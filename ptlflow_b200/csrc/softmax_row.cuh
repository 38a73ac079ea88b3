// One attention row softmax held in shared memory: one CTA of kRowThreads per row, the row read once with 16-byte loads, its
// adjusted logits kept in shared memory between the max, exp-sum and normalise passes, and written once.  Shared by GMA's
// relative-position softmax (misc.cu) and CRAFT's windowed-bias softmax (craft.cu), which differ only in the term added to a logit.
#pragma once

#include "common.cuh"

namespace pfb {

constexpr int kRowThreads = 256;

template <bool MAX>
__device__ __forceinline__ float row_block_reduce(float v, float* red) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = MAX ? fmaxf(v, w) : v + w;
  }
  if (lane == 0) red[warp] = v;
  __syncthreads();
  v = red[0];
  for (int i = 1; i < kRowThreads / 32; ++i) v = MAX ? fmaxf(v, red[i]) : v + red[i];
  __syncthreads();
  return v;
}

// arow[j] = softmax_j(term(lrow[j] or 0, u, v)) over the N = H*W keys j = u*W + v, fp32 math.  srow: N floats of shared memory
// (16-byte aligned); red: kRowThreads / 32 floats.  VEC: N a multiple of 16 bytes of T and both rows 16-byte aligned.
template <typename T, bool VEC, typename Term>
__device__ __forceinline__ void softmax_row_smem(const T* lrow, T* arow, int N, int W, float* srow, float* red, Term term) {
  constexpr int EV = VEC ? 16 / (int)sizeof(T) : 1;
  const int nvec = N / EV;
  float m = -INFINITY;
  for (int c = threadIdx.x; c < nvec; c += kRowThreads) {
    const int j0 = c * EV;
    float f[EV];
    if (lrow) {
      if constexpr (VEC) {
        const uint4 raw = *reinterpret_cast<const uint4*>(lrow + j0);
        const T* e = reinterpret_cast<const T*>(&raw);
#pragma unroll
        for (int k = 0; k < EV; ++k) f[k] = to_f32(e[k]);
      } else {
        f[0] = to_f32(lrow[j0]);
      }
    } else {
#pragma unroll
      for (int k = 0; k < EV; ++k) f[k] = 0.f;
    }
    int u = j0 / W, v = j0 - u * W;
#pragma unroll
    for (int k = 0; k < EV; ++k) {
      f[k] = term(f[k], u, v);
      m = fmaxf(m, f[k]);
      if (++v == W) { v = 0; ++u; }
    }
#pragma unroll
    for (int k = 0; k < EV; k += 4 > EV ? EV : 4) {
      if constexpr (EV >= 4) *reinterpret_cast<float4*>(srow + j0 + k) = make_float4(f[k], f[k + 1], f[k + 2], f[k + 3]);
      else srow[j0 + k] = f[k];
    }
  }
  m = row_block_reduce<true>(m, red);

  float sum = 0.f;  // every thread revisits the entries it wrote: no barrier needed before this pass
  for (int c = threadIdx.x; c < nvec; c += kRowThreads) {
    const int j0 = c * EV;
#pragma unroll
    for (int k = 0; k < EV; ++k) {
      const float e = __expf(srow[j0 + k] - m);
      srow[j0 + k] = e;
      sum += e;
    }
  }
  sum = row_block_reduce<false>(sum, red);
  const float inv = 1.f / sum;

  for (int c = threadIdx.x; c < nvec; c += kRowThreads) {
    const int j0 = c * EV;
    if constexpr (VEC) {
      uint4 raw;
      T* e = reinterpret_cast<T*>(&raw);
#pragma unroll
      for (int k = 0; k < EV; ++k) e[k] = from_f32<T>(srow[j0 + k] * inv);
      *reinterpret_cast<uint4*>(arow + j0) = raw;
    } else {
      arow[j0] = from_f32<T>(srow[j0] * inv);
    }
  }
}

}  // namespace pfb
