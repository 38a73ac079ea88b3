// Flow1D's 1D attention and 1D correlation (flow1d/attention.py, correlation.py) and the per-iteration 1D lookup of its two
// volumes.  A "sequence" is one row (axis 0, length W) or one column (axis 1, length H) of a pixel-major [B,H,W,C] map; every
// operand is read straight from the map with the sequence's pixel step, so column sequences need no transpose.
//
// pfb_attn1d, two implementations of one contract:
//   mode 1 (correlation): out[query pixel * L + key] = scale * q . k in the storage type;
//   mode 2 (attention):   out[query pixel] = softmax(scale * q . K^T) V, the softmax in fp32, P rounded to the storage type
//                         before P V (the reference half model's softmax output is half), fp32 accumulation.  The L x L scores
//                         stay on chip.  Padded keys get a logit of -inf, so they weigh exactly zero.
// * wgmma (f16 / bf16, C in {64, 128, 256}, 16-byte aligned pointers and pixel strides): one warpgroup per CTA = 64 queries of
//   one sequence.  TMA tensor maps over [B][H][W][C] whose second dimension steps along the sequence's axis load the query
//   tile once and each 64-key tile of K and V (pixels past the sequence zero-filled); S = Q K^T on wgmma (both operands
//   K-major), the online softmax on the accumulator fragments, P rounded into shared memory, V transposed in shared memory
//   into a K-major [C][64 keys] operand, O += P V^T on wgmma (N = C).  The next tile's K / V loads overlap P V.
// * SIMT (fp32, impl = 1, and the shapes above that wgmma does not take): one CTA = 32 queries; keys in tiles of 32, operands
//   converted to fp32 in shared memory; each warp owns 4 queries, lane j computes the 4 logits of key j, then the online
//   softmax and P V with lane j holding channels j, j+32, ...
// pfb_corr1d_lookup: one warp per query stages the 2r+2 values of each row window that the 2r+1 taps read (each loaded
// once), then lane j writes output channels j, j+32, ... from them.
#include <math.h>

#include <type_traits>

#include "umma.cuh"

namespace pfb {

constexpr int A1_TQ = 32;       // queries per CTA (8 warps x 4)
constexpr int A1_TK = 32;       // keys per tile (one per lane)
constexpr int A1_QPW = 4;       // queries per warp
constexpr int A1_THREADS = 256;
constexpr int A1_MAX_NJ = 8;    // C / 32 channels per lane in P V (C <= 256)

// pixel index of element l of sequence `seq`: rows (axis 0) are contiguous, columns step by W
struct SeqAddr {
  size_t base, step;
  __device__ SeqAddr(int seq, int axis, int H, int W) {
    if (axis == 0) { base = (size_t)seq * W; step = 1; }
    else { const int b = seq / W, x = seq - b * W; base = (size_t)b * H * W + x; step = W; }
  }
  __device__ size_t operator()(int l) const { return base + (size_t)l * step; }
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T>
__device__ __forceinline__ void load_tile(float* dst, int dst_stride, const T* __restrict__ src, int src_stride, const SeqAddr& at,
                                          int l0, int rows, int L, int C) {
  for (int i = threadIdx.x; i < rows * C; i += A1_THREADS) {
    const int r = i / C, c = i - r * C, l = l0 + r;
    dst[r * dst_stride + c] = l < L ? to_f32(src[at(l) * src_stride + c]) : 0.f;
  }
}

template <typename T, bool ATTN>
__global__ void __launch_bounds__(A1_THREADS, 2)
attn1d_kernel(const T* __restrict__ q, int q_stride, const T* __restrict__ k, int k_stride, const T* __restrict__ v, int v_stride,
              T* __restrict__ out, int out_stride, int H, int W, int C, int axis, float scale) {
  extern __shared__ __align__(16) float a1_smem[];
  const int L = axis == 0 ? W : H;
  const SeqAddr at(blockIdx.x, axis, H, W);
  const int q0 = blockIdx.y * A1_TQ;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int nj = C >> 5;
  float* Qs = a1_smem;                  // [TQ][C]
  float* Ks = Qs + A1_TQ * C;           // [TK][C + 1]: lane j reads row j, conflict-free
  float* Vs = Ks + A1_TK * (C + 1);     // [TK][C]           (attention)
  float* Ps = Vs + A1_TK * C;           // [8 warps][QPW][TK] (attention)

  load_tile(Qs, C, q, q_stride, at, q0, A1_TQ, L, C);

  float m[A1_QPW], den[A1_QPW], o[A1_QPW][A1_MAX_NJ];
#pragma unroll
  for (int i = 0; i < A1_QPW; ++i) {
    m[i] = -INFINITY;
    den[i] = 0.f;
#pragma unroll
    for (int j = 0; j < A1_MAX_NJ; ++j) o[i][j] = 0.f;
  }

  for (int k0 = 0; k0 < L; k0 += A1_TK) {
    __syncthreads();  // the previous tile is consumed (and, first time round, Qs is complete after the next barrier)
    load_tile(Ks, C + 1, k, k_stride, at, k0, A1_TK, L, C);
    if (ATTN) load_tile(Vs, C, v, v_stride, at, k0, A1_TK, L, C);
    __syncthreads();

    float s[A1_QPW] = {0.f, 0.f, 0.f, 0.f};
    const float* kr = Ks + lane * (C + 1);
    for (int c = 0; c < C; c += 4) {
      const float k_0 = kr[c], k_1 = kr[c + 1], k_2 = kr[c + 2], k_3 = kr[c + 3];
#pragma unroll
      for (int i = 0; i < A1_QPW; ++i) {
        const float4 qv = *reinterpret_cast<const float4*>(Qs + (warp * A1_QPW + i) * C + c);
        s[i] = fmaf(qv.x, k_0, fmaf(qv.y, k_1, fmaf(qv.z, k_2, fmaf(qv.w, k_3, s[i]))));
      }
    }
    const int key = k0 + lane;
    const bool key_ok = key < L;

    if (!ATTN) {
#pragma unroll
      for (int i = 0; i < A1_QPW; ++i) {
        const int qi = q0 + warp * A1_QPW + i;
        if (qi < L && key_ok) out[at(qi) * (size_t)L + key] = from_f32<T>(s[i] * scale);
      }
      continue;
    }

    float* pw = Ps + warp * A1_QPW * A1_TK;
#pragma unroll
    for (int i = 0; i < A1_QPW; ++i) {
      const float logit = key_ok ? s[i] * scale : -INFINITY;  // k0 < L: every tile holds at least one real key
      const float m_new = fmaxf(m[i], warp_max(logit));
      const float rescale = __expf(m[i] - m_new);             // exp(-inf) = 0 on the first tile
      const float p = key_ok ? __expf(logit - m_new) : 0.f;
      den[i] = den[i] * rescale + warp_sum(p);
      m[i] = m_new;
      pw[i * A1_TK + lane] = to_f32(from_f32<T>(p));
#pragma unroll
      for (int j = 0; j < A1_MAX_NJ; ++j) o[i][j] *= rescale;
    }
    __syncwarp();
    const int nk = min(A1_TK, L - k0);
    for (int kk = 0; kk < nk; ++kk) {
      float p[A1_QPW];
#pragma unroll
      for (int i = 0; i < A1_QPW; ++i) p[i] = pw[i * A1_TK + kk];
      const float* vr = Vs + kk * C + lane;
#pragma unroll
      for (int j = 0; j < A1_MAX_NJ; ++j) {
        if (j < nj) {
          const float vv = vr[j * 32];
#pragma unroll
          for (int i = 0; i < A1_QPW; ++i) o[i][j] = fmaf(p[i], vv, o[i][j]);
        }
      }
    }
    __syncwarp();
  }

  if (ATTN) {
#pragma unroll
    for (int i = 0; i < A1_QPW; ++i) {
      const int qi = q0 + warp * A1_QPW + i;
      if (qi >= L) continue;
      const float inv = 1.f / den[i];
      T* dst = out + at(qi) * out_stride + lane;
#pragma unroll
      for (int j = 0; j < A1_MAX_NJ; ++j)
        if (j < nj) dst[j * 32] = from_f32<T>(o[i][j] * inv);
    }
  }
}

// ---------------------------------------------------------------- wgmma path
constexpr int AT_Q = 64, AT_K = 64, AT_THREADS = 128;
constexpr int AT_TILE = 64 * 128;  // 64 rows x 64 halves, 128-byte swizzle

// byte offset of element (row, col) of a K-major 128-byte-swizzled tile of 64-element rows (TMA's SWIZZLE_128B pattern)
__device__ __forceinline__ uint32_t sw128(int row, int col) {
  return row * 128 + ((((col >> 3) ^ (row & 7)) & 7) << 4) + ((col & 7) << 1);
}

struct __align__(8) AttnBars {  // must fit the 1024-byte header of the shared-memory carve
  uint64_t q_full, kv_full;
};

template <typename T, int C, bool ATTN>
__global__ void __launch_bounds__(AT_THREADS, 1)
attn1d_umma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK, const __grid_constant__ CUtensorMap tmV,
                   T* __restrict__ out, int out_stride, int H, int W, int axis, float scale) {
  using namespace sm90;
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int KC = C / 64;  // 64-channel chunks
  extern __shared__ __align__(1024) uint8_t at_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(at_smem_raw) + 1023) & ~uintptr_t(1023));
  AttnBars* bars = reinterpret_cast<AttnBars*>(smem);  // the first 1024 bytes; the tiles stay 1024-byte aligned after it
  uint8_t* sQ = smem + 1024;                // KC tiles [64 queries][64 ch]
  uint8_t* sK = sQ + KC * AT_TILE;          // KC tiles [64 keys][64 ch]
  uint8_t* sV = sK + KC * AT_TILE;          // KC tiles [64 keys][64 ch]        (attention)
  uint8_t* sVt = sV + KC * AT_TILE;         // [C][64 keys], one K-major tile   (attention)
  uint8_t* sP = sVt + C * 128;              // [64 queries][64 keys]            (attention)

  const int L = axis == 0 ? W : H;
  const int seq = blockIdx.x, q0 = blockIdx.y * AT_Q;
  const int other = axis == 0 ? H : W;   // the sequence's index in the dimension across the axis
  const int b = seq / other, o = seq - b * other;
  const SeqAddr at(seq, axis, H, W);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t kv_bytes = (ATTN ? 2 : 1) * KC * AT_TILE;

  if (tid == 0) {
    mbar_init(&bars->q_full, 1);
    mbar_init(&bars->kv_full, 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_kv = [&](int k0) {
    mbar_arrive_expect_tx(&bars->kv_full, kv_bytes);
    for (int k = 0; k < KC; ++k) {
      tma_load_4d(sK + k * AT_TILE, &tmK, &bars->kv_full, k * 64, k0, o, b);
      if (ATTN) tma_load_4d(sV + k * AT_TILE, &tmV, &bars->kv_full, k * 64, k0, o, b);
    }
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars->q_full, KC * AT_TILE);
    for (int k = 0; k < KC; ++k) tma_load_4d(sQ + k * AT_TILE, &tmQ, &bars->q_full, k * 64, q0, o, b);
    load_kv(0);
  }
  mbar_wait(&bars->q_full, 0);

  // fragment rows of this thread: r0 and r0 + 8; columns 8 j + 2 (tid & 3) + {0, 1}
  const int r0 = 16 * warp + (lane >> 2);
  float m[2] = {-INFINITY, -INFINITY}, den[2] = {0.f, 0.f};
  float acc[C / 2];  // O (attention; the correlation instances drop it)
#pragma unroll
  for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;

  int phase = 0;
  for (int k0 = 0; k0 < L; k0 += AT_K, phase ^= 1) {
    mbar_wait(&bars->kv_full, phase);
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < KC; ++k) {
      const uint32_t al = gdesc_lo(smem_u32(sQ + k * AT_TILE), 16), bl = gdesc_lo(smem_u32(sK + k * AT_TILE), 16);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma<64, BF16>(sc, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), (k == 0 && kk == 0) ? 0u : 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sc);

    if (!ATTN) {
#pragma unroll
      for (int e = 0; e < 32; e += 2) {
        const int row = r0 + 8 * ((e >> 1) & 1), col = 8 * (e >> 2) + 2 * (lane & 3);
        const int qi = q0 + row, key = k0 + col;
        if (qi < L) {
          T* dst = out + at(qi) * (size_t)L + key;
          if (key + 1 < L && (((size_t)at(qi) * L + key) & 1) == 0) {
            using T2 = typename std::conditional<BF16, __nv_bfloat162, __half2>::type;
            T2 v2;
            v2.x = from_f32<T>(sc[e] * scale);
            v2.y = from_f32<T>(sc[e + 1] * scale);
            *reinterpret_cast<T2*>(dst) = v2;
          } else {
            if (key < L) dst[0] = from_f32<T>(sc[e] * scale);
            if (key + 1 < L) dst[1] = from_f32<T>(sc[e + 1] * scale);
          }
        }
      }
      __syncthreads();  // every thread's wgmma has read sK before the next tile overwrites it
      if (tid == 0 && k0 + AT_K < L) load_kv(k0 + AT_K);
      continue;
    }

    // online softmax over this tile's 64 keys, rows r0 / r0 + 8 (the 4 lanes of a quad share a row)
    float rescale[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        if (((e >> 1) & 1) != h) continue;
        const int key = k0 + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1);
        sc[e] = key < L ? sc[e] * scale : -INFINITY;
        mx = fmaxf(mx, sc[e]);
      }
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m[h], mx);  // finite: k0 < L, so every tile holds a real key
      rescale[h] = __expf(m[h] - m_new);
      m[h] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int e = 0; e < 32; ++e) {
        if (((e >> 1) & 1) != h) continue;
        sc[e] = __expf(sc[e] - m_new);  // exp(-inf) = 0 for padded keys
        sum += sc[e];
      }
      den[h] = den[h] * rescale[h] + sum;  // this thread's share of the row; the quad is summed at the end
    }
    // P (rounded to the storage type) into its K-major tile
#pragma unroll
    for (int e = 0; e < 32; e += 2) {
      const int row = r0 + 8 * ((e >> 1) & 1), col = 8 * (e >> 2) + 2 * (lane & 3);
      T p2[2] = {from_f32<T>(sc[e]), from_f32<T>(sc[e + 1])};
      *reinterpret_cast<uint32_t*>(sP + sw128(row, col)) = *reinterpret_cast<uint32_t*>(p2);
    }
    // V^T: row c of sVt holds the 64 keys of channel c (16 bytes = 8 keys per store)
    for (int i = tid; i < C * 8; i += AT_THREADS) {
      const int c = i >> 3, j = i & 7, kc = c >> 6, cc = c & 63;
      const uint8_t* src = sV + kc * AT_TILE;
      T v8[8];
#pragma unroll
      for (int t = 0; t < 8; ++t) v8[t] = *reinterpret_cast<const T*>(src + sw128(8 * j + t, cc));
      *reinterpret_cast<uint4*>(sVt + sw128(c, 8 * j)) = *reinterpret_cast<uint4*>(v8);
    }
#pragma unroll
    for (int i = 0; i < C / 2; ++i) acc[i] *= rescale[(i >> 1) & 1];
    fence_proxy_async();  // the generic-proxy writes of sP / sVt become visible to wgmma
    __syncthreads();      // ... from every thread; sK and sV are consumed, so the next tile may land there
    if (tid == 0 && k0 + AT_K < L) load_kv(k0 + AT_K);
    wgmma_fence();
    {
      const uint32_t al = gdesc_lo(smem_u32(sP), 16), bl = gdesc_lo(smem_u32(sVt), 16);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) wgmma<C, BF16>(acc, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(acc);
    __syncthreads();  // sP / sVt are read before the next tile rewrites them
  }

  if (ATTN) {
    float inv[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float d = den[h];
      d += __shfl_xor_sync(0xffffffffu, d, 1);
      d += __shfl_xor_sync(0xffffffffu, d, 2);
      inv[h] = 1.f / d;
    }
    using T2 = typename std::conditional<BF16, __nv_bfloat162, __half2>::type;
#pragma unroll
    for (int e = 0; e < C / 2; e += 2) {
      const int h = (e >> 1) & 1, row = r0 + 8 * h, col = 8 * (e >> 2) + 2 * (lane & 3);
      const int qi = q0 + row;
      if (qi >= L) continue;
      T2 v2;
      v2.x = from_f32<T>(acc[e] * inv[h]);
      v2.y = from_f32<T>(acc[e + 1] * inv[h]);
      *reinterpret_cast<T2*>(out + at(qi) * out_stride + col) = v2;
    }
  }
}

static size_t attn1d_umma_smem(int C, bool attn) {
  const size_t kc = C / 64;
  // alignment slack, the barrier header, then Q and K (and V, V^T, P) -- the kernel's carve
  return 1024 + 1024 + (attn ? 3 * kc * AT_TILE + (size_t)C * 128 + AT_TILE : 2 * kc * AT_TILE);
}

// the tensor map of a [B,H,W,*] map with pixel stride ps (elements) whose dimension 1 runs along the sequence axis
static int attn1d_tmap(CUtensorMap* m, const void* base, int ps, int B, int H, int W, int C, int axis, pfb_dtype dt) {
  const uint64_t px = (uint64_t)ps * 2, row = (uint64_t)W * px, img = (uint64_t)H * row;
  const uint64_t dims[4] = {(uint64_t)C, (uint64_t)(axis == 0 ? W : H), (uint64_t)(axis == 0 ? H : W), (uint64_t)B};
  const uint64_t str[3] = {axis == 0 ? px : row, axis == 0 ? row : px, img};
  const uint32_t box[4] = {64, (uint32_t)AT_K, 1, 1};
  return make_tensor_map(m, base, dt, 4, dims, str, box);
}

static bool attn1d_umma_supported(const void* q, int qs, const void* k, int ks, const void* v, int vs, const void* out, int os, int C,
                                  bool attn, pfb_dtype dt) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (dt == PFB_F32 || !(C == 64 || C == 128 || C == 256)) return false;
  if (!al16(q) || !al16(k) || qs % 8 || ks % 8) return false;
  if (attn && (!al16(v) || vs % 8 || !al16(out) || os % 2)) return false;
  return true;
}

template <typename T, int C, bool ATTN>
static int launch_attn1d_umma(const void* q, int qs, const void* k, int ks, const void* v, int vs, void* out, int os, int B, int H, int W,
                              int axis, float scale, pfb_dtype dt, cudaStream_t s) {
  CUtensorMap tq, tk, tv;
  PFB_TRY(attn1d_tmap(&tq, q, qs, B, H, W, C, axis, dt));
  PFB_TRY(attn1d_tmap(&tk, k, ks, B, H, W, C, axis, dt));
  if (ATTN) PFB_TRY(attn1d_tmap(&tv, v, vs, B, H, W, C, axis, dt));
  else tv = tk;
  const int L = axis == 0 ? W : H, seqs = axis == 0 ? B * H : B * W;
  const size_t smem = attn1d_umma_smem(C, ATTN);
  auto kern = attn1d_umma_kernel<T, C, ATTN>;
  PFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfScope prof(KC_ATTN1D, s);
  kern<<<dim3(seqs, ceil_div(L, AT_Q)), AT_THREADS, smem, s>>>(tq, tk, tv, reinterpret_cast<T*>(out), os, H, W, axis, scale);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

template <typename T>
static int dispatch_attn1d_umma(const void* q, int qs, const void* k, int ks, const void* v, int vs, void* out, int os, int B, int H,
                                int W, int C, int axis, bool attn, float scale, pfb_dtype dt, cudaStream_t s) {
#define PFB_AT_CASE(CC)                                                                                                  \
  if (C == CC) {                                                                                                         \
    if (attn) return launch_attn1d_umma<T, CC, true>(q, qs, k, ks, v, vs, out, os, B, H, W, axis, scale, dt, s);         \
    return launch_attn1d_umma<T, CC, false>(q, qs, k, ks, v, vs, out, os, B, H, W, axis, scale, dt, s);                   \
  }
  PFB_AT_CASE(64)
  PFB_AT_CASE(128)
  PFB_AT_CASE(256)
#undef PFB_AT_CASE
  return PFB_ERR_ARG;
}

static size_t attn1d_smem(int C, bool attn) {
  size_t f = (size_t)A1_TQ * C + (size_t)A1_TK * (C + 1);
  if (attn) f += (size_t)A1_TK * C + (size_t)(A1_THREADS / 32) * A1_QPW * A1_TK;
  return f * sizeof(float);
}

template <typename T, bool ATTN>
static int launch_attn1d(const void* q, int qs, const void* k, int ks, const void* v, int vs, void* out, int os, int B, int H, int W,
                         int C, int axis, float scale, cudaStream_t s) {
  const int L = axis == 0 ? W : H;
  const int seqs = axis == 0 ? B * H : B * W;
  const size_t smem = attn1d_smem(C, ATTN);
  auto kern = attn1d_kernel<T, ATTN>;
  PFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  ProfScope prof(KC_ATTN1D, s);
  kern<<<dim3(seqs, ceil_div(L, A1_TQ)), A1_THREADS, smem, s>>>(
      reinterpret_cast<const T*>(q), qs, reinterpret_cast<const T*>(k), ks, reinterpret_cast<const T*>(v), vs, reinterpret_cast<T*>(out),
      os, H, W, C, axis, scale);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

constexpr int LK_WARPS = 8;
constexpr int LK_WIN = 2 * 64 + 2;  // 2r + 2 values per row window at r = 64

// one warp per query: stage the 2r+2 values row[floor(c) - r .. floor(c) + r + 1] of each volume (zero outside the row; each value
// loaded once), then lane j writes output channels j, j + 32, ...: tap d reads window entries d + r and d + r + 1
template <typename T>
__global__ void __launch_bounds__(LK_WARPS * 32)
corr1d_lookup_kernel(const T* __restrict__ corr_x, const T* __restrict__ corr_y, const float* __restrict__ coords, T* __restrict__ out,
                     size_t P, int H, int W, int r, int out_stride) {
  __shared__ float win[LK_WARPS][2][LK_WIN];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const size_t qp = (size_t)blockIdx.x * LK_WARPS + warp;
  if (qp >= P) return;
  const int K = 2 * r + 1;
  float frac[2];
#pragma unroll
  for (int a = 0; a < 2; ++a) {
    const int L = a == 0 ? W : H;
    const T* row = (a == 0 ? corr_x : corr_y) + qp * L;
    const float c = coords[2 * qp + a];
    const float f = floorf(c);
    // a window that cannot reach the row (this also keeps huge coordinates away from the int conversion; NaN fails both tests)
    const bool reach = f >= -(float)(r + 1) && f <= (float)(L + r);
    const int x0 = reach ? (int)f - r : 0;
    frac[a] = reach ? c - f : 0.f;
    for (int i = lane; i < K + 1; i += 32) {
      const int x = x0 + i;
      win[warp][a][i] = reach && x >= 0 && x < L ? to_f32(row[x]) : 0.f;
    }
  }
  __syncwarp();
  T* dst = out + qp * out_stride;
  for (int j = lane; j < out_stride; j += 32) {
    float val = 0.f;
    if (j < 2 * K) {
      const int a = j < K ? 0 : 1, d = j - a * K;
      val = (1.f - frac[a]) * win[warp][a][d] + frac[a] * win[warp][a][d + 1];
    }
    dst[j] = from_f32<T>(val);
  }
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_attn1d(const void* q, int q_stride, const void* k, int k_stride, const void* v, int v_stride, void* out,
                                  int out_stride, int B, int H, int W, int C, int axis, int mode, float scale, pfb_dtype dtype, int impl,
                                  pfb_stream stream) {
  PFB_CHECK_ARG(dtype_ok(dtype), "attn1d: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(mode == PFB_ATTN1D_CORR || mode == PFB_ATTN1D_ATTN, "attn1d: mode=%d (1 correlation, 2 attention)", mode);
  PFB_CHECK_ARG(axis == 0 || axis == 1, "attn1d: axis=%d (0 rows, 1 columns)", axis);
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0, "attn1d: bad grid %dx%dx%d", B, H, W);
  PFB_CHECK_ARG(C >= 64 && C <= 256 && C % 64 == 0, "attn1d: C=%d (a multiple of 64, at most 256)", C);
  const int L = axis == 0 ? W : H;
  PFB_CHECK_ARG(L >= 1 && L <= PFB_ATTN1D_MAX_L, "attn1d: sequence length %d outside 1..%d", L, PFB_ATTN1D_MAX_L);
  PFB_CHECK_ARG((long long)B * (axis == 0 ? H : W) <= 0x7fffffffLL, "attn1d: too many sequences");
  PFB_CHECK_ARG(q && k && out && q_stride >= C && k_stride >= C, "attn1d: null operand or pixel stride < C");
  const bool attn = mode == PFB_ATTN1D_ATTN;
  if (attn) PFB_CHECK_ARG(v && v_stride >= C && out_stride >= C, "attn1d: attention needs v and pixel strides >= C");
  PFB_CHECK_ARG(impl >= 0 && impl <= 2, "attn1d: impl=%d (0 auto, 1 SIMT, 2 wgmma)", impl);
  const cudaStream_t s = as_stream(stream);
  const bool tc = attn1d_umma_supported(q, q_stride, k, k_stride, v, v_stride, out, out_stride, C, attn, dtype);
  PFB_CHECK_ARG(impl != 2 || tc, "attn1d: the wgmma path needs f16 / bf16, C in {64, 128, 256}, 16-byte aligned operands and pixel "
                "strides that are multiples of 8 elements");
  if (tc && impl != 1) {
    if (dtype == PFB_F16) return dispatch_attn1d_umma<__half>(q, q_stride, k, k_stride, v, v_stride, out, out_stride, B, H, W, C, axis,
                                                              attn, scale, dtype, s);
    return dispatch_attn1d_umma<__nv_bfloat16>(q, q_stride, k, k_stride, v, v_stride, out, out_stride, B, H, W, C, axis, attn, scale,
                                               dtype, s);
  }
  PFB_DISPATCH_DTYPE(dtype, T, {
    if (attn) return launch_attn1d<T, true>(q, q_stride, k, k_stride, v, v_stride, out, out_stride, B, H, W, C, axis, scale, s);
    return launch_attn1d<T, false>(q, q_stride, k, k_stride, v, v_stride, out, out_stride, B, H, W, C, axis, scale, s);
  });
  return PFB_OK;
}

extern "C" PFB_API int pfb_corr1d_lookup(const void* corr_x, const void* corr_y, const float* coords, void* out, int B, int H, int W,
                                         int radius, pfb_dtype dtype, int out_stride, pfb_stream stream) {
  PFB_CHECK_ARG(dtype_ok(dtype), "corr1d_lookup: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(corr_x && corr_y && coords && out, "corr1d_lookup: null pointer");
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0, "corr1d_lookup: bad grid %dx%dx%d", B, H, W);
  PFB_CHECK_ARG(radius >= 1 && radius <= 64, "corr1d_lookup: radius=%d (1..64)", radius);
  PFB_CHECK_ARG(out_stride >= 2 * (2 * radius + 1), "corr1d_lookup: out_stride %d < %d", out_stride, 2 * (2 * radius + 1));
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_LOOKUP, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    corr1d_lookup_kernel<T><<<(unsigned)ceil_div_sz(P, LK_WARPS), LK_WARPS * 32, 0, s>>>(reinterpret_cast<const T*>(corr_x),
                                                                       reinterpret_cast<const T*>(corr_y), coords,
                                                                       reinterpret_cast<T*>(out), P, H, W, radius, out_stride);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
