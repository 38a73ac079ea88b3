// a22: LLA-Flow (ptlflow/models/llaflow/llaflow.py:140-217, aggregate.py, corr.py): local 5 x 5 similarity attention on the context
// features, the local aggregation of fmap2 (LSA), and the shift-aggregated term gamma corr2 of the correlation volume (ShiftLSA).
//
// With delta_l = (l / 5 - 2, l % 5 - 2) (dy, dx), l = 0..24, and clamp() replicate padding (PatchExtra / ImgShift):
//   a[n, l]  = softmax_l(<q[n], k[clamp(n + delta_l)]> / sqrt(128))                                     pfb_local_similar
//   fmap2'   = fmap2 + lsa_gamma sum_l a2[n, l] v[clamp(n + delta_l)]                                    pfb_local_aggregate
//   volume   = <fmap1[n], fmap2'[m]> / 16 + gamma sum_l a1[n, l] <f1'[clamp(n + delta_l)], f2''[clamp(m + delta_l)]> / 16
// The volume is ONE GEMM of K = 26 x 256 = 6656 (pfb_shift_pack writes its operands):
//   A'[n] = [fmap1[n] / 16 | gamma a1[n, l] f1'[clamp(n + delta_l)] / 16 for l = 0..24]
//   B'[m] = [fmap2'[m]     | f2''[clamp(m + delta_l)]                    for l = 0..24]
// B' is never needed in full on the tensor-core path: [fmap2' | f2''] stored replicate-padded by 2 pixels ([B, H+4, W+4, 512])
// turns clamp(m + delta_l) into a plain offset, so every B tile is the 16 x 8 target box of corr_volume_tiled_kernel moved by
// (2 + dx, 2 + dy) (pfb_shift_volume_tiled).
#include "corr_umma.cuh"

namespace pfb {

constexpr int kLlaC = 256;              // feature channels (fmap1, fmap2, f1', f2'')
constexpr int kLlaD = 128;              // query / key channels of LocalSimilar
constexpr int kLlaTaps = 25;            // 5 x 5
constexpr int kLlaK = (kLlaTaps + 1) * kLlaC;  // 6656

__device__ __forceinline__ int clampi(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

__device__ __forceinline__ float lla_warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float lla_warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- pfb_local_similar: one warp per (pixel, table); lane j holds channels 4j .. 4j+3 of q, lane l < 25 ends with logit l ----
constexpr int kLsWarps = 8;

template <typename T>
__global__ void __launch_bounds__(kLsWarps * 32)
local_similar_kernel(const T* __restrict__ qk, float* __restrict__ a1, float* __restrict__ a2, int B, int H, int W, float scale) {
  const int lane = threadIdx.x & 31;
  const size_t g = (size_t)blockIdx.x * kLsWarps + (threadIdx.x >> 5);
  const size_t P = (size_t)B * H * W;
  if (g >= 2 * P) return;
  const size_t p = g >> 1;
  const int t = (int)(g & 1);  // table: 0 = ls1 (channels 0..255 of qk), 1 = ls2 (256..511)
  const int x = (int)(p % W), y = (int)((p / W) % H);
  const size_t b0 = p - ((size_t)y * W + x);  // first pixel of the sample
  const T* qp = qk + p * (4 * kLlaD) + t * (2 * kLlaD) + 4 * lane;
  float q[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) q[j] = to_f32(qp[j]);
  float mine = -INFINITY;
#pragma unroll 5
  for (int l = 0; l < kLlaTaps; ++l) {
    const int yy = clampi(y + l / 5 - 2, H - 1), xx = clampi(x + l % 5 - 2, W - 1);
    const T* kp = qk + (b0 + (size_t)yy * W + xx) * (4 * kLlaD) + t * (2 * kLlaD) + kLlaD + 4 * lane;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) s += q[j] * to_f32(kp[j]);
    s = lla_warp_sum(s);
    if (lane == l) mine = s * scale;
  }
  const float m = lla_warp_max(mine);
  const float e = lane < kLlaTaps ? expf(mine - m) : 0.f;
  const float sum = lla_warp_sum(e);
  if (lane < kLlaTaps) (t ? a2 : a1)[p * kLlaTaps + lane] = e / sum;
}

// ---- pfb_local_aggregate: one thread per output element ----
template <typename T>
__global__ void __launch_bounds__(256)
local_aggregate_kernel(const T* __restrict__ fmap2, const T* __restrict__ v, const float* __restrict__ a2, float gamma, T* __restrict__ out,
                       int B, int H, int W) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * H * W * kLlaC) return;
  const int c = (int)(i % kLlaC);
  const size_t p = i / kLlaC;
  const int x = (int)(p % W), y = (int)((p / W) % H);
  const size_t b0 = p - ((size_t)y * W + x);
  const float* a = a2 + p * kLlaTaps;
  float s = 0.f;
#pragma unroll 5
  for (int l = 0; l < kLlaTaps; ++l) {
    const int yy = clampi(y + l / 5 - 2, H - 1), xx = clampi(x + l % 5 - 2, W - 1);
    s += a[l] * to_f32(v[(b0 + (size_t)yy * W + xx) * kLlaC + c]);
  }
  out[i] = from_f32<T>(to_f32(fmap2[i]) + gamma * s);
}

// ---- pfb_shift_pack: the GEMM operands, one thread per output element ----
template <typename T>
__global__ void __launch_bounds__(256)
shift_pack_a_kernel(const T* __restrict__ fmap1, const T* __restrict__ f1, const float* __restrict__ a1, float gamma, T* __restrict__ A,
                    int B, int H, int W) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * H * W * kLlaK) return;
  const int k = (int)(i % kLlaK), seg = k / kLlaC, c = k - seg * kLlaC;
  const size_t p = i / kLlaK;
  float v;
  if (seg == 0) {
    v = to_f32(fmap1[p * kLlaC + c]) * 0.0625f;
  } else {
    const int l = seg - 1;
    const int x = (int)(p % W), y = (int)((p / W) % H);
    const size_t b0 = p - ((size_t)y * W + x);
    const int yy = clampi(y + l / 5 - 2, H - 1), xx = clampi(x + l % 5 - 2, W - 1);
    v = gamma * a1[p * kLlaTaps + l] * to_f32(f1[(b0 + (size_t)yy * W + xx) * kLlaC + c]) * 0.0625f;
  }
  A[i] = from_f32<T>(v);
}

// [fmap2' | f2''] replicate-padded by 2 pixels: [B, H+4, W+4, 512]
template <typename T>
__global__ void __launch_bounds__(256)
shift_pack_bpad_kernel(const T* __restrict__ fmap2, const T* __restrict__ f2, T* __restrict__ Bp, int B, int H, int W) {
  const int Hp = H + 4, Wp = W + 4;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * Hp * Wp * 2 * kLlaC) return;
  const int k = (int)(i % (2 * kLlaC));
  const size_t pp = i / (2 * kLlaC);
  const int xp = (int)(pp % Wp), yp = (int)((pp / Wp) % Hp), b = (int)(pp / ((size_t)Wp * Hp));
  const size_t src = ((size_t)b * H + clampi(yp - 2, H - 1)) * W + clampi(xp - 2, W - 1);
  Bp[i] = k < kLlaC ? fmap2[src * kLlaC + k] : f2[src * kLlaC + k - kLlaC];
}

// B' materialised: [B*H*W, 6656]
template <typename T>
__global__ void __launch_bounds__(256)
shift_pack_bmat_kernel(const T* __restrict__ fmap2, const T* __restrict__ f2, T* __restrict__ Bm, int B, int H, int W) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * H * W * kLlaK) return;
  const int k = (int)(i % kLlaK), seg = k / kLlaC, c = k - seg * kLlaC;
  const size_t p = i / kLlaK;
  if (seg == 0) {
    Bm[i] = fmap2[p * kLlaC + c];
  } else {
    const int l = seg - 1;
    const int x = (int)(p % W), y = (int)((p / W) % H);
    const size_t b0 = p - ((size_t)y * W + x);
    const int yy = clampi(y + l / 5 - 2, H - 1), xx = clampi(x + l % 5 - 2, W - 1);
    Bm[i] = f2[(b0 + (size_t)yy * W + xx) * kLlaC + c];
  }
}

// ---- pfb_shift_volume_tiled: the K = 6656 GEMM on wgmma, written as the tiled pyramid ----
//
// CTA = 13 warps as corr_volume_tiled_kernel: 0-3 epilogue (thread = query row), 4-11 two MMA warpgroups (64 query rows each),
// 12 TMA producer.  One work item per CTA: 128 queries x one 16 x 8 target patch, K streamed in 104 chunks of 64 channels, each
// chunk's A' tile (3D map over [B][N][6656]) and shifted B box (4D map over the padded [B][H+4][W+4][512]) arriving together in
// a 3-stage mbarrier ring of 32 KB stages.  The MMA warpgroups keep one chunk's wgmma group in flight and free a stage once the
// group after it is issued.  The epilogue is the tiled kernel's (tiled_epilogue_item), scale 1.
//
// Grid: x = target patch (fastest), y = query block, z = sample.  Consecutive CTAs share a query block, so the ~2 query blocks
// resident at a time keep their A' rows (1.7 MB each) in L2 while every patch streams past them; A' (94 MB per pair at
// 1024 x 436) leaves HBM about once, and the padded B operand (8 MB) stays in L2.
//
// Targets of a patch beyond W or H read the padded buffer's replicate border or the TMA unit's zero fill; they only reach the
// level-0 pad cells of the last tiles, which the lookup masks (corr_tiled.cu), and the floor-sized 2 x 2 pooling never reads them.
constexpr int kShiftStages = 3;
constexpr int kShiftChunks = kLlaK / 64;  // 104

struct __align__(8) ShiftBars {
  uint64_t full[kShiftStages];
  uint64_t empty[kShiftStages];
  uint64_t acc_full;
  uint64_t acc_empty;
};

template <typename T>
__global__ void __launch_bounds__(kCorrThreads, 1)
shift_volume_tiled_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                          const __grid_constant__ CUtensorMap tmO, TiledOut out, int W, int N1, int levels) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sStage = smem;                                                      // kShiftStages x (A 16 KB | B 16 KB)
  float* sacc = reinterpret_cast<float*>(sStage + kShiftStages * 2 * kTileBytes);  // fp32 accumulator tile, 128 columns
  uint8_t* sC = reinterpret_cast<uint8_t*>(sacc) + acc_tile_bytes(128);        // 32 KB level-0 staging
  ShiftBars* bars = reinterpret_cast<ShiftBars*>(sC + 2 * kTileBytes);

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int PW = (W + 15) / 16;
  const int ph = blockIdx.x / PW, pw = blockIdx.x - ph * PW;
  const int m_tile = blockIdx.y, b = blockIdx.z;

  if (threadIdx.x == 0) {
    for (int s = 0; s < kShiftStages; ++s) {
      mbar_init(&bars->full[s], 1);
      mbar_init(&bars->empty[s], 8);  // one arrival per MMA warp
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, 4);
    fence_barrier_init();
  }
  if (warp == 12 && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
    prefetch_tmap(&tmO);
  }
  __syncthreads();

  if (warp == 12) {
    // ================= TMA producer =================
    if (lane == 0) {
      for (int k = 0; k < kShiftChunks; ++k) {
        const int st = k % kShiftStages, use = k / kShiftStages;
        mbar_wait(&bars->empty[st], (use & 1) ^ 1);
        mbar_arrive_expect_tx(&bars->full[st], 2 * kTileBytes);
        uint8_t* sa = sStage + st * 2 * kTileBytes;
        tma_load_3d(sa, &tmA, &bars->full[st], k * 64, m_tile * 128, b);
        // chunk k: segment k / 4 of B' (0: fmap2', channels 0..255 of the padded buffer; 1 + l: f2'' at delta_l, channels 256..511)
        const int seg = k >> 2, c0 = (k & 3) * 64;
        const int l = seg - 1;
        const int ch = seg == 0 ? c0 : kLlaC + c0;
        const int dy = seg == 0 ? 0 : l / 5 - 2, dx = seg == 0 ? 0 : l % 5 - 2;
        tma_load_4d(sa + kTileBytes, &tmB, &bars->full[st], ch, pw * 16 + 2 + dx, ph * 8 + 2 + dy, b);
      }
    }
  } else if (warp >= 4) {
    // ================= MMA warpgroups =================
    float d[64];
    for (int k = 0; k < kShiftChunks; ++k) {
      const int st = k % kShiftStages, use = k / kShiftStages;
      mbar_wait(&bars->full[st], use & 1);
      const uint32_t sa = smem_u32(sStage + st * 2 * kTileBytes);
      wgmma_fence();
      corr_mma_k<std::is_same<T, __nv_bfloat16>::value>(d, sa, sa + kTileBytes, 1, k == 0);
      wgmma_commit();
      wgmma_wait<1>();  // chunk k - 1's group has retired: its stage can be refilled
      __syncwarp();
      if (k > 0 && lane == 0) mbar_arrive(&bars->empty[(k - 1) % kShiftStages]);
    }
    wgmma_wait<0>();
    reg_fence(d);
    corr_acc_handoff(d, sacc, &bars->acc_empty, &bars->acc_full, 0);
  } else {
    // ================= epilogue: 4 warps, thread <-> query row =================
    const int row = (warp & 3) * 32 + lane;
    const int n1 = m_tile * 128 + row;
    const bool row_ok = n1 < N1;
    const size_t q = (size_t)b * N1 + (row_ok ? n1 : 0);
    T* o1 = levels > 1 ? reinterpret_cast<T*>(out.ptr[1]) + q * out.map_elems[1] : nullptr;
    T* o2 = levels > 2 ? reinterpret_cast<T*>(out.ptr[2]) + q * out.map_elems[2] : nullptr;
    T* o3 = levels > 3 ? reinterpret_cast<T*>(out.ptr[3]) + q * out.map_elems[3] : nullptr;
    tiled_epilogue_item<T>(sacc, sC, &tmO, out, row, row_ok, o1, o2, o3, 0, ph, pw, m_tile, b, 1.0f, &bars->acc_full, &bars->acc_empty);
    if (row == 0) tma_store_wait_read();
  }
}

static int check_lla_grid(int B, int H, int W, const char* name) {
  PFB_CHECK_ARG(B > 0 && H > 0 && W > 0, "%s: bad grid %dx%dx%d", name, B, H, W);
  return PFB_OK;
}

static unsigned blocks_for(size_t n, int threads) { return (unsigned)ceil_div_sz(n, (size_t)threads); }

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API int pfb_local_similar(const void* qk, float* a1, float* a2, int B, int H, int W, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(qk && a1 && a2, "local_similar: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "local_similar: bad dtype %d", (int)dtype);
  PFB_TRY(check_lla_grid(B, H, W, "local_similar"));
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    local_similar_kernel<T><<<blocks_for(2 * P, kLsWarps), kLsWarps * 32, 0, s>>>(reinterpret_cast<const T*>(qk), a1, a2, B, H, W,
                                                                                   1.0f / sqrtf((float)kLlaD));
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_local_aggregate(const void* fmap2, const void* v, const float* a2, float gamma, void* out, int B, int H, int W,
                                           pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(fmap2 && v && a2 && out, "local_aggregate: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "local_aggregate: bad dtype %d", (int)dtype);
  PFB_TRY(check_lla_grid(B, H, W, "local_aggregate"));
  const size_t n = (size_t)B * H * W * kLlaC;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    local_aggregate_kernel<T><<<blocks_for(n, 256), 256, 0, s>>>(reinterpret_cast<const T*>(fmap2), reinterpret_cast<const T*>(v), a2, gamma,
                                                                 reinterpret_cast<T*>(out), B, H, W);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_shift_pack(const void* fmap1, const void* f1, const float* a1, const void* fmap2, const void* f2, float gamma,
                                      void* a_pack, void* b_pad, void* b_pack, int B, int H, int W, pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(a_pack || b_pad || b_pack, "shift_pack: nothing to write");
  PFB_CHECK_ARG(!a_pack || (fmap1 && f1 && a1), "shift_pack: a_pack needs fmap1, f1 and a1");
  PFB_CHECK_ARG(!(b_pad || b_pack) || (fmap2 && f2), "shift_pack: b_pad / b_pack need fmap2 and f2");
  PFB_CHECK_ARG(dtype_ok(dtype), "shift_pack: bad dtype %d", (int)dtype);
  PFB_TRY(check_lla_grid(B, H, W, "shift_pack"));
  const size_t P = (size_t)B * H * W;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_MISC, s);
  PFB_DISPATCH_DTYPE(dtype, T, {
    const T* m1 = reinterpret_cast<const T*>(fmap1);
    const T* m2 = reinterpret_cast<const T*>(fmap2);
    if (a_pack)
      shift_pack_a_kernel<T><<<blocks_for(P * kLlaK, 256), 256, 0, s>>>(m1, reinterpret_cast<const T*>(f1), a1, gamma,
                                                                        reinterpret_cast<T*>(a_pack), B, H, W);
    if (b_pad)
      shift_pack_bpad_kernel<T><<<blocks_for((size_t)B * (H + 4) * (W + 4) * 2 * kLlaC, 256), 256, 0, s>>>(
          m2, reinterpret_cast<const T*>(f2), reinterpret_cast<T*>(b_pad), B, H, W);
    if (b_pack)
      shift_pack_bmat_kernel<T><<<blocks_for(P * kLlaK, 256), 256, 0, s>>>(m2, reinterpret_cast<const T*>(f2), reinterpret_cast<T*>(b_pack),
                                                                           B, H, W);
  });
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

extern "C" PFB_API int pfb_shift_volume_tiled(const void* a_pack, const void* b_pad, void* const* pyramid, int B, int H, int W, int levels,
                                              pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(a_pack && b_pad && pyramid, "shift_volume_tiled: null pointer");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "shift_volume_tiled: f16 / bf16 only (dtype=%d)", (int)dtype);
  PFB_CHECK_ARG(B > 0 && B <= 65535 && H > 0 && W > 0, "shift_volume_tiled: bad grid %dx%dx%d", B, H, W);
  PFB_CHECK_ARG(levels >= 1 && levels <= 4 && (H >> (levels - 1)) >= 1 && (W >> (levels - 1)) >= 1,
                "shift_volume_tiled: %dx%d grid cannot hold %d levels (1..4)", H, W, levels);
  PFB_CHECK_ARG((reinterpret_cast<uintptr_t>(a_pack) & 15) == 0 && (reinterpret_cast<uintptr_t>(b_pad) & 15) == 0,
                "shift_volume_tiled: operands must be 16-byte aligned");
  for (int l = 0; l < levels; ++l)
    PFB_CHECK_ARG(pyramid[l] && (reinterpret_cast<uintptr_t>(pyramid[l]) & 15) == 0, "shift_volume_tiled: pyramid[%d] null or not 16-byte aligned", l);
  const int N1 = H * W;
  const int m_tiles = ceil_div(N1, 128), n_patches = ceil_div(W, 16) * ceil_div(H, 8);
  PFB_CHECK_ARG(m_tiles <= 65535, "shift_volume_tiled: %d queries per sample exceed the grid", N1);
  CUtensorMap tmA, tmB, tmO;
  {
    uint64_t dims[3] = {(uint64_t)kLlaK, (uint64_t)N1, (uint64_t)B};
    uint64_t str[2] = {(uint64_t)kLlaK * 2, (uint64_t)N1 * kLlaK * 2};
    uint32_t box[3] = {64, 128, 1};
    PFB_TRY(make_tensor_map(&tmA, a_pack, dtype, 3, dims, str, box));
  }
  {
    const uint64_t Hp = H + 4, Wp = W + 4;
    uint64_t dims[4] = {2 * kLlaC, Wp, Hp, (uint64_t)B};
    uint64_t str[3] = {2 * kLlaC * 2, Wp * 2 * kLlaC * 2, Hp * Wp * 2 * kLlaC * 2};
    uint32_t box[4] = {64, 16, 8, 1};
    PFB_TRY(make_tensor_map(&tmB, b_pad, dtype, 4, dims, str, box));
  }
  TiledOut out{};
  PFB_TRY(tiled_out_maps(pyramid, B, N1, H, W, levels, dtype, &out, &tmO));
  const size_t smem = (size_t)kShiftStages * 2 * kTileBytes + acc_tile_bytes(128) + 2 * kTileBytes + sizeof(ShiftBars) + 1024;
  const dim3 grid(n_patches, m_tiles, B);
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_VOLUME, s);
  if (dtype == PFB_F16) {
    PFB_CUDA(cudaFuncSetAttribute(shift_volume_tiled_kernel<__half>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    shift_volume_tiled_kernel<__half><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, W, N1, levels);
  } else {
    PFB_CUDA(cudaFuncSetAttribute(shift_volume_tiled_kernel<__nv_bfloat16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    shift_volume_tiled_kernel<__nv_bfloat16><<<grid, kCorrThreads, smem, s>>>(tmA, tmB, tmO, out, W, N1, levels);
  }
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}
