// a21: SCV's k-NN (ptlflow/models/scv/scv.py:48-83, knn.py:88-116): for every query of f1 the k targets of f2 (same sample) with the
// largest inner product.  The N x N scores never leave the CTA.
//
// Both implementations give a CTA 64 queries and stream 64-target tiles of the sample; each tile's scores go to shared memory, and
// one warp per query folds them into the query's running top-k.  The list lives in registers, lane j holding entry j, sorted by
// (score descending, target ascending); a score that does not beat entry k-1 is dropped with one compare and a ballot, a survivor is
// inserted with one ballot (its rank) and one shuffle.  The list is the exact top-k of that total order whatever order tiles and
// survivors arrive in: no atomics, bit-identical across runs and graph replays.
//
// wgmma (f16 / bf16, C = 64, 128, 192 or 256): one warpgroup; the query block is loaded once by TMA (3D maps over [B][N][C], 128-byte
//   swizzle, K-major, rows past N zero-filled), target tiles through a two-stage TMA ring; S = Q T^T is KC x 4 wgmma m64n64k16 with
//   fp32 accumulators (products of f16 / bf16 values are exact in fp32).
// SIMT (fp32, impl = 1, or operands the TMA cannot address): a 64 x 64 fp32 FMA GEMM, 4 x 4 outputs per thread, 32-channel chunks.
// Split targets: when B x ceil(N / 64) query blocks would leave SMs idle, blockIdx.y splits the target tiles into contiguous ranges;
//   each split writes its raw top-k list to the workspace and knn_merge_kernel folds the lists of a query in split order (the same
//   exact top-k, so the result does not depend on the split count).
#include <limits.h>
#include <math.h>

#include <type_traits>

#include "umma.cuh"

namespace pfb {

constexpr int KQ = 64, KT = 64, KNN_MAX_K = 32;
constexpr unsigned FULL = 0xffffffffu;

// (a, ia) ranks before (b, ib): larger score, then the lower target
__device__ __forceinline__ bool knn_better(float a, int ia, float b, int ib) { return a > b || (a == b && ia < ib); }

// every lane offers one candidate (v, t) when ok; the warp's list (bv, bi: lane j holds entry j, j < k) keeps the best k
__device__ __forceinline__ void knn_offer(float v, int t, bool ok, int k, int lane, float& bv, int& bi) {
  const float kv = __shfl_sync(FULL, bv, k - 1);
  const int ki = __shfl_sync(FULL, bi, k - 1);
  unsigned surv = __ballot_sync(FULL, ok && knn_better(v, t, kv, ki));
  while (surv) {
    const int src = __ffs(surv) - 1;
    surv &= surv - 1;
    const float cv = __shfl_sync(FULL, v, src);
    const int ci = __shfl_sync(FULL, t, src);
    const int pos = __popc(__ballot_sync(FULL, lane < k && knn_better(bv, bi, cv, ci)));
    const float up_v = __shfl_up_sync(FULL, bv, 1);
    const int up_i = __shfl_up_sync(FULL, bi, 1);
    if (lane == pos) { bv = cv; bi = ci; }
    else if (lane > pos && lane < k) { bv = up_v; bi = up_i; }
  }
}

// the split's result: final (scaled) when the targets are not split, the raw list in the workspace otherwise
__device__ __forceinline__ void knn_store(int b, int q, int N, int k, int lane, float bv, int bi, float scale, float* val, int* idx,
                                          float* part_v, int* part_i, int split, int splits) {
  if (q >= N || lane >= k) return;
  const size_t row = (size_t)b * N + q;
  if (splits == 1) {
    val[row * k + lane] = bv * scale;
    idx[row * k + lane] = bi;
  } else {
    const size_t o = (row * splits + split) * k + lane;
    part_v[o] = bv;
    part_i[o] = bi;
  }
}

// ---------------------------------------------------------------- SIMT path
constexpr int KS_C = 32, KS_THREADS = 256, KS_QPW = KQ / (KS_THREADS / 32);

template <typename T>
__global__ void __launch_bounds__(KS_THREADS)
knn_simt_kernel(const T* __restrict__ f1, const T* __restrict__ f2, float* __restrict__ val, int* __restrict__ idx, float* __restrict__ part_v,
                int* __restrict__ part_i, int N, int C, int k, float scale, int tiles_per_split, int splits) {
  // rows padded by one: the staging stores (consecutive lanes on the channel) hit 32 different banks
  __shared__ float qs[KS_C][KQ + 1];
  __shared__ float ts[KS_C][KT + 1];
  __shared__ float sc[KQ][KT + 1];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int b = blockIdx.z, split = blockIdx.y, q0 = blockIdx.x * KQ;
  const int j0 = split * tiles_per_split, j1 = min(j0 + tiles_per_split, (N + KT - 1) / KT);
  const T* F1 = f1 + (size_t)b * N * C;
  const T* F2 = f2 + (size_t)b * N * C;
  const int tx = tid & 15, ty = tid >> 4;  // outputs (query ty + 16 i, target tx + 16 j)
  float bv[KS_QPW];
  int bi[KS_QPW];
#pragma unroll
  for (int i = 0; i < KS_QPW; ++i) { bv[i] = -INFINITY; bi[i] = INT_MAX; }

  for (int jt = j0; jt < j1; ++jt) {
    const int t0 = jt * KT;
    float acc[4][4] = {};
    for (int c0 = 0; c0 < C; c0 += KS_C) {
      // element e = row * KS_C + c: consecutive lanes read consecutive channels of a row; rows past N, channels past C are zero
      for (int e = tid; e < KQ * KS_C; e += KS_THREADS) {
        const int r = e / KS_C, c = e % KS_C;
        const int q = q0 + r, t = t0 + r, cc = c0 + c;
        qs[c][r] = (q < N && cc < C) ? to_f32(F1[(size_t)q * C + cc]) : 0.f;
        ts[c][r] = (t < N && cc < C) ? to_f32(F2[(size_t)t * C + cc]) : 0.f;
      }
      __syncthreads();
#pragma unroll 8
      for (int c = 0; c < KS_C; ++c) {
        float a[4], bb[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i] = qs[c][ty + 16 * i]; bb[i] = ts[c][tx + 16 * i]; }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], bb[j], acc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) sc[ty + 16 * i][tx + 16 * j] = acc[i][j];
    __syncthreads();
#pragma unroll
    for (int i = 0; i < KS_QPW; ++i) {
      const float* row = sc[warp * KS_QPW + i];
      knn_offer(row[lane], t0 + lane, t0 + lane < N, k, lane, bv[i], bi[i]);
      knn_offer(row[lane + 32], t0 + lane + 32, t0 + lane + 32 < N, k, lane, bv[i], bi[i]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < KS_QPW; ++i)
    knn_store(b, q0 + warp * KS_QPW + i, N, k, lane, bv[i], bi[i], scale, val, idx, part_v, part_i, split, splits);
}

// ---------------------------------------------------------------- wgmma path
constexpr int KU_THREADS = 128, KU_TILE = 64 * 128, KU_QPW = KQ / (KU_THREADS / 32), KU_SPITCH = KT + 1;

struct __align__(8) KnnBars {  // in the 1024-byte header of the shared-memory carve
  uint64_t q_full, t_full[2];
};

template <typename T, int C>
__global__ void __launch_bounds__(KU_THREADS, 1)
knn_umma_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmT, float* __restrict__ val,
                int* __restrict__ idx, float* __restrict__ part_v, int* __restrict__ part_i, int N, int k, float scale, int tiles_per_split,
                int splits) {
  using namespace sm90;
  constexpr bool BF16 = std::is_same<T, __nv_bfloat16>::value;
  constexpr int KCH = C / 64;  // 64-channel chunks
  extern __shared__ __align__(1024) uint8_t ku_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(ku_smem_raw) + 1023) & ~uintptr_t(1023));
  KnnBars* bars = reinterpret_cast<KnnBars*>(smem);
  uint8_t* sQ = smem + 1024;                                   // KCH tiles [64 queries][64 ch]
  uint8_t* sT = sQ + KCH * KU_TILE;                            // 2 stages x KCH tiles [64 targets][64 ch]
  float* sS = reinterpret_cast<float*>(sT + 2 * KCH * KU_TILE);  // [64 queries][KU_SPITCH] scores of the tile

  const int b = blockIdx.z, split = blockIdx.y, q0 = blockIdx.x * KQ;
  const int j0 = split * tiles_per_split, j1 = min(j0 + tiles_per_split, (N + KT - 1) / KT);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;

  if (tid == 0) {
    mbar_init(&bars->q_full, 1);
    mbar_init(&bars->t_full[0], 1);
    mbar_init(&bars->t_full[1], 1);
    fence_barrier_init();
  }
  __syncthreads();
  auto load_t = [&](int j) {
    const int st = (j - j0) & 1;
    mbar_arrive_expect_tx(&bars->t_full[st], KCH * KU_TILE);
    for (int kc = 0; kc < KCH; ++kc) tma_load_3d(sT + (st * KCH + kc) * KU_TILE, &tmT, &bars->t_full[st], kc * 64, j * KT, b);
  };
  if (tid == 0) {
    mbar_arrive_expect_tx(&bars->q_full, KCH * KU_TILE);
    for (int kc = 0; kc < KCH; ++kc) tma_load_3d(sQ + kc * KU_TILE, &tmQ, &bars->q_full, kc * 64, q0, b);
    if (j0 < j1) load_t(j0);
    if (j0 + 1 < j1) load_t(j0 + 1);
  }
  mbar_wait(&bars->q_full, 0);

  const int r0 = 16 * warp + (lane >> 2);  // fragment rows r0, r0 + 8; columns 8 (e >> 2) + 2 (lane & 3) + (e & 1)
  float bv[KU_QPW];
  int bi[KU_QPW];
#pragma unroll
  for (int i = 0; i < KU_QPW; ++i) { bv[i] = -INFINITY; bi[i] = INT_MAX; }

  for (int j = j0; j < j1; ++j) {
    const int st = (j - j0) & 1;
    mbar_wait(&bars->t_full[st], ((j - j0) >> 1) & 1);
    float sc[32];
    wgmma_fence();
#pragma unroll
    for (int kc = 0; kc < KCH; ++kc) {
      const uint32_t al = gdesc_lo(smem_u32(sQ + kc * KU_TILE), 16), bl = gdesc_lo(smem_u32(sT + (st * KCH + kc) * KU_TILE), 16);
#pragma unroll
      for (int kk = 0; kk < 4; ++kk)
        wgmma<64, BF16>(sc, gdesc(al + 2 * kk, kDescHiSw128), gdesc(bl + 2 * kk, kDescHiSw128), (kc == 0 && kk == 0) ? 0u : 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    reg_fence(sc);
#pragma unroll
    for (int e = 0; e < 32; ++e) sS[(r0 + 8 * ((e >> 1) & 1)) * KU_SPITCH + 8 * (e >> 2) + 2 * (lane & 3) + (e & 1)] = sc[e];
    __syncthreads();  // every warp's wgmma has read stage st, and the tile's scores are complete
    if (tid == 0 && j + 2 < j1) load_t(j + 2);
    const int t0 = j * KT;
#pragma unroll
    for (int i = 0; i < KU_QPW; ++i) {
      const float* row = sS + (warp * KU_QPW + i) * KU_SPITCH;
      knn_offer(row[lane], t0 + lane, t0 + lane < N, k, lane, bv[i], bi[i]);
      knn_offer(row[lane + 32], t0 + lane + 32, t0 + lane + 32 < N, k, lane, bv[i], bi[i]);
    }
    __syncthreads();  // the scores are read before the next tile rewrites them
  }
#pragma unroll
  for (int i = 0; i < KU_QPW; ++i)
    knn_store(b, q0 + warp * KU_QPW + i, N, k, lane, bv[i], bi[i], scale, val, idx, part_v, part_i, split, splits);
}

// one warp per query: the splits' lists, in split order, folded into the final top-k
constexpr int KM_WARPS = 8;
__global__ void __launch_bounds__(KM_WARPS * 32)
knn_merge_kernel(const float* __restrict__ part_v, const int* __restrict__ part_i, float* __restrict__ val, int* __restrict__ idx, size_t rows,
                 int k, int splits, float scale) {
  const int lane = threadIdx.x & 31;
  const size_t row = (size_t)blockIdx.x * KM_WARPS + (threadIdx.x >> 5);
  if (row >= rows) return;  // whole warps leave together
  float bv = -INFINITY;
  int bi = INT_MAX;
  for (int s = 0; s < splits; ++s) {
    const size_t o = (row * splits + s) * k + lane;
    knn_offer(lane < k ? part_v[o] : 0.f, lane < k ? part_i[o] : 0, lane < k, k, lane, bv, bi);
  }
  if (lane < k) {
    val[row * k + lane] = bv * scale;
    idx[row * k + lane] = bi;
  }
}

static size_t knn_umma_smem(int C) { return 1024 + 1024 + 3 * (size_t)(C / 64) * KU_TILE + (size_t)KQ * KU_SPITCH * 4; }

static bool knn_umma_supported(const void* f1, const void* f2, int C, pfb_dtype dt) {
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  return dt != PFB_F32 && C % 64 == 0 && C >= 64 && C <= 256 && al16(f1) && al16(f2);
}

struct KnnPlan {
  bool umma;
  int tiles_per_split, splits;
};

// the split count: enough CTAs for two per SM when the query blocks alone are fewer, at least 4 target tiles per split
static KnnPlan knn_plan(const void* f1, const void* f2, int B, int N, int C, int impl, pfb_dtype dt) {
  KnnPlan p{};
  p.umma = impl != 1 && knn_umma_supported(f1, f2, C, dt);
  const int tiles = ceil_div(N, KT);
  const long qblocks = (long)B * ceil_div(N, KQ);
  const long want = 2L * sm_count();
  int splits = qblocks >= want ? 1 : (int)std::min<long>((want + qblocks - 1) / qblocks, std::max(1, tiles / 4));
  p.tiles_per_split = ceil_div(tiles, splits);
  p.splits = ceil_div(tiles, p.tiles_per_split);
  return p;
}

static size_t knn_workspace(const KnnPlan& p, int B, int N, int k) {
  return p.splits > 1 ? (size_t)B * N * p.splits * k * (sizeof(float) + sizeof(int)) : 0;
}

static int knn_check(const void* f1, const void* f2, int B, int N, int C, int k, pfb_dtype dtype, int impl) {
  PFB_CHECK_ARG(f1 && f2, "knn_topk: null pointer");
  PFB_CHECK_ARG(dtype_ok(dtype), "knn_topk: bad dtype %d", (int)dtype);
  PFB_CHECK_ARG(B > 0 && N > 0 && C > 0, "knn_topk: bad shape B=%d N=%d C=%d", B, N, C);
  PFB_CHECK_ARG(k >= 1 && k <= KNN_MAX_K && k <= N, "knn_topk: k=%d (1..%d and at most N=%d)", k, KNN_MAX_K, N);
  PFB_CHECK_ARG(impl >= 0 && impl <= 2, "knn_topk: impl=%d (0 auto, 1 SIMT, 2 wgmma)", impl);
  PFB_CHECK_ARG(impl != 2 || knn_umma_supported(f1, f2, C, dtype),
                "knn_topk: impl=2 needs f16 / bf16, C a multiple of 64 up to 256 and 16-byte aligned features (C=%d dtype=%d)", C, (int)dtype);
  return PFB_OK;
}

template <typename T, int C>
static int launch_knn_umma(const void* f1, const void* f2, float* val, int* idx, float* pv, int* pi, int B, int N, int k, float scale,
                           const KnnPlan& p, pfb_dtype dt, cudaStream_t s) {
  CUtensorMap tq, tt;
  const uint64_t dims[3] = {(uint64_t)C, (uint64_t)N, (uint64_t)B};
  const uint64_t str[2] = {(uint64_t)C * 2, (uint64_t)N * C * 2};
  const uint32_t box[3] = {64, (uint32_t)KQ, 1};
  PFB_TRY(make_tensor_map(&tq, f1, dt, 3, dims, str, box));
  PFB_TRY(make_tensor_map(&tt, f2, dt, 3, dims, str, box));
  const size_t smem = knn_umma_smem(C);
  auto kern = knn_umma_kernel<T, C>;
  PFB_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kern<<<dim3(ceil_div(N, KQ), p.splits, B), KU_THREADS, smem, s>>>(tq, tt, val, idx, pv, pi, N, k, scale, p.tiles_per_split, p.splits);
  PFB_LAUNCH_CHECK();
  return PFB_OK;
}

}  // namespace pfb

using namespace pfb;

extern "C" PFB_API size_t pfb_knn_topk_workspace_bytes(const void* f1, const void* f2, int B, int N, int C, int k, pfb_dtype dtype,
                                                       int impl) {
  if (knn_check(f1, f2, B, N, C, k, dtype, impl) != PFB_OK) return 0;
  return knn_workspace(knn_plan(f1, f2, B, N, C, impl, dtype), B, N, k);
}

extern "C" PFB_API int pfb_knn_topk(const void* f1, const void* f2, float* val, int* idx, void* workspace, size_t workspace_bytes, int B, int N,
                                    int C, int k, float scale, pfb_dtype dtype, int impl, pfb_stream stream) {
  PFB_TRY(knn_check(f1, f2, B, N, C, k, dtype, impl));
  PFB_CHECK_ARG(val && idx, "knn_topk: null output");
  const KnnPlan p = knn_plan(f1, f2, B, N, C, impl, dtype);
  const size_t need = knn_workspace(p, B, N, k);
  PFB_CHECK_ARG(workspace_bytes >= need && (need == 0 || workspace), "knn_topk: workspace %zu bytes < required %zu", workspace_bytes, need);
  float* pv = need ? reinterpret_cast<float*>(workspace) : nullptr;
  int* pi = need ? reinterpret_cast<int*>(pv + (size_t)B * N * p.splits * k) : nullptr;
  const cudaStream_t s = as_stream(stream);
  ProfScope prof(KC_VOLUME, s);
  if (p.umma) {
    const bool bf = dtype == PFB_BF16;
#define PFB_KNN_CASE(CC)                                                                                             \
  if (C == CC) {                                                                                                     \
    const int rc = bf ? launch_knn_umma<__nv_bfloat16, CC>(f1, f2, val, idx, pv, pi, B, N, k, scale, p, dtype, s)    \
                      : launch_knn_umma<__half, CC>(f1, f2, val, idx, pv, pi, B, N, k, scale, p, dtype, s);          \
    PFB_TRY(rc);                                                                                                     \
  }
    PFB_KNN_CASE(64)
    PFB_KNN_CASE(128)
    PFB_KNN_CASE(192)
    PFB_KNN_CASE(256)
#undef PFB_KNN_CASE
  } else {
    PFB_DISPATCH_DTYPE(dtype, T, {
      knn_simt_kernel<T><<<dim3(ceil_div(N, KQ), p.splits, B), KS_THREADS, 0, s>>>(
          reinterpret_cast<const T*>(f1), reinterpret_cast<const T*>(f2), val, idx, pv, pi, N, C, k, scale, p.tiles_per_split, p.splits);
    });
    PFB_LAUNCH_CHECK();
  }
  if (p.splits > 1) {
    const size_t rows = (size_t)B * N;
    knn_merge_kernel<<<(unsigned)ceil_div_sz(rows, KM_WARPS), KM_WARPS * 32, 0, s>>>(pv, pi, val, idx, rows, k, p.splits, scale);
    PFB_LAUNCH_CHECK();
  }
  return PFB_OK;
}
