// Encoder 3x3 stride-1 "same" convolution on the Hopper tensor cores, output channels on the MMA's M dimension.
//
//   out[p, co] = epilogue( sum_{ky, kx, c} W[co][c][ky][kx] * X[p + (ky - 1, kx - 1), c] )
//
// The update-block kernel (conv_umma.cu) puts pixels on M and output channels on N.  At the encoders' widths (64, 96, 128
// output channels) that is the small-N case: an m64n64k16 reads 4 KB of operands from shared memory for 131 kFLOP, as
// long as the MMA itself takes.  Here the product is transposed: A = a 64-row block of the weights, B = 128 pixels of the
// activation patch, one m64n128k16 per 16-channel K step (2 KB + 4 KB for 262 kFLOP).
//
//   Work item : TW pixels of one image row.  Cout = 64: TW = 256, the two MMA warpgroups take 128 pixels each with the
//               same weight block.  Cout = 96 / 128: TW = 128, warpgroup w takes output channels 64w .. 64w + 63 of all
//               of them (for 96 the rows 96..127 of the second block are computed from whatever follows in the weight
//               tensor and never stored).
//   K loop    : (64-channel chunk, ky, kx).  One activation patch of TW + 2 pixels per (chunk, ky), loaded by TMA with the
//               x halo; out-of-image pixels and channels beyond Cin are zero-filled by the TMA unit ("same" padding).  Tap
//               kx reads the patch through a descriptor advanced by kx pixel rows (128 B): the swizzle is a function of
//               the absolute shared-memory address.  A 32-channel last chunk issues 2 of its 4 K steps.
//   Weights   : the K-major packing of ops.PackedConv, [9][Cout_pad_k][Cin_pad].  One tap for all M blocks per weight
//               stage; when every tap fits next to the patch ring (Cout = 64, Cin <= 64: 72 KB), the weights are loaded
//               once per CTA and stay resident.
//   Epilogue  : in the MMA warpgroups, from the fp32 accumulators (rounded once).  stmatrix .trans turns the channel-major
//               fragments into pixel-major 128-byte rows of a swizzled staging tile, which leaves with one TMA store per
//               warpgroup (clipped at the image's right edge and at Cout).  The residual epilogue first TMA-loads the
//               residual tile into the same staging buffer (issued before the tile's MMAs) and reads it back in fragment
//               order with ldmatrix .trans.
//
// Persistent CTAs (one per SM) walk the work items round-robin; warpgroup 0 is the TMA producer, 1 and 2 the MMA +
// epilogue warpgroups.
#include <atomic>
#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

constexpr int kEcThreads = 3 * 128;
constexpr int kEcNW = 128;                 // pixels per MMA warpgroup (wgmma N)
constexpr int kEcPatchBox = kEcNW + 2;     // pixels per patch TMA box (128 + the x halo)
constexpr int kEcStageOut = kEcNW * 128;   // [128 pixels][64 channels] staging tile per MMA warpgroup
constexpr int kEcMaxA = 8, kEcMaxW = 18;
// Register budget per role: 384 threads at one CTA per SM launch with 170 each; the producer keeps 40, the MMA warpgroups
// (64 fp32 accumulators + addressing) take up to 232.
constexpr int kEcProducerRegs = 40, kEcMmaRegs = 232;
static_assert(128 * (kEcProducerRegs + 2 * kEcMmaRegs) <= 65536, "register budget exceeds the register file");

struct __align__(8) EcBars {
  uint64_t a_full[kEcMaxA];
  uint64_t a_empty[kEcMaxA];
  uint64_t w_full[kEcMaxW];
  uint64_t w_empty[kEcMaxW];
  uint64_t res_full[2];
};

struct EcPlan {
  int mb;                  // 64-row M blocks (1: Cout = 64, 2: Cout = 96 / 128)
  int TW;                  // pixels per work item
  int chunks;              // 64-channel chunks of the input
  int a_stages, a_slot_bytes;
  int w_stages, w_slot_bytes;
  int w_resident;          // 1: w_stages == 9 * chunks, every tap loaded once
  int tiles_x, n_work;
  size_t smem;
};

struct EncConvArgs {
  int B, H, W, Cin, Cout, Cout_pad_k;
  int mb, TW, chunks, tiles_x, n_work;
  int a_stages, a_slot_bytes, w_stages, w_slot_bytes, w_resident;
  int out_offset;
  const float* bias;
};

// Everything about a launch but its operands.  pfb_enc_conv3x3_supported and pfb_enc_conv3x3 both call it.
static bool plan_enc_conv(int B, int H, int W, int Cin, int Cout, EcPlan& pl) {
  if (B < 1 || H < 1 || W < 1) return false;
  if (Cin < 32 || Cin % 32) return false;
  if (Cout != 64 && Cout != 96 && Cout != 128) return false;
  pl.mb = Cout > 64 ? 2 : 1;
  pl.TW = pl.mb == 1 ? 2 * kEcNW : kEcNW;
  pl.chunks = ceil_div(Cin, 64);
  pl.a_slot_bytes = (int)align_up((size_t)(pl.TW + 2) * 128, 1024);
  pl.w_slot_bytes = pl.mb * 64 * 128;
  const int fixed = 2 * kEcStageOut + (int)sizeof(EcBars) + 1024;  // staging, barriers, alignment slack
  const int budget = 227 * 1024 - fixed;
  const int taps = 9 * pl.chunks;
  // resident weights when all taps fit next to three patches
  pl.w_resident = taps <= kEcMaxW && taps * pl.w_slot_bytes + 3 * pl.a_slot_bytes <= budget;
  int best = -1;
  if (pl.w_resident) {
    pl.w_stages = taps;
    pl.a_stages = (budget - taps * pl.w_slot_bytes) / pl.a_slot_bytes;
    if (pl.a_stages > kEcMaxA) pl.a_stages = kEcMaxA;
    best = 0;
  } else {
    // a slot is reused once per round trip (release -> producer -> TMA -> MMA): maximise the K steps in flight, counted
    // in taps (a patch serves 3)
    for (int as = 2; as <= kEcMaxA; ++as) {
      int ws = (budget - as * pl.a_slot_bytes) / pl.w_slot_bytes;
      if (ws > kEcMaxW) ws = kEcMaxW;
      if (ws < 2) continue;
      const int cover_a = (as - 1) * 3, cover_w = ws - 1;
      const int cover = cover_a < cover_w ? cover_a : cover_w;
      if (cover > best || (cover == best && ws > pl.w_stages)) { best = cover; pl.a_stages = as; pl.w_stages = ws; }
    }
  }
  if (best < 0) return false;
  pl.tiles_x = ceil_div(W, pl.TW);
  const long n_work = (long)pl.tiles_x * H * B;
  if (n_work > (1l << 30)) return false;
  pl.n_work = (int)n_work;
  pl.smem = (size_t)pl.a_stages * pl.a_slot_bytes + (size_t)pl.w_stages * pl.w_slot_bytes + fixed;
  return true;
}

// stmatrix / ldmatrix of four 8x8 b16 matrices, transposed: lane l gives the row address of row l & 7 of matrix l >> 3;
// register i holds (row = lane >> 2, columns 2 (lane & 3), +1) of matrix i, the accumulator fragment order
__device__ __forceinline__ void stmatrix_x4_trans(uint32_t addr, const uint32_t (&r)[4]) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};"
               ::"r"(addr), "r"(r[0]), "r"(r[1]), "r"(r[2]), "r"(r[3]) : "memory");
}
__device__ __forceinline__ void ldmatrix_x4_trans(uint32_t addr, uint32_t (&r)[4]) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr) : "memory");
}

template <typename T>
__device__ __forceinline__ uint32_t ec_pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t ec_pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t ec_pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <typename T>
__device__ __forceinline__ void ec_unpack2(uint32_t u, float& a, float& b) {
  const T* h = reinterpret_cast<const T*>(&u);
  a = to_f32(h[0]);
  b = to_f32(h[1]);
}

// one tap: KS K steps of 16 channels, committed as one wgmma group (fence and commit in the MMAs' own basic block)
template <bool BF16, int KS>
__device__ __forceinline__ void ec_issue(float (&d)[kEcNW / 2], uint32_t w_lo, uint32_t x_lo, uint32_t acc) {
  wgmma_fence();
#pragma unroll
  for (int kk = 0; kk < KS; ++kk)
    wgmma<kEcNW, BF16>(d, gdesc(w_lo + 2 * kk, kDescHiSw128), gdesc(x_lo + 2 * kk, kDescHiSw128), kk == 0 ? acc : 1u);
  wgmma_commit();
}

template <typename T, int EPI>
__global__ void __launch_bounds__(kEcThreads, 1)
enc_conv_umma_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                     const __grid_constant__ CUtensorMap tmO, const __grid_constant__ CUtensorMap tmR, const EncConvArgs a) {
  constexpr bool kBF16 = std::is_same<T, __nv_bfloat16>::value;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemW = smemA + a.a_stages * a.a_slot_bytes;
  uint8_t* smemO = smemW + a.w_stages * a.w_slot_bytes;
  EcBars* bars = reinterpret_cast<EcBars*>(smemO + 2 * kEcStageOut);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.a_stages; ++s) {
      mbar_init(&bars->a_full[s], 1);
      mbar_init(&bars->a_empty[s], 8);  // one arrival per MMA warp
    }
    for (int s = 0; s < a.w_stages; ++s) {
      mbar_init(&bars->w_full[s], 1);
      mbar_init(&bars->w_empty[s], 8);
    }
    mbar_init(&bars->res_full[0], 1);
    mbar_init(&bars->res_full[1], 1);
    fence_barrier_init();
  }
  if (warp == 0 && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmW);
    prefetch_tmap(&tmO);
    if (EPI == PFB_ENC_CONV_BIAS_RELU_RESIDUAL) prefetch_tmap(&tmR);
  }
  __syncthreads();
  pdl_wait();
  pdl_trigger();

  auto decode = [&](int w, int& b, int& y, int& x0) {
    const int px = w % a.tiles_x;
    const int r = w / a.tiles_x;
    y = r % a.H;
    b = r / a.H;
    x0 = px * a.TW;
  };

  if (warp < 4) {
    setmaxnreg_dec<kEcProducerRegs>();
    if (warp == 0) {
      // ================= TMA producer =================
      const int boxes = a.TW / kEcNW;
      const uint32_t a_tx = boxes * kEcPatchBox * 128;
      int sa = 0, sw = 0;
      uint32_t pa = 0, pw = 0;
      if (a.w_resident) {  // every tap once, each on its own barrier so the first tile starts on the first tap
        for (int t = 0; t < a.w_stages; ++t) {
          if (elect_one()) {
            mbar_arrive_expect_tx(&bars->w_full[t], a.w_slot_bytes);
            tma_load_2d(smemW + t * a.w_slot_bytes, &tmW, &bars->w_full[t], (t / 9) * 64, (t % 9) * a.Cout_pad_k);
          }
          __syncwarp();
        }
      }
      for (int w = blockIdx.x; w < a.n_work; w += gridDim.x) {
        int b, y, x0;
        decode(w, b, y, x0);
        for (int c = 0; c < a.chunks; ++c) {
          for (int ky = 0; ky < 3; ++ky) {
            mbar_wait(&bars->a_empty[sa], pa ^ 1);
            if (elect_one()) {
              mbar_arrive_expect_tx(&bars->a_full[sa], a_tx);
              // boxes of 130 pixels that overlap by two: each destination starts on the 1024-byte swizzle period
              for (int h = 0; h < boxes; ++h)
                tma_load_4d(smemA + sa * a.a_slot_bytes + h * kEcNW * 128, &tmX, &bars->a_full[sa], c * 64, x0 - 1 + h * kEcNW,
                            y + ky - 1, b);
            }
            __syncwarp();
            if (++sa == a.a_stages) { sa = 0; pa ^= 1; }
            if (!a.w_resident) {
              for (int kx = 0; kx < 3; ++kx) {
                mbar_wait(&bars->w_empty[sw], pw ^ 1);
                if (elect_one()) {
                  mbar_arrive_expect_tx(&bars->w_full[sw], a.w_slot_bytes);
                  tma_load_2d(smemW + sw * a.w_slot_bytes, &tmW, &bars->w_full[sw], c * 64, (ky * 3 + kx) * a.Cout_pad_k);
                }
                __syncwarp();
                if (++sw == a.w_stages) { sw = 0; pw ^= 1; }
              }
            }
          }
        }
      }
    }
  } else {
    setmaxnreg_inc<kEcMmaRegs>();
    // ================= MMA + epilogue warpgroups =================
    const int wg = (threadIdx.x >> 7) - 1, tid = threadIdx.x & 127, wq = tid >> 5;
    const int mrow = a.mb == 2 ? wg : 0;          // this warpgroup's 64-row block of output channels
    const int pix0 = a.mb == 2 ? 0 : wg * kEcNW;  // and its first pixel of the work item
    uint8_t* stage = smemO + wg * kEcStageOut;
    const uint32_t stage_u32 = smem_u32(stage);
    const uint32_t a_slot16 = (uint32_t)a.a_slot_bytes >> 4, w_slot16 = (uint32_t)a.w_slot_bytes >> 4;
    const uint32_t a_lo0 = gdesc_lo(smem_u32(smemA) + pix0 * 128, 16);
    const uint32_t w_lo0 = gdesc_lo(smem_u32(smemW) + mrow * 64 * 128, 16);
    const uint32_t bar_a_full = smem_u32(&bars->a_full[0]);
    const uint32_t bar_w_full = smem_u32(&bars->w_full[0]);
    // bias of this thread's two fragment rows (channels ch and ch + 8)
    const int ch = mrow * 64 + 16 * wq + (lane >> 2);
    float bias_lo = 0.f, bias_hi = 0.f;
    if (EPI != PFB_ENC_CONV_LINEAR) {
      if (ch < a.Cout) bias_lo = a.bias[ch];
      if (ch + 8 < a.Cout) bias_hi = a.bias[ch + 8];
    }
    int sa = 0, sw = 0, held_a = -1, held_w = -1;
    uint32_t pha = 0, phw = 0, res_phase = 0;
    uint32_t a_lo = a_lo0, w_lo = w_lo0;
    auto release_held = [&]() {
      __syncwarp();
      if (lane == 0) {
        if (held_w >= 0) mbar_arrive(&bars->w_empty[held_w]);
        if (held_a >= 0) mbar_arrive(&bars->a_empty[held_a]);
      }
      held_a = held_w = -1;
    };
    // the residual tile goes into the staging buffer once the previous item's store has read it
    auto load_residual = [&](int b, int y, int x0) {
      if (EPI == PFB_ENC_CONV_BIAS_RELU_RESIDUAL && x0 + pix0 < a.W && tid == 0) {
        tma_store_wait_read();
        mbar_arrive_expect_tx(&bars->res_full[wg], kEcStageOut);
        tma_load_4d(stage, &tmR, &bars->res_full[wg], mrow * 64, x0 + pix0, y, b);
      }
    };
    auto epilogue = [&](float (&dd)[kEcNW / 2], int b, int y, int x0) {
      if (x0 + pix0 >= a.W) return;  // (Cout = 64 on narrow images: the second half may lie beyond the edge)
      // ---- fragments -> pixel-major staging rows -> one TMA store ----
      if (EPI == PFB_ENC_CONV_BIAS_RELU_RESIDUAL) {
        mbar_wait(&bars->res_full[wg], res_phase);
        res_phase ^= 1;
      } else {
        if (tid == 0) tma_store_wait_read();
        named_barrier_sync(1 + wg, 128);
      }
#pragma unroll
      for (int j = 0; j < kEcNW / 8; j += 2) {
        // matrix m = lane >> 3: pixel group j + (m >> 1), channels 16 wq + 8 (m & 1) .. + 7; this lane addresses pixel
        // (lane & 7) of it.  128-byte swizzle: 16-byte piece q of row p lives at piece q ^ (p & 7).
        const int m = lane >> 3;
        const int px = 8 * (j + (m >> 1)) + (lane & 7);
        const int piece = 2 * wq + (m & 1);
        const uint32_t addr = stage_u32 + px * 128 + ((piece ^ (px & 7)) << 4);
        float v[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) v[q] = dd[4 * j + q] + ((q & 2) ? bias_hi : bias_lo);
        if (EPI != PFB_ENC_CONV_LINEAR) {
#pragma unroll
          for (int q = 0; q < 8; ++q) v[q] = fmaxf(v[q], 0.f);
        }
        uint32_t r[4];
        if (EPI == PFB_ENC_CONV_BIAS_RELU_RESIDUAL) {
          ldmatrix_x4_trans(addr, r);
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float r0, r1;
            ec_unpack2<T>(r[q], r0, r1);
            v[2 * q] = fmaxf(v[2 * q] + r0, 0.f);
            v[2 * q + 1] = fmaxf(v[2 * q + 1] + r1, 0.f);
          }
        }
#pragma unroll
        for (int q = 0; q < 4; ++q) r[q] = ec_pack2<T>(v[2 * q], v[2 * q + 1]);
        stmatrix_x4_trans(addr, r);
      }
      fence_proxy_async();
      named_barrier_sync(1 + wg, 128);
      if (tid == 0) {
        tma_store_4d(&tmO, stage, a.out_offset + mrow * 64, x0 + pix0, y, b);
        tma_store_commit();
      }
    };
    // The epilogue does not overlap the warpgroup's own MMAs: with the next item's MMAs in flight across its divergent
    // code (the elected TMA store, the clipped edge), ptxas serialises every wgmma of the kernel (C7518), measured 1.4x
    // slower on layer1.  The producer keeps loading the next item's patches meanwhile.
    float d[kEcNW / 2];
    for (int w = blockIdx.x; w < a.n_work; w += gridDim.x) {
      int b, y, x0;
      decode(w, b, y, x0);
      load_residual(b, y, x0);
      uint32_t acc = 0;  // the first MMA of the item overwrites the accumulator
      for (int c = 0; c < a.chunks; ++c) {
        const bool full_chunk = a.Cin - 64 * c >= 64;  // else 32 channels: 2 K steps
        for (int ky = 0; ky < 3; ++ky) {
          mbar_wait_uniform(bar_a_full + 8 * sa, pha);
          for (int kx = 0; kx < 3; ++kx) {
            uint32_t wl;
            if (a.w_resident) {
              const int t = c * 9 + ky * 3 + kx;
              mbar_wait_uniform(bar_w_full + 8 * t, 0);
              wl = w_lo0 + w_slot16 * t;
            } else {
              mbar_wait_uniform(bar_w_full + 8 * sw, phw);
              wl = w_lo;
            }
            const uint32_t xl = a_lo + 8u * kx;  // tap kx: the patch from pixel row kx (128 B each)
            if (full_chunk) ec_issue<kBF16, 4>(d, wl, xl, acc);
            else ec_issue<kBF16, 2>(d, wl, xl, acc);
            // one group stays in flight: the previous tap's slots are free once it has completed
            wgmma_wait<1>();
            reg_fence(d);
            release_held();
            if (!a.w_resident) {
              held_w = sw;
              w_lo += w_slot16;
              if (++sw == a.w_stages) { sw = 0; phw ^= 1; w_lo = w_lo0; }
            }
            if (kx == 2) held_a = sa;
            acc = 1;
          }
          a_lo += a_slot16;
          if (++sa == a.a_stages) { sa = 0; pha ^= 1; a_lo = a_lo0; }
        }
      }
      wgmma_wait<0>();
      reg_fence(d);
      release_held();
      epilogue(d, b, y, x0);
    }
    if (tid == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete before the CTA exits
  }
}

template <typename T, int EPI>
static int launch_enc_conv_e(const CUtensorMap& tmX, const CUtensorMap& tmW, const CUtensorMap& tmO, const CUtensorMap& tmR,
                             const EncConvArgs& a, int grid, size_t smem, cudaStream_t s) {
  static std::atomic<unsigned long long> attr_done{0};  // once per (instantiation, device)
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(enc_conv_umma_kernel<T, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  PFB_CUDA(launch_pdl(enc_conv_umma_kernel<T, EPI>, dim3(grid), dim3(kEcThreads), smem, s, tmX, tmW, tmO, tmR, a));
  return PFB_OK;
}

template <typename T>
static int launch_enc_conv(int epilogue, const CUtensorMap& tmX, const CUtensorMap& tmW, const CUtensorMap& tmO,
                           const CUtensorMap& tmR, const EncConvArgs& a, int grid, size_t smem, cudaStream_t s) {
  switch (epilogue) {
    case PFB_ENC_CONV_LINEAR: return launch_enc_conv_e<T, PFB_ENC_CONV_LINEAR>(tmX, tmW, tmO, tmR, a, grid, smem, s);
    case PFB_ENC_CONV_BIAS_RELU: return launch_enc_conv_e<T, PFB_ENC_CONV_BIAS_RELU>(tmX, tmW, tmO, tmR, a, grid, smem, s);
    default: return launch_enc_conv_e<T, PFB_ENC_CONV_BIAS_RELU_RESIDUAL>(tmX, tmW, tmO, tmR, a, grid, smem, s);
  }
}

}  // namespace pfb

using namespace pfb;

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

extern "C" PFB_API int pfb_enc_conv3x3_supported(int Cin, int Cout, pfb_dtype dtype) {
  if (dtype != PFB_F16 && dtype != PFB_BF16) return 0;
  EcPlan pl{};
  return plan_enc_conv(1, 1, 1, Cin, Cout, pl) ? 1 : 0;
}

extern "C" PFB_API int pfb_enc_conv3x3(const void* x, const void* weight_k, const float* bias, const void* residual, void* out,
                                       int B, int H, int W, int Cin, int Cout, int out_stride, int out_offset, int epilogue,
                                       pfb_dtype dtype, pfb_stream stream) {
  PFB_CHECK_ARG(x && weight_k && out, "enc_conv3x3: null pointer");
  PFB_CHECK_ARG(dtype == PFB_F16 || dtype == PFB_BF16, "enc_conv3x3: f16 / bf16 storage only");
  PFB_CHECK_ARG(epilogue == PFB_ENC_CONV_LINEAR || epilogue == PFB_ENC_CONV_BIAS_RELU || epilogue == PFB_ENC_CONV_BIAS_RELU_RESIDUAL,
                "enc_conv3x3: unknown epilogue %d", epilogue);
  PFB_CHECK_ARG(epilogue == PFB_ENC_CONV_LINEAR || bias, "enc_conv3x3: epilogue %d needs a bias", epilogue);
  PFB_CHECK_ARG(epilogue != PFB_ENC_CONV_BIAS_RELU_RESIDUAL || (residual && aligned16(residual)),
                "enc_conv3x3: the residual epilogue needs a 16-byte aligned residual [B,H,W,Cout]");
  PFB_CHECK_ARG(aligned16(x) && aligned16(weight_k) && aligned16(out), "enc_conv3x3: 16-byte alignment");
  PFB_CHECK_ARG(out_stride % 8 == 0 && out_offset % 8 == 0 && out_offset >= 0 && out_offset + Cout <= out_stride,
                "enc_conv3x3: out_stride / out_offset must be multiples of 8 with out_offset + Cout <= out_stride");
  EcPlan pl{};
  PFB_CHECK_ARG(plan_enc_conv(B, H, W, Cin, Cout, pl), "enc_conv3x3: unsupported shape B=%d H=%d W=%d Cin=%d Cout=%d", B, H, W, Cin, Cout);
  cudaStream_t s = as_stream(stream);
  const int Cin_pad = pl.chunks * 64, Cout_pad_k = (Cout + 31) / 32 * 32;  // ops.PackedConv's K-major packing
  CUtensorMap tmX, tmW, tmO, tmR;
  {
    uint64_t dims[4] = {(uint64_t)Cin, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)Cin * 2, (uint64_t)W * Cin * 2, (uint64_t)H * W * Cin * 2};
    uint32_t box[4] = {64, (uint32_t)kEcPatchBox, 1, 1};
    int rc = make_tensor_map(&tmX, x, dtype, 4, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[2] = {(uint64_t)Cin_pad, (uint64_t)9 * Cout_pad_k};
    uint64_t str[1] = {(uint64_t)Cin_pad * 2};
    uint32_t box[2] = {64, (uint32_t)(64 * pl.mb)};
    int rc = make_tensor_map(&tmW, weight_k, dtype, 2, dims, str, box);
    if (rc) return rc;
  }
  {
    uint64_t dims[4] = {(uint64_t)(out_offset + Cout), (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)out_stride * 2, (uint64_t)W * out_stride * 2, (uint64_t)H * W * out_stride * 2};
    uint32_t box[4] = {64, (uint32_t)kEcNW, 1, 1};
    int rc = make_tensor_map(&tmO, out, dtype, 4, dims, str, box);
    if (rc) return rc;
  }
  tmR = tmO;
  if (epilogue == PFB_ENC_CONV_BIAS_RELU_RESIDUAL) {
    uint64_t dims[4] = {(uint64_t)Cout, (uint64_t)W, (uint64_t)H, (uint64_t)B};
    uint64_t str[3] = {(uint64_t)Cout * 2, (uint64_t)W * Cout * 2, (uint64_t)H * W * Cout * 2};
    uint32_t box[4] = {64, (uint32_t)kEcNW, 1, 1};
    int rc = make_tensor_map(&tmR, residual, dtype, 4, dims, str, box);
    if (rc) return rc;
  }
  EncConvArgs a{};
  a.B = B; a.H = H; a.W = W; a.Cin = Cin; a.Cout = Cout; a.Cout_pad_k = Cout_pad_k;
  a.mb = pl.mb; a.TW = pl.TW; a.chunks = pl.chunks; a.tiles_x = pl.tiles_x; a.n_work = pl.n_work;
  a.a_stages = pl.a_stages; a.a_slot_bytes = pl.a_slot_bytes; a.w_stages = pl.w_stages; a.w_slot_bytes = pl.w_slot_bytes;
  a.w_resident = pl.w_resident;
  a.out_offset = out_offset;
  a.bias = bias;
  int grid = sm_count();
  if (grid > pl.n_work) grid = pl.n_work;
  ProfScope prof(KC_ENC_CONV1, s);  // the encoder-convolution class (bench.py's enc_conv1 field)
  if (dtype == PFB_F16) return launch_enc_conv<__half>(epilogue, tmX, tmW, tmO, tmR, a, grid, pl.smem, s);
  return launch_enc_conv<__nv_bfloat16>(epilogue, tmX, tmW, tmO, tmR, a, grid, pl.smem, s);
}
