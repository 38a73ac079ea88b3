// Implicit-GEMM convolution on the Hopper tensor cores (wgmma; f16 / bf16 storage, fp32 accumulate).
//
//   out[p, n] = epilogue( bias[n] + sum_{tap, src, c} X_src[p + tap, c] * Wk[tap][n][kpos(src, c)] )
//
//   M tile : 128 pixels = TW x TH of one image, chosen per shape for the least padding.  The A operand of a tap is a TMA
//            box of the pixel-major activation tensor: out-of-image elements are zero-filled by the TMA unit, which is
//            exactly "same" zero padding -- no im2col, no torch.cat (each concatenated source has its own tensor map).
//            Halo reuse: with row tiles one patch of TW + KW - 1 pixels serves all KW horizontal taps (tap kx = the same
//            patch read through a descriptor advanced by kx * 128 B); vertical kernels use (TH + KH - 1) x TW patches the
//            same way (advance TW * 128 B, a multiple of the 1024-byte swizzle period).
//   N tile : up to 128 output channels (equal tiles, multiples of 32): the two MMA warpgroups hold 64 x N fp32 each in
//            registers.
//   K loop : (64-channel chunk of a source, ky, kx).  Two rings: activation patches and weight tiles; a weight stage
//            holds one tap or all taps of a patch ("b_group").
//
// Persistent CTAs (one per SM) walk the output tiles round-robin.  The rings run continuously across tiles; at the end of
// a tile the MMA warpgroups park their fragments in a shared-memory accumulator tile and go on with the next tile while
// the epilogue warps read it.  The epilogue fuses bias + ReLU / sigmoid / tanh + the GRU gate arithmetic of
// ptlflow/models/raft/update.py:58-73 and writes pixel-major f16/bf16 with 16-byte stores; its h / z / residual
// operands are requested before the accumulator wait.  Launched with programmatic stream serialization: the
// prologue (barriers, bias, tensor-map prefetch) overlaps the previous kernel's drain (pdl_wait below).
// PFB_CONV_TRACE=<file> records a per-CTA timeline of every launch (tools/conv_trace_report.py).
#include <stdio.h>
#include <stdlib.h>

#include <atomic>
#include <type_traits>

#include "umma.cuh"

namespace pfb {
using namespace sm90;

constexpr int kATileBytes = 128 * 128;
constexpr int kMaxBias = 1024;  // output channels per layer whose bias is kept in shared memory (Cout_pad_k <= 1024)
constexpr int kMaxAStages = 8, kMaxBStages = 32;
// warp roles (conv_umma_kernel): epilogue warpgroup, two MMA warpgroups, producer warpgroup
constexpr int kEpilogueWarps = 4, kMmaWarp0 = 4, kProducerWarp = 12;

struct __align__(8) ConvBars {
  uint64_t a_full[kMaxAStages];
  uint64_t a_empty[kMaxAStages];
  uint64_t b_full[kMaxBStages];
  uint64_t b_empty[kMaxBStages];
  uint64_t acc_full;
  uint64_t acc_empty;
};

struct ConvUmmaArgs {
  int nsrc;
  int src_chunks[PFB_MAX_SRC];   // 64-channel chunks per source
  int src_coff[PFB_MAX_SRC];     // first channel inside the source tensor
  int B, H, W, KH, KW;
  int NT;                        // N tile (multiple of 32, <= 128)
  int n_tiles;                   // N tiles per M tile
  int TW, TH, tw_shift;          // M tile = TW x TH pixels (TW * TH = 128, powers of two)
  int tiles_x, tiles_y, n_work;  // work items = tiles_x * tiles_y * B * n_tiles
  int Cout, Cout_pad_k;
  // Two rings: activation patches (A) and weight tiles (B).  With row tiles (TH == 1, "halo" mode) one A patch of
  // TW + KW - 1 pixels serves all KW horizontal taps of a (chunk, ky): tap kx reads it through a descriptor whose
  // start address is advanced by kx pixel rows (128 B each) -- the swizzle is a function of the absolute shared-memory
  // address, so TMA writes and wgmma reads stay consistent.  Otherwise every tap loads its own patch.
  int halo;
  int a_stages, a_slot_bytes, a_tx_bytes, b_stages, b_slot_bytes;
  int b_group, b_tap_bytes;      // weight stage = b_group consecutive taps of one activation patch (1, or all of them)
  const float* bias;
  int epilogue;
  float scale;
  void* out;
  int out_stride, out_offset;
  const void* aux_h;
  void* aux_z;
  int hidden;
  const float* flow;
  int w_rows_per_sample;         // > 0: every sample b has its own weight matrix, rows [b * w_rows_per_sample, ...) of the weight map
  const void* addend;            // optional per-pixel pre-activation term [B*H*W][addend_stride] (storage type), added instead of the bias
  int addend_stride;
  const void* residual;          // PFB_EPI_RESIDUAL_GELU: residual operand [B*H*W][residual_stride] (storage type) from residual_offset
  int residual_stride, residual_offset;
  const float* post_w;           // PFB_EPI_RESIDUAL_GELU: optional per-channel second step gelu(y * (1 + post_w) + post_b)
  const float* post_b;
  int ab_fmt;
  int tma_out;                   // 1: outputs leave through shared-memory staging + TMA bulk stores (tmO0 = out, tmO1 = aux_z)
  unsigned long long* trace;     // debug timeline (PFB_CONV_TRACE): 32 clock64 slots per CTA, null in production
};

#define PFB_TR(slot) do { if (a.trace && lane == 0) a.trace[blockIdx.x * 32 + (slot)] = clock64(); } while (0)

// two fp32 -> one packed pair of the storage type: a single cvt.rn.{f16x2,bf16x2}.f32 (the epilogues convert 256 values per row)
template <typename T>
__device__ __forceinline__ uint32_t pack2(float a, float b);
template <>
__device__ __forceinline__ uint32_t pack2<__half>(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <>
__device__ __forceinline__ uint32_t pack2<__nv_bfloat16>(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
template <typename T>
__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  const T* h = reinterpret_cast<const T*>(&u);
#pragma unroll
  for (int i = 0; i < 8; ++i) f[i] = to_f32(h[i]);
}

// store 32 consecutive channels starting at element pointer dst (16-byte aligned), of which `valid` are real
template <typename T>
__device__ __forceinline__ void store32(T* dst, const float (&v)[32], int valid) {
  if (valid >= 32) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      uint4 u;
      u.x = pack2<T>(v[8 * q + 0], v[8 * q + 1]);
      u.y = pack2<T>(v[8 * q + 2], v[8 * q + 3]);
      u.z = pack2<T>(v[8 * q + 4], v[8 * q + 5]);
      u.w = pack2<T>(v[8 * q + 6], v[8 * q + 7]);
      reinterpret_cast<uint4*>(dst)[q] = u;
    }
  } else {
#pragma unroll
    for (int e = 0; e < 32; ++e)
      if (e < valid) dst[e] = from_f32<T>(v[e]);
  }
}
template <typename T>
__device__ __forceinline__ void load32(const T* src, float (&v)[32]) {
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 u = reinterpret_cast<const uint4*>(src)[q];
    float f[8];
    unpack8<T>(u, f);
#pragma unroll
    for (int i = 0; i < 8; ++i) v[8 * q + i] = f[i];
  }
}

// The MMA role: two warpgroups, rows 0-63 and 64-127 of the M tile, each m64nNT per 16-channel K step with the
// accumulator in registers.  A pipeline step (b_group taps x 4 K steps) is committed as one wgmma group and the next
// step is issued before it has completed; its ring slots are released once it has (so the role holds one step more of
// each ring than it computes on).  At the end of a tile the fragments go to the shared-memory accumulator tile
// (once the epilogue has released it), so the epilogue of tile i overlaps the MMAs of tile i + 1.
template <int NT, bool BF16, int G>
__device__ __forceinline__ void issue_taps(float (&d)[NT / 2], uint32_t a_lo, uint32_t a_tap16, uint32_t b_lo, uint32_t b_tap16, uint32_t acc) {
  // fence and commit in the MMAs' own basic block: ptxas injects warpgroup.arrive instructions of its own when they are outside it
  wgmma_fence();
#pragma unroll
  for (int g = 0; g < G; ++g) {
#pragma unroll
    for (int kk = 0; kk < 4; ++kk) {
      const uint32_t en = (g == 0 && kk == 0) ? acc : 1u;
      wgmma<NT, BF16>(d, gdesc(a_lo + g * a_tap16 + 2 * kk, kDescHiSw128), gdesc(b_lo + g * b_tap16 + 2 * kk, kDescHiSw128), en);
    }
  }
  wgmma_commit();
}

template <int NT, bool BF16>
__device__ __forceinline__ void conv_mma_role(const ConvUmmaArgs& a, ConvBars* bars, uint8_t* smemA, uint8_t* smemB, float* sacc,
                                              int chunks, int group0, int group_stride) {
  const int wg = (threadIdx.x >> 7) - kMmaWarp0 / 4, tid = threadIdx.x & 127, lane = threadIdx.x & 31;
  const uint32_t a_slot16 = (uint32_t)a.a_slot_bytes >> 4, b_slot16 = (uint32_t)a.b_slot_bytes >> 4;
  const uint32_t a_lo0 = gdesc_lo(smem_u32(smemA) + wg * 64 * 128, 16);  // this warpgroup's 64 pixel rows
  const uint32_t b_lo0 = gdesc_lo(smem_u32(smemB), 16);
  const uint32_t bar_a_full = smem_u32(&bars->a_full[0]);
  const uint32_t bar_b_full = smem_u32(&bars->b_full[0]);
  const int kw_halo = a.halo == 1 ? a.KW : (a.halo == 2 ? a.KH : 1);  // taps served by one activation patch
  const int groups = chunks * (a.halo == 1 ? a.KH : (a.halo == 2 ? 1 : a.KH * a.KW));  // patches per tile
  const uint32_t tap_step16 = a.halo == 2 ? (uint32_t)a.TW * 8u : 8u;  // descriptor advance per tap (16-B units)
  const uint32_t b_tap16 = (uint32_t)a.b_tap_bytes >> 4;
  int sa = 0, sb = 0, i = 0;
  uint32_t pha = 0, phb = 0;
  uint32_t a_lo = a_lo0, b_lo = b_lo0;
  // slots of the step still in flight: weight stage (-1: none) and activation slot (-1: the step does not finish its patch)
  int held_b = -1, held_a = -1;
  auto release_held = [&]() {
    __syncwarp();
    if (lane == 0 && held_b >= 0) {
      mbar_arrive(&bars->b_empty[held_b]);
      if (held_a >= 0) mbar_arrive(&bars->a_empty[held_a]);
    }
  };
  float d[NT / 2];
  for (int w = group0; w < a.n_work; w += group_stride, ++i) {
    uint32_t acc = 0;  // first MMA of the tile overwrites the accumulator
    for (int g = 0; g < groups; ++g) {
      mbar_wait_uniform(bar_a_full + 8 * sa, pha);
      for (int kx = 0; kx < kw_halo; kx += a.b_group) {
        mbar_wait_uniform(bar_b_full + 8 * sb, phb);
        const uint32_t al = a_lo + tap_step16 * kx;  // x halo: +1 pixel row (128 B) per tap; y halo: +TW rows
        switch (a.b_group) {
          case 5: issue_taps<NT, BF16, 5>(d, al, tap_step16, b_lo, b_tap16, acc); break;
          case 3: issue_taps<NT, BF16, 3>(d, al, tap_step16, b_lo, b_tap16, acc); break;
          default: issue_taps<NT, BF16, 1>(d, al, tap_step16, b_lo, b_tap16, acc); break;
        }
        // one group stays in flight: this step's MMAs queue behind the previous step's, whose slots are free once it has
        // completed
        wgmma_wait<1>();
        reg_fence(d);
        release_held();
        held_b = sb;
        held_a = kx + a.b_group >= kw_halo ? sa : -1;
        acc = 1;
        b_lo += b_slot16;
        if (++sb == a.b_stages) { sb = 0; phb ^= 1; b_lo = b_lo0; }
      }
      a_lo += a_slot16;
      if (++sa == a.a_stages) { sa = 0; pha ^= 1; a_lo = a_lo0; }
    }
    wgmma_wait<0>();
    reg_fence(d);
    release_held();
    held_b = -1;
    mbar_wait(&bars->acc_empty, (i & 1) ^ 1);
    acc_store<NT>(sacc, d, wg * 64, tid);
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars->acc_full);
  }
}

// Four warpgroups: warps 0-3 the epilogue (thread = pixel row, all NT columns), 4-11 the two MMA warpgroups, 12-15 the
// producer warpgroup (warp 12 issues the TMA loads; 13-15 only give their registers away).
// EPI (the pfb_epilogue) is a template parameter: with a run-time switch the register allocation of every epilogue was the
// union of all of them (h, z, addend and bias operands live together), and the staged-store version spilled.
constexpr int kConvThreads = 16 * 32;
// Register budget per role (setmaxnreg).  512 threads at one CTA per SM launch with 128 registers each: 65536 for the CTA.
// The producer warpgroup drops to 48 (at 40 its loop spills) and the epilogue takes what it frees; the MMA warpgroups keep
// 128 (they need 96 for NT = 128 without spilling).  The gate epilogues (GRU z|r and q, which hold h / z / addend operands
// one chunk ahead) need 168: with two epilogue warpgroups (640 threads, 96 registers each at launch) no split of the 61440
// registers gives them that next to the MMA and producer warpgroups, hence one epilogue warpgroup.
constexpr int kProducerRegs = 48, kEpilogueRegs = 208, kMmaRegs = 128;
static_assert(128 * (kProducerRegs + kEpilogueRegs + 2 * kMmaRegs) <= 65536, "register budget exceeds the register file");
template <typename T, int EPI>
__global__ void __launch_bounds__(kConvThreads, 1)
conv_umma_kernel(const __grid_constant__ CUtensorMap tm0, const __grid_constant__ CUtensorMap tm1,
                 const __grid_constant__ CUtensorMap tm2, const __grid_constant__ CUtensorMap tmW,
                 const __grid_constant__ CUtensorMap tmO0, const __grid_constant__ CUtensorMap tmO1, const ConvUmmaArgs a) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  // only the plain epilogues stage their outputs (compile-time: the gate instantiations carry none of the staging state)
  constexpr bool kPlain = EPI == PFB_EPI_LINEAR || EPI == PFB_EPI_RELU || EPI == PFB_EPI_RELU_APPEND_FLOW || EPI == PFB_EPI_GELU ||
                          EPI == PFB_EPI_LINEAR_APPEND_FLOW;
  const bool tma_out = kPlain && a.tma_out;
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* smemA = smem;
  uint8_t* smemB = smem + a.a_stages * a.a_slot_bytes;
  // output staging: [128 pixels][64 channels] (16 KB), 128-byte swizzled like an operand tile.  The epilogue's thread <-> pixel
  // mapping makes every direct global access a 16-byte piece per lane at a 256..768-byte stride; staged, the stores are
  // conflict-free 16-byte shared-memory writes and the global side is the TMA unit writing whole 128-byte rows.
  uint8_t* smemO = smemB + a.b_stages * a.b_slot_bytes;
  float* sacc = reinterpret_cast<float*>(smemO + (tma_out ? kATileBytes : 0));  // fp32 accumulator tile, NT columns
  float* sbias = sacc + a.NT * kAccPitch;  // n_tiles * NT <= kMaxBias floats
  ConvBars* bars = reinterpret_cast<ConvBars*>(reinterpret_cast<uint8_t*>(sbias) + kMaxBias * sizeof(float));

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (a.trace && threadIdx.x == 0) {
    a.trace[blockIdx.x * 32 + 0] = global_timer_ns();
    a.trace[blockIdx.x * 32 + 1] = clock64();
  }
  int chunks = 0;
  for (int s = 0; s < a.nsrc; ++s) chunks += a.src_chunks[s];
  const int tiles_m = a.tiles_x * a.tiles_y * a.B;
  const int group0 = blockIdx.x, group_stride = gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < a.a_stages; ++s) {
      mbar_init(&bars->a_full[s], 1);
      mbar_init(&bars->a_empty[s], 8);  // one arrival per MMA warp
    }
    for (int s = 0; s < a.b_stages; ++s) {
      mbar_init(&bars->b_full[s], 1);
      mbar_init(&bars->b_empty[s], 8);
    }
    mbar_init(&bars->acc_full, 8);
    mbar_init(&bars->acc_empty, kEpilogueWarps);  // one arrival per epilogue warp
    fence_barrier_init();
  }
  // the bias vector is read by every epilogue thread for every 32-column chunk: one copy in shared memory instead of 8
  // dependent global loads per chunk
  for (int k = threadIdx.x; k < a.n_tiles * a.NT && k < kMaxBias; k += blockDim.x) sbias[k] = a.bias ? a.bias[k] : 0.f;
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tm0);
    prefetch_tmap(&tmW);
    if (tma_out) prefetch_tmap(&tmO0);
  }
  __syncthreads();
  // PDL: everything above (barriers, bias, tensor-map prefetch) overlapped the previous kernel's drain
  pdl_wait();
  pdl_trigger();
  if (warp == 0) PFB_TR(2);

  // work item j -> (n tile, image, tile row, tile col) of THIS CTA; n-tile major so concurrent CTAs share the weight
  // tile in L2
  auto decode = [&](int j, int& n0, int& b, int& y0, int& x0) {
    const int nt = j / tiles_m;
    int m = j - nt * tiles_m;
    const int px = m % a.tiles_x;
    m /= a.tiles_x;
    const int py = m % a.tiles_y;
    b = m / a.tiles_y;
    n0 = nt * a.NT;
    y0 = py * a.TH;
    x0 = px * a.TW;
  };

  if (warp >= kProducerWarp) {
    setmaxnreg_dec<kProducerRegs>();
    if (warp == kProducerWarp) {
      // ================= TMA producer (warp-uniform loop, one elected lane issues) =================
      const int ph2 = a.KH >> 1, pw2 = a.KW >> 1;
      const uint32_t btx = a.NT * 128;  // bytes of one weight tap
      // ring positions advance incrementally (stage index + phase bit): no integer division on the issue path
      int sta = 0, stb = 0, bg = 0;
      uint32_t pha = 0, phb = 0;
      PFB_TR(3);
      for (int w = group0; w < a.n_work; w += group_stride) {
        int n0, b, y0, x0;
        decode(w, n0, b, y0, x0);
        int kidx = 0;
        const int wrow0 = b * a.w_rows_per_sample;  // per-sample weights (GMA aggregate: the sample's v^T)
        for (int s = 0; s < a.nsrc; ++s) {
          const CUtensorMap* tm = s == 0 ? &tm0 : (s == 1 ? &tm1 : &tm2);
          for (int c = 0; c < a.src_chunks[s]; ++c, ++kidx) {
            int wrow = wrow0;  // + (ky * KW + kx) * Cout_pad_k
            for (int ky = 0; ky < a.KH; ++ky) {
              for (int kx = 0; kx < a.KW; ++kx) {
                // activation patch: once per (chunk, ky) with the x halo, once per chunk with the y halo, else per tap
                if (a.halo == 0 || (a.halo == 1 && kx == 0) || (a.halo == 2 && ky == 0)) {
                  mbar_wait(&bars->a_empty[sta], pha ^ 1);
                  if (elect_one()) {
                    mbar_arrive_expect_tx(&bars->a_full[sta], a.a_tx_bytes);
                    tma_load_4d(smemA + sta * a.a_slot_bytes, tm, &bars->a_full[sta], a.src_coff[s] + c * 64,
                                x0 - pw2 + (a.halo ? 0 : kx), y0 + ky - ph2, b);
                  }
                  __syncwarp();
                  if (++sta == a.a_stages) { sta = 0; pha ^= 1; }
                }
                // weight stage: b_group consecutive taps of this patch share one barrier (fewer, larger pipeline steps)
                if (bg == 0) mbar_wait(&bars->b_empty[stb], phb ^ 1);
                if (elect_one()) {
                  if (bg == 0) mbar_arrive_expect_tx(&bars->b_full[stb], btx * a.b_group);
                  tma_load_2d(smemB + stb * a.b_slot_bytes + bg * a.b_tap_bytes, &tmW, &bars->b_full[stb], kidx * 64, wrow + n0);
                }
                __syncwarp();
                wrow += a.Cout_pad_k;
                if (++bg == a.b_group) {
                  bg = 0;
                  if (++stb == a.b_stages) { stb = 0; phb ^= 1; }
                }
              }
            }
          }
        }
      }
      PFB_TR(4);
    }
  } else if (warp >= kMmaWarp0) {
    // ================= MMA warpgroups (kMmaRegs: the launch budget) =================
    switch (a.NT) {
      case 32: conv_mma_role<32, std::is_same<T, __nv_bfloat16>::value>(a, bars, smemA, smemB, sacc, chunks, group0, group_stride); break;
      case 64: conv_mma_role<64, std::is_same<T, __nv_bfloat16>::value>(a, bars, smemA, smemB, sacc, chunks, group0, group_stride); break;
      case 96: conv_mma_role<96, std::is_same<T, __nv_bfloat16>::value>(a, bars, smemA, smemB, sacc, chunks, group0, group_stride); break;
      default: conv_mma_role<128, std::is_same<T, __nv_bfloat16>::value>(a, bars, smemA, smemB, sacc, chunks, group0, group_stride); break;
    }
  } else {
    setmaxnreg_inc<kEpilogueRegs>();
    // ================= epilogue: thread <-> pixel, 32 output channels at a time =================
    const int row = warp * 32 + lane;
    const int hd = a.hidden;
    int i = 0;
    for (int w = group0; w < a.n_work; w += group_stride, ++i) {
      int n0, b, y0, x0;
      decode(w, n0, b, y0, x0);
      const int y = y0 + (row >> a.tw_shift), x = x0 + (row & (a.TW - 1));
      const bool ok = (y < a.H) && (x < a.W) && (b < a.B);
      const size_t p = ((size_t)b * a.H + (ok ? y : 0)) * a.W + (ok ? x : 0);
      // Operands that do not depend on the accumulator (h, z, residual) are requested BEFORE waiting for the MMAs
      // of this tile, and the next chunk's while the current one is processed (exposed L2 latency otherwise makes the
      // GRU layers epilogue-bound).
      const bool aux_h_any = EPI == PFB_EPI_GRU_ZR || EPI == PFB_EPI_GRU_Q || EPI == PFB_EPI_AXPY || EPI == PFB_EPI_RESIDUAL_GELU;
      auto issue_h = [&](int c, uint4 (&hq)[4]) {
        const int n = n0 + c;
        const bool need_h = ok && ((EPI == PFB_EPI_GRU_ZR && n >= hd) || EPI == PFB_EPI_GRU_Q || ((EPI == PFB_EPI_AXPY || EPI == PFB_EPI_RESIDUAL_GELU) && n + 32 <= a.Cout));
        if (need_h) {
          const T* hp = EPI == PFB_EPI_RESIDUAL_GELU
                            ? reinterpret_cast<const T*>(a.residual) + p * a.residual_stride + a.residual_offset + n
                            : reinterpret_cast<const T*>(a.aux_h) + p * hd + (EPI == PFB_EPI_GRU_ZR ? n - hd : n);
#pragma unroll
          for (int q = 0; q < 4; ++q) hq[q] = reinterpret_cast<const uint4*>(hp)[q];
        }
      };
      auto issue_z = [&](int c, uint4 (&zq)[4]) {
        if (ok && EPI == PFB_EPI_GRU_Q) {
          const T* zp = reinterpret_cast<const T*>(a.aux_z) + p * hd + n0 + c;
#pragma unroll
          for (int q = 0; q < 4; ++q) zq[q] = reinterpret_cast<const uint4*>(zp)[q];
        }
      };
      // per-pixel addend (the iteration-invariant context part of the GRU gates, computed once per forward and carrying the
      // bias): requested one chunk ahead like h / z
      const T* addp = a.addend ? reinterpret_cast<const T*>(a.addend) + p * a.addend_stride + n0 : nullptr;
      auto issue_add = [&](int c, uint4 (&aq)[4]) {
        if (ok && addp) {
#pragma unroll
          for (int q = 0; q < 4; ++q) aq[q] = reinterpret_cast<const uint4*>(addp + c)[q];
        }
      };
      uint4 hnext[4], znext[4], anext[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) hnext[q] = znext[q] = anext[q] = make_uint4(0u, 0u, 0u, 0u);
      // Operand prefetch.  Plain epilogues: the next chunk's accumulator / residual is requested as soon as the current chunk
      // has been moved out of r[] ("early").  Gate epilogues (z|r, q, axpy) also hold h / z / addend: they request the next
      // chunk's operands only AFTER the current chunk has been packed ("late"), when its registers are dead -- the loads then
      // fly under the staging barriers and the TMA issue.  That keeps every instantiation inside its register budget
      // without spills and without exposing the L2 latency per chunk (in-place loads cost +2..6 us per gate launch, r02e).
      // Measured (launch lists r02c / r02e / r02f): the staged stores win on the plain epilogues (convc1 27.7 -> 20.8 us, flow
      // head 35.1 -> 29.4 us) but lose on the gate epilogues, whose warps are unevenly loaded (r half vs z half) and meet at two
      // barriers per 64-column block: z|r 41.7 -> 45.0 us, q 40.0 -> 49.2 us.  The host therefore stages only plain epilogues
      // (conv2d_umma: tma_out), and the gates keep direct stores with everything requested one chunk ahead.
      constexpr bool kLate = false;
      if (aux_h_any) issue_h(0, hnext);
      issue_z(0, znext);
      issue_add(0, anext);
      mbar_wait(&bars->acc_full, i & 1);
      if (warp == 0 && i < 3) PFB_TR(12 + i);
      // accumulator reads are software-pipelined too: chunk c + 32 is loaded as soon as chunk c has been moved to v[]
      uint32_t r[32];
      acc_ld32(sacc, row, 0, r);
      // 32 packed values -> half `half` of this thread's pixel's 128-byte row in the staging buffer
      auto stage32 = [&](const uint4 (&pk)[4], int half) {
        uint8_t* sb = smemO + row * 128;
#pragma unroll
        for (int q = 0; q < 4; ++q) *reinterpret_cast<uint4*>(sb + (((half * 4 + q) ^ (row & 7)) << 4)) = pk[q];
      };
      for (int c = 0; c < a.NT; c += 32) {
       uint4 pk[4];  // the chunk's 32 results, converted: what stays live across the staging barrier
       {
        float v[32];
        const int n = n0 + c;  // first output channel of this chunk
        uint4 hraw[4], zraw[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { hraw[q] = hnext[q]; zraw[q] = znext[q]; }
        if (addp) {  // warp-uniform: per-pixel addend instead of the per-channel bias
          uint4 araw[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) araw[q] = anext[q];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            float f[8];
            unpack8<T>(araw[q], f);
#pragma unroll
            for (int e = 0; e < 8; ++e) v[8 * q + e] = __uint_as_float(r[8 * q + e]) + f[e];
          }
        } else {
          float4 bb[8];
#pragma unroll
          for (int q = 0; q < 8; ++q) bb[q] = reinterpret_cast<const float4*>(sbias + n)[q];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
            v[4 * q + 0] = __uint_as_float(r[4 * q + 0]) + bb[q].x;
            v[4 * q + 1] = __uint_as_float(r[4 * q + 1]) + bb[q].y;
            v[4 * q + 2] = __uint_as_float(r[4 * q + 2]) + bb[q].z;
            v[4 * q + 3] = __uint_as_float(r[4 * q + 3]) + bb[q].w;
          }
        }
        if (!kLate && c + 32 < a.NT) {  // warp-uniform
          acc_ld32(sacc, row, c + 32, r);
          if (aux_h_any) issue_h(c + 32, hnext);
          issue_z(c + 32, znext);
          issue_add(c + 32, anext);
        }
        if (ok || tma_out) {  // (staged rows of out-of-image pixels are clipped by the TMA unit)
        T* out = reinterpret_cast<T*>(a.out);
        switch (EPI) {
          case PFB_EPI_LINEAR: {
#pragma unroll
            for (int e = 0; e < 32; ++e) v[e] *= a.scale;
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, a.Cout - n);
            break;
          }
          case PFB_EPI_RELU: {
#pragma unroll
            for (int e = 0; e < 32; ++e) v[e] = fmaxf(v[e], 0.f);
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, a.Cout - n);
            break;
          }
          case PFB_EPI_LINEAR_F32: {  // fp32 output (16-byte aligned rows: out_stride % 4 == 0)
            float* o32 = reinterpret_cast<float*>(a.out) + p * a.out_stride + a.out_offset + n;
            const int valid = a.Cout - n;
#pragma unroll
            for (int q = 0; q < 8; ++q)
              if (4 * q + 4 <= valid)
                reinterpret_cast<float4*>(o32)[q] = make_float4(v[4 * q] * a.scale, v[4 * q + 1] * a.scale, v[4 * q + 2] * a.scale, v[4 * q + 3] * a.scale);
              else
                for (int e = 4 * q; e < 4 * q + 4; ++e)
                  if (e < valid) o32[e] = v[e] * a.scale;
            break;
          }
          case PFB_EPI_AXPY: {  // residual + scale * acc   (residual = aux_h[p * hidden + n])
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float h[8];
              unpack8<T>(hraw[q], h);
#pragma unroll
              for (int e = 0; e < 8; ++e) v[8 * q + e] = h[e] + a.scale * v[8 * q + e];
            }
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, a.Cout - n);
            break;
          }
          case PFB_EPI_GELU: {
#pragma unroll
            for (int e = 0; e < 32; ++e) v[e] = gelu_f32(v[e]);
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, a.Cout - n);
            break;
          }
          case PFB_EPI_RESIDUAL_GELU: {  // gelu(residual + acc + bias) (+ the optional per-channel step)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float h[8];
              unpack8<T>(hraw[q], h);
#pragma unroll
              for (int e = 0; e < 8; ++e) v[8 * q + e] = gelu_f32(h[e] + v[8 * q + e]);
            }
            if (a.post_w) {  // warp-uniform
#pragma unroll
              for (int q = 0; q < 8; ++q) {
                const float4 w4 = __ldg(reinterpret_cast<const float4*>(a.post_w + n) + q);
                const float4 b4 = __ldg(reinterpret_cast<const float4*>(a.post_b + n) + q);
                v[4 * q + 0] = gelu_f32(fmaf(v[4 * q + 0], 1.f + w4.x, b4.x));
                v[4 * q + 1] = gelu_f32(fmaf(v[4 * q + 1], 1.f + w4.y, b4.y));
                v[4 * q + 2] = gelu_f32(fmaf(v[4 * q + 2], 1.f + w4.z, b4.z));
                v[4 * q + 3] = gelu_f32(fmaf(v[4 * q + 3], 1.f + w4.w, b4.w));
              }
            }
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, a.Cout - n);
            break;
          }
          case PFB_EPI_RELU_APPEND_FLOW:
          case PFB_EPI_LINEAR_APPEND_FLOW: {
            if (EPI == PFB_EPI_RELU_APPEND_FLOW) {
#pragma unroll
              for (int e = 0; e < 32; ++e) v[e] = fmaxf(v[e], 0.f);
            }
            int valid = a.Cout - n;
            if (valid > 0 && valid <= 30) {  // the chunk that holds the last real channel also takes the 2 flow columns
              const float fx = a.flow[2 * p], fy = a.flow[2 * p + 1];
#pragma unroll
              for (int e = 0; e < 32; ++e) {
                if (e == valid) v[e] = fx;
                if (e == valid + 1) v[e] = fy;
              }
              valid += 2;
            }
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, valid);
            break;
          }
          case PFB_EPI_GRU_ZR: {
#pragma unroll
            for (int e = 0; e < 32; ++e) v[e] = __fdividef(1.f, 1.f + __expf(-v[e]));  // sigmoid: 2 MUFU ops
            if (n < hd) {
              if (!tma_out) store32<T>(reinterpret_cast<T*>(a.aux_z) + p * hd + n, v, 32);
            } else {
#pragma unroll
              for (int q = 0; q < 4; ++q) {
                float h[8];
                unpack8<T>(hraw[q], h);
#pragma unroll
                for (int e = 0; e < 8; ++e) v[8 * q + e] *= h[e];
              }
              if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + (n - hd), v, 32);
            }
            break;
          }
          case PFB_EPI_GRU_Q: {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              float h[8], z[8];
              unpack8<T>(hraw[q], h);
              unpack8<T>(zraw[q], z);
#pragma unroll
              for (int e = 0; e < 8; ++e) {
                // tanh(x) = 1 - 2 / (1 + exp(2x)): two MUFU ops, ~1e-7 absolute error, saturates cleanly
                const float th = 1.f - __fdividef(2.f, 1.f + __expf(2.f * v[8 * q + e]));
                v[8 * q + e] = (1.f - z[e]) * h[e] + z[e] * th;
              }
            }
            if (!tma_out) store32<T>(out + p * a.out_stride + a.out_offset + n, v, 32);
            break;
          }
          default:
            break;
        }
        }
        if (tma_out) {
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            pk[q].x = pack2<T>(v[8 * q + 0], v[8 * q + 1]);
            pk[q].y = pack2<T>(v[8 * q + 2], v[8 * q + 3]);
            pk[q].z = pack2<T>(v[8 * q + 4], v[8 * q + 5]);
            pk[q].w = pack2<T>(v[8 * q + 6], v[8 * q + 7]);
          }
        }
        if (kLate && c + 32 < a.NT) {  // warp-uniform
          acc_ld32(sacc, row, c + 32, r);
          if (aux_h_any) issue_h(c + 32, hnext);
          issue_z(c + 32, znext);
          issue_add(c + 32, anext);
        }
       }
       if (tma_out) {
         // One 64-column block (two chunks) leaves as one bulk store (single staging buffer: the previous block's store has
         // had this chunk's arithmetic to drain; thread 0 confirms it before anybody overwrites the buffer).
         if ((c & 32) == 0) {
           if (threadIdx.x == 0) tma_store_wait_read();
           named_barrier_sync(1, 32 * kEpilogueWarps);
         }
         stage32(pk, (c >> 5) & 1);
         if ((c & 32) != 0 || c + 32 >= a.NT) {
          fence_proxy_async();
          named_barrier_sync(1, 32 * kEpilogueWarps);
          if (threadIdx.x == 0) {
           const int nb = n0 + (c & ~63);
           if (EPI == PFB_EPI_GRU_ZR && nb < hd) tma_store_4d(&tmO1, smemO, nb, x0, y0, b);
           else tma_store_4d(&tmO0, smemO, a.out_offset + (EPI == PFB_EPI_GRU_ZR ? nb - hd : nb), x0, y0, b);
           tma_store_commit();
          }
         }
       }
      }
      __syncwarp();
      if (warp == 0 && i < 3) PFB_TR(15 + i);
      if (warp == kEpilogueWarps - 1 && i < 3) PFB_TR(21 + i);
      if (lane == 0) mbar_arrive(&bars->acc_empty);
    }
  }
  if (tma_out && threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores complete (not only read)
  __syncthreads();
  if (warp == 0) PFB_TR(18);
  if (a.trace && threadIdx.x == 0) a.trace[blockIdx.x * 32 + 20] = global_timer_ns();
}

// ------------------------------------------------------------------------------------------------
static int eff_channels(const pfb_conv_src& s) { return (int)align_up((size_t)s.channels, 64); }

// N tiling: the fewest equal tiles of <= 128 columns that are multiples of 32 (epilogue chunk); 0 if there is none
static int conv_n_tiles(int cout_pad) {
  for (int n = ceil_div(cout_pad, 128); n <= cout_pad / 32; ++n)
    if (cout_pad % n == 0 && (cout_pad / n) % 32 == 0) return n;
  return 0;
}

static bool aligned16(const void* ptr) { return (reinterpret_cast<uintptr_t>(ptr) & 15) == 0; }

static bool plan_conv_umma(const pfb_conv_params* p, ConvUmmaArgs& a);

bool conv2d_umma_supported(const pfb_conv_params* p) {
  if (p->dtype != PFB_F16 && p->dtype != PFB_BF16) return false;
  if (!p->weight_k || p->Cout_pad_k < 16 || p->Cout_pad_k % 16 || p->Cout_pad_k > kMaxBias) return false;
  // the epilogue writes out (and reads / writes aux_h, aux_z below) 16 bytes at a time; the weight tensor map needs an
  // aligned base
  if (!aligned16(p->out) || !aligned16(p->weight_k)) return false;
  if (p->nsrc > 3) return false;
  int cin_pad = 0;
  for (int i = 0; i < p->nsrc; ++i) {
    const pfb_conv_src& s = p->src[i];
    if (s.is_f32) return false;
    if (s.offset % 8 || s.stride % 8) return false;  // 16-byte aligned channel vectors / TMA strides
    if ((reinterpret_cast<uintptr_t>(s.ptr) & 15) != 0) return false;
    cin_pad += eff_channels(s);
  }
  if (cin_pad != p->Cin_pad) return false;
  switch (p->epilogue) {
    case PFB_EPI_LINEAR: case PFB_EPI_RELU: case PFB_EPI_GELU: break;
    case PFB_EPI_RELU_APPEND_FLOW: case PFB_EPI_LINEAR_APPEND_FLOW:
      // the two flow columns go into the 32-column chunk that holds the last real channel, after it
      if (p->Cout % 32 == 0 || p->Cout % 32 == 31) return false;
      break;
    case PFB_EPI_RESIDUAL_GELU:
      if (!p->residual || p->residual_stride % 8 || p->residual_offset % 8 || p->Cout % 32 ||
          (reinterpret_cast<uintptr_t>(p->residual) & 15))
        return false;
      if (p->post_w && ((reinterpret_cast<uintptr_t>(p->post_w) & 15) || (reinterpret_cast<uintptr_t>(p->post_b) & 15))) return false;
      break;
    case PFB_EPI_LINEAR_F32:
      if (p->out_stride % 4 || p->out_offset % 4) return false;
      break;
    case PFB_EPI_AXPY:
      if (!p->aux_h || !aligned16(p->aux_h) || p->hidden % 8 || p->Cout % 32) return false;
      break;
    case PFB_EPI_GRU_ZR:
      if (p->hidden % 32 || p->Cout_pad_k != 2 * p->hidden || p->Cout_pad_k > 256) return false;
      if (!aligned16(p->aux_h) || !aligned16(p->aux_z)) return false;
      break;
    case PFB_EPI_GRU_Q:
      if (p->hidden % 32 || p->Cout_pad_k != p->hidden) return false;
      if (!aligned16(p->aux_h) || !aligned16(p->aux_z)) return false;
      break;
    default: return false;
  }
  if (p->out_stride % 8 || p->out_offset % 8) return false;
  if (p->w_rows_per_sample && (p->KH != 1 || p->KW != 1 || p->w_rows_per_sample < p->Cout_pad_k)) return false;
  if (p->addend && (p->addend_stride % 8 || (reinterpret_cast<uintptr_t>(p->addend) & 15) || p->addend_stride < p->Cout_pad_k)) return false;
  ConvUmmaArgs a{};
  return plan_conv_umma(p, a);
}

template <typename T, int EPI>
static int launch_conv_umma_e(const CUtensorMap* tms, const CUtensorMap& tmW, const CUtensorMap* tmO, const ConvUmmaArgs& a, int grid,
                              size_t smem, cudaStream_t s) {
  // once per (instantiation, device): correct when one process drives several devices, and off the per-launch path
  static std::atomic<unsigned long long> attr_done{0};
  int dev = 0;
  PFB_CUDA(cudaGetDevice(&dev));
  if (!(attr_done.load(std::memory_order_acquire) & (1ull << (dev & 63)))) {
    PFB_CUDA(cudaFuncSetAttribute(conv_umma_kernel<T, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_done.fetch_or(1ull << (dev & 63), std::memory_order_release);
  }
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(kConvThreads);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = s;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = pdl_enabled();
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  PFB_CUDA(cudaLaunchKernelEx(&cfg, conv_umma_kernel<T, EPI>, tms[0], tms[1], tms[2], tmW, tmO[0], tmO[1], a));
  return PFB_OK;
}

template <typename T>
static int launch_conv_umma(const CUtensorMap* tms, const CUtensorMap& tmW, const CUtensorMap* tmO, const ConvUmmaArgs& a, int grid,
                            size_t smem, cudaStream_t s) {
  switch (a.epilogue) {
    case PFB_EPI_LINEAR: return launch_conv_umma_e<T, PFB_EPI_LINEAR>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_RELU: return launch_conv_umma_e<T, PFB_EPI_RELU>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_GRU_ZR: return launch_conv_umma_e<T, PFB_EPI_GRU_ZR>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_GRU_Q: return launch_conv_umma_e<T, PFB_EPI_GRU_Q>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_RELU_APPEND_FLOW: return launch_conv_umma_e<T, PFB_EPI_RELU_APPEND_FLOW>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_AXPY: return launch_conv_umma_e<T, PFB_EPI_AXPY>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_LINEAR_F32: return launch_conv_umma_e<T, PFB_EPI_LINEAR_F32>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_GELU: return launch_conv_umma_e<T, PFB_EPI_GELU>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_RESIDUAL_GELU: return launch_conv_umma_e<T, PFB_EPI_RESIDUAL_GELU>(tms, tmW, tmO, a, grid, smem, s);
    case PFB_EPI_LINEAR_APPEND_FLOW: return launch_conv_umma_e<T, PFB_EPI_LINEAR_APPEND_FLOW>(tms, tmW, tmO, a, grid, smem, s);
    default: break;
  }
  set_error("conv_umma: epilogue %d has no tensor-core instantiation", a.epilogue);
  return PFB_ERR_UNSUPPORTED;
}

// M tile shape: TW x TH = 128 with the least padded area (ties -> the wider tile: fewer, longer TMA rows)
static void pick_tile(int H, int W, int& TW, int& TH) {
  long best = -1;
  for (int tw = 128; tw >= 8; tw >>= 1) {
    const int th = 128 / tw;
    const long area = (long)ceil_div(W, tw) * tw * ceil_div(H, th) * th;
    if (best < 0 || area < best) { best = area; TW = tw; TH = th; }
  }
}

// The activation patch of the M tile in `a` (TW, TH, halo) and the rings around it: b_group, a_stages, b_stages.  False when
// not even two stages of each ring fit next to each other.
static bool plan_rings(const pfb_conv_params* p, ConvUmmaArgs& a, int ring_budget) {
  const int patch_w = a.TW + (a.halo == 1 ? p->KW - 1 : 0);
  const int patch_h = a.TH + (a.halo == 2 ? p->KH - 1 : 0);
  a.a_tx_bytes = patch_w * patch_h * 128;
  a.a_slot_bytes = (int)align_up((size_t)a.a_tx_bytes, 1024);
  const int taps_per_patch = a.halo == 1 ? p->KW : (a.halo == 2 ? p->KH : 1);
  {
    static const int env_group = getenv("PFB_CONV_TAP_GROUP") ? atoi(getenv("PFB_CONV_TAP_GROUP")) : 1;
    a.b_group = 1;
    // all taps of a patch in one weight stage when at least 3 such stages fit next to 3 activation patches
    if (env_group && (taps_per_patch == 3 || taps_per_patch == 5) && 3 * taps_per_patch * a.b_tap_bytes + 3 * a.a_slot_bytes <= ring_budget)
      a.b_group = taps_per_patch;
  }
  a.b_slot_bytes = a.b_group * a.b_tap_bytes;
  // Split the rest between the rings.  A slot is reused only once per round trip (release -> producer wake-up -> TMA ->
  // MMA), so the number of K steps in flight, not the bytes, sets the pace of the small-N layers: maximise min(steps
  // covered by the activation ring, weight stages).  The MMA warpgroups hold the stage of the step in flight on top of
  // the one they issue from, so one stage of each ring counts as consumed: 2 weight stages (the least that does not
  // deadlock) leave the producer no lead and are chosen only where the activation patches leave room for no more.
  int best = -1;
  for (int as = 2; as <= kMaxAStages; ++as) {
    int bs = (ring_budget - as * a.a_slot_bytes) / a.b_slot_bytes;
    if (bs > kMaxBStages) bs = kMaxBStages;
    if (bs < 2) continue;
    const int cover_a = (as - 1) * taps_per_patch, cover_b = (bs - 1) * a.b_group;
    const int cover = cover_a < cover_b ? cover_a : cover_b;
    if (cover > best || (cover == best && bs > a.b_stages)) { best = cover; a.a_stages = as; a.b_stages = bs; }
  }
  return best >= 0;
}

// Everything about a launch but its operands: N tiling, output staging, M tile, halo mode, rings and work items.
// conv2d_umma_supported and conv2d_umma both call it, so every shape the predicate accepts can be launched.  The M tiles are
// tried in order of preference until the rings fit: for vertical kernels the vertical-halo tiles (fewest tiles first, then
// the smallest patch), whose patches of TH + KH - 1 rows can leave no room for two weight stages on short or wide grids;
// then the generic tile, with the horizontal halo where it applies and without any halo (one 16 KB patch per tap, which
// always fits).
static bool plan_conv_umma(const pfb_conv_params* p, ConvUmmaArgs& a) {
  a.n_tiles = conv_n_tiles(p->Cout_pad_k);
  if (a.n_tiles == 0) return false;
  a.NT = p->Cout_pad_k / a.n_tiles;
  a.b_tap_bytes = a.NT * 128;
  {
    static const int env_tma_out = getenv("PFB_CONV_TMA_STORE") ? atoi(getenv("PFB_CONV_TMA_STORE")) : 1;
    const bool plain = p->epilogue == PFB_EPI_LINEAR || p->epilogue == PFB_EPI_RELU || p->epilogue == PFB_EPI_RELU_APPEND_FLOW ||
                       p->epilogue == PFB_EPI_GELU || p->epilogue == PFB_EPI_LINEAR_APPEND_FLOW;
    // a staged store writes whole 64-channel blocks: with several N tiles of NT % 64 == 32 the last block of a tile would
    // overwrite the first 32 channels of the next one (a single tile is clipped at the layer's last channel by the tensor map)
    a.tma_out = env_tma_out && plain && aligned16(p->out) && (a.NT % 64 == 0 || a.n_tiles == 1);
  }
  // 227 KB less the accumulator tile, the output staging, the bias, the barriers and the alignment slack
  const int ring_budget = 227 * 1024 - acc_tile_bytes(a.NT) - (a.tma_out ? kATileBytes : 0) - kMaxBias * (int)sizeof(float) -
                          (int)sizeof(ConvBars) - 1024;
  static const int env_halo = getenv("PFB_CONV_HALO") ? atoi(getenv("PFB_CONV_HALO")) : 1;
  static const int env_vhalo = getenv("PFB_CONV_VHALO") ? atoi(getenv("PFB_CONV_VHALO")) : 1;
  int cand_tw[6], cand_th[6], cand_halo[6], nc = 0;
  if (env_vhalo && p->KW == 1 && p->KH > 1) {
    // vertical taps: a (TH + KH - 1) x TW patch serves all KH taps of a chunk when the per-tap offset TW * 128 B keeps
    // the 1024-byte swizzle phase (TW % 8 == 0).  Insertion by (tiles, patch); equal keys keep the wider tile first.
    long tiles[4], patch[4];
    for (int tw = 64; tw >= 8; tw >>= 1) {
      const int th = 128 / tw;
      const long t = (long)ceil_div(p->W, tw) * ceil_div(p->H, th), pt = (long)(th + p->KH - 1) * tw;
      int i = nc++;
      for (; i > 0 && (t < tiles[i - 1] || (t == tiles[i - 1] && pt < patch[i - 1])); --i) {
        tiles[i] = tiles[i - 1]; patch[i] = patch[i - 1]; cand_tw[i] = cand_tw[i - 1]; cand_th[i] = cand_th[i - 1];
      }
      tiles[i] = t; patch[i] = pt; cand_tw[i] = tw; cand_th[i] = th;
    }
    for (int i = 0; i < nc; ++i) cand_halo[i] = 2;
  }
  int TW = 128, TH = 1;
  pick_tile(p->H, p->W, TW, TH);
  const int hx = (env_halo && TH == 1 && p->KW > 1) ? 1 : 0;
  cand_tw[nc] = TW; cand_th[nc] = TH; cand_halo[nc++] = hx;
  if (hx) { cand_tw[nc] = TW; cand_th[nc] = TH; cand_halo[nc++] = 0; }
  for (int i = 0; i < nc; ++i) {
    a.TW = cand_tw[i]; a.TH = cand_th[i]; a.halo = cand_halo[i];
    if (!plan_rings(p, a, ring_budget)) continue;
    a.tw_shift = 0;
    while ((1 << a.tw_shift) < a.TW) ++a.tw_shift;
    a.tiles_x = ceil_div(p->W, a.TW);
    a.tiles_y = ceil_div(p->H, a.TH);
    a.n_work = a.tiles_x * a.tiles_y * p->B * a.n_tiles;
    return true;
  }
  return false;
}

int conv2d_umma(const pfb_conv_params* p, cudaStream_t s) {
  ConvUmmaArgs a{};
  if (!plan_conv_umma(p, a)) {
    set_error("conv_umma: no tile and ring plan fits in shared memory");
    return PFB_ERR_UNSUPPORTED;
  }
  const int patch_w = a.TW + (a.halo == 1 ? p->KW - 1 : 0);
  const int patch_h = a.TH + (a.halo == 2 ? p->KH - 1 : 0);
  CUtensorMap tms[3];
  a.nsrc = p->nsrc;
  for (int i = 0; i < p->nsrc; ++i) {
    const pfb_conv_src& src = p->src[i];
    a.src_chunks[i] = eff_channels(src) / 64;
    a.src_coff[i] = src.offset;
    // dim 0 ends at the source's last real channel: a partial last 64-chunk is zero-filled by the TMA unit
    uint64_t dims[4] = {(uint64_t)(src.offset + src.channels), (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->B};
    uint64_t str[3] = {(uint64_t)src.stride * 2, (uint64_t)p->W * src.stride * 2, (uint64_t)p->H * p->W * src.stride * 2};
    uint32_t box[4] = {64, (uint32_t)patch_w, (uint32_t)patch_h, 1};
    int rc = make_tensor_map(&tms[i], src.ptr, p->dtype, 4, dims, str, box);
    if (rc) return rc;
  }
  for (int i = p->nsrc; i < 3; ++i) tms[i] = tms[0];
  CUtensorMap tmW;
  {
    uint64_t dims[2] = {(uint64_t)p->Cin_pad, p->w_rows_per_sample > 0 ? (uint64_t)p->B * p->w_rows_per_sample : (uint64_t)p->KH * p->KW * p->Cout_pad_k};
    uint64_t str[1] = {(uint64_t)p->Cin_pad * 2};
    uint32_t box[2] = {64, (uint32_t)a.NT};
    int rc = make_tensor_map(&tmW, p->weight_k, p->dtype, 2, dims, str, box);
    if (rc) return rc;
  }
  a.B = p->B; a.H = p->H; a.W = p->W; a.KH = p->KH; a.KW = p->KW;
  a.Cout = p->Cout; a.Cout_pad_k = p->Cout_pad_k;
  // ---- outputs through staging + TMA bulk stores (everything but the fp32 tap products) ----
  CUtensorMap tmO[2];
  tmO[0] = tms[0];
  tmO[1] = tms[0];
  {
    const bool zr = p->epilogue == PFB_EPI_GRU_ZR;
    if (a.tma_out) {
      const bool append = p->epilogue == PFB_EPI_RELU_APPEND_FLOW || p->epilogue == PFB_EPI_LINEAR_APPEND_FLOW;
      const int ncols = zr ? p->hidden : (append ? p->Cout + 2 : p->Cout);
      uint64_t dims[4] = {(uint64_t)(p->out_offset + ncols), (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->B};
      uint64_t str[3] = {(uint64_t)p->out_stride * 2, (uint64_t)p->W * p->out_stride * 2, (uint64_t)p->H * p->W * p->out_stride * 2};
      uint32_t box[4] = {64, (uint32_t)a.TW, (uint32_t)a.TH, 1};
      int rc = make_tensor_map(&tmO[0], p->out, p->dtype, 4, dims, str, box);
      if (rc) return rc;
      if (zr) {
        uint64_t dz[4] = {(uint64_t)p->hidden, (uint64_t)p->W, (uint64_t)p->H, (uint64_t)p->B};
        uint64_t sz[3] = {(uint64_t)p->hidden * 2, (uint64_t)p->W * p->hidden * 2, (uint64_t)p->H * p->W * p->hidden * 2};
        rc = make_tensor_map(&tmO[1], p->aux_z, p->dtype, 4, dz, sz, box);
        if (rc) return rc;
      }
    }
  }
  a.bias = p->bias; a.epilogue = p->epilogue; a.scale = p->scale;
  a.out = p->out; a.out_stride = p->out_stride; a.out_offset = p->out_offset;
  a.aux_h = p->aux_h; a.aux_z = p->aux_z; a.hidden = p->hidden; a.flow = p->flow;
  a.addend = p->addend; a.addend_stride = p->addend_stride;
  a.residual = p->residual; a.residual_stride = p->residual_stride; a.residual_offset = p->residual_offset;
  a.post_w = p->post_w; a.post_b = p->post_b;
  a.w_rows_per_sample = p->w_rows_per_sample;
  a.ab_fmt = p->dtype == PFB_F16 ? 0 : 1;
  const size_t smem = (size_t)a.a_stages * a.a_slot_bytes + (size_t)a.b_stages * a.b_slot_bytes + (a.tma_out ? kATileBytes : 0) +
                      acc_tile_bytes(a.NT) + kMaxBias * sizeof(float) + sizeof(ConvBars) + 1024;
  int grid = sm_count();
  if (grid > a.n_work) grid = a.n_work;
  static const char* env_trace = getenv("PFB_CONV_TRACE");  // debug: per-CTA timeline of every launch -> JSON lines
  if (env_trace) {
    static unsigned long long* dbuf = nullptr;
    if (!dbuf) PFB_CUDA(cudaMalloc(&dbuf, 256 * 32 * 8));
    PFB_CUDA(cudaMemsetAsync(dbuf, 0, 256 * 32 * 8, s));
    a.trace = dbuf;
    int rc;
    rc = p->dtype == PFB_F16 ? launch_conv_umma<__half>(tms, tmW, tmO, a, grid, smem, s) : launch_conv_umma<__nv_bfloat16>(tms, tmW, tmO, a, grid, smem, s);
    if (rc) return rc;
    PFB_CUDA(cudaStreamSynchronize(s));
    static unsigned long long host[256 * 32];
    PFB_CUDA(cudaMemcpy(host, dbuf, sizeof(host), cudaMemcpyDeviceToHost));
    if (FILE* f = fopen(env_trace, "a")) {
      fprintf(f, "{\"KH\":%d,\"KW\":%d,\"NT\":%d,\"Cin_pad\":%d,\"halo\":%d,\"TW\":%d,\"TH\":%d,\"epi\":%d,\"grid\":%d,\"n_work\":%d,\"a_stages\":%d,\"b_stages\":%d,\"b_group\":%d,\"t\":[",
              a.KH, a.KW, a.NT, p->Cin_pad, a.halo, a.TW, a.TH, a.epilogue, grid, a.n_work, a.a_stages, a.b_stages, a.b_group);
      for (int i = 0; i < grid * 32; ++i) fprintf(f, "%s%llu", i ? "," : "", host[i]);
      fprintf(f, "]}\n");
      fclose(f);
    }
    return PFB_OK;
  }
  ProfScope prof(KC_CONV, s);
  if (p->dtype == PFB_F16) return launch_conv_umma<__half>(tms, tmW, tmO, a, grid, smem, s);
  return launch_conv_umma<__nv_bfloat16>(tms, tmW, tmO, a, grid, smem, s);
}

}  // namespace pfb
