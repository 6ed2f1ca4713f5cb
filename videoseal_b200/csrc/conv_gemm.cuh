// K1/K2: implicit-GEMM convolution / linear layer on the Hopper tensor cores (wgmma, fp32 accumulators in registers),
// persistent and warp-specialised:
//
//   warps 0..E-1  : epilogue, E = 8 (LD_TMA) or 4 (accumulator tile in shared memory -> registers -> fused bias/BN-fold/act/
//                   residual/LN/tanh/GRN-stats -> HBM); warp w owns rows 32*(w%4) .. +31 (one row per lane) and the 16-column
//                   chunks c with c % (E/4) == w/4
//   warps E..E+3  : A-tile builders (all loaders except LD_TMA):
//       LD_HALO_CONV3 : on-chip im2col - the (8+2)x(16+2) input halo of an 8x16 output tile is TMA-loaded ONCE per channel
//                       chunk (zero fill = conv padding) and the tap tiles are copied smem->smem into the 128-byte-swizzled
//                       wgmma operand layout (input pixels cross L2->SM once instead of nine times)
//       LD_GATHER_CONV: generic strided / reflect-padded conv gathered from global memory (stride-2 3x3, k2s2 patchify,
//                       reflect-padded head conv, the 3x3 conv of a nearest x2 up-sample read from the low-resolution map)
//
//   next 8 warps  : two MMA warpgroups; warpgroup h issues the wgmma of rows [64h, 64h + 64) of the tile
//   last warp     : TMA producer (weights unless resident; activations for LD_TMA; input halo tiles for LD_HALO_CONV3)
//
// GEMM view: D[M = output pixels, N = C_out] = A[M, K = taps*C_in] * W[N, K]^T, fp16 operands, fp32 accumulation.
// BLOCK_M = 128, BLOCK_N <= 128.  The MMA warpgroups hand each finished accumulator round to the epilogue through one
// [128 x 128] fp32 tile in shared memory (the epilogue reads one row per thread) and meanwhile run the main loop of the
// next round in registers, so the epilogue of tile i overlaps the main loop of tile i+1.  Small weight matrices stay
// resident in shared memory.
//
// Replaces: nn.Conv2d / nn.Linear + BatchNorm2d(eval) + ReLU / LayerNorm / GELU / GRN / tanh call sites of
// videoseal/modules/unet.py:17-197, modules/common.py:45-52,150-169, modules/convnext.py:41-57,
// modules/pixel_decoder.py:44-55 (see DESIGN.md for the per-layer mapping).
#pragma once
#include "ptx.cuh"

namespace vsb {

enum : int { LD_TMA = 0, LD_GATHER_CONV = 1, LD_HALO_CONV3 = 4 };
enum : int { EPI_AFFINE = 0, EPI_LN = 1 };
enum : int { ACT_NONE = 0, ACT_RELU = 1, ACT_GELU = 2 };

constexpr int kBlockM = 128;
constexpr int kMaxStages = 24;
constexpr int kMaxHalo = 8;
constexpr int kMaxBlockN = 128;
constexpr int kAccCols = 128;       // columns of one accumulator round (group * block_n)
constexpr int kAccPitch = kAccCols + 4;   // floats per row of the shared accumulator tile: row-per-thread float4 reads are conflict-free
constexpr uint32_t kAccBytes = (uint32_t)kBlockM * kAccPitch * 4;
constexpr int kEpiWarps = 8;       // LD_TMA; the loaders with 4 builder warps have 4 epilogue warps (17 warps either way: 96 registers)
constexpr int kMmaThreads = 256;    // two MMA warpgroups
constexpr int kHeaderBytes = 11264;  // barriers | bias x2 | LN w,b / outc rows | outc partials (3 x [128][3])
constexpr int kHaloTW = 16, kHaloTH = 8;
constexpr int kHaloW = kHaloTW + 2, kHaloH = kHaloTH + 2;   // 18 x 10 input halo of an 8x16 output tile

// division by a runtime constant as multiply-high + shift (valid for 0 <= n < 2^31); the host precomputes (mul, shr)
struct FastDiv {
  uint32_t mul, shr;
  int d;
  __device__ __forceinline__ int div(int n) const { return d == 1 ? n : (int)(__umulhi((uint32_t)n, mul) >> shr); }
};

struct ConvGemmParams {
  FastDiv fd_ntiles, fd_tpi, fd_tx, fd_tw, fd_group, fd_rps, fd_hw, fd_cc, fd_ow, fd_oh, fd_ct, fd_s;
  // ---- GEMM view
  int M, N, num_kb, kblk, block_n, n_tiles, m_tiles, num_tiles, stages;
  uint32_t a_stage_bytes, b_stage_bytes, stage_bytes;
  int group;                      // consecutive M tiles that share one accumulator round (amortises per-tile handshakes for small N)
  int b_resident;                 // whole [block_n x K] weight slab lives in shared memory for the kernel's lifetime
  int b_fixed_ntile;              // b_resident with several N tiles: this CTA only ever sees N tile blockIdx.x % n_tiles
  int tma_store;                  // 1: fp16, 2: fp32 output tiles leave through TMA stores: every epilogue warp stages its 16-column chunks
  int cpw;                        //   ([32 rows][16 cols] boxes) in shared memory and one lane issues a bulk store per chunk; the warps of a
                                  //   lane quadrant own consecutive chunks (cpw = the largest count; the split may be uneven)
  uint32_t ostage_off, ostage_bytes;   // staging area: [epilogue warp][boxes][32 rows][ost_cpb * 16 cols]
  int ost_cpb;                    //   chunks per staging box (cpw: one box per warp; 1: one box per chunk)
  uint32_t ost_rowb;              //   bytes per box row
  int ost_swz;                    //   0 linear, 1 / 2 / 3: 32 / 64 / 128-byte TMA swizzle of the box rows
  int bias_global;                // epilogue reads the bias straight from global memory (warp-uniform 16-byte loads, L1 hits) instead
                                  // of a shared copy: no per-tile barrier between the epilogue warps (whole tiles only)
  uint32_t bres_off, acc_off;
  // ---- output-tile geometry: tile_mode 0: rows are consecutive GEMM rows; 1: tile_h x tile_w pixel patch of an H x W map
  int tile_mode, H, W, tile_w, tile_h, tiles_x, tiles_per_img;
  // ---- A via TMA (LD_TMA): a_is_conv 0: 2D map (K, M); 1: 4D map (C, W, H, B) with zero-fill halo, one load per tap
  int a_is_conv, R, S, pad, c_blocks;
  // ---- halo loaders: the input is cut into `c_blocks` channel chunks of `cc` (= min(C, 64)) channels, the first c0_blocks
  //      from source 0; each chunk contributes kb_per_c K-blocks of 64 (K order inside a chunk: (tap, channel), zero padded)
  int c0_blocks, cc, kb_per_c;
  uint32_t halo_bytes /*TMA box bytes*/, halo_stride /*buffer pitch*/, halo_off;
  // ---- residual prefetch ring (thread-private slots)
  uint32_t resid_off, resid_stride;
  int resid_depth;
  int resid_direct;               // 1: no shared-memory ring, the epilogue reads the fp16 residual straight from global memory (long-K layers:
                                  //    their epilogue is hidden behind the main loop, the 48 KB buy one more TMA pipeline stage)
  // (declared here, not with the halo fields: this keeps the 8-byte pairing of the int fields above, without which ptxas gives
  //  the gather and halo kernels more stack)
  int halo_bufs;                  // ring depth of the halo tiles (prefetch distance of the producer)
  // ---- gather loaders (NHWC fp16 sources; K order = (r, s, c) with c over the virtual concat [src0 | src1])
  const __half* src0;
  const __half* src1;
  int C0, C1, ld0, ld1, IH, IW, OH, OW, stride, pad_mode /*0 zero, 1 reflect, 2 zero on the nearest x2 up-sample*/, Ktot;
  int rows_per_sample;            // GEMM rows per sample (GRN statistics, per-sample weights)
  int b_sample_rows;              // > 0: per-sample weights [samples][N][K] (GRN folded into pwconv2); = N
  FastDiv fd_tps;                 // M tiles per sample
  // ---- epilogue
  int epi, act;
  const float* bias;     // [N] or null
  const __half* resid16; int ld_res16;   // added AFTER the activation (ResnetBlock: act(norm(conv)) + res)
  const float* resid32;  int ld_res32;
  __half* out16; int ld_out16;
  float* out32;  int ld_out32;
  const float* ln_w; const float* ln_b; float ln_eps;     // EPI_LN (requires n_tiles == 1)
  const float* outc_w; const float* outc_b; float* delta; int n_out, hw, outc_tanh;  // fused 1x1 outc (+tanh)
  float* grn_stats;      // [num_samples, N] sum of squares of the epilogue output (GRN), or null
  int grn_part;          // 1: grn_stats is [M / 32, N]: every epilogue warp STORES the column sums of its 32 rows (no atomics: the
                         //    consumer adds the rows of a sample in a fixed order -> bit-reproducible logits); needs
                         //    rows_per_sample % 32 == 0
};

// exact-erf GELU (nn.GELU default) with ONE special-function op per element:
//   gelu(x) = 0.5 x (1 + erf(x / sqrt2)) = max(x, 0) - 0.5 |x| erfc(|x| / sqrt2),   erfc(|x| / sqrt2) = 2^Q(|x|)
// Q = degree-5 polynomial without constant term (erfc(0) = 1), weighted minimax fit of log2 erfc on [0, 3.3 sqrt2] (oracle-side
// check in tests/test_cpu_library.py): |gelu - exact| <= 1.0e-6 for every fp32 x in [-30, 30] (the tail runs to 2^-88 -> 0 on its
// own).  Abramowitz-Stegun 7.1.25 would need rcp AND ex2 per element, and its error is 2.5e-5.
constexpr float kGeluQ0 = -1.1510894298553467f, kGeluQ1 = -0.4592657685279846f, kGeluQ2 = -0.05254320427775383f,
                kGeluQ3 = 0.007386638317257166f, kGeluQ4 = -0.0005183160537853837f;
__device__ __forceinline__ float ex2_approx(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float gelu_erf(float x) {
  const float ax = fabsf(x);
  float q = fmaf(kGeluQ4, ax, kGeluQ3);
  q = fmaf(q, ax, kGeluQ2);
  q = fmaf(q, ax, kGeluQ1);
  q = fmaf(q, ax, kGeluQ0);
  const float e = ex2_approx(q * ax);
  return fmaf(-0.5f * ax, e, fmaxf(x, 0.f));
}

// two GELUs at once, written on float2 pairs (each component rounds exactly like the scalar fma / mul / add)
__device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 f2mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
// packed in, packed out; max(x, 0) as 0.5 (x + |x|) so that the tail is two packed FMAs: gelu = 0.5 x + 0.5 |x| (1 - e)
__device__ __forceinline__ float2 gelu_erf_p(float2 x) {
  const float2 ax = make_float2(fabsf(x.x), fabsf(x.y));
  float2 q = f2fma(make_float2(kGeluQ4, kGeluQ4), ax, make_float2(kGeluQ3, kGeluQ3));
  q = f2fma(q, ax, make_float2(kGeluQ2, kGeluQ2));
  q = f2fma(q, ax, make_float2(kGeluQ1, kGeluQ1));
  q = f2fma(q, ax, make_float2(kGeluQ0, kGeluQ0));
  q = f2mul(q, ax);
  const float2 e = make_float2(ex2_approx(q.x), ex2_approx(q.y));
  const float2 hax = f2mul(ax, make_float2(0.5f, 0.5f));
  const float2 t = f2fma(make_float2(-e.x, -e.y), hax, hax);            // 0.5 |x| (1 - e)
  return f2fma(x, make_float2(0.5f, 0.5f), t);
}
__device__ __forceinline__ void gelu_erf2(float& x0, float& x1) {
  const float2 ax = make_float2(fabsf(x0), fabsf(x1));
  float2 q = f2fma(make_float2(kGeluQ4, kGeluQ4), ax, make_float2(kGeluQ3, kGeluQ3));
  q = f2fma(q, ax, make_float2(kGeluQ2, kGeluQ2));
  q = f2fma(q, ax, make_float2(kGeluQ1, kGeluQ1));
  q = f2fma(q, ax, make_float2(kGeluQ0, kGeluQ0));
  q = f2mul(q, ax);
  const float2 e = make_float2(ex2_approx(q.x), ex2_approx(q.y));
  const float2 r = f2fma(f2mul(ax, make_float2(-0.5f, -0.5f)), e, make_float2(fmaxf(x0, 0.f), fmaxf(x1, 0.f)));
  x0 = r.x; x1 = r.y;
}

__device__ __forceinline__ int reflect_idx(int i, int n) {
  if (i < 0) i = -i;
  if (i >= n) i = 2 * n - 2 - i;
  return i;
}

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async16_zfill(void* smem_dst, const void* gsrc, uint32_t src_bytes) {   // src_bytes 16 or 0
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(src_bytes) : "memory");
}
// the mbarrier receives one (counted) arrival once all prior cp.async of this thread have completed
__device__ __forceinline__ void cp_async_mbar_arrive_noinc(uint64_t* bar) {
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_pending(int n) {   // wait until at most n groups are pending
  switch (n) {
    case 0: asm volatile("cp.async.wait_group 0;" ::: "memory"); break;
    case 1: asm volatile("cp.async.wait_group 1;" ::: "memory"); break;
    case 2: asm volatile("cp.async.wait_group 2;" ::: "memory"); break;
    default: asm volatile("cp.async.wait_group 3;" ::: "memory"); break;
  }
}
template <int NT> __device__ __forceinline__ void epi_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(NT) : "memory"); }

// one row of the shared accumulator tile -> 16 registers
__device__ __forceinline__ void acc_ld16(const float* src, uint32_t (&r)[16]) {
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const float4 t = reinterpret_cast<const float4*>(src)[u];
    r[4 * u] = __float_as_uint(t.x); r[4 * u + 1] = __float_as_uint(t.y); r[4 * u + 2] = __float_as_uint(t.z); r[4 * u + 3] = __float_as_uint(t.w);
  }
}
__device__ __forceinline__ void acc_ld16(const float* src, float (&v)[16]) {
#pragma unroll
  for (int u = 0; u < 4; ++u) {
    const float4 t = reinterpret_cast<const float4*>(src)[u];
    v[4 * u] = t.x; v[4 * u + 1] = t.y; v[4 * u + 2] = t.z; v[4 * u + 3] = t.w;
  }
}

// The MMA warpgroups: warpgroup wg computes rows [64 wg, 64 wg + 64) of every sub-tile in registers (BN = block_n columns),
// keeping one wgmma group in flight, then writes them into the shared accumulator tile once the epilogue has drained it.
template <int BN, int LOADER>
__device__ __forceinline__ void mma_warpgroup(const ConvGemmParams& p, uint8_t* tiles, uint8_t* bres, uint64_t* full_bar,
                                              uint64_t* empty_bar, uint64_t* tfull_bar, uint64_t* tempty_bar, uint64_t* bres_bar,
                                              float* acc_s, int wg) {
  const int lane = threadIdx.x & 31, wq = (threadIdx.x >> 5) & 3;
  float d[BN / 2];
  int stage = 0;
  uint32_t phase = 0, aphase = 0;
  const uint32_t row_bytes = (uint32_t)p.kblk * 2u;
  const uint32_t a_off = (uint32_t)wg * 64u * row_bytes;   // 8-row swizzle atoms: a multiple of 1024 bytes
  const int nmma = p.kblk >> 4;
  if (p.b_resident) mbar_wait(bres_bar, 0u);
  const uint32_t bres_addr = smem_u32(bres);
  const int r0 = wg * 64 + wq * 16 + (lane >> 2), c0 = 2 * (lane & 3);
  auto release = [&](int s) {
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty_bar[s]);
  };
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
    const int st = p.fd_ntiles.div(tile);
    for (int g = 0; g < p.group; ++g) {
      if (st * p.group + g >= p.m_tiles) break;
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        mbar_wait(&full_bar[stage], phase);
        if (LOADER == LD_GATHER_CONV) fence_proxy_async_smem();   // cp.async-written A tile -> async proxy
        const uint32_t sa = smem_u32(tiles + (size_t)stage * p.stage_bytes);
        const uint64_t adesc = make_smem_desc(sa + a_off, row_bytes);
        const uint64_t bdesc = make_smem_desc(p.b_resident ? bres_addr + (uint32_t)kb * p.b_stage_bytes : sa + p.a_stage_bytes, row_bytes);
        wgmma_fence_regs(d);
        wgmma_fence();
        for (int j = 0; j < nmma; ++j) {
          // advance 16 K-elements = 32 bytes inside the swizzled row: +2 in the (addr >> 4) field
          Wgmma<BN>::mma(d, adesc + (uint64_t)(2 * j), bdesc + (uint64_t)(2 * j), (uint32_t)((kb | j) != 0));
        }
        wgmma_commit();
        wgmma_fence_regs(d);
        if (prev >= 0) {
          wgmma_wait<1>();   // the previous K-block's wgmma have read their slot
          release(prev);
        }
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
      wgmma_wait<0>();
      wgmma_fence_regs(d);
      release(prev);
      if (g == 0) mbar_wait(tempty_bar, aphase ^ 1u);   // the epilogue has read the previous round
      float* dst = acc_s + g * BN;
#pragma unroll
      for (int i = 0; i < BN / 2; i += 2) {
        const int r = r0 + 8 * ((i >> 1) & 1), c = 8 * (i >> 2) + c0;
        *reinterpret_cast<float2*>(dst + r * kAccPitch + c) = make_float2(d[i], d[i + 1]);
      }
    }
    mbar_arrive(tfull_bar);
    aphase ^= 1u;
  }
}

template <int LOADER, int ACT>
__global__ void __launch_bounds__(544, 1)
conv_gemm_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmA2,
                 const __grid_constant__ CUtensorMap tmB, const __grid_constant__ CUtensorMap tmO,
                 const __grid_constant__ ConvGemmParams p) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  // header (kHeaderBytes): barriers | s_bias[2][256] | s_lnw[256] s_lnb[256] s_oc2[256] | s_dot[128][3]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint64_t* tfull_bar = empty_bar + kMaxStages;    // accumulator tile written by the MMA warpgroups
  uint64_t* tempty_bar = tfull_bar + 1;            // accumulator tile read by the epilogue
  uint64_t* hfull_bar = tempty_bar + 1;
  uint64_t* hempty_bar = hfull_bar + kMaxHalo;
  uint64_t* bres_bar = hempty_bar + kMaxHalo;
  float* s_bias = reinterpret_cast<float*>(smem + 1024);        // [2][256]
  float* s_lnw = reinterpret_cast<float*>(smem + 3072);         // [256]  (LN weight | outc row 0)
  float* s_lnb = reinterpret_cast<float*>(smem + 4096);         // [256]  (LN bias   | outc row 1)
  float* s_oc2 = reinterpret_cast<float*>(smem + 5120);         // [256]  (            outc row 2)
  float* s_dot = reinterpret_cast<float*>(smem + 6144);         // [128][3]
  uint8_t* tiles = smem + kHeaderBytes;
  uint8_t* halo = smem + p.halo_off;
  uint8_t* bres = smem + p.bres_off;
  uint8_t* rbuf = smem + p.resid_off;
  float* acc_s = reinterpret_cast<float*>(smem + p.acc_off);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  constexpr uint32_t kNumBuilders = 128;
  constexpr bool kHalo = LOADER == LD_HALO_CONV3;
  constexpr int kEpiW = LOADER == LD_TMA ? kEpiWarps : 4;
  constexpr int kEpiThreads = kEpiW * 32;
  constexpr int kEpiSplit = kEpiW / 4;              // warps sharing one 32-row quadrant (interleaved 16-column chunks)
  constexpr int kBuilderWarp0 = kEpiW;
  constexpr int kMmaWarp0 = kBuilderWarp0 + (LOADER == LD_TMA ? 0 : 4);   // warpgroup-aligned
  constexpr int kProducerWarp = kMmaWarp0 + kMmaThreads / 32;

  if (threadIdx.x == 0) {
    const uint32_t full_count = LOADER == LD_TMA ? 1u : kNumBuilders + (p.b_resident ? 0u : 1u);
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], full_count);
      mbar_init(&empty_bar[s], (uint32_t)(kMmaThreads / 32));
    }
    mbar_init(tfull_bar, (uint32_t)kMmaThreads);
    mbar_init(tempty_bar, (uint32_t)kEpiThreads);
    for (int s = 0; s < kMaxHalo; ++s) {
      mbar_init(&hfull_bar[s], 1u);
      mbar_init(&hempty_bar[s], kNumBuilders);
    }
    mbar_init(bres_bar, 1u);
    fence_barrier_init();
    if (LOADER == LD_TMA || kHalo) tma_prefetch_desc(&tmA);
    if (LOADER == LD_TMA && p.c0_blocks != 0) tma_prefetch_desc(&tmA2);
    tma_prefetch_desc(&tmB);
    if (p.tma_store) tma_prefetch_desc(&tmO);
  }
  if (p.epi == EPI_LN) {
    for (int i = threadIdx.x; i < p.N; i += blockDim.x) { s_lnw[i] = p.ln_w[i]; s_lnb[i] = p.ln_b[i]; }
  } else if (p.outc_w != nullptr) {  // fused 1x1 outc: N <= 256 (n_tiles == 1), up to 3 output channels
    for (int i = threadIdx.x; i < p.N; i += blockDim.x) {
      s_lnw[i] = p.outc_w[i];
      s_lnb[i] = p.n_out > 1 ? p.outc_w[p.N + i] : 0.f;
      s_oc2[i] = p.n_out > 2 ? p.outc_w[2 * p.N + i] : 0.f;
    }
  }
  __syncthreads();
  // nothing above reads or writes a tensor produced by an earlier kernel: only parameters and weights
  pdl_launch_dependents();
  pdl_wait();

  if (warp == kProducerWarp) {
    // ===================================================================== TMA producer
    if (elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      int hb = 0;
      uint32_t hphase = 0;
      if (p.b_resident) {  // n_tiles == 1: the whole weight slab once
        mbar_arrive_expect_tx(bres_bar, (uint32_t)p.num_kb * p.b_stage_bytes);
        const int brow0 = p.b_fixed_ntile ? ((int)blockIdx.x - p.fd_ntiles.div((int)blockIdx.x) * p.n_tiles) * p.block_n : 0;
        for (int kb = 0; kb < p.num_kb; ++kb) tma_load_2d(&tmB, bres_bar, bres + (size_t)kb * p.b_stage_bytes, kb * p.kblk, brow0);
      }
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
       const int st = p.fd_ntiles.div(tile), n_tile = tile - st * p.n_tiles;
       for (int g = 0; g < p.group; ++g) {
        const int m_tile = st * p.group + g;
        if (m_tile >= p.m_tiles) break;
        int cb = 0, cx = 0, cy = 0;
        if (p.tile_mode == 1) {
          cb = p.fd_tpi.div(m_tile);
          const int rem = m_tile - cb * p.tiles_per_img;
          const int ty = p.fd_tx.div(rem);
          cy = ty * p.tile_h;
          cx = (rem - ty * p.tiles_x) * p.tile_w;
        }
        if (kHalo) {
          for (int c = 0; c < p.c_blocks; ++c) {
            mbar_wait(&hempty_bar[hb], hphase ^ 1u);
            mbar_arrive_expect_tx(&hfull_bar[hb], p.halo_bytes);
            tma_load_4d(&tmA, &hfull_bar[hb], halo + (size_t)hb * p.halo_stride, c * p.cc, cx - 1, cy - 1, cb);
            if (++hb == p.halo_bufs) { hb = 0; hphase ^= 1u; }
            if (!p.b_resident) {
              int kcoord = c * p.kb_per_c * 64;
              for (int kbi = 0; kbi < p.kb_per_c; ++kbi, kcoord += 64) {
                mbar_wait(&empty_bar[stage], phase ^ 1u);
                mbar_arrive_expect_tx(&full_bar[stage], p.b_stage_bytes);
                tma_load_2d(&tmB, &full_bar[stage], tiles + (size_t)stage * p.stage_bytes + p.a_stage_bytes, kcoord, n_tile * p.block_n);
                if (++stage == p.stages) { stage = 0; phase ^= 1u; }
              }
            }
          }
        } else if (LOADER == LD_TMA) {
          int tap_r = 0, tap_s = 0, cblk = 0;
          const int brow = n_tile * p.block_n + (p.b_sample_rows ? p.fd_tps.div(m_tile) * p.b_sample_rows : 0);
          for (int kb = 0; kb < p.num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* sa = tiles + (size_t)stage * p.stage_bytes;
            mbar_arrive_expect_tx(&full_bar[stage], p.a_stage_bytes + (p.b_resident ? 0u : p.b_stage_bytes));
            if (p.a_is_conv) {
              tma_load_4d(&tmA, &full_bar[stage], sa, cblk * p.kblk, cx + tap_s - p.pad, cy + tap_r - p.pad, cb);
              if (++cblk == p.c_blocks) { cblk = 0; if (++tap_s == p.S) { tap_s = 0; ++tap_r; } }
            } else {
              // 2D GEMM operand, optionally the virtual concat [A0 | A1] along K (c0_blocks K-blocks come from A0)
              if (p.c0_blocks == 0 || kb < p.c0_blocks) tma_load_2d(&tmA, &full_bar[stage], sa, kb * p.kblk, m_tile * kBlockM);
              else tma_load_2d(&tmA2, &full_bar[stage], sa, (kb - p.c0_blocks) * p.kblk, m_tile * kBlockM);
            }
            if (!p.b_resident) tma_load_2d(&tmB, &full_bar[stage], sa + p.a_stage_bytes, kb * p.kblk, brow);
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
          }
        } else if (!p.b_resident) {  // gather loaders: weights only
          for (int kb = 0; kb < p.num_kb; ++kb) {
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            mbar_arrive_expect_tx(&full_bar[stage], p.b_stage_bytes);
            tma_load_2d(&tmB, &full_bar[stage], tiles + (size_t)stage * p.stage_bytes + p.a_stage_bytes, kb * p.kblk, n_tile * p.block_n);
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
          }
        }
       }
      }
    }
  } else if (warp >= kMmaWarp0) {
    // ===================================================================== MMA warpgroups
    const int wg = (warp - kMmaWarp0) >> 2;
    switch (p.block_n) {
      case 16: mma_warpgroup<16, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 32: mma_warpgroup<32, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 48: mma_warpgroup<48, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 64: mma_warpgroup<64, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 80: mma_warpgroup<80, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 96: mma_warpgroup<96, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      case 112: mma_warpgroup<112, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
      default: mma_warpgroup<128, LOADER>(p, tiles, bres, full_bar, empty_bar, tfull_bar, tempty_bar, bres_bar, acc_s, wg); break;
    }
  } else if (warp < kEpiW) {
    // ===================================================================== epilogue (4 or 8 warps)
    const int q = warp & 3;            // 32-row quadrant of the tile this warp owns
    const int half = warp >> 2;        // which 16-column chunks: chunk index modulo kEpiSplit
    const int row = q * 32 + lane;
    const int et = threadIdx.x;        // 0..kEpiThreads-1
    const int nchunks = p.block_n >> 4;
    // 16-column chunks of this warp: interleaved (half, half + kEpiSplit, ...) or, with TMA stores, cpw consecutive ones
    int c_beg = half, c_end = nchunks, c_step = kEpiSplit;
    if (p.tma_store) {
      const int base = nchunks / kEpiSplit, rem = nchunks - base * kEpiSplit;
      c_beg = half * base + min(half, rem);
      c_end = c_beg + base + (half < rem ? 1 : 0);
      c_step = 1;
    }
    uint8_t* ost = smem + p.ostage_off + (size_t)warp * p.ostage_bytes;   // this warp's output staging boxes
    const uint32_t ost_box = 32u * p.ost_rowb;
    const uint32_t ost_upc = p.tma_store == 2 ? 4u : 2u;                         // 16-byte units per chunk
    // 16-byte unit u of row r of a swizzled box lives at unit u ^ f(r) (CU_TENSOR_MAP_SWIZZLE_{32,64,128}B)
    const uint32_t ost_x = p.ost_swz == 3 ? (uint32_t)(lane & 7) : (p.ost_swz == 2 ? (uint32_t)((lane >> 1) & 3) : (p.ost_swz == 1 ? (uint32_t)((lane >> 2) & 1) : 0u));
    auto ost_ptr = [&](int k /*chunk of this warp*/, uint32_t t /*16-byte unit inside the chunk*/) -> uint4* {
      const int box = p.ost_cpb == 1 ? k : 0, kin = p.ost_cpb == 1 ? 0 : k;
      return reinterpret_cast<uint4*>(ost + (size_t)box * ost_box + (size_t)lane * p.ost_rowb + (((uint32_t)kin * ost_upc + t) ^ ost_x) * 16u);
    };
    const int D = p.resid_depth;
    const bool has_res = (p.resid16 != nullptr) || (p.resid32 != nullptr);

    // geometry of this thread's row in M tile `m_tile`
    auto tile_row = [&](int m_tile, long& m, bool& mvalid) {
      if (p.tile_mode == 1) {
        const int b = p.fd_tpi.div(m_tile);
        const int rem = m_tile - b * p.tiles_per_img;
        const int ty = p.fd_tx.div(rem), tx = rem - ty * p.tiles_x;
        const int ry = p.fd_tw.div(row), rx = row - ry * p.tile_w;
        m = ((long)b * p.H + (ty * p.tile_h + ry)) * p.W + (tx * p.tile_w + rx);
        mvalid = true;
      } else {
        m = (long)m_tile * kBlockM + row;
        mvalid = m < p.M;
      }
    };
    // residual row of sub-tile number `sq` (= iteration * group + g of this CTA) -> ring slot (thread-private region,
    // layout [16-byte chunk][row] = conflict-free)
    const int G = p.group;
    auto prefetch_resid = [&](int sq, int slot) {
      if (has_res && !p.resid_direct) {
        const int it = p.fd_group.div(sq), g = sq - it * G;
        const int tile = (int)blockIdx.x + it * (int)gridDim.x;
        const int st = p.fd_ntiles.div(tile);
        const int m_tile = st * G + g;
        if (tile < p.num_tiles && m_tile < p.m_tiles) {
          const int n0 = (tile - st * p.n_tiles) * p.block_n;
          long m; bool mvalid;
          tile_row(m_tile, m, mvalid);
          if (mvalid && n0 + p.block_n <= p.N) {
            uint8_t* dst = rbuf + (size_t)slot * p.resid_stride;
            if (p.resid16 != nullptr) {
              const __half* r = p.resid16 + m * p.ld_res16 + n0;
              for (int ch = c_beg; ch < c_end; ch += c_step) {
                cp_async16(dst + ((size_t)(2 * ch) * 128 + row) * 16, r + ch * 16);
                cp_async16(dst + ((size_t)(2 * ch + 1) * 128 + row) * 16, r + ch * 16 + 8);
              }
            } else {
              const float* r = p.resid32 + m * p.ld_res32 + n0;
              for (int ch = c_beg; ch < c_end; ch += c_step) {
#pragma unroll
                for (int u = 0; u < 4; ++u) cp_async16(dst + ((size_t)(4 * ch + u) * 128 + row) * 16, r + ch * 16 + 4 * u);
              }
            }
          }
        }
      }
      cp_async_commit();
    };

    uint32_t aphase = 0;
    int bsel = 0;
    int slot = 0;
    int sq = 0;
    for (int i = 0; i < D - 1; ++i) prefetch_resid(i, i);
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int st = p.fd_ntiles.div(tile);
      const int n0 = (tile - st * p.n_tiles) * p.block_n;
      // ---- prologue, overlapped with the main loop: bias -> smem
      const float* sb = s_bias + bsel * 256;
      if (p.bias_global) {
        sb = p.bias + n0;
      } else {
        if (et < p.block_n) s_bias[bsel * 256 + et] = (p.bias != nullptr && n0 + et < p.N) ? __ldg(p.bias + n0 + et) : 0.f;
        epi_bar_sync<kEpiThreads>();  // bias visible to all epilogue warps (double-buffered across tiles)
      }
     for (int g = 0; g < G; ++g, ++sq) {
      // residual of the sub-tile D-1 ahead -> ring (issued before waiting for this group's accumulators)
      {
        int pslot = slot + D - 1;
        if (pslot >= D) pslot -= D;
        prefetch_resid(sq + D - 1, pslot);
      }
      if (g == 0) mbar_wait(tfull_bar, aphase);
      cp_async_wait_pending(D - 1);
      const int m_tile = st * G + g;
      const uint8_t* rb_ = rbuf + (size_t)slot * p.resid_stride;
      if (++slot == D) slot = 0;
      if (m_tile >= p.m_tiles) continue;     // ragged last group (uniform across the CTA)
      long m; bool mvalid;
      tile_row(m_tile, m, mvalid);
      const bool res_fast = mvalid && (n0 + p.block_n <= p.N);
      const float* trow = acc_s + row * kAccPitch + g * p.block_n;

      if (p.epi == EPI_LN) {
        // channels-first LayerNorm over the full C_out row (biased variance), then activation.  The kEpiSplit warps that share a
        // 32-row quadrant split the 16-column chunks: pass 1 = per-warp partial (sum, sum of squares) of its chunks, exchanged
        // through shared memory and added in a fixed order; pass 2 = normalise + store its chunks.
        {
          const int N = p.N;
          float* s_part = s_dot;                                  // [kEpiSplit][128][2]
          float sum = 0.f, sq = 0.f;
          for (int ch = half; ch < nchunks; ch += kEpiSplit) {
            const int c = ch * 16;
            float v[16];
            acc_ld16(trow + c, v);
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const float x = (c + j < N) ? v[j] + sb[c + j] : 0.f;
              sum += x;
              sq = fmaf(x, x, sq);
            }
          }
          s_part[(half * 128 + row) * 2] = sum;
          s_part[(half * 128 + row) * 2 + 1] = sq;
          epi_bar_sync<kEpiThreads>();
          sum = 0.f; sq = 0.f;
#pragma unroll
          for (int h2 = 0; h2 < kEpiSplit; ++h2) { sum += s_part[(h2 * 128 + row) * 2]; sq += s_part[(h2 * 128 + row) * 2 + 1]; }
          const float mean = sum / (float)N;
          const float rstd = 1.0f / sqrtf(fmaxf(sq / (float)N - mean * mean, 0.f) + p.ln_eps);
          for (int ch = half; ch < nchunks; ch += kEpiSplit) {
            const int c = ch * 16;
            float v[16];
            acc_ld16(trow + c, v);
            if (c >= N) continue;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const int n = c + j;
              float y = 0.f;
              if (n < N) {
                y = (v[j] + sb[c + j] - mean) * rstd * s_lnw[n] + s_lnb[n];
                if (ACT == ACT_RELU) y = fmaxf(y, 0.f);
                else if (ACT == ACT_GELU) y = gelu_erf(y);
              }
              v[j] = y;
            }
            if (mvalid) {
              if (p.out32 != nullptr) {
                float* o = p.out32 + m * p.ld_out32 + c;
                if (c + 16 <= N) {
#pragma unroll
                  for (int u = 0; u < 4; ++u)
                    reinterpret_cast<float4*>(o)[u] = make_float4(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
                } else {
                  for (int j = 0; j < 16 && c + j < N; ++j) o[j] = v[j];
                }
              }
              if (p.out16 != nullptr) {
                __align__(16) __half h[16];
#pragma unroll
                for (int j = 0; j < 16; ++j) h[j] = __float2half_rn(v[j]);
                __half* o = p.out16 + m * p.ld_out16 + c;
                if (c + 16 <= N) {
                  reinterpret_cast<uint4*>(o)[0] = reinterpret_cast<const uint4*>(h)[0];
                  reinterpret_cast<uint4*>(o)[1] = reinterpret_cast<const uint4*>(h)[1];
                } else {
                  for (int j = 0; j < 16 && c + j < N; ++j) o[j] = h[j];
                }
              }
            }
          }
          epi_bar_sync<kEpiThreads>();     // s_part is rewritten by the next sub-tile
        }
      } else {
        float dot0 = 0.f, dot1 = 0.f, dot2 = 0.f;
        const bool grn_uniform =
            p.grn_stats != nullptr &&
            p.fd_rps.div(m_tile * kBlockM + q * 32) == p.fd_rps.div(m_tile * kBlockM + q * 32 + 31) &&
            (m_tile * kBlockM + q * 32 + 31) < p.M;
        float* grn_row = !grn_uniform ? nullptr
                         : (p.grn_part ? p.grn_stats + (long)(m_tile * 4 + q) * p.N
                                       : p.grn_stats + (long)p.fd_rps.div(m_tile * kBlockM + q * 32) * p.N);
        // whole tile, fp16 output only, no residual / fused 1x1, statistics (if any) uniform per warp
        const bool whole = (m_tile + 1) * kBlockM <= p.M && n0 + p.block_n <= p.N && p.out16 != nullptr && p.out32 == nullptr &&
                           p.outc_w == nullptr && (p.ld_out16 & 7) == 0;
        const bool lean32 = ACT == ACT_NONE && (m_tile + 1) * kBlockM <= p.M && n0 + p.block_n <= p.N && p.out32 != nullptr &&
                            p.outc_w == nullptr && p.grn_stats == nullptr && p.resid32 != nullptr && res_fast && (p.ld_out32 & 3) == 0 &&
                            (p.out16 == nullptr || (p.ld_out16 & 7) == 0);
        const bool lean = ACT == ACT_GELU ? (whole && !has_res && (p.grn_stats == nullptr || grn_uniform))
                                          : (whole && p.grn_stats == nullptr && (!has_res || (p.resid16 != nullptr && res_fast)));
        uint32_t vnext[16];
        if (c_beg < c_end) acc_ld16(trow + c_beg * 16, vnext);
        const bool use_ts = p.tma_store == 1 && lean;      // this warp's part of the tile leaves through its staging boxes + TMA stores
        const bool use_ts32 = p.tma_store == 2 && lean32 && p.out16 == nullptr;
        if (use_ts || use_ts32) {                          // the previous stores of this warp have finished reading the staging boxes
          if (lane == 0) bulk_wait_group_read0();
          __syncwarp();
        }
        if (ACT == ACT_GELU && lean) {
          // pwconv1 on whole tiles (every shipped card): bias + GELU + fp16 store + GRN column statistics and nothing else, in packed
          // fp32 arithmetic throughout; one saturating F2FP per output pair.
          const __half* orow = p.out16 + m * p.ld_out16 + n0;
          for (int ch = c_beg; ch < c_end; ch += c_step) {
            const int c = ch * 16;
            const float4* sb4 = reinterpret_cast<const float4*>(sb + c);
            float2 w2[8];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float4 bq = sb4[u];
              w2[2 * u] = f2add(make_float2(__uint_as_float(vnext[4 * u]), __uint_as_float(vnext[4 * u + 1])), make_float2(bq.x, bq.y));
              w2[2 * u + 1] = f2add(make_float2(__uint_as_float(vnext[4 * u + 2]), __uint_as_float(vnext[4 * u + 3])), make_float2(bq.z, bq.w));
            }
            if (ch + c_step < c_end) acc_ld16(trow + c + 16 * c_step, vnext);   // overlaps the math below
#pragma unroll
            for (int j = 0; j < 8; ++j) w2[j] = gelu_erf_p(w2[j]);
            {
              uint32_t h[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h[j]) : "f"(w2[j].y), "f"(w2[j].x));   // {hi, lo}
              if (use_ts) {
                *ost_ptr(ch - c_beg, 0) = make_uint4(h[0], h[1], h[2], h[3]);
                *ost_ptr(ch - c_beg, 1) = make_uint4(h[4], h[5], h[6], h[7]);
              } else {
                uint4* o = reinterpret_cast<uint4*>(const_cast<__half*>(orow) + c);
                o[0] = make_uint4(h[0], h[1], h[2], h[3]);
                o[1] = make_uint4(h[4], h[5], h[6], h[7]);
              }
            }
            if (grn_row != nullptr) {
              float sq[16];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                const float2 t2 = f2mul(w2[j], w2[j]);
                sq[2 * j] = t2.x; sq[2 * j + 1] = t2.y;
              }
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float send = (lane & 16) ? sq[i] : sq[i + 8];
                const float keep = (lane & 16) ? sq[i + 8] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float send = (lane & 8) ? sq[i] : sq[i + 4];
                const float keep = (lane & 8) ? sq[i + 4] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const float send = (lane & 4) ? sq[i] : sq[i + 2];
                const float keep = (lane & 4) ? sq[i + 2] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
              }
              {
                const float send = (lane & 2) ? sq[0] : sq[1];
                const float keep = (lane & 2) ? sq[1] : sq[0];
                sq[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
              }
              sq[0] += __shfl_xor_sync(0xffffffffu, sq[0], 1);
              if ((lane & 1) == 0) {
                if (p.grn_part) grn_row[n0 + c + ((lane >> 1) & 15)] = sq[0];
                else atomicAdd(grn_row + n0 + c + ((lane >> 1) & 15), sq[0]);
              }
            }
          }
        } else
        for (int ch = c_beg; ch < c_end; ch += c_step) {
          const int c = ch * 16;
          float v[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) v[j] = __uint_as_float(vnext[j]);
          if (ch + c_step < c_end) acc_ld16(trow + c + 16 * c_step, vnext);   // overlaps the math below
          const int n = n0 + c;
          if (ACT == ACT_NONE && lean32) {
            // pwconv2 on whole tiles: bias + fp32 residual stream from the prefetch ring, updated in place (+ fp16 copy)
            const float4* sb4 = reinterpret_cast<const float4*>(sb + c);
            float4* o = reinterpret_cast<float4*>(p.out32 + m * p.ld_out32 + n);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float4 bq = sb4[u];
              const float4 t = *reinterpret_cast<const float4*>(rb_ + ((size_t)(4 * ch + u) * 128 + row) * 16);
              v[4 * u + 0] += bq.x + t.x; v[4 * u + 1] += bq.y + t.y; v[4 * u + 2] += bq.z + t.z; v[4 * u + 3] += bq.w + t.w;
              float4* dst = use_ts32 ? reinterpret_cast<float4*>(ost_ptr(ch - c_beg, (uint32_t)u)) : o + u;
              *dst = make_float4(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
            }
            if (p.out16 != nullptr) {
              __align__(16) __half2 h2[8];
#pragma unroll
              for (int j = 0; j < 8; ++j)
                h2[j] = __floats2half2_rn(fminf(fmaxf(v[2 * j], -65504.f), 65504.f), fminf(fmaxf(v[2 * j + 1], -65504.f), 65504.f));
              uint4* o16 = reinterpret_cast<uint4*>(p.out16 + m * p.ld_out16 + n);
              o16[0] = reinterpret_cast<const uint4*>(h2)[0];
              o16[1] = reinterpret_cast<const uint4*>(h2)[1];
            }
            continue;
          }
          if (ACT != ACT_GELU && lean) {
            // whole-tile conv / GEMM with an fp16 output: bias, ReLU, optional fp16 residual from the prefetch ring, store
            const float4* sb4 = reinterpret_cast<const float4*>(sb + c);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float4 bq = sb4[u];
              v[4 * u + 0] += bq.x; v[4 * u + 1] += bq.y; v[4 * u + 2] += bq.z; v[4 * u + 3] += bq.w;
            }
            if (ACT == ACT_RELU) {
#pragma unroll
              for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
            }
            if (has_res) {
              __align__(16) __half h[16];
              if (p.resid_direct) {
                const uint4* rg = reinterpret_cast<const uint4*>(p.resid16 + m * p.ld_res16 + n);
                reinterpret_cast<uint4*>(h)[0] = __ldg(rg);
                reinterpret_cast<uint4*>(h)[1] = __ldg(rg + 1);
              } else {
                reinterpret_cast<uint4*>(h)[0] = *reinterpret_cast<const uint4*>(rb_ + ((size_t)(2 * ch) * 128 + row) * 16);
                reinterpret_cast<uint4*>(h)[1] = *reinterpret_cast<const uint4*>(rb_ + ((size_t)(2 * ch + 1) * 128 + row) * 16);
              }
#pragma unroll
              for (int j = 0; j < 16; ++j) v[j] += __half2float(h[j]);
            }
            __align__(16) __half2 h2[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              float a = fminf(v[2 * j], 65504.f), b2 = fminf(v[2 * j + 1], 65504.f);
              if (ACT == ACT_NONE || has_res) { a = fmaxf(a, -65504.f); b2 = fmaxf(b2, -65504.f); }
              h2[j] = __floats2half2_rn(a, b2);
            }
            if (use_ts) {
              *ost_ptr(ch - c_beg, 0) = reinterpret_cast<const uint4*>(h2)[0];
              *ost_ptr(ch - c_beg, 1) = reinterpret_cast<const uint4*>(h2)[1];
            } else {
              uint4* o = reinterpret_cast<uint4*>(p.out16 + m * p.ld_out16 + n);
              o[0] = reinterpret_cast<const uint4*>(h2)[0];
              o[1] = reinterpret_cast<const uint4*>(h2)[1];
            }
            continue;
          }
          if (n >= p.N) continue;  // uniform across the warp
          const int nval = min(16, p.N - n);   // 16 on every full chunk (all shipped tiny/pixelseal layers)
          {
            const float4* sb4 = reinterpret_cast<const float4*>(sb + c);
#pragma unroll
            for (int u = 0; u < 4; ++u) {
              const float4 bq = sb4[u];
              v[4 * u + 0] += bq.x; v[4 * u + 1] += bq.y; v[4 * u + 2] += bq.z; v[4 * u + 3] += bq.w;
            }
          }
          if (ACT == ACT_GELU) {
#pragma unroll
            for (int j = 0; j < 16; j += 2) gelu_erf2(v[j], v[j + 1]);
          } else if (ACT == ACT_RELU) {
#pragma unroll
            for (int j = 0; j < 16; ++j) v[j] = fmaxf(v[j], 0.f);
          }
          if (nval < 16) {
#pragma unroll
            for (int j = 0; j < 16; ++j) if (j >= nval) v[j] = 0.f;   // ragged last chunk (chunky widths): keep the tail inert
          }
          if (has_res && mvalid) {
            if (res_fast && !p.resid_direct) {
              if (p.resid16 != nullptr) {
                __align__(16) __half h[16];
                reinterpret_cast<uint4*>(h)[0] = *reinterpret_cast<const uint4*>(rb_ + ((size_t)(2 * ch) * 128 + row) * 16);
                reinterpret_cast<uint4*>(h)[1] = *reinterpret_cast<const uint4*>(rb_ + ((size_t)(2 * ch + 1) * 128 + row) * 16);
#pragma unroll
                for (int j = 0; j < 16; ++j) v[j] += __half2float(h[j]);
              } else {
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                  const float4 t = *reinterpret_cast<const float4*>(rb_ + ((size_t)(4 * ch + u) * 128 + row) * 16);
                  v[4 * u + 0] += t.x; v[4 * u + 1] += t.y; v[4 * u + 2] += t.z; v[4 * u + 3] += t.w;
                }
              }
            } else if (p.resid16 != nullptr) {
              const __half* r = p.resid16 + m * p.ld_res16 + n;
#pragma unroll
              for (int j = 0; j < 16; ++j) if (j < nval) v[j] += __half2float(r[j]);
            } else {
              const float* r = p.resid32 + m * p.ld_res32 + n;
#pragma unroll
              for (int j = 0; j < 16; ++j) if (j < nval) v[j] += r[j];
            }
          }
          if (p.outc_w != nullptr) {   // N <= 256 and a multiple of 16 here (host-checked): no tail
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              dot0 += v[j] * s_lnw[n + j];
              dot1 += v[j] * s_lnb[n + j];
              dot2 += v[j] * s_oc2[n + j];
            }
          }
          if (mvalid) {
            if (p.out16 != nullptr) {
              __half* o = p.out16 + m * p.ld_out16 + n;
              __align__(16) __half2 h[8];
#pragma unroll
              for (int j = 0; j < 8; ++j) {
                float a = fminf(v[2 * j], 65504.f), b2 = fminf(v[2 * j + 1], 65504.f);
                if (ACT == ACT_NONE || has_res) { a = fmaxf(a, -65504.f); b2 = fmaxf(b2, -65504.f); }   // ReLU >= 0, GELU >= -0.17
                h[j] = __floats2half2_rn(a, b2);
              }
              if (nval == 16) {
                reinterpret_cast<uint4*>(o)[0] = reinterpret_cast<const uint4*>(h)[0];
                reinterpret_cast<uint4*>(o)[1] = reinterpret_cast<const uint4*>(h)[1];
              } else {
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                  if (2 * j < nval) o[2 * j] = __low2half(h[j]);
                  if (2 * j + 1 < nval) o[2 * j + 1] = __high2half(h[j]);
                }
              }
            }
            if (p.out32 != nullptr) {
              float* o = p.out32 + m * p.ld_out32 + n;
              if (nval == 16) {
#pragma unroll
                for (int u = 0; u < 4; ++u)
                  reinterpret_cast<float4*>(o)[u] = make_float4(v[4 * u], v[4 * u + 1], v[4 * u + 2], v[4 * u + 3]);
              } else {
#pragma unroll
                for (int j = 0; j < 16; ++j) if (j < nval) o[j] = v[j];
              }
            }
          }
          if (p.grn_stats != nullptr) {
            // column sums of squares over this warp's 32 rows (GRN: ||x||_2 over H,W per (sample, channel))
            float sq[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) sq[j] = mvalid ? v[j] * v[j] : 0.f;
            if (grn_uniform) {
              // halving butterfly: after xor 16,8,4,2 each lane holds one column summed over 16 rows
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const float send = (lane & 16) ? sq[i] : sq[i + 8];
                const float keep = (lane & 16) ? sq[i + 8] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
              }
#pragma unroll
              for (int i = 0; i < 4; ++i) {
                const float send = (lane & 8) ? sq[i] : sq[i + 4];
                const float keep = (lane & 8) ? sq[i + 4] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
              }
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                const float send = (lane & 4) ? sq[i] : sq[i + 2];
                const float keep = (lane & 4) ? sq[i + 2] : sq[i];
                sq[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
              }
              {
                const float send = (lane & 2) ? sq[0] : sq[1];
                const float keep = (lane & 2) ? sq[1] : sq[0];
                sq[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
              }
              sq[0] += __shfl_xor_sync(0xffffffffu, sq[0], 1);
              const int col = (lane >> 1) & 15;
              if ((lane & 1) == 0 && col < nval) {
                if (p.grn_part) grn_row[n + col] = sq[0];
                else atomicAdd(grn_row + n + col, sq[0]);
              }
            } else if (mvalid) {
              float* gr = p.grn_stats + (long)p.fd_rps.div((int)m) * p.N + n;
#pragma unroll
              for (int j = 0; j < 16; ++j) if (j < nval) atomicAdd(gr + j, sq[j]);
            }
          }
        }
        if (use_ts || use_ts32) {
          // staging boxes complete: make the generic-proxy writes visible to the async proxy, then ONE lane hands the 32 x 16 boxes to
          // the TMA unit (full 32-byte sectors, no LSU tag traffic: the 16-byte-per-row register stores this replaces cost 32 tag
          // cycles per warp instruction and were the bottleneck of every short-K layer)
          fence_proxy_async_smem();
          __syncwarp();
          if (lane == 0) {
            for (int k = 0; k < c_end - c_beg; k += p.ost_cpb)
              tma_store_2d(&tmO, ost + (size_t)(p.ost_cpb == 1 ? k : 0) * ost_box, n0 + (c_beg + k) * 16, (int)(m - lane));
            bulk_commit_group();
          }
        }
        if (p.outc_w != nullptr) {
          // the warps sharing a row each hold a partial dot product: combine through shared memory
          if (half != 0) {
            float* d = s_dot + ((half - 1) * 128 + row) * 3;
            d[0] = dot0; d[1] = dot1; d[2] = dot2;
          }
          epi_bar_sync<kEpiThreads>();
          if (half == 0 && mvalid) {
#pragma unroll
            for (int h2 = 1; h2 < kEpiSplit; ++h2) {
              const float* d = s_dot + ((h2 - 1) * 128 + row) * 3;
              dot0 += d[0]; dot1 += d[1]; dot2 += d[2];
            }
            const int b = p.fd_hw.div((int)m), pix = (int)m - b * p.hw;
            const float dd[3] = {dot0, dot1, dot2};
#pragma unroll
            for (int o = 0; o < 3; ++o) {
              if (o < p.n_out) {
                float d = dd[o] + __ldg(p.outc_b + o);
                if (p.outc_tanh) d = tanhf(d);
                p.delta[((long)b * p.n_out + o) * p.hw + pix] = d;
              }
            }
          }
        }
      }
     }  // g
      mbar_arrive(tempty_bar);
      aphase ^= 1u;
      bsel ^= 1;
    }
    if (p.tma_store && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all stores of this warp have landed
  } else if (LOADER != LD_TMA && warp >= kBuilderWarp0) {
    // ===================================================================== A-tile builders (4 warps)
    const int gt = threadIdx.x - kBuilderWarp0 * 32;  // 0..127
    const int j = gt & 7;              // 16-byte chunk (8 fp16 K-elements) within the 128-byte swizzled row
    const int rg = gt >> 3;            // rows rg + 16*i
    int stage = 0;
    uint32_t phase = 0;
    if (kHalo) {
      const uint32_t pb = (uint32_t)p.cc * 2u;   // bytes per halo pixel
      int hb = 0;
      uint32_t hphase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
       for (int g = 0; g < p.group; ++g) {
        const int m_tile = p.fd_ntiles.div(tile) * p.group + g;
        if (m_tile >= p.m_tiles) break;
        int cy, cx;
        {
          const int b = p.fd_tpi.div(m_tile);
          const int rem = m_tile - b * p.tiles_per_img;
          const int ty = p.fd_tx.div(rem);
          cy = ty * p.tile_h;
          cx = (rem - ty * p.tiles_x) * p.tile_w;
        }
        for (int c = 0; c < p.c_blocks; ++c) {
          mbar_wait(&hfull_bar[hb], hphase);
          const uint8_t* hsrc = halo + (size_t)hb * p.halo_stride;
          // tap tiles.  K-block kbi of this chunk holds K indices [64*kbi, 64*kbi+64) of the (tap, channel)
          // order; 16-byte chunk j covers k = 64*kbi + 8*j -> tap = k / cc, channel offset = k % cc
          const int stage0 = stage;
          const uint32_t phase0 = phase;
          for (int kbi = 0; kbi < p.kb_per_c; ++kbi) {
            const int k = kbi * 64 + j * 8;
            const int tap = p.fd_cc.div(k);
            const int coff = (k - tap * p.cc) * 2;
            const int tr = tap / 3, ts = tap - tr * 3;
            mbar_wait(&empty_bar[stage], phase ^ 1u);
            uint8_t* sa = tiles + (size_t)stage * p.stage_bytes;
            if (tap < 9) {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int r = rg + 16 * i;
                const int ry = r >> 4, rx = r & 15;
                const uint4 val = *reinterpret_cast<const uint4*>(hsrc + (size_t)((ry + tr) * kHaloW + rx + ts) * pb + coff);
                *reinterpret_cast<uint4*>(sa + r * 128 + ((j ^ (r & 7)) << 4)) = val;
              }
            } else {
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int r = rg + 16 * i;
                *reinterpret_cast<uint4*>(sa + r * 128 + ((j ^ (r & 7)) << 4)) = make_uint4(0, 0, 0, 0);
              }
            }
            if (p.kb_per_c > p.stages) {   // ring shorter than the chunk: publish each K-block immediately
              fence_proxy_async_smem();
              mbar_arrive(&full_bar[stage]);
            }
            if (++stage == p.stages) { stage = 0; phase ^= 1u; }
          }
          if (p.kb_per_c <= p.stages) {
            // one generic->async proxy fence for the whole chunk, then publish its K-blocks
            fence_proxy_async_smem();
            int sp = stage0;
            for (int kbi = 0; kbi < p.kb_per_c; ++kbi) {
              mbar_arrive(&full_bar[sp]);
              if (++sp == p.stages) sp = 0;
            }
          }
          (void)phase0;
          mbar_arrive(&hempty_bar[hb]);
          if (++hb == p.halo_bufs) { hb = 0; hphase ^= 1u; }
        }
       }
      }
    } else {
      const int Ct = p.C0 + p.C1;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
       for (int g = 0; g < p.group; ++g) {
        const int m_tile = p.fd_ntiles.div(tile) * p.group + g;
        if (m_tile >= p.m_tiles) break;
        int pb[8], py[8], px[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int m = m_tile * kBlockM + rg + 16 * i;      // M < 2^31 (host-checked)
          if (m < p.M) {
            const int t = p.fd_ow.div(m);
            px[i] = m - t * p.OW;
            pb[i] = p.fd_oh.div(t);
            py[i] = t - pb[i] * p.OH;
          } else {
            pb[i] = -1; py[i] = 0; px[i] = 0;
          }
        }
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = tiles + (size_t)stage * p.stage_bytes;
          const int k = kb * 64 + j * 8;
          const bool kvalid = k < p.Ktot;
          const int tap = kvalid ? p.fd_ct.div(k) : 0;
          const int c = k - tap * Ct;
          const int tr = p.fd_s.div(tap), ts = tap - tr * p.S;
          const __half* src = (c < p.C0) ? p.src0 : p.src1;
          const int ld = (c < p.C0) ? p.ld0 : p.ld1;
          const int cc = (c < p.C0) ? c : c - p.C0;
          // asynchronous gather: 16-byte cp.async per (row, chunk) with zero fill for padding / tails; the mbarrier
          // arrival fires when this thread's copies have landed, so the builder runs ahead by the ring depth
#pragma unroll
          for (int i = 0; i < 8; ++i) {
            const __half* gsrc = p.src0;   // always a valid address (no bytes are read when nbytes == 0)
            uint32_t nbytes = 0;
            if (kvalid && pb[i] >= 0) {
              int iy = py[i] * p.stride + tr - p.pad;
              int ix = px[i] * p.stride + ts - p.pad;
              bool ok = true;
              if (p.pad_mode == 1) {
                iy = reflect_idx(iy, p.IH);
                ix = reflect_idx(ix, p.IW);
              } else if (p.pad_mode == 2) {   // zero padding around the nearest x2 up-sample of the 2x smaller source
                ok = (iy >= 0) && (iy < 2 * p.IH) && (ix >= 0) && (ix < 2 * p.IW);
                iy >>= 1; ix >>= 1;
              } else {
                ok = (iy >= 0) && (iy < p.IH) && (ix >= 0) && (ix < p.IW);
              }
              if (ok) { gsrc = src + (((long)pb[i] * p.IH + iy) * p.IW + ix) * ld + cc; nbytes = 16; }
            }
            const int r = rg + 16 * i;
            cp_async16_zfill(sa + r * 128 + ((j ^ (r & 7)) << 4), gsrc, nbytes);
          }
          cp_async_mbar_arrive_noinc(&full_bar[stage]);
          if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
       }
      }
    }
  }

  __syncthreads();
}

// ------------------------------------------------------------------------------------------------------------------------------
// Long-K variant of the LD_TMA kernel: 256 x BN output tiles, the accumulators stay in registers through the epilogue.
//
//   warpgroup 0    : producer; gives its registers away (setmaxnreg) and one elected thread runs the TMA loop: per K block of 64
//                    a [256 x 64] A tile (one box: tile_h x tile_w = 256 pixels of the map, or 256 GEMM rows) and a [BN x 64] B tile
//                    (of the tile's sample with per-sample weights)
//   warpgroups 1,2 : consumers; warpgroup h owns rows [128h, 128h + 128) of the tile as two m64 wgmma chains that read the same B
//                    tile, 2 x BN / 2 accumulators per thread, and runs the epilogue of its rows straight from the fragments.  Chain c
//                    reads the 8-row groups 2g + c (g = 0..7) of the warpgroup's rows (descriptor group stride 2048 B), so warp wq
//                    holds the 32 consecutive rows [32 wq, 32 wq + 32): fragment half hh of chain c is row 32 wq + 8c + 16hh + lane / 4.
//   epilogues      : F32 = false, ACT ReLU / none: acc + bias -> ReLU -> + fp16 residual -> clamp -> fp16
//                    F32 = false, ACT GELU:        acc + bias -> GELU -> fp16, and the column sums of squares of every 32 rows (GRN
//                                                  partial rows, [M / 32][N])
//                    F32 = true (ACT none):        fp32 stream += acc + bias in place (pwconv2), optional fp16 copy
//                    fp16 outputs are staged per warp in swizzled [8 rows] boxes that leave through TMA stores.
//
// Against the 128-row kernel a K block moves 48 KB instead of 2 x 32 KB from L2 for the same 4.2 MFLOP, a pipeline stage is worth
// twice the MMA time, and no accumulator crosses shared memory.  The price: a warpgroup's epilogue does not overlap its own next
// main loop (the producer keeps filling the ring meanwhile).  The K-block order, the k16 order inside a block, the epilogue
// arithmetic and the order of the GRN row sums (32 rows paired by row bit 4, 3, 2, 1, 0) are those of conv_gemm_kernel's lean
// paths: both kernels produce the same bits.
//
// BN = 192 (lean affine epilogue only): a K block moves 32 KB of A and 24 KB of B for 6.3 MFLOP, 0.78x the operand bytes per FLOP of
// BN = 128.  Shared memory: 1 KB barriers + 3 stages x 56 KB + 8 warps x 6 KB staging (one chain's [16 rows][192] fp16) = 217 KB,
// + 1 KB alignment slack <= 227 KB.  Each consumer thread holds 2 x 96 accumulators in the 232 registers setmaxnreg gives it.
constexpr int kLongM = 256;
constexpr int kLongThreads = 384;
constexpr int kLongHeaderBytes = 1024;                // full / empty barriers
constexpr int kLongWideN = 192;                       // the widest block_n (lean affine epilogue only)
// staging of one consumer warp: one chain's [16 rows][BN] fp16, 4 KB for every block_n up to 128 and 6 KB at kLongWideN
__host__ __device__ constexpr uint32_t long_ost_warp_bytes(int bn) { return 16u * (uint32_t)(bn > kMaxBlockN ? bn : kMaxBlockN) * 2u; }
constexpr int kLongConsumerWarps = 8;

// read-only global loads that keep their place among the barrier / wgmma statements
__device__ __forceinline__ uint32_t ld_nc_u32(const void* g) {
  uint32_t v;
  asm volatile("ld.global.nc.b32 %0, [%1];" : "=r"(v) : "l"(g));
  return v;
}
__device__ __forceinline__ float2 ld_nc_f32x2(const float* g) {
  float2 v;
  asm volatile("ld.global.nc.v2.f32 {%0, %1}, [%2];" : "=f"(v.x), "=f"(v.y) : "l"(g));
  return v;
}

template <int BN, int ACT, bool F32 = false>
__global__ void __launch_bounds__(kLongThreads, 1)
conv_gemm_longk_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                       const __grid_constant__ CUtensorMap tmO, const __grid_constant__ ConvGemmParams p) {
  static_assert(!F32 || ACT == ACT_NONE, "the fp32 residual-stream epilogue has no activation");
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem);
  uint64_t* empty_bar = full_bar + kMaxStages;
  uint8_t* tiles = smem + kLongHeaderBytes;
  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(&full_bar[s], 1u);
      mbar_init(&empty_bar[s], (uint32_t)kLongConsumerWarps);
    }
    fence_barrier_init();
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    if (!F32) tma_prefetch_desc(&tmO);
  }
  __syncthreads();
  // nothing above reads or writes a tensor produced by an earlier kernel
  pdl_launch_dependents();
  pdl_wait();

  if (warp < 4) {
    // ===================================================================== TMA producer
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const int m_tile = p.fd_ntiles.div(tile);
        const int brow = (tile - m_tile * p.n_tiles) * BN + (p.b_sample_rows ? p.fd_tps.div(m_tile) * p.b_sample_rows : 0);
        int cb = 0, cx = 0, cy = 0;
        if (p.a_is_conv) {
          cb = p.fd_tpi.div(m_tile);
          const int rem = m_tile - cb * p.tiles_per_img;
          const int ty = p.fd_tx.div(rem);
          cy = ty * p.tile_h;
          cx = (rem - ty * p.tiles_x) * p.tile_w;
        }
        int tap_r = 0, tap_s = 0, cblk = 0;
        for (int kb = 0; kb < p.num_kb; ++kb) {
          mbar_wait(&empty_bar[stage], phase ^ 1u);
          uint8_t* sa = tiles + (size_t)stage * p.stage_bytes;
          mbar_arrive_expect_tx(&full_bar[stage], p.a_stage_bytes + p.b_stage_bytes);
          if (p.a_is_conv) {
            tma_load_4d(&tmA, &full_bar[stage], sa, cblk * 64, cx + tap_s - p.pad, cy + tap_r - p.pad, cb);
            if (++cblk == p.c_blocks) { cblk = 0; if (++tap_s == p.S) { tap_s = 0; ++tap_r; } }
          } else {
            tma_load_2d(&tmA, &full_bar[stage], sa, kb * 64, m_tile * kLongM);
          }
          tma_load_2d(&tmB, &full_bar[stage], sa + p.a_stage_bytes, kb * 64, brow);
          if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    // ===================================================================== consumers: MMA + epilogue of rows [128h, 128h + 128)
    setmaxnreg_inc<232>();
    const int h = (warp >> 2) - 1, wq = warp & 3;
    const int rl = lane >> 2, q = lane & 3;
    // staging boxes of this warp: [BN / kBoxCols][2 halves] boxes of [8 rows][kBoxCols] fp16 in the TMA swizzle of that row width;
    // the 4-byte stores of a warp instruction (8 rows x 4 lanes) fall into 32 different banks
    constexpr int kBoxCols = BN % 64 == 0 ? 64 : 16;
    constexpr uint32_t kBoxRowB = kBoxCols * 2, kBoxBytes = 8 * kBoxRowB;
    const uint32_t swz_x = kBoxCols == 64 ? (uint32_t)rl : (uint32_t)((rl >> 2) & 1);
    uint8_t* ost = smem + p.ostage_off + (size_t)(warp - 4) * long_ost_warp_bytes(BN);
    auto box_ptr = [&](int j /*8-column group*/, int hh) -> uint8_t* {
      return ost + (uint32_t)(((8 * j) / kBoxCols) * 2 + hh) * kBoxBytes + (uint32_t)rl * kBoxRowB +
             (((uint32_t)(((8 * j) % kBoxCols) >> 3) ^ swz_x) << 4) + 4u * q;
    };
    const bool has_res = !F32 && p.resid16 != nullptr;
    constexpr uint32_t kRowBytes = 128;                           // K block of 64 fp16
    const uint32_t a_off = (uint32_t)h * 128u * kRowBytes;
    float d[2][BN / 2];
    // The fp16 affine epilogue walks the 2 x BN / 8 eight-column groups of the two chains in kGrp-sized steps; the bias pairs and
    // residual half2 of step t + 1 are loaded while step t is converted.  Only two steps' worth sit in registers beside the
    // 2 x BN / 2 accumulators (the whole tile's would not fit), and the loads are ordered statements so that they stay where they
    // are put.
    constexpr int kGrp = BN > kMaxBlockN ? 2 : (BN % 32 == 0 ? 4 : 5), kSteps = BN / 8 / kGrp;     // steps per chain
    static_assert(kGrp * kSteps * 8 == BN, "block_n must split into whole epilogue steps");
    float2 gb0[kGrp], gb1[kGrp];
    uint32_t gr0[2 * kGrp], gr1[2 * kGrp];
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const int m_tile = p.fd_ntiles.div(tile), n0 = (tile - m_tile * p.n_tiles) * BN;
      const long m_warp = (long)m_tile * kLongM + h * 128 + wq * 32;     // first of this warp's 32 rows
      int prev = -1;
      for (int kb = 0; kb < p.num_kb; ++kb) {
        // 192 accumulators per thread only stay in registers with the watchdog's trap out of line (mbar_wait_cold_trap)
        if constexpr (BN > kMaxBlockN) mbar_wait_cold_trap(&full_bar[stage], phase);
        else mbar_wait(&full_bar[stage], phase);
        const uint32_t sa = smem_u32(tiles + (size_t)stage * p.stage_bytes);
        const uint64_t adesc0 = make_smem_desc(sa + a_off, kRowBytes, 16 * kRowBytes);
        const uint64_t adesc1 = make_smem_desc(sa + a_off + 8u * kRowBytes, kRowBytes, 16 * kRowBytes);
        const uint64_t bdesc = make_smem_desc(sa + p.a_stage_bytes, kRowBytes);
        wgmma_fence_regs(d[0]);
        wgmma_fence_regs(d[1]);
        wgmma_fence();
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          // advance 16 K-elements = 32 bytes inside the swizzled row: +2 in the (addr >> 4) field
          Wgmma<BN>::mma(d[0], adesc0 + (uint64_t)(2 * j), bdesc + (uint64_t)(2 * j), (uint32_t)((kb | j) != 0));
          Wgmma<BN>::mma(d[1], adesc1 + (uint64_t)(2 * j), bdesc + (uint64_t)(2 * j), (uint32_t)((kb | j) != 0));
        }
        wgmma_commit();
        wgmma_fence_regs(d[0]);
        wgmma_fence_regs(d[1]);
        if (prev >= 0) {
          wgmma_wait<1>();   // the previous K-block's wgmma have read their slot
          __syncwarp();
          if (lane == 0) mbar_arrive(&empty_bar[prev]);
        }
        prev = stage;
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
      }
      // TMA stores of chain c's staging boxes
      auto store_chain = [&](int c) {
        fence_proxy_async_smem();     // generic-proxy writes of the staging boxes -> async proxy
        __syncwarp();
        if (lane == 0) {
#pragma unroll
          for (int b = 0; b < BN / kBoxCols; ++b)
#pragma unroll
            for (int hh = 0; hh < 2; ++hh)
              tma_store_2d(&tmO, ost + (2 * b + hh) * kBoxBytes, n0 + b * kBoxCols, (int)(m_warp + 8 * c + 16 * hh));
          bulk_commit_group();
        }
      };
      if (F32) {
        // pwconv2: the fp32 residual stream, read and written in place by the same thread, += acc + bias (+ fp16 copy).  Row t =
        // (chain t / 2, half t % 2) of the thread: its residual is loaded while the last wgmma group drains (t = 0) or, below
        // block_n 128 (where a second row buffer fits in registers), while row t - 1 is written.
        constexpr bool kPipe = BN < 128;
        float2 ra[BN / 8], rb[kPipe ? BN / 8 : 1];
        auto load_row = [&](float2 (&r)[BN / 8], int t) {
          const float* rr = p.resid32 + (m_warp + 8 * (t >> 1) + 16 * (t & 1) + rl) * p.ld_res32 + n0 + 2 * q;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) r[j] = *reinterpret_cast<const float2*>(rr + 8 * j);
        };
        auto store_row = [&](const float2 (&r)[BN / 8], int t) {
          const int c = t >> 1, hh = t & 1;
          const long row = m_warp + 8 * c + 16 * hh + rl;
          float* o = p.out32 + row * p.ld_out32 + n0 + 2 * q;
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const float2 b = p.bias != nullptr ? ld_nc_f32x2(p.bias + n0 + 8 * j + 2 * q) : make_float2(0.f, 0.f);
            const float v0 = d[c][4 * j + 2 * hh] + (b.x + r[j].x), v1 = d[c][4 * j + 2 * hh + 1] + (b.y + r[j].y);
            *reinterpret_cast<float2*>(o + 8 * j) = make_float2(v0, v1);
            if (p.out16 != nullptr)
              *reinterpret_cast<__half2*>(p.out16 + row * p.ld_out16 + n0 + 8 * j + 2 * q) =
                  __floats2half2_rn(fminf(fmaxf(v0, -65504.f), 65504.f), fminf(fmaxf(v1, -65504.f), 65504.f));
          }
        };
        load_row(ra, 0);
        wgmma_wait<0>();
        wgmma_fence_regs(d[0]);
        wgmma_fence_regs(d[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
        if constexpr (kPipe) {
          load_row(rb, 1);
          store_row(ra, 0);
          load_row(ra, 2);
          store_row(rb, 1);
          load_row(rb, 3);
          store_row(ra, 2);
          store_row(rb, 3);
        } else {
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            if (t > 0) load_row(ra, t);
            store_row(ra, t);
          }
        }
      } else if (ACT == ACT_GELU) {
        // pwconv1: bias + GELU + fp16 store, then the GRN column sums of squares of the warp's 32 rows
        wgmma_wait<0>();
        wgmma_fence_regs(d[0]);
        wgmma_fence_regs(d[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          if (lane == 0) bulk_wait_group_read0();     // the previous stores of this warp have finished reading the staging boxes
          __syncwarp();
#pragma unroll
          for (int j = 0; j < BN / 8; ++j) {
            const float2 b = p.bias != nullptr ? ld_nc_f32x2(p.bias + n0 + 8 * j + 2 * q) : make_float2(0.f, 0.f);
#pragma unroll
            for (int hh = 0; hh < 2; ++hh) {
              const float2 w = gelu_erf_p(f2add(make_float2(d[c][4 * j + 2 * hh], d[c][4 * j + 2 * hh + 1]), b));
              d[c][4 * j + 2 * hh] = w.x; d[c][4 * j + 2 * hh + 1] = w.y;
              uint32_t hv;
              asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(hv) : "f"(w.y), "f"(w.x));   // {hi, lo}
              *reinterpret_cast<uint32_t*>(box_ptr(j, hh)) = hv;
            }
          }
          store_chain(c);
        }
        if (p.grn_stats != nullptr) {
          // row x of the 32 is (c, hh, rl) = (bit 3, bit 4, bits 0-2): pair rows x, x + 16 (hh), then x, x + 8 (c) in the thread,
          // then rows 4, 2, 1 apart across lanes 16, 8, 4 apart (halving butterfly).  Column of value i: 8 (i / 2) + 2q + i % 2.
          constexpr int kV = BN / 4;
          float s[kV];
#pragma unroll
          for (int i = 0; i < kV; ++i) {
            const int k = 4 * (i >> 1) + (i & 1);
            const float t0 = __fmul_rn(d[0][k], d[0][k]) + __fmul_rn(d[0][k + 2], d[0][k + 2]);
            const float t1 = __fmul_rn(d[1][k], d[1][k]) + __fmul_rn(d[1][k + 2], d[1][k + 2]);
            s[i] = t0 + t1;
          }
          int base = 0;
#pragma unroll
          for (int i = 0; i < kV / 2; ++i) {
            const float send = (lane & 16) ? s[i] : s[i + kV / 2];
            const float keep = (lane & 16) ? s[i + kV / 2] : s[i];
            s[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
          }
          if (lane & 16) base += kV / 2;
#pragma unroll
          for (int i = 0; i < kV / 4; ++i) {
            const float send = (lane & 8) ? s[i] : s[i + kV / 4];
            const float keep = (lane & 8) ? s[i + kV / 4] : s[i];
            s[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
          }
          if (lane & 8) base += kV / 4;
#pragma unroll
          for (int i = 0; i < kV / 8; ++i) {
            const float send = (lane & 4) ? s[i] : s[i + kV / 8];
            const float keep = (lane & 4) ? s[i + kV / 8] : s[i];
            s[i] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
          }
          if (lane & 4) base += kV / 8;
          float* grow = p.grn_stats + (m_warp >> 5) * p.N + n0 + 2 * q;
#pragma unroll
          for (int i = 0; i < kV / 8; ++i) {
            const int v = base + i;
            grow[8 * (v >> 1) + (v & 1)] = s[i];
          }
        }
      } else {
        auto load_step = [&](float2 (&gb)[kGrp], uint32_t (&gr)[2 * kGrp], int t) {
          const int c = t / kSteps, j0 = (t % kSteps) * kGrp;
          const __half* r0 = p.resid16 + (m_warp + 8 * c + rl) * p.ld_res16 + n0 + 8 * j0 + 2 * q;
          const __half* r1 = r0 + 16 * (long)p.ld_res16;
#pragma unroll
          for (int jj = 0; jj < kGrp; ++jj) {
            gb[jj] = p.bias != nullptr ? ld_nc_f32x2(p.bias + n0 + 8 * (j0 + jj) + 2 * q) : make_float2(0.f, 0.f);
            if (has_res) {
              gr[2 * jj] = ld_nc_u32(r0 + 8 * jj);
              gr[2 * jj + 1] = ld_nc_u32(r1 + 8 * jj);
            }
          }
        };
        load_step(gb0, gr0, 0);       // in flight while the last wgmma group drains
        wgmma_wait<0>();
        wgmma_fence_regs(d[0]);
        wgmma_fence_regs(d[1]);
        __syncwarp();
        if (lane == 0) mbar_arrive(&empty_bar[prev]);
#pragma unroll
        for (int t = 0; t < 2 * kSteps; ++t) {
          const int c = t / kSteps, g = t % kSteps;
          if (g == 0) {
            if (lane == 0) bulk_wait_group_read0();     // the previous stores of this warp have finished reading the staging boxes
            __syncwarp();
          }
          auto convert_step = [&](const float2 (&gb)[kGrp], const uint32_t (&gr)[2 * kGrp]) {
#pragma unroll
            for (int jj = 0; jj < kGrp; ++jj) {
              const int j = g * kGrp + jj;
#pragma unroll
              for (int hh = 0; hh < 2; ++hh) {
                float v0 = d[c][4 * j + 2 * hh] + gb[jj].x, v1 = d[c][4 * j + 2 * hh + 1] + gb[jj].y;
                if (ACT == ACT_RELU) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
                if (has_res) {
                  const uint32_t rbits = gr[2 * jj + hh];
                  const float2 rf = __half22float2(*reinterpret_cast<const __half2*>(&rbits));
                  v0 += rf.x; v1 += rf.y;
                }
                v0 = fminf(v0, 65504.f); v1 = fminf(v1, 65504.f);
                if (ACT == ACT_NONE || has_res) { v0 = fmaxf(v0, -65504.f); v1 = fmaxf(v1, -65504.f); }   // ReLU >= 0
                *reinterpret_cast<__half2*>(box_ptr(j, hh)) = __floats2half2_rn(v0, v1);
              }
            }
          };
          if ((t & 1) == 0) {
            if (t + 1 < 2 * kSteps) load_step(gb1, gr1, t + 1);
            convert_step(gb0, gr0);
          } else {
            if (t + 1 < 2 * kSteps) load_step(gb0, gr0, t + 1);
            convert_step(gb1, gr1);
          }
          if (g == kSteps - 1) store_chain(c);
        }
      }
    }
    if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all stores of this warp have landed
  }
}

}  // namespace vsb
