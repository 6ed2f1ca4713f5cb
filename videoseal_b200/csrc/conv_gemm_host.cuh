// Host-side construction + launch of conv_gemm_kernel instances (tensor maps, tiling, smem budget).
#pragma once
#include <atomic>
#include <cstdio>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "conv_gemm.cuh"

namespace vsb {

// status codes of include/vsb200.h (static_assert-ed equal in vsb200.cu): every throw site names its code, the C ABI returns it
enum : int { kErrInvalid = -1, kErrUnsupported = -2, kErrCuda = -3, kErrState = -4 };
struct Error : std::runtime_error {
  int code;
  explicit Error(const std::string& m, int c = kErrInvalid) : std::runtime_error(m), code(c) {}
};

#define VSB_CHECK(cond, msg)                                                                      \
  do {                                                                                            \
    if (!(cond)) throw ::vsb::Error(std::string(msg) + " [" #cond "] at " __FILE__ ":" + std::to_string(__LINE__)); \
  } while (0)

#define VSB_CUDA(expr)                                                                            \
  do {                                                                                            \
    cudaError_t _e = (expr);                                                                      \
    if (_e != cudaSuccess)                                                                        \
      throw ::vsb::Error(std::string("CUDA error ") + cudaGetErrorString(_e) + " in " #expr " at " __FILE__ ":" + std::to_string(__LINE__), ::vsb::kErrCuda); \
  } while (0)

// device allocations owned by one object, freed together
struct DevicePool {
  std::vector<void*> ptrs;
  void* alloc(size_t n) {
    void* p = nullptr;
    n = (n + 255) & ~size_t(255);
    if (n == 0) n = 256;
    VSB_CUDA(cudaMalloc(&p, n));
    ptrs.push_back(p);
    return p;
  }
  template <class T> T* alloc_n(size_t n) { return reinterpret_cast<T*>(alloc(n * sizeof(T))); }
  // zeroed before it returns: plans run on the caller's stream, which need not be ordered after stream 0
  template <class T> T* alloc_zeroed(size_t n) {
    T* p = alloc_n<T>(n);
    VSB_CUDA(cudaMemset(p, 0, n * sizeof(T)));
    VSB_CUDA(cudaDeviceSynchronize());
    return p;
  }
  template <class T> T* upload(const std::vector<T>& v) {
    T* p = alloc_n<T>(v.size());
    VSB_CUDA(cudaMemcpy(p, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice));
    return p;
  }
  ~DevicePool() { for (void* p : ptrs) cudaFree(p); }
};

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                    const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                    CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    VSB_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q));
    VSB_CHECK(p != nullptr && q == cudaDriverEntryPointSuccess, "cuTensorMapEncodeTiled not available");
    fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

inline CUtensorMapSwizzle swizzle_for(int kblk) {
  return kblk == 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (kblk == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
}

// fp16 (or fp32: f32 = true, always unswizzled) tensor map, dims innermost-first; strides (bytes) for dims 1..rank-1
inline void encode_map(CUtensorMap* tm, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                       const uint32_t* box, int kblk, bool no_swizzle = false, bool f32 = false, int swz_bytes = -1 /* >= 0: explicit 0/32/64/128 */) {
  cuuint64_t gd[5], gs[4];
  cuuint32_t bx[5], es[5];
  for (int i = 0; i < rank; ++i) { gd[i] = dims[i]; bx[i] = box[i]; es[i] = 1; }
  for (int i = 0; i + 1 < rank; ++i) gs[i] = strides_bytes[i];
  VSB_CHECK((reinterpret_cast<uintptr_t>(base) & 15) == 0, "TMA base must be 16B aligned");
  for (int i = 0; i + 1 < rank; ++i) VSB_CHECK(gs[i] % 16 == 0, "TMA strides must be multiples of 16B");
  CUresult r = get_encode_fn()(tm, f32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank,
                               const_cast<void*>(base), gd, gs, bx, es,
                               CU_TENSOR_MAP_INTERLEAVE_NONE,
                               swz_bytes >= 0 ? (swz_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : swz_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B
                                                 : swz_bytes == 32 ? CU_TENSOR_MAP_SWIZZLE_32B : CU_TENSOR_MAP_SWIZZLE_NONE)
                                              : ((no_swizzle || f32) ? CU_TENSOR_MAP_SWIZZLE_NONE : swizzle_for(kblk)),
                               CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  VSB_CHECK(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (" + std::to_string((int)r) + ")");
}

inline FastDiv make_fastdiv(int d) {
  FastDiv f; f.d = d < 1 ? 1 : d; f.mul = 0; f.shr = 0;
  if (f.d > 1) {
    int l = 0; while ((1u << l) < (uint32_t)f.d) ++l;       // ceil(log2 d)
    const int pp = 31 + l;
    const unsigned long long m = ((1ull << pp) + (unsigned long long)f.d - 1) / (unsigned long long)f.d;
    f.mul = (uint32_t)m; f.shr = (uint32_t)(pp - 32);
  }
  return f;
}

struct ConvGemmOp {
  int loader = LD_TMA;
  ConvGemmParams p;
  CUtensorMap tmA, tmA2, tmB, tmO;
  int grid = 0, threads = 0;
  int w_samples = 1;   // > 1: weights are [w_samples][N][K], sample = row / rows_per_sample (finalize_op)
  size_t smem = 0;
  const char* name = "";
  // the A operand as setup_tma_conv / setup_tma_gemm encoded it (a_rank 4 / 2; 0: another loader or the two-source GEMM), kept so
  // that finalize_op can encode the same tensor with the 256-row box of the long-K kernel
  const void* a_base = nullptr;
  int a_rank = 0;
  uint64_t a_dims[4] = {0, 0, 0, 0}, a_strides[3] = {0, 0, 0};
  int longk = 0;       // 1: conv_gemm_longk_kernel runs this op (finalize_op)
  ConvGemmOp() { memset(&p, 0, sizeof(p)); memset(&tmA, 0, sizeof(tmA)); memset(&tmA2, 0, sizeof(tmA2)); memset(&tmB, 0, sizeof(tmB)); memset(&tmO, 0, sizeof(tmO)); }
};

// the largest tile in {max_bn, ..., 32} (multiples of 16) that divides N rounded up to 16; else max_bn with a ragged last tile
inline int pick_block_n(int N, int max_bn = kMaxBlockN) {
  const int n16 = (N + 15) / 16 * 16;
  if (n16 <= max_bn) return n16;
  for (int bn = max_bn / 16 * 16; bn >= 32; bn -= 16)
    if (n16 % bn == 0) return bn;
  return max_bn / 16 * 16;
}

// ---- the long-K kernel (conv_gemm_longk_kernel): which ops may run on it, and its tiling / shared-memory plan
enum : int { kKernelAuto = 0, kKernel128 = 1, kKernelLongK = 2 };   // kernel_sel of finalize_op (1, 2: test seam of vsb_debug_conv)

// 256-pixel patch of an H x W map as one TMA box (each box dimension <= 256); false when the map does not tile by it
inline bool longk_conv_tile(int H, int W, int& tile_w, int& tile_h) {
  tile_w = W < kLongM ? W : kLongM;
  tile_h = kLongM / tile_w;
  return tile_w * tile_h == kLongM && W % tile_w == 0 && H % tile_h == 0;
}

// The output-tile width the long-K kernel would run this op at, or 0 when it cannot run it.  Everything but the tile count: a
// TMA-fed op with 64-wide K blocks in whole 256-row tiles, and one of the kernel's epilogues at a width it is instantiated for:
//   - the lean affine one (bias, ReLU or none, optional fp16 residual, fp16 output) on long main loops, at the 128-row kernel's
//     block_n (128 or 80), or at kLongWideN (192) where that block_n is 128, N splits into 192-wide tiles and those still make
//     at least two tiles per SM: a 256 x 192 tile moves 56 KB per K block for 3.1 M MACs where 256 x 128 moves 48 KB for 2.1 M;
//   - ConvNeXt pwconv1: bias + GELU, fp16 output, GRN statistics as per-32-row partial rows, block_n 128 (the float-atomic GRN
//     mode and GELU GEMMs without GRN, the ViT MLP, stay on the 128-row kernel: not measured on this one);
//   - ConvNeXt pwconv2: no activation, fp32 residual stream updated in place, optional fp16 copy, per-sample weights whose samples
//     are whole 256-row tiles, block_n 128 or 96.
// longk_bn (test seam of vsb_debug_conv): 0 = choose as above, else the long-K width to take (0 is returned when the op cannot run
// at it).  It does not change the 128-row kernel's block_n, which block_n_override sets.
inline int longk_block_n(const ConvGemmOp& op, int N, int block_n_override, int num_sms, int longk_bn = 0) {
  const ConvGemmParams& p = op.p;
  int tw, th;
  if (!(op.loader == LD_TMA && op.a_rank != 0 && p.kblk == 64 && p.num_kb >= 2 && p.epi == EPI_AFFINE && p.outc_w == nullptr &&
        p.M % kLongM == 0 && (reinterpret_cast<uintptr_t>(p.bias) & 7) == 0 && (!p.a_is_conv || longk_conv_tile(p.H, p.W, tw, th))))
    return 0;
  const bool out16_ok = p.out16 != nullptr && (reinterpret_cast<uintptr_t>(p.out16) & 15) == 0 && p.ld_out16 % 8 == 0;
  int bn = 0;
  if (p.act == ACT_GELU) {
    if (out16_ok && p.out32 == nullptr && p.resid16 == nullptr && p.resid32 == nullptr && op.w_samples == 1 &&
        p.grn_stats != nullptr && p.grn_part && p.rows_per_sample > 0 && p.rows_per_sample % 32 == 0)
      bn = 128;
  } else if (p.resid32 != nullptr) {
    if (p.act == ACT_NONE && p.out32 != nullptr && p.resid16 == nullptr && p.grn_stats == nullptr &&
        (reinterpret_cast<uintptr_t>(p.out32) & 7) == 0 && p.ld_out32 % 2 == 0 &&
        (reinterpret_cast<uintptr_t>(p.resid32) & 7) == 0 && p.ld_res32 % 2 == 0 &&
        (p.out16 == nullptr || ((reinterpret_cast<uintptr_t>(p.out16) & 3) == 0 && p.ld_out16 % 2 == 0)) &&
        (op.w_samples == 1 || (!p.a_is_conv && p.rows_per_sample > 0 && p.rows_per_sample % kLongM == 0)))
      bn = N % 128 == 0 ? 128 : (N % 96 == 0 ? 96 : 0);
  } else if (p.num_kb >= 24 && (p.act == ACT_NONE || p.act == ACT_RELU) && out16_ok && p.out32 == nullptr && p.grn_stats == nullptr &&
             op.w_samples == 1 && (p.resid16 == nullptr || ((reinterpret_cast<uintptr_t>(p.resid16) & 3) == 0 && p.ld_res16 % 8 == 0)) &&
             (p.block_n == 128 || p.block_n == 80)) {
    bn = p.block_n;
    if (bn == 128 && block_n_override == 0 && N % kLongWideN == 0 &&
        (longk_bn == kLongWideN || (longk_bn == 0 && (long)(p.M / kLongM) * (N / kLongWideN) >= 2L * num_sms)))
      bn = kLongWideN;
  }
  if (bn == 0 || N % bn != 0 || (block_n_override != 0 && block_n_override != bn) || (longk_bn != 0 && longk_bn != bn)) return 0;
  return bn;
}

inline void finalize_longk(ConvGemmOp& op, const __half* W, int N, int Kw, int ldw, int num_sms, int block_n) {
  ConvGemmParams& p = op.p;
  op.longk = 1;
  p.block_n = block_n;
  p.n_tiles = N / block_n;
  p.group = 1;
  p.m_tiles = p.M / kLongM;
  p.num_tiles = p.m_tiles * p.n_tiles;
  uint32_t abox[4] = {64u, (uint32_t)kLongM, 1u, 1u};
  if (p.a_is_conv) {
    longk_conv_tile(p.H, p.W, p.tile_w, p.tile_h);
    p.tiles_x = p.W / p.tile_w;
    p.tiles_per_img = p.tiles_x * (p.H / p.tile_h);
    abox[1] = (uint32_t)p.tile_w; abox[2] = (uint32_t)p.tile_h;
  }
  encode_map(&op.tmA, op.a_base, op.a_rank, op.a_dims, op.a_strides, abox, 64);
  p.fd_ntiles = make_fastdiv(p.n_tiles); p.fd_tpi = make_fastdiv(p.tiles_per_img); p.fd_tx = make_fastdiv(p.tiles_x);
  p.b_sample_rows = 0;
  if (op.w_samples > 1) {   // weights [w_samples][N][K]; every 256-row tile lies inside one sample (longk_block_n)
    p.b_sample_rows = N;
    p.fd_tps = make_fastdiv(p.rows_per_sample / kLongM);
  }
  p.a_stage_bytes = (uint32_t)(kLongM * 64 * 2);
  p.b_stage_bytes = (uint32_t)(p.block_n * 64 * 2);
  p.stage_bytes = p.a_stage_bytes + ((p.b_stage_bytes + 1023u) & ~1023u);
  // shared memory: [barriers | stages x (A|B) | staging boxes of the 8 consumer warps (fp16 outputs)] within 226 KB:
  //   block_n 128: 1 KB + 4 x 48 KB + 8 x 4 KB = 225 KB;  block_n 192: 1 KB + 3 x 56 KB + 8 x 6 KB = 217 KB
  // (+ 1 KB alignment slack, <= 227 KB).  The fp32 residual-stream epilogue stores from registers and spends the staging bytes on
  // a pipeline stage.
  const bool staged = p.resid32 == nullptr;
  const size_t ostage_total = staged ? (size_t)kLongConsumerWarps * long_ost_warp_bytes(p.block_n) : 0;
  int stages = (int)((226 * 1024 - kLongHeaderBytes - ostage_total) / p.stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  VSB_CHECK(stages >= 3, "long-K tile does not fit in shared memory");
  p.stages = stages;
  p.ostage_off = (uint32_t)(kLongHeaderBytes + (size_t)stages * p.stage_bytes);
  op.smem = 1024 /*align slack*/ + p.ostage_off + ostage_total;
  if (staged) {  // output map [M rows][N cols]; box = one staging box: 8 fragment rows x 64 columns (128-byte swizzle) or x 16 (32-byte)
    const int box_cols = p.block_n % 64 == 0 ? 64 : 16;
    uint64_t odims[2] = {(uint64_t)N, (uint64_t)p.M};
    uint64_t ostrides[1] = {(uint64_t)p.ld_out16 * 2};
    uint32_t obox[2] = {(uint32_t)box_cols, 8u};
    encode_map(&op.tmO, p.out16, 2, odims, ostrides, obox, 0, /*no_swizzle=*/true, false, box_cols * 2);
  }
  uint64_t dims[2] = {(uint64_t)Kw, (uint64_t)N * (uint64_t)op.w_samples};
  uint64_t strides[1] = {(uint64_t)ldw * 2};
  uint32_t box[2] = {64u, (uint32_t)p.block_n};
  encode_map(&op.tmB, W, 2, dims, strides, box, 64);
  op.grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  op.threads = kLongThreads;
  VSB_CHECK((long)p.M < (1L << 31), "M too large for 32-bit row indices");
}

// Common finalisation: weights map, tiling, stage count, smem, grid.
// W: [N, Kw] fp16 row-major (K-major), Kw >= num_kb*kblk need not hold (TMA zero-fills out-of-bounds K).
inline void finalize_op(ConvGemmOp& op, const __half* W, int N, int Kw, int ldw, int num_sms, int block_n_override = 0,
                        int kernel_sel = kKernelAuto, int longk_bn = 0) {
  ConvGemmParams& p = op.p;
  p.N = N;
  // block_n <= 128: the two MMA warpgroups hold a 128 x block_n fp32 accumulator in registers (block_n / 2 per thread); an fp32
  // residual tile is prefetched into shared memory beside the accumulator tile: keep it <= 32 KB
  p.block_n = block_n_override ? block_n_override : pick_block_n(N, p.resid32 ? 64 : kMaxBlockN);
  VSB_CHECK(p.block_n % 16 == 0 && p.block_n >= 16 && p.block_n <= kMaxBlockN, "bad block_n");
  p.n_tiles = (N + p.block_n - 1) / p.block_n;
  {
    // Long main loops run on 256-row tiles when there are at least two of them per SM.  Below that the 128-row kernel fills the
    // machine better: it has twice the tiles to spread, and the last wave of 256-row tiles would leave SMs idle for a whole
    // 256-row main loop.  (Not measured below the threshold; the bottleneck convs at 64 frames have 5.8 tiles per SM, the
    // ConvNeXt pwconv1s and stage 1's pwconv2 at 64 frames 2.9 or more.)
    const int lbn = longk_block_n(op, N, block_n_override, num_sms, longk_bn);
    VSB_CHECK(kernel_sel != kKernelLongK || lbn != 0, "the long-K kernel cannot run this op");
    // The fp32 residual-stream epilogue also needs 12 K blocks: below that the tile's 8 bytes of stream traffic per output outlast
    // its main loop, and the 128-row kernel, which overlaps the two, is faster (videoseal_1.0 stage 0's pwconv2, K = 384: 188
    // against 196 us on an H100 SXM at 700 W).
    const long ltiles = (long)(p.M / kLongM) * (lbn ? N / lbn : 0);
    const bool long_enough = p.resid32 == nullptr || p.num_kb >= 12;
    if (lbn != 0 && kernel_sel != kKernel128 && (kernel_sel == kKernelLongK || (ltiles >= 2L * num_sms && long_enough))) {
      finalize_longk(op, W, N, Kw, ldw, num_sms, lbn);
      return;
    }
  }
  // small-N layers: several consecutive M tiles share one accumulator round (columns g*block_n of the accumulator tile) so that
  // the per-tile barrier handshakes / index math are amortised
  p.group = p.block_n <= 32 ? kAccCols / p.block_n : 1;
  if (p.group > 4) p.group = 4;
  if (p.group < 1) p.group = 1;
  if (p.m_tiles < 4 * num_sms) p.group = 1;   // keep enough tiles for load balance
  p.num_tiles = ((p.m_tiles + p.group - 1) / p.group) * p.n_tiles;
  p.fd_ntiles = make_fastdiv(p.n_tiles); p.fd_tpi = make_fastdiv(p.tiles_per_img); p.fd_tx = make_fastdiv(p.tiles_x);
  p.fd_tw = make_fastdiv(p.tile_w); p.fd_group = make_fastdiv(p.group); p.fd_rps = make_fastdiv(p.rows_per_sample);
  p.fd_hw = make_fastdiv(p.hw); p.fd_cc = make_fastdiv(p.cc); p.fd_ow = make_fastdiv(p.OW); p.fd_oh = make_fastdiv(p.OH);
  p.fd_ct = make_fastdiv(p.C0 + p.C1); p.fd_s = make_fastdiv(p.S);
  p.a_stage_bytes = (uint32_t)(kBlockM * p.kblk * 2);
  p.b_stage_bytes = (uint32_t)(p.block_n * p.kblk * 2);
  p.stage_bytes = p.a_stage_bytes + ((p.b_stage_bytes + 1023u) & ~1023u);
  VSB_CHECK(p.a_stage_bytes % 1024 == 0, "A stage must be 1024B aligned");
  // shared memory: [header | stages x (A|B) | halo tiles | resident weights | residual ring | output staging | accumulator tile]
  size_t resid_one = 0;
  p.resid_direct = 0;
  if (p.resid16 && op.loader == LD_TMA && p.num_kb >= 24 && (p.ld_res16 % 8) == 0 && N % p.block_n == 0 && (long)p.m_tiles * kBlockM == (long)p.M &&
      p.out32 == nullptr && p.outc_w == nullptr)
    p.resid_direct = 1;     // whole tiles only (the lean affine path is the one that implements the direct read)
  if (p.resid16 && !p.resid_direct) resid_one = (size_t)kBlockM * p.block_n * 2;
  if (p.resid32) resid_one = (size_t)kBlockM * p.block_n * 4;
  int depth = 1;
  if (resid_one) { depth = (int)(32768 / resid_one); if (depth > 4) depth = 4; if (depth < 1) depth = 1; }
  p.resid_depth = depth;
  p.resid_stride = (uint32_t)resid_one;
  const size_t resid_bytes = resid_one * depth;
  p.halo_stride = (uint32_t)(((size_t)p.halo_bytes + 1023) & ~size_t(1023));
  // halo ring: as deep as ~24 KB allows (2..8): the producer prefetches that many tiles ahead of the builders
  p.halo_bufs = 2;
  if (p.halo_stride) { p.halo_bufs = (int)(24576 / p.halo_stride); if (p.halo_bufs > kMaxHalo) p.halo_bufs = kMaxHalo; if (p.halo_bufs < 2) p.halo_bufs = 2; }
  const size_t halo_total = (size_t)p.halo_bufs * p.halo_stride;
  // resident weights: one N tile, whole K slab <= 48 KB -> loaded once per CTA instead of once per tile
  const size_t bslab = (size_t)p.num_kb * p.b_stage_bytes;
  p.b_resident = (p.n_tiles == 1 && bslab <= 48 * 1024 && op.w_samples == 1) ? 1 : 0;
  // several N tiles: every CTA keeps ONE N tile for its whole life (grid a multiple of n_tiles, tile = blockIdx.x + k * gridDim.x),
  // so its [block_n x K] weight slab can stay resident too when it fits beside >= 4 A stages.  Without this the slab is re-streamed
  // from L2 for every M tile (res 1x1 384->384: 295 KB of weights per M tile against 98 KB of activations).
  p.b_fixed_ntile = 0;
  if (!p.b_resident && p.n_tiles > 1 && p.n_tiles <= 8 && op.w_samples == 1 && op.loader == LD_TMA &&
      kHeaderBytes + resid_bytes + bslab + kAccBytes + 4 * (size_t)p.a_stage_bytes + 64 * 1024 <= 225 * 1024 && p.num_tiles >= 2 * num_sms) {
    p.b_resident = 1;
    p.b_fixed_ntile = 1;
  }
  // a resident slab that leaves fewer than 2 pipeline stages beside the rest is streamed instead
  if (p.b_resident && !p.b_fixed_ntile &&
      kHeaderBytes + resid_bytes + halo_total + bslab + kAccBytes + 2 * (size_t)p.a_stage_bytes + 1024 > 225 * 1024)
    p.b_resident = 0;
  const size_t bres_bytes = p.b_resident ? bslab : 0;
  if (p.b_resident) p.stage_bytes = p.a_stage_bytes;
  // TMA-store epilogue (short main loops only: there the epilogue is the critical path; long-K layers keep their shared memory for
  // pipeline stages): whole tiles, fp16 output (affine / GELU epilogues) or the in-place fp32 residual stream of pwconv2
  p.tma_store = 0; p.cpw = 0; p.ostage_bytes = 0;
  {
    const int nchunks = p.block_n / 16, epw = kEpiWarps / 4;     // epilogue warps per 32-row quadrant
    const bool common = op.loader == LD_TMA && p.outc_w == nullptr && p.epi == EPI_AFFINE && (long)p.m_tiles * kBlockM == (long)p.M &&
                        N % p.block_n == 0 && p.num_kb <= 12;
    if (common && p.out16 != nullptr && p.out32 == nullptr && (p.ld_out16 % 8) == 0 && (reinterpret_cast<uintptr_t>(p.out16) & 15) == 0)
      p.tma_store = 1;
    else if (common && p.out32 != nullptr && p.out16 == nullptr && p.act == ACT_NONE && p.resid32 != nullptr && p.grn_stats == nullptr &&
             (p.ld_out32 % 4) == 0 && (reinterpret_cast<uintptr_t>(p.out32) & 15) == 0)
      p.tma_store = 2;
    if (p.tma_store) {
      p.cpw = (nchunks + epw - 1) / epw;
      const uint32_t cb = p.tma_store == 2 ? 64u : 32u;          // bytes per row of one 16-column chunk
      // staging boxes: all cpw chunks of a warp in one box when the split is even and the row is 32 / 64 / 96 / 128 bytes, else one box
      // per chunk.  Rows of 32 / 64 / 128 bytes use the matching TMA swizzle so that the 16-byte register stores of the 32 lanes (one
      // row each) are bank-conflict free; 96-byte rows stay linear (2-way conflicts).
      p.ost_cpb = (nchunks % epw == 0 && p.cpw * cb <= 128u) ? p.cpw : 1;
      p.ost_rowb = (uint32_t)p.ost_cpb * cb;
      p.ost_swz = p.ost_rowb == 128u ? 3 : (p.ost_rowb == 64u ? 2 : (p.ost_rowb == 32u ? 1 : 0));
      p.ostage_bytes = (uint32_t)p.cpw * 32u * cb;               // per warp: multiples of 1024 bytes (swizzle atoms stay aligned)
    }
  }
  size_t ostage_total = p.tma_store ? (size_t)kEpiWarps * p.ostage_bytes + 1024 : 0;
  size_t fixed = kHeaderBytes + resid_bytes + halo_total + bres_bytes + ostage_total + kAccBytes;
  if (p.tma_store && fixed + 2 * (size_t)p.stage_bytes > 225 * 1024) {   // no room for the staging boxes: plain stores
    fixed -= ostage_total;
    ostage_total = 0;
    p.tma_store = 0; p.cpw = 0; p.ostage_bytes = 0;
  }
  VSB_CHECK(fixed + 2 * (size_t)p.stage_bytes <= 225 * 1024, "tile does not fit in shared memory (" + std::to_string(fixed) + " + 2 x " +
            std::to_string(p.stage_bytes) + " bytes)");
  int stages = (int)((225 * 1024 - fixed) / p.stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  p.stages = stages;
  p.halo_off = (uint32_t)(kHeaderBytes + (size_t)stages * p.stage_bytes);
  p.bres_off = (uint32_t)(p.halo_off + halo_total);
  p.resid_off = (uint32_t)(p.bres_off + bres_bytes);
  p.ostage_off = (uint32_t)((p.resid_off + resid_bytes + 1023) & ~size_t(1023));   // swizzle atoms of the staging boxes need 1024-byte alignment
  p.acc_off = (uint32_t)(p.ostage_off + ostage_total);
  op.smem = 1024 /*align slack*/ + p.acc_off + kAccBytes;
  if (p.tma_store) {   // output map: [M rows][N cols], box = one staging box (32 rows x 16 columns), dense rows
    uint64_t odims[2] = {(uint64_t)N, (uint64_t)p.M};
    uint32_t obox[2] = {(uint32_t)(p.ost_cpb * 16), 32u};
    const int swzb = p.ost_swz == 3 ? 128 : (p.ost_swz == 2 ? 64 : (p.ost_swz == 1 ? 32 : 0));
    if (p.tma_store == 1) {
      uint64_t ostrides[1] = {(uint64_t)p.ld_out16 * 2};
      encode_map(&op.tmO, p.out16, 2, odims, ostrides, obox, 0, /*no_swizzle=*/true, false, swzb);
    } else {
      uint64_t ostrides[1] = {(uint64_t)p.ld_out32 * 4};
      encode_map(&op.tmO, p.out32, 2, odims, ostrides, obox, 0, /*no_swizzle=*/true, /*f32=*/true, swzb);
    }
  }
  if (p.epi == EPI_LN || p.outc_w) VSB_CHECK(p.n_tiles == 1 && N <= kMaxBlockN, "LN / fused-outc epilogues need the full row in one tile");
  // weights: dims (K, N)
  if (op.w_samples > 1) {
    VSB_CHECK(op.loader == LD_TMA && !p.a_is_conv && p.rows_per_sample > 0 && p.rows_per_sample % kBlockM == 0 && N % p.block_n == 0,
              "per-sample weights: plain GEMM with whole tiles per sample only");
    p.b_sample_rows = N;
    p.fd_tps = make_fastdiv(p.rows_per_sample / kBlockM);
  }
  uint64_t dims[2] = {(uint64_t)Kw, (uint64_t)N * (uint64_t)op.w_samples};
  uint64_t strides[1] = {(uint64_t)ldw * 2};
  uint32_t box[2] = {(uint32_t)p.kblk, (uint32_t)p.block_n};
  encode_map(&op.tmB, W, 2, dims, strides, box, p.kblk);
  // whole tiles and an aligned bias vector: the epilogue warps read it from global memory and never meet at a barrier (the fused
  // 1x1 outc epilogue keeps its own barrier, so it keeps the shared copy)
  p.bias_global = (p.bias != nullptr && N % p.block_n == 0 && p.epi == EPI_AFFINE && p.outc_w == nullptr &&
                   (reinterpret_cast<uintptr_t>(p.bias) & 15) == 0) ? 1 : 0;
  op.grid = p.num_tiles < num_sms ? p.num_tiles : num_sms;
  if (p.b_fixed_ntile) op.grid = (num_sms / p.n_tiles) * p.n_tiles;
  // 8 epilogue warps (LD_TMA) or 4 epilogue + 4 builder warps, 2 MMA warpgroups, the producer warp
  op.threads = 544;
  VSB_CHECK((long)p.m_tiles * kBlockM < (1L << 31), "M too large for 32-bit row indices");
}

// A = NHWC fp16 activation [B, H, W, C] (pixel pitch ld elements); conv RxS stride 1, zero padding `pad`
// (R = S = 1, pad = 0 for 1x1).  Weights [N][R*S*C] with K order (r, s, c).
inline void setup_tma_conv(ConvGemmOp& op, const __half* src, int B, int H, int W, int C, int ld, int R, int S, int pad) {
  ConvGemmParams& p = op.p;
  op.loader = LD_TMA;
  p.a_is_conv = 1;
  p.tile_mode = 1;
  p.kblk = C >= 64 ? 64 : C;
  VSB_CHECK(p.kblk == 64 || p.kblk == 32 || p.kblk == 16, "TMA conv: C must be 16, 32 or a multiple of 64");
  VSB_CHECK(C % p.kblk == 0, "TMA conv: C must be a multiple of the K block");
  p.c_blocks = C / p.kblk;
  p.R = R; p.S = S; p.pad = pad;
  p.H = H; p.W = W;
  p.tile_w = W < kBlockM ? W : kBlockM;
  p.tile_h = kBlockM / p.tile_w;
  VSB_CHECK(p.tile_w * p.tile_h == kBlockM && W % p.tile_w == 0 && H % p.tile_h == 0, "TMA conv: map size must tile by 128 pixels");
  p.tiles_x = W / p.tile_w;
  p.tiles_per_img = p.tiles_x * (H / p.tile_h);
  p.m_tiles = B * p.tiles_per_img;
  p.M = B * H * W;
  p.num_kb = R * S * p.c_blocks;
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)W * ld * 2, (uint64_t)H * W * ld * 2};
  uint32_t box[4] = {(uint32_t)p.kblk, (uint32_t)p.tile_w, (uint32_t)p.tile_h, 1u};
  encode_map(&op.tmA, src, 4, dims, strides, box, p.kblk);
  op.a_base = src; op.a_rank = 4;
  for (int i = 0; i < 4; ++i) op.a_dims[i] = dims[i];
  for (int i = 0; i < 3; ++i) op.a_strides[i] = strides[i];
}


// 3x3 stride-1 zero-padded conv with on-chip im2col: the (8+2)x(16+2) input halo of each 8x16 output tile is loaded once
// per channel chunk.  Weights [N][9*C] with K order (r, s, c).
inline int halo_kpad(int C0, int C1) {   // padded K of the chunk-major halo weight layout
  const int cc = C0 < 64 ? C0 : 64;
  const int kb_per_c = (9 * cc + 63) / 64;
  return ((C0 + C1) / cc) * kb_per_c * 64;
}

// Halo-loader weight layout: [N][chunk][tap][cc] with each chunk zero-padded to kb_per_c*64 (see ConvGemmParams).
inline void setup_halo_common(ConvGemmParams& p, int C0, int C1, int B, int OH, int OW) {
  p.tile_mode = 1;
  p.kblk = 64;
  p.cc = C0 < 64 ? C0 : 64;
  VSB_CHECK(p.cc == 64 || p.cc == 32 || p.cc == 16, "halo loader: C must be 16, 32 or a multiple of 64");
  VSB_CHECK(C0 % p.cc == 0 && C1 % p.cc == 0, "halo loader: channels must be multiples of the chunk size");
  VSB_CHECK(OW % kHaloTW == 0 && OH % kHaloTH == 0, "halo loader: output map must tile by 8x16");
  p.c0_blocks = C0 / p.cc;
  p.c_blocks = (C0 + C1) / p.cc;
  p.kb_per_c = (9 * p.cc + 63) / 64;
  p.R = 3; p.S = 3; p.pad = 1;
  p.H = OH; p.W = OW; p.tile_w = kHaloTW; p.tile_h = kHaloTH;
  p.tiles_x = OW / kHaloTW;
  p.tiles_per_img = p.tiles_x * (OH / kHaloTH);
  p.m_tiles = B * p.tiles_per_img;
  p.M = B * OH * OW;
  p.num_kb = p.c_blocks * p.kb_per_c;
}

// 3x3 stride-1 zero-padded conv with on-chip im2col: the (8+2)x(16+2) input halo of each 8x16 output tile is loaded once
// per channel chunk.
inline void setup_halo_conv3(ConvGemmOp& op, const __half* src, int B, int H, int W, int C, int ld) {
  ConvGemmParams& p = op.p;
  op.loader = LD_HALO_CONV3;
  setup_halo_common(p, C, 0, B, H, W);
  p.halo_bytes = (uint32_t)(kHaloH * kHaloW * p.cc * 2);
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)ld * 2, (uint64_t)W * ld * 2, (uint64_t)H * W * ld * 2};
  uint32_t box[4] = {(uint32_t)p.cc, (uint32_t)kHaloW, (uint32_t)kHaloH, 1u};
  encode_map(&op.tmA, src, 4, dims, strides, box, 64, /*no_swizzle=*/true);
}

// A = [M, K] fp16 row-major (row pitch ld elements)
inline void setup_tma_gemm(ConvGemmOp& op, const __half* A, long M, int K, int ld) {
  ConvGemmParams& p = op.p;
  op.loader = LD_TMA;
  p.a_is_conv = 0;
  p.kblk = K >= 64 ? 64 : K;
  VSB_CHECK(p.kblk == 64 || p.kblk == 32 || p.kblk == 16, "TMA gemm: K must be 16, 32 or >= 64");
  p.M = (int)M;
  p.m_tiles = (int)((M + kBlockM - 1) / kBlockM);
  p.num_kb = (K + p.kblk - 1) / p.kblk;
  uint64_t dims[2] = {(uint64_t)K, (uint64_t)M};
  uint64_t strides[1] = {(uint64_t)ld * 2};
  uint32_t box[2] = {(uint32_t)p.kblk, (uint32_t)kBlockM};
  encode_map(&op.tmA, A, 2, dims, strides, box, p.kblk);
  op.a_base = A; op.a_rank = 2;
  op.a_dims[0] = dims[0]; op.a_dims[1] = dims[1]; op.a_strides[0] = strides[0];
}

// A = [A0 | A1] virtual concat along K of two [M, K0] / [M, K1] fp16 matrices (row pitches ld0 / ld1)
inline void setup_tma_gemm2(ConvGemmOp& op, const __half* A0, int K0, int ld0, const __half* A1, int K1, int ld1, long M) {
  ConvGemmParams& p = op.p;
  op.loader = LD_TMA;
  p.a_is_conv = 0;
  p.kblk = K0 >= 64 ? 64 : K0;
  VSB_CHECK(p.kblk == 64 || p.kblk == 32 || p.kblk == 16, "TMA gemm2: K0 must be 16, 32 or a multiple of 64");
  VSB_CHECK(K0 % p.kblk == 0 && K1 % p.kblk == 0, "TMA gemm2: K0, K1 must be multiples of the K block");
  p.M = (int)M;
  p.m_tiles = (int)((M + kBlockM - 1) / kBlockM);
  p.c0_blocks = K0 / p.kblk;
  p.num_kb = (K0 + K1) / p.kblk;
  uint32_t box[2] = {(uint32_t)p.kblk, (uint32_t)kBlockM};
  {
    uint64_t dims[2] = {(uint64_t)K0, (uint64_t)M};
    uint64_t strides[1] = {(uint64_t)ld0 * 2};
    encode_map(&op.tmA, A0, 2, dims, strides, box, p.kblk);
  }
  {
    uint64_t dims[2] = {(uint64_t)K1, (uint64_t)M};
    uint64_t strides[1] = {(uint64_t)ld1 * 2};
    encode_map(&op.tmA2, A1, 2, dims, strides, box, p.kblk);
  }
}

// generic gathered conv: out[b,oy,ox,:] over taps (r,s) of the virtual concat [src0 (C0 ch) | src1 (C1 ch)]
inline void setup_gather_conv(ConvGemmOp& op, int loader, const __half* src0, int C0, int ld0, const __half* src1, int C1, int ld1,
                              int B, int IH, int IW, int OH, int OW, int R, int S, int stride, int pad, int pad_mode) {
  ConvGemmParams& p = op.p;
  op.loader = loader;
  p.kblk = 64;
  p.src0 = src0; p.src1 = src1; p.C0 = C0; p.C1 = C1; p.ld0 = ld0; p.ld1 = ld1;
  VSB_CHECK(C0 % 8 == 0 && C1 % 8 == 0 && ld0 % 8 == 0 && (C1 == 0 || ld1 % 8 == 0), "gather conv: channels must be multiples of 8");
  p.IH = IH; p.IW = IW; p.OH = OH; p.OW = OW; p.R = R; p.S = S; p.stride = stride; p.pad = pad; p.pad_mode = pad_mode;
  p.Ktot = R * S * (C0 + C1);
  p.M = B * OH * OW;
  p.m_tiles = (p.M + kBlockM - 1) / kBlockM;
  p.num_kb = (p.Ktot + 63) / 64;
}

// stride-1 3x3 zero-padded conv of x [B][h*h][C] (pixel pitch ld), weights [N][9*C] with K order (r, s, c): the TMA conv where the
// h x h map tiles by 128 pixels (sides 16, 32, 64 or a multiple of 128), else the gather loader, which reads the same weights (sides
// such as 48, 80, 96, 160, 192 and 320, the maps at and below processing sizes that are odd multiples of 128).  op.loader tells which.
inline void setup_conv3x3(ConvGemmOp& op, const __half* x, int B, int h, int C, int ld) {
  if (h >= kBlockM ? h % kBlockM == 0 : kBlockM % h == 0 && h % (kBlockM / h) == 0) setup_tma_conv(op, x, B, h, h, C, ld, 3, 3, 1);
  else setup_gather_conv(op, LD_GATHER_CONV, x, C, ld, nullptr, 0, 0, B, h, h, h, h, 3, 3, 1, 1, 0);
}

// launch with programmatic stream serialization: the kernel may begin while its predecessor drains and synchronises
// itself with pdl_wait() (ptx.cuh).
template <class... KArgs, class... Args>
inline void launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t st, Args&&... args) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  VSB_CUDA(cudaLaunchKernelEx(&cfg, kernel, KArgs(args)...));
}

// Device the C entry point on this thread runs on (set by its DeviceGuard, vsb200.cu); -1 outside one.
inline thread_local int t_device = -1;

// Allow kernel K `bytes` of dynamic shared memory on the current device, the first time K is launched there.  The limit is a
// per-device attribute (cuKernelSetAttribute takes the device), so a process with models on several GPUs opts in on each of
// them.  One bit per device; threads that race both set the same value.
template <auto K>
inline void smem_optin(size_t bytes) {
  static std::atomic<uint64_t> done{0};
  int dev = t_device;
  if (dev < 0) VSB_CUDA(cudaGetDevice(&dev));
  VSB_CHECK(dev < 64, "device index above 63");
  const uint64_t bit = 1ull << dev;
  if (done.load(std::memory_order_acquire) & bit) return;
  VSB_CUDA(cudaFuncSetAttribute(K, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes));
  done.fetch_or(bit, std::memory_order_release);
}

template <int LOADER, int ACT>
inline void launch_one(const ConvGemmOp& op, cudaStream_t st) {
  smem_optin<conv_gemm_kernel<LOADER, ACT>>(227 * 1024);
  launch_pdl(conv_gemm_kernel<LOADER, ACT>, dim3(op.grid), dim3(op.threads), op.smem, st, op.tmA, op.tmA2, op.tmB, op.tmO, op.p);
}

template <int BN, int ACT, bool F32 = false>
inline void launch_longk(const ConvGemmOp& op, cudaStream_t st) {
  smem_optin<conv_gemm_longk_kernel<BN, ACT, F32>>(227 * 1024);
  launch_pdl(conv_gemm_longk_kernel<BN, ACT, F32>, dim3(op.grid), dim3(op.threads), op.smem, st, op.tmA, op.tmB, op.tmO, op.p);
}

// instantiated (loader, activation) pairs: only what the networks need, to bound compile time
inline void launch(const ConvGemmOp& op, cudaStream_t st) {
  const int a = op.p.act;
  if (op.longk) {   // the (block_n, epilogue) pairs of longk_block_n
    const int bn = op.p.block_n;
    if (op.p.resid32 != nullptr) { if (bn == 128) launch_longk<128, ACT_NONE, true>(op, st); else launch_longk<96, ACT_NONE, true>(op, st); }
    else if (a == ACT_GELU) launch_longk<128, ACT_GELU>(op, st);
    else if (bn == kLongWideN) { if (a == ACT_RELU) launch_longk<kLongWideN, ACT_RELU>(op, st); else launch_longk<kLongWideN, ACT_NONE>(op, st); }
    else if (bn == 128) { if (a == ACT_RELU) launch_longk<128, ACT_RELU>(op, st); else launch_longk<128, ACT_NONE>(op, st); }
    else { if (a == ACT_RELU) launch_longk<80, ACT_RELU>(op, st); else launch_longk<80, ACT_NONE>(op, st); }
    VSB_CUDA(cudaGetLastError());
    return;
  }
  switch (op.loader) {
    case LD_TMA:
      if (a == ACT_NONE) launch_one<LD_TMA, ACT_NONE>(op, st);
      else if (a == ACT_RELU) launch_one<LD_TMA, ACT_RELU>(op, st);
      else launch_one<LD_TMA, ACT_GELU>(op, st);
      break;
    case LD_GATHER_CONV:
      if (a == ACT_NONE) launch_one<LD_GATHER_CONV, ACT_NONE>(op, st);
      else if (a == ACT_RELU) launch_one<LD_GATHER_CONV, ACT_RELU>(op, st);
      else throw Error("gather conv: unsupported activation", kErrUnsupported);
      break;
    case LD_HALO_CONV3:
      if (a == ACT_RELU) launch_one<LD_HALO_CONV3, ACT_RELU>(op, st);
      else throw Error("halo conv3: unsupported activation", kErrUnsupported);
      break;
    default: throw Error("bad loader");
  }
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
