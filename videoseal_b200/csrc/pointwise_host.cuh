// Host side of pointwise.cuh and dwconv_ring.cuh: grid, shared memory and template dispatch of each kernel family.
#pragma once
#include <algorithm>
#include "conv_gemm_host.cuh"
#include "dwconv_ring.cuh"
#include "pointwise.cuh"

namespace vsb {

// inc block's first conv + 1x1 residual (K0), S x S maps of Z channels; Z = 8 has its own kernel
inline void launch_unet_first(const float* src, int B, int S, int Z, int cin, const float* w1, const float* b1, const float* wr,
                              const float* br, __half* h1, __half* r0, int yuv, cudaStream_t st) {
  if (Z == 8) {
    const dim3 grid((S + 63) / 64, (S + 15) / 16, B);
    if (cin == 1) unet_first_z8_kernel<1><<<grid, 256, 0, st>>>(src, B, S, S, w1, b1, wr, br, h1, r0, yuv);
    else unet_first_z8_kernel<3><<<grid, 256, 0, st>>>(src, B, S, S, w1, b1, wr, br, h1, r0, yuv);
  } else {
    const dim3 grid((S + 31) / 32, (S + 15) / 16, B);
    if (cin == 1) unet_first_kernel<1><<<grid, 256, 0, st>>>(src, B, S, S, Z, w1, b1, wr, br, h1, r0, yuv);
    else unet_first_kernel<3><<<grid, 256, 0, st>>>(src, B, S, S, Z, w1, b1, wr, br, h1, r0, yuv);
  }
  VSB_CUDA(cudaGetLastError());
}

inline void launch_msg_embed(const uint8_t* msgs, int msg_stride, const float* table, int K, int hidden, __half* cat, int B, int hw,
                             int ld, int c_off, cudaStream_t st) {
  msg_embed_kernel<<<dim3(B, 8), 256, hidden * sizeof(float), st>>>(msgs, table, K, hidden, cat, hw, ld, c_off, msg_stride);
  VSB_CUDA(cudaGetLastError());
}

// ups_gather_ln_{tiled_,}kernel: bilinear x F + reflect pad + 3x3 tap sum + LayerNorm + activation of the tap GEMM output y
struct UpsGather {
  const __half* y = nullptr;
  int B = 0, IH = 0, C = 0;
  const float *lnw = nullptr, *lnb = nullptr;
  __half* out = nullptr;
  int ld_out = 0;
  size_t smem = 0;     // > 0: the tiled kernel with this much dynamic shared memory (ups_tile_smem, + the head's weights)
  size_t optin = 0;    // the caller's cap on `smem`, requested once per kernel and device
  int num_sms = 0;
  const float *hw = nullptr, *hb = nullptr;   // fused 1x1 head (HEAD): NO fp32 maps [B][NO][F*IH][F*IH]
  int NO = 0;
  float* maps = nullptr;
};
// dynamic shared memory of the tiled kernel: the 9 taps of (16/F + 2)^2 low-resolution pixels
inline size_t ups_tile_smem(int F, int C) { const int T = 16 / F; return (size_t)(T + 2) * (T + 2) * 9 * C * sizeof(__half); }

template <int VPT, int F, int ACT, bool HEAD = false>
inline void launch_ups_gather_t(const UpsGather& g, cudaStream_t st) {
  if constexpr (!HEAD) {   // the head is only fused into the tiled kernel
    if (!g.smem) {
      const int ppb = 256 / (g.C / (8 * VPT));
      const long npix = (long)g.B * F * g.IH * F * g.IH;
      // the G lanes of a pixel share LayerNorm sums through full-warp shuffles, which every lane of a warp must reach: no warp may
      // hold pixels past npix.  Processing sizes are multiples of 128, so every map is a multiple of 4 pixels and this holds.
      VSB_CHECK(npix % (32 / (g.C / (8 * VPT))) == 0, "up-gather: pixel count not a multiple of the pixels per warp");
      const unsigned grid = (unsigned)std::min<long>((npix + ppb - 1) / ppb, (long)g.num_sms * 32);
      ups_gather_ln_kernel<VPT, F, ACT><<<grid, 256, 0, st>>>(g.y, g.B, g.IH, g.IH, g.C, g.lnw, g.lnb, 1e-6f, g.out, g.ld_out);
      VSB_CUDA(cudaGetLastError());
      return;
    }
  }
  smem_optin<ups_gather_ln_tiled_kernel<VPT, F, ACT, HEAD>>(g.optin);
  const int tiles = g.IH / (16 / F);
  ups_gather_ln_tiled_kernel<VPT, F, ACT, HEAD><<<(unsigned)((long)g.B * tiles * tiles), 256, g.smem, st>>>(
      g.y, g.B, g.IH, g.IH, g.C, g.lnw, g.lnb, 1e-6f, g.out, g.ld_out, g.hw, g.hb, g.NO, g.maps);
  VSB_CUDA(cudaGetLastError());
}
// U-Net up-convs: factor 2, ReLU; 16-byte channel vectors per thread vpt = 1, or 2 for 512 channels
inline void launch_unet_upgather(const UpsGather& g, int vpt, cudaStream_t st) {
  if (vpt == 1) launch_ups_gather_t<1, 2, kUpRelu>(g, st);
  else launch_ups_gather_t<2, 2, kUpRelu>(g, st);
}
// pixel-decoder stages (F in {2, 4}, GELU): vpt 1 or 3; the last stage with the head (g.NO > 0) has C = 8 * vpt, vpt 1..4
inline void launch_pd_gather(const UpsGather& g, int F, int vpt, cudaStream_t st) {
  if (g.NO) {
    if (F == 2 && vpt == 1) launch_ups_gather_t<1, 2, kUpGelu, true>(g, st);
    else if (F == 2 && vpt == 2) launch_ups_gather_t<2, 2, kUpGelu, true>(g, st);
    else if (F == 2 && vpt == 3) launch_ups_gather_t<3, 2, kUpGelu, true>(g, st);
    else if (F == 2 && vpt == 4) launch_ups_gather_t<4, 2, kUpGelu, true>(g, st);
    else if (F == 4 && vpt == 1) launch_ups_gather_t<1, 4, kUpGelu, true>(g, st);
    else if (F == 4 && vpt == 2) launch_ups_gather_t<2, 4, kUpGelu, true>(g, st);
    else if (F == 4 && vpt == 3) launch_ups_gather_t<3, 4, kUpGelu, true>(g, st);
    else if (F == 4 && vpt == 4) launch_ups_gather_t<4, 4, kUpGelu, true>(g, st);
    else throw Error("pixel-wise head: no kernel for this width", kErrUnsupported);
  } else if (F == 2 && vpt == 1) launch_ups_gather_t<1, 2, kUpGelu>(g, st);
  else if (F == 2 && vpt == 3) launch_ups_gather_t<3, 2, kUpGelu>(g, st);
  else if (F == 4 && vpt == 1) launch_ups_gather_t<1, 4, kUpGelu>(g, st);
  else if (F == 4 && vpt == 3) launch_ups_gather_t<3, 4, kUpGelu>(g, st);
  else throw Error("pixel decoder: no gather kernel for this stage", kErrUnsupported);
}

// exact outermost rows / columns of a phase-folded up-conv (conv3_direct_host.cuh, setup_up_phase_direct): 64 = 2 x C channels in
inline void launch_up_border_fix(const __half* x0, const __half* x1, int C, int B, int IH, const float* wk, const float* lnw,
                                 const float* lnb, __half* out, int num_sms, cudaStream_t st) {
  smem_optin<up_border_fix_kernel>(kUpFixSmem);
  const long nb = (long)B * (2 * (2 * IH) + 2 * (2 * IH - 2));
  up_border_fix_kernel<<<(unsigned)std::min<long>((nb + kUpFixPPB - 1) / kUpFixPPB, (long)num_sms * 3), 256, kUpFixSmem, st>>>(
      x0, C, x1, C, B, IH, IH, wk, lnw, lnb, 1e-6f, out);
  VSB_CUDA(cudaGetLastError());
}

// ConvNeXt stem on S x S RGB frames -> OH x OH: CUDA-core conv + LayerNorm (one warp per output pixel), or the k4 patches of the
// tensor-core stem GEMM
inline void launch_stem_ln(const float* imgs, int B, int S, int OH, int stride, const float* wk, const float* bias, const float* lnw,
                           const float* lnb, int C, float* out, int ldo, int num_sms, cudaStream_t st) {
  const long npix = (long)B * OH * OH;
  const int grid = (int)std::min<long>((npix + 7) / 8, (long)num_sms * 16);
  stem_ln_kernel<<<grid, 256, (size_t)8 * (48 + C) * sizeof(float), st>>>(imgs, B, S, S, OH, OH, stride, wk, bias, lnw, lnb, C, out, ldo);
  VSB_CUDA(cudaGetLastError());
}
inline void launch_stem_im2col(const float* imgs, int B, int S, int OH, int stride, __half* patches, int num_sms, cudaStream_t st) {
  const long total = (long)B * OH * OH * 4;
  const int grid = (int)std::min<long>((total + 255) / 256, (long)num_sms * 32);
  stem_im2col_kernel<<<grid, 256, 0, st>>>(imgs, B, S, S, OH, OH, stride, patches);
  VSB_CUDA(cudaGetLastError());
}

// eps: 1e-6 for the ConvNeXt downsample layers and the SAM-ViT neck, 1e-5 for the ViT blocks' nn.LayerNorm
inline void launch_ln_rows(const float* x, long M, int C, int ldx, const float* lnw, const float* lnb, float eps, __half* out, int ld_out,
                           int num_sms, cudaStream_t st) {
  const int grid = (int)std::min<long>((M + 7) / 8, (long)num_sms * 16);
  ln_rows_kernel<<<grid, 256, 0, st>>>(x, M, C, ldx, lnw, lnb, eps, out, ld_out);
  VSB_CUDA(cudaGetLastError());
}

// GRN multiplier of K = 4C channels: folded into per-sample copies w2s of W2 [N][K] (K2e), or, w2s == nullptr, applied to g in
// place over row-slabs that fill the GPU (~8 blocks per SM)
inline void launch_grn(const float* stats, float* stats_next, const float* gamma, int K, int part_rows, int B, const __half* w2,
                       __half* w2s, int N, __half* g, int rows_per_sample, int num_sms, cudaStream_t st) {
  if (w2s) {
    smem_optin<grn_scale_weights_kernel>(200 * 1024);
    grn_scale_weights_kernel<<<dim3(B, 4), 256, 2 * K * sizeof(float), st>>>(stats, stats_next, gamma, w2, w2s, N, K, part_rows);
  } else {
    smem_optin<grn_apply_kernel>(200 * 1024);
    const int slabs = std::max(1, std::min(rows_per_sample, (num_sms * 8 + B - 1) / B));
    grn_apply_kernel<<<B * slabs, 256, 2 * K * sizeof(float), st>>>(g, rows_per_sample, K, K, stats, stats_next, gamma, slabs, part_rows);
  }
  VSB_CUDA(cudaGetLastError());
}

// pooled head: LayerNorm + mean over the P pixels of each frame, then the linear layer to NO logits
inline void launch_head(const float* y, int B, int P, int C, int ldy, const float* lnw, const float* lnb, float* pooled, const float* hw,
                        const float* hb, int NO, float* logits, cudaStream_t st) {
  smem_optin<head_pool_kernel>(160 * 1024);
  head_pool_kernel<<<B, 256, (size_t)8 * C * sizeof(float), st>>>(y, P, C, ldy, lnw, lnb, pooled);
  head_linear_kernel<<<(int)(((long)B * NO + 7) / 8), 256, 0, st>>>(pooled, hw, hb, B, C, NO, logits);
  VSB_CUDA(cudaGetLastError());
}

// JND heat-map of F frames H x W times the key-frame delta (delta == nullptr: the heat-map alone)
inline void launch_jnd_lowres(const float* imgs, const float* delta, float* out, int F, int H, int W, int CD, int step, int alternate,
                              int interp_chunk, int jin, int jout, cudaStream_t st) {
  const dim3 grid((W + kBlendTW - 1) / kBlendTW, (H + kBlendTH - 1) / kBlendTH, F);
  jnd_lowres_kernel<<<grid, 256, 0, st>>>(imgs, delta, out, H, W, CD, step, alternate, interp_chunk, jin, jout);
  VSB_CUDA(cudaGetLastError());
}

// RGB24 [npx][3] uint8 <-> planar fp32 [npx / plane][3][plane]; requant (optional) receives the re-quantised fp32 frames
inline void launch_u8_to_f32(const uint8_t* src, float* dst, long npx, long plane, int num_sms, cudaStream_t st) {
  u8hwc_to_f32chw_kernel<<<(unsigned)std::min<long>((npx + 255) / 256, (long)num_sms * 16), 256, 0, st>>>(src, dst, npx, plane);
  VSB_CUDA(cudaGetLastError());
}
inline void launch_f32_to_u8(const float* src, uint8_t* dst, float* requant, long npx, long plane, int num_sms, cudaStream_t st) {
  f32chw_to_u8hwc_kernel<<<(unsigned)std::min<long>((npx + 255) / 256, (long)num_sms * 16), 256, 0, st>>>(src, dst, requant, npx, plane);
  VSB_CUDA(cudaGetLastError());
}

// Depthwise 7x7 + LayerNorm of a ConvNeXt block: fp32 NHWC x [B,H,H,C] (pitch ld) -> fp16 out (pitch ld).  The TMA ring of rows
// (dwconv_ring.cuh, map built at plan time) takes 96 / 192 dense channels on maps that tile by 16; the strip kernel the rest of
// 96 to 768 (at 16 x 16 maps a 384-channel ring block would run one 192-thread block per SM with a 14-step prologue per 8 rows); the
// wide kernel any even width / odd map size (chunkyseal's proportional trunk), its threads looping over the channel pairs.
// The variant is chosen here and named in the plan's step names: ring (TMA ring), row (strip kernel, one strip = the whole row),
// strip (strip kernel, 8-pixel strips with predicated edge columns), wide (any even width, padded rows).
enum DwKind : int { DW_RING, DW_ROW, DW_STRIP, DW_WIDE };
inline const char* dw_kind_name(int k) { return k == DW_RING ? "ring" : k == DW_ROW ? "row" : k == DW_STRIP ? "strip" : "wide"; }
struct DwConvOp {
  CUtensorMap tm;
  int kind = DW_WIDE;
  const float* x = nullptr;
  int B = 0, H = 0, C = 0, ld = 0, R = 0;
  const float *dww = nullptr, *dwb = nullptr, *lnw = nullptr, *lnb = nullptr;
  __half* out = nullptr;
};
inline DwConvOp setup_dwconv(const float* x, int B, int H, int C, int ld, const float* dww, const float* dwb, const float* lnw,
                             const float* lnb, __half* out) {
  DwConvOp op;
  op.x = x; op.B = B; op.H = H; op.C = C; op.ld = ld;
  op.dww = dww; op.dwb = dwb; op.lnw = lnw; op.lnb = lnb; op.out = out;
  if (ld == C && (C == 96 || C == 192) && H % 16 == 0) op.kind = DW_RING;
  else if (!(C == 96 || C == 192 || C == 384 || C == 768)) op.kind = DW_WIDE;
  else op.kind = (C == 384 && H == 16) || (C == 768 && H == 8) ? DW_ROW : DW_STRIP;
  if (op.kind == DW_RING) {
    op.R = H % 32 == 0 ? 32 : 16;    // rows per block: 6 halo rows + the block prologue are amortised over R
    const int BW = (C == 96 ? 8 : 4) + 6;
    uint64_t dims[4] = {(uint64_t)C, (uint64_t)H, (uint64_t)H, (uint64_t)B};
    uint64_t strides[3] = {(uint64_t)C * 4, (uint64_t)H * C * 4, (uint64_t)H * H * C * 4};
    uint32_t box[4] = {(uint32_t)C, (uint32_t)BW, 1u, 1u};
    encode_map(&op.tm, x, 4, dims, strides, box, 0, true, /*f32=*/true);
  }
  return op;
}
template <int C, int NS, int SX, int NSLOT>
inline void launch_dw_ring_t(const DwConvOp& op, cudaStream_t st) {
  constexpr size_t smem = dw_ring_smem<C, NS, SX, NSLOT>();
  smem_optin<dwconv7_ln_ring_kernel<C, NS, SX, NSLOT>>(smem);
  const unsigned blocks = (unsigned)((long)op.B * (op.H / op.R) * (op.H / (NS * SX)));
  launch_pdl(dwconv7_ln_ring_kernel<C, NS, SX, NSLOT>, dim3(blocks), dim3(NS * C / 2 + 32), smem, st, op.tm, op.B, op.H, op.H, op.dww,
             op.dwb, op.lnw, op.lnb, op.out, op.R);
}
// spb strips per block over ngroups strips (or whole rows: FR)
template <int C, int ST, bool FR>
inline void launch_dw_strip_t(const DwConvOp& op, int spb, long ngroups, cudaStream_t st) {
  dwconv7_ln_c_kernel<C, ST, FR><<<(unsigned)((ngroups + spb - 1) / spb), spb * C / 2, (size_t)spb * ST * C * sizeof(float), st>>>(
      op.x, op.B, op.H, op.H, op.dww, op.dwb, op.lnw, op.lnb, op.out, op.C, spb, (int)ngroups);
}
inline void launch_dwconv(const DwConvOp& op, cudaStream_t st) {
  const int C = op.C, H = op.H;
  const long nstrips = (long)op.B * H * ((H + kDwStrip - 1) / kDwStrip);
  if (op.kind == DW_RING) {
    if (C == 96) launch_dw_ring_t<96, 2, 4, 8>(op, st);
    else launch_dw_ring_t<192, 1, 4, 8>(op, st);
  } else if (op.kind == DW_WIDE) {
    const int threads = std::min(512, (C / 2 + 31) / 32 * 32);
    const size_t smem_w = (size_t)kDwStrip * C * sizeof(float);
    smem_optin<dwconv7_ln_wide_kernel>(200 * 1024);
    if (smem_w > 200 * 1024) throw Error("dwconv7: more than 6400 channels is not implemented", kErrUnsupported);
    dwconv7_ln_wide_kernel<<<(unsigned)nstrips, threads, smem_w, st>>>(op.x, op.B, H, H, C, op.ld, op.dww, op.dwb, op.lnw, op.lnb, op.out, op.ld);
  } else {
    const int C2 = C / 2;
    int spb = 1;
    for (int s2 = 1; s2 <= 4; s2 *= 2) if ((s2 * C2) % 32 == 0 && s2 * C2 <= 512) { spb = s2; break; }
    if (spb * C2 > 512) throw Error("dwconv7: C/2 > 512 threads is not implemented (unsupported chunky extractor width)", kErrUnsupported);
    // narrow maps: one strip = the whole row, so no column is ever out of the image
    const long nrows = (long)op.B * H;
    if (op.kind == DW_ROW && C == 384) launch_dw_strip_t<384, 16, true>(op, 1, nrows, st);
    else if (op.kind == DW_ROW) launch_dw_strip_t<768, 8, true>(op, 1, nrows, st);
    else if (C == 96) launch_dw_strip_t<96, 8, false>(op, spb, nstrips, st);
    else if (C == 192) launch_dw_strip_t<192, 8, false>(op, spb, nstrips, st);
    else if (C == 384) launch_dw_strip_t<384, 8, false>(op, spb, nstrips, st);
    else launch_dw_strip_t<768, 8, false>(op, spb, nstrips, st);
  }
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
