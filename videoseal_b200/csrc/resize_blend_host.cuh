// Host side of resize_blend.cuh: ATen-compatible resample tables, the resize launch geometry and the blend kernel choice.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>
#include "conv_gemm_host.cuh"
#include "resize_blend.cuh"

namespace vsb {

// ATen-compatible separable resample tables (host) ------------------------------------------------
struct ResampleHost {
  std::vector<int> start, cnt;
  std::vector<float> w;
  int maxt = 0;
};

// aten/src/ATen/native/cpu/UpSampleKernel.cpp (_compute_indices_weights_aa, bilinear filter) for antialias=True;
// plain half-pixel bilinear (align_corners=False) otherwise.  Upscaling with antialias=True degenerates to plain bilinear.
inline ResampleHost make_resample(int in, int out, bool antialias) {
  ResampleHost t;
  const double scale = (double)in / (double)out;
  if (antialias && scale > 1.0) {
    const double support = scale;  // interp_size/2 * scale with interp_size = 2
    t.maxt = (int)std::ceil(support) * 2 + 1;
    t.start.resize(out); t.cnt.resize(out); t.w.assign((size_t)out * t.maxt, 0.f);
    for (int i = 0; i < out; ++i) {
      const double center = scale * (i + 0.5);
      const double invscale = 1.0 / scale;
      int xmin = (int)(center - support + 0.5); if (xmin < 0) xmin = 0;
      int xmax = (int)(center + support + 0.5); if (xmax > in) xmax = in;
      const int n = xmax - xmin;
      double total = 0.0;
      std::vector<double> ww(n);
      for (int j = 0; j < n; ++j) {
        double x = (j + xmin - center + 0.5) * invscale;
        if (x < 0) x = -x;
        ww[j] = x < 1.0 ? 1.0 - x : 0.0;
        total += ww[j];
      }
      t.start[i] = xmin; t.cnt[i] = n;
      for (int j = 0; j < n; ++j) t.w[(size_t)i * t.maxt + j] = (float)(total != 0.0 ? ww[j] / total : 0.0);
    }
  } else {
    t.maxt = 2;
    t.start.resize(out); t.cnt.resize(out); t.w.assign((size_t)out * 2, 0.f);
    for (int i = 0; i < out; ++i) {
      // area_pixel_compute_source_index(scale, dst, align_corners=false, cubic=false)
      // single rounding (fused multiply-add), like the vectorised ATen CPU kernel and the CUDA one
      float src = std::fmaf((float)scale, i + 0.5f, -0.5f);
      if (src < 0.f) src = 0.f;
      int x0 = (int)src; if (x0 > in - 1) x0 = in - 1;
      const int x1 = x0 + ((x0 < in - 1) ? 1 : 0);
      const float l1 = src - (float)x0, l0 = 1.f - l1;
      t.start[i] = x0;
      if (x1 == x0) { t.cnt[i] = 1; t.w[(size_t)i * 2] = 1.f; }
      else { t.cnt[i] = 2; t.w[(size_t)i * 2] = l0; t.w[(size_t)i * 2 + 1] = l1; }
    }
  }
  return t;
}

struct ResampleDev {
  DevicePool pool;
  ResampleTab tab;
  // geometry of resize_sep_kernel for this (in -> out) pair: output rows per block, input rows per staging round, the largest
  // number of input rows one block touches, dynamic shared memory
  int toy = 8, gstage = 1, rin_max = 1;
  size_t smem = 0;
  ResampleDev(int ih, int iw, int oh, int ow, bool aa) {
    ResampleHost y = make_resample(ih, oh, aa), x = make_resample(iw, ow, aa);
    tab.ystart = pool.upload(y.start); tab.ycnt = pool.upload(y.cnt); tab.yw = pool.upload(y.w); tab.maxt_y = y.maxt;
    tab.xstart = pool.upload(x.start); tab.xcnt = pool.upload(x.cnt); tab.xw = pool.upload(x.w); tab.maxt_x = x.maxt;
    gstage = iw * 4 * 4 <= 16 * 1024 ? 4 : (iw * 4 * 2 <= 16 * 1024 ? 2 : 1);    // rows per staging round (kRsStages - 1 rounds in flight): 4, 2 or 1
    for (toy = 8; toy >= 1; toy >>= 1) {
      rin_max = 1;
      for (int o0 = 0; o0 < oh; o0 += toy) {
        const int o1 = std::min(oh, o0 + toy) - 1;
        rin_max = std::max(rin_max, y.start[o1] + y.cnt[o1] - y.start[o0]);
      }
      smem = ((((size_t)rin_max * ow + 3) & ~(size_t)3) + kRsStages * (((size_t)gstage * iw + 8 + 3) & ~(size_t)3)) * sizeof(float);
      if (smem <= 100 * 1024 || toy == 1) break;
    }
  }
};

// resample n <= 16384 frames that are `frame_stride` floats apart, H x W -> S x S (the table pair r); rec: MT, GST, vec, toy, OW
inline void launch_resize(const ResampleDev& r, const float* src, long frame_stride, int n, int H, int W, int S, float* dst, int32_t rec[5],
                          cudaStream_t st) {
  // (checked here, not when the table is built: the blend only reads the delta up-sampler's table, whatever its width)
  if (r.smem > 200 * 1024) throw Error("resize: image too wide for the shared-memory resample kernel (not implemented)", kErrUnsupported);
  const int vec = (W % 4 == 0) && (reinterpret_cast<uintptr_t>(src) % 16 == 0) && (frame_stride % 4 == 0);
  const dim3 grid((S + r.toy - 1) / r.toy, n * 3);
  const int mt = r.tab.maxt_x <= 2 ? 2 : (r.tab.maxt_x <= 8 ? 8 : 0);
  const int32_t rc[5] = {mt, r.gstage, vec, r.toy, S};
  std::copy(rc, rc + 5, rec);
#define VSB_RS(MT, GS) do { smem_optin<resize_sep_kernel<MT, GS>>(200 * 1024); \
    resize_sep_kernel<MT, GS><<<grid, 256, r.smem, st>>>(src, frame_stride, dst, H, W, S, S, r.tab, r.toy, r.rin_max, vec); } while (0)
  if (r.gstage == 4) { if (mt == 2) VSB_RS(2, 4); else if (mt == 8) VSB_RS(8, 4); else VSB_RS(0, 4); }
  else if (r.gstage == 2) { if (mt == 2) VSB_RS(2, 2); else if (mt == 8) VSB_RS(8, 2); else VSB_RS(0, 2); }
  else { if (mt == 2) VSB_RS(2, 1); else if (mt == 8) VSB_RS(8, 1); else VSB_RS(0, 1); }
#undef VSB_RS
  VSB_CUDA(cudaGetLastError());
}

// JND blend of bp.F frames; rec: 3 (jnd_blend3_kernel) or 2 (jnd_blend2_kernel), VEC, FASTUP, CD, JIN
inline void launch_blend(const BlendParams& bp, int32_t rec[5], cudaStream_t st) {
  VSB_CHECK(bp.F <= 65535, "too many frames per blend launch");
  dim3 grid((bp.W + kB2TW - 1) / kB2TW, (bp.H + kB2TH - 1) / kB2TH, bp.F);
  const bool vec = (bp.W % 4 == 0) && ((reinterpret_cast<uintptr_t>(bp.imgs) | reinterpret_cast<uintptr_t>(bp.imgs_w) |
                                        reinterpret_cast<uintptr_t>(bp.preds_w)) % 16 == 0);
  // delta read in place, or through <= 2 taps per axis (plain bilinear up-scale: every input at least as large as the processing size)
  const bool fastup = bp.identity_resample || (bp.tab.maxt_x <= 2 && bp.tab.maxt_y <= 2 && bp.H >= bp.PH && bp.W >= bp.PW);
  VSB_CHECK(bp.CD == 1 || bp.CD == 3, "delta must have 1 or 3 channels");
  // TMA-fed kernel (jnd_blend3_kernel): vector layout, delta in place or <= 2 taps per axis; the delta tile needs a TMA-legal row pitch
  const bool delta_tma = bp.identity_resample || (bp.PW % 4 == 0 && reinterpret_cast<uintptr_t>(bp.delta) % 16 == 0);
  // (boxes never exceed the tensor they are cut from: tiny frames / processing sizes take the load-then-compute kernel)
  const bool tma = vec && fastup && delta_tma && bp.W >= kB2LP && bp.H >= kB2TH + 4 &&
                   (bp.identity_resample || (bp.PW >= kB3DW && bp.PH >= kB2DH)) &&
                   (!bp.identity_resample || (bp.PW % 4 == 0 && reinterpret_cast<uintptr_t>(bp.delta) % 16 == 0));
  CUtensorMap tmI, tmD;
  if (tma) {
    const uint64_t idims[3] = {(uint64_t)bp.W, (uint64_t)bp.H, (uint64_t)bp.F * 3};
    const uint64_t istr[2] = {(uint64_t)bp.W * 4, (uint64_t)bp.H * bp.W * 4};
    const uint32_t ibox[3] = {(uint32_t)kB2LP, (uint32_t)(kB2TH + 4), 3};
    encode_map(&tmI, bp.imgs, 3, idims, istr, ibox, 0, true, /*f32=*/true);
    tmD = tmI;
    if (!bp.identity_resample) {
      const int nkeys = (bp.F + bp.step - 1) / bp.step;
      const uint64_t ddims[3] = {(uint64_t)bp.PW, (uint64_t)bp.PH, (uint64_t)nkeys * bp.CD};
      const uint64_t dstr[2] = {(uint64_t)bp.PW * 4, (uint64_t)bp.PH * bp.PW * 4};
      const uint32_t dbox[3] = {(uint32_t)kB3DW, (uint32_t)kB2DH, 1};
      encode_map(&tmD, bp.delta, 3, ddims, dstr, dbox, 0, true, /*f32=*/true);
    }
  }
  const int32_t rc[5] = {tma ? 3 : 2, vec ? 4 : 1, fastup ? 1 : 0, bp.CD, (bp.use_jnd && bp.jnd_in == 3) ? 3 : 1};
  std::copy(rc, rc + 5, rec);
#define VSB_BL(V, FU, CDV, JI) do { smem_optin<jnd_blend2_kernel<V, FU, CDV, JI>>(b2_smem(JI)); \
    jnd_blend2_kernel<V, FU, CDV, JI><<<grid, 256, b2_smem(JI), st>>>(bp); } while (0)
#define VSB_BL2(CDV, JI) do { \
    if (vec) { if (fastup) VSB_BL(4, 1, CDV, JI); else VSB_BL(4, 0, CDV, JI); } else { if (fastup) VSB_BL(1, 1, CDV, JI); else VSB_BL(1, 0, CDV, JI); } } while (0)
#define VSB_BL3(CDV, JI) do { smem_optin<jnd_blend3_kernel<CDV, JI>>(b3_smem(JI)); \
    jnd_blend3_kernel<CDV, JI><<<grid3, 256, b3_smem(JI), st>>>(bp, tmI, tmD); } while (0)
  const dim3 grid3(grid.x, (bp.H + kB2TH * kB3NT - 1) / (kB2TH * kB3NT), bp.F);
  const bool j3 = bp.use_jnd && bp.jnd_in == 3;      // one heat-map per RGB channel (jnd_3_1 / jnd_3_3): rarely used, own instantiation
  if (tma) {
    if (bp.CD == 1) { if (j3) VSB_BL3(1, 3); else VSB_BL3(1, 1); }
    else            { if (j3) VSB_BL3(3, 3); else VSB_BL3(3, 1); }
  } else if (bp.CD == 1) { if (j3) VSB_BL2(1, 3); else VSB_BL2(1, 1); }
  else                   { if (j3) VSB_BL2(3, 3); else VSB_BL2(3, 1); }
#undef VSB_BL3
#undef VSB_BL2
#undef VSB_BL
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
