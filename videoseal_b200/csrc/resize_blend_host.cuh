// Host side of resize_blend.cuh: ATen-compatible resample tables, the resize launch geometry and the blend kernel choice.
#pragma once
#include <algorithm>
#include <cmath>
#include <vector>
#include "../../include/vsb200.h"
#include "conv_gemm_host.cuh"
#include "resize_blend.cuh"

namespace vsb {

// ATen-compatible separable resample tables (host) ------------------------------------------------
struct ResampleHost {
  std::vector<int> start, cnt;
  std::vector<float> w;
  int maxt = 0;
};

// F.interpolate's `mode` (vsb200.h VSB_RESIZE_*), `align_corners` and `antialias`
struct ResampleMode {
  int mode = VSB_RESIZE_BILINEAR;
  bool align_corners = false, antialias = true;
};

// the resize fields of vsb_flags; what F.interpolate rejects is rejected here (ValueError there, VSB_ERR_INVALID here)
inline ResampleMode resample_mode(int flags) {
  ResampleMode m;
  m.mode = (flags & VSB_FLAG_RESIZE_MODE_MASK) >> VSB_FLAG_RESIZE_MODE_SHIFT;
  m.align_corners = (flags & VSB_FLAG_RESIZE_ALIGN_CORNERS) != 0;
  m.antialias = !(flags & VSB_FLAG_RESIZE_NO_AA);
  if (m.mode == VSB_RESIZE_NEAREST || m.mode == VSB_RESIZE_AREA) {
    VSB_CHECK(!m.antialias, "anti-aliasing is restricted to bilinear and bicubic resizes (set VSB_FLAG_RESIZE_NO_AA)");
    VSB_CHECK(!m.align_corners, "align_corners can only be set with bilinear and bicubic resizes");
  }
  return m;
}

// aten/src/ATen/native/cpu/UpSampleKernel.cpp _compute_indices_min_size_weights_aa in double: a normalised separable filter of
// half-width `half` source pixels at scale 1, stretched by the scale when down-scaling; taps whose centres lie within the support
inline void aa_table(ResampleHost& t, int in, int out, double scale, double half, double (*filter)(double)) {
  const double support = scale >= 1.0 ? half * scale : half;
  const double invscale = scale >= 1.0 ? 1.0 / scale : 1.0;
  t.maxt = (int)std::ceil(support) * 2 + 1;
  t.start.resize(out); t.cnt.resize(out); t.w.assign((size_t)out * t.maxt, 0.f);
  for (int i = 0; i < out; ++i) {
    const double center = scale * (i + 0.5);
    int xmin = (int)(center - support + 0.5); if (xmin < 0) xmin = 0;
    int xmax = (int)(center + support + 0.5); if (xmax > in) xmax = in;
    const int n = std::min(xmax - xmin, t.maxt);
    double total = 0.0;
    std::vector<double> ww(n);
    for (int j = 0; j < n; ++j) {
      ww[j] = filter((j + xmin - center + 0.5) * invscale);
      total += ww[j];
    }
    t.start[i] = xmin; t.cnt[i] = n;
    for (int j = 0; j < n; ++j) t.w[(size_t)i * t.maxt + j] = (float)(total != 0.0 ? ww[j] / total : 0.0);
  }
}
inline double aa_triangle(double x) { if (x < 0) x = -x; return x < 1.0 ? 1.0 - x : 0.0; }
// Keys cubic convolution kernel (aten/src/ATen/native/UpSample.h cubic_convolution1 / 2) with A = -0.75 (plain bicubic) or -0.5
// (the anti-aliased filter, as PIL)
template <typename T> inline T cubic_conv1(T x, T A) { return ((A + 2) * x - (A + 3)) * x * x + 1; }
template <typename T> inline T cubic_conv2(T x, T A) { return ((A * x - 5 * A) * x + 8 * A) * x - 4 * A; }
inline double aa_cubic(double x) {
  if (x < 0) x = -x;
  return x < 1.0 ? cubic_conv1(x, -0.5) : (x < 2.0 ? cubic_conv2(x, -0.5) : 0.0);
}

// repack a table to maxt = its largest tap count (the filters' maxt of ATen leaves room for a tap that never has weight)
inline void compact(ResampleHost& t) {
  const int out = (int)t.start.size();
  const int m = std::max(1, *std::max_element(t.cnt.begin(), t.cnt.end()));
  if (m == t.maxt) return;
  std::vector<float> w((size_t)out * m, 0.f);
  for (int i = 0; i < out; ++i)
    for (int j = 0; j < t.cnt[i]; ++j) w[(size_t)i * m + j] = t.w[(size_t)i * t.maxt + j];
  t.w.swap(w);
  t.maxt = m;
}

inline ResampleHost make_resample(int in, int out, bool antialias);

// The separable table of F.interpolate(size=out, mode, align_corners, antialias) along one axis of length in, for fp32 tensors
// (aten/src/ATen/native/UpSample.h, cpu/UpSampleKernel.cpp, AdaptiveAveragePooling.cpp):
//   bilinear, align_corners=False   antialias and down-scaling: triangle filter of half-width 1 stretched by the scale; otherwise
//                                   plain half-pixel bilinear (up-scaling with antialias=True degenerates to it)
//   bilinear, align_corners=True    antialias: the triangle filter at scale (in-1)/(out-1); otherwise source i*(in-1)/(out-1)
//   bicubic                         antialias: cubic filter (a = -0.5) of half-width 2, stretched when down-scaling; otherwise Keys
//                                   (A = -0.75) at 4 taps floor-1 .. floor+2, the out-of-range ones folded into the edge tap
//   nearest                         one tap at min(floor(i * (float)in/out), in - 1)
//   area                            adaptive_avg_pool: equal weights over [floor(i*in/out), ceil((i+1)*in/out))
// Every table is (start, cnt <= maxt, w[maxt]) with contiguous taps inside [0, in).
inline ResampleHost make_resample(int in, int out, ResampleMode m) {
  ResampleHost t;
  const bool ac = m.align_corners;
  if (m.mode == VSB_RESIZE_BILINEAR && !ac) return make_resample(in, out, m.antialias);
  if (m.antialias && (m.mode == VSB_RESIZE_BILINEAR || m.mode == VSB_RESIZE_BICUBIC)) {
    const double scale = ac ? (out > 1 ? (double)(in - 1) / (out - 1) : 0.0) : (double)in / out;
    if (m.mode == VSB_RESIZE_BILINEAR) aa_table(t, in, out, scale, 1.0, aa_triangle);
    else aa_table(t, in, out, scale, 2.0, aa_cubic);
    compact(t);
    return t;
  }
  t.start.resize(out); t.cnt.resize(out);
  if (m.mode == VSB_RESIZE_NEAREST) {
    t.maxt = 1;
    t.w.assign(out, 1.f);
    const float s = (float)in / (float)out;
    for (int i = 0; i < out; ++i) {
      t.start[i] = out == in ? i : (out == 2 * in ? i >> 1 : std::min((int)std::floor((float)i * s), in - 1));
      t.cnt[i] = 1;
    }
    return t;
  }
  if (m.mode == VSB_RESIZE_AREA) {
    t.maxt = 0;
    for (int i = 0; i < out; ++i) {
      t.start[i] = (int)((long)i * in / out);
      t.cnt[i] = (int)(((long)(i + 1) * in + out - 1) / out) - t.start[i];
      t.maxt = std::max(t.maxt, t.cnt[i]);
    }
    t.w.assign((size_t)out * t.maxt, 0.f);
    for (int i = 0; i < out; ++i)
      for (int j = 0; j < t.cnt[i]; ++j) t.w[(size_t)i * t.maxt + j] = (float)(1.0 / t.cnt[i]);
    return t;
  }
  // plain bilinear with align_corners=True, or plain bicubic: fp32 source coordinate (area_pixel_compute_source_index) and weights
  const float scale = ac ? (out > 1 ? (float)(in - 1) / (float)(out - 1) : 0.f) : (float)in / (float)out;
  const bool cubic = m.mode == VSB_RESIZE_BICUBIC;
  VSB_CHECK(cubic || m.mode == VSB_RESIZE_BILINEAR, "unknown resize mode");
  t.maxt = cubic ? 4 : 2;
  t.w.assign((size_t)out * t.maxt, 0.f);
  for (int i = 0; i < out; ++i) {
    // cubic: no clamp at 0 (the taps are clamped instead); the half-pixel form is one fused multiply-add, as ATen's kernels compute it
    const float src = ac ? scale * (float)i : std::fmaf(scale, i + 0.5f, -0.5f);
    const int x0 = std::min((int)std::floor(src), in - 1);                   // guard_index_and_lambda
    const float l = std::min(std::max(src - (float)x0, 0.f), 1.f);
    float* w = &t.w[(size_t)i * t.maxt];
    if (!cubic) {
      const int x1 = x0 + ((x0 < in - 1) ? 1 : 0);
      t.start[i] = x0;
      if (x1 == x0) { t.cnt[i] = 1; w[0] = 1.f; }
      else { t.cnt[i] = 2; w[0] = 1.f - l; w[1] = l; }
      continue;
    }
    const float A = -0.75f, l1 = 1.f - l;
    const float c[4] = {cubic_conv2(l + 1.f, A), cubic_conv1(l, A), cubic_conv1(l1, A), cubic_conv2(l1 + 1.f, A)};
    const int lo = std::max(0, std::min(x0 - 1, in - 1)), hi = std::max(0, std::min(x0 + 2, in - 1));
    t.start[i] = lo; t.cnt[i] = hi - lo + 1;
    for (int j = 0; j < 4; ++j) w[std::max(lo, std::min(x0 - 1 + j, hi)) - lo] += c[j];   // edge-clamped taps fold into the edge tap
  }
  return t;
}

// the rules every table obeys and the kernels rely on: taps inside the source, 1 <= cnt <= maxt, and first and last taps that never
// move backwards (a block of consecutive outputs reads the source range from its first output's first tap to its last output's last)
inline void check_table(const ResampleHost& t, int in) {
  for (size_t i = 0; i < t.start.size(); ++i) {
    VSB_CHECK(t.start[i] >= 0 && t.cnt[i] >= 1 && t.cnt[i] <= t.maxt && t.start[i] + t.cnt[i] <= in, "resample table: tap out of range");
    VSB_CHECK(i == 0 || (t.start[i] >= t.start[i - 1] && t.start[i] + t.cnt[i] >= t.start[i - 1] + t.cnt[i - 1]),
              "resample table: taps move backwards");
  }
}

// The source samples one blend tile of `tile` outputs (tiles start at multiples of `tile`) reads: from its first output's first
// tap, rounded down to a multiple of `align` (the TMA box's 16-byte start), to its last output's last tap, or to that output's
// start + `reads` - 1 when the kernel reads a fixed number of taps.  The staged tile / TMA box must hold this many.
inline int tile_span(const ResampleHost& t, int tile, int align, int reads) {
  const int out = (int)t.start.size();
  int span = 0;
  for (int o0 = 0; o0 < out; o0 += tile) {
    const int o1 = std::min(out, o0 + tile) - 1;
    span = std::max(span, std::max(t.start[o1] + t.cnt[o1], t.start[o1] + reads) - t.start[o0] / align * align);
  }
  return span;
}

// aten/src/ATen/native/cpu/UpSampleKernel.cpp (_compute_indices_weights_aa, bilinear filter) for antialias=True;
// plain half-pixel bilinear (align_corners=False) otherwise.  Upscaling with antialias=True degenerates to plain bilinear.
inline ResampleHost make_resample(int in, int out, bool antialias) {
  ResampleHost t;
  const double scale = (double)in / (double)out;
  if (antialias && scale > 1.0) {
    aa_table(t, in, out, scale, 1.0, aa_triangle);
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
  // when this table pair up-scales the delta in the blend: the source rows / columns one tile reads (tile_span), [0] through the
  // table's own taps (the <= 2-tap path), [1] through 4 taps from each output's start (the 4-tap path); columns also from the TMA
  // box's 16-byte-rounded first column
  int blend_rows[2], blend_cols[2], blend_cols_tma[2];
  ResampleDev(int ih, int iw, int oh, int ow, ResampleMode m) {
    ResampleHost y = make_resample(ih, oh, m), x = make_resample(iw, ow, m);
    check_table(y, ih);
    check_table(x, iw);
    tab.ystart = pool.upload(y.start); tab.ycnt = pool.upload(y.cnt); tab.yw = pool.upload(y.w); tab.maxt_y = y.maxt;
    tab.xstart = pool.upload(x.start); tab.xcnt = pool.upload(x.cnt); tab.xw = pool.upload(x.w); tab.maxt_x = x.maxt;
    for (int k = 0; k < 2; ++k) {
      blend_rows[k] = tile_span(y, kB2TH, 1, 4 * k);
      blend_cols[k] = tile_span(x, kB2TW, 1, 4 * k);
      blend_cols_tma[k] = tile_span(x, kB2TW, 4, 4 * k);
    }
    gstage = iw * 4 * 4 <= 16 * 1024 ? 4 : (iw * 4 * 2 <= 16 * 1024 ? 2 : 1);    // rows per staging round (kRsStages - 1 rounds in flight): 4, 2 or 1
    for (toy = 8; toy >= 1; toy >>= 1) {
      rin_max = std::max(1, tile_span(y, toy, 1, 0));                            // (the tables' taps never move backwards)
      smem = ((((size_t)rin_max * ow + 3) & ~(size_t)3) + kRsStages * (((size_t)gstage * iw + 8 + 3) & ~(size_t)3)) * sizeof(float);
      if (smem <= 100 * 1024 || toy == 1) break;
    }
  }
};

// the MT template argument of resize_sep_kernel for this table pair: taps per output column, 2, <= 8, or any (0)
inline int resize_mt(const ResampleDev& r) { return r.tab.maxt_x <= 2 ? 2 : (r.tab.maxt_x <= 8 ? 8 : 0); }

// resample n <= 16384 frames that are `frame_stride` floats apart, H x W -> OH x OW (the table pair r); rec: MT, GST, vec, toy, OW
inline void launch_resize(const ResampleDev& r, const float* src, long frame_stride, int n, int H, int W, int OH, int OW, float* dst,
                          int32_t rec[5], cudaStream_t st) {
  // (checked here, not when the table is built: the blend only reads the delta up-sampler's table, whatever its width)
  if (r.smem > 200 * 1024) throw Error("resize: image too wide for the shared-memory resample kernel (not implemented)", kErrUnsupported);
  const int vec = (W % 4 == 0) && (reinterpret_cast<uintptr_t>(src) % 16 == 0) && (frame_stride % 4 == 0);
  const dim3 grid((OH + r.toy - 1) / r.toy, n * 3);
  const int mt = resize_mt(r);
  const int32_t rc[5] = {mt, r.gstage, vec, r.toy, OW};
  std::copy(rc, rc + 5, rec);
#define VSB_RS(MT, GS) do { smem_optin<resize_sep_kernel<MT, GS>>(200 * 1024); \
    resize_sep_kernel<MT, GS><<<grid, 256, r.smem, st>>>(src, frame_stride, dst, H, W, OH, OW, r.tab, r.toy, r.rin_max, vec); } while (0)
  if (r.gstage == 4) { if (mt == 2) VSB_RS(2, 4); else if (mt == 8) VSB_RS(8, 4); else VSB_RS(0, 4); }
  else if (r.gstage == 2) { if (mt == 2) VSB_RS(2, 2); else if (mt == 8) VSB_RS(8, 2); else VSB_RS(0, 2); }
  else { if (mt == 2) VSB_RS(2, 1); else if (mt == 8) VSB_RS(8, 1); else VSB_RS(0, 1); }
#undef VSB_RS
  VSB_CUDA(cudaGetLastError());
}

// JND blend of bp.F frames, the delta up-scaled through up's tables (nullptr: read in place); rec: 3 (jnd_blend3_kernel) or 2
// (jnd_blend2_kernel), VEC, FASTUP, CD, JIN
inline void launch_blend(const BlendParams& bp, const ResampleDev* up, int32_t rec[5], cudaStream_t st) {
  VSB_CHECK(bp.F <= 65535, "too many frames per blend launch");
  VSB_CHECK(bp.identity_resample || up != nullptr, "blend: no delta up-sampler");
  dim3 grid((bp.W + kB2TW - 1) / kB2TW, (bp.H + kB2TH - 1) / kB2TH, bp.F);
  const bool vec = (bp.W % 4 == 0) && ((reinterpret_cast<uintptr_t>(bp.imgs) | reinterpret_cast<uintptr_t>(bp.imgs_w) |
                                        reinterpret_cast<uintptr_t>(bp.preds_w)) % 16 == 0);
  // FASTUP 1: delta read in place, or through <= 2 taps per axis; 4: through 3 or 4 taps per axis (bicubic), both from a staged tile
  // (every input at least as large as the processing size); 0: the generic tables straight from global memory
  const int taps = std::max(bp.tab.maxt_x, bp.tab.maxt_y);
  const int fastup = bp.identity_resample ? 1 : (bp.H < bp.PH || bp.W < bp.PW) ? 0 : (taps <= 2 ? 1 : (taps <= 4 ? 4 : 0));
  const int dh = fastup == 4 ? kB2DH4 : kB2DH;           // delta tile rows (staged tile and TMA box)
  VSB_CHECK(bp.CD == 1 || bp.CD == 3, "delta must have 1 or 3 channels");
  if (fastup && !bp.identity_resample) {
    const int k = fastup == 4 ? 1 : 0;
    VSB_CHECK(up->blend_rows[k] <= dh && up->blend_cols[k] <= kB2DW, "blend: the delta tile does not hold the up-scale's taps");
  }
  // TMA-fed kernel (jnd_blend3_kernel): vector layout, delta in place or staged; the delta tile needs a TMA-legal row pitch
  const bool delta_tma = bp.identity_resample || (bp.PW % 4 == 0 && reinterpret_cast<uintptr_t>(bp.delta) % 16 == 0);
  // (boxes never exceed the tensor they are cut from: tiny frames / processing sizes take the load-then-compute kernel)
  const bool tma = vec && fastup && delta_tma && bp.W >= kB2LP && bp.H >= kB2TH + 4 &&
                   (bp.identity_resample || (bp.PW >= kB3DW && bp.PH >= dh)) &&
                   (!bp.identity_resample || (bp.PW % 4 == 0 && reinterpret_cast<uintptr_t>(bp.delta) % 16 == 0));
  if (tma && !bp.identity_resample)
    VSB_CHECK(up->blend_cols_tma[fastup == 4 ? 1 : 0] <= kB3DW, "blend: the delta box does not hold the up-scale's taps");
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
      const uint32_t dbox[3] = {(uint32_t)kB3DW, (uint32_t)dh, 1};
      encode_map(&tmD, bp.delta, 3, ddims, dstr, dbox, 0, true, /*f32=*/true);
    }
  }
  const int32_t rc[5] = {tma ? 3 : 2, vec ? 4 : 1, fastup, bp.CD, (bp.use_jnd && bp.jnd_in == 3) ? 3 : 1};
  std::copy(rc, rc + 5, rec);
#define VSB_BL(V, FU, CDV, JI) do { smem_optin<jnd_blend2_kernel<V, FU, CDV, JI>>(b2_smem(JI, FU)); \
    jnd_blend2_kernel<V, FU, CDV, JI><<<grid, 256, b2_smem(JI, FU), st>>>(bp); } while (0)
#define VSB_BL2V(V, CDV, JI) do { \
    if (fastup == 1) VSB_BL(V, 1, CDV, JI); else if (fastup == 4) VSB_BL(V, 4, CDV, JI); else VSB_BL(V, 0, CDV, JI); } while (0)
#define VSB_BL2(CDV, JI) do { if (vec) VSB_BL2V(4, CDV, JI); else VSB_BL2V(1, CDV, JI); } while (0)
#define VSB_BL3F(CDV, JI, FU) do { smem_optin<jnd_blend3_kernel<CDV, JI, FU>>(b3_smem(JI, FU)); \
    jnd_blend3_kernel<CDV, JI, FU><<<grid3, 256, b3_smem(JI, FU), st>>>(bp, tmI, tmD); } while (0)
#define VSB_BL3(CDV, JI) do { if (fastup == 4) VSB_BL3F(CDV, JI, 4); else VSB_BL3F(CDV, JI, 1); } while (0)
  const dim3 grid3(grid.x, (bp.H + kB2TH * kB3NT - 1) / (kB2TH * kB3NT), bp.F);
  const bool j3 = bp.use_jnd && bp.jnd_in == 3;      // one heat-map per RGB channel (jnd_3_1 / jnd_3_3): rarely used, own instantiation
  if (tma) {
    if (bp.CD == 1) { if (j3) VSB_BL3(1, 3); else VSB_BL3(1, 1); }
    else            { if (j3) VSB_BL3(3, 3); else VSB_BL3(3, 1); }
  } else if (bp.CD == 1) { if (j3) VSB_BL2(1, 3); else VSB_BL2(1, 1); }
  else                   { if (j3) VSB_BL2(3, 3); else VSB_BL2(3, 1); }
#undef VSB_BL3
#undef VSB_BL3F
#undef VSB_BL2
#undef VSB_BL2V
#undef VSB_BL
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
