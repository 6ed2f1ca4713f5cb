// Host side of quality.cuh: the workspace layout of vsb_ssim (host-only, so sizes and argument errors need no GPU) and the
// launch sequence of one SSIM / MS-SSIM call.
#pragma once
#include <cmath>
#include <string>
#include "plan.cuh"
#include "quality.cuh"

namespace vsb {

// Levels of one call and where their block sums and pooled planes live in the caller's workspace.
struct QualityLayout {
  int levels = 1;
  int H[kQLevels] = {}, W[kQLevels] = {};
  int KH = 11, KW = 11;               // level 0 taps per axis (1: the axis is shorter than 11 and not filtered)
  int tiles[kQLevels] = {}, strips[kQLevels] = {}, nb[kQLevels] = {};
  size_t part_off[kQLevels] = {};     // byte offsets of the [planes][nb][2] fp64 block sums
  size_t px_off[kQLevels] = {}, py_off[kQLevels] = {};   // levels 1..4: pooled x / y [planes][H][W] fp32
  size_t bytes = 0;
};

// Argument rules of vsb_ssim that need no device (throws Error(kErrInvalid) with the reason).
inline QualityLayout quality_layout(int B, int C, int H, int W, bool multiscale) {
  VSB_CHECK(B >= 1 && C >= 1, "quality: B and C must be positive");
  VSB_CHECK(H >= 2 && W >= 2, "quality: H and W must be at least 2 (pytorch_msssim squeezes singleton spatial dims)");
  VSB_CHECK(!multiscale || std::min(H, W) > (kQTaps - 1) * 16, "quality: MS-SSIM needs min(H, W) > 160 (4 downsamplings of an 11-tap window)");
  const int64_t planes = (int64_t)B * C;
  QualityLayout L;
  L.levels = multiscale ? kQLevels : 1;
  L.KH = H >= kQTaps ? kQTaps : 1;
  L.KW = W >= kQTaps ? kQTaps : 1;
  auto align = [](size_t n) { return (n + 255) & ~(size_t)255; };
  size_t off = 0;
  int h = H, w = W;
  for (int l = 0; l < L.levels; ++l) {
    L.H[l] = h; L.W[l] = w;
    if (l == 0 && (L.KH == 1 || L.KW == 1)) {
      const int64_t npix = (int64_t)(h - L.KH + 1) * (w - L.KW + 1);
      VSB_CHECK(npix < (1ll << 31) - kQNT, "quality: frame too large for an unfiltered axis");
      L.tiles[l] = (int)((npix + kQNT - 1) / kQNT); L.strips[l] = 1;
    } else {
      L.tiles[l] = (w - 10 + kQTW - 1) / kQTW;
      L.strips[l] = (h - 10 + kQRS - 1) / kQRS;
    }
    L.nb[l] = L.tiles[l] * L.strips[l];
    VSB_CHECK(planes * L.nb[l] < (1ll << 31), "quality: too many blocks for one launch");
    L.part_off[l] = off;
    off += align((size_t)planes * L.nb[l] * 2 * sizeof(double));
    if (l > 0) {
      L.px_off[l] = off; off += align((size_t)planes * h * w * sizeof(float));
      L.py_off[l] = off; off += align((size_t)planes * h * w * sizeof(float));
    }
    // avg_pool2d(kernel 2, stride 2, padding = size % 2): (n + 2 p - 2) / 2 + 1
    h = (h + 2 * (h & 1) - 2) / 2 + 1;
    w = (w + 2 * (w & 1) - 2) / 2 + 1;
  }
  L.bytes = off;
  return L;
}

// The normalised 11-tap Gaussian (sigma 1.5) of pytorch_msssim's _fspecial_gauss_1d.
inline void quality_taps(float g[kQTaps]) {
  double e[kQTaps], s = 0.0;
  for (int i = 0; i < kQTaps; ++i) { e[i] = std::exp(-(double)((i - 5) * (i - 5)) / (2.0 * 1.5 * 1.5)); s += e[i]; }
  for (int i = 0; i < kQTaps; ++i) g[i] = (float)(e[i] / s);
}

// All launches of one call on `st`: the level passes (level l writes level l+1's planes), then the finalize.
inline void quality_run(const QualityLayout& L, const float* x, const float* y, int B, int C, float data_range, float* ssim_out,
                        float* msssim_out, char* ws, cudaStream_t st) {
  const int64_t planes = (int64_t)B * C;
  QualityFinal f{};
  f.levels = L.levels; f.B = B; f.C = C; f.ssim = ssim_out; f.msssim = msssim_out;
  for (int l = 0; l < L.levels; ++l) {
    QualityLevel q{};
    q.x = l == 0 ? x : (const float*)(ws + L.px_off[l]);
    q.y = l == 0 ? y : (const float*)(ws + L.py_off[l]);
    const bool pool = l + 1 < L.levels;
    q.px = pool ? (float*)(ws + L.px_off[l + 1]) : nullptr;
    q.py = pool ? (float*)(ws + L.py_off[l + 1]) : nullptr;
    q.part = (double*)(ws + L.part_off[l]);
    q.H = L.H[l]; q.W = L.W[l];
    q.PH = pool ? L.H[l + 1] : 0; q.PW = pool ? L.W[l + 1] : 0;
    q.tiles = L.tiles[l]; q.strips = L.strips[l]; q.nb = L.nb[l];
    q.C1 = (float)((0.01 * data_range) * (0.01 * data_range));   // (K * R)^2 in double, then used in fp32, as the package does
    q.C2 = (float)((0.03 * data_range) * (0.03 * data_range));
    quality_taps(q.g);
    const bool direct = l == 0 && (L.KH == 1 || L.KW == 1);
    const int64_t oh = L.H[l] - (direct ? L.KH : kQTaps) + 1, ow = L.W[l] - (direct ? L.KW : kQTaps) + 1;
    f.part[l] = q.part; f.nb[l] = q.nb; f.count[l] = (double)oh * (double)ow;
    const dim3 grid((unsigned)(planes * q.nb));
    prof_scope("quality.l" + std::to_string(l) + "@" + std::to_string(q.H) + "x" + std::to_string(q.W), st, 1, [&] {
      if (direct) launch_pdl(quality_direct_kernel, grid, dim3(kQNT), 0, st, q, L.KH, L.KW);
      else launch_pdl(quality_level_kernel, grid, dim3(kQNT), 0, st, q);
    });
  }
  prof_scope("quality.finalize@" + std::to_string(B), st, 1, [&] {
    launch_pdl(quality_finalize_kernel, dim3((B + 127) / 128), dim3(128), 0, st, f);
  });
}

}  // namespace vsb
