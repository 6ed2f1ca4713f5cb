// Host side of augment.cuh: argument rules and workspace sizes of vsb_augment (host-only, so they hold without a GPU) and the
// launches of one call.
#pragma once
#include <algorithm>
#include <cmath>
#include <string>
#include <type_traits>
#include "augment.cuh"
#include "plan.cuh"
#include "resize_blend_host.cuh"

namespace vsb {

inline int aug_blocks(int64_t n, int per_block_items = 256) {
  return (int)std::max<int64_t>(1, std::min<int64_t>((n + per_block_items - 1) / per_block_items, 4096));
}
// fp64 partial sums per image of the contrast mean: enough blocks to fill the GPU at 1080p, a fixed count for a given H x W
inline int aug_sum_blocks(int64_t HW) { return (int)std::max<int64_t>(1, std::min<int64_t>(HW / (kAugSumThreads * 16), 256)); }

inline size_t aug_align(size_t n) { return (n + 255) & ~(size_t)255; }

// Workspace bytes of one call (0 when the op needs none); throws Error(kErrInvalid) on a bad op or shape.
inline size_t aug_workspace_bytes(int op, int B, int H, int W) {
  VSB_CHECK(B >= 1 && H >= 1 && W >= 1, "augment: B, H and W must be positive");
  VSB_CHECK(op >= VSB_AUG_CROP_FLIP && op <= VSB_AUG_WINDOW_AVG, "augment: unknown op");
  const int64_t HW = (int64_t)H * W;
  if (op == VSB_AUG_CONTRAST) return aug_align((size_t)B * aug_sum_blocks(HW) * sizeof(double));
  if (op == VSB_AUG_BLUR) return aug_align((size_t)B * 3 * HW * sizeof(float));
  if (op == VSB_AUG_JPEG) return aug_align((size_t)B * HW) + aug_align((size_t)B * 2 * ((H + 1) / 2) * ((W + 1) / 2));
  return 0;
}

// Argument rules that need no device.
inline void aug_check(int op, int B, int C, int H, int W, int OH, int OW, const float* params, int n_params, const float* aux) {
  aug_workspace_bytes(op, B, H, W);
  VSB_CHECK(C == 3, "augment: images must have 3 channels");
  VSB_CHECK(OH >= 1 && OW >= 1, "augment: output size must be positive");
  VSB_CHECK((int64_t)H * W < (1ll << 31) && (int64_t)OH * OW < (1ll << 31) && B <= 16384, "augment: tensor too large");
  auto need = [&](int n) { VSB_CHECK(params != nullptr && n_params == n, "augment: op expects " + std::to_string(n) + " parameters"); };
  switch (op) {
    case VSB_AUG_CROP_FLIP: {
      need(3);
      const int i0 = (int)params[0], j0 = (int)params[1];
      VSB_CHECK(i0 >= 0 && j0 >= 0 && i0 + OH <= H && j0 + OW <= W, "augment: crop window outside the image");
      break;
    }
    case VSB_AUG_GRID_NEAREST: case VSB_AUG_GRID_BILINEAR:
      need(9);
      VSB_CHECK(aux != nullptr, "augment: grid ops need the base-grid coordinates in aux");
      break;
    case VSB_AUG_BRIGHTNESS: case VSB_AUG_CONTRAST: case VSB_AUG_SATURATION: need(2); break;
    case VSB_AUG_HUE: need(1); break;
    case VSB_AUG_GRAYSCALE: VSB_CHECK(n_params == 0, "augment: grayscale takes no parameters"); break;
    case VSB_AUG_BLUR:
      VSB_CHECK(params != nullptr && n_params >= 1 && n_params <= kAugMaxTaps && n_params % 2 == 1, "augment: blur needs an odd tap count <= 33");
      VSB_CHECK(n_params / 2 < H && n_params / 2 < W, "augment: reflect padding needs the image larger than half the kernel");
      break;
    case VSB_AUG_JPEG:
      need(1);
      VSB_CHECK(params[0] >= 1.f && params[0] <= 100.f && params[0] == (float)(int)params[0], "augment: JPEG quality must be an integer in 1..100");
      break;
    case VSB_AUG_WINDOW_AVG: {
      need(3);
      VSB_CHECK(params[0] >= 1.f && params[0] <= 16777216.f && params[0] == std::floor(params[0]), "augment: the averaging window must be an integer >= 1");
      VSB_CHECK(std::isfinite(params[1]) && std::isfinite(params[2]), "augment: the window-averaging alpha must be finite");
      const int64_t window = std::min<int64_t>((int64_t)params[0], B);
      if (window / 2 > kAugMaxHalfWindow)
        throw Error("augment: window averaging implements windows of at most " + std::to_string(2 * kAugMaxHalfWindow + 1) +
                        " frames (after window = min(window, T)); got " + std::to_string(window), kErrUnsupported);
      break;
    }
    default: break;
  }
  if (op != VSB_AUG_CROP_FLIP && op != VSB_AUG_GRID_NEAREST && op != VSB_AUG_GRID_BILINEAR && op != VSB_AUG_RESIZE)
    VSB_CHECK(OH == H && OW == W, "augment: this op keeps the image size");
  if (op == VSB_AUG_GRID_NEAREST || op == VSB_AUG_GRID_BILINEAR || op == VSB_AUG_RESIZE)
    VSB_CHECK(OH <= 65535 * 8, "augment: output too tall");
}

// IJG quality scaling of an Annex K table, baseline-clamped to 1..255
inline void jpeg_tables(int quality, JpegQ& q) {
  static const int luma[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                               14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                               49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
  static const int chroma_rows[4][4] = {{17, 18, 24, 47}, {18, 21, 26, 66}, {24, 26, 56, 99}, {47, 66, 99, 99}};   // 99 elsewhere
  const int scale = quality < 50 ? 5000 / quality : 200 - 2 * quality;
  for (int i = 0; i < 64; ++i) {
    const int r = i / 8, c = i % 8;
    const int cb = (r < 4 && c < 4) ? chroma_rows[r][c] : 99;
    q.q[0][i] = std::min(255, std::max(1, (luma[i] * scale + 50) / 100));
    q.q[1][i] = std::min(255, std::max(1, (cb * scale + 50) / 100));
  }
}

inline void aug_run(int op, const float* x, float* y, int B, int H, int W, int OH, int OW, const float* params, int n_params, const float* aux,
                    char* ws, cudaStream_t st) {
  const int64_t HW = (int64_t)H * W, OHW = (int64_t)OH * OW;
  const std::string tag = "@" + std::to_string(B) + "x" + std::to_string(H) + "x" + std::to_string(W);
  switch (op) {
    case VSB_AUG_CROP_FLIP:
      prof_scope("aug.crop_flip" + tag, st, 1, [&] {
        aug_gather_kernel<<<dim3(aug_blocks(OHW), B * 3), 256, 0, st>>>(x, y, H, W, OH, OW, (int)params[0], (int)params[1], params[2] != 0.f);
      });
      break;
    case VSB_AUG_GRID_NEAREST: case VSB_AUG_GRID_BILINEAR: {
      AugGrid g{};
      for (int i = 0; i < 6; ++i) g.t[i] = params[i];
      g.p[0] = params[6]; g.p[1] = params[7]; g.persp = params[8] != 0.f;
      g.xs = aux; g.ys = aux + OW;
      const dim3 grid(aug_blocks(OHW), B);
      if (op == VSB_AUG_GRID_NEAREST) prof_scope("aug.grid_nearest" + tag, st, 1, [&] { aug_grid_kernel<true><<<grid, 256, 0, st>>>(x, y, 3, H, W, OH, OW, g); });
      else prof_scope("aug.grid_bilinear" + tag, st, 1, [&] { aug_grid_kernel<false><<<grid, 256, 0, st>>>(x, y, 3, H, W, OH, OW, g); });
      break;
    }
    case VSB_AUG_BRIGHTNESS: case VSB_AUG_CONTRAST: case VSB_AUG_SATURATION: case VSB_AUG_HUE: case VSB_AUG_GRAYSCALE: {
      static const int cop[] = {kAugBrightness, kAugContrast, kAugSaturation, kAugHue, kAugGrayscale};
      const int c = cop[op - VSB_AUG_BRIGHTNESS];
      const int nblk = aug_sum_blocks(HW);
      double* part = (double*)ws;
      if (c == kAugContrast)
        prof_scope("aug.gray_sum" + tag, st, 1, [&] { aug_gray_sum_kernel<<<dim3(nblk, B), kAugSumThreads, 0, st>>>(x, HW, part); });
      const float f = n_params > 0 ? params[0] : 0.f, f1 = n_params > 1 ? params[1] : 0.f;
      prof_scope("aug.color" + std::to_string(c) + tag, st, 1, [&] {
        aug_color_kernel<<<dim3(aug_blocks(HW), B), 256, 0, st>>>(x, y, HW, c, f, f1, part, nblk);
      });
      break;
    }
    case VSB_AUG_BLUR: {
      AugTaps t{};
      t.k = n_params;
      for (int i = 0; i < n_params; ++i) t.w[i] = params[i];
      float* tmp = (float*)ws;
      const size_t smem = (size_t)(W + 2 * (n_params / 2)) * sizeof(float);
      VSB_CHECK(smem <= 48 * 1024, "augment: image too wide for the blur row buffer");
      prof_scope("aug.blur_h" + tag, st, 1, [&] { aug_blur_h_kernel<<<dim3(H, B * 3), 256, smem, st>>>(x, tmp, H, W, t); });
      prof_scope("aug.blur_v" + tag, st, 1, [&] { aug_blur_v_kernel<<<dim3(aug_blocks(HW), B * 3), 256, 0, st>>>(tmp, y, H, W, t); });
      break;
    }
    case VSB_AUG_JPEG: {
      JpegQ q;
      jpeg_tables((int)params[0], q);
      uint8_t* yp = (uint8_t*)ws;
      uint8_t* cp = (uint8_t*)(ws + aug_align((size_t)B * HW));
      prof_scope("aug.jpeg_mcu" + tag, st, 1, [&] { jpeg_mcu_kernel<<<dim3((W + 15) / 16, (H + 15) / 16, B), 256, 0, st>>>(x, yp, cp, H, W, q); });
      prof_scope("aug.jpeg_rgb" + tag, st, 1, [&] { jpeg_rgb_kernel<<<dim3(aug_blocks(HW), B), 256, 0, st>>>(x, yp, cp, y, H, W); });
      break;
    }
    case VSB_AUG_RESIZE: {
      // F.resize(size, antialias=True): the embedder's own separable resample tables and kernel (bilinear, align_corners=False);
      // the profile name carries the variant, resize_sep_kernel<MT, GST>
      ResampleDev r(H, W, OH, OW, ResampleMode{});
      int32_t rec[5];
      const std::string variant = ".mt" + std::to_string(resize_mt(r)) + "g" + std::to_string(r.gstage);
      prof_scope("aug.resize" + variant + tag, st, 1, [&] { launch_resize(r, x, 3 * HW, B, H, W, OH, OW, y, rec, st); });
      VSB_CUDA(cudaStreamSynchronize(st));   // the tables are freed with r
      break;
    }
    case VSB_AUG_WINDOW_AVG: {
      // x is a clip of B = T frames; a thread per VEC-float vector of a frame: float4 when a frame is a whole number of them and x
      // and y are 16-byte aligned (a contiguous fp32 view may start at any 4-byte offset), one float otherwise
      const int T = B, hh = (int)(std::min<int64_t>((int64_t)params[0], T) / 2);
      const int64_t n = 3 * HW;
      const bool v4 = n % 4 == 0 && (reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) % 16 == 0;
      const int64_t nvec = v4 ? n / 4 : n;
      const unsigned blocks = (unsigned)((nvec + 255) / 256);
      const float a_avg = params[1], a_keep = params[2];
      auto go = [&](auto hc) {
        constexpr int HH = decltype(hc)::value;
        prof_scope("aug.window_avg.h" + std::to_string(HH) + (v4 ? ".v4" : ".v1") + tag, st, 1, [&] {
          if (v4) aug_window_avg_kernel<HH, 4><<<blocks, 256, 0, st>>>(x, y, T, nvec, a_keep, a_avg);
          else aug_window_avg_kernel<HH, 1><<<blocks, 256, 0, st>>>(x, y, T, nvec, a_keep, a_avg);
        });
      };
      switch (hh) {
        case 0: go(std::integral_constant<int, 0>{}); break;
        case 1: go(std::integral_constant<int, 1>{}); break;
        case 2: go(std::integral_constant<int, 2>{}); break;
        case 3: go(std::integral_constant<int, 3>{}); break;
        case 4: go(std::integral_constant<int, 4>{}); break;
        case 5: go(std::integral_constant<int, 5>{}); break;
        case 6: go(std::integral_constant<int, 6>{}); break;
        case 7: go(std::integral_constant<int, 7>{}); break;
        default: go(std::integral_constant<int, kAugMaxHalfWindow>{}); break;
      }
      break;
    }
    default: break;
  }
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
