// Validation augmentations of the reference's robustness evaluation (videoseal/augmentation/*.py, evals/full.py:188-239), fp32
// NCHW in and out.  Each kernel restates the torchvision / PIL function the reference calls:
//   aug_gather_kernel     F.crop at (i, j) and F.hflip: an offset copy with an optional mirror
//   aug_grid_kernel       F.rotate / F.perspective: torchvision's fp32 grid (base grid, then theta through a 3-term dot product
//                         rounded as the CPU bmm rounds it, x*t0 then fma(y, t1, .) then + t2), grid_sample with align_corners=False,
//                         zero padding, nearest (nearbyint, exact) or bilinear
//   aug_color_kernel      adjust_brightness / adjust_contrast / adjust_saturation (_blend and clamp), adjust_hue (_rgb2hsv, shift,
//                         _hsv2rgb) and the reference's own 0.299 / 0.587 / 0.114 Grayscale
//   aug_gray_sum_kernel   the per-image sum of rgb_to_grayscale that adjust_contrast blends with: fixed-order fp64 partials per
//                         block (no atomics), summed in a fixed order by aug_color_kernel
//   aug_blur_h/v_kernel   F.gaussian_blur: the separable form of the 2-D kernel torchvision builds, reflect padding
//   jpeg_mcu_kernel       PIL's JPEG save at quality q (libjpeg-turbo: 4:2:0, islow DCT) and its decode, up to the chroma
//   jpeg_rgb_kernel       upsampling: integer arithmetic throughout, so the round trip is bit-exact (tests/jpeg_oracle.py)
//   aug_window_avg_kernel video.py's WindowAveraging: each frame blended with the mean of its temporal window, one pass over the clip
// Every fp32 expression that has to match torchvision's rounding is written with __f*_rn intrinsics so that nvcc cannot contract it.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace vsb {

enum AugColorOp { kAugBrightness = 0, kAugContrast = 1, kAugSaturation = 2, kAugHue = 3, kAugGrayscale = 4 };
constexpr int kAugSumThreads = 256;

// ---------------------------------------------------------------- crop / flip
__global__ void __launch_bounds__(256) aug_gather_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int OH, int OW,
                                                         int i0, int j0, int flip) {
  const int64_t n = (int64_t)OH * OW;
  const int64_t plane = blockIdx.y;
  const float* src = x + plane * H * W;
  float* dst = y + plane * n;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(k / OW), ox = (int)(k - (int64_t)oy * OW);
    dst[k] = __ldg(src + (int64_t)(i0 + oy) * W + j0 + (flip ? OW - 1 - ox : ox));
  }
}

// ---------------------------------------------------------------- rotate / perspective
struct AugGrid {
  float t[6];      // rescaled theta as [3][2]: row k multiplies base-grid coordinate k (x, y, 1)
  float p[2];      // perspective: the denominator's x and y coefficients (c6, c7); unused for an affine grid
  int persp;
  const float* xs; // [OW] base-grid x values, [OH] y values (torch.linspace, as torchvision builds them)
  const float* ys;
};

__device__ __forceinline__ float aug_dot3(float x, float y, float a, float b, float c) {
  return __fadd_rn(__fmaf_rn(y, b, __fmul_rn(x, a)), c);
}

template <bool NEAREST>
__global__ void __launch_bounds__(256) aug_grid_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int H, int W, int OH,
                                                       int OW, AugGrid g) {
  const int64_t n = (int64_t)OH * OW;
  const int b = blockIdx.y;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(k / OW), ox = (int)(k - (int64_t)oy * OW);
    const float bx = __ldg(g.xs + ox), by = __ldg(g.ys + oy);
    float gx = aug_dot3(bx, by, g.t[0], g.t[2], g.t[4]);
    float gy = aug_dot3(bx, by, g.t[1], g.t[3], g.t[5]);
    if (g.persp) {
      const float den = aug_dot3(bx, by, g.p[0], g.p[1], 1.f);
      gx = __fsub_rn(__fdiv_rn(gx, den), 1.f);
      gy = __fsub_rn(__fdiv_rn(gy, den), 1.f);
    }
    // grid_sample, align_corners=False, as ATen's CPU kernel computes it: (g + 1) * (size / 2) - 0.5
    const float ix = __fsub_rn(__fmul_rn(__fadd_rn(gx, 1.f), 0.5f * (float)W), 0.5f);
    const float iy = __fsub_rn(__fmul_rn(__fadd_rn(gy, 1.f), 0.5f * (float)H), 0.5f);
    const float* src = x + (int64_t)b * C * H * W;
    float* dst = y + (int64_t)b * C * n + k;
    if (NEAREST) {
      const float rx = nearbyintf(ix), ry = nearbyintf(iy);
      const bool in = rx >= 0.f && rx < (float)W && ry >= 0.f && ry < (float)H;
      const int64_t off = in ? (int64_t)ry * W + (int64_t)rx : 0;
      for (int c = 0; c < C; ++c) dst[(int64_t)c * n] = in ? __ldg(src + (int64_t)c * H * W + off) : 0.f;
    } else {
      const float x0 = floorf(ix), y0 = floorf(iy);
      const float wx = __fsub_rn(ix, x0), ex = __fsub_rn(1.f, wx), wy = __fsub_rn(iy, y0), sy = __fsub_rn(1.f, wy);
      const float w4[4] = {__fmul_rn(sy, ex), __fmul_rn(sy, wx), __fmul_rn(wy, ex), __fmul_rn(wy, wx)};
      int64_t off[4];
      bool in[4];
      for (int q = 0; q < 4; ++q) {
        const float cx = x0 + (float)(q & 1), cy = y0 + (float)(q >> 1);
        in[q] = cx >= 0.f && cx < (float)W && cy >= 0.f && cy < (float)H;
        off[q] = in[q] ? (int64_t)cy * W + (int64_t)cx : 0;
      }
      for (int c = 0; c < C; ++c) {
        const float* s = src + (int64_t)c * H * W;
        float acc = __fmul_rn(in[0] ? __ldg(s + off[0]) : 0.f, w4[0]);
        for (int q = 1; q < 4; ++q) acc = __fadd_rn(acc, __fmul_rn(in[q] ? __ldg(s + off[q]) : 0.f, w4[q]));
        dst[(int64_t)c * n] = acc;
      }
    }
  }
}

// ---------------------------------------------------------------- colour
// torchvision's rgb_to_grayscale: (0.2989 r + 0.587 g) + 0.114 b in fp32
__device__ __forceinline__ float aug_tv_gray(float r, float g, float b) {
  return __fadd_rn(__fadd_rn(__fmul_rn(0.2989f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, b));
}

// grid (nblk, B): block (blk, b) writes the fp64 sum of its grid-strided pixels of image b to part[b * nblk + blk]
__global__ void __launch_bounds__(kAugSumThreads) aug_gray_sum_kernel(const float* __restrict__ x, int64_t HW, double* __restrict__ part) {
  const float* img = x + (int64_t)blockIdx.y * 3 * HW;
  double s = 0.0;
  for (int64_t k = (int64_t)blockIdx.x * kAugSumThreads + threadIdx.x; k < HW; k += (int64_t)gridDim.x * kAugSumThreads)
    s += (double)aug_tv_gray(__ldg(img + k), __ldg(img + HW + k), __ldg(img + 2 * HW + k));
  __shared__ double red[kAugSumThreads];
  red[threadIdx.x] = s;
  __syncthreads();
  for (int h = kAugSumThreads / 2; h > 0; h >>= 1) {
    if (threadIdx.x < h) red[threadIdx.x] += red[threadIdx.x + h];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[(int64_t)blockIdx.y * gridDim.x + blockIdx.x] = red[0];
}

__device__ __forceinline__ float aug_clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// _rgb2hsv, hue shift, _hsv2rgb (torchvision/transforms/_functional_tensor.py) in fp32
__device__ __forceinline__ void aug_hue(float& r, float& g, float& b, float shift) {
  const float maxc = fmaxf(fmaxf(r, g), b), minc = fminf(fminf(r, g), b);
  const bool eqc = maxc == minc;
  const float cr = __fsub_rn(maxc, minc);
  const float s = __fdiv_rn(cr, eqc ? 1.f : maxc);
  const float crd = eqc ? 1.f : cr;
  const float rc = __fdiv_rn(__fsub_rn(maxc, r), crd), gc = __fdiv_rn(__fsub_rn(maxc, g), crd), bc = __fdiv_rn(__fsub_rn(maxc, b), crd);
  const float hr = maxc == r ? __fsub_rn(bc, gc) : 0.f;
  const float hg = (maxc == g && maxc != r) ? __fsub_rn(__fadd_rn(2.f, rc), bc) : 0.f;
  const float hb = (maxc != g && maxc != r) ? __fsub_rn(__fadd_rn(4.f, gc), rc) : 0.f;
  float h = __fadd_rn(__fadd_rn(hr, hg), hb);
  h = fmodf(__fadd_rn(__fdiv_rn(h, 6.f), 1.f), 1.f);
  // (h + hue_factor) % 1.0: Python-style remainder, the sign of the divisor
  h = __fadd_rn(h, shift);
  h = __fsub_rn(h, floorf(h));
  const float v = maxc;
  const float h6 = __fmul_rn(h, 6.f);
  const float fi = floorf(h6);
  const float f = __fsub_rn(h6, fi);
  int i = ((int)fi) % 6;
  if (i < 0) i += 6;
  const float p = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, s)));
  const float q = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, f))));
  const float t = aug_clamp01(__fmul_rn(v, __fsub_rn(1.f, __fmul_rn(s, __fsub_rn(1.f, f)))));
  switch (i) {
    case 0: r = v; g = t; b = p; break;
    case 1: r = q; g = v; b = p; break;
    case 2: r = p; g = v; b = t; break;
    case 3: r = p; g = q; b = v; break;
    case 4: r = t; g = p; b = v; break;
    default: r = v; g = p; b = q; break;
  }
}

// grid (blocks, B); one thread per pixel.  f = ratio, f1 = 1 - ratio (both rounded to fp32 on the host, as torch rounds the Python
// scalars); contrast reads its image's nblk partial sums from `part`.
__global__ void __launch_bounds__(256) aug_color_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t HW, int op, float f,
                                                        float f1, const double* __restrict__ part, int nblk) {
  const int b = blockIdx.y;
  float other = 0.f;
  if (op == kAugContrast) {
    __shared__ float mean_s;
    if (threadIdx.x == 0) {
      double s = 0.0;
      for (int i = 0; i < nblk; ++i) s += part[(int64_t)b * nblk + i];
      mean_s = (float)(s / (double)HW);
    }
    __syncthreads();
    other = mean_s;
  }
  const float* src = x + (int64_t)b * 3 * HW;
  float* dst = y + (int64_t)b * 3 * HW;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < HW; k += (int64_t)gridDim.x * blockDim.x) {
    float r = __ldg(src + k), g = __ldg(src + HW + k), bl = __ldg(src + 2 * HW + k);
    if (op == kAugGrayscale) {
      const float l = __fadd_rn(__fadd_rn(__fmul_rn(0.299f, r), __fmul_rn(0.587f, g)), __fmul_rn(0.114f, bl));
      r = g = bl = l;
    } else if (op == kAugHue) {
      aug_hue(r, g, bl, f);
    } else {
      const float o = op == kAugSaturation ? aug_tv_gray(r, g, bl) : other;
      const float ob = __fmul_rn(f1, o);
      r = aug_clamp01(__fadd_rn(__fmul_rn(f, r), ob));
      g = aug_clamp01(__fadd_rn(__fmul_rn(f, g), ob));
      bl = aug_clamp01(__fadd_rn(__fmul_rn(f, bl), ob));
    }
    dst[k] = r; dst[HW + k] = g; dst[2 * HW + k] = bl;
  }
}

// ---------------------------------------------------------------- Gaussian blur (reflect padding, taps in constant memory)
constexpr int kAugMaxTaps = 33;
struct AugTaps { float w[kAugMaxTaps]; int k; };

__device__ __forceinline__ int aug_reflect(int i, int n) { return i < 0 ? -i : (i >= n ? 2 * n - 2 - i : i); }

// one block per (row strip of 1 row, plane): the row and its halo in shared memory
__global__ void __launch_bounds__(256) aug_blur_h_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, AugTaps t) {
  extern __shared__ float row[];
  const int pad = t.k / 2;
  const int64_t base = ((int64_t)blockIdx.y * H + blockIdx.x) * W;
  for (int i = threadIdx.x; i < W + 2 * pad; i += blockDim.x) row[i] = __ldg(x + base + aug_reflect(i - pad, W));
  __syncthreads();
  for (int i = threadIdx.x; i < W; i += blockDim.x) {
    float acc = 0.f;
    for (int j = 0; j < t.k; ++j) acc = __fmaf_rn(t.w[j], row[i + j], acc);
    y[base + i] = acc;
  }
}

__global__ void __launch_bounds__(256) aug_blur_v_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, AugTaps t) {
  const int pad = t.k / 2;
  const int64_t plane = (int64_t)blockIdx.y * H * W;
  const int64_t n = (int64_t)H * W;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < n; k += (int64_t)gridDim.x * blockDim.x) {
    const int r = (int)(k / W), c = (int)(k - (int64_t)r * W);
    float acc = 0.f;
    for (int j = 0; j < t.k; ++j) acc = __fmaf_rn(t.w[j], __ldg(x + plane + (int64_t)aug_reflect(r + j - pad, H) * W + c), acc);
    y[plane + k] = acc;
  }
}

// ---------------------------------------------------------------- temporal window averaging
// The reference's WindowAveraging (augmentation/video.py:455-485) on a clip x [T, n] (n = 3 H W floats per frame), with
// HH = window // 2 after window = min(window, T):
//   y[i] = (1 - alpha) x[i] + alpha mean(x[max(0, i - HH) : min(T, i + HH + 1)])
// The mean is what torch.mean computes there: a fresh fp32 sum of the window's frames in frame order, divided by their count; the
// blend is the three rounded operations of the Python expression, with a_keep = fp32(1 - alpha) and a_avg = fp32(alpha).
// Each thread owns one VEC-float vector of a frame position and walks the T frames, keeping the 2 HH + 1 newest frame vectors in a
// register ring (frame j in slot j % K), so every input byte is read once and every output byte written once.  The time loop is
// unrolled by K so that every slot index is a compile-time constant.
template <int VEC> struct AugVec;
template <> struct AugVec<4> { using T = float4; };
template <> struct AugVec<1> { using T = float; };

template <int VEC>
__device__ __forceinline__ void aug_vadd(float* s, const typename AugVec<VEC>::T& v) {
  const float* f = reinterpret_cast<const float*>(&v);
#pragma unroll
  for (int e = 0; e < VEC; ++e) s[e] = __fadd_rn(s[e], f[e]);
}

constexpr int kAugMaxHalfWindow = 8;   // windows of up to 17 frames

template <int HH, int VEC>
__global__ void __launch_bounds__(256) aug_window_avg_kernel(const float* __restrict__ x, float* __restrict__ y, int T, int64_t nvec,
                                                             float a_keep, float a_avg) {
  using V = typename AugVec<VEC>::T;
  constexpr int K = 2 * HH + 1;
  const int64_t p = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (p >= nvec) return;
  const V* src = reinterpret_cast<const V*>(x) + p;
  V* dst = reinterpret_cast<V*>(y) + p;
  V ring[K];
#pragma unroll
  for (int j = 0; j < HH; ++j)
    if (j < T) ring[j] = __ldg(src + (int64_t)j * nvec);
  for (int i0 = 0; i0 < T; i0 += K) {
#pragma unroll
    for (int s = 0; s < K; ++s) {
      const int i = i0 + s;
      if (i < T) {
        if (i + HH < T) ring[(s + HH) % K] = __ldg(src + (int64_t)(i + HH) * nvec);
        float sum[VEC];
#pragma unroll
        for (int e = 0; e < VEC; ++e) sum[e] = 0.f;
#pragma unroll
        for (int k = 0; k < K; ++k) {          // frames i - HH .. i + HH, in order
          const int j = i - HH + k;
          if (j >= 0 && j < T) aug_vadd<VEC>(sum, ring[(s + k + K - HH % K) % K]);
        }
        const float cnt = (float)(min(T, i + HH + 1) - max(0, i - HH));
        const float* xi = reinterpret_cast<const float*>(&ring[s % K]);
        V o;
        float* of = reinterpret_cast<float*>(&o);
#pragma unroll
        for (int e = 0; e < VEC; ++e) of[e] = __fadd_rn(__fmul_rn(a_keep, xi[e]), __fmul_rn(a_avg, __fdiv_rn(sum[e], cnt)));
        dst[(int64_t)i * nvec] = o;
      }
    }
  }
}

// ---------------------------------------------------------------- JPEG
struct JpegQ { int32_t q[2][64]; };          // luma / chroma quantisation tables, natural order

__device__ __forceinline__ int jp_descale(long long x, int n) { return (int)((x + (1ll << (n - 1))) >> n); }

// one pass of the islow forward DCT over 8 values `stride` apart (pass 1: rows, pass 2: columns)
__device__ void jp_fdct8(int* d, int stride, bool pass1) {
  const long long t0 = d[0] + d[7 * stride], t7 = d[0] - d[7 * stride], t1 = d[stride] + d[6 * stride], t6 = d[stride] - d[6 * stride];
  const long long t2 = d[2 * stride] + d[5 * stride], t5 = d[2 * stride] - d[5 * stride];
  const long long t3 = d[3 * stride] + d[4 * stride], t4 = d[3 * stride] - d[4 * stride];
  const long long t10 = t0 + t3, t13 = t0 - t3, t11 = t1 + t2, t12 = t1 - t2;
  const int sh = pass1 ? 11 : 15;
  d[0] = pass1 ? (int)((t10 + t11) << 2) : jp_descale(t10 + t11, 2);
  d[4 * stride] = pass1 ? (int)((t10 - t11) << 2) : jp_descale(t10 - t11, 2);
  const long long z1 = (t12 + t13) * 4433;
  d[2 * stride] = jp_descale(z1 + t13 * 6270, sh);
  d[6 * stride] = jp_descale(z1 - t12 * 15137, sh);
  const long long z5 = (t4 + t6 + t5 + t7) * 9633;
  const long long a1 = -(t4 + t7) * 7373, a2 = -(t5 + t6) * 20995, a3 = -(t4 + t6) * 16069 + z5, a4 = -(t5 + t7) * 3196 + z5;
  d[7 * stride] = jp_descale(t4 * 2446 + a1 + a3, sh);
  d[5 * stride] = jp_descale(t5 * 16819 + a2 + a4, sh);
  d[3 * stride] = jp_descale(t6 * 25172 + a2 + a3, sh);
  d[stride] = jp_descale(t7 * 12299 + a1 + a4, sh);
}

// one pass of the islow inverse DCT (pass 1: columns, descale 11; pass 2: rows, descale 18 and the post-IDCT range limit)
__device__ void jp_idct8(int* d, int stride, bool pass1) {
  const long long z2 = d[2 * stride], z3 = d[6 * stride];
  const long long z1 = (z2 + z3) * 4433;
  const long long e2 = z1 - z3 * 15137, e3 = z1 + z2 * 6270;
  const long long e0 = (long long)(d[0] + d[4 * stride]) << 13, e1 = (long long)(d[0] - d[4 * stride]) << 13;
  const long long t10 = e0 + e3, t13 = e0 - e3, t11 = e1 + e2, t12 = e1 - e2;
  long long o0 = d[7 * stride], o1 = d[5 * stride], o2 = d[3 * stride], o3 = d[stride];
  const long long z5 = (o0 + o2 + o1 + o3) * 9633;
  const long long a1 = -(o0 + o3) * 7373, a2 = -(o1 + o2) * 20995, a3 = -(o0 + o2) * 16069 + z5, a4 = -(o1 + o3) * 3196 + z5;
  o0 = o0 * 2446 + a1 + a3; o1 = o1 * 16819 + a2 + a4; o2 = o2 * 25172 + a2 + a3; o3 = o3 * 12299 + a1 + a4;
  const int sh = pass1 ? 11 : 18;
  int r[8] = {jp_descale(t10 + o3, sh), jp_descale(t11 + o2, sh), jp_descale(t12 + o1, sh), jp_descale(t13 + o0, sh),
              jp_descale(t13 - o0, sh), jp_descale(t12 - o1, sh), jp_descale(t11 - o2, sh), jp_descale(t10 - o3, sh)};
  for (int i = 0; i < 8; ++i) {
    int v = r[i];
    if (!pass1) {   // libjpeg's range-limit table on the low ten bits: clamp(v + 128, 0, 255) for |v| <= 512
      const int m = v & 1023;
      v = m < 128 ? m + 128 : (m < 512 ? 255 : (m < 896 ? 0 : m - 896));
    }
    d[i * stride] = v;
  }
}

// libjpeg-turbo's quantiser: (|t| + corr) * recip >> shift with its 16-bit reciprocal of 8q, sign restored; then dequantised
__device__ __forceinline__ int jp_quant_dequant(int t, int q) {
  const int d = q * 8;
  const int b = 31 - __clz(d);
  int r = 16 + b;
  long long fq = (1ll << r) / d;
  const long long fr = (1ll << r) % d;
  long long c = d / 2;
  if (fr == 0) { fq >>= 1; --r; }
  else if (fr <= d / 2) ++c;
  else ++fq;
  const long long a = t < 0 ? -(long long)t : t;
  const int qv = (int)(((a + c) * fq) >> r);
  return (t < 0 ? -qv : qv) * q;
}

__device__ __forceinline__ int jp_u8(float v) { return (int)__fmul_rn(aug_clamp01(v), 255.f); }   // ToPILImage: x * 255, truncated

// grid (ceil(W/16), ceil(H/16), B), 256 threads: one 16x16 MCU.  Y -> yp [B][H][W], Cb / Cr -> cp [B][2][CH][CW] (CH, CW = ceil / 2)
__global__ void __launch_bounds__(256) jpeg_mcu_kernel(const float* __restrict__ x, uint8_t* __restrict__ yp, uint8_t* __restrict__ cp, int H,
                                                       int W, JpegQ qt) {
  __shared__ int yb[16][16];
  __shared__ int cf[2][16][16];   // full-resolution chroma, then the 8x8 downsampled block in [.][0..7][0..7]
  __shared__ int blk[6][64];      // 4 luma blocks, Cb, Cr
  const int tid = threadIdx.x, b = blockIdx.z;
  const int x0 = blockIdx.x * 16, y0 = blockIdx.y * 16;
  const int64_t HW = (int64_t)H * W;
  const float* img = x + (int64_t)b * 3 * HW;
  {
    const int r = tid >> 4, c = tid & 15;
    const int gy = min(y0 + r, H - 1), gx = min(x0 + c, W - 1);   // edge replication up to whole MCUs
    const int64_t o = (int64_t)gy * W + gx;
    const int R = jp_u8(__ldg(img + o)), G = jp_u8(__ldg(img + HW + o)), B = jp_u8(__ldg(img + 2 * HW + o));
    yb[r][c] = (19595 * R + 38470 * G + 7471 * B + 32768) >> 16;
    cf[0][r][c] = (-11059 * R - 21709 * G + 32768 * B + (128 << 16) + 32767) >> 16;
    cf[1][r][c] = (32768 * R - 27439 * G - 5329 * B + (128 << 16) + 32767) >> 16;
  }
  __syncthreads();
  // h2v2 downsample with the 1, 2 bias; rows past the even-rounded height repeat the last downsampled row of the image
  const int he2 = (H + 1) >> 1;   // downsampled rows computed from image rows
  int cds = 0;
  if (tid < 128) {
    const int comp = tid >> 6, r = (tid >> 3) & 7, c = tid & 7;
    const int rr = min(blockIdx.y * 8 + r, he2 - 1) - blockIdx.y * 8;
    cds = (cf[comp][2 * rr][2 * c] + cf[comp][2 * rr][2 * c + 1] + cf[comp][2 * rr + 1][2 * c] + cf[comp][2 * rr + 1][2 * c + 1] + 1 + (c & 1)) >> 2;
  }
  for (int i = tid; i < 256; i += 256) {
    const int r = i >> 4, c = i & 15;
    blk[(r >> 3) * 2 + (c >> 3)][(r & 7) * 8 + (c & 7)] = yb[r][c] - 128;
  }
  __syncthreads();
  if (tid < 128) blk[4 + (tid >> 6)][tid & 63] = cds - 128;
  __syncthreads();
  if (tid < 48) jp_fdct8(&blk[tid >> 3][(tid & 7) * 8], 1, true);
  __syncthreads();
  if (tid < 48) jp_fdct8(&blk[tid >> 3][tid & 7], 8, false);
  __syncthreads();
  for (int i = tid; i < 384; i += 256) {
    const int k = i >> 6, e = i & 63;
    blk[k][e] = jp_quant_dequant(blk[k][e], qt.q[k >= 4][e]);
  }
  __syncthreads();
  if (tid < 48) jp_idct8(&blk[tid >> 3][tid & 7], 8, true);
  __syncthreads();
  if (tid < 48) jp_idct8(&blk[tid >> 3][(tid & 7) * 8], 1, false);
  __syncthreads();
  {
    const int r = tid >> 4, c = tid & 15;
    if (y0 + r < H && x0 + c < W) yp[(int64_t)b * HW + (int64_t)(y0 + r) * W + x0 + c] = (uint8_t)blk[(r >> 3) * 2 + (c >> 3)][(r & 7) * 8 + (c & 7)];
  }
  if (tid < 128) {
    const int comp = tid >> 6, r = (tid >> 3) & 7, c = tid & 7;
    const int CH = (H + 1) >> 1, CW = (W + 1) >> 1;
    const int gy = blockIdx.y * 8 + r, gx = blockIdx.x * 8 + c;
    if (gy < CH && gx < CW) cp[(((int64_t)b * 2 + comp) * CH + gy) * CW + gx] = (uint8_t)blk[4 + comp][tid & 63];
  }
}

// triangle (fancy) h2v2 upsampling of one chroma sample for output pixel (oy, ox); 2x2 replication when CW <= 2
__device__ __forceinline__ int jp_upsample(const uint8_t* __restrict__ p, int CH, int CW, int oy, int ox) {
  const int r = oy >> 1, c = ox >> 1;
  if (CW <= 2) return __ldg(p + (int64_t)r * CW + c);
  const int rn = (oy & 1) ? min(r + 1, CH - 1) : max(r - 1, 0);
  const int cn = (ox & 1) ? min(c + 1, CW - 1) : max(c - 1, 0);
  const uint8_t* a = p + (int64_t)r * CW;
  const uint8_t* n = p + (int64_t)rn * CW;
  const int s = 3 * __ldg(a + c) + __ldg(n + c), sn = 3 * __ldg(a + cn) + __ldg(n + cn);
  return (3 * s + sn + ((ox & 1) ? 7 : 8)) >> 4;
}

// one thread per pixel: upsample, YCbCr -> RGB, u8 / 255, then the reference's pass-through (jpeg - x) + x on the clamped input
__global__ void __launch_bounds__(256) jpeg_rgb_kernel(const float* __restrict__ x, const uint8_t* __restrict__ yp, const uint8_t* __restrict__ cp,
                                                       float* __restrict__ y, int H, int W) {
  const int64_t HW = (int64_t)H * W;
  const int b = blockIdx.y;
  const int CH = (H + 1) >> 1, CW = (W + 1) >> 1;
  const uint8_t* cb = cp + (int64_t)b * 2 * CH * CW;
  const uint8_t* cr = cb + (int64_t)CH * CW;
  for (int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; k < HW; k += (int64_t)gridDim.x * blockDim.x) {
    const int oy = (int)(k / W), ox = (int)(k - (int64_t)oy * W);
    const int Y = __ldg(yp + (int64_t)b * HW + k);
    const int xb = jp_upsample(cb, CH, CW, oy, ox) - 128, xr = jp_upsample(cr, CH, CW, oy, ox) - 128;
    const int rgb[3] = {Y + ((91881 * xr + 32768) >> 16), Y + ((-22554 * xb + 32768 - 46802 * xr) >> 16), Y + ((116130 * xb + 32768) >> 16)};
    for (int c = 0; c < 3; ++c) {
      const float j = __fdiv_rn((float)min(max(rgb[c], 0), 255), 255.f);
      const float xc = aug_clamp01(__ldg(x + ((int64_t)b * 3 + c) * HW + k));
      y[((int64_t)b * 3 + c) * HW + k] = __fadd_rn(__fsub_rn(j, xc), xc);
    }
  }
}

}  // namespace vsb
