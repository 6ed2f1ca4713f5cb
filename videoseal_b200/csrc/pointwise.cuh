// CUDA-core kernels of the hot path that are bound by HBM / L2 bandwidth, not by the tensor pipe:
//   K5  resample_kernel        antialiased / plain bilinear resize with precomputed separable taps
//   K0  unet_first_kernel      U-Net `inc` first conv (C_in = 1 or 3) + folded BN + ReLU, and the 1x1 res conv
//   K6  msg_embed_kernel       message bits -> embedding sum -> per-sample constant channels of the bottleneck input
//   K7  jnd_blend_kernel       delta up-resample x JND heat-map x scaling_w + scaling_i * img, clamp (128-bit vectorised)
//   K9  stem_ln_kernel         ConvNeXt stem conv k4 (stride 4 / 2) + channels-first LayerNorm
//   K4  dwconv7_ln_kernel      depthwise 7x7 + channels-last LayerNorm -> fp16 GEMM operand
//   K4b ln_rows_kernel         per-pixel LayerNorm over C (downsample layers) -> fp16
//   K8  head_pool_kernel / head_linear_kernel   LN + GELU + spatial mean, then Linear(C -> 1 + nbits)
#pragma once
#include <type_traits>
#include "conv_gemm.cuh"
#include "ptx.cuh"

namespace vsb {

// ------------------------------------------------------------------------------------------------
// K5: generic separable resample.  For each output index o along an axis: taps [start[o], start[o]+cnt[o]) with
// weights w[o*maxt + j].  Tables are built on the host to match ATen exactly
// (aten/src/ATen/native/cpu/UpSampleKernel.cpp: _compute_indices_weights_aa; F.interpolate call sites
// videoseal/models/wam.py:163,184,224 and models/videoseal.py:305,329).
struct ResampleTab {
  const int* ystart; const int* ycnt; const float* yw;
  const int* xstart; const int* xcnt; const float* xw;
  int maxt_y, maxt_x;
};

// (the kernel that consumes these tables is resize_sep_kernel in resize_blend.cuh)

// ------------------------------------------------------------------------------------------------
// K0: first U-Net layer.  imgs: [B, 3, H, W] fp32 RGB in [0,1] (H = W = processing size).  If yuv: x = 2*Y-1 with
// Y = .299R + .587G + .114B (data/transforms.py:15-27, wam.py:168-172, embedder.py:23), else x = 2*rgb-1 (3 ch).
// h1 = relu(conv3x3(x; w1') + b1')   (BN folded)      -> NHWC fp16 [B,H,W,Z]
// r  = conv1x1(x; wr) + br                             -> NHWC fp16 [B,H,W,Z]
// (modules/unet.py:24-39 for the `inc` block).  Zero padding applies to the preprocessed x.
// Thread = 4 horizontally adjacent pixels x 8 of every 16 output channels (block = 16 rows x 32 columns; lane bit 0 picks the channel
// half): every weight load feeds 4 FMAs, the 3 x 6 input window of the 4 pixels lives in registers, and the two lanes of a pair
// store the two 16-byte halves of a pixel's 32-byte channel group in the SAME instruction (full sectors).  The first version (1 pixel
// per thread, all channels) executed one weight load per FMA and was issue-bound at 152 us for a 64-frame batch against a 49 us HBM
// bound (318 MB).  Z % 16 == 0.
template <int CIN>
__global__ void __launch_bounds__(256) unet_first_kernel(const float* __restrict__ imgs, int B, int H, int W, int Z,
                                                         const float* __restrict__ w1 /*[Z][CIN][3][3]*/, const float* __restrict__ b1,
                                                         const float* __restrict__ wr /*[Z][CIN]*/, const float* __restrict__ br,
                                                         __half* __restrict__ h1, __half* __restrict__ res, int yuv) {
  constexpr int NP = 4, TW = 8 * NP, TH = 16;
  __shared__ float tile[CIN][TH + 2][TW + 2 + 2];
  const int zh = threadIdx.x & 1, tx = (threadIdx.x >> 1) & 7, ty = threadIdx.x >> 4;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH, b = blockIdx.z;
  const float* img = imgs + (long)b * 3 * H * W;
  for (int i = threadIdx.x; i < (TH + 2) * (TW + 2); i += 256) {
    const int ly = i / (TW + 2), lx = i - ly * (TW + 2);
    const int gy = y0 + ly - 1, gx = x0 + lx - 1;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    if (CIN == 1) {
      float v = 0.f;
      if (in) {
        const long o = (long)gy * W + gx;
        const float y = 0.299f * __ldg(img + o) + 0.587f * __ldg(img + (long)H * W + o) + 0.114f * __ldg(img + 2L * H * W + o);
        v = 2.f * y - 1.f;
      }
      tile[0][ly][lx] = v;
    } else {
#pragma unroll
      for (int c = 0; c < CIN; ++c) tile[c][ly][lx] = in ? 2.f * __ldg(img + (long)c * H * W + (long)gy * W + gx) - 1.f : 0.f;
    }
  }
  __syncthreads();
  const int gx = x0 + tx * NP, gy = y0 + ty;
  if (gx >= W || gy >= H) return;
  const long pix = ((long)b * H + gy) * W + gx;
  const int npx = min(NP, W - gx);
  for (int zb = 0; zb < Z; zb += 16) {
    const int z0 = zb + 8 * zh;
    float a[8][NP], rr[8][NP];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float bz = __ldg(b1 + z0 + q), brz = __ldg(br + z0 + q);
#pragma unroll
      for (int p = 0; p < NP; ++p) { a[q][p] = bz; rr[q][p] = brz; }
    }
#pragma unroll
    for (int c = 0; c < CIN; ++c) {
#pragma unroll
      for (int r = 0; r < 3; ++r) {
        float xr[NP + 2];
#pragma unroll
        for (int s = 0; s < NP + 2; ++s) xr[s] = tile[c][ty + r][tx * NP + s];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
#pragma unroll
          for (int s = 0; s < 3; ++s) {
            const float wv = __ldg(w1 + ((z0 + q) * CIN + c) * 9 + r * 3 + s);
#pragma unroll
            for (int p = 0; p < NP; ++p) a[q][p] = fmaf(xr[p + s], wv, a[q][p]);
          }
          if (r == 1) {
            const float wv = __ldg(wr + (z0 + q) * CIN + c);
#pragma unroll
            for (int p = 0; p < NP; ++p) rr[q][p] = fmaf(xr[p + 1], wv, rr[q][p]);
          }
        }
      }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      if (p < npx) {
        __align__(16) __half ho[8];
        __align__(16) __half ro[8];
#pragma unroll
        for (int q = 0; q < 8; ++q) { ho[q] = __float2half_rn(fmaxf(a[q][p], 0.f)); ro[q] = __float2half_rn(rr[q][p]); }
        *reinterpret_cast<uint4*>(h1 + (pix + p) * Z + z0) = *reinterpret_cast<const uint4*>(ho);
        *reinterpret_cast<uint4*>(res + (pix + p) * Z + z0) = *reinterpret_cast<const uint4*>(ro);
      }
    }
  }
}

// K0 for Z = 8 (unet_tiny_*): the same arithmetic with the whole 16-byte pixel per thread.  Thread = 4 horizontally adjacent
// pixels x all 8 channels (block = 16 rows x 64 columns); the 16 lanes of a half-warp store 64 consecutive pixels' 1 KB.
template <int CIN>
__global__ void __launch_bounds__(256) unet_first_z8_kernel(const float* __restrict__ imgs, int B, int H, int W,
                                                            const float* __restrict__ w1 /*[8][CIN][3][3]*/, const float* __restrict__ b1,
                                                            const float* __restrict__ wr /*[8][CIN]*/, const float* __restrict__ br,
                                                            __half* __restrict__ h1, __half* __restrict__ res, int yuv) {
  constexpr int NP = 4, TW = 16 * NP, TH = 16;
  __shared__ float tile[CIN][TH + 2][TW + 2 + 2];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH, b = blockIdx.z;
  const float* img = imgs + (long)b * 3 * H * W;
  for (int i = threadIdx.x; i < (TH + 2) * (TW + 2); i += 256) {
    const int ly = i / (TW + 2), lx = i - ly * (TW + 2);
    const int gy = y0 + ly - 1, gx = x0 + lx - 1;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W;
    if (CIN == 1) {
      float v = 0.f;
      if (in) {
        const long o = (long)gy * W + gx;
        const float y = 0.299f * __ldg(img + o) + 0.587f * __ldg(img + (long)H * W + o) + 0.114f * __ldg(img + 2L * H * W + o);
        v = 2.f * y - 1.f;
      }
      tile[0][ly][lx] = v;
    } else {
#pragma unroll
      for (int c = 0; c < CIN; ++c) tile[c][ly][lx] = in ? 2.f * __ldg(img + (long)c * H * W + (long)gy * W + gx) - 1.f : 0.f;
    }
  }
  __syncthreads();
  const int gx = x0 + tx * NP, gy = y0 + ty;
  if (gx >= W || gy >= H) return;
  const long pix = ((long)b * H + gy) * W + gx;
  const int npx = min(NP, W - gx);
  float a[8][NP], rr[8][NP];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const float bz = __ldg(b1 + q), brz = __ldg(br + q);
#pragma unroll
    for (int p = 0; p < NP; ++p) { a[q][p] = bz; rr[q][p] = brz; }
  }
#pragma unroll
  for (int c = 0; c < CIN; ++c) {
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      float xr[NP + 2];
#pragma unroll
      for (int s = 0; s < NP + 2; ++s) xr[s] = tile[c][ty + r][tx * NP + s];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
#pragma unroll
        for (int s = 0; s < 3; ++s) {
          const float wv = __ldg(w1 + (q * CIN + c) * 9 + r * 3 + s);
#pragma unroll
          for (int p = 0; p < NP; ++p) a[q][p] = fmaf(xr[p + s], wv, a[q][p]);
        }
        if (r == 1) {
          const float wv = __ldg(wr + q * CIN + c);
#pragma unroll
          for (int p = 0; p < NP; ++p) rr[q][p] = fmaf(xr[p + 1], wv, rr[q][p]);
        }
      }
    }
  }
#pragma unroll
  for (int p = 0; p < NP; ++p) {
    if (p < npx) {
      __align__(16) __half ho[8];
      __align__(16) __half ro[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) { ho[q] = __float2half_rn(fmaxf(a[q][p], 0.f)); ro[q] = __float2half_rn(rr[q][p]); }
      *reinterpret_cast<uint4*>(h1 + (pix + p) * 8) = *reinterpret_cast<const uint4*>(ho);
      *reinterpret_cast<uint4*>(res + (pix + p) * 8) = *reinterpret_cast<const uint4*>(ro);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K6: modules/msg_processor.py:88-115 (binary + concat).  msgs: [B, K] uint8 {0,1}; table: [2K, hidden] fp32.
// Writes the `hidden` message channels (constant over the h x w map) into channels [c_off, c_off+hidden) of the
// NHWC fp16 bottleneck input `cat` ([B, h*w, ld]).
__global__ void msg_embed_kernel(const uint8_t* __restrict__ msgs, const float* __restrict__ table, int K, int hidden,
                                 __half* __restrict__ cat, int hw, int ld, int c_off, int msg_stride /*0: one message for all*/) {
  extern __shared__ float emb[];  // [hidden]
  const int b = blockIdx.x;
  const uint8_t* m = msgs + (long)b * msg_stride;
  for (int d = threadIdx.x; d < hidden; d += blockDim.x) {
    float a = 0.f;
    for (int k = 0; k < K; ++k) a += __ldg(table + (long)(2 * k + (m[k] ? 1 : 0)) * hidden + d);
    emb[d] = a;
  }
  __syncthreads();
  const int chunk = (hw + gridDim.y - 1) / gridDim.y;
  const int p0 = blockIdx.y * chunk, p1 = min(hw, p0 + chunk);
  const int h2 = hidden >> 1;
  for (long i = (long)p0 * h2 + threadIdx.x; i < (long)p1 * h2; i += blockDim.x) {
    const int pix = (int)(i / h2), d2 = (int)(i - (long)pix * h2);
    *reinterpret_cast<__half2*>(cat + ((long)b * hw + pix) * ld + c_off + 2 * d2) = __floats2half2_rn(emb[2 * d2], emb[2 * d2 + 1]);
  }
}

// ------------------------------------------------------------------------------------------------
// K7: JND heat-map (modules/jnd.py:63-108, jnd_1_1) x up-resampled delta, additive blend, clamp
// (models/wam.py:183-201, models/blender.py:61-68, models/videoseal.py:80-118 `repeat`/`alternate`).
//   imgs   [F, 3, H, W] fp32;  delta [Nk, CD, PH, PW] fp32 (CD = 1 or 3), key frame of frame f = f / step
//   imgs_w [F, 3, H, W];  preds_w (optional) [F, CD, H, W] = hmap * delta_up  (NOT yet multiplied by scaling_w)
struct BlendParams {
  const float* imgs; const float* delta; float* imgs_w; float* preds_w;
  int F, H, W, PH, PW, CD, step, alternate;
  int interp_chunk;  // > 0: video_mode 'interpolate' with this many key frames per chunk (frame 0 starts a chunk)
  int use_jnd, clamp, identity_resample;
  int jnd_in, jnd_out;   // configs/attenuation.yaml in_channels / out_channels (1 or 3 each); preds_w has max(CD, jnd_out) channels
  float scaling_i, scaling_w;
  ResampleTab tab;  // delta (PH x PW) -> (H x W); unused when identity_resample
};

constexpr int kBlendTW = 128, kBlendTH = 8;

// Which key-frame deltas feed frame f (models/videoseal.py:80-118).  repeat: key f/step.  alternate: key f/step on the
// key frames, nothing in between.  interpolate: inside a chunk of `interp_chunk` keys, frames before the chunk's last key
// mix key k and k+1 with alpha = 1 - (f % step)/(step-1) (torch.linspace(0,1,step)); from the last key on, that key alone.
struct FrameKeys { int k0, k1; float a; bool has; };
__device__ __forceinline__ FrameKeys frame_keys(int f, int F, int step, int alternate, int interp_chunk) {
  FrameKeys r;
  const int kf = f / step, ph = f - kf * step;
  r.k0 = kf; r.k1 = kf; r.a = 1.f; r.has = !(alternate && ph != 0);
  if (interp_chunk > 0) {
    const int nkeys = (F + step - 1) / step;
    const int c0 = (kf / interp_chunk) * interp_chunk;
    const int nc = min(interp_chunk, nkeys - c0);
    if (kf - c0 < nc - 1 && step > 1) { r.k1 = kf + 1; r.a = 1.f - (float)ph / (float)(step - 1); }
  }
  return r;
}

__device__ __forceinline__ float jnd_from_lum(const float (*lum)[kBlendTW + 4 + 1], int ly, int lx) {
  // lum holds L = 255 * Y with a 2-pixel zero halo; (ly, lx) index the centre pixel inside the halo tile
  const float* r0 = lum[ly - 2] + lx; const float* r1 = lum[ly - 1] + lx; const float* r2 = lum[ly] + lx;
  const float* r3 = lum[ly + 1] + lx; const float* r4 = lum[ly + 2] + lx;
  float la = (r0[-2] + r0[-1] + r0[0] + r0[1] + r0[2]) + (r1[-2] + r1[2]) + (r2[-2] + r2[2]) + (r3[-2] + r3[2]) +
             (r4[-2] + r4[-1] + r4[0] + r4[1] + r4[2]) + 2.f * (r1[-1] + r1[0] + r1[1] + r2[-1] + r2[1] + r3[-1] + r3[0] + r3[1]);
  la *= (1.f / 32.f);
  la = (la <= 127.f) ? 17.f * (1.f - sqrtf(la / 127.f + 1e-5f)) : (3.f / 128.f) * (la - 127.f) + 3.f;
  const float gx = (r1[1] - r1[-1]) + 2.f * (r2[1] - r2[-1]) + (r3[1] - r3[-1]);
  const float gy = (r1[-1] + 2.f * r1[0] + r1[1]) - (r3[-1] + 2.f * r3[0] + r3[1]);
  const float g2 = gx * gx + gy * gy;
  float pw;   // g^2.4 = (g^2)^1.2 on the SFU (lg2 / ex2, ~1e-6 relative); g2 == 0 -> lg2 = -inf -> 0
  asm("{\n\t.reg .f32 t;\n\tlg2.approx.ftz.f32 t, %1;\n\tmul.f32 t, t, 0f3F99999A;\n\tex2.approx.ftz.f32 %0, t;\n\t}" : "=f"(pw) : "f"(g2));
  const float cm = 0.117f * (16.f * pw / (g2 + 676.f));
  return fmaxf(la + cm - 0.3f * fminf(la, cm), 0.f) * (1.f / 255.f);
}

// low-resolution attenuation (wam.py:177-180): delta[k] *= hmap(imgs_res[k*step ... ]) is per FRAME in video mode, so this
// kernel writes a per-frame attenuated delta:  out[f] = hmap(imgs_res[f]) * delta[f / step]   (all at PH x PW).
// JND configurations (configs/attenuation.yaml, modules/jnd.py:80-108): jin = 1: heat-map of the luminance; jin = 3: one heat-map per
// RGB channel (255 * channel through the same filters); jout = 1 with jin = 3: their mean; jout = 3 with jin = 1: the luminance map
// for all three channels.  Output channels PC = max(CD, jout): delta (CD = 1 or 3 channels) and heat-map broadcast against each
// other like `hmaps * preds_w` does.  delta == nullptr: heat-maps only (jout channels).
__global__ void __launch_bounds__(256) jnd_lowres_kernel(const float* __restrict__ imgs_res, const float* __restrict__ delta,
                                                         float* __restrict__ out, int PH, int PW, int CD, int step, int alternate,
                                                         int interp_chunk, int jin, int jout) {
  __shared__ float lum[kBlendTH + 4][kBlendTW + 4 + 1];
  const int f = blockIdx.z;
  const int x0 = blockIdx.x * kBlendTW, y0 = blockIdx.y * kBlendTH;
  const long plane = (long)PH * PW;
  const float* img = imgs_res + (long)f * 3 * plane;
  const int tx = (threadIdx.x & 31) * 4, ty = threadIdx.x >> 5;
  const int gy = y0 + ty;
  float hm[3][4];
  for (int pass = 0; pass < jin; ++pass) {
    if (pass) __syncthreads();
    for (int i = threadIdx.x; i < (kBlendTH + 4) * (kBlendTW + 4); i += 256) {
      const int ly = i / (kBlendTW + 4), lx = i - ly * (kBlendTW + 4);
      const int yy = y0 + ly - 2, xx = x0 + lx - 2;
      float v = 0.f;
      if (yy >= 0 && yy < PH && xx >= 0 && xx < PW) {
        const long o = (long)yy * PW + xx;
        v = jin == 1 ? 0.299f * (255.f * img[o]) + 0.587f * (255.f * img[plane + o]) + 0.114f * (255.f * img[2 * plane + o])
                     : 255.f * img[pass * plane + o];
      }
      lum[ly][lx] = v;
    }
    __syncthreads();
#pragma unroll
    for (int q = 0; q < 4; ++q) hm[pass][q] = (gy < PH && x0 + tx + q < PW) ? jnd_from_lum(lum, ty + 2, tx + q + 2) : 0.f;
  }
  if (gy >= PH) return;
  if (jin == 3 && jout == 1) {
#pragma unroll
    for (int q = 0; q < 4; ++q) hm[0][q] = hm[0][q] / 3.f + hm[1][q] / 3.f + hm[2][q] / 3.f;     // sum(hmaps / 3) / 255, jnd.py:101
  }
  const FrameKeys fk = frame_keys(f, (int)gridDim.z, step, alternate, interp_chunk);
  const int PC = delta == nullptr ? jout : max(CD, jout);
  for (int q = 0; q < 4; ++q) {
    const int gx = x0 + tx + q;
    if (gx >= PW) break;
    const long o = (long)gy * PW + gx;
    for (int c = 0; c < PC; ++c) {
      const float h = (jin == 3 && jout == 3) ? hm[c][q] : hm[0][q];
      float dv = 0.f;
      if (fk.has) {
        if (delta == nullptr) {
          dv = 1.f;          // heat-map only
        } else {
          const int dc = CD == 1 ? 0 : c;
          dv = delta[((long)fk.k0 * CD + dc) * plane + o];
          if (fk.k1 != fk.k0) dv = fk.a * dv + (1.f - fk.a) * delta[((long)fk.k1 * CD + dc) * plane + o];
        }
      }
      out[((long)f * PC + c) * plane + o] = h * dv;
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K3: second half of the UBlock up-conv (modules/common.py:45-52 after unet.py:187-190).  Because bilinear up-sampling,
// reflection padding and the 3x3 taps are all linear, conv3x3(pad(up(x))) == sum_taps shift_tap(pad(up(W_tap x))): the channel
// mixing is done FIRST at low resolution by one tensor-core GEMM  y[b,i,j, tap*C + co] = sum_c W[co,c,tap] x[b,i,j,c]
// (4x fewer MACs than convolving the up-sampled map, no im2col), and this kernel does the cheap spatial part
//   out[b,oy,ox,co] = act(LN_c( sum_{r,s} bilinear_x2( y[.., (3r+s)*C + co] )(reflect(oy+r-1), reflect(ox+s-1)) ))
// One group of C/8 threads per output pixel (8 channels = one 16-byte load per thread and tap corner).
// VPT = 16-byte channel vectors per thread: C = 8 * VPT * G with G <= 32 threads per pixel (C <= 256: VPT 1; chunkyseal's
// 512-channel first up-conv: VPT 2; the pixel decoder's 192 / 48 / 24: VPT 3); thread lane_g owns the vectors lane_g + G*j.
// F = up-sampling factor (2: U-Net; 2 or 4: pixel decoder, pixel_decoder.py:44-50), ACT = kUpRelu (U-Net) or kUpGelu (pixel decoder).
constexpr int kUpRelu = 0, kUpGelu = 1;

// Source rows of row u (already reflected into [0, 4*IH)) of a bilinear x4 up-sampling with align_corners=False: rows a <= b and
// the weight of a (src = (u + 0.5) / 4 - 0.5 clamped at 0; the weights are multiples of 1/8, exact in fp16).  Factor 2 is written
// out in the kernels themselves, as the U-Net has always had it.
template <int F>
__device__ __forceinline__ void up_src(int u, int IH, int& a, int& b, float& wa) {
  static_assert(F == 4, "factor 2 is inlined in the kernels");
  const int i = u >> 2, p = u & 3;
  if (p < 2) { a = max(i - 1, 0); b = i; wa = (float)(3 - 2 * p) * 0.125f; }
  else       { a = i; b = min(i + 1, IH - 1); wa = (float)(11 - 2 * p) * 0.125f; }
}

template <int ACT>
__device__ __forceinline__ float up_act(float v) {
  if constexpr (ACT == kUpRelu) return fmaxf(v, 0.f);
  else return 0.5f * v * (1.f + erff(v * 0.70710678118654752f));    // nn.GELU (exact erf), pixel_decoder.py:24
}

template <int VPT, int F = 2, int ACT = kUpRelu>
__global__ void __launch_bounds__(256) ups_gather_ln_kernel(const __half* __restrict__ y, int B, int IH, int IW, int C,
                                                            const float* __restrict__ lnw, const float* __restrict__ lnb, float eps,
                                                            __half* __restrict__ out, int ld_out) {
  const int G = C / (8 * VPT);                // threads per pixel (power of two, <= 32)
  const int OH = F * IH, OW = F * IW;
  const long npix = (long)B * OH * OW;
  const int ppb = 256 / G;                    // pixels per block
  const int lane_g = threadIdx.x % G;
  const long ldy = 9L * C;
  for (long pix = (long)blockIdx.x * ppb + threadIdx.x / G; pix < npix; pix += (long)gridDim.x * ppb) {
    const int pix32 = (int)pix;                 // B*OH*OW < 2^31
    const int t = pix32 / OW;
    const int ox = pix32 - t * OW;
    const int b = t / OH, oy = t - b * OH;
    int ya[3], yb[3], xa[3], xb[3];
    float wy[3], wx[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      int u = oy + r - 1;
      if (u < 0) u = -u;
      if (u >= OH) u = 2 * OH - 2 - u;
      if constexpr (F == 2) {
        const int i = u >> 1;
        if (u & 1) { ya[r] = i; yb[r] = min(i + 1, IH - 1); wy[r] = 0.75f; }
        else       { ya[r] = max(i - 1, 0); yb[r] = i; wy[r] = 0.25f; }
      } else {
        up_src<F>(u, IH, ya[r], yb[r], wy[r]);
      }
      int v = ox + r - 1;
      if (v < 0) v = -v;
      if (v >= OW) v = 2 * OW - 2 - v;
      if constexpr (F == 2) {
        const int jx = v >> 1;
        if (v & 1) { xa[r] = jx; xb[r] = min(jx + 1, IW - 1); wx[r] = 0.75f; }
        else       { xa[r] = max(jx - 1, 0); xb[r] = jx; wx[r] = 0.25f; }
      } else {
        up_src<F>(v, IW, xa[r], xb[r], wx[r]);
      }
    }
    float acc[8 * VPT];
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) acc[k] = 0.f;
    const __half* yb_ = y + (long)b * IH * IW * ldy + lane_g * 8;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        // the 4-corner bilinear mix of one tap runs in packed half precision (weights 1/16, 3/16, 9/16 are exact, the
        // operands are fp16 already); the 9 taps accumulate in fp32
        const __half2 w00 = __float2half2_rn(wy[r] * wx[s]), w01 = __float2half2_rn(wy[r] * (1.f - wx[s]));
        const __half2 w10 = __float2half2_rn((1.f - wy[r]) * wx[s]), w11 = __float2half2_rn((1.f - wy[r]) * (1.f - wx[s]));
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
          const __half* base = yb_ + (r * 3 + s) * C + j * G * 8;
          const uint4 v00 = __ldg(reinterpret_cast<const uint4*>(base + ((long)ya[r] * IW + xa[s]) * ldy));
          const uint4 v01 = __ldg(reinterpret_cast<const uint4*>(base + ((long)ya[r] * IW + xb[s]) * ldy));
          const uint4 v10 = __ldg(reinterpret_cast<const uint4*>(base + ((long)yb[r] * IW + xa[s]) * ldy));
          const uint4 v11 = __ldg(reinterpret_cast<const uint4*>(base + ((long)yb[r] * IW + xb[s]) * ldy));
          const __half2* p00 = reinterpret_cast<const __half2*>(&v00);
          const __half2* p01 = reinterpret_cast<const __half2*>(&v01);
          const __half2* p10 = reinterpret_cast<const __half2*>(&v10);
          const __half2* p11 = reinterpret_cast<const __half2*>(&v11);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const __half2 t = __hfma2(w00, p00[k], __hfma2(w01, p01[k], __hfma2(w10, p10[k], __hmul2(w11, p11[k]))));
            const float2 f = __half22float2(t);
            acc[8 * j + 2 * k] += f.x;
            acc[8 * j + 2 * k + 1] += f.y;
          }
        }
      }
    }
    // channels-first LayerNorm over the C channels of this pixel (biased variance) + ReLU
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) sum += acc[k];
    for (int o = G >> 1; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) { const float d = acc[k] - mean; var += d * d; }
    for (int o = G >> 1; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + eps);
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
      __align__(16) __half h[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = (lane_g + j * G) * 8 + k;
        h[k] = __float2half_rn(up_act<ACT>((acc[8 * j + k] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c)));
      }
      *reinterpret_cast<uint4*>(out + pix * ld_out + (lane_g + j * G) * 8) = *reinterpret_cast<const uint4*>(h);
    }
  }
}

// K3 (tiled): the same operation with the low-resolution taps staged in shared memory.  A block owns a 16 x 16 tile of OUTPUT pixels;
// the (8 + 2) x (8 + 2) low-resolution pixels x 9C channels its 36 bilinear corners touch are copied once (16-byte cp.async, rows /
// columns clamped at the image border), then every corner is a 128-bit shared load.  The untiled kernel above re-read each
// low-resolution vector ~16 times through L1/L2 (2.4 GB of L1 traffic for 151 MB of input at 32@128: 203 us against a 34 us bound).
// Factor F: the tile is 16 x 16 output pixels = T x T low-resolution pixels with T = 16 / F, (T + 2)^2 of them staged.
// Requires IH, IW multiples of T.  Dynamic shared memory: (T + 2)^2 * 9C halves (+ the head below).
// HEAD (last pixel-decoder stage, pixel_decoder.py:76-78): the activated C = 8 * VPT channels of each pixel (G = 1) stay in
// registers and the 1x1 conv head (hw fp32 [NO][C], hb [NO], staged in shared memory after the taps) writes the NO fp32 NCHW
// planes `maps` [B][NO][OH][OW] directly: a warp's 32 pixels are two 16-pixel rows, i.e. two full 64-byte segments per plane.
template <int VPT, int F = 2, int ACT = kUpRelu, bool HEAD = false>
__global__ void __launch_bounds__(256) ups_gather_ln_tiled_kernel(const __half* __restrict__ y, int B, int IH, int IW, int C,
                                                                  const float* __restrict__ lnw, const float* __restrict__ lnb, float eps,
                                                                  __half* __restrict__ out, int ld_out, const float* __restrict__ hw = nullptr,
                                                                  const float* __restrict__ hb = nullptr, int NO = 0,
                                                                  float* __restrict__ maps = nullptr) {
  constexpr int T = 16 / F, TS = T + 2, LT = F == 2 ? 3 : 2;   // low-resolution tile, staged tile side, log2(T)
  extern __shared__ __align__(16) uint8_t ugt_smem[];
  __half* tile = reinterpret_cast<__half*>(ugt_smem);       // [TS][TS][9C]
  const int G = C / (8 * VPT);                // threads per pixel (power of two, <= 32)
  const int OH = F * IH, OW = F * IW;
  const int tiles_x = IW >> LT, tiles_y = IH >> LT;
  int t = blockIdx.x;
  const int tx = t % tiles_x; t /= tiles_x;
  const int ty = t % tiles_y;
  const int b = t / tiles_y;
  const int I0 = ty * T, J0 = tx * T;          // low-resolution origin of the tile; the staged region starts at (I0 - 1, J0 - 1)
  const int ldy = 9 * C, cpp = ldy >> 3;       // 16-byte chunks per low-resolution pixel
  const __half* yb_ = y + (long)b * IH * IW * ldy;
  float* hws = reinterpret_cast<float*>(ugt_smem + (size_t)TS * TS * ldy * sizeof(__half));   // HEAD: [NO][C] then [NO]
  if constexpr (HEAD) {
    for (int i = threadIdx.x; i < NO * C; i += 256) hws[i] = __ldg(hw + i);
    for (int i = threadIdx.x; i < NO; i += 256) hws[NO * C + i] = __ldg(hb + i);
  }
  for (int i = threadIdx.x; i < TS * TS * cpp; i += 256) {
    const int px = i / cpp, ch = i - px * cpp;
    const int ly = px / TS, lx = px - ly * TS;
    const int gy = min(max(I0 - 1 + ly, 0), IH - 1), gx = min(max(J0 - 1 + lx, 0), IW - 1);
    cp_async16(tile + (long)px * ldy + ch * 8, yb_ + ((long)gy * IW + gx) * ldy + ch * 8);
  }
  cp_async_commit();
  cp_async_wait_pending(0);
  __syncthreads();
  const int lane_g = threadIdx.x % G;
  const int ppb = 256 / G;
  for (int lp = threadIdx.x / G; lp < 256; lp += ppb) {      // local output pixel of the 16 x 16 tile
    const int loy = lp >> 4, lox = lp & 15;
    const int oy = F * I0 + loy, ox = F * J0 + lox;
    int ya[3], yb[3], xa[3], xb[3];
    float wy[3], wx[3];
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      int u = oy + r - 1;
      if (u < 0) u = -u;
      if (u >= OH) u = 2 * OH - 2 - u;
      if constexpr (F == 2) {
        const int i = u >> 1;
        if (u & 1) { ya[r] = i; yb[r] = min(i + 1, IH - 1); wy[r] = 0.75f; }
        else       { ya[r] = max(i - 1, 0); yb[r] = i; wy[r] = 0.25f; }
      } else {
        up_src<F>(u, IH, ya[r], yb[r], wy[r]);
      }
      ya[r] -= I0 - 1; yb[r] -= I0 - 1;           // tile rows (the clamped copies make the border rows valid)
      int v = ox + r - 1;
      if (v < 0) v = -v;
      if (v >= OW) v = 2 * OW - 2 - v;
      if constexpr (F == 2) {
        const int jx = v >> 1;
        if (v & 1) { xa[r] = jx; xb[r] = min(jx + 1, IW - 1); wx[r] = 0.75f; }
        else       { xa[r] = max(jx - 1, 0); xb[r] = jx; wx[r] = 0.25f; }
      } else {
        up_src<F>(v, IW, xa[r], xb[r], wx[r]);
      }
      xa[r] -= J0 - 1; xb[r] -= J0 - 1;
    }
    float acc[8 * VPT];
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) acc[k] = 0.f;
    const __half* tb = tile + lane_g * 8;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
#pragma unroll
      for (int s2 = 0; s2 < 3; ++s2) {
        const __half2 w00 = __float2half2_rn(wy[r] * wx[s2]), w01 = __float2half2_rn(wy[r] * (1.f - wx[s2]));
        const __half2 w10 = __float2half2_rn((1.f - wy[r]) * wx[s2]), w11 = __float2half2_rn((1.f - wy[r]) * (1.f - wx[s2]));
#pragma unroll
        for (int j = 0; j < VPT; ++j) {
          const __half* base = tb + (r * 3 + s2) * C + j * G * 8;
          const uint4 v00 = *reinterpret_cast<const uint4*>(base + (ya[r] * TS + xa[s2]) * ldy);
          const uint4 v01 = *reinterpret_cast<const uint4*>(base + (ya[r] * TS + xb[s2]) * ldy);
          const uint4 v10 = *reinterpret_cast<const uint4*>(base + (yb[r] * TS + xa[s2]) * ldy);
          const uint4 v11 = *reinterpret_cast<const uint4*>(base + (yb[r] * TS + xb[s2]) * ldy);
          const __half2* p00 = reinterpret_cast<const __half2*>(&v00);
          const __half2* p01 = reinterpret_cast<const __half2*>(&v01);
          const __half2* p10 = reinterpret_cast<const __half2*>(&v10);
          const __half2* p11 = reinterpret_cast<const __half2*>(&v11);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const __half2 tt = __hfma2(w00, p00[k], __hfma2(w01, p01[k], __hfma2(w10, p10[k], __hmul2(w11, p11[k]))));
            const float2 f = __half22float2(tt);
            acc[8 * j + 2 * k] += f.x;
            acc[8 * j + 2 * k + 1] += f.y;
          }
        }
      }
    }
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) sum += acc[k];
    for (int o = G >> 1; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < 8 * VPT; ++k) { const float d = acc[k] - mean; var += d * d; }
    for (int o = G >> 1; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + eps);
    if constexpr (HEAD) {
      constexpr int CH = 8 * VPT;             // G == 1: this thread holds all channels of its pixel
#pragma unroll
      for (int k = 0; k < CH; ++k) acc[k] = up_act<ACT>((acc[k] - mean) * rstd * __ldg(lnw + k) + __ldg(lnb + k));
      const long plane = (long)OH * OW;
      float* dst = maps + (long)b * NO * plane + (long)oy * OW + ox;
      for (int o = 0; o < NO; ++o) {
        const float4* w4 = reinterpret_cast<const float4*>(hws + o * CH);
        float a0 = hws[NO * CH + o], a1 = 0.f;
#pragma unroll
        for (int k = 0; k < CH / 4; ++k) {
          const float4 w = w4[k];
          a0 = fmaf(w.x, acc[4 * k], a0); a1 = fmaf(w.y, acc[4 * k + 1], a1);
          a0 = fmaf(w.z, acc[4 * k + 2], a0); a1 = fmaf(w.w, acc[4 * k + 3], a1);
        }
        __stcs(dst + o * plane, a0 + a1);      // streamed: the maps are not read again by this library
      }
    } else {
    const long pix = ((long)b * OH + oy) * OW + ox;
#pragma unroll
    for (int j = 0; j < VPT; ++j) {
      __align__(16) __half h[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) {
        const int c = (lane_g + j * G) * 8 + k;
        h[k] = __float2half_rn(up_act<ACT>((acc[8 * j + k] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c)));
      }
      *reinterpret_cast<uint4*>(out + pix * ld_out + (lane_g + j * G) * 8) = *reinterpret_cast<const uint4*>(h);
    }
    }
  }
}

// K3b: exact border pixels of the UBlock up-conv for the phase-folded tensor-core path (conv3_direct_host.cuh,
// setup_up_phase_direct): the outermost rows/columns of the 2H x 2W output see the reflect padding of the up-sampled map,
// which breaks the per-phase weight pattern.  One block = 8 border pixels x 16 output channels; the 9 bilinear-sampled
// input vectors of a pixel (64 channels, two sources) are staged in shared memory, then each thread does its 576 MACs in
// fp32 and the 16 threads of a pixel finish with LayerNorm + ReLU.  wk: fp32 [9][16][64] (input scale folded).
constexpr int kUpFixPPB = 16;   // border pixels per block (x 16 output channels = 256 threads)
constexpr size_t kUpFixSmem = (size_t)(9 * 16 * 16 * 4 + kUpFixPPB * 9 * 64) * sizeof(float);
__global__ void __launch_bounds__(256) up_border_fix_kernel(const __half* __restrict__ x0, int C0, const __half* __restrict__ x1, int C1,
                                                            int B, int IH, int IW, const float* __restrict__ wk,
                                                            const float* __restrict__ lnw, const float* __restrict__ lnb, float eps,
                                                            __half* __restrict__ out) {
  constexpr int PPB = kUpFixPPB, CT = 64;
  extern __shared__ __align__(16) float upfix_smem[];
  float* Ws = upfix_smem;                     // [tap][c4][co][4]: conflict-free float4 reads across the 16 co threads
  float* U = upfix_smem + 9 * 16 * 16 * 4;    // [PPB][9][CT]
  const int OH = 2 * IH, OW = 2 * IW;
  const int per_img = 2 * OW + 2 * (OH - 2);
  const int total = B * per_img;              // < 2^31: B * 4 * 2W
  auto decode = [&](int q, int& b, int& oy, int& ox) {
    b = q / per_img;
    int r = q - b * per_img;
    if (r < OW) { oy = 0; ox = r; }
    else if (r < 2 * OW) { oy = OH - 1; ox = r - OW; }
    else { r -= 2 * OW; const int side = r / (OH - 2); oy = 1 + r - side * (OH - 2); ox = side ? OW - 1 : 0; }
  };
  // weights wk [tap][co][c] -> Ws [tap][c4][co][4]
  for (int i = threadIdx.x; i < 9 * 16 * 16; i += 256) {
    const int c4 = i & 15, co = (i >> 4) & 15, tap = i >> 8;
    const float4 w4 = __ldg(reinterpret_cast<const float4*>(wk + ((long)tap * 16 + co) * CT) + c4);
    *reinterpret_cast<float4*>(Ws + (((tap * 16 + c4) * 16 + co) << 2)) = w4;
  }
  // the block keeps its weights and walks over groups of PPB border pixels
  for (int q0 = (int)blockIdx.x * PPB; q0 < total; q0 += (int)gridDim.x * PPB) {
  __syncthreads();   // U of the previous group has been consumed (and Ws is complete on the first pass)
  // (a two-pass variant that issues all 36 loads of a thread first needs 178 registers -> one block per SM; the kernel is bound by the
  //  shared-memory reads of its fp32 MAC loop, not by these loads)
  for (int it = threadIdx.x; it < PPB * 9 * 16; it += 256) {
    const int g4 = it & 15, tap = (it >> 4) % 9, pp = it / 144;
    const int q = q0 + pp;
    float4 val = make_float4(0.f, 0.f, 0.f, 0.f);
    if (q < total) {
      int b, oy, ox;
      decode(q, b, oy, ox);
      const int r = tap / 3, s2 = tap - r * 3;
      int u = oy + r - 1;
      if (u < 0) u = -u;
      if (u >= OH) u = 2 * OH - 2 - u;
      int v = ox + s2 - 1;
      if (v < 0) v = -v;
      if (v >= OW) v = 2 * OW - 2 - v;
      int ya, yb, xa, xb; float wy, wx;
      { const int i = u >> 1; if (u & 1) { ya = i; yb = min(i + 1, IH - 1); wy = 0.75f; } else { ya = max(i - 1, 0); yb = i; wy = 0.25f; } }
      { const int i = v >> 1; if (v & 1) { xa = i; xb = min(i + 1, IW - 1); wx = 0.75f; } else { xa = max(i - 1, 0); xb = i; wx = 0.25f; } }
      const int c = g4 * 4;
      const __half* src = c < C0 ? x0 + c : x1 + (c - C0);
      const int ld = c < C0 ? C0 : C1;
      auto ld4 = [&](int yy, int xx) {
        const uint2 raw = __ldg(reinterpret_cast<const uint2*>(src + (((long)b * IH + yy) * IW + xx) * ld));
        const float2 lo = __half22float2(*reinterpret_cast<const __half2*>(&raw.x)), hi = __half22float2(*reinterpret_cast<const __half2*>(&raw.y));
        return make_float4(lo.x, lo.y, hi.x, hi.y);
      };
      const float4 a = ld4(ya, xa), bq = ld4(ya, xb), cq = ld4(yb, xa), d = ld4(yb, xb);
      const float w00 = wy * wx, w01 = wy * (1.f - wx), w10 = (1.f - wy) * wx, w11 = (1.f - wy) * (1.f - wx);
      val.x = w00 * a.x + w01 * bq.x + w10 * cq.x + w11 * d.x;
      val.y = w00 * a.y + w01 * bq.y + w10 * cq.y + w11 * d.y;
      val.z = w00 * a.z + w01 * bq.z + w10 * cq.z + w11 * d.z;
      val.w = w00 * a.w + w01 * bq.w + w10 * cq.w + w11 * d.w;
    }
    *reinterpret_cast<float4*>(U + ((pp * 9 + tap) * CT + g4 * 4)) = val;
  }
  __syncthreads();
  const int pp = threadIdx.x >> 4, co = threadIdx.x & 15;
  float acc = 0.f;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const float4* up = reinterpret_cast<const float4*>(U + (pp * 9 + tap) * CT);
    const float4* wp = reinterpret_cast<const float4*>(Ws + ((tap * 16 * 16 + co) << 2));
#pragma unroll
    for (int c4 = 0; c4 < CT / 4; ++c4) {
      const float4 u4 = up[c4];
      const float4 w4 = wp[c4 * 16];
      acc += u4.x * w4.x + u4.y * w4.y + u4.z * w4.z + u4.w * w4.w;
    }
  }
  float sum = acc;
#pragma unroll
  for (int o = 8; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  const float mean = sum * (1.f / 16.f);
  const float dv = acc - mean;
  float var = dv * dv;
#pragma unroll
  for (int o = 8; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
  const float rstd = 1.0f / sqrtf(var * (1.f / 16.f) + eps);
  const int q = q0 + pp;
  if (q < total) {
    int b, oy, ox;
    decode(q, b, oy, ox);
    out[(((long)b * OH + oy) * OW + ox) * 16 + co] = __float2half_rn(fmaxf(dv * rstd * __ldg(lnw + co) + __ldg(lnb + co), 0.f));
  }
  }  // pixel groups
}

// K10: uint8 frame I/O around the path (SURVEY 8(f)1, inference_streaming.py:26,31,118): the streaming caller holds RGB24
// frames [F,H,W,3] uint8; moving those over PCIe instead of fp32 planes is 4x less traffic each way.
//   in : x[f,c,y,x] = float(u8[f,y,x,c]) / 255                               (torch: tensor(clip).permute(0,3,1,2) / 255.0)
//   out: u8[f,y,x,c] = (uint8) trunc(imgs_w * 255)  and  imgs_q = float(u8) / 255   ((imgs_w * 255.0).byte(); the detector
//        of the streaming pipeline sees the re-quantised frames)
__global__ void __launch_bounds__(256) u8hwc_to_f32chw_kernel(const uint8_t* __restrict__ src, float* __restrict__ dst, long npix_total,
                                                              long plane) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npix_total; i += (long)gridDim.x * blockDim.x) {
    const long f = i / plane, o = i - f * plane;
    const uint8_t* s = src + i * 3;
    float* d = dst + f * 3 * plane + o;
    d[0] = __fdiv_rn((float)s[0], 255.f);
    d[plane] = __fdiv_rn((float)s[1], 255.f);
    d[2 * plane] = __fdiv_rn((float)s[2], 255.f);
  }
}
__global__ void __launch_bounds__(256) f32chw_to_u8hwc_kernel(const float* __restrict__ src, uint8_t* __restrict__ dst, float* __restrict__ requant,
                                                              long npix_total, long plane) {
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < npix_total; i += (long)gridDim.x * blockDim.x) {
    const long f = i / plane, o = i - f * plane;
    const float* s = src + f * 3 * plane + o;
    uint8_t* d = dst + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float v = __fmul_rn(s[c * plane], 255.f);
      const int q = min(max((int)v, 0), 255);   // .byte(): truncation toward zero; inputs are clamped to [0, 1] by the blend
      d[c] = (uint8_t)q;
      if (requant != nullptr) requant[f * 3 * plane + o + c * plane] = __fdiv_rn((float)q, 255.f);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// K9: ConvNeXt stem: x = 2*img-1 (extractor.py:25); conv k4 stride s (no padding) + bias; channels-first LN eps 1e-6
// (convnext.py:108-111).  imgs [B,3,H,W] fp32 -> out NHWC fp32 [B,OH,OW,C] (row pitch ld).  One warp per output pixel.
__global__ void __launch_bounds__(256) stem_ln_kernel(const float* __restrict__ imgs, int B, int H, int W, int OH, int OW, int stride,
                                                      const float* __restrict__ w /*[48][C] (k = c*16 + r*4 + s)*/, const float* __restrict__ bias,
                                                      const float* __restrict__ lnw, const float* __restrict__ lnb, int C,
                                                      float* __restrict__ out, int ld) {
  extern __shared__ float sm[];  // per warp: 48 inputs + C outputs
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* xin = sm + warp * (48 + C);
  float* yo = xin + 48;
  const long npix = (long)B * OH * OW;
  for (long pix = (long)blockIdx.x * 8 + warp; pix < npix; pix += (long)gridDim.x * 8) {
    const int ox = (int)(pix % OW);
    const long t = pix / OW;
    const int oy = (int)(t % OH), b = (int)(t / OH);
    for (int k = lane; k < 48; k += 32) {
      const int c = k >> 4, r = (k >> 2) & 3, s = k & 3;
      xin[k] = 2.f * __ldg(imgs + ((long)(b * 3 + c) * H + (oy * stride + r)) * W + ox * stride + s) - 1.f;
    }
    __syncwarp();
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) {
      float a = __ldg(bias + c);
#pragma unroll 8
      for (int k = 0; k < 48; ++k) a += xin[k] * __ldg(w + k * C + c);
      yo[c] = a;
      sum += a;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = yo[c] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + 1e-6f);
    for (int c = lane; c < C; c += 32) out[pix * ld + c] = (yo[c] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c);
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------------
// K4: depthwise 7x7 (pad 3, bias) + channels-last LayerNorm (eps 1e-6) -> fp16 [M, ld_out]   (convnext.py:42-45)
// x: NHWC fp32 [B, H, W, C] (pixel pitch ldx).  One block = one strip of kDwStrip output pixels along x; each thread owns
// a channel pair and slides over the 7 x (strip+6) input window; pre-LN results go to smem, then LN per pixel by warps.
constexpr int kDwStrip = 8;
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) { return f2fma(a, b, c); }
// K4 for arbitrary (even) widths, used for the proportional chunkyseal trunk (362 / 724 / 1448 / 2896 channels on 127 / 63 / 31 /
// 15 pixel maps): one block per strip of kDwStrip output pixels; the threads LOOP over the channel pairs (C/2 may exceed the
// block size) and the LayerNorm stage re-reads the pre-LN strip from shared memory instead of holding it in registers.
__global__ void __launch_bounds__(512) dwconv7_ln_wide_kernel(const float* __restrict__ x, int B, int H, int W, int C, int ldx,
                                                              const float* __restrict__ wdw /*[49][C]*/, const float* __restrict__ bdw,
                                                              const float* __restrict__ lnw, const float* __restrict__ lnb,
                                                              __half* __restrict__ out, int ld_out) {
  extern __shared__ float pre[];  // [kDwStrip][C]
  const int strips_x = (W + kDwStrip - 1) / kDwStrip;
  const int C2 = C >> 1;
  const unsigned strip = blockIdx.x;
  const unsigned t = strip / (unsigned)strips_x;
  const int sx = (int)(strip - t * (unsigned)strips_x);
  const int b = (int)(t / (unsigned)H), oy = (int)(t - (unsigned)b * (unsigned)H);
  const int ox0 = sx * kDwStrip;
  for (int cp = threadIdx.x; cp < C2; cp += blockDim.x) {
    const int c = cp * 2;
    float2 acc[kDwStrip];
    const float2 bb = __ldg(reinterpret_cast<const float2*>(bdw + c));
#pragma unroll
    for (int i = 0; i < kDwStrip; ++i) acc[i] = bb;
    for (int r = 0; r < 7; ++r) {
      const int iy = oy + r - 3;
      if (iy < 0 || iy >= H) continue;
      float2 wr[7];
#pragma unroll
      for (int s2 = 0; s2 < 7; ++s2) wr[s2] = __ldg(reinterpret_cast<const float2*>(wdw + (r * 7 + s2) * C + c));
      const float* rowp = x + (((long)b * H + iy) * W) * ldx + c;
#pragma unroll
      for (int u = 0; u < kDwStrip + 6; ++u) {
        const int ix = ox0 + u - 3;
        float2 v = make_float2(0.f, 0.f);
        if (ix >= 0 && ix < W) v = __ldg(reinterpret_cast<const float2*>(rowp + (long)ix * ldx));
#pragma unroll
        for (int s2 = 0; s2 < 7; ++s2) {
          const int i = u - s2;  // output pixel index within the strip
          if (i >= 0 && i < kDwStrip) acc[i] = ffma2(v, wr[s2], acc[i]);
        }
      }
    }
#pragma unroll
    for (int i = 0; i < kDwStrip; ++i) { pre[i * C + c] = acc[i].x; pre[i * C + c + 1] = acc[i].y; }
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int i = warp; i < kDwStrip; i += nwarps) {   // one warp per output pixel of the strip
    const int ox = ox0 + i;
    if (ox >= W) continue;
    const float* pr = pre + (size_t)i * C;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += pr[c];
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = pr[c] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + 1e-6f);
    __half* dst = out + (((long)b * H + oy) * W + ox) * ld_out;
    for (int c2 = lane; c2 < C2; c2 += 32) {
      const float2 g = __ldg(reinterpret_cast<const float2*>(lnw) + c2), bt = __ldg(reinterpret_cast<const float2*>(lnb) + c2);
      const float a = (pr[2 * c2] - mean) * rstd * g.x + bt.x;
      const float bq = (pr[2 * c2 + 1] - mean) * rstd * g.y + bt.y;
      *reinterpret_cast<__half2*>(dst + 2 * c2) = __floats2half2_rn(a, bq);
    }
  }
}

// K4, fixed-width variant used for the ConvNeXt trunk widths (96/192/384/768).  Same mapping as above, but written around
// the instruction count: the generic kernel spends most of its instructions on 64-bit address arithmetic, bounds tests and
// the divergence bookkeeping of branchy conditional loads.  Here C is a template
// constant, so every input and weight load is `base + immediate`; rows advance by one pointer add; interior strips take a
// path with no predicates at all and edge strips use a single predicated load per tap column (inline PTX, no branches).
template <int OFF>
__device__ __forceinline__ float2 ldg_f2_pred(const float* p, unsigned pred) {
  float2 v;
  asm("{\n\t.reg .pred q;\n\tsetp.ne.u32 q, %3, 0;\n\tmov.f32 %0, 0f00000000;\n\tmov.f32 %1, 0f00000000;\n\t"
      "@q ld.global.nc.v2.f32 {%0, %1}, [%2+%4];\n\t}"
      : "=f"(v.x), "=f"(v.y)
      : "l"(p), "r"(pred), "n"(OFF));
  return v;
}
// MODE 0: interior strip (no predicates), 1: edge strip (predicated loads), 2: the strip is the whole row (W == STRIP): the
// out-of-image columns are dropped at compile time
template <int C, int STRIP, int U, int MODE>
struct DwCol {
  static __device__ __forceinline__ void run(const float* prow, unsigned cmask, const float2 (&wr)[7], float2 (&acc)[STRIP]) {
    if (MODE != 2 || (U >= 3 && U < STRIP + 3)) {
    float2 v;
    if (MODE == 1) v = ldg_f2_pred<U * C * 4>(prow, cmask & (1u << U));
    else v = __ldg(reinterpret_cast<const float2*>(prow + U * C));
#pragma unroll
    for (int s2 = 0; s2 < 7; ++s2) {
      const int i = U - s2;  // output pixel index within the strip
      if (i >= 0 && i < STRIP) acc[i] = ffma2(v, wr[s2], acc[i]);
    }
    }
    DwCol<C, STRIP, U + 1, MODE>::run(prow, cmask, wr, acc);
  }
};
template <int C, int STRIP, int MODE>
struct DwCol<C, STRIP, STRIP + 6, MODE> {
  static __device__ __forceinline__ void run(const float*, unsigned, const float2 (&)[7], float2 (&)[STRIP]) {}
};

template <int C, int STRIP, bool FULLROW>
__global__ void __launch_bounds__(768) dwconv7_ln_c_kernel(const float* __restrict__ x, int B, int H, int W,
                                                           const float* __restrict__ wdw /*[49][C]*/, const float* __restrict__ bdw,
                                                           const float* __restrict__ lnw, const float* __restrict__ lnb,
                                                           __half* __restrict__ out, int ld_out, int spb, int ngroups) {
  constexpr int C2 = C / 2, KP = (C + 63) / 64;
  extern __shared__ float pre[];  // [spb][STRIP][C]
  const int strips_x = (W + STRIP - 1) / STRIP;
  const int ls = threadIdx.x / C2;                 // local strip
  const int cp = threadIdx.x - ls * C2;            // channel pair
  // A block owns `spb` strips of one output row each (group = (b*H + oy) * strips_x + strip column)
  const unsigned group = blockIdx.x * (unsigned)spb + (unsigned)ls;
  const unsigned tg = group / (unsigned)strips_x;
  const int sx = (int)(group - tg * (unsigned)strips_x);
  const int b = (int)(tg / (unsigned)H), oy = (int)(tg - (unsigned)b * (unsigned)H);
  if (ls < spb && group < (unsigned)ngroups) {
    const int ox0 = sx * STRIP;
    const int c = cp * 2;
    float2 acc[STRIP];
    const float2 bb = __ldg(reinterpret_cast<const float2*>(bdw + c));
#pragma unroll
    for (int i = 0; i < STRIP; ++i) acc[i] = bb;
    unsigned cmask = 0;
#pragma unroll
    for (int u = 0; u < STRIP + 6; ++u) cmask |= ((unsigned)(ox0 + u - 3) < (unsigned)W) ? (1u << u) : 0u;
    const bool interior = cmask == (1u << (STRIP + 6)) - 1u;
    const long rowpitch = (long)W * C;
    // (oy - 3, ox0 - 3): may lie outside the image; only dereferenced where the masks allow
    const float* prow = x + (((long)b * H + oy) * W + ox0) * C + c - 3 * rowpitch - 3 * C;
    const float* wrow = wdw + c;
#pragma unroll 1
    for (int r = 0; r < 7; ++r, prow += rowpitch, wrow += 7 * C) {
      if ((unsigned)(oy + r - 3) >= (unsigned)H) continue;
      float2 wr[7];
#pragma unroll
      for (int s2 = 0; s2 < 7; ++s2) wr[s2] = __ldg(reinterpret_cast<const float2*>(wrow + s2 * C));
      if (FULLROW) DwCol<C, STRIP, 0, 2>::run(prow, cmask, wr, acc);
      else if (interior) DwCol<C, STRIP, 0, 0>::run(prow, cmask, wr, acc);
      else DwCol<C, STRIP, 0, 1>::run(prow, cmask, wr, acc);
    }
    float* pr = pre + (size_t)ls * STRIP * C;
#pragma unroll
    for (int i = 0; i < STRIP; ++i) *reinterpret_cast<float2*>(pr + i * C + c) = acc[i];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
  for (int item = warp; item < spb * STRIP; item += nwarps) {
    const int l2 = item / STRIP, i = item - l2 * STRIP;
    const unsigned st2 = blockIdx.x * (unsigned)spb + (unsigned)l2;
    if (st2 >= (unsigned)ngroups) continue;
    const unsigned t2 = st2 / (unsigned)strips_x;   // b*H + oy
    const int sx2 = (int)(st2 - t2 * (unsigned)strips_x);
    const int ox = sx2 * STRIP + i;
    if (ox >= W) continue;
    const float2* pr2 = reinterpret_cast<const float2*>(pre + ((size_t)l2 * STRIP + i) * C);
    float2 vv[KP];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int c2 = lane + 32 * k;
      vv[k] = c2 < C2 ? pr2[c2] : make_float2(0.f, 0.f);
      sum += vv[k].x + vv[k].y;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum * (1.0f / (float)C);
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      if (lane + 32 * k < C2) { const float dx = vv[k].x - mean, dy = vv[k].y - mean; var += dx * dx + dy * dy; }
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + 1e-6f);
    __half* dst = out + ((long)t2 * W + ox) * ld_out;   // t2 = b*H + oy
#pragma unroll
    for (int k = 0; k < KP; ++k) {
      const int c2 = lane + 32 * k;
      if (c2 < C2) {
        const float2 g = __ldg(reinterpret_cast<const float2*>(lnw) + c2), bt = __ldg(reinterpret_cast<const float2*>(lnb) + c2);
        const float a = (vv[k].x - mean) * rstd * g.x + bt.x;
        const float bq = (vv[k].y - mean) * rstd * g.y + bt.y;
        *reinterpret_cast<__half2*>(dst + 2 * c2) = __floats2half2_rn(a, bq);
      }
    }
  }
}


// K4b: per-row LayerNorm over C (biased variance, eps) of fp32 rows -> fp16 rows.  One warp per row.
__global__ void __launch_bounds__(256) ln_rows_kernel(const float* __restrict__ x, long M, int C, int ldx, const float* __restrict__ w,
                                                      const float* __restrict__ bvec, float eps, __half* __restrict__ out, int ld_out) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (long m = (long)blockIdx.x * 8 + warp; m < M; m += (long)gridDim.x * 8) {
    const float* r = x + m * ldx;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += r[c];
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = r[c] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + eps);
    for (int c = lane; c < C; c += 32) out[m * ld_out + c] = __float2half_rn((r[c] - mean) * rstd * __ldg(w + c) + __ldg(bvec + c));
  }
}

// K2d: GRN (common.py:166-169) applied in place on the fp16 pwconv1 output, fused with the statistics -> multiplier step:
//   Gx = sqrt(stats[b,k]);  Nx = Gx / (mean_k Gx + 1e-6);  g[m,k] *= gamma[k] * Nx + 1     (beta is folded into pwconv2's bias)
// One block per (sample, row-slab); the per-sample mean is recomputed by every block (K <= 3072 values).  `stats_next` (the
// ping-pong buffer the NEXT block's pwconv1 accumulates into) is cleared here.  At batch 64 x 256^2 g is 201 / 100 / 50 / 25 MB in
// the four stages, so on the H100's 50 MB L2 only the last stage's pass runs out of L2 and the others stream g from HBM (one
// read + one write of g, against the pwconv2 GEMM that reads it again); pwconv2 is then a plain TMA-fed GEMM.
// part_rows > 0: `stats` holds part_rows partial rows per sample ([B * part_rows][K], written by the pwconv1 epilogue warps without
// atomics).  They are added here in a FIXED order (so the result does not depend on the order in which the tiles finished): 128-bit
// loads, 8 rows in flight per thread, and two row groups per column when the block has the threads for it (combined lower rows first).
// Fills sc[k] = sqrt(sum_rows) for all k; tmp is K floats of scratch.  Ends with a block barrier.
__device__ __forceinline__ void grn_colnorms(const float* __restrict__ stats, int b, int K, int part_rows, float* sc, float* tmp) {
  if (part_rows <= 0) {
    for (int k = threadIdx.x; k < K; k += blockDim.x) sc[k] = sqrtf(stats[(long)b * K + k]);
    __syncthreads();
    return;
  }
  const int K4 = K >> 2;
  const float4* base = reinterpret_cast<const float4*>(stats + (long)b * part_rows * K);
  const bool two = (int)blockDim.x >= 2 * K4 && (part_rows & 1) == 0;
  auto sum_rows = [&](int c4, int r0, int r1) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
    int r = r0;
    for (; r + 8 <= r1; r += 8) {
      float4 v[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) v[u] = base[(long)(r + u) * K4 + c4];
#pragma unroll
      for (int u = 0; u < 8; ++u) { a.x += v[u].x; a.y += v[u].y; a.z += v[u].z; a.w += v[u].w; }
    }
    for (; r < r1; ++r) { const float4 v = base[(long)r * K4 + c4]; a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w; }
    return a;
  };
  if (two) {
    const int rg = threadIdx.x / K4, c4 = threadIdx.x - rg * K4, half = part_rows >> 1;
    if (rg < 2) {
      const float4 a = sum_rows(c4, rg * half, (rg + 1) * half);
      *reinterpret_cast<float4*>((rg ? tmp : sc) + 4 * c4) = a;
    }
    __syncthreads();
    for (int k = threadIdx.x; k < K; k += blockDim.x) sc[k] = sqrtf(sc[k] + tmp[k]);
  } else {
    for (int c4 = threadIdx.x; c4 < K4; c4 += blockDim.x) {
      float4 a = sum_rows(c4, 0, part_rows);
      *reinterpret_cast<float4*>(sc + 4 * c4) = make_float4(sqrtf(a.x), sqrtf(a.y), sqrtf(a.z), sqrtf(a.w));
    }
  }
  __syncthreads();
}
__global__ void __launch_bounds__(256) grn_apply_kernel(__half* __restrict__ g, int rows_per_sample, int K, int ld,
                                                        const float* __restrict__ stats, float* __restrict__ stats_next,
                                                        const float* __restrict__ gamma, int slabs, int part_rows) {
  extern __shared__ __align__(16) float sc[];   // [K] multipliers of this sample | [K] scratch
  __shared__ float red[8];
  __shared__ float mean_s;
  const int b = blockIdx.x / slabs, slab = blockIdx.x - b * slabs;
  grn_colnorms(stats, b, K, part_rows, sc, sc + K);
  float sum = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sum += sc[k];
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    mean_s = t / (float)K;
  }
  __syncthreads();
  const float inv = 1.0f / (mean_s + 1e-6f);
  for (int k = threadIdx.x; k < K; k += blockDim.x) sc[k] = __ldg(gamma + k) * (sc[k] * inv) + 1.0f;
  if (slab == 0 && stats_next != nullptr) for (int k = threadIdx.x; k < K; k += blockDim.x) stats_next[(long)b * K + k] = 0.f;
  __syncthreads();
  const int k8 = K >> 3;
  const int r0 = (int)(((long)rows_per_sample * slab) / slabs), r1 = (int)(((long)rows_per_sample * (slab + 1)) / slabs);
  __half* base = g + ((long)b * rows_per_sample + r0) * ld;
  // thread -> (row m, 16-byte column chunk kc), advanced incrementally (no division in the loop)
  const int dm = (int)blockDim.x / k8, dk = (int)blockDim.x - dm * k8;
  int m = (int)threadIdx.x / k8, kc = (int)threadIdx.x - m * k8;
  const int nrows = r1 - r0;
  while (m < nrows) {
    const int k = kc * 8;
    uint4* ptr = reinterpret_cast<uint4*>(base + (long)m * ld + k);
    uint4 v = *ptr;
    __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float2 f = __half22float2(h[q]);
      f.x *= sc[k + 2 * q]; f.y *= sc[k + 2 * q + 1];
      h[q] = __float22half2_rn(f);
    }
    *ptr = v;
    m += dm; kc += dk;
    if (kc >= k8) { kc -= k8; ++m; }
  }
}

// K2e: GRN folded into the NEXT GEMM's weights instead of the activations (stages where C_out << rows per sample):
//   pwconv2(g * s[b,:]) = (W2 * diag(s[b,:])) g,   s[b,k] = gamma[k] * Gx[b,k] / (mean_k Gx[b,:] + 1e-6) + 1
// so each sample gets its own fp16 copy of W2 [N][K] (64 x 72 KB at stage 0) and the 200 MB activation tensor is neither
// re-read nor re-written.  grid (samples, splits); `stats_next` is cleared like grn_apply_kernel does.
__global__ void __launch_bounds__(256) grn_scale_weights_kernel(const float* __restrict__ stats, float* __restrict__ stats_next,
                                                                const float* __restrict__ gamma, const __half* __restrict__ w,
                                                                __half* __restrict__ out, int N, int K, int part_rows) {
  extern __shared__ __align__(16) float sc[];   // [K] | [K] scratch
  __shared__ float red[8];
  __shared__ float mean_s;
  const int b = blockIdx.x;
  grn_colnorms(stats, b, K, part_rows, sc, sc + K);
  float sum = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) sum += sc[k];
#pragma unroll
  for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = sum;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) t += red[i];
    mean_s = t / (float)K;
  }
  __syncthreads();
  const float inv = 1.0f / (mean_s + 1e-6f);
  for (int k = threadIdx.x; k < K; k += blockDim.x) sc[k] = __ldg(gamma + k) * (sc[k] * inv) + 1.0f;
  if (blockIdx.y == 0 && stats_next != nullptr) for (int k = threadIdx.x; k < K; k += blockDim.x) stats_next[(long)b * K + k] = 0.f;
  __syncthreads();
  const int k8 = K >> 3;
  const int n0 = (int)(((long)N * blockIdx.y) / gridDim.y), n1 = (int)(((long)N * (blockIdx.y + 1)) / gridDim.y);
  const int dm = (int)blockDim.x / k8, dk = (int)blockDim.x - dm * k8;
  int n = n0 + (int)threadIdx.x / k8, kc = (int)threadIdx.x % k8;
  while (n < n1) {
    const int k = kc * 8;
    uint4 v = __ldg(reinterpret_cast<const uint4*>(w + (long)n * K + k));
    __half2* h = reinterpret_cast<__half2*>(&v);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float2 f = __half22float2(h[q]);
      f.x *= sc[k + 2 * q]; f.y *= sc[k + 2 * q + 1];
      h[q] = __float22half2_rn(f);
    }
    *reinterpret_cast<uint4*>(out + ((long)b * N + n) * K + k) = v;
    n += dm; kc += dk;
    if (kc >= k8) { kc -= k8; ++n; }
  }
}

// K9a: stem im2col: x = 2*img-1 (extractor.py:25) patches of the k4 conv (stride s, no padding) -> fp16 [M, 64] rows
// (k = c*16 + r*4 + t for k < 48, zero for 48..63) for the tensor-core stem GEMM.  One thread per (pixel, channel c).
__global__ void __launch_bounds__(256) stem_im2col_kernel(const float* __restrict__ imgs, int B, int H, int W, int OH, int OW, int stride,
                                                          __half* __restrict__ out) {
  const long total = (long)B * OH * OW * 4;
  for (long i = (long)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c = (int)(i & 3);
    const long pix = i >> 2;
    __align__(16) __half h[16];
    if (c < 3) {
      const int ox = (int)(pix % OW);
      const long t = pix / OW;
      const int oy = (int)(t % OH), b = (int)(t / OH);
      const float* src = imgs + ((long)(b * 3 + c) * H + oy * stride) * W + ox * stride;
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int q = 0; q < 4; ++q) h[r * 4 + q] = __float2half_rn(2.f * __ldg(src + (long)r * W + q) - 1.f);
    } else {
#pragma unroll
      for (int q = 0; q < 16; ++q) h[q] = __float2half_rn(0.f);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + pix * 64 + c * 16);
    dst[0] = reinterpret_cast<const uint4*>(h)[0];
    dst[1] = reinterpret_cast<const uint4*>(h)[1];
  }
}

// K8a: per sample: channels-first LN (eps 1e-6) over C for each of the P pixels, GELU, mean over pixels -> pooled [B, C]
// (pixel_decoder.py:44-55,77 with common.py:50-51).  y: [B*P, ld] fp32.  One block per sample, one warp per pixel (loop).
__global__ void __launch_bounds__(256) head_pool_kernel(const float* __restrict__ y, int P, int C, int ld, const float* __restrict__ lnw,
                                                        const float* __restrict__ lnb, float* __restrict__ pooled) {
  // acc [nw][C]: every warp adds its own pixels in a fixed order into its own row, the rows are added in warp order at the end:
  // no atomics, bit-reproducible logits
  extern __shared__ float acc_all[];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
  float* acc = acc_all + warp * C;
  for (int c = lane; c < C; c += 32) acc[c] = 0.f;
  __syncwarp();
  for (int pix = warp; pix < P; pix += nw) {
    const float* r = y + ((long)b * P + pix) * ld;
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += r[c];
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float mean = sum / (float)C;
    float var = 0.f;
    for (int c = lane; c < C; c += 32) { const float d = r[c] - mean; var += d * d; }
#pragma unroll
    for (int o = 16; o; o >>= 1) var += __shfl_xor_sync(0xffffffffu, var, o);
    const float rstd = 1.0f / sqrtf(var / (float)C + 1e-6f);
    for (int c = lane; c < C; c += 32) {
      const float v = (r[c] - mean) * rstd * __ldg(lnw + c) + __ldg(lnb + c);
      acc[c] += 0.5f * v * (1.0f + erff(v * 0.70710678118654752f));     // lane-private element of this warp's row
    }
  }
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float t = 0.f;
    for (int w = 0; w < nw; ++w) t += acc_all[w * C + c];
    pooled[(long)b * C + c] = t / (float)P;
  }
}

// K8b: logits[b, o] = bias[o] + sum_c pooled[b, c] * w[o, c]     (pixel_decoder.py:78).  One warp per output.
__global__ void __launch_bounds__(256) head_linear_kernel(const float* __restrict__ pooled, const float* __restrict__ w,
                                                          const float* __restrict__ bias, int B, int C, int NO, float* __restrict__ logits) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long total = (long)B * NO;
  for (long idx = (long)blockIdx.x * 8 + warp; idx < total; idx += (long)gridDim.x * 8) {
    const int o = (int)(idx % NO);
    const long b = idx / NO;
    float a = 0.f;
    for (int c = lane; c < C; c += 32) a += pooled[b * C + c] * __ldg(w + (long)o * C + c);
#pragma unroll
    for (int q = 16; q; q >>= 1) a += __shfl_xor_sync(0xffffffffu, a, q);
    if (lane == 0) logits[idx] = a + __ldg(bias + o);
  }
}

}  // namespace vsb
