// HBM-bound full-resolution stage of the path (round 2):
//   K5  resize_sep_kernel    F.interpolate(size, **interpolation) as a SEPARABLE resample (any table of resize_blend_host.cuh:
//                            bilinear / bicubic with or without antialias and align_corners, nearest, area): groups of input
//                            rows arrive in shared memory as single bulk copies on an mbarrier ring, the horizontal pass runs out of
//                            shared memory with the thread's taps in registers, the vertical pass out of a second shared buffer.  One
//                            launch handles key frames that are `frame_stride` apart (video mode).  Replaces the scalar per-output-pixel
//                            gather of round 1 (49 global loads per output at 768 -> 256).
//                            (models/wam.py:161-164,222-226; videoseal.py:303-310)
//   K7  jnd_blend3_kernel    JND heat-map x up-resampled delta, additive blend, clamp (modules/jnd.py:63-108, wam.py:183-201,
//                            blender.py:61-68, videoseal.py:80-118), TMA-fed: one box per 128 x 16 tile brings the RGB tile with its
//                            2-pixel halo (out-of-image = zero fill = the conv padding), a second one the delta tile; double buffer
//                            over 4 tiles per block; separable 5x5 / Sobel sums and jnd_value in packed fp32, SFU transcendentals.
//       jnd_blend2_kernel    the same arithmetic with per-thread loads: widths that are not multiples of 4, unaligned tensors,
//                            delta down-scale, frames smaller than a TMA box.
//       Both up-scale the delta through <= 2 taps per axis (FASTUP 1) or, for bicubic tables, 3-4 taps (FASTUP 4).
#pragma once
#include "conv_gemm.cuh"
#include "pointwise.cuh"

namespace vsb {

// ------------------------------------------------------------------------------------------------ K5
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(gsrc) : "memory");
}
// in: planes [n][3][IH][IW] with frames `frame_stride` floats apart; out: [n*3][OH][OW] contiguous.
// grid (ceil(OH / toy), n*3); block 256.  Shared: hbuf [rin_max][OW] | stage [kRsStages][GST * IW + 8] (ring of staging rounds: the rows of
// round r+1 are in flight while the horizontal pass of round r runs; consecutive input rows of a plane are contiguous in memory,
// so a round is ONE flat asynchronous copy of GST * IW floats, 16 bytes per request when IW % 4 == 0).
// The tap loops carry no predicates: taps beyond an output's support have weight 0 and read whatever FINITE value follows in the
// staging buffer (the buffers are zero-filled once, an 8-float zero pad ends each of them) -- ncu of the first version showed
// 33 % of its instructions were predicate bookkeeping (LOP3 / ISETP / P2R) and 17 % address IMADs against 8 % FFMA.
constexpr int kRsStages = 3;
template <int MAXT, int GST>   // MAXT: x taps per output held in registers (2 or 8); 0 = any count (weights from the table, predicated)
__global__ void __launch_bounds__(256) resize_sep_kernel(const float* __restrict__ in, long frame_stride, float* __restrict__ out, int IH,
                                                         int IW, int OH, int OW, ResampleTab t, int toy, int rin_max, int vec) {
  extern __shared__ __align__(16) float rs_smem[];
  float* hbuf = rs_smem;
  const int stg_stride = (GST * IW + 8 + 3) & ~3;
  float* stg = rs_smem + (((size_t)rin_max * OW + 3) & ~(size_t)3);
  const int pl = blockIdx.y;
  const int n = pl / 3, c = pl - n * 3;
  const float* src = in + (long)n * frame_stride + (long)c * IH * IW;
  const int oy0 = blockIdx.x * toy, oy1 = min(OH, oy0 + toy);
  const int r0 = __ldg(t.ystart + oy0);
  const int nr = __ldg(t.ystart + oy1 - 1) + __ldg(t.ycnt + oy1 - 1) - r0;   // <= rin_max (host-computed from the same table)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rounds = (nr + GST - 1) / GST;
  for (int i = threadIdx.x * 4; i < kRsStages * stg_stride; i += 1024) *reinterpret_cast<float4*>(stg + i) = make_float4(0.f, 0.f, 0.f, 0.f);
  if (vec) fence_proxy_async_smem();     // every writer orders its zero fill before the bulk copies (async proxy) into the same buffers
  __shared__ uint64_t rs_full[kRsStages];
  if (vec && threadIdx.x == 0) {
    for (int i = 0; i < kRsStages; ++i) mbar_init(&rs_full[i], 1);
    fence_barrier_init();
  }
  __syncthreads();
  // vec (IW % 4 == 0, 16-byte aligned planes): a round is ONE bulk copy issued by thread 0 instead of a cp.async loop in every thread,
  // kRsStages - 1 rounds in flight.
  // otherwise: 4-byte cp.async by every thread, one round in flight.
  const int depth = vec ? kRsStages - 1 : 1;
  auto issue = [&](int rd) {
    if (vec) {
      if (rd < rounds && threadIdx.x == 0) {
        const int g0 = rd * GST;
        const uint32_t bytes = (uint32_t)(min(GST, nr - g0) * IW) * 4u;
        const int b = rd % kRsStages;
        fence_proxy_async_smem();            // the buffer was zero-filled / read through the generic proxy
        mbar_arrive_expect_tx(&rs_full[b], bytes);
        bulk_load_1d(stg + b * stg_stride, src + (long)(r0 + g0) * IW, bytes, &rs_full[b]);
      }
    } else {
      if (rd < rounds) {
        const int g0 = rd * GST, nfl = min(GST, nr - g0) * IW;
        const float* sp = src + (long)(r0 + g0) * IW;
        float* d = stg + (rd & 1) * stg_stride;
        for (int i = threadIdx.x; i < nfl; i += 256) cp_async4(d + i, sp + i);
      }
      cp_async_commit();
    }
  };
  // OW <= 256 (every card: processing size 256): a thread owns ONE output column for the whole block, so its taps are loaded once
  // instead of every round, and the row / column predicates and addresses are computed once
  const bool single = MAXT > 0 && OW <= 256;
  const bool act = (int)threadIdx.x < OW;
  int xs1 = 0;
  float w1[MAXT > 0 ? MAXT : 1];
  if (single && act) {
    const int xc = __ldg(t.xcnt + threadIdx.x);
    xs1 = __ldg(t.xstart + threadIdx.x);
#pragma unroll
    for (int i = 0; i < MAXT; ++i) w1[i] = i < xc ? __ldg(t.xw + threadIdx.x * t.maxt_x + i) : 0.f;
  }
  for (int rd = 0; rd < depth; ++rd) issue(rd);
  for (int rd = 0; rd < rounds; ++rd) {
    issue(rd + depth);                 // its buffer was released by the barrier that ended round rd - 1
    if (vec) {
      mbar_wait(&rs_full[rd % kRsStages], (rd / kRsStages) & 1);
    } else {
      cp_async_wait_pending(1);        // round rd has landed (this thread's part); the barrier makes it everybody's
      __syncthreads();
    }
    const int g0 = rd * GST, ng = min(GST, nr - g0);
    const float* sb = stg + (vec ? rd % kRsStages : (rd & 1)) * stg_stride;
    if (single) {
      if (act) {
        const float* s = sb + xs1;
        float* hb = hbuf + g0 * OW + threadIdx.x;
        if (ng == GST) {
#pragma unroll
          for (int r = 0; r < GST; ++r) {
            float acc = w1[0] * s[0];
#pragma unroll
            for (int i = 1; i < MAXT; ++i) acc = fmaf(w1[i], s[i], acc);
            hb[r * OW] = acc;
            s += IW;
          }
        } else {
          for (int r = 0; r < ng; ++r) {
            float acc = w1[0] * s[0];
#pragma unroll
            for (int i = 1; i < MAXT; ++i) acc = fmaf(w1[i], s[i], acc);
            hb[r * OW] = acc;
            s += IW;
          }
        }
      }
    } else {
      for (int ox = threadIdx.x; ox < OW; ox += 256) {
        const int xs = __ldg(t.xstart + ox), xc = __ldg(t.xcnt + ox);
        const float* wp = t.xw + (long)ox * t.maxt_x;
        float* hb = hbuf + g0 * OW + ox;
        if (MAXT > 0) {
          float w[MAXT > 0 ? MAXT : 1];
#pragma unroll
          for (int i = 0; i < MAXT; ++i) w[i] = i < xc ? __ldg(wp + i) : 0.f;
          const float* s = sb + xs;
#pragma unroll
          for (int r = 0; r < GST; ++r) {
            if (r < ng) {
              float acc = w[0] * s[0];
#pragma unroll
              for (int i = 1; i < MAXT; ++i) acc = fmaf(w[i], s[i], acc);
              hb[r * OW] = acc;
            }
            s += IW;
          }
        } else {
          for (int r = 0; r < ng; ++r) {
            const float* s = sb + r * IW + xs;
            float acc = __ldg(wp) * s[0];
            for (int i = 1; i < xc; ++i) acc = fmaf(__ldg(wp + i), s[i], acc);
            hb[r * OW] = acc;
          }
        }
      }
    }
    __syncthreads();                   // this round's buffer may be refilled; hbuf complete after the last round
  }
  float* dst = out + (long)pl * OH * OW;
  const bool ow_full = (OW & 255) == 0;                    // no column predicates in the vertical pass
  for (int oy = oy0 + warp; oy < oy1; oy += 8) {          // one warp per output row: the y taps are warp-uniform
    const int ys = __ldg(t.ystart + oy) - r0, yc = __ldg(t.ycnt + oy);
    const float* wy = t.yw + oy * t.maxt_y;
    for (int oxb = 0; oxb < OW; oxb += 256) {              // 8 outputs per lane: accumulators in registers, one weight load per tap
      const float* h = hbuf + ys * OW + oxb + lane;
      float acc[8];
      const float w0 = __ldg(wy);
      if (ow_full) {
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = w0 * h[32 * k];
        for (int j = 1; j < yc; ++j) {
          const float wj = __ldg(wy + j);
          const float* hj = h + j * OW;
#pragma unroll
          for (int k = 0; k < 8; ++k) acc[k] = fmaf(wj, hj[32 * k], acc[k]);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) dst[oy * OW + oxb + lane + 32 * k] = acc[k];
      } else {
#pragma unroll
        for (int k = 0; k < 8; ++k) acc[k] = (oxb + lane + 32 * k < OW) ? w0 * h[32 * k] : 0.f;
        for (int j = 1; j < yc; ++j) {
          const float wj = __ldg(wy + j);
          const float* hj = h + j * OW;
#pragma unroll
          for (int k = 0; k < 8; ++k) if (oxb + lane + 32 * k < OW) acc[k] = fmaf(wj, hj[32 * k], acc[k]);
        }
#pragma unroll
        for (int k = 0; k < 8; ++k) if (oxb + lane + 32 * k < OW) dst[oy * OW + oxb + lane + 32 * k] = acc[k];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ K7
constexpr int kB2TW = 128, kB2TH = 16, kB2LP = 136;   // tile, and the pitch of the luminance tile (image column x0 + j at index 4 + j)
constexpr int kB2DH = kB2TH + 2, kB2DW = kB2TW + 4;   // delta tile at processing resolution (up-scale: at most 1 source pixel per output pixel + 1)
// 4-tap up-scale (bicubic): taps floor - 1 .. floor + 2 reach one source row further on each side; the rows / columns read are at most
// tile + 3 (the host checks every table against these sizes: ResampleDev::blend_rows / blend_cols)
constexpr int kB2DH4 = kB2TH + 4;
constexpr size_t b2_smem(int jin, int fastup = 1) {
  return (size_t)(jin * (kB2TH + 4) * kB2LP + 3 * kB2TH * kB2TW + (fastup == 4 ? kB2DH4 : kB2DH) * kB2DW) * sizeof(float);
}

__device__ __forceinline__ float lg2_approx(float x) { float y; asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float ex2_approx_f(float x) { float y; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float sqrt_approx(float x) { float y; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
__device__ __forceinline__ float rcp_approx_f(float x) { float y; asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x)); return y; }
// L = 255 * Y with the factor folded into the weights (1 FMUL + 2 FFMA per pixel instead of 6 operations; differs from the
// reference's (255 x) . w by one rounding, 1e-7 relative)
__device__ __forceinline__ float lum255(float r, float g, float b) {
  return fmaf(0.114f * 255.f, b, fmaf(0.587f * 255.f, g, (0.299f * 255.f) * r));
}
// modules/jnd.py:63-108 on L = 255*Y: la = conv5x5(L)/32 -> piecewise; cm = .117 * 16 g^2.4 / (g^2 + 26^2), g = |Sobel|;
// hmap = max(la + cm - .3 min(la, cm), 0) / 255.  la_sum = the 5x5 weighted sum (weights 1 / 2 / 0, jnd.py:37-43).
// Transcendentals on the SFU (sqrt / lg2 / ex2 / rcp .approx, each <= 2 ulp-ish): 4 MUFU + ~16 FP32 instructions per pixel.
__device__ __forceinline__ float jnd_value(float la_sum, float gx, float gy) {
  const float la0 = la_sum * (1.f / 32.f);
  const float lo = fmaf(-17.f, sqrt_approx(fmaf(la0, 1.f / 127.f, 1e-5f)), 17.f);
  const float hi = fmaf(3.f / 128.f, la0 - 127.f, 3.f);
  const float la = (la0 <= 127.f) ? lo : hi;
  const float g2 = fmaf(gx, gx, gy * gy);
  const float pw = ex2_approx_f(1.2f * lg2_approx(g2));    // g^2.4 = (g^2)^1.2;  g2 == 0 -> lg2 = -inf -> 0
  const float cm = (0.117f * 16.f) * pw * rcp_approx_f(g2 + 676.f);
  return fmaxf(la + cm - 0.3f * fminf(la, cm), 0.f) * (1.f / 255.f);
}

// Heat-map of a thread's 2 rows x 4 consecutive pixels from a luminance tile with halo (pitch kB2LP; pixel (row yl, column j) of
// the tile sits at [(yl + 2) * kB2LP + 4 + j]); thread = rows 2 warp, 2 warp + 1, columns 4 lane .. 4 lane + 3.
// VERTICAL sums first (they are shared by the pixels of a row segment):
//   output row j in {0, 1} sees luminance rows j .. j+4 of the six rows L0..L5 this thread reads; per column
//     V5_j = sum of its 5 rows, V3_j = sum of its 3 middle rows, VS_j = [1 2 1] smooth of the middle rows = V3_j + centre row,
//     VD_j = row j+1 - row j+3;
//   then per pixel  la = sum_5 V5 + sum_3 V3 - 2 centre,  gx = VS[x+1] - VS[x-1],  gy = VD[x-1] + 2 VD[x] + VD[x+1]
//   (the 5x5 kernel of modules/jnd.py:37-43 is ones(5,5) + ones(3,3) - 2 delta; Sobel pair jnd.py:44-53).
__device__ __forceinline__ float2 f2sub(float2 a, float2 b) { return f2fma(b, make_float2(-1.f, -1.f), a); }
__device__ __forceinline__ float2 f2s(float v) { return make_float2(v, v); }
// jnd_value of two pixels on float2 pairs (add / mul / fma per component).  Same operations in the same order as jnd_value, except that hi's (la0 - 127) * 3/128 + 3
// is one FMA with the constant folded (1 rounding less).
__device__ __forceinline__ float2 jnd_value2(float2 la_sum, float2 gx, float2 gy) {
  const float2 la0 = f2mul(la_sum, f2s(1.f / 32.f));
  const float2 t = f2fma(la0, f2s(1.f / 127.f), f2s(1e-5f));
  const float2 lo = f2fma(f2s(-17.f), make_float2(sqrt_approx(t.x), sqrt_approx(t.y)), f2s(17.f));
  const float2 hi = f2fma(f2s(3.f / 128.f), la0, f2s(3.f - 127.f * 3.f / 128.f));
  const float2 la = make_float2(la0.x <= 127.f ? lo.x : hi.x, la0.y <= 127.f ? lo.y : hi.y);
  const float2 g2 = f2fma(gx, gx, f2mul(gy, gy));
  const float2 e = f2mul(f2s(1.2f), make_float2(lg2_approx(g2.x), lg2_approx(g2.y)));     // g^2.4 = (g^2)^1.2;  g2 == 0 -> lg2 = -inf -> 0
  const float2 den = f2add(g2, f2s(676.f));
  const float2 cm = f2mul(f2mul(f2s(0.117f * 16.f), make_float2(ex2_approx_f(e.x), ex2_approx_f(e.y))),
                          make_float2(rcp_approx_f(den.x), rcp_approx_f(den.y)));
  const float2 r = f2fma(f2s(-0.3f), make_float2(fminf(la.x, cm.x), fminf(la.y, cm.y)), f2add(la, cm));
  return f2mul(make_float2(fmaxf(r.x, 0.f), fmaxf(r.y, 0.f)), f2s(1.f / 255.f));
}

__device__ __forceinline__ void jnd_hm_vec4(const float* __restrict__ lum_, int warp, int lane, float (&hm)[2][4]) {
  // columns 2..9 of the 12 floats at shared column lane*4, as the four aligned pairs the 128-bit loads deliver; pixel q's centre = column 2 + q of them
  float2 L[6][4];
#pragma unroll
  for (int r = 0; r < 6; ++r) {
    const float4* s4 = reinterpret_cast<const float4*>(lum_ + (warp * 2 + r) * kB2LP + lane * 4);
    const float4 t0 = s4[0], t1 = s4[1], t2 = s4[2];
    L[r][0] = make_float2(t0.z, t0.w); L[r][1] = make_float2(t1.x, t1.y); L[r][2] = make_float2(t1.z, t1.w); L[r][3] = make_float2(t2.x, t2.y);
  }
  float V5[2][8], V3[2][8], VS[2][8], VD[2][8];       // [output row][column 0..7]; V3 / VS / VD are used on columns 1..6 only
#pragma unroll
  for (int h = 0; h < 4; ++h) {
    const float2 mid4 = f2add(f2add(L[1][h], L[2][h]), f2add(L[3][h], L[4][h]));
    const float2 a0 = f2add(mid4, L[0][h]), a1 = f2add(mid4, L[5][h]);
    const float2 c23 = f2add(L[2][h], L[3][h]);
    const float2 b0 = f2add(c23, L[1][h]), b1 = f2add(c23, L[4][h]);
    const float2 s0 = f2add(b0, L[2][h]), s1 = f2add(b1, L[3][h]);
    const float2 d0 = f2sub(L[1][h], L[3][h]), d1 = f2sub(L[2][h], L[4][h]);
    V5[0][2 * h] = a0.x; V5[0][2 * h + 1] = a0.y; V5[1][2 * h] = a1.x; V5[1][2 * h + 1] = a1.y;
    V3[0][2 * h] = b0.x; V3[0][2 * h + 1] = b0.y; V3[1][2 * h] = b1.x; V3[1][2 * h + 1] = b1.y;
    VS[0][2 * h] = s0.x; VS[0][2 * h + 1] = s0.y; VS[1][2 * h] = s1.x; VS[1][2 * h + 1] = s1.y;
    VD[0][2 * h] = d0.x; VD[0][2 * h + 1] = d0.y; VD[1][2 * h] = d1.x; VD[1][2 * h + 1] = d1.y;
  }
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int q = 0; q < 4; q += 2) {
      float lac[2], gx[2], gy[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int x = q + u;                                   // centre column x + 2
        const float la = ((V5[j][x] + V5[j][x + 1]) + (V5[j][x + 2] + V5[j][x + 3])) + V5[j][x + 4] +
                         (V3[j][x + 1] + V3[j][x + 2] + V3[j][x + 3]);
        const float ctr = (x & 1) ? L[2 + j][(x + 2) >> 1].y : L[2 + j][(x + 2) >> 1].x;
        lac[u] = fmaf(-2.f, ctr, la);
        gx[u] = VS[j][x + 3] - VS[j][x + 1];
        gy[u] = fmaf(2.f, VD[j][x + 2], VD[j][x + 1] + VD[j][x + 3]);
      }
      const float2 v = jnd_value2(make_float2(lac[0], lac[1]), make_float2(gx[0], gx[1]), make_float2(gy[0], gy[1]));
      hm[j][q] = v.x; hm[j][q + 1] = v.y;
    }
}

// Delta up-scale through 4 taps per axis (bicubic tables, 3 or 4 taps): the taps of output o, as the offset of its first tap from
// `base` and its weights, zero past its tap count.  The kernels read all 4 samples; those past the count have weight 0 and lie
// inside the staged tile (kB2DH4 rows; columns: see kB2DH4), which holds finite values everywhere.
__device__ __forceinline__ int taps4(const int* __restrict__ start, const int* __restrict__ cnt, const float* __restrict__ w, int maxt,
                                     int o, int base, float (&wo)[4]) {
  const int c = __ldg(cnt + o);
#pragma unroll
  for (int i = 0; i < 4; ++i) wo[i] = i < c ? __ldg(w + (long)o * maxt + i) : 0.f;
  return __ldg(start + o) - base;
}
// sum over the 4 x 4 staged samples from `a` (row pitch P): horizontal sums per source row first, then the vertical one
template <int P>
__device__ __forceinline__ float up4(const float* a, const float (&xw)[4], const float (&yw)[4]) {
  float v = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float* r = a + i * P;
    const float h = fmaf(xw[3], r[3], fmaf(xw[2], r[2], fmaf(xw[1], r[1], xw[0] * r[0])));
    v = i == 0 ? yw[0] * h : fmaf(yw[i], h, v);
  }
  return v;
}

// VEC 4: W % 4 == 0 and 16-byte aligned tensors: thread = 4 consecutive pixels (128-bit global / shared accesses).
// VEC 1: any W / alignment: thread = pixels lane, lane+32, lane+64, lane+96 of the tile row (32-bit accesses, fully coalesced).
// FASTUP 1: the delta is read in place (identity) or up-scaled through <= 2 taps per axis from a tile staged in shared memory
//           (every input at least as large as the processing size); 4: the same through 3 or 4 taps per axis (kB2DH4 x kB2DW tile,
//           zero outside the delta); 0: generic separable tables straight from global memory.
// Thread = 2 rows x 4 pixels.  The 5x5 luminance filter and the Sobel pair are evaluated SEPARABLY while the six luminance rows
// of the two output rows stream through registers (per row: 5- and 3-sums, the horizontal difference and the [1 2 1] smooth).
// CD: delta channels (1 for the Y-channel cards, 3 for RGB U-Nets) as a compile-time constant: the per-channel loops and their
// accumulators disappear from the single-channel instantiation.
// JIN: heat-map inputs (1: luminance; 3: one map per RGB channel, configs/attenuation.yaml jnd_3_*), compile-time for the same reason.
template <int VEC, int FASTUP, int CD, int JIN>
__global__ void __launch_bounds__(256, 3) jnd_blend2_kernel(const BlendParams p) {
  extern __shared__ __align__(16) float b2_smem_[];
  constexpr int LUMP = (kB2TH + 4) * kB2LP;               // floats per luminance plane
  float* lum = b2_smem_;                                  // [JIN][TH + 4][LP]
  float* rgb = lum + JIN * LUMP;                          // [3][TH][TW]
  float* dl = rgb + 3 * kB2TH * kB2TW;                    // [DH][DW]
  const int f = blockIdx.z, x0 = blockIdx.x * kB2TW, y0 = blockIdx.y * kB2TH;
  const long plane = (long)p.H * p.W;
  const float* img = p.imgs + (long)f * 3 * plane;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  auto col_of = [&](int q) { return VEC == 4 ? lane * 4 + q : lane + 32 * q; };
  const FrameKeys fk = frame_keys(f, p.F, p.step, p.alternate, p.interp_chunk);
  const bool has_delta = fk.has;
  const int nsrc = (fk.k1 != fk.k0 && fk.a != 1.f) ? 2 : 1;
  const bool staged = FASTUP && !p.identity_resample && has_delta;

  // delta tile geometry (staged path): source rows / columns touched by this output tile
  int sy0 = 0, sx0 = 0, dnr = 0, dnc = 0;
  if (staged) {
    const int ylast = min(y0 + kB2TH, p.H) - 1, xlast = min(x0 + kB2TW, p.W) - 1;
    sy0 = __ldg(p.tab.ystart + y0);
    sx0 = __ldg(p.tab.xstart + x0);
    dnr = min(__ldg(p.tab.ystart + ylast) + __ldg(p.tab.ycnt + ylast), p.PH) - sy0;    // <= DH (host guarantees H >= PH, W >= PW)
    dnc = min(__ldg(p.tab.xstart + xlast) + __ldg(p.tab.xcnt + xlast), p.PW) - sx0;    // <= DW
  }
  auto stage_delta = [&](int c, int s) {
    const float* src = p.delta + ((long)(s ? fk.k1 : fk.k0) * CD + c) * p.PH * p.PW + (long)sy0 * p.PW + sx0;
    if constexpr (FASTUP == 4) {         // the whole tile: the 4-tap reads pass the last tap of an edge output (with weight 0)
      for (int r = warp; r < kB2DH4; r += 8)
        for (int cc = lane; cc < kB2DW; cc += 32)
          dl[r * kB2DW + cc] = (sy0 + r < p.PH && sx0 + cc < p.PW) ? __ldg(src + (long)r * p.PW + cc) : 0.f;
    } else {
      for (int r = warp; r < dnr; r += 8)
        for (int cc = lane; cc < dnc; cc += 32) dl[r * kB2DW + cc] = __ldg(src + (long)r * p.PW + cc);
    }
  };

  // ---- phase 1: this thread's pixels (2 rows x 4 pixels x RGB) -> shared; luminance tile with a 2-pixel zero halo
#pragma unroll
  for (int k = 0; k < 2; ++k) {
    const int yl = warp * 2 + k, gy = y0 + yl;
    if (VEC == 4) {
      const int gx = x0 + lane * 4;
      float4 v[3];
      v[0] = v[1] = v[2] = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gy < p.H && gx < p.W) {
        const float* s = img + (long)gy * p.W + gx;
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = __ldg(reinterpret_cast<const float4*>(s + c * plane));
      }
#pragma unroll
      for (int c = 0; c < 3; ++c) *reinterpret_cast<float4*>(rgb + (c * kB2TH + yl) * kB2TW + lane * 4) = v[c];
      if (p.use_jnd) {
        if (JIN == 1) {
          *reinterpret_cast<float4*>(lum + (yl + 2) * kB2LP + 4 + lane * 4) =
              make_float4(lum255(v[0].x, v[1].x, v[2].x), lum255(v[0].y, v[1].y, v[2].y), lum255(v[0].z, v[1].z, v[2].z),
                          lum255(v[0].w, v[1].w, v[2].w));
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c)
            *reinterpret_cast<float4*>(lum + c * LUMP + (yl + 2) * kB2LP + 4 + lane * 4) =
                make_float4(255.f * v[c].x, 255.f * v[c].y, 255.f * v[c].z, 255.f * v[c].w);
        }
      }
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int col = lane + 32 * q, gx = x0 + col;
        float v[3] = {0.f, 0.f, 0.f};
        if (gy < p.H && gx < p.W) {
          const float* s = img + (long)gy * p.W + gx;
#pragma unroll
          for (int c = 0; c < 3; ++c) v[c] = __ldg(s + c * plane);
        }
#pragma unroll
        for (int c = 0; c < 3; ++c) rgb[(c * kB2TH + yl) * kB2TW + col] = v[c];
        if (p.use_jnd) {
          if (JIN == 1) lum[(yl + 2) * kB2LP + 4 + col] = lum255(v[0], v[1], v[2]);
          else {
#pragma unroll
            for (int c = 0; c < 3; ++c) lum[c * LUMP + (yl + 2) * kB2LP + 4 + col] = 255.f * v[c];
          }
        }
      }
    }
  }
  if (p.use_jnd) {
    if (warp < 4) {   // halo rows: shared rows 0, 1, TH+2, TH+3 <-> image rows y0-2, y0-1, y0+TH, y0+TH+1
      const int s = warp < 2 ? warp : kB2TH + warp;
      const int gy = y0 + s - 2;
      const bool rowok = gy >= 0 && gy < p.H;
      if (VEC == 4) {
        const int gx = x0 + lane * 4;
        float4 l4 = make_float4(0.f, 0.f, 0.f, 0.f);
        if (rowok && gx < p.W) {
          const float* sp = img + (long)gy * p.W + gx;
          const float4 r = __ldg(reinterpret_cast<const float4*>(sp)), g = __ldg(reinterpret_cast<const float4*>(sp + plane)),
                       b = __ldg(reinterpret_cast<const float4*>(sp + 2 * plane));
          l4 = make_float4(lum255(r.x, g.x, b.x), lum255(r.y, g.y, b.y), lum255(r.z, g.z, b.z), lum255(r.w, g.w, b.w));
          if (JIN == 3) {
            *reinterpret_cast<float4*>(lum + 1 * LUMP + s * kB2LP + 4 + lane * 4) = make_float4(255.f * g.x, 255.f * g.y, 255.f * g.z, 255.f * g.w);
            *reinterpret_cast<float4*>(lum + 2 * LUMP + s * kB2LP + 4 + lane * 4) = make_float4(255.f * b.x, 255.f * b.y, 255.f * b.z, 255.f * b.w);
            l4 = make_float4(255.f * r.x, 255.f * r.y, 255.f * r.z, 255.f * r.w);
          }
        } else if (JIN == 3) {
          *reinterpret_cast<float4*>(lum + 1 * LUMP + s * kB2LP + 4 + lane * 4) = l4;
          *reinterpret_cast<float4*>(lum + 2 * LUMP + s * kB2LP + 4 + lane * 4) = l4;
        }
        *reinterpret_cast<float4*>(lum + s * kB2LP + 4 + lane * 4) = l4;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int col = lane + 32 * q, gx = x0 + col;
          float l3[3] = {0.f, 0.f, 0.f};
          if (rowok && gx < p.W) {
            const float* sp = img + (long)gy * p.W + gx;
            const float r = __ldg(sp), g = __ldg(sp + plane), bb = __ldg(sp + 2 * plane);
            if (JIN == 1) l3[0] = lum255(r, g, bb);
            else { l3[0] = 255.f * r; l3[1] = 255.f * g; l3[2] = 255.f * bb; }
          }
#pragma unroll
          for (int c = 0; c < JIN; ++c) lum[c * LUMP + s * kB2LP + 4 + col] = l3[c];
        }
      }
    } else {          // warps 4..7: halo columns x0-2, x0-1, x0+TW, x0+TW+1 of all TH+4 rows
      const int ht = (int)threadIdx.x - 128;
      if (ht < 4 * (kB2TH + 4)) {
        const int s = ht >> 2, j = ht & 3;
        const int col = j < 2 ? j - 2 : kB2TW + j - 2;
        const int gy = y0 + s - 2, gx = x0 + col;
        float l3[3] = {0.f, 0.f, 0.f};
        if (gy >= 0 && gy < p.H && gx >= 0 && gx < p.W) {
          const float* sp = img + (long)gy * p.W + gx;
          const float r = __ldg(sp), g = __ldg(sp + plane), bb = __ldg(sp + 2 * plane);
          if (JIN == 1) l3[0] = lum255(r, g, bb);
          else { l3[0] = 255.f * r; l3[1] = 255.f * g; l3[2] = 255.f * bb; }
        }
#pragma unroll
        for (int c = 0; c < JIN; ++c) lum[c * LUMP + s * kB2LP + 4 + col] = l3[c];
      }
    }
  }
  if (staged) stage_delta(0, 0);
  __syncthreads();

  // ---- phase 2a: heat-map of this thread's 2 x 4 pixels.  VERTICAL sums first (they are shared by the pixels of a row segment):
  //   output row j in {0, 1} sees luminance rows j .. j+4 of the six rows L0..L5 this thread reads; per column
  //     V5_j = sum of its 5 rows, V3_j = sum of its 3 middle rows, VS_j = [1 2 1] smooth of the middle rows = V3_j + centre row,
  //     VD_j = row j+1 - row j+3;
  //   then per pixel  la = sum_5 V5 + sum_3 V3 - 2 centre,  gx = VS[x+1] - VS[x-1],  gy = VD[x-1] + 2 VD[x] + VD[x+1]
  //   (the 5x5 kernel of modules/jnd.py:37-43 is ones(5,5) + ones(3,3) - 2 delta; Sobel pair jnd.py:44-53).
  float hmc[JIN][2][4];
#pragma unroll
  for (int c = 0; c < JIN; ++c)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) hmc[c][j][q] = 1.f;
  if (p.use_jnd) {
#pragma unroll
   for (int jc = 0; jc < JIN; ++jc) {
    const float* lum_ = lum + jc * LUMP;
    float (&hm)[2][4] = hmc[jc];
    if (VEC == 4) {
      jnd_hm_vec4(lum_, warp, lane, hm);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float* cpt = lum_ + (warp * 2) * kB2LP + 4 + lane + 32 * q;      // row 0 of the window, centre column
        float L[6][5];
#pragma unroll
        for (int r = 0; r < 6; ++r)
#pragma unroll
          for (int i = 0; i < 5; ++i) L[r][i] = cpt[r * kB2LP + i - 2];
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          float la = 0.f, gx = 0.f, gy = 0.f;
#pragma unroll
          for (int i = 0; i < 5; ++i) {
            const float v5 = L[j][i] + L[j + 1][i] + L[j + 2][i] + L[j + 3][i] + L[j + 4][i];
            la += v5;
            if (i >= 1 && i <= 3) {
              const float v3 = L[j + 1][i] + L[j + 2][i] + L[j + 3][i];
              la += v3;
              const float vs = v3 + L[j + 2][i], vd = L[j + 1][i] - L[j + 3][i];
              if (i == 1) { gx -= vs; gy += vd; }
              if (i == 2) gy = fmaf(2.f, vd, gy);
              if (i == 3) { gx += vs; gy += vd; }
            }
          }
          la = fmaf(-2.f, L[j + 2][2], la);
          hm[j][q] = jnd_value(la, gx, gy);
        }
      }
    }
   }
    if (JIN == 3 && p.jnd_out == 1) {      // hmaps = sum(hmaps / 3) over the channels (jnd.py:101); /255 is inside jnd_value
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) hmc[0][j][q] = hmc[0][j][q] / 3.f + hmc[JIN - 1 > 0 ? 1 : 0][j][q] / 3.f + hmc[JIN - 1][j][q] / 3.f;
    }
  }
  const bool hm_per_channel = JIN == 3 && p.jnd_out == 3;

  // ---- phase 2b: delta of the 2 x 4 pixels (up-resampled from PH x PW), x heat-map
  float d[CD][2][4];
#pragma unroll
  for (int c = 0; c < CD; ++c)
#pragma unroll
    for (int j = 0; j < 2; ++j)
#pragma unroll
      for (int q = 0; q < 4; ++q) d[c][j][q] = 0.f;
  if constexpr (FASTUP == 4) {           // (launched for up-scales only: never in place)
    if (has_delta) {
      int xr[4], yr[2];
      float xw[4][4], yw[2][4];
#pragma unroll
      for (int q = 0; q < 4; ++q) xr[q] = taps4(p.tab.xstart, p.tab.xcnt, p.tab.xw, p.tab.maxt_x, min(x0 + col_of(q), p.W - 1), sx0, xw[q]);
#pragma unroll
      for (int j = 0; j < 2; ++j) yr[j] = taps4(p.tab.ystart, p.tab.ycnt, p.tab.yw, p.tab.maxt_y, min(y0 + warp * 2 + j, p.H - 1), sy0, yw[j]);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (c >= CD) break;
        for (int s = 0; s < nsrc; ++s) {
          if ((c | s) != 0) {
            __syncthreads();
            stage_delta(c, s);
            __syncthreads();
          }
          const float ws = nsrc == 1 ? 1.f : (s ? 1.f - fk.a : fk.a);
#pragma unroll
          for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              const float vs = up4<kB2DW>(dl + yr[j] * kB2DW + xr[q], xw[q], yw[j]);
              d[c][j][q] = fmaf(ws, vs, d[c][j][q]);
            }
        }
      }
    }
  } else if (has_delta) {
    int xr[4] = {0, 0, 0, 0}, xo[4] = {0, 0, 0, 0};
    float xw0[4] = {1.f, 1.f, 1.f, 1.f}, xw1[4] = {0.f, 0.f, 0.f, 0.f};
    int yr[2] = {0, 0}, yo[2] = {0, 0};
    float yw0[2] = {1.f, 1.f}, yw1[2] = {0.f, 0.f};
    if (staged) {
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int ox = min(x0 + col_of(q), p.W - 1);
        const int xc = __ldg(p.tab.xcnt + ox);
        xr[q] = __ldg(p.tab.xstart + ox) - sx0;
        xw0[q] = __ldg(p.tab.xw + (long)ox * p.tab.maxt_x);
        xw1[q] = xc > 1 ? __ldg(p.tab.xw + (long)ox * p.tab.maxt_x + 1) : 0.f;
        xo[q] = xc > 1 ? 1 : 0;
      }
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const int oy = min(y0 + warp * 2 + j, p.H - 1);
        const int yc = __ldg(p.tab.ycnt + oy);
        yr[j] = __ldg(p.tab.ystart + oy) - sy0;
        yw0[j] = __ldg(p.tab.yw + (long)oy * p.tab.maxt_y);
        yw1[j] = yc > 1 ? __ldg(p.tab.yw + (long)oy * p.tab.maxt_y + 1) : 0.f;
        yo[j] = yc > 1 ? 1 : 0;
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      if (c >= CD) break;
      for (int s = 0; s < nsrc; ++s) {
        if (staged && (c | s) != 0) {      // the tile of the first (channel, key) was staged together with the image
          __syncthreads();
          stage_delta(c, s);
          __syncthreads();
        }
        const float ws = nsrc == 1 ? 1.f : (s ? 1.f - fk.a : fk.a);
        const bool same_rows = staged && yr[0] == yr[1] && yo[0] == yo[1];
        float hra[4], hrb[4];
#pragma unroll
        for (int q = 0; q < 4; ++q) { hra[q] = 0.f; hrb[q] = 0.f; }
        const float* src = p.delta + ((long)(s ? fk.k1 : fk.k0) * CD + c) * p.PH * p.PW;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int gy = y0 + warp * 2 + j;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const int gx = x0 + col_of(q);
            float vs = 0.f;
            if (gy < p.H && gx < p.W) {
              if (p.identity_resample) {
                vs = __ldg(src + (long)gy * p.PW + gx);
              } else if (FASTUP) {
                if (j == 0 || !same_rows) {     // (warp-uniform) at scale 3 two of three row pairs share both source rows
                  const float* a0 = dl + yr[j] * kB2DW + xr[q];
                  const float* b0 = a0 + yo[j] * kB2DW;
                  hra[q] = xw0[q] * a0[0] + xw1[q] * a0[xo[q]];
                  hrb[q] = xw0[q] * b0[0] + xw1[q] * b0[xo[q]];
                }
                vs = yw0[j] * hra[q] + yw1[j] * hrb[q];
              } else {
                const int ys2 = p.tab.ystart[gy], yc = p.tab.ycnt[gy], xs2 = p.tab.xstart[gx], xc = p.tab.xcnt[gx];
                for (int jj = 0; jj < yc; ++jj) {
                  float racc = 0.f;
                  for (int i = 0; i < xc; ++i) racc += p.tab.xw[gx * p.tab.maxt_x + i] * __ldg(src + (long)(ys2 + jj) * p.PW + xs2 + i);
                  vs += p.tab.yw[gy * p.tab.maxt_y + jj] * racc;
                }
              }
            }
            d[c][j][q] = fmaf(ws, vs, d[c][j][q]);
          }
        }
      }
    }
  }

  // ---- phase 2c: preds_w = hmap * delta (optional output; max(CD, jnd_out) channels, broadcast like `hmaps * preds_w`) and the blend
  const int PC = (p.use_jnd && p.jnd_out == 3) ? 3 : CD;
#pragma unroll
  for (int j = 0; j < 2; ++j) {
    const int yl = warp * 2 + j, gy = y0 + yl;
    if (gy >= p.H) break;
    const long o = (long)gy * p.W + x0;
    const bool vfull = VEC == 4 && (x0 + lane * 4 < p.W);      // W % 4 == 0: a 4-pixel group is inside or outside as a whole
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float pw[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) pw[q] = d[CD == 1 ? 0 : c][j][q] * (JIN == 3 ? (hm_per_channel ? hmc[JIN == 3 ? c : 0][j][q] : hmc[0][j][q]) : hmc[0][j][q]);
      if (p.preds_w != nullptr && c < PC) {
        float* dst = p.preds_w + ((long)f * PC + c) * plane + o;
        if (VEC == 4) {
          if (vfull) *reinterpret_cast<float4*>(dst + lane * 4) = make_float4(pw[0], pw[1], pw[2], pw[3]);
        } else {
#pragma unroll
          for (int q = 0; q < 4; ++q) if (x0 + lane + 32 * q < p.W) dst[lane + 32 * q] = pw[q];
        }
      }
      float in[4], out[4];
      if (VEC == 4) {
        const float4 t4 = *reinterpret_cast<const float4*>(rgb + (c * kB2TH + yl) * kB2TW + lane * 4);
        in[0] = t4.x; in[1] = t4.y; in[2] = t4.z; in[3] = t4.w;
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) in[q] = rgb[(c * kB2TH + yl) * kB2TW + lane + 32 * q];
      }
      if (p.clamp) {       // FFMA.SAT
#pragma unroll
        for (int q = 0; q < 4; ++q) out[q] = __saturatef(fmaf(p.scaling_i, in[q], p.scaling_w * pw[q]));
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) out[q] = fmaf(p.scaling_i, in[q], p.scaling_w * pw[q]);
      }
      float* dst = p.imgs_w + ((long)f * 3 + c) * plane + o;
      if (VEC == 4) {
        if (vfull) *reinterpret_cast<float4*>(dst + lane * 4) = make_float4(out[0], out[1], out[2], out[3]);
      } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) if (x0 + lane + 32 * q < p.W) dst[lane + 32 * q] = out[q];
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ K7, TMA-fed
// The same blend for the common layout (W % 4 == 0, 16-byte aligned tensors, delta read in place or up-scaled through <= 2 taps per
// axis): a block walks kB3NT vertically adjacent 128 x 16 tiles.  ONE TMA box per tile brings the raw RGB tile with its 2-pixel
// halo ([3][20][136] floats at (x0 - 4, y0 - 2); the engine zero-fills what lies outside the image, which is exactly the zero padding of
// the reference's conv2d), a second one the delta tile at processing resolution; both land in the other half of a double buffer while
// the current tile is computed.  Unlike the load-then-compute kernel above, the loads cost one instruction per tile and the per-block
// set-up is amortised over kB3NT tiles.
constexpr int kB3NT = 4;
constexpr int kB3RAW = 3 * (kB2TH + 4) * kB2LP;             // floats of one raw tile (32 640 B, a multiple of 128)
constexpr int kB3DW = kB2DW + 4;                            // delta tile pitch: the box starts at a 16-byte aligned source column (TMA faults otherwise)
constexpr int kB3DL = 2464;                                 // floats reserved per delta tile (kB2DH * kB3DW = 2448, rounded to 128 B)
constexpr int kB3DL4 = kB2DH4 * kB3DW;                      // the same for the 4-tap up-scale (2720 floats, a multiple of 128 B)
constexpr size_t b3_smem(int jin, int fastup = 1) {
  return (size_t)(2 * kB3RAW + 2 * (fastup == 4 ? kB3DL4 : kB3DL) + jin * (kB2TH + 4) * kB2LP) * sizeof(float) + 2 * sizeof(uint64_t) + 128;
}

// FASTUP 1: delta in place or through <= 2 taps per axis; 4: through 3 or 4 taps per axis, from a kB2DH4-row box
template <int CD, int JIN, int FASTUP = 1>
__global__ void __launch_bounds__(256, 2) jnd_blend3_kernel(const BlendParams p, const __grid_constant__ CUtensorMap tmI,
                                                            const __grid_constant__ CUtensorMap tmD) {
  extern __shared__ uint8_t b3_smem_[];
  constexpr int LUMP = (kB2TH + 4) * kB2LP;
  constexpr int DL = FASTUP == 4 ? kB3DL4 : kB3DL, DH = FASTUP == 4 ? kB2DH4 : kB2DH;
  float* raw = reinterpret_cast<float*>(b3_smem_ + ((128u - (smem_u32(b3_smem_) & 127u)) & 127u));   // [2][3][TH + 4][LP], 128-byte aligned
  float* dlb = raw + 2 * kB3RAW;                          // [2][DH][kB3DW]
  float* lum = dlb + 2 * DL;                              // [JIN][TH + 4][LP]
  uint64_t* full = reinterpret_cast<uint64_t*>(lum + JIN * LUMP);
  const int f = blockIdx.z, x0 = blockIdx.x * kB2TW, Y0 = blockIdx.y * (kB3NT * kB2TH);
  const int plane = p.H * p.W;                            // < 2^31 (host-checked)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const FrameKeys fk = frame_keys(f, p.F, p.step, p.alternate, p.interp_chunk);
  const bool has_delta = fk.has;
  const int nsrc = (fk.k1 != fk.k0 && fk.a != 1.f) ? 2 : 1;
  const bool staged = !p.identity_resample && has_delta;
  const int ntl = min(kB3NT, (p.H - Y0 + kB2TH - 1) / kB2TH);
  const int sx0 = staged ? (__ldg(p.tab.xstart + x0) & ~3) : 0;      // first source column of the delta tile, rounded down to 16 bytes
  const uint32_t tx_bytes = (uint32_t)(kB3RAW * sizeof(float)) + (staged ? (uint32_t)(DH * kB3DW * sizeof(float)) : 0u);

  auto issue = [&](int t) {                               // thread 0: both boxes of tile t
    const int buf = t & 1, y0 = Y0 + t * kB2TH;
    fence_proxy_async_smem();                             // the buffer was last touched through the generic proxy
    mbar_arrive_expect_tx(&full[buf], tx_bytes);
    tma_load_3d(&tmI, &full[buf], raw + buf * kB3RAW, x0 - 4, y0 - 2, f * 3);
    if (staged) tma_load_3d(&tmD, &full[buf], dlb + buf * DL, sx0, __ldg(p.tab.ystart + y0), fk.k0 * CD);
  };
  if (threadIdx.x == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    fence_barrier_init();
    issue(0);
  }
  // x taps of this thread's 4 pixels for the delta up-sample (the same for every tile of the block)
  int xr[4] = {0, 0, 0, 0}, xo[4] = {0, 0, 0, 0};
  float xw0[4] = {1.f, 1.f, 1.f, 1.f}, xw1[4] = {0.f, 0.f, 0.f, 0.f};
  float xw4[FASTUP == 4 ? 4 : 1][4];                      // 4-tap weights
  if constexpr (FASTUP == 4) {
    if (staged) {
#pragma unroll
      for (int q = 0; q < 4; ++q) xr[q] = taps4(p.tab.xstart, p.tab.xcnt, p.tab.xw, p.tab.maxt_x, min(x0 + lane * 4 + q, p.W - 1), sx0, xw4[q]);
    }
  } else if (staged) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int ox = min(x0 + lane * 4 + q, p.W - 1);
      const int xc = __ldg(p.tab.xcnt + ox);
      xr[q] = __ldg(p.tab.xstart + ox) - sx0;
      xw0[q] = __ldg(p.tab.xw + ox * p.tab.maxt_x);
      xw1[q] = xc > 1 ? __ldg(p.tab.xw + ox * p.tab.maxt_x + 1) : 0.f;
      xo[q] = xc > 1 ? 1 : 0;
    }
  }
  const bool vfull = x0 + lane * 4 < p.W;                 // W % 4 == 0: a 4-pixel group is inside or outside as a whole
  const int PC = (p.use_jnd && p.jnd_out == 3) ? 3 : CD;
  const bool hm_per_channel = JIN == 3 && p.jnd_out == 3;
  __syncthreads();                                        // barrier initialisation visible to every waiter

  for (int t = 0; t < ntl; ++t) {
    const int y0 = Y0 + t * kB2TH, buf = t & 1;
    const float* rawb = raw + buf * kB3RAW;
    float* dl = dlb + buf * DL;
    if (t + 1 < ntl && threadIdx.x == 0) issue(t + 1);    // buffer buf^1 was released by the barrier that ended tile t - 1
    mbar_wait(&full[buf], (t >> 1) & 1);

    // ---- luminance planes (with halo) from the raw tile
    if (p.use_jnd) {
      for (int i = threadIdx.x; i < (kB2TH + 4) * (kB2LP / 4); i += 256) {
        const float4 r = *reinterpret_cast<const float4*>(rawb + i * 4), g = *reinterpret_cast<const float4*>(rawb + LUMP + i * 4),
                     bq = *reinterpret_cast<const float4*>(rawb + 2 * LUMP + i * 4);
        if (JIN == 1) {
          *reinterpret_cast<float4*>(lum + i * 4) =
              make_float4(lum255(r.x, g.x, bq.x), lum255(r.y, g.y, bq.y), lum255(r.z, g.z, bq.z), lum255(r.w, g.w, bq.w));
        } else {
          *reinterpret_cast<float4*>(lum + i * 4) = make_float4(255.f * r.x, 255.f * r.y, 255.f * r.z, 255.f * r.w);
          *reinterpret_cast<float4*>(lum + (JIN > 1 ? LUMP : 0) + i * 4) = make_float4(255.f * g.x, 255.f * g.y, 255.f * g.z, 255.f * g.w);
          *reinterpret_cast<float4*>(lum + (JIN > 2 ? 2 * LUMP : 0) + i * 4) = make_float4(255.f * bq.x, 255.f * bq.y, 255.f * bq.z, 255.f * bq.w);
        }
      }
      __syncthreads();
    }

    // ---- heat-map of this thread's 2 x 4 pixels
    float hmc[JIN][2][4];
#pragma unroll
    for (int c = 0; c < JIN; ++c)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) hmc[c][j][q] = 1.f;
    if (p.use_jnd) {
#pragma unroll
      for (int jc = 0; jc < JIN; ++jc) jnd_hm_vec4(lum + jc * LUMP, warp, lane, hmc[jc]);
      if (JIN == 3 && p.jnd_out == 1) {      // hmaps = sum(hmaps / 3) over the channels (jnd.py:101); /255 is inside jnd_value
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
          for (int q = 0; q < 4; ++q) hmc[0][j][q] = hmc[0][j][q] / 3.f + hmc[JIN - 1 > 0 ? 1 : 0][j][q] / 3.f + hmc[JIN - 1][j][q] / 3.f;
      }
    }

    // ---- delta of the 2 x 4 pixels (read in place, or up-sampled from the staged PH x PW tile)
    float d[CD][2][4];
#pragma unroll
    for (int c = 0; c < CD; ++c)
#pragma unroll
      for (int j = 0; j < 2; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) d[c][j][q] = 0.f;
    if (has_delta) {
      int yr[2] = {0, 0}, yo[2] = {0, 0};
      float yw0[2] = {1.f, 1.f}, yw1[2] = {0.f, 0.f};
      int sy0 = 0, dnr = 0, dnc = 0;
      float yw4[FASTUP == 4 ? 2 : 1][4];                  // 4-tap weights
      if (staged) {
        sy0 = __ldg(p.tab.ystart + y0);
        if constexpr (FASTUP == 4) {
#pragma unroll
          for (int j = 0; j < 2; ++j) yr[j] = taps4(p.tab.ystart, p.tab.ycnt, p.tab.yw, p.tab.maxt_y, min(y0 + warp * 2 + j, p.H - 1), sy0, yw4[j]);
        } else {
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const int oy = min(y0 + warp * 2 + j, p.H - 1);
          const int yc = __ldg(p.tab.ycnt + oy);
          yr[j] = __ldg(p.tab.ystart + oy) - sy0;
          yw0[j] = __ldg(p.tab.yw + oy * p.tab.maxt_y);
          yw1[j] = yc > 1 ? __ldg(p.tab.yw + oy * p.tab.maxt_y + 1) : 0.f;
          yo[j] = yc > 1 ? 1 : 0;
        }
        }
        if (CD * nsrc > 1) {                 // geometry of the tiles staged by hand below
          const int ylast = min(y0 + kB2TH, p.H) - 1, xlast = min(x0 + kB2TW, p.W) - 1;
          dnr = min(__ldg(p.tab.ystart + ylast) + __ldg(p.tab.ycnt + ylast), p.PH) - sy0;
          dnc = min(__ldg(p.tab.xstart + xlast) + __ldg(p.tab.xcnt + xlast), p.PW) - sx0;
        }
      }
      const bool same_rows = staged && yr[0] == yr[1] && yo[0] == yo[1];
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        if (c >= CD) break;
        for (int s = 0; s < nsrc; ++s) {
          const float* src = p.delta + ((long)(s ? fk.k1 : fk.k0) * CD + c) * p.PH * p.PW;
          if (staged && (c | s) != 0) {      // the tile of the first (channel, key) arrived with the image tile; the others are staged here
            __syncthreads();
            for (int r = warp; r < dnr; r += 8)
              for (int cc = lane; cc < dnc; cc += 32) dl[r * kB3DW + cc] = __ldg(src + (long)(sy0 + r) * p.PW + sx0 + cc);
            __syncthreads();
          }
          const float ws = nsrc == 1 ? 1.f : (s ? 1.f - fk.a : fk.a);
          float hra[4] = {0.f, 0.f, 0.f, 0.f}, hrb[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int j = 0; j < 2; ++j) {
            const int gy = y0 + warp * 2 + j;
            float vs[4] = {0.f, 0.f, 0.f, 0.f};
            if (gy < p.H && vfull) {
              if (p.identity_resample) {
                const float4 v4 = __ldg(reinterpret_cast<const float4*>(src + (long)gy * p.PW + x0 + lane * 4));
                vs[0] = v4.x; vs[1] = v4.y; vs[2] = v4.z; vs[3] = v4.w;
              } else if constexpr (FASTUP == 4) {
#pragma unroll
                for (int q = 0; q < 4; ++q) vs[q] = up4<kB3DW>(dl + yr[j] * kB3DW + xr[q], xw4[q], yw4[j]);
              } else {
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                  if (j == 0 || !same_rows) {     // (warp-uniform) at scale 3 two of three row pairs share both source rows
                    const float* a0 = dl + yr[j] * kB3DW + xr[q];
                    const float* b0 = a0 + yo[j] * kB3DW;
                    hra[q] = xw0[q] * a0[0] + xw1[q] * a0[xo[q]];
                    hrb[q] = xw0[q] * b0[0] + xw1[q] * b0[xo[q]];
                  }
                  vs[q] = yw0[j] * hra[q] + yw1[j] * hrb[q];
                }
              }
            }
#pragma unroll
            for (int q = 0; q < 4; ++q) d[c][j][q] = fmaf(ws, vs[q], d[c][j][q]);
          }
        }
      }
    }

    // ---- preds_w = hmap * delta (optional output; max(CD, jnd_out) channels, broadcast like `hmaps * preds_w`) and the blend
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const int yl = warp * 2 + j, gy = y0 + yl;
      if (gy < p.H && vfull) {
        const int o = gy * p.W + x0 + lane * 4;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          float pw[4], out[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) pw[q] = d[CD == 1 ? 0 : c][j][q] * (hm_per_channel ? hmc[JIN == 3 ? c : 0][j][q] : hmc[0][j][q]);
          if (p.preds_w != nullptr && c < PC)
            *reinterpret_cast<float4*>(p.preds_w + ((long)f * PC + c) * plane + o) = make_float4(pw[0], pw[1], pw[2], pw[3]);
          const float4 t4 = *reinterpret_cast<const float4*>(rawb + (c * (kB2TH + 4) + yl + 2) * kB2LP + 4 + lane * 4);
          const float in[4] = {t4.x, t4.y, t4.z, t4.w};
          if (p.clamp) {
#pragma unroll
            for (int q = 0; q < 4; ++q) out[q] = __saturatef(fmaf(p.scaling_i, in[q], p.scaling_w * pw[q]));
          } else {
#pragma unroll
            for (int q = 0; q < 4; ++q) out[q] = fmaf(p.scaling_i, in[q], p.scaling_w * pw[q]);
          }
          *reinterpret_cast<float4*>(p.imgs_w + ((long)f * 3 + c) * plane + o) = make_float4(out[0], out[1], out[2], out[3]);
        }
      }
    }
    if (CD * nsrc > 1) fence_proxy_async_smem();   // hand-staged delta tiles (generic proxy) before the next TMA box into the same buffer
    __syncthreads();       // every read of raw[buf] / lum / dl[buf] is done: the next iteration may refill them
  }
}

}  // namespace vsb
