// The temporal U-Net's own kernels (unet.conv_layer 'conv3d', modules/common.py Conv3dWrapper): a group of G consecutive frames of a
// sub-batch is one reference embedder call, [G, C, H, W] -> [1, C, T = G, H, W], with one zero frame of padding at both ends of the
// group.  A sub-batch of B frames holds whole groups: frames [g*G, min((g+1)*G, B)), so only the last one may be shorter.
//   temporal_stack_kernel      the time taps of a 3x3x3 conv as channels: xs[b, p] = [x[b-1, p] | x[b, p] | x[b+1, p] | 0 ...], a
//                              neighbour outside b's group reading as zeros.  The 3x3x3 conv over x is then the 3x3 conv over xs
//                              (K = 9 * Cs, spatial tap major, then time, then channel), which runs on the tensor-core convs.  It
//                              can stack a slice of the batch's frames, and (POOL) the 2x2 mean of x (the DVMark extractor, dvmark.cuh).
//   unet_first_t_kernel        the `inc` block's first conv as 3x3x3 over 1 or 3 input channels (27 taps) + folded BN + ReLU, and
//                              its 1x1x1 res conv, on CUDA cores (the temporal form of unet_first_kernel).
#pragma once
#include "conv_gemm_host.cuh"

namespace vsb {

// channels of the stacked operand of a C-channel 3x3x3 conv: 3C rounded up to the 64-channel K block of the TMA conv
inline int temporal_stack_width(int C) { return (3 * C + 63) / 64 * 64; }

// frame b + dt lies in frame b's group (groups of G frames from frame 0, B frames in all)
__device__ __forceinline__ bool same_group(int b, int dt, int B, int G) {
  const int t = b + dt;
  return t >= 0 && t < B && t / G == b / G;
}

// xs [n, HW, Cs] fp16 (dense): frames b0 .. b0 + n - 1 of the B-frame batch.  x [B, HW, C] fp16 with pixel pitch ldx, or with POOL
// x [B, 2h, 2h, C] (HW = h * h), stacked as its 2x2 mean (AvgPool3d (1,2,2): the four fp16 values summed in fp32, rounded once).
// C and ldx multiples of 8.  One 16-byte vector per thread.
template <bool POOL>
__global__ void __launch_bounds__(256) temporal_stack_kernel(const __half* __restrict__ x, int ldx, int C, long HW, int h, int b0, int n,
                                                             int B, int G, __half* __restrict__ xs, int Cs) {
  const int vpp = Cs / 8;
  const long total = (long)n * HW * vpp;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long pix = i / vpp;
    const int c8 = (int)(i - pix * vpp) * 8;
    const int b = b0 + (int)(pix / HW), dt = c8 / C, c = c8 - dt * C;
    const long p = pix % HW;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (dt < 3 && same_group(b, dt - 1, B, G)) {
      const int bs = b + dt - 1;
      if (!POOL) {
        v = __ldg(reinterpret_cast<const uint4*>(x + ((long)bs * HW + p) * ldx + c));
      } else {
        const int y = (int)(p / h), xx = (int)(p % h), w2 = 2 * h;
        const __half* s0 = x + (((long)bs * w2 + 2 * y) * w2 + 2 * xx) * ldx + c;
        const uint4 u[4] = {__ldg(reinterpret_cast<const uint4*>(s0)), __ldg(reinterpret_cast<const uint4*>(s0 + ldx)),
                            __ldg(reinterpret_cast<const uint4*>(s0 + (long)w2 * ldx)),
                            __ldg(reinterpret_cast<const uint4*>(s0 + (long)w2 * ldx + ldx))};
        __align__(16) __half o[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float s = 0.f;
#pragma unroll
          for (int q = 0; q < 4; ++q) s += __half2float(reinterpret_cast<const __half*>(&u[q])[j]);
          o[j] = __float2half_rn(0.25f * s);
        }
        v = *reinterpret_cast<const uint4*>(o);
      }
    }
    reinterpret_cast<uint4*>(xs)[i] = v;
  }
}

// frames [b0, b0 + n) of the batch; pool: x is at 2h x 2h and HW = h * h
inline void launch_temporal_stack(const __half* x, int ldx, int C, long HW, int b0, int n, int B, int G, __half* xs, int Cs, int num_sms,
                                  cudaStream_t st, bool pool = false, int h = 0) {
  VSB_CHECK(C % 8 == 0 && ldx % 8 == 0 && Cs % 8 == 0 && Cs >= 3 * C && G >= 1, "temporal stack: channel layout");
  VSB_CHECK(b0 >= 0 && n >= 1 && b0 + n <= B && (!pool || (long)h * h == HW), "temporal stack: frame slice / pooled map");
  const long total = (long)n * HW * (Cs / 8);
  const long blocks = std::min<long>((total + 255) / 256, (long)num_sms * 16);
  if (pool) temporal_stack_kernel<true><<<(unsigned)blocks, 256, 0, st>>>(x, ldx, C, HW, h, b0, n, B, G, xs, Cs);
  else temporal_stack_kernel<false><<<(unsigned)blocks, 256, 0, st>>>(x, ldx, C, HW, h, b0, n, B, G, xs, Cs);
  VSB_CUDA(cudaGetLastError());
}

// imgs [B, 3, H, W] fp32 RGB in [0,1]; x = 2*Y-1 (CIN 1) or 2*rgb-1 (CIN 3) as in unet_first_kernel, zero padded in space and in time.
// h1 = relu(conv3x3x3(x; w1') + b1')  -> NHWC fp16 [B,H,W,Z];  r = conv1x1x1(x; wr) + br -> NHWC fp16 [B,H,W,Z].  w1 is the checkpoint's
// [Z][CIN][3 (t)][3][3] with the BN scale folded per row.  Thread = 4 horizontally adjacent pixels x 8 of every 16 output channels,
// block = 16 rows x 32 columns of one frame; the three frames' input windows are staged in shared memory.  Z % 16 == 0.
template <int CIN>
__global__ void __launch_bounds__(256) unet_first_t_kernel(const float* __restrict__ imgs, int B, int G, int H, int W, int Z,
                                                           const float* __restrict__ w1, const float* __restrict__ b1,
                                                           const float* __restrict__ wr, const float* __restrict__ br,
                                                           __half* __restrict__ h1, __half* __restrict__ res) {
  constexpr int NP = 4, TW = 8 * NP, TH = 16;
  __shared__ float tile[3][CIN][TH + 2][TW + 2 + 2];
  const int zh = threadIdx.x & 1, tx = (threadIdx.x >> 1) & 7, ty = threadIdx.x >> 4;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH, b = blockIdx.z;
  for (int i = threadIdx.x; i < 3 * (TH + 2) * (TW + 2); i += 256) {
    const int dt = i / ((TH + 2) * (TW + 2)), j = i - dt * (TH + 2) * (TW + 2);
    const int ly = j / (TW + 2), lx = j - ly * (TW + 2);
    const int gy = y0 + ly - 1, gx = x0 + lx - 1;
    const bool in = gy >= 0 && gy < H && gx >= 0 && gx < W && same_group(b, dt - 1, B, G);
    const float* img = imgs + (long)(in ? b + dt - 1 : b) * 3 * H * W;
    if (CIN == 1) {
      float v = 0.f;
      if (in) {
        const long o = (long)gy * W + gx;
        const float y = 0.299f * __ldg(img + o) + 0.587f * __ldg(img + (long)H * W + o) + 0.114f * __ldg(img + 2L * H * W + o);
        v = 2.f * y - 1.f;
      }
      tile[dt][0][ly][lx] = v;
    } else {
#pragma unroll
      for (int c = 0; c < CIN; ++c) tile[dt][c][ly][lx] = in ? 2.f * __ldg(img + (long)c * H * W + (long)gy * W + gx) - 1.f : 0.f;
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
    for (int dt = 0; dt < 3; ++dt) {
#pragma unroll
      for (int c = 0; c < CIN; ++c) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          float xr[NP + 2];
#pragma unroll
          for (int s = 0; s < NP + 2; ++s) xr[s] = tile[dt][c][ty + r][tx * NP + s];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const float wv = __ldg(w1 + (((z0 + q) * CIN + c) * 3 + dt) * 9 + r * 3 + s);
#pragma unroll
              for (int p = 0; p < NP; ++p) a[q][p] = fmaf(xr[p + s], wv, a[q][p]);
            }
            if (dt == 1 && r == 1) {
              const float wv = __ldg(wr + (z0 + q) * CIN + c);
#pragma unroll
              for (int p = 0; p < NP; ++p) rr[q][p] = fmaf(xr[p + 1], wv, rr[q][p]);
            }
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

inline void launch_unet_first_t(const float* src, int B, int G, int S, int Z, int cin, const float* w1, const float* b1, const float* wr,
                                const float* br, __half* h1, __half* r0, cudaStream_t st) {
  VSB_CHECK(Z % 16 == 0 && G >= 1, "temporal first layer: Z % 16 == 0");
  const dim3 grid((S + 31) / 32, (S + 15) / 16, B);
  if (cin == 1) unet_first_t_kernel<1><<<grid, 256, 0, st>>>(src, B, G, S, S, Z, w1, b1, wr, br, h1, r0);
  else unet_first_t_kernel<3><<<grid, 256, 0, st>>>(src, B, G, S, S, Z, w1, b1, wr, br, h1, r0);
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
