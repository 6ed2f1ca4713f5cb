// The DVMark extractor (modules/dvmark.py DVMarkDecoder; models/extractor.py build_extractor 'dvmark'): four 3x3x3 Conv3d (zero
// padding 1 in space and time, bias) over the frames of one reference detector call, [G, 3, S, S] -> [1, 3, T = G, S, S], on the
// frames in [0, 1] (no preprocess):
//   layer1 3 -> 128, ReLU, layer2 128 -> 128, ReLU, avgpool (1,2,2), layer3 128 -> 256, ReLU, avgpool (1,2,2), layer4 256 -> 1 + K,
//   then the mean over the S/4 x S/4 map: the pooled logits [G, 1 + K].
// A detect sub-batch of B frames holds whole groups of G frames (frames [g G, min((g + 1) G, B))); frames of different groups never
// interact (same_group, temporal.cuh).
//
// Kernels:
//   dvmark_first_kernel   layer1 (K = 81) on CUDA cores from the planar fp32 frames -> NHWC fp16.
//   temporal_stack_kernel (temporal.cuh)   the time taps of a 3x3x3 conv as channels [x(t-1) | x(t) | x(t+1)] for a slice of the
//                         frames, with layer3's (1,2,2) average pool fused (POOL); the 3x3 tensor-core conv over that operand is the 3x3x3 conv (layer2, layer3; bias + ReLU in
//                         its epilogue).  The stacked operand of one conv launch is bounded by kDvStackBudget: a conv runs over
//                         slices of frames, so the scratch does not grow with the batch (at 256^2 a 64-frame operand would take
//                         3 GiB, at 768^2 27 GiB).
//   dvmark_rowsum_kernel, dvmark_head_kernel   layer4 and the spatial mean together.  The mean of a zero-padded 3x3x3 conv is, per
//                         time tap and spatial tap (r, s), the weight times the sum of its input over the window that tap reads:
//                         the whole map minus its last / first row (r = 0 / 2) and last / first column (s = 0 / 2).  So the head
//                         needs, per frame and channel, the sums of every row and of the first and last columns of the pooled
//                         layer3 map (rowsum: one block per row, pooled on the fly), and then 27 x 256 weights per logit.  Every
//                         sum runs in a fixed order with plain stores: the logits are bit-identical run to run.
#pragma once
#include "temporal.cuh"
#include "weights.cuh"

namespace vsb {

constexpr int kDvC1 = 128, kDvC3 = 256;            // widths of layers 1-2 and of layer 3
constexpr size_t kDvStackBudget = (size_t)512 << 20;   // bytes of time-stacked operand per conv launch

// layer1: imgs [B][3][S][S] fp32, out = relu(conv3x3x3(imgs; w) + b) -> NHWC fp16 [B][S][S][128].  w is the checkpoint's
// [128][3][3 (t)][3][3].  Thread = 4 horizontally adjacent pixels x 8 of every 16 output channels, block = 16 rows x 32 columns of one
// frame; the three frames' input windows are staged in shared memory.
__global__ void __launch_bounds__(256) dvmark_first_kernel(const float* __restrict__ imgs, int B, int G, int S,
                                                           const float* __restrict__ w, const float* __restrict__ bias,
                                                           __half* __restrict__ out) {
  constexpr int NP = 4, TW = 8 * NP, TH = 16;
  __shared__ float tile[3][3][TH + 2][TW + 2 + 2];
  const int zh = threadIdx.x & 1, tx = (threadIdx.x >> 1) & 7, ty = threadIdx.x >> 4;
  const int x0 = blockIdx.x * TW, y0 = blockIdx.y * TH, b = blockIdx.z;
  for (int i = threadIdx.x; i < 3 * (TH + 2) * (TW + 2); i += 256) {
    const int dt = i / ((TH + 2) * (TW + 2)), j = i - dt * (TH + 2) * (TW + 2);
    const int ly = j / (TW + 2), lx = j - ly * (TW + 2);
    const int gy = y0 + ly - 1, gx = x0 + lx - 1;
    const bool in = gy >= 0 && gy < S && gx >= 0 && gx < S && same_group(b, dt - 1, B, G);
    const float* img = imgs + (long)(in ? b + dt - 1 : b) * 3 * S * S;
#pragma unroll
    for (int c = 0; c < 3; ++c) tile[dt][c][ly][lx] = in ? __ldg(img + (long)c * S * S + (long)gy * S + gx) : 0.f;
  }
  __syncthreads();
  const int gx = x0 + tx * NP, gy = y0 + ty;
  const long pix = ((long)b * S + gy) * S + gx;
  for (int zb = 0; zb < kDvC1; zb += 16) {
    const int z0 = zb + 8 * zh;
    float a[8][NP];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const float bz = __ldg(bias + z0 + q);
#pragma unroll
      for (int p = 0; p < NP; ++p) a[q][p] = bz;
    }
#pragma unroll
    for (int dt = 0; dt < 3; ++dt) {
#pragma unroll
      for (int c = 0; c < 3; ++c) {
#pragma unroll
        for (int r = 0; r < 3; ++r) {
          float xr[NP + 2];
#pragma unroll
          for (int s = 0; s < NP + 2; ++s) xr[s] = tile[dt][c][ty + r][tx * NP + s];
#pragma unroll
          for (int q = 0; q < 8; ++q) {
#pragma unroll
            for (int s = 0; s < 3; ++s) {
              const float wv = __ldg(w + (((z0 + q) * 3 + c) * 3 + dt) * 9 + r * 3 + s);
#pragma unroll
              for (int p = 0; p < NP; ++p) a[q][p] = fmaf(xr[p + s], wv, a[q][p]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int p = 0; p < NP; ++p) {
      __align__(16) __half ho[8];
#pragma unroll
      for (int q = 0; q < 8; ++q) ho[q] = __float2half_rn(fmaxf(a[q][p], 0.f));
      *reinterpret_cast<uint4*>(out + (pix + p) * kDvC1 + z0) = *reinterpret_cast<const uint4*>(ho);
    }
  }
}

// part [B][h][3][256]: for row y of the 2x2-pooled layer3 map (h x h, pooled from x [B][2h][2h][256] fp16 as in temporal_stack_kernel
// but kept in fp32): the row's sum, its first and its last value, per channel.  Block = one row of one frame, thread = channel.
__global__ void __launch_bounds__(kDvC3) dvmark_rowsum_kernel(const __half* __restrict__ x, int h, float* __restrict__ part) {
  const int y = blockIdx.x, b = blockIdx.y, c = threadIdx.x, w2 = 2 * h;
  const __half* row = x + (((long)b * w2 + 2 * y) * w2) * kDvC3 + c;
  float sum = 0.f, first = 0.f, last = 0.f;
  for (int xx = 0; xx < h; ++xx) {
    const __half* s0 = row + (long)2 * xx * kDvC3;
    const float v = 0.25f * (__half2float(s0[0]) + __half2float(s0[kDvC3]) + __half2float(s0[(long)w2 * kDvC3]) +
                             __half2float(s0[(long)w2 * kDvC3 + kDvC3]));
    sum += v;
    if (xx == 0) first = v;
    if (xx == h - 1) last = v;
  }
  float* o = part + (((long)b * h + y) * 3) * kDvC3 + c;
  o[0] = sum; o[kDvC3] = first; o[2 * kDvC3] = last;
}

// logits [B][NO]: layer4 (w4 [NO][27][256], (dt, r, s) major, bias b4) over the pooled layer3 map, averaged over its h x h pixels.
// ws[dt][r*3+s][c] = sum of channel c of frame b + dt - 1 over the window tap (r, s) reads (zero outside b's group); then one warp
// per logit: lanes over the 27 x 256 products, a fixed shuffle tree.
__global__ void __launch_bounds__(kDvC3) dvmark_head_kernel(const float* __restrict__ part, int h, int B, int G,
                                                            const float* __restrict__ w4, const float* __restrict__ b4, int NO,
                                                            float* __restrict__ ws_out, float* __restrict__ logits) {
  __shared__ float ws[27 * kDvC3];
  const int b = blockIdx.x, c = threadIdx.x;
  for (int dt = 0; dt < 3; ++dt) {
    float win[9];
    if (same_group(b, dt - 1, B, G)) {
      const float* pf = part + ((long)(b + dt - 1) * h * 3) * kDvC3 + c;
      float T = 0.f, C0 = 0.f, CL = 0.f;
      for (int y = 0; y < h; ++y) { T += pf[(long)y * 3 * kDvC3]; C0 += pf[((long)y * 3 + 1) * kDvC3]; CL += pf[((long)y * 3 + 2) * kDvC3]; }
      const float R0 = pf[0], RL = pf[((long)(h - 1) * 3) * kDvC3];
      const float f0 = pf[kDvC3], l0 = pf[2 * kDvC3];                                                       // row 0: first, last
      const float fL = pf[((long)(h - 1) * 3 + 1) * kDvC3], lL = pf[((long)(h - 1) * 3 + 2) * kDvC3];        // last row
      // tap (r, s) leaves out the last row (r = 0) or the first (r = 2), and the last column (s = 0) or the first (s = 2)
      const float row_out[3] = {RL, 0.f, R0}, col_out[3] = {CL, 0.f, C0};
      const float corner[3][3] = {{lL, 0.f, fL}, {0.f, 0.f, 0.f}, {l0, 0.f, f0}};
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s) win[r * 3 + s] = T - row_out[r] - col_out[s] + corner[r][s];
    } else {
#pragma unroll
      for (int k = 0; k < 9; ++k) win[k] = 0.f;
    }
#pragma unroll
    for (int k = 0; k < 9; ++k) ws[(dt * 9 + k) * kDvC3 + c] = win[k];
  }
  __syncthreads();
  if (ws_out)
    for (int j = c; j < 27 * kDvC3; j += kDvC3) ws_out[(long)b * 27 * kDvC3 + j] = ws[j];
  const int lane = c & 31, warp = c >> 5;
  const float inv = 1.f / ((float)h * (float)h);
  for (int n = warp; n < NO; n += kDvC3 / 32) {
    const float* wr = w4 + (long)n * 27 * kDvC3;
    float a = 0.f;
    for (int j = lane; j < 27 * kDvC3; j += 32) a = fmaf(__ldg(wr + j), ws[j], a);
#pragma unroll
    for (int o = 16; o; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    if (lane == 0) logits[(long)b * NO + n] = __ldg(b4 + n) + a * inv;
  }
}

// frames of one conv launch whose stacked operand (frame_elems fp16 values per frame) stays within kDvStackBudget, at least one
inline int dv_slice_frames(size_t frame_elems, int B) {
  return (int)std::max<size_t>(1, std::min<size_t>(B, kDvStackBudget / (frame_elems * sizeof(__half))));
}

// A 3x3x3 conv over the time taps of x [B][h*h][C] (pitch C; POOL: of the 2x2 mean of x [B][2h][2h][C]) at h x h, in groups of G:
// per slice of at most `fps` frames, temporal_stack_kernel into xs (xs_cap fp16 values), then the tensor-core 3x3 conv over xs,
// whose epilogue `epi(op, b0)` sets for the slice that starts at frame b0.  The DVMark extractor and embedder share it.
template <bool POOL, class Epi>
void add_conv3d_sliced(Plan& pl, const ConvW& w, const __half* x, int C, int h, int B, int G, __half* xs, size_t xs_cap, int fps,
                       int nsm, const std::string& unit, const std::string& name, Epi epi) {
  const int Cs = temporal_stack_width(C);
  const long hw = (long)h * h;
  VSB_CHECK((size_t)fps * hw * Cs <= xs_cap, "DVMark: a frame slice's stacked operand exceeds its scratch buffer");
  for (int b0 = 0; b0 < B; b0 += fps) {
    const int n = std::min(fps, B - b0);
    pl.add(unit + ".tstack" + std::string(POOL ? "+pool." : ".") + std::to_string(C) + "-" + std::to_string(Cs) + "@" + std::to_string(h),
           [=](cudaStream_t st) { launch_temporal_stack(x, C, C, hw, b0, n, B, G, xs, Cs, nsm, st, POOL, h); });
    ConvGemmOp op;
    setup_conv3x3(op, xs, n, h, Cs, Cs);
    epi(op, b0);
    vsb::add_conv(pl, op, w, name, nsm);
  }
}

struct DVMark {
  bool on = false;
  int nbits = 0, nsm = 0;
  float *w1 = nullptr, *b1 = nullptr;   // layer1 as the checkpoint holds it
  ConvW c2, c3;                         // layers 2-3 as 3x3 convs over the time-stacked operand
  float *w4 = nullptr, *b4 = nullptr;   // layer4 [1 + K][27][256]

  // vsb_model_set_dvmark_extractor: the rules (no CUDA calls)
  void set(int nb, const vsb_model_desc& d) {
    VSB_CHECK(nb >= 1, "DVMark extractor: nbits must be at least 1");
    VSB_CHECK(nb == d.nbits, "DVMark extractor: nbits must equal the descriptor's nbits");
    // layer2's map (S) tiles the TMA conv by 128 pixels; layer3's (S / 2) does only when S is a multiple of 256, else it runs on the
    // gather loader (setup_conv3x3); layer4's (S / 4) has a row of its own per block
    if (d.img_size < 128 || d.img_size % 128 != 0)
      throw Error("DVMark extractor: processing size " + std::to_string(d.img_size) + " is not implemented (a positive multiple of 128)",
                  kErrUnsupported);
    nbits = nb; on = true;
  }

  // a group of G frames (one reference detector call) must fit one 64-frame sub-batch
  static int group(int G, int max_batch) {
    VSB_CHECK(G >= 1, "DVMark extractor: the detect group length must be at least 1");
    if (G > max_batch)
      throw Error("DVMark extractor: a group of " + std::to_string(G) + " frames convolved together (one video chunk, or the whole "
                  "batch in image mode) does not fit one " + std::to_string(max_batch) + "-frame sub-batch; at most " +
                  std::to_string(max_batch) + " are implemented", kErrUnsupported);
    return G;
  }

  const HostTensor& conv_w(Weights& ws, int i, int cin, int cout) const {
    const std::string k = "detector.layers.layer" + std::to_string(i) + ".weight";
    const HostTensor& w = ws.get(k);
    VSB_CHECK(w.shape.size() == 5 && w.shape[0] == cout && w.shape[1] == cin && w.shape[2] == 3 && w.shape[3] == 3 && w.shape[4] == 3,
              k + ": expected a [" + std::to_string(cout) + "][" + std::to_string(cin) + "][3][3][3] Conv3d weight (DVMarkDecoder)");
    return w;
  }
  std::vector<float> conv_b(Weights& ws, int i, int cout) const {
    const std::string k = "detector.layers.layer" + std::to_string(i) + ".bias";
    const HostTensor& b = ws.get(k);
    VSB_CHECK(b.numel() == cout, k + ": expected " + std::to_string(cout) + " values");
    return b.data;
  }

  void pack(Weights& ws, int num_sms) {
    nsm = num_sms;
    const int NO = 1 + nbits;
    w1 = ws.pool.upload(conv_w(ws, 1, 3, kDvC1).data);
    b1 = ws.pool.upload(conv_b(ws, 1, kDvC1));
    c2 = ws.gemm(conv3d_taps(conv_w(ws, 2, kDvC1, kDvC1), nullptr, temporal_stack_width(kDvC1)), conv_b(ws, 2, kDvC1));
    c3 = ws.gemm(conv3d_taps(conv_w(ws, 3, kDvC1, kDvC3), nullptr, temporal_stack_width(kDvC1)), conv_b(ws, 3, kDvC3));
    const HostTensor& w = conv_w(ws, 4, kDvC3, NO);
    std::vector<float> p((size_t)NO * 27 * kDvC3);
    for (int n = 0; n < NO; ++n)
      for (int c = 0; c < kDvC3; ++c)
        for (int k = 0; k < 27; ++k) p[((size_t)n * 27 + k) * kDvC3 + c] = w.data[((size_t)n * kDvC3 + c) * 27 + k];
    w4 = ws.pool.upload(p);
    b4 = ws.pool.upload(conv_b(ws, 4, NO));
  }

  // layer2 / layer3: bias + ReLU -> out [B][h*h][N]
  template <bool POOL>
  void add_conv3d(Plan& pl, const ConvW& w, const __half* x, int C, int h, int B, int G, __half* xs, size_t xs_cap, int fps,
                  __half* out, const std::string& name) const {
    const long hw = (long)h * h;
    const float* bias = w.bias;
    const int N = w.N;
    add_conv3d_sliced<POOL>(pl, w, x, C, h, B, G, xs, xs_cap, fps, nsm, "dvmark", name, [=](ConvGemmOp& op, int b0) {
      op.p.epi = EPI_AFFINE; op.p.act = ACT_RELU; op.p.bias = bias; op.p.out16 = out + b0 * hw * N; op.p.ld_out16 = N;
    });
  }

  // the detect plan of B frames at S x S in groups of G -> pl.logits [B][1 + nbits].  Taps: dvm.l1, dvm.l2 (NHWC fp16 at S), dvm.l3
  // (at S / 2), dvm.rows (the row sums, fp32 [B][S/4][3][256]), dvm.win (the window sums the head read, fp32 [B][27][256]).
  void build(Plan& pl, int B, int G, int S) const {
    VSB_CHECK(G >= 1, "DVMark detect plan: group length");
    const int h2 = S / 2, h4 = S / 4, NO = 1 + nbits;
    const long hw = (long)S * S, hw2 = (long)h2 * h2;
    const Plan* plp = &pl;
    __half* l1 = pl.pool.alloc_n<__half>((size_t)B * hw * kDvC1);
    __half* l2 = pl.pool.alloc_n<__half>((size_t)B * hw * kDvC1);
    __half* l3 = pl.pool.alloc_n<__half>((size_t)B * hw2 * kDvC3);
    // frames per conv launch: as many as the budget holds (at least one); the scratch fits the larger of the two layers' slices
    const size_t frame2 = (size_t)hw * temporal_stack_width(kDvC1), frame3 = (size_t)hw2 * temporal_stack_width(kDvC1);
    const int fps2 = dv_slice_frames(frame2, B), fps3 = dv_slice_frames(frame3, B);
    const size_t xs_cap = std::max((size_t)fps2 * frame2, (size_t)fps3 * frame3);
    __half* xs = pl.pool.alloc_n<__half>(xs_cap);
    const std::string at = "@" + std::to_string(S);
    const float *w1_ = w1, *b1_ = b1;
    pl.add("dvmark.conv3x3x3.3-128" + at, [=](cudaStream_t st) {
      dvmark_first_kernel<<<dim3(S / 32, S / 16, B), 256, 0, st>>>(plp->in_imgs, B, G, S, w1_, b1_, l1);
      VSB_CUDA(cudaGetLastError());
    });
    pl.tap("dvm.l1", l1, 1, B, S, S, kDvC1, kDvC1);
    add_conv3d<false>(pl, c2, l1, kDvC1, S, B, G, xs, xs_cap, fps2, l2, "dvmark.conv3x3x3.128-128" + at);
    pl.tap("dvm.l2", l2, 1, B, S, S, kDvC1, kDvC1);
    add_conv3d<true>(pl, c3, l2, kDvC1, h2, B, G, xs, xs_cap, fps3, l3, "dvmark.conv3x3x3.128-256@" + std::to_string(h2));
    pl.tap("dvm.l3", l3, 1, B, h2, h2, kDvC3, kDvC3);
    float* rows = pl.pool.alloc_n<float>((size_t)B * h4 * 3 * kDvC3);
    float* win = pl.pool.alloc_n<float>((size_t)B * 27 * kDvC3);
    const float *w4_ = w4, *b4_ = b4;
    float* logits = pl.logits;
    pl.add("dvmark.pool+conv3x3x3+mean.256-" + std::to_string(NO) + "@" + std::to_string(h4), [=](cudaStream_t st) {
      dvmark_rowsum_kernel<<<dim3(h4, B), kDvC3, 0, st>>>(l3, h4, rows);
      dvmark_head_kernel<<<B, kDvC3, 0, st>>>(rows, h4, B, G, w4_, b4_, NO, win, logits);
      VSB_CUDA(cudaGetLastError());
    }, 2);
    pl.tap("dvm.rows", rows, 0, B, h4, 3, kDvC3, kDvC3);
    pl.tap("dvm.win", win, 0, B, 27, 1, kDvC3, kDvC3);
  }
};

}  // namespace vsb
