// The DVMark embedder (modules/dvmark.py DVMarkEncoder; models/embedder.py DVMarkEmbedder, build_embedder 'dvmark'): Conv3d layers
// (bias, zero padding) over the key frames of one reference embedder call, [G, 3, S, S] -> [1, 3, T = G, S, S], on x = 2 imgs - 1,
// with the message bits of frame t as K constant planes of 0 / 1:
//   transform_layer  (1,3,3) convs 3 -> 64 -> 64 -> 64, then 3x3x3 64 -> 64, each + ReLU                          at S
//   emb_layer1       [x | msg planes] (64 + K) -> 256 -> 128 -> 128, 3x3x3 + ReLU: x_skip                            at S
//   emb_layer2       [avgpool (1,2,2) of x_skip | msg planes] (128 + K) -> 512 -> 256 -> 256, 3x3x3 + ReLU           at S / 2
//   up               bilinear, align_corners=True (F.upsample_bilinear), S / 2 -> S
//   emb_layer3       [x_skip | up] 384 -> 256 -> 128 (3x3x3 + ReLU) -> 3 (3x3x3), tanh: the delta                    at S
// A sub-batch of B frames holds whole groups of G frames (temporal.cuh same_group); frames of different groups never interact.
//
// Kernels:
//   hidden_c3_kernel (hidden.cuh)     transform_layer.0 on CUDA cores from the planar fp32 frames (x = 2 imgs - 1 folded in).
//   tensor-core 3x3 conv              transform_layer.2 / .4 (bias + ReLU epilogue).
//   add_conv3d_sliced (dvmark.cuh)    every 3x3x3 conv: temporal_stack_kernel + the tensor-core 3x3 conv, in frame slices whose
//                                     stacked operand stays within kDvStackBudget.  transform_layer.6 and emb_layer1.4 write with
//                                     an output pitch straight into their concat buffers.  The output layer runs with N padded to
//                                     16 (zero weight rows) and the conv's fused 1x1 outc epilogue as the identity on its first 3
//                                     columns + tanh, which writes the planar fp32 delta: no fp16 rounding of the pre-tanh value
//                                     and no extra pass (a CUDA-core 128 -> 3 conv would need 10 368 fp32 FMAs per pixel, 1.3 ms
//                                     at 64 x 256^2 at the FP32 peak, on top of reading the same operand).
//   dvmark_planes_kernel              the message planes (exact fp16 0 / 1) and the zero pad channels of a concat buffer, with the
//                                     2x2 average pool of x_skip at S / 2.  The planes are materialised, so the zero padding at map
//                                     borders and group ends is the reference's by construction.
//   dvmark_upsample_kernel            the align_corners=True bilinear up-sample, one block per output row, into the 384 concat.
// Concat pitches are padded to a multiple of 8 channels with zero channels and zero weight columns.
#pragma once
#include "dvmark.cuh"
#include "hidden.cuh"

namespace vsb {

constexpr int kDvEncMaxSize = 512;   // processing sizes above it would need more than ~34 GB at 64 frames (DESIGN row a13f)

// out [B][hw][ld] fp16, channels [c0, ld): frame b's K message bits (msgs + b * msg_stride, exact 0 / 1), then zeros.  With src
// (the 2x2 pool, hw = h * h): channels [0, c0) are the 2x2 mean of src [B][2h][2h] (pitch lds), the four fp16 values summed in fp32
// and rounded once, as temporal_stack_kernel pools.  One 16-byte vector per thread; c0 and ld multiples of 8.
__global__ void __launch_bounds__(256) dvmark_planes_kernel(const uint8_t* __restrict__ msgs, int msg_stride, int K,
                                                            const __half* __restrict__ src, int lds, int h, long hw, int c0, int ld,
                                                            long total, __half* __restrict__ out) {
  const int vpp = (ld - (src ? 0 : c0)) / 8, v0 = src ? 0 : c0 / 8;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const long pix = i / vpp;
    const int c8 = ((int)(i - pix * vpp) + v0) * 8;
    const int b = (int)(pix / hw);
    __align__(16) __half o[8];
    if (c8 < c0) {
      const long p = pix - (long)b * hw;
      const int y = (int)(p / h), xx = (int)(p % h), w2 = 2 * h;
      const __half* s0 = src + (((long)b * w2 + 2 * y) * w2 + 2 * xx) * lds + c8;
      const uint4 u[4] = {__ldg(reinterpret_cast<const uint4*>(s0)), __ldg(reinterpret_cast<const uint4*>(s0 + lds)),
                          __ldg(reinterpret_cast<const uint4*>(s0 + (long)w2 * lds)),
                          __ldg(reinterpret_cast<const uint4*>(s0 + (long)w2 * lds + lds))};
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float s = 0.f;
#pragma unroll
        for (int q = 0; q < 4; ++q) s += __half2float(reinterpret_cast<const __half*>(&u[q])[j]);
        o[j] = __float2half_rn(0.25f * s);
      }
    } else {
      const uint8_t* m = msgs + (long)b * msg_stride;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int k = c8 + j - c0;
        o[j] = __float2half_rn(k < K && m[k] ? 1.f : 0.f);
      }
    }
    *reinterpret_cast<uint4*>(out + pix * ld + c8) = *reinterpret_cast<const uint4*>(o);
  }
}

// out [B][2h][2h] (pitch ldo, channels [0, C)) = bilinear align_corners=True up-sample of x [B][h][h][C] (dense), source coordinates
// as ATen computes them: fp32 scale (h - 1) / (2h - 1), times the output index.  Block = one output row of one frame, thread = one
// 16-byte channel vector of a pixel; the two source rows it reads stay in L1 / L2 for the block.
__global__ void __launch_bounds__(256) dvmark_upsample_kernel(const __half* __restrict__ x, int h, int C, __half* __restrict__ out,
                                                              int ldo) {
  const int OW = 2 * h, y = blockIdx.x, b = blockIdx.y, vpp = C / 8;
  const float scale = (float)(h - 1) / (float)(OW - 1);
  const float ry = scale * (float)y;
  const int y0 = (int)ry, y1 = y0 + (y0 < h - 1 ? 1 : 0);
  const float ly = ry - (float)y0, hy = 1.f - ly;
  const __half* r0 = x + ((long)b * h + y0) * h * C;
  const __half* r1 = x + ((long)b * h + y1) * h * C;
  __half* o = out + ((long)b * OW + y) * OW * ldo;
  for (int i = threadIdx.x; i < OW * vpp; i += blockDim.x) {
    const int ox = i / vpp, c = (i - ox * vpp) * 8;
    const float rx = scale * (float)ox;
    const int x0 = (int)rx, x1 = x0 + (x0 < h - 1 ? 1 : 0);
    const float lx = rx - (float)x0, hx = 1.f - lx;
    const uint4 u00 = __ldg(reinterpret_cast<const uint4*>(r0 + (long)x0 * C + c));
    const uint4 u01 = __ldg(reinterpret_cast<const uint4*>(r0 + (long)x1 * C + c));
    const uint4 u10 = __ldg(reinterpret_cast<const uint4*>(r1 + (long)x0 * C + c));
    const uint4 u11 = __ldg(reinterpret_cast<const uint4*>(r1 + (long)x1 * C + c));
    __align__(16) __half v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float a = __half2float(reinterpret_cast<const __half*>(&u00)[j]), bb = __half2float(reinterpret_cast<const __half*>(&u01)[j]);
      const float cc = __half2float(reinterpret_cast<const __half*>(&u10)[j]), d = __half2float(reinterpret_cast<const __half*>(&u11)[j]);
      v[j] = __float2half_rn(hy * (hx * a + lx * bb) + ly * (hx * cc + lx * d));
    }
    *reinterpret_cast<uint4*>(o + (long)ox * ldo + c) = *reinterpret_cast<const uint4*>(v);
  }
}

struct DVMarkEnc {
  bool on = false;
  int nbits = 0, nsm = 0;
  float *w0 = nullptr, *b0 = nullptr;          // transform_layer.0 in hidden_c3_kernel's [27][64] layout
  ConvW t2, t4;                                // transform_layer.2 / .4 as 3x3 convs
  ConvW t6, e10, e12, e14, e20, e22, e24, e30, e32;   // 3x3x3 convs over the time-stacked operand
  ConvW e34;                                   // emb_layer3.4, N padded to 16
  float *id_w = nullptr, *zero_b = nullptr;    // the identity outc [3][16] and its zero bias

  static int pad8(int c) { return (c + 7) / 8 * 8; }
  int p1() const { return pad8(64 + nbits); }    // pitch of [x | msg planes] at S
  int p2() const { return pad8(128 + nbits); }   // pitch of [pool(x_skip) | msg planes] at S / 2

  // vsb_model_set_dvmark_embedder: the rules (no CUDA calls)
  void set(int nb, const vsb_model_desc& d) {
    VSB_CHECK(nb >= 1, "DVMark embedder: nbits must be at least 1");
    VSB_CHECK(nb == d.nbits, "DVMark embedder: nbits must equal the descriptor's nbits");
    // the half-resolution maps tile the TMA conv by 128 pixels when S is a multiple of 256, else their convs run on the gather loader
    // (setup_conv3x3); above 512 a 64-frame plan outgrows the card (row a13f)
    if (d.img_size < 128 || d.img_size % 128 != 0 || d.img_size > kDvEncMaxSize)
      throw Error("DVMark embedder: processing size " + std::to_string(d.img_size) + " is not implemented (a positive multiple of 128, "
                  "at most " + std::to_string(kDvEncMaxSize) + ")", kErrUnsupported);
    nbits = nb; on = true;
  }

  // checkpoint weight embedder.unet.<key>.weight [cout][cin][kt][3][3], its columns zero-padded to cin_pad and its rows to cout_pad
  static HostTensor conv_w(Weights& ws, const std::string& key, int cin, int cout, int kt, int cin_pad = 0, int cout_pad = 0) {
    const std::string k = "embedder.unet." + key + ".weight";
    const HostTensor& w = ws.get(k);
    VSB_CHECK(w.shape.size() == 5 && w.shape[0] == cout && w.shape[1] == cin && w.shape[2] == kt && w.shape[3] == 3 && w.shape[4] == 3,
              k + ": expected a [" + std::to_string(cout) + "][" + std::to_string(cin) + "][" + std::to_string(kt) +
              "][3][3] Conv3d weight (DVMarkEncoder)");
    const int ci = std::max(cin, cin_pad), co = std::max(cout, cout_pad), per = kt * 9;
    HostTensor t;
    t.shape = {co, ci, kt, 3, 3};
    t.data.assign((size_t)co * ci * per, 0.f);
    for (int n = 0; n < cout; ++n)
      for (int c = 0; c < cin; ++c)
        for (int j = 0; j < per; ++j) t.data[((size_t)n * ci + c) * per + j] = w.data[((size_t)n * cin + c) * per + j];
    return t;
  }
  static std::vector<float> conv_b(Weights& ws, const std::string& key, int cout, int cout_pad = 0) {
    const std::string k = "embedder.unet." + key + ".bias";
    const HostTensor& b = ws.get(k);
    VSB_CHECK(b.numel() == cout, k + ": expected " + std::to_string(cout) + " values");
    std::vector<float> v(b.data);
    v.resize(std::max(cout, cout_pad), 0.f);
    return v;
  }
  ConvW conv3(Weights& ws, const std::string& key, int cin, int cout, int cin_pad = 0, int cout_pad = 0) {
    const HostTensor w = conv_w(ws, key, cin, cout, 3, cin_pad, cout_pad);
    return ws.gemm(conv3d_taps(w, nullptr, temporal_stack_width((int)w.shape[1])), conv_b(ws, key, cout, cout_pad));
  }
  ConvW conv2(Weights& ws, const std::string& key) {   // a (1,3,3) Conv3d as the 3x3 conv it is
    HostTensor w = conv_w(ws, key, 64, 64, 1);
    w.shape = {64, 64, 3, 3};
    return ws.gemm(conv_taps(w), conv_b(ws, key, 64));
  }

  void pack(Weights& ws, int num_sms) {
    nsm = num_sms;
    const int K = nbits;
    {
      const HostTensor w = conv_w(ws, "transform_layer.0", 3, 64, 1);
      std::vector<float> o((size_t)27 * 64);
      for (int n = 0; n < 64; ++n)
        for (int k = 0; k < 27; ++k) o[(size_t)k * 64 + n] = w.data[(size_t)n * 27 + k];   // k = c * 9 + r * 3 + s
      w0 = ws.pool.upload(o);
      b0 = ws.pool.upload(conv_b(ws, "transform_layer.0", 64));
    }
    t2 = conv2(ws, "transform_layer.2");
    t4 = conv2(ws, "transform_layer.4");
    t6 = conv3(ws, "transform_layer.6", 64, 64);
    e10 = conv3(ws, "emb_layer1.0", 64 + K, 256, p1());
    e12 = conv3(ws, "emb_layer1.2", 256, 128);
    e14 = conv3(ws, "emb_layer1.4", 128, 128);
    e20 = conv3(ws, "emb_layer2.0", 128 + K, 512, p2());
    e22 = conv3(ws, "emb_layer2.2", 512, 256);
    e24 = conv3(ws, "emb_layer2.4", 256, 256);
    e30 = conv3(ws, "emb_layer3.0", 384, 256);
    e32 = conv3(ws, "emb_layer3.2", 256, 128);
    e34 = conv3(ws, "emb_layer3.4", 128, 3, 0, 16);
    std::vector<float> id((size_t)3 * 16, 0.f);
    for (int o = 0; o < 3; ++o) id[(size_t)o * 16 + o] = 1.f;
    id_w = ws.pool.upload(id);
    zero_b = ws.pool.upload(std::vector<float>(3, 0.f));
  }

  // the embed plan of B frames at S x S in groups of G -> pl.delta [B][3][S][S].  Buffers by lifetime (2 bytes per channel per pixel):
  // at S a wide map X (max(384, p1) channels: [x | msg planes], later [x_skip | up]), F256 and F128; at S / 2 Y (max(p2, 256):
  // [pool(x_skip) | msg planes], later emb_layer2.2's output) and H (512: emb_layer2.0's, later emb_layer2.4's); the stack slice.
  // keep (test seam, vsb_debug_keep_inputs): every map gets a buffer of its own, so that each step's input stays readable as a tap.
  // Taps: dve.t0 .t2 .t4 (64 at S), dve.cat1 (p1), dve.e1_0 (256), dve.e1_2 (128), dve.cat3 (384), dve.cat2 (p2 at S / 2),
  // dve.e2_0 (512), dve.e2_2 (256), dve.e2_4 (256), dve.e3_0 (256 at S), dve.e3_2 (128), delta.
  void build(Plan& pl, int B, int G, int S, bool keep) const {
    VSB_CHECK(G >= 1, "DVMark embed plan: group length");
    const int h = S / 2, K = nbits, P1 = p1(), P2 = p2();
    const long hw = (long)S * S, hw2 = (long)h * h, M = (long)B * hw, M2 = (long)B * hw2;
    const std::string at = "@" + std::to_string(S), at2 = "@" + std::to_string(h);
    Plan* plp = &pl;
    auto alloc = [&](long n) { return pl.pool.alloc_n<__half>((size_t)n); };
    __half* X = alloc(M * std::max(384, P1));
    __half* F256 = alloc(M * 256);
    __half* F128 = alloc(M * 128);
    __half* Y = alloc(M2 * std::max(P2, 256));
    __half* H = alloc(M2 * 512);
    auto buf = [&](__half* shared, long n) { return keep ? alloc(n) : shared; };
    // each map takes a buffer whose previous tenant the step before it consumed
    __half *t0 = buf(F128, M * 64), *t2o = buf(F256, M * 64), *t4o = buf(F128, M * 64);
    __half *cat1 = buf(X, M * P1), *e10o = buf(F256, M * 256), *e12o = buf(F128, M * 128), *cat3 = buf(X, M * 384);
    __half *cat2 = buf(Y, M2 * P2), *e20o = buf(H, M2 * 512), *e22o = buf(Y, M2 * 256), *e24o = buf(H, M2 * 256);
    __half *e30o = buf(F256, M * 256), *e32o = buf(F128, M * 128);
    // frames per conv launch: the scratch holds the largest slice of any 3x3x3 conv
    struct C3 { int C; int h; };
    const C3 convs[] = {{64, S}, {P1, S}, {256, S}, {128, S}, {P2, h}, {512, h}, {256, h}, {384, S}, {256, S}, {128, S}};
    size_t xs_cap = 0;
    for (const C3& c : convs) {
      const size_t fe = (size_t)c.h * c.h * temporal_stack_width(c.C);
      xs_cap = std::max(xs_cap, (size_t)dv_slice_frames(fe, B) * fe);
    }
    __half* xs = alloc((long)xs_cap);
    pl.delta = pl.pool.alloc_n<float>((size_t)B * 3 * hw);
    const int sms = nsm;
    // ---- transform_layer
    {
      const float *w = w0, *bb = b0;
      const long fstride = 3 * hw;
      pl.add("dvmark_enc.conv1x3x3.3-64" + at, [=](cudaStream_t st) {
        hidden_c3_kernel<<<dim3((unsigned)(hw / kHidPix), B), kHidPix, 0, st>>>(plp->in_imgs, fstride, S, w, bb, nullptr, ACT_RELU, t0);
        VSB_CUDA(cudaGetLastError());
      });
      pl.tap("dve.t0", t0, 1, B, S, S, 64, 64);
    }
    auto conv2d = [&](const ConvW& w, const __half* x, __half* out, const std::string& tap) {
      ConvGemmOp op;
      setup_tma_conv(op, x, B, S, S, 64, 64, 3, 3, 1);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_RELU; op.p.bias = w.bias; op.p.out16 = out; op.p.ld_out16 = 64;
      vsb::add_conv(pl, op, w, "dvmark_enc.conv1x3x3.64-64" + at, nsm);
      pl.tap(tap, out, 1, B, S, S, 64, 64);
    };
    conv2d(t2, t0, t2o, "dve.t2");
    conv2d(t4, t2o, t4o, "dve.t4");
    // a 3x3x3 conv + bias + ReLU over x [B][hh*hh][C] (pitch C) into out (pitch ld)
    auto conv3 = [&](const ConvW& w, const __half* x, int C, int hh, __half* out, int ld) {
      const long hwx = (long)hh * hh;
      const float* bias = w.bias;
      const int fps = dv_slice_frames((size_t)hwx * temporal_stack_width(C), B);
      add_conv3d_sliced<false>(pl, w, x, C, hh, B, G, xs, xs_cap, fps, sms, "dvmark_enc",
                               "dvmark_enc.conv3x3x3." + std::to_string(C) + "-" + std::to_string(w.N) + "@" + std::to_string(hh),
                               [=](ConvGemmOp& op, int bs) {
                                 op.p.epi = EPI_AFFINE; op.p.act = ACT_RELU; op.p.bias = bias;
                                 op.p.out16 = out + bs * hwx * ld; op.p.ld_out16 = ld;
                               });
    };
    // message planes (+ the pool at S / 2) into channels [c0, ld) of `out`
    auto planes = [&](const __half* src, int hh, int c0, int ld, __half* out, const std::string& name) {
      const long hwx = (long)hh * hh, total = (long)B * hwx * ((ld - (src ? 0 : c0)) / 8);
      const long blocks = std::min<long>((total + 255) / 256, (long)sms * 16);
      pl.add(name, [=](cudaStream_t st) {
        dvmark_planes_kernel<<<(unsigned)blocks, 256, 0, st>>>(plp->in_msgs, plp->in_msg_stride, K, src, 384, hh, hwx, c0, ld, total, out);
        VSB_CUDA(cudaGetLastError());
      });
    };
    conv3(t6, t4o, 64, S, cat1, P1);                                 // channels [0, 64) of [x | msg planes]
    planes(nullptr, S, 64, P1, cat1, "dvmark_enc.msg_planes." + std::to_string(P1) + at);
    pl.tap("dve.cat1", cat1, 1, B, S, S, P1, P1);
    // ---- emb_layer1
    conv3(e10, cat1, P1, S, e10o, 256);
    pl.tap("dve.e1_0", e10o, 1, B, S, S, 256, 256);
    conv3(e12, e10o, 256, S, e12o, 128);
    pl.tap("dve.e1_2", e12o, 1, B, S, S, 128, 128);
    conv3(e14, e12o, 128, S, cat3, 384);                             // x_skip: channels [0, 128) of [x_skip | up]
    // ---- emb_layer2 at S / 2
    planes(cat3, h, 128, P2, cat2, "dvmark_enc.pool+msg_planes." + std::to_string(P2) + at2);
    pl.tap("dve.cat2", cat2, 1, B, h, h, P2, P2);
    conv3(e20, cat2, P2, h, e20o, 512);
    pl.tap("dve.e2_0", e20o, 1, B, h, h, 512, 512);
    conv3(e22, e20o, 512, h, e22o, 256);
    pl.tap("dve.e2_2", e22o, 1, B, h, h, 256, 256);
    conv3(e24, e22o, 256, h, e24o, 256);
    pl.tap("dve.e2_4", e24o, 1, B, h, h, 256, 256);
    // ---- up-sample into channels [128, 384) of [x_skip | up]
    pl.add("dvmark_enc.upsample_ac.256" + at, [=](cudaStream_t st) {
      dvmark_upsample_kernel<<<dim3(S, B), 256, 0, st>>>(e24o, h, 256, cat3 + 128, 384);
      VSB_CUDA(cudaGetLastError());
    });
    pl.tap("dve.cat3", cat3, 1, B, S, S, 384, 384);
    // ---- emb_layer3
    conv3(e30, cat3, 384, S, e30o, 256);
    pl.tap("dve.e3_0", e30o, 1, B, S, S, 256, 256);
    conv3(e32, e30o, 256, S, e32o, 128);
    pl.tap("dve.e3_2", e32o, 1, B, S, S, 128, 128);
    {
      // 128 -> 3 (N padded to 16) + bias, then the fused outc epilogue as the identity on columns 0..2 + tanh -> planar fp32 delta
      const float *bias = e34.bias, *idw = id_w, *zb = zero_b;
      float* delta = pl.delta;
      const int fps = dv_slice_frames((size_t)hw * temporal_stack_width(128), B);
      add_conv3d_sliced<false>(pl, e34, e32o, 128, S, B, G, xs, xs_cap, fps, sms, "dvmark_enc", "dvmark_enc.conv3x3x3+tanh.128-3" + at,
                               [=](ConvGemmOp& op, int bs) {
                                 op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = bias;
                                 op.p.outc_w = idw; op.p.outc_b = zb; op.p.n_out = 3; op.p.outc_tanh = 1;
                                 op.p.delta = delta + (long)bs * 3 * hw; op.p.hw = (int)hw;
                               });
    }
    pl.tap("delta", pl.delta, 0, B, 3, S, S, S);
  }
};

}  // namespace vsb
