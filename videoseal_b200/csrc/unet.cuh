// The U-Net embedder (modules/unet.py, BatchNorm + ReLU blocks): its rules and the kernel of every layer, its packed weights and its
// embed plan.  A temporal U-Net (`temporal`, conv_layer 'conv3d') differs in the ResnetBlocks only: their 3x3 convs are 3x3x3 over
// the frames of a group (temporal.cuh; the first one on CUDA cores, the others as the tensor-core 3x3 conv over the time-stacked
// operand, never the direct ring conv) and their res_conv is 1x1x1, i.e. an ordinary 1x1 conv.
#pragma once
#include "pointwise_host.cuh"
#include "temporal.cuh"
#include "weights.cuh"

namespace vsb {

constexpr size_t kUpGatherSmem = 160 * 1024;   // tiling cap of the up-conv gather kernels

struct UNet {
  // ---- the kernel of every layer at the map width it runs at, chosen once by check.  pack packs only the weights that kernel
  // reads, and build follows them: ConvW::wd (direct ring conv) or ::w (tensor-core GEMM), down_conv[i].wd (space-to-depth ring
  // conv) or .w (gather GEMM), up_phase_w[j] (phase-folded ring conv + border fix) or up_conv[j] (tap GEMM + gather with `vpt`
  // 16-byte channel vectors per thread, tiled when smem > 0).
  struct ResBlockK { bool res, c1, c2; };   // true: the direct ring conv
  struct UpK { bool phase; int vpt; size_t smem; };
  bool inc_k = false;
  std::vector<bool> down_k;
  std::vector<ResBlockK> down_rb_k, up_rb_k;
  ResBlockK bott_rb_k{};
  std::vector<UpK> up_k;

  // ---- packed weights
  struct ResBlockW { ConvW c1, c2, res; };
  float *first_w1 = nullptr, *first_b1 = nullptr, *first_wr = nullptr, *first_br = nullptr;  // inc (CUDA-core layer)
  ConvW inc_c2;
  std::vector<ConvW> down_conv;
  std::vector<ResBlockW> down_rb, bott_rb, up_rb;
  std::vector<ConvW> up_conv;
  std::vector<float*> up_lnw, up_lnb;
  std::vector<__half*> up_phase_w;   // per level: phase-folded weights (direct layout) or nullptr
  std::vector<float*> up_border_w;   // per level: fp32 taps [9][Cout][Ct] for the border fix-up, or nullptr
  float *outc_w = nullptr, *outc_b = nullptr;
  float* msg_table = nullptr;

  vsb_model_desc d{};
  bool temporal = false;   // conv_layer 'conv3d' (vsb_model_set_unet_temporal)
  int nsm = 0;   // SMs of the model's device

  // vsb_model_create: the U-Net's rules (no CUDA calls)
  void check(const vsb_model_desc& desc) {
    d = desc;
    if (d.unet_act != 0 || d.unet_norm != 0) throw Error("unsupported card: only BatchNorm+ReLU U-Nets are implemented on the GPU path", kErrUnsupported);
    VSB_CHECK(d.unet_levels >= 2 && d.unet_levels <= 6, "unet levels");
    VSB_CHECK(d.unet_in_ch == 1 || d.unet_in_ch == 3, "unet in_channels must be 1 or 3");
    VSB_CHECK(d.unet_out_ch >= 1 && d.unet_out_ch <= 3, "unet out_channels must be <= 3");
    VSB_CHECK((d.yuv != 0) == (d.unet_in_ch == 1), "yuv cards use 1 input channel");
    const int S = d.img_size, L = d.unet_levels;
    const int* z = d.unet_z;
    for (int i = 0; i < L; ++i) {
      // widths the kernels implement: 8 (a leading run of levels, not the last: the direct conv's 8-channel instantiations),
      // 16, 32 and multiples of 64
      const bool ok8 = z[i] == 8 && i < L - 1 && (i == 0 || z[i - 1] == 8);
      if (!(ok8 || z[i] == 16 || z[i] == 32 || (z[i] > 0 && z[i] % 64 == 0)))
        throw Error("U-Net width " + std::to_string(z[i]) + " at level " + std::to_string(i) + " is not implemented (8 in the "
                    "leading levels, 16, 32 or a multiple of 64)", kErrUnsupported);
    }
    // the time-stacked operand of a 3x3x3 conv feeds the TMA conv, which has no 8-channel form
    if (temporal)
      for (int i = 0; i < L; ++i)
        if (z[i] < 16)
          throw Error("temporal U-Net width " + std::to_string(z[i]) + " at level " + std::to_string(i) + " is not implemented (16, 32 or "
                      "a multiple of 64)", kErrUnsupported);
    // the tensor-core convs tile maps by 128 pixels
    if ((S >> (L - 1)) < 16)
      throw Error("img_size=" + std::to_string(S) + ": the U-Net's " + std::to_string(L) + " levels leave a " +
                  std::to_string(S >> (L - 1)) + "-pixel bottleneck map; at least 16 is implemented", kErrUnsupported);
    // policy, also where the 8-channel rings would still fit: unet_tiny_yuv_quant's first ring to overflow is at 896
    if (z[0] == 8 && S > 768)
      throw Error("img_size=" + std::to_string(S) + ": an 8-channel U-Net runs at processing sizes up to 768", kErrUnsupported);
    VSB_CHECK(S % 128 == 0, "processing size must be a multiple of 128");
    VSB_CHECK(d.hidden % 8 == 0, "hidden must be a multiple of 8");
  }
  // the kernel of every layer (no CUDA calls); after the model's other descriptor rules
  void choose_kernels() {
    const int S = d.img_size, L = d.unet_levels, zb = d.unet_z[L - 1] + d.hidden;
    const int* z = d.unet_z;
    // 8-channel layers have no GEMM path: where their ring does not fit, the model is not implemented
    auto ring8 = [](bool ring, int C, int W) {
      if (C == 8 && !ring)
        throw Error("8-channel layer on a " + std::to_string(W) + "-wide map: the direct conv's ring does not fit (processing size "
                    "too large for an 8-channel U-Net)", kErrUnsupported);
      return ring;
    };
    // ResnetBlock of C channels on a W-wide map; dense_out: its output has pitch C (the last down level writes the concat buffer)
    auto resblock = [&](int C, int W, bool dense_out) {
      if (temporal) return ResBlockK{conv3_direct_ok(C, C, W, 1), false, false};
      return ResBlockK{ring8(conv3_direct_ok(C, C, W, 1), C, W), ring8(conv3_direct_ok(C, C, W), C, W),
                       ring8(dense_out && conv3_direct_ok(C, C, W), C, W)};
    };
    inc_k = !temporal && ring8(conv3_direct_ok(z[0], z[0], S), z[0], S);
    for (int i = 0; i < L - 1; ++i) {
      down_k.push_back(ring8(conv3_direct_s2d_ok(z[i], z[i + 1], S >> (i + 1)), z[i + 1], S >> (i + 1)));
      down_rb_k.push_back(resblock(z[i + 1], S >> (i + 1), i < L - 2));
    }
    bott_rb_k = resblock(zb, S >> (L - 1), true);
    for (int ii = L - 2; ii >= 0; --ii) {
      const int hs = S >> (ii + 1), Cin = ii == L - 2 ? zb : z[ii + 1], Cout = z[ii];
      UpK k{Cout == 16 && 2 * Cin == 64 && conv3_direct_ok(64, 64, hs), 0, 0};
      if (!k.phase) {
        // Cout / (8 * vpt) threads per output pixel, a power of two <= 32: VPT 2 only above 256 channels, which no shipped card has
        // (chunkyseal's widest up block outputs 256)
        k.vpt = Cout <= 256 ? 1 : 2;
        const int g = Cout / (8 * k.vpt);
        if (Cout % (8 * k.vpt) != 0 || g > 32 || (g & (g - 1)) != 0)
          throw Error("U-Net up-conv to " + std::to_string(Cout) + " channels is not implemented (8 * 2^k, at most 512)", kErrUnsupported);
        // low-resolution taps of a 16 x 16 output tile staged in shared memory (ups_gather_ln_tiled_kernel) when they fit
        k.smem = hs % 8 == 0 && ups_tile_smem(2, Cout) <= kUpGatherSmem ? ups_tile_smem(2, Cout) : 0;
      }
      up_k.push_back(k);
      up_rb_k.push_back(resblock(Cout, 2 * hs, true));
    }
  }

  static bool use_halo(int C) { return C <= 16; }
  // a conv (3x3 or 1x1, stride 1) in the layout its kernel reads: the direct ring conv's, or the GEMM's (for 3x3 convs up to 16
  // input channels, the halo loader's)
  static ConvW pack_conv(Weights& ws, const std::string& wkey, const std::vector<float>* out_scale, const std::vector<float>& bias, bool direct) {
    return pack_taps(ws, ws.taps(wkey, out_scale), bias, direct);
  }
  static ConvW pack_taps(Weights& ws, const Taps& t, const std::vector<float>& bias, bool direct) {
    if (!direct) return t.R == 3 && use_halo(t.C) ? ws.halo(t, bias) : ws.gemm(t, bias);
    ConvW cw;
    cw.N = t.N;
    cw.wd = ws.direct(t);
    return ws.with_bias(cw, bias);
  }
  // a temporal ResnetBlock: Conv3dWrapper keys (`.conv.` inside), 5-D weights
  static ResBlockW pack_resblock3d(Weights& ws, const std::string& key, const ResBlockK& k) {
    auto conv = [&](const std::string& wkey, const std::vector<float>* s, const std::vector<float>& b, bool direct) {
      const HostTensor& w = ws.get(wkey);
      VSB_CHECK(w.shape.size() == 5, wkey + ": a temporal U-Net needs 5-D Conv3d weights");
      return pack_taps(ws, conv3d_taps(w, s, temporal_stack_width((int)w.shape[1])), b, direct);
    };
    ResBlockW rb;
    std::vector<float> s, b;
    ws.bn_fold(key + ".double_conv.1", s, b);
    rb.c1 = conv(key + ".double_conv.0.conv.weight", &s, b, false);
    ws.bn_fold(key + ".double_conv.4", s, b);
    rb.c2 = conv(key + ".double_conv.3.conv.weight", &s, b, false);
    rb.res = conv(key + ".res_conv.conv.weight", nullptr, ws.get(key + ".res_conv.conv.bias").data, k.res);
    return rb;
  }
  ResBlockW pack_block(Weights& ws, const std::string& key, const ResBlockK& k) const {
    return temporal ? pack_resblock3d(ws, key, k) : pack_resblock(ws, key, k);
  }
  static ResBlockW pack_resblock(Weights& ws, const std::string& key, const ResBlockK& k) {
    ResBlockW rb;
    std::vector<float> s, b;
    ws.bn_fold(key + ".double_conv.1", s, b);
    rb.c1 = pack_conv(ws, key + ".double_conv.0.weight", &s, b, k.c1);
    ws.bn_fold(key + ".double_conv.4", s, b);
    rb.c2 = pack_conv(ws, key + ".double_conv.3.weight", &s, b, k.c2);
    rb.res = pack_conv(ws, key + ".res_conv.weight", nullptr, ws.get(key + ".res_conv.bias").data, k.res);
    return rb;
  }

  void pack(Weights& ws, int num_sms) {
    nsm = num_sms;
    const std::string P = "embedder.unet.";
    const int L = d.unet_levels;
    std::vector<int> z(d.unet_z, d.unet_z + L);
    // ---- inc: first conv on CUDA cores, fp32 weights with BN folded
    {
      const std::string cv = temporal ? ".conv" : "";   // Conv3dWrapper keys
      std::vector<float> s, b;
      ws.bn_fold(P + "inc.double_conv.1", s, b);
      const HostTensor& w = ws.get(P + "inc.double_conv.0" + cv + ".weight");
      VSB_CHECK((int)w.shape[0] == z[0] && (int)w.shape[1] == d.unet_in_ch && (int)w.shape.size() == (temporal ? 5 : 4), "inc conv shape");
      std::vector<float> w1(w.data);   // the CUDA-core kernel reads the checkpoint's own layout: each output row scaled
      const size_t per = (size_t)d.unet_in_ch * (temporal ? 27 : 9);
      VSB_CHECK(w1.size() == per * z[0], "inc conv shape");
      for (int n = 0; n < z[0]; ++n) for (size_t k = 0; k < per; ++k) w1[n * per + k] *= s[n];
      first_w1 = ws.pool.upload(w1); first_b1 = ws.pool.upload(b);
      first_wr = ws.vec(P + "inc.res_conv" + cv + ".weight", (int64_t)z[0] * d.unet_in_ch);
      first_br = ws.vec(P + "inc.res_conv" + cv + ".bias");
      ws.bn_fold(P + "inc.double_conv.4", s, b);
      if (temporal) {
        const HostTensor& w2 = ws.get(P + "inc.double_conv.3.conv.weight");
        inc_c2 = pack_taps(ws, conv3d_taps(w2, &s, temporal_stack_width(z[0])), b, false);
      } else {
        inc_c2 = pack_conv(ws, P + "inc.double_conv.3.weight", &s, b, inc_k);
      }
    }
    for (int i = 0; i < L - 1; ++i) {
      const std::string D = P + "downs." + std::to_string(i);
      const std::vector<float>& bias = ws.get(D + ".down.bias").data;
      ConvW dc;
      if (down_k[i]) { dc.wd = ws.down_s2d(ws.taps(D + ".down.weight")); dc = ws.with_bias(dc, bias); }
      else dc = ws.gemm(ws.taps(D + ".down.weight"), bias);
      down_conv.push_back(dc);
      down_rb.push_back(pack_block(ws, D + ".conv", down_rb_k[i]));
    }
    for (int i = 0; i < d.unet_num_blocks; ++i) bott_rb.push_back(pack_block(ws, P + "bottleneck.model." + std::to_string(i), bott_rb_k));
    std::vector<int> zz(z);
    zz[L - 1] += d.hidden;
    int j = 0;
    for (int ii = L - 2; ii >= 0; --ii, ++j) {
      const std::string U = P + "ups." + std::to_string(j);
      // virtual concat (x | skip * 2^-1/2): fold the skip scale into the second half of the input channels
      std::vector<float> in_scale(2 * zz[ii + 1], 1.0f);
      for (int c = zz[ii + 1]; c < 2 * zz[ii + 1]; ++c) in_scale[c] = 0.70710678118654752440f;
      const Taps t = ws.taps(U + ".up.upsample_block.2.weight", nullptr, &in_scale);
      __half* pw = nullptr; float* bw = nullptr;
      if (up_k[j].phase) ws.upconv_phase(t, &pw, &bw);
      // 8-channel sources go through the gather loader, whose K block is 64: pad K to one block
      up_conv.push_back(up_k[j].phase ? ConvW{} : ws.upconv_taps(t, zz[ii + 1] == 8 ? 64 : 0));
      up_phase_w.push_back(pw); up_border_w.push_back(bw);
      up_lnw.push_back(ws.vec(U + ".up.upsample_block.3.weight"));
      up_lnb.push_back(ws.vec(U + ".up.upsample_block.3.bias"));
      up_rb.push_back(pack_block(ws, U + ".conv", up_rb_k[j]));
    }
    outc_w = ws.vec(P + "outc.weight");  // [n_out][z0][1][1]
    outc_b = ws.vec(P + "outc.bias");
    const HostTensor& t = ws.get(P + "msg_processor.msg_embeddings.weight");
    VSB_CHECK((int)t.shape[0] == 2 * d.nbits && (int)t.shape[1] == d.hidden, "message table shape");
    msg_table = ws.pool.upload(t.data);
  }

  // One conv step, R x R (3: stride 1, zero pad 1; or 1) over x [B,H,W,Cin] (pitch ldx): the direct ring conv when its weights were
  // packed for it, else the tensor-core GEMM.  Epilogue: bias, ReLU (relu), + the fp16 residual `resid` (pitch w.N), output `out`
  // (pitch ld_out; nullptr: not written) and, fuse_outc, the 1x1 outc + tanh into pl.delta.
  void add_conv(Plan& pl, const ConvW& w, int R, const __half* x, int B, int H, int W, int Cin, int ldx,
                bool relu, const __half* resid, __half* out, int ld_out, bool fuse_outc = false, const std::string& label = "") const {
    const int N = w.N;
    const bool direct = w.wd != nullptr;
    VSB_CHECK(!direct || (ldx == Cin && (out == nullptr || ld_out == N)), "direct conv: dense input and output");
    const std::string name = !label.empty() ? label :
                             std::string("unet.conv") + (R == 3 ? "3x3" : "1x1") + (direct ? "d" : "") + (fuse_outc ? "+outc." : ".") +
                             std::to_string(Cin) + "-" + std::to_string(N) + "@" + std::to_string(H);
    if (direct) {
      Conv3DirectOp op; setup_conv3_direct(op, x, B, H, W, Cin, N, w.wd, nsm, R);
      op.p.bias = w.bias; op.p.relu = relu ? 1 : 0; op.p.resid = resid; op.p.out = out;
      if (fuse_outc) {
        op.p.outc_w = outc_w; op.p.outc_b = outc_b; op.p.n_out = d.unet_out_ch; op.p.delta = pl.delta; op.p.outc_tanh = d.unet_last_tanh;
      }
      pl.add(name, [op](cudaStream_t st) { launch_direct(op, st); });
      return;
    }
    // 3x3 up to 16 input channels: on-chip im2col from a shared-memory halo tile (input crosses L2->SM once), one TMA load per tap
    // above; the weight layout follows the same rule (pack_conv)
    ConvGemmOp op;
    if (R == 3 && use_halo(Cin)) setup_halo_conv3(op, x, B, H, W, Cin, ldx);
    else setup_tma_conv(op, x, B, H, W, Cin, ldx, R, R, R / 2);
    op.p.epi = EPI_AFFINE; op.p.act = relu ? ACT_RELU : ACT_NONE; op.p.bias = w.bias;
    if (resid) { op.p.resid16 = resid; op.p.ld_res16 = N; }
    if (out) { op.p.out16 = out; op.p.ld_out16 = ld_out; }
    if (fuse_outc) {
      op.p.outc_w = outc_w; op.p.outc_b = outc_b; op.p.n_out = d.unet_out_ch; op.p.delta = pl.delta; op.p.hw = H * W;
      op.p.outc_tanh = d.unet_last_tanh;
    }
    vsb::add_conv(pl, op, w, name, nsm);
  }

  // 3x3x3 conv (stride 1, zero pad 1 in space and time) over x [B,H,W,Cin] (pitch ldx) in groups of G frames: the frames' time taps
  // stacked into the plan's scratch `xs`, then the tensor-core 3x3 conv over it (K = 9 * Cs).  Arguments after ldx as in add_conv.
  void add_conv3d(Plan& pl, const ConvW& w, const __half* x, int B, int G, int H, int W, int Cin, int ldx, __half* xs,
                  bool relu, const __half* resid, __half* out, int ld_out, bool fuse_outc = false) const {
    const int Cs = temporal_stack_width(Cin), sms = nsm;
    const std::string at = std::to_string(H);
    pl.add("unet.tstack." + std::to_string(Cin) + "-" + std::to_string(Cs) + "@" + at,
           [=](cudaStream_t st) { launch_temporal_stack(x, ldx, Cin, (long)H * W, 0, B, B, G, xs, Cs, sms, st); });
    add_conv(pl, w, 3, xs, B, H, W, Cs, Cs, relu, resid, out, ld_out, fuse_outc,
             std::string("unet.conv3x3x3") + (fuse_outc ? "+outc." : ".") + std::to_string(Cin) + "-" + std::to_string(w.N) + "@" + at);
  }

  // ResnetBlock on NHWC fp16 (modules/unet.py:17-39):  out = relu(conv3'(relu(conv3'(x)))) + (conv1(x) + b)
  // `x` has pixel pitch ldx; output written with pitch ld_out.  If fuse_outc: the 1x1 outc + tanh is fused and the
  // block output itself is not written.
  // G > 0: a temporal block (3x3x3 convs over groups of G frames through the scratch xs, 1x1x1 res conv)
  __half* add_resblock(Plan& pl, const std::string& name, const ResBlockW& w, const __half* x, int B, int G, __half* xs,
                       int H, int W, int Cin, int ldx, __half* out, int ld_out, bool fuse_outc = false) const {
    const int Cout = w.c1.N;
    const long M = (long)B * H * W;
    __half* r = pl.pool.alloc_n<__half>(M * Cout);
    __half* h = pl.pool.alloc_n<__half>(M * Cout);
    if (!out && !fuse_outc) { out = pl.pool.alloc_n<__half>(M * Cout); ld_out = Cout; }
    add_conv(pl, w.res, 1, x, B, H, W, Cin, ldx, false, nullptr, r, Cout);
    if (G > 0) {
      add_conv3d(pl, w.c1, x, B, G, H, W, Cin, ldx, xs, true, nullptr, h, Cout);
      add_conv3d(pl, w.c2, h, B, G, H, W, Cout, Cout, xs, true, r, out, ld_out, fuse_outc);
    } else {
      add_conv(pl, w.c1, 3, x, B, H, W, Cin, ldx, true, nullptr, h, Cout);
      add_conv(pl, w.c2, 3, h, B, H, W, Cout, Cout, true, r, out, ld_out, fuse_outc);
    }
    pl.tap(name + ".h", h, 1, B, H, W, Cout, Cout);
    pl.tap(name + ".r", r, 1, B, H, W, Cout, Cout);
    if (out) pl.tap(name, out, 1, B, H, W, Cout, ld_out);
    return out;
  }

  // the embed plan of B frames; a temporal U-Net convolves across groups of G consecutive frames (G >= 1, the last group may be
  // shorter), a 2-D one takes G = 0
  void build(Plan& pl, int B, int G = 0) const {
    const int S = d.img_size, L = d.unet_levels;
    std::vector<int> z(d.unet_z, d.unet_z + L);
    VSB_CHECK((G > 0) == (temporal), "temporal group length");
    // one time-stacked operand buffer for every 3x3x3 conv of the plan (they run one after the other on one stream)
    __half* xs = nullptr;
    if (G > 0) {
      size_t n = 0;
      for (int i = 0; i < L; ++i) {
        const int C = (i == L - 1 ? z[i] + d.hidden : z[i]), h = S >> i;
        n = std::max(n, (size_t)B * h * h * temporal_stack_width(C));
      }
      xs = pl.pool.alloc_n<__half>(n);
    }
    pl.x_res = pl.pool.alloc_n<float>((size_t)B * 3 * S * S);
    pl.tap("x_res", pl.x_res, 0, B, 3, S, S, S);
    pl.delta = pl.pool.alloc_n<float>((size_t)B * d.unet_out_ch * S * S);
    Plan* plp = &pl;
    // ---- inc
    const long M0 = (long)B * S * S;
    __half* h1 = pl.pool.alloc_n<__half>(M0 * z[0]);
    __half* r0 = pl.pool.alloc_n<__half>(M0 * z[0]);
    {
      const int Z = z[0], yuv = d.yuv, cin = d.unet_in_ch;
      const float *w1 = first_w1, *b1 = first_b1, *wr = first_wr, *br = first_br;
      if (G > 0)
        pl.add("unet.first3x3x3", [=](cudaStream_t st) { launch_unet_first_t(plp->in_imgs, B, G, S, Z, cin, w1, b1, wr, br, h1, r0, st); });
      else
        pl.add("unet.first", [=](cudaStream_t st) { launch_unet_first(plp->in_imgs, B, S, Z, cin, w1, b1, wr, br, h1, r0, yuv, st); });
    }
    pl.tap("first_h", h1, 1, B, S, S, z[0], z[0]);
    pl.tap("first_r", r0, 1, B, S, S, z[0], z[0]);
    std::vector<__half*> skips;  // outputs of inc, downs[0..]
    std::vector<int> skip_ld;
    __half* x = pl.pool.alloc_n<__half>(M0 * z[0]);
    if (G > 0) add_conv3d(pl, inc_c2, h1, B, G, S, S, z[0], z[0], xs, true, r0, x, z[0]);
    else add_conv(pl, inc_c2, 3, h1, B, S, S, z[0], z[0], true, r0, x, z[0]);
    pl.tap("inc", x, 1, B, S, S, z[0], z[0]);
    int ldx = z[0], hs = S;
    const int zb = z[L - 1] + d.hidden;
    __half* cat = nullptr;
    for (int i = 0; i < L - 1; ++i) {
      const int ho = hs / 2;
      const long Mo = (long)B * ho * ho;
      __half* dn = pl.pool.alloc_n<__half>(Mo * z[i + 1]);
      const std::string shape = std::to_string(z[i]) + "-" + std::to_string(z[i + 1]) + "@" + std::to_string(ho);
      if (down_conv[i].wd) {
        Conv3DirectOp op;
        setup_down_s2d_direct(op, x, z[i], B, ho, ho, z[i + 1], down_conv[i].wd, down_conv[i].bias, dn, nsm);
        pl.add("unet.down3x3s2d." + shape, [op](cudaStream_t st) { launch_direct(op, st); });
      } else {
        ConvGemmOp op;
        setup_gather_conv(op, LD_GATHER_CONV, x, z[i], ldx, nullptr, 0, 0, B, hs, hs, ho, ho, 3, 3, 2, 1, 0);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = down_conv[i].bias; op.p.out16 = dn; op.p.ld_out16 = z[i + 1];
        vsb::add_conv(pl, op, down_conv[i], "unet.down3x3s2." + shape, nsm);
      }
      pl.tap("down" + std::to_string(i) + "_conv", dn, 1, B, ho, ho, z[i + 1], z[i + 1]);
      __half* out = nullptr; int ld_out = 0;
      if (i == L - 2) {  // last level writes straight into the message-concat buffer (channels [0, z))
        cat = pl.pool.alloc_n<__half>(Mo * zb);
        out = cat; ld_out = zb;
      }
      x = add_resblock(pl, "down" + std::to_string(i), down_rb[i], dn, B, G, xs, ho, ho, z[i + 1], z[i + 1], out, ld_out);
      ldx = (i == L - 2) ? zb : z[i + 1];
      hs = ho;
      skips.push_back(x); skip_ld.push_back(ldx);
    }
    // ---- message channels
    {
      const int K = d.nbits, hidden = d.hidden, hw = hs * hs, coff = z[L - 1];
      const float* table = msg_table;
      pl.add("unet.msg", [=](cudaStream_t st) { launch_msg_embed(plp->in_msgs, plp->in_msg_stride, table, K, hidden, cat, B, hw, zb, coff, st); });
      pl.tap("cat", cat, 1, B, hs, hs, zb, zb);
    }
    // ---- bottleneck
    x = cat; ldx = zb;
    for (int i = 0; i < d.unet_num_blocks; ++i) {
      x = add_resblock(pl, "bott" + std::to_string(i), bott_rb[i], x, B, G, xs, hs, hs, zb, ldx, nullptr, 0);
      ldx = zb;
    }
    // ---- ups
    std::vector<int> zz(z); zz[L - 1] = zb;
    int j = 0;
    for (int ii = L - 2; ii >= 0; --ii, ++j) {
      const int Cin = zz[ii + 1], Cout = zz[ii];
      // hiddens stack (unet.py:175-191): first pop is the message-concatenated latent, then downs[L-3], ...
      const __half* skip = (j == 0) ? cat : skips[L - 2 - j];
      const int ld_skip = (j == 0) ? zb : skip_ld[L - 2 - j];
      const int ho = hs * 2;
      const long Mo = (long)B * ho * ho;
      __half* u = pl.pool.alloc_n<__half>(Mo * Cout);
      if (up_phase_w[j]) {
        // one tensor-core conv on the low-resolution grid (bilinear weights folded per output phase) + exact border pixels
        Conv3DirectOp op;
        setup_up_phase_direct(op, x, Cin, skip, Cin, B, hs, hs, up_phase_w[j], up_lnw[j], up_lnb[j], 1e-6f, u, nsm);
        pl.add("unet.upphase." + std::to_string(2 * Cin) + "-" + std::to_string(Cout) + "@" + std::to_string(ho),
               [op](cudaStream_t st) { launch_direct(op, st); });
        const __half *x0 = x, *x1 = skip;
        const int IH = hs, Ci = Cin;
        const float *wk = up_border_w[j], *lw = up_lnw[j], *lb = up_lnb[j];
        pl.add("unet.upborder." + std::to_string(Cout) + "@" + std::to_string(ho),
               [=](cudaStream_t st) { launch_up_border_fix(x0, x1, Ci, B, IH, wk, lw, lb, u, nsm, st); });
      } else {
        // channel mixing first, at low resolution: y[b,i,j, tap*Cout + co] = sum_c W[co,c,tap] * [x | skip/sqrt2][b,i,j,c]
        const long Mi = (long)B * hs * hs;
        __half* ytap = pl.pool.alloc_n<__half>(Mi * 9 * Cout);
        ConvGemmOp op;
        if (Cin == 8)   // 8-channel sources: a 1x1 gathered conv over [x | skip] (the TMA GEMM's K block is at least 16 per source)
          setup_gather_conv(op, LD_GATHER_CONV, x, Cin, ldx, skip, Cin, ld_skip, B, hs, hs, hs, hs, 1, 1, 1, 0, 0);
        else
          setup_tma_gemm2(op, x, Cin, ldx, skip, Cin, ld_skip, Mi);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out16 = ytap; op.p.ld_out16 = 9 * Cout;
        vsb::add_conv(pl, op, up_conv[j], "unet.uptap1x1." + std::to_string(2 * Cin) + "-" + std::to_string(9 * Cout) + "@" + std::to_string(hs), nsm);
        pl.tap("up" + std::to_string(j) + "_taps", ytap, 1, B, hs, hs, 9 * Cout, 9 * Cout);
        // then bilinear x2 + reflect pad + 3x3 tap sum + LayerNorm + ReLU (CUDA cores, memory-bound)
        const int vpt = up_k[j].vpt;
        UpsGather g;
        g.y = ytap; g.B = B; g.IH = hs; g.C = Cout; g.lnw = up_lnw[j]; g.lnb = up_lnb[j]; g.out = u; g.ld_out = Cout; g.num_sms = nsm;
        g.optin = kUpGatherSmem;
        g.smem = up_k[j].smem;
        pl.add("unet.upgather." + std::to_string(Cout) + "@" + std::to_string(ho), [g, vpt](cudaStream_t st) { launch_unet_upgather(g, vpt, st); });
      }
      pl.tap("up" + std::to_string(j) + "_conv", u, 1, B, ho, ho, Cout, Cout);
      const bool last = (ii == 0);
      x = add_resblock(pl, "up" + std::to_string(j), up_rb[j], u, B, G, xs, ho, ho, Cout, Cout, nullptr, 0, /*fuse_outc=*/last);
      ldx = Cout; hs = ho;
    }
    pl.tap("delta", pl.delta, 0, B, d.unet_out_ch, S, S, S);
  }
};

}  // namespace vsb
