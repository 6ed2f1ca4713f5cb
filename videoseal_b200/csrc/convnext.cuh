// The ConvNeXt-V2 extractor trunk (modules/convnext.py): its rules, its packed weights and its part of the detect plan.
#pragma once
#include "pointwise_host.cuh"
#include "weights.cuh"

namespace vsb {

struct ConvNeXt {
  __half* stem_w16 = nullptr;
  float* stem_wk = nullptr;   // widths > 256 (chunkyseal): fp32 [48][C0] for the CUDA-core stem kernel
  float *stem_b = nullptr, *stem_lnw = nullptr, *stem_lnb = nullptr;
  struct DsW { float* lnw; float* lnb; ConvW conv; };
  std::vector<DsW> ds;
  struct CnBlockW { float* dww; float* dwb; float* lnw; float* lnb; ConvW pw1; float* gamma; ConvW pw2; };
  std::vector<std::vector<CnBlockW>> cn;

  static void check(const vsb_model_desc& d) {
    for (int s = 0; s < 4; ++s) {
      VSB_CHECK(d.ext_dims[s] % 2 == 0, "extractor widths must be even (channel pairs in the depthwise kernel)");
      VSB_CHECK(s == 0 || d.ext_dims[s] >= d.ext_dims[s - 1], "extractor widths must not shrink along the trunk");
    }
  }
  // side of stage s's map: stem k4 / stride st, then a k2 s2 downsampling layer before each later stage (odd maps 127, 63, 31:
  // the last row / column is dropped, like nn.Conv2d k2 s2)
  static int map(const vsb_model_desc& d, int s) {
    int h = (d.img_size - 4) / d.ext_stem_stride + 1;
    for (int i = 1; i <= s; ++i) h = (h - 2) / 2 + 1;
    return h;
  }

  void pack(Weights& ws, const vsb_model_desc& d) {
    const std::string Q = "detector.convnext.";
    {
      const HostTensor& w = ws.get(Q + "downsample_layers.0.0.weight");  // [C0][3][4][4]
      const int C0 = d.ext_dims[0];
      VSB_CHECK((int)w.shape[0] == C0 && w.shape[1] == 3 && w.shape[2] == 4, "stem shape");
      const Taps t = conv_taps(w);
      if (C0 <= 256) {   // tensor-core stem GEMM with the LayerNorm fused in the epilogue (needs the whole row in one N tile)
        std::vector<float> p((size_t)C0 * 64, 0.f);   // GEMM operand [C0][64], K = (c, r, s) zero-padded 48 -> 64
        for (int n = 0; n < C0; ++n) for (int c = 0; c < 3; ++c) for (int k = 0; k < 16; ++k) p[(size_t)n * 64 + c * 16 + k] = t(n, k, c);
        stem_w16 = ws.pool.upload(to_half(p));
      } else {           // stem_ln_kernel: [48][C0]
        std::vector<float> p((size_t)48 * C0);
        for (int n = 0; n < C0; ++n) for (int c = 0; c < 3; ++c) for (int k = 0; k < 16; ++k) p[(size_t)(c * 16 + k) * C0 + n] = t(n, k, c);
        stem_wk = ws.pool.upload(p);
      }
      stem_b = ws.vec(Q + "downsample_layers.0.0.bias");
      stem_lnw = ws.vec(Q + "downsample_layers.0.1.weight");
      stem_lnb = ws.vec(Q + "downsample_layers.0.1.bias");
    }
    for (int i = 1; i < 4; ++i) {
      DsW w;
      const std::string K = Q + "downsample_layers." + std::to_string(i);
      w.lnw = ws.vec(K + ".0.weight");
      w.lnb = ws.vec(K + ".0.bias");
      w.conv = ws.gemm(ws.taps(K + ".1.weight"), ws.get(K + ".1.bias").data, /*pad_taps=*/true);
      ds.push_back(w);
    }
    cn.resize(4);
    for (int s = 0; s < 4; ++s) {
      const int C = d.ext_dims[s];
      for (int j = 0; j < d.ext_depths[s]; ++j) {
        const std::string B = Q + "stages." + std::to_string(s) + "." + std::to_string(j) + ".";
        CnBlockW w;
        const Taps dw = ws.taps(B + "dwconv.weight");  // [C][1][7][7] -> [49][C]
        std::vector<float> p((size_t)49 * C);
        for (int c = 0; c < C; ++c) for (int k = 0; k < 49; ++k) p[(size_t)k * C + c] = dw(c, k, 0);
        w.dww = ws.pool.upload(p);
        w.dwb = ws.vec(B + "dwconv.bias");
        w.lnw = ws.vec(B + "norm.weight");
        w.lnb = ws.vec(B + "norm.bias");
        w.pw1 = ws.gemm(ws.taps(B + "pwconv1.weight"), ws.get(B + "pwconv1.bias").data);
        w.gamma = ws.vec(B + "grn.gamma");
        // GRN: gamma*(x*Nx) + beta + x  ==  x*(gamma*Nx + 1) + beta ; beta goes through pwconv2 into its bias
        const Taps w2 = ws.taps(B + "pwconv2.weight");
        const HostTensor &b2 = ws.get(B + "pwconv2.bias"), &beta = ws.get(B + "grn.beta");
        std::vector<float> bias2(C);
        for (int n = 0; n < C; ++n) {
          double a = b2.data[n];
          for (int k = 0; k < 4 * C; ++k) a += (double)w2(n, 0, k) * (double)beta.data[k];
          bias2[n] = (float)a;
        }
        w.pw2 = ws.gemm(w2, bias2);
        cn[s].push_back(w);
      }
    }
  }

  // The trunk on the plan's input frames (pl.in_imgs).  keep_inputs (vsb_debug_keep_inputs): the residual stream is updated in place
  // by every block, so the values a stage's first and last blocks read are copied aside as they pass: s{s}_ds after the stem / down
  // conv, s{s}_in before the last block.
  FeatureMap build(Plan& pl, int B, const vsb_model_desc& d, int nsm, bool keep_inputs) const {
    Plan* plp = &pl;
    const int S = d.img_size, st_ = d.ext_stem_stride;
    int hs = map(d, 0);
    int C = d.ext_dims[0];
    // pixel pitch of every NHWC buffer of the trunk: the width rounded up to 8 channels (16-byte fp16 rows for TMA / vector
    // access; the proportional chunkyseal widths 362 / 724 are not multiples of 8).  Pad channels are never read through a
    // TMA map (its K extent is the true width); the buffers the gather loaders read are zeroed once below.
    auto pitch = [](int c) { return (c + 7) / 8 * 8; };
    int Cp = pitch(C);
    float* x = pl.pool.alloc_n<float>((size_t)B * hs * hs * Cp);
    if (stem_wk != nullptr) {
      // widths > 256: CUDA-core stem conv + LayerNorm (one warp per output pixel); the fused-LN GEMM epilogue needs N <= 256
      const int OH = hs, Cc = C, ldo = Cp;
      const float *wk = stem_wk, *sb = stem_b, *lw = stem_lnw, *lb = stem_lnb;
      pl.add("cnx.stem_ln." + std::to_string(C) + "@" + std::to_string(hs),
             [=](cudaStream_t st) { launch_stem_ln(plp->in_imgs, B, S, OH, st_, wk, sb, lw, lb, Cc, x, ldo, nsm, st); });
    } else {
      // stem (convnext.py:108-111): im2col of the k4 patches (x = 2*img-1 folded) -> tensor-core GEMM [M,64]x[64,C0] with the
      // conv bias and the channels-first LayerNorm fused into the epilogue, fp32 NHWC output (the residual stream)
      const int OH = hs;
      const long M = (long)B * OH * OH;
      __half* patches = pl.pool.alloc_n<__half>(M * 64);
      pl.add("cnx.stem_im2col", [=](cudaStream_t st) { launch_stem_im2col(plp->in_imgs, B, S, OH, st_, patches, nsm, st); });
      ConvGemmOp op; setup_tma_gemm(op, patches, M, 64, 64);
      op.p.epi = EPI_LN; op.p.act = ACT_NONE; op.p.bias = stem_b; op.p.ln_w = stem_lnw; op.p.ln_b = stem_lnb; op.p.ln_eps = 1e-6f;
      op.p.out32 = x; op.p.ld_out32 = Cp;
      ConvW sw; sw.w = stem_w16; sw.N = C; sw.K = 64; sw.bias = stem_b;
      add_conv(pl, op, sw, "cnx.stem_gemm." + std::to_string(C) + "@" + std::to_string(hs), nsm);
    }
    auto keep = [&](const std::string& name, const float* src, int h, int c, int cp) {
      const size_t bytes = (size_t)B * h * h * cp * sizeof(float);
      float* dst = pl.pool.alloc_n<float>((size_t)B * h * h * cp);
      pl.add("dbg.keep." + name, [=](cudaStream_t st) { VSB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st)); }, 0);
      pl.tap(name, dst, 0, B, h, h, c, cp);
      return dst;
    };
    int maxK4 = 0;
    for (int s = 0; s < 4; ++s) maxK4 = std::max(maxK4, 4 * d.ext_dims[s]);
    // GRN statistics ping-pong: block j's pwconv1 accumulates into stats_pp[j&1]; its apply pass clears stats_pp[(j+1)&1] over
    // B*K_j floats, which covers what block j-1 left there because the widths never shrink along the trunk.  Both buffers are
    // zeroed at the start of every run (the last block of the previous run leaves its statistics behind).
    const size_t stats_n = (size_t)B * maxK4;
    float* stats_all = pl.pool.alloc_n<float>(2 * stats_n);
    float* stats_pp[2] = {stats_all, stats_all + stats_n};
    int blk_counter = 0;
    // Deterministic mode (every stage's rows per sample a multiple of 32: the tiny and base trunks at S a multiple of 256): the
    // pwconv1 epilogue warps STORE per-warp partial column sums ([M/32][4C]) and the GRN kernels add them in a fixed order: no
    // atomics, no clearing, bit-reproducible logits.  Otherwise (chunkyseal's odd maps; the tiny and base trunks at S = 128, 384,
    // 640, ...) float atomics into [B][4C], cleared here and by the GRN kernels.
    bool all_part = true;
    size_t part_n = 0;
    for (int s = 0; s < 4; ++s) {
      const long rps = (long)map(d, s) * map(d, s), Ms = (long)B * rps;
      if (rps % 32 != 0) all_part = false;      // every epilogue warp (32 rows) then lies inside one sample, also in a ragged last tile
      part_n = std::max(part_n, (size_t)((Ms + kBlockM - 1) / kBlockM * 4) * 4 * d.ext_dims[s]);
    }
    float* part_buf = all_part ? pl.pool.alloc_n<float>(part_n) : nullptr;
    if (!all_part)
      pl.add("cnx.grn_clear", [=](cudaStream_t st) { VSB_CUDA(cudaMemsetAsync(stats_all, 0, 2 * stats_n * sizeof(float), st)); }, 0);
    __half* x16 = nullptr;
    for (int s = 0; s < 4; ++s) {
      if (s > 0) {
        const int Cv = d.ext_dims[s - 1], Cvp = Cp, Cn = d.ext_dims[s], Cnp = pitch(Cn);
        const long Mp = (long)B * hs * hs;
        // pad channels stay zero: ln_rows writes [0, Cv)
        __half* xn = Cvp != Cv ? pl.pool.alloc_zeroed<__half>(Mp * Cvp) : pl.pool.alloc_n<__half>(Mp * Cvp);
        {
          const float *lw = ds[s - 1].lnw, *lb = ds[s - 1].lnb, *xin = x;
          pl.add("cnx.ln_rows", [=](cudaStream_t st) { launch_ln_rows(xin, Mp, Cv, Cvp, lw, lb, 1e-6f, xn, Cvp, nsm, st); });
        }
        pl.tap("s" + std::to_string(s) + "_ln", xn, 1, B, hs, hs, Cv, Cvp);
        const int ho = map(d, s);
        float* xo = pl.pool.alloc_n<float>((size_t)B * ho * ho * Cnp);
        ConvGemmOp op;
        // K order (r, s, c) with c over the PADDED width: matches Weights::gemm(..., pad_taps)
        setup_gather_conv(op, LD_GATHER_CONV, xn, Cvp, Cvp, nullptr, 0, 0, B, hs, hs, ho, ho, 2, 2, 2, 0, 0);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = ds[s - 1].conv.bias; op.p.out32 = xo; op.p.ld_out32 = Cnp;
        add_conv(pl, op, ds[s - 1].conv, "cnx.down2x2s2." + std::to_string(Cv) + "-" + std::to_string(Cn) + "@" + std::to_string(ho), nsm);
        x = xo; hs = ho; C = Cn; Cp = Cnp;
      }
      const std::string ss = "s" + std::to_string(s);
      const float* kept_ds = keep_inputs ? keep(ss + "_ds", x, hs, C, Cp) : nullptr;
      const long M = (long)B * hs * hs;
      const int rows_per_sample = hs * hs;
      __half* a = pl.pool.alloc_n<__half>(M * Cp);
      __half* g = pl.pool.alloc_n<__half>(M * 4 * C);   // 4C is a multiple of 8 for every even width
      // GRN multiplier: folded into per-sample pwconv2 weights where a sample has many more rows than W2 has output
      // channels (stages 0-1 of the tiny trunk), applied to g in place otherwise
      const bool wscale = 4 * C <= rows_per_sample && rows_per_sample % kBlockM == 0 && C % 16 == 0;
      __half* w2s = wscale ? pl.pool.alloc_n<__half>((size_t)B * C * 4 * C) : nullptr;
      const std::string tag = std::to_string(C) + "@" + std::to_string(hs);
      for (int jb = 0; jb < d.ext_depths[s]; ++jb) {
        const CnBlockW& w = cn[s][jb];
        const bool last = jb == d.ext_depths[s] - 1;
        if (keep_inputs && last) {
          if (jb == 0) pl.tap(ss + "_in", kept_ds, 0, B, hs, hs, C, Cp);
          else keep(ss + "_in", x, hs, C, Cp);
        }
        {
          const DwConvOp op = setup_dwconv(x, B, hs, C, Cp, w.dww, w.dwb, w.lnw, w.lnb, a);
          pl.add(std::string("cnx.dwconv7_ln.") + dw_kind_name(op.kind) + "." + tag, [op](cudaStream_t st) { launch_dwconv(op, st); });
        }
        {
          ConvGemmOp op; setup_tma_gemm(op, a, M, C, Cp);
          op.p.epi = EPI_AFFINE; op.p.act = ACT_GELU; op.p.bias = w.pw1.bias; op.p.out16 = g; op.p.ld_out16 = 4 * C;
          float* stats = all_part ? part_buf : stats_pp[blk_counter & 1];
          ++blk_counter;
          op.p.grn_stats = stats; op.p.rows_per_sample = rows_per_sample; op.p.grn_part = all_part ? 1 : 0;
          add_conv(pl, op, w.pw1, "cnx.pwconv1." + tag, nsm);
        }
        {
          const int K4 = 4 * C, Cc = C, part_rows = all_part ? rows_per_sample / 32 : 0;
          const float* gamma = w.gamma;
          float* stats = all_part ? part_buf : stats_pp[(blk_counter - 1) & 1];
          float* stats_next = all_part ? nullptr : stats_pp[blk_counter & 1];
          // GRN multiplier folded into per-sample copies of W2 (pointwise.cuh K2e: no pass over g at all), or applied to g in place
          const __half* w2 = w.pw2.w;
          pl.add((wscale ? "cnx.grn_wscale." : "cnx.grn_apply.") + tag, [=](cudaStream_t st) {
            launch_grn(stats, stats_next, gamma, K4, part_rows, B, w2, w2s, Cc, g, rows_per_sample, nsm, st);
          });
        }
        {
          ConvGemmOp op; setup_tma_gemm(op, g, M, 4 * C, 4 * C);
          op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.pw2.bias; op.p.resid32 = x; op.p.ld_res32 = Cp;
          op.p.out32 = x; op.p.ld_out32 = Cp;  // in place: each element is read and written by the same thread
          if (wscale) { op.w_samples = B; op.p.rows_per_sample = rows_per_sample; }
          if (s == 3 && last) {
            // the head conv's gather reads the pad channels
            x16 = Cp != C ? pl.pool.alloc_zeroed<__half>(M * Cp) : pl.pool.alloc_n<__half>(M * Cp);
            op.p.out16 = x16; op.p.ld_out16 = Cp;
            pl.tap("stage3_16", x16, 1, B, hs, hs, C, Cp);
          }
          add_conv(pl, op, w.pw2, "cnx.pwconv2." + tag, nsm, wscale ? w2s : nullptr);
        }
      }
      // a, g and w2s are reused by every block of the stage: after a run they hold the last block's values (g after the in-place
      // GRN where it is applied)
      pl.tap(ss + "_a", a, 1, B, hs, hs, C, Cp);
      pl.tap(ss + "_g", g, 1, B, hs, hs, 4 * C, 4 * C);
      if (wscale) pl.tap(ss + "_w2s", w2s, 1, B, C, 1, 4 * C, 4 * C);
      pl.tap("stage" + std::to_string(s), x, 0, B, hs, hs, C, Cp);
    }
    return FeatureMap{x16, hs, C, Cp};
  }
};

}  // namespace vsb
