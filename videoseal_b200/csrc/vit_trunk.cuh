// The SAM-ViT extractor trunk (modules/vit.py ImageEncoderViT): its rules (vsb_model_set_vit_extractor), its packed weights and its
// part of the detect plan.
#pragma once
#include "attention_host.cuh"
#include "pointwise_host.cuh"
#include "weights.cuh"

namespace vsb {

struct VitTrunk {
  bool on = false;   // replaces the ConvNeXt trunk
  vsb_vit_desc vd{};
  ConvW patch;                          // [E][768] fp16, x*2-1 folded: W' = 2W (K order c, r, s); no bias (it is in pos)
  float* pos = nullptr;                 // fp32 [grid^2][E]: pos_embed + b - sum(W)
  struct BlockW { float *n1w, *n1b, *n2w, *n2b; ConvW qkv, proj, lin1, lin2; __half *rel_h, *rel_w; };
  std::vector<BlockW> blk;
  ConvW neck1, neck3;
  float *nln1w = nullptr, *nln1b = nullptr, *nln2w = nullptr, *nln2b = nullptr;

  // the ViT rules (include/vsb200.h) at processing size S, no CUDA calls
  void set(const vsb_vit_desc& v, int S) {
    VSB_CHECK(v.depth >= 1 && v.num_heads >= 1 && v.embed_dim >= 1 && v.window_size >= 0, "ViT: depth, num_heads and embed_dim must be positive");
    VSB_CHECK(v.depth >= 32 || (v.global_mask >> v.depth) == 0, "ViT: global_mask has bits at or above depth");
    VSB_CHECK((v.qkv_bias == 0 || v.qkv_bias == 1) && (v.use_rel_pos == 0 || v.use_rel_pos == 1), "ViT: qkv_bias / use_rel_pos must be 0 or 1");
    auto unsup = [](const std::string& m) { throw Error("SAM-ViT extractor: " + m, kErrUnsupported); };
    if (v.embed_dim % v.num_heads != 0 || v.embed_dim / v.num_heads != kAttnHd)
      unsup("head dim " + std::to_string(v.embed_dim) + " / " + std::to_string(v.num_heads) + " is not implemented (64 only)");
    if (v.mlp_dim <= 0 || v.mlp_dim % 64 != 0) unsup("mlp_dim " + std::to_string(v.mlp_dim) + " is not a multiple of 64");
    if (v.out_chans <= 0 || v.out_chans % 64 != 0) unsup("out_chans " + std::to_string(v.out_chans) + " is not a multiple of 64");
    if (v.patch_size != kVitPatch) unsup("patch_size " + std::to_string(v.patch_size) + " is not implemented (16 only)");
    if (v.depth > 32) unsup("depth " + std::to_string(v.depth) + " above 32 is not implemented");
    const int G = S / kVitPatch;
    const uint32_t all = v.depth == 32 ? ~0u : (1u << v.depth) - 1u;
    if (v.global_mask != all) {   // some block attends over windows
      if (v.window_size <= 0 || G % v.window_size != 0)
        unsup("a " + std::to_string(G) + "-token grid is not divisible by window_size " + std::to_string(v.window_size) + " (window padding is not implemented)");
      if (v.window_size * v.window_size % kAttnTile != 0)
        unsup("window_size " + std::to_string(v.window_size) + " holds " + std::to_string(v.window_size * v.window_size) + " tokens, not a multiple of 64");
    }
    if (v.global_mask != 0 && G * G > 1024)
      unsup("global attention over " + std::to_string(G * G) + " tokens (img_size " + std::to_string(S) + ") is not implemented (at most 1024, img_size <= 512)");
    // the kernel stages the 2n - 1 rows of each relative-position table in 64 rows: region sides n <= 32 (global blocks: the cap above)
    if (v.use_rel_pos && v.global_mask != all && v.window_size > kAttnMaxRelSide)
      unsup("relative positions over " + std::to_string(v.window_size) + "-token-wide windows are not implemented (at most " +
            std::to_string(kAttnMaxRelSide) + ")");
    vd = v;
    on = true;
  }
  int width() const { return vd.out_chans; }
  static int map(int S) { return S / kVitPatch; }   // the token grid

  // modules/vit.py:14-143, :146-210, :302-353, :494-525
  void pack(Weights& ws, int S) {
    const std::string Q = "detector.image_encoder.";
    const int E = vd.embed_dim, G = map(S);
    auto shape_is = [](const HostTensor& t, std::vector<int64_t> s) { return t.shape == s; };
    {
      const HostTensor& w = ws.get(Q + "patch_embed.proj.weight");
      VSB_CHECK(shape_is(w, {E, 3, kVitPatch, kVitPatch}), Q + "patch_embed.proj.weight: expected [embed_dim, 3, 16, 16]");
      const HostTensor& b = ws.get(Q + "patch_embed.proj.bias");
      const HostTensor& pe = ws.get(Q + "pos_embed");
      if (!shape_is(pe, {1, G, G, E}))
        throw Error(Q + "pos_embed: a " + std::to_string(G) + " x " + std::to_string(G) + " grid of " + std::to_string(E) +
                    " is needed at img_size " + std::to_string(S), kErrInvalid);
      // x*2-1 folded (extractor.py:64): W (2x - 1) + b = (2W) x + (b - sum W), K and the sum in the im2col order (c, r, s)
      const Taps t = conv_taps(w);
      std::vector<float> wp((size_t)E * 768), table((size_t)G * G * E);
      std::vector<double> bias(E);
      for (int e = 0; e < E; ++e) {
        double s = 0.0;
        for (int c = 0; c < 3; ++c)
          for (int k = 0; k < 256; ++k) { s += t(e, k, c); wp[(size_t)e * 768 + c * 256 + k] = 2.f * t(e, k, c); }
        bias[e] = (double)b.data[e] - s;
      }
      for (int pidx = 0; pidx < G * G; ++pidx)
        for (int e = 0; e < E; ++e) table[(size_t)pidx * E + e] = (float)((double)pe.data[(size_t)pidx * E + e] + bias[e]);
      patch.N = E; patch.K = 768;
      patch.w = ws.pool.upload(to_half(wp));
      pos = ws.pool.upload(table);
    }
    auto lin = [&](const std::string& k, int N, int K, bool bias) {
      VSB_CHECK(shape_is(ws.get(k + ".weight"), {N, K}), k + ".weight: expected [" + std::to_string(N) + ", " + std::to_string(K) + "]");
      return ws.gemm(ws.taps(k + ".weight"), bias ? ws.get(k + ".bias").data : std::vector<float>{});
    };
    for (int i = 0; i < vd.depth; ++i) {
      const std::string B = Q + "blocks." + std::to_string(i) + ".";
      BlockW w{};
      w.n1w = ws.vec(B + "norm1.weight", E); w.n1b = ws.vec(B + "norm1.bias", E);
      w.n2w = ws.vec(B + "norm2.weight", E); w.n2b = ws.vec(B + "norm2.bias", E);
      w.qkv = lin(B + "attn.qkv", 3 * E, E, vd.qkv_bias != 0);
      w.proj = lin(B + "attn.proj", E, E, true);
      w.lin1 = lin(B + "mlp.lin1", vd.mlp_dim, E, true);
      w.lin2 = lin(B + "mlp.lin2", E, vd.mlp_dim, true);
      if (vd.use_rel_pos) {
        const int n = (vd.global_mask >> i) & 1u ? G : vd.window_size;
        auto rel = [&](const std::string& k) {
          const HostTensor& t = ws.get(k);
          // the reference interpolates a table of another length (vit.py:398-428, for checkpoints of another size): not here
          if (!shape_is(t, {2 * n - 1, kAttnHd}))
            throw Error(k + ": expected [" + std::to_string(2 * n - 1) + ", 64] (2 * " + std::to_string(n) + " - 1 relative positions); "
                        "tables of another length are not interpolated", kErrInvalid);
          VSB_CHECK(n <= kAttnMaxRelSide, k + ": more than 63 relative positions (set_vit_extractor's rule)");
          std::vector<float> p((size_t)kAttnTile * kAttnHd, 0.f);   // zero rows past 2n-1: the kernel reads whole 8-row tiles
          std::copy(t.data.begin(), t.data.end(), p.begin());
          return ws.pool.upload(to_half(p));
        };
        w.rel_h = rel(B + "attn.rel_pos_h");
        w.rel_w = rel(B + "attn.rel_pos_w");
      }
      blk.push_back(w);
    }
    const int oc = vd.out_chans;
    VSB_CHECK(shape_is(ws.get(Q + "neck.0.weight"), {oc, E, 1, 1}), Q + "neck.0.weight: expected [out_chans, embed_dim, 1, 1]");
    VSB_CHECK(shape_is(ws.get(Q + "neck.2.weight"), {oc, oc, 3, 3}), Q + "neck.2.weight: expected [out_chans, out_chans, 3, 3]");
    neck1 = ws.gemm(ws.taps(Q + "neck.0.weight"), {});
    neck3 = ws.gemm(ws.taps(Q + "neck.2.weight"), {}, /*pad_taps=*/true);
    nln1w = ws.vec(Q + "neck.1.weight", oc); nln1b = ws.vec(Q + "neck.1.bias", oc);
    nln2w = ws.vec(Q + "neck.3.weight", oc); nln2b = ws.vec(Q + "neck.3.bias", oc);
  }

  // modules/vit.py:111-143 on the fp32 residual stream x [B*G*G][E] (token rows in raster order), ending in the fp16 [B, G, G,
  // out_chans] map the head reads.  keep_inputs (vsb_debug_keep_inputs): the values the last block and the neck read from buffers
  // that a later step overwrites are copied aside as they pass (vit.blk{L}.in / .ln1 / .mid, vit.neck1x1)
  FeatureMap build(Plan& pl, int B, int S, int nsm, bool keep_inputs) const {
    Plan* plp = &pl;
    const int G = map(S), E = vd.embed_dim, H3 = 3 * E, MLP = vd.mlp_dim, oc = vd.out_chans;
    const long M = (long)B * G * G;
    float* x = pl.pool.alloc_n<float>(M * E);
    float* x0 = pl.pool.alloc_n<float>(M * E);         // patch embedding + position table: block 0 reads it, its proj writes x
    __half* xn = pl.pool.alloc_n<__half>(M * E);       // LayerNorm output, the A operand of qkv / lin1
    __half* qkv = pl.pool.alloc_n<__half>(M * H3);
    __half* att = pl.pool.alloc_n<__half>(M * E);
    __half* hid = pl.pool.alloc_n<__half>(M * MLP);
    __half* x16 = pl.pool.alloc_n<__half>(M * E);      // fp16 copy of the last block's output: the neck's A operand
    // GEMM on the fp16 rows a [M][K] into the fp32 / fp16 outputs the caller sets in op.p
    auto gemm = [&](const __half* a, int K, const ConvW& w, int act, const char* name, auto&& epi) {
      ConvGemmOp op; setup_tma_gemm(op, a, M, K, K);
      op.p.epi = EPI_AFFINE; op.p.act = act; op.p.bias = w.bias;
      epi(op.p);
      add_conv(pl, op, w, name, nsm);
    };
    auto ln = [&](const char* name, const float* in, int C, const float* lw, const float* lb, float eps, __half* out) {
      pl.add(name, [=](cudaStream_t st) { launch_ln_rows(in, M, C, C, lw, lb, eps, out, C, nsm, st); });
    };
    auto keep = [&](const std::string& name, const void* src, int dtype, int C) {
      const size_t bytes = (size_t)M * C * (dtype == 0 ? sizeof(float) : sizeof(__half));
      void* dst = pl.pool.alloc_n<char>(bytes);
      pl.add("dbg.keep." + name, [=](cudaStream_t st) { VSB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st)); }, 0);
      pl.tap(name, dst, dtype, B, G, G, C, C);
    };
    {
      // patch embed (vit.py:494-525): im2col of the 16 x 16 patches, GEMM into the fp32 stream, + (pos_embed + folded bias)
      __half* patches = pl.pool.alloc_n<__half>(M * 768);
      pl.add("vit.patch", [=](cudaStream_t st) { launch_vit_patch_im2col(plp->in_imgs, B, S, patches, nsm, st); });
      gemm(patches, 768, patch, ACT_NONE, "vit.patch", [&](ConvGemmParams& p) { p.out32 = x0; p.ld_out32 = E; });
      const float* table = pos;
      pl.add("vit.patch", [=](cudaStream_t st) { launch_vit_pos_add(x0, M, G * G, E, table, nsm, st); });
      pl.tap("vit.patches", patches, 1, B, G, G, 768, 768);
      pl.tap("vit.embed", x0, 0, B, G, G, E, E);
    }
    for (int i = 0; i < vd.depth; ++i) {
      const BlockW& w = blk[i];
      const std::string bi = "vit.blk" + std::to_string(i);
      const bool global = (vd.global_mask >> i) & 1u;
      const float* xin = i == 0 ? x0 : x;   // the block's input stream
      const bool last = i + 1 == vd.depth;
      if (keep_inputs && last) keep(bi + ".in", xin, 0, E);
      ln("vit.ln", xin, E, w.n1w, w.n1b, 1e-5f, xn);
      if (keep_inputs && last) keep(bi + ".ln1", xn, 1, E);
      gemm(xn, E, w.qkv, ACT_NONE, "vit.qkv", [&](ConvGemmParams& p) { p.out16 = qkv; p.ld_out16 = H3; });
      {
        AttnParams ap{};
        ap.qkv = qkv; ap.out = att; ap.rel_h = w.rel_h; ap.rel_w = w.rel_w;
        ap.G = G; ap.n = global ? G : vd.window_size; ap.heads = vd.num_heads; ap.E = E;
        ap.regions = (G / ap.n) * (G / ap.n); ap.scale = 1.0f / std::sqrt((float)kAttnHd);
        pl.add(global ? "vit.attn_global." + std::to_string(G * G) : "vit.attn_win." + std::to_string(ap.n * ap.n),
               [=](cudaStream_t st) { launch_vit_attention(ap, B, st); });
      }
      // in place after block 0: each element is read and written by the same thread
      gemm(att, E, w.proj, ACT_NONE, "vit.proj", [&](ConvGemmParams& p) { p.resid32 = xin; p.ld_res32 = E; p.out32 = x; p.ld_out32 = E; });
      if (keep_inputs && last) keep(bi + ".mid", x, 0, E);
      ln("vit.ln", x, E, w.n2w, w.n2b, 1e-5f, xn);
      gemm(xn, E, w.lin1, ACT_GELU, "vit.lin1", [&](ConvGemmParams& p) { p.out16 = hid; p.ld_out16 = MLP; });
      gemm(hid, MLP, w.lin2, ACT_NONE, "vit.lin2", [&](ConvGemmParams& p) {
        p.resid32 = x; p.ld_res32 = E; p.out32 = x; p.ld_out32 = E;
        if (last) { p.out16 = x16; p.ld_out16 = E; }
      });
      // the stream, qkv and att buffers are reused by every block, so they hold the LAST block's values after a run: only its taps
      // exist.  Per-block copies would cost ~0.9 GB per 64-frame 256^2 plan; block k - 1 of a model is compared through the model
      // of depth k built from the same checkpoint prefix (tests/test_vit_gpu.py)
      if (last) {
        pl.tap(bi + ".qkv", qkv, 1, B, G, G, H3, H3);
        pl.tap(bi + ".attn", att, 1, B, G, G, E, E);
        pl.tap(bi + ".ln2", xn, 1, B, G, G, E, E);
        pl.tap(bi + ".hid", hid, 1, B, G, G, MLP, MLP);
        pl.tap(bi, x, 0, B, G, G, E, E);
        pl.tap("vit.x16", x16, 1, B, G, G, E, E);
      }
    }
    // neck (vit.py:90-109): 1x1 conv, LayerNorm2d, 3x3 conv (zero padding 1), LayerNorm2d; both without bias, eps 1e-6
    float* y = pl.pool.alloc_n<float>(M * oc);
    __half* yn = pl.pool.alloc_n<__half>(M * oc);
    __half* out = pl.pool.alloc_n<__half>(M * oc);
    gemm(x16, E, neck1, ACT_NONE, "vit.neck1x1", [&](ConvGemmParams& p) { p.out32 = y; p.ld_out32 = oc; });
    if (keep_inputs) keep("vit.neck1x1", y, 0, oc);
    ln("vit.neck_ln", y, oc, nln1w, nln1b, 1e-6f, yn);
    pl.tap("vit.neck_ln1", yn, 1, B, G, G, oc, oc);
    {
      ConvGemmOp op;
      setup_gather_conv(op, LD_GATHER_CONV, yn, oc, oc, nullptr, 0, 0, B, G, G, G, G, 3, 3, 1, 1, 0);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = y; op.p.ld_out32 = oc;
      add_conv(pl, op, neck3, "vit.neck3x3", nsm);
    }
    pl.tap("vit.neck3x3", y, 0, B, G, G, oc, oc);   // the 3x3 output: the last LayerNorm only reads y
    ln("vit.neck_ln", y, oc, nln2w, nln2b, 1e-6f, out);
    pl.tap("vit.neck", out, 1, B, G, G, oc, oc);
    return FeatureMap{out, G, oc, oc};
  }
};

}  // namespace vsb
