// The extractor's pixel decoder (modules/pixel_decoder.py:44-83) on a trunk's feature map: the pooled head (logits) or the
// pixel-wise stages (per-pixel maps).  Its rules, its packed weights and its part of the detect plan.
#pragma once
#include "pointwise_host.cuh"
#include "weights.cuh"

namespace vsb {

constexpr size_t kPdMaxSmem = 227 * 1024;   // tiling cap of the gather kernels: the opt-in shared memory of one H100 block

struct Decoder {
  // vsb_model_set_pixel_decoder: stage i = bilinear x pd[i].f, reflect-padded 3x3 conv C -> C / f, LayerNorm, GELU; then the 1x1
  // conv head C_last -> 1 + nbits per pixel
  bool pixelwise = false;
  // geometry and gather kernel (16-byte vectors per thread; tiled when smem > 0) from set, weights from pack
  struct StageW { ConvW taps; float* lnw; float* lnb; int f, cin, cout, kin, vpt; size_t smem; };
  std::vector<StageW> pd;
  float *pd_hw = nullptr, *pd_hb = nullptr;   // fp32 [1+nbits][C_last], [1+nbits]
  // pooled head
  ConvW head_conv;
  float *head_lnw = nullptr, *head_lnb = nullptr, *head_lw = nullptr, *head_lb = nullptr;

  // K of a stage GEMM over C input channels: the TMA GEMM loader takes K in {16, 32} or >= 64, narrower widths are zero-padded (in
  // the packed weights and in the pitch of the activation buffer, whose pad channels are zeroed once)
  static int gemm_k(int C) { return (C == 16 || C == 32 || C >= 64) ? C : (C < 16 ? 16 : (C < 32 ? 32 : 64)); }
  // 16-byte channel vectors per gather thread for a non-final stage of C channels: C = 8 * VPT * G, G a power of two <= 32
  static int vpt(int C) {
    for (int v : {1, 3}) {
      if (C % (8 * v)) continue;
      const int g = C / (8 * v);
      if (g <= 32 && (g & (g - 1)) == 0) return v;
    }
    return 0;
  }

  // the stage rules (include/vsb200.h) and each stage's gather kernel, no CUDA calls.  stem4: a trunk the pixel-wise decoder runs
  // on; trunk() gives its width and map side, asked only for a pixel-wise decoder on such a trunk (a ConvNeXt stride of 0 has no
  // map).  Stage i maps c -> c / f_i channels; the last stage's kernel holds one pixel's channels in registers and the head's
  // weights beside its staged taps.
  template <class Trunk> void set(int n, const int32_t* f, int pw, bool stem4, int nbits, Trunk&& trunk) {
    VSB_CHECK(pw == 0 || pw == 1, "pixelwise must be 0 or 1");
    VSB_CHECK(n >= 1 && n <= 8, "pixel decoder: 1 to 8 upscale stages");
    for (int i = 0; i < n; ++i) VSB_CHECK(f[i] >= 1, "pixel decoder: upscale factors must be positive");
    if (!pw) {
      if (n != 1 || f[0] != 1) throw Error("pooled pixel decoder: only upscale_stages [1] is implemented", kErrUnsupported);
      pixelwise = false;
      pd.clear();
      return;
    }
    for (int i = 0; i < n; ++i)
      if (f[i] != 2 && f[i] != 4) throw Error("pixel-wise decoder: upscale factors must be 2 or 4", kErrUnsupported);
    if (!stem4) throw Error("pixel-wise decoder: needs a ConvNeXt trunk with stem stride 4", kErrUnsupported);
    const std::pair<int, int> geom = trunk();
    int c = geom.first, h = geom.second;
    std::vector<StageW> stages;
    for (int i = 0; i < n; ++i) {
      const int F = f[i], co = c / F, T = 16 / F;
      const bool last = i + 1 == n;
      if (c % F != 0 || co % 8 != 0 || (last ? co > 32 : vpt(co) == 0) || (i == 0 && gemm_k(c) != c))
        throw Error("pixel decoder: stage " + std::to_string(i) + " (" + std::to_string(c) + " channels / " + std::to_string(F) +
                    ") is not implemented (a trunk width of 16, 32 or >= 64; stage widths multiples of 8 of the form 8 * {1,3} * 2^k, "
                    "the last one at most 32)", kErrUnsupported);
      StageW s{};
      s.f = F; s.cin = c; s.cout = co; s.kin = gemm_k(c);
      const size_t tsmem = ups_tile_smem(F, co);
      if (last) {
        s.vpt = co / 8;
        s.smem = tsmem + (size_t)(1 + nbits) * (co + 1) * sizeof(float);
        if (h % T != 0 || s.smem > kPdMaxSmem)
          throw Error("pixel-wise head: a " + std::to_string(h) + "-pixel map with " + std::to_string(1 + nbits) + " outputs is not implemented", kErrUnsupported);
      } else {
        s.vpt = vpt(co);
        s.smem = h % T == 0 && tsmem <= kPdMaxSmem ? tsmem : 0;
      }
      stages.push_back(s);
      c = co; h *= F;
    }
    pixelwise = true;
    pd = std::move(stages);
  }
  // side of the maps the pixel-wise decoder writes from an h-pixel trunk map
  int out_side(int h) const {
    for (const StageW& s : pd) h *= s.f;
    return h;
  }

  void pack(Weights& ws, int nbits) {
    const std::string D = "detector.pixel_decoder.";
    if (pixelwise) {
      for (size_t i = 0; i < pd.size(); ++i) {
        const std::string K = D + "output_upscaling." + std::to_string(i) + ".upsample_block.";
        StageW& sw = pd[i];
        const HostTensor& w = ws.get(K + "2.weight");
        VSB_CHECK(w.shape.size() == 4 && (int)w.shape[0] == sw.cout && (int)w.shape[1] == sw.cin && w.shape[2] == 3 && w.shape[3] == 3,
                  "pixel decoder stage " + std::to_string(i) + ": weight must be [C/f, C, 3, 3]");
        sw.taps = ws.upconv_taps(conv_taps(w), sw.kin);
        sw.lnw = ws.vec(K + "3.weight");
        sw.lnb = ws.vec(K + "3.bias");
      }
      const HostTensor& lw = ws.get(D + "linear.weight");
      VSB_CHECK(lw.shape.size() == 4 && (int)lw.shape[0] == 1 + nbits && (int)lw.shape[1] == pd.back().cout && lw.shape[2] == 1 && lw.shape[3] == 1,
                "pixel-wise head: linear.weight must be [1+nbits, C, 1, 1]");
      pd_hw = ws.pool.upload(lw.data);
      pd_hb = ws.vec(D + "linear.bias");
    } else {
      head_conv = ws.gemm(ws.taps(D + "output_upscaling.0.upsample_block.2.weight"), {}, /*pad_taps=*/true);
      head_lnw = ws.vec(D + "output_upscaling.0.upsample_block.3.weight");
      head_lnb = ws.vec(D + "output_upscaling.0.upsample_block.3.bias");
      const HostTensor& lw = ws.get(D + "linear.weight");
      VSB_CHECK((int)lw.shape[0] == 1 + nbits, "head linear shape");
      head_lw = ws.pool.upload(lw.data);
      head_lb = ws.vec(D + "linear.bias");
    }
  }

  // on the trunk's map; `prefix` names the pooled head's steps after the trunk
  void build(Plan& pl, int B, const FeatureMap& m, const std::string& prefix, int nbits, int nsm) const {
    if (pixelwise) add_pixel_decoder(pl, B, m, nbits, nsm);
    else add_head(pl, B, m, prefix, nbits, nsm);
  }

  // pixel_decoder.py:61-83: 3x3 conv, LayerNorm, GELU, mean pool and the linear layer into pl.logits
  void add_head(Plan& pl, int B, const FeatureMap& m, const std::string& prefix, int nbits, int nsm) const {
    const int hs = m.h, C = m.C, Cp = m.ld;
    const long M = (long)B * hs * hs;
    float* y = pl.pool.alloc_n<float>(M * Cp);
    ConvGemmOp op;
    setup_gather_conv(op, LD_GATHER_CONV, m.x16, Cp, Cp, nullptr, 0, 0, B, hs, hs, hs, hs, 3, 3, 1, 1, 1);
    op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = y; op.p.ld_out32 = Cp;
    add_conv(pl, op, head_conv, prefix + "head3x3." + std::to_string(C) + "@" + std::to_string(hs), nsm);
    pl.tap("head_conv", y, 0, B, hs, hs, C, Cp);
    float* pooled = pl.pool.alloc_n<float>((size_t)B * C);
    pl.tap("head_pooled", pooled, 0, B, 1, 1, C, C);
    const int P = hs * hs, NO = 1 + nbits;
    const float *lw = head_lnw, *lb = head_lnb, *hw = head_lw, *hb = head_lb;
    float* logits = pl.logits;
    pl.add(prefix + "head_tail", [=](cudaStream_t st) { launch_head(y, B, P, C, Cp, lw, lb, pooled, hw, hb, NO, logits, st); }, 2);
  }

  // Pixel-wise stages.  Each stage is one tensor-core GEMM at the LOW resolution, Y[p, tap*C_out + co] (the tap trick of the U-Net's
  // up-convolutions: bilinear up-sampling, reflection padding and the 3x3 taps are linear, so the channel mixing commutes with the
  // spatial gather), then ups_gather_ln_*_kernel forms each output pixel from 9 taps x 4 bilinear corners + LN + GELU.  The last
  // stage's kernel also applies the 1x1 head and writes the 1+K NCHW maps straight into the caller's buffer (plp->out_maps): the
  // full-resolution activation never goes to HBM.
  void add_pixel_decoder(Plan& pl, int B, const FeatureMap& m, int nbits, int nsm) const {
    Plan* plp = &pl;
    const __half* x = m.x16;
    int h = m.h, ldx = m.ld;
    const int NO = 1 + nbits;
    for (size_t i = 0; i < pd.size(); ++i) {
      const StageW& s = pd[i];
      const int F = s.f, ho = F * h, Co = s.cout, IH = h;
      const bool last = i + 1 == pd.size();
      const long Mi = (long)B * h * h;
      __half* ytap = pl.pool.alloc_n<__half>(Mi * 9 * Co);
      ConvGemmOp op; setup_tma_gemm(op, x, Mi, s.kin, ldx);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out16 = ytap; op.p.ld_out16 = 9 * Co;
      add_conv(pl, op, s.taps, "pd.uptap1x1." + std::to_string(s.cin) + "-" + std::to_string(9 * Co) + "@" + std::to_string(h), nsm);
      pl.tap("pd" + std::to_string(i) + "_y", ytap, 1, B, h, h, 9 * Co, 9 * Co);
      UpsGather g;
      g.y = ytap; g.B = B; g.IH = IH; g.C = Co; g.lnw = s.lnw; g.lnb = s.lnb; g.num_sms = nsm; g.optin = kPdMaxSmem;
      g.smem = s.smem;
      const int v = s.vpt;
      const std::string tag = std::to_string(Co) + "x" + std::to_string(F) + "@" + std::to_string(ho);
      if (last) {
        g.hw = pd_hw; g.hb = pd_hb; g.NO = NO;
        pl.add("pd.gather_head." + tag, [g, F, v, plp](cudaStream_t st) mutable { g.maps = plp->out_maps; launch_pd_gather(g, F, v, st); });
      } else {
        const int ldo = gemm_k(Co);
        // pad channels stay zero: the gather writes [0, Co)
        __half* u = ldo != Co ? pl.pool.alloc_zeroed<__half>((size_t)B * ho * ho * ldo) : pl.pool.alloc_n<__half>((size_t)B * ho * ho * ldo);
        g.out = u; g.ld_out = ldo;
        pl.add(std::string(g.smem ? "pd.upgather." : "pd.upgather_untiled.") + tag, [g, F, v](cudaStream_t st) { launch_pd_gather(g, F, v, st); });
        pl.tap("pd" + std::to_string(i), u, 1, B, ho, ho, Co, ldo);
        x = u; ldx = ldo;
      }
      h = ho;
    }
  }
};

}  // namespace vsb
