// The host checkpoint and the weight layouts the kernels read.  conv_taps is the one reader of the checkpoint's NCHW order: every
// packed layout below re-indexes the fp32 [N][T][C] taps it returns.
#pragma once
#include <algorithm>
#include <cmath>
#include <map>
#include <string>
#include <vector>

#include "../../include/vsb200.h"
#include "conv3_direct_host.cuh"
#include "plan.cuh"

namespace vsb {

struct HostTensor {
  std::vector<float> data;
  std::vector<int64_t> shape;
  int64_t numel() const { int64_t n = 1; for (auto s : shape) n *= s; return n; }
};

struct ConvW {          // packed conv / linear weights: fp16 [N][K] (K order r,s,c) + fp32 bias
  __half* w = nullptr;
  __half* wd = nullptr;  // 3x3 convs eligible for conv3_direct.cuh: the same weights in its core-matrix layout
  float* bias = nullptr;
  int N = 0, K = 0;
  int ld = 0;            // row pitch of `w` in elements (0 = K): rows are padded to a multiple of 8 (16-byte TMA strides)
};

inline std::vector<__half> to_half(const std::vector<float>& v) {
  std::vector<__half> h(v.size());
  for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
  return h;
}

// fp32 conv taps [N][T = R*S][C] (K order r, s, c)
struct Taps {
  int N = 0, C = 0, R = 1, S = 1, T = 1;
  std::vector<float> v;
  float operator()(int n, int t, int c) const { return v[((size_t)n * T + t) * C + c]; }
};

// conv weight [N][C][R][S] or linear [N][C], times out_scale[n] and then in_scale[c] -> taps
inline Taps conv_taps(const HostTensor& w, const std::vector<float>* out_scale = nullptr, const std::vector<float>* in_scale = nullptr) {
  VSB_CHECK(w.shape.size() == 4 || w.shape.size() == 2, "conv weight rank");
  Taps t;
  t.N = (int)w.shape[0]; t.C = (int)w.shape[1];
  if (w.shape.size() == 4) { t.R = (int)w.shape[2]; t.S = (int)w.shape[3]; }
  t.T = t.R * t.S;
  t.v.resize((size_t)t.N * t.T * t.C);
  for (int n = 0; n < t.N; ++n)
    for (int c = 0; c < t.C; ++c)
      for (int k = 0; k < t.T; ++k) {
        float v = w.data[((size_t)n * t.C + c) * t.T + k];
        if (out_scale) v *= (*out_scale)[n];
        if (in_scale) v *= (*in_scale)[c];
        t.v[((size_t)n * t.T + k) * t.C + c] = v;
      }
  return t;
}

// Conv3d weight [N][C][3][3][3] (3x3x3) or [N][C][1][1][1] times out_scale[n] -> taps.  1x1x1: the 1x1 taps.  3x3x3: the taps of the 3x3
// conv over the time-stacked operand of temporal.cuh, Cs >= 3C channels [x(t-1) | x(t) | x(t+1) | zeros], K order (r, s, dt, c).
inline Taps conv3d_taps(const HostTensor& w, const std::vector<float>* out_scale, int Cs) {
  VSB_CHECK(w.shape.size() == 5 && w.shape[2] == w.shape[3] && w.shape[3] == w.shape[4] && (w.shape[2] == 1 || w.shape[2] == 3),
            "conv3d weight shape: [N, C, 3, 3, 3] or [N, C, 1, 1, 1]");
  Taps t;
  t.N = (int)w.shape[0];
  const int C = (int)w.shape[1];
  if (w.shape[2] == 1) {
    HostTensor w2{w.data, {w.shape[0], w.shape[1], 1, 1}};
    return conv_taps(w2, out_scale);
  }
  VSB_CHECK(Cs >= 3 * C, "conv3d: stacked width");
  t.C = Cs; t.R = t.S = 3; t.T = 9;
  t.v.assign((size_t)t.N * 9 * Cs, 0.f);
  for (int n = 0; n < t.N; ++n)
    for (int c = 0; c < C; ++c)
      for (int dt = 0; dt < 3; ++dt)
        for (int k = 0; k < 9; ++k) {
          float v = w.data[(((size_t)n * C + c) * 3 + dt) * 9 + k];
          if (out_scale) v *= (*out_scale)[n];
          t.v[((size_t)n * 9 + k) * Cs + dt * C + c] = v;
        }
  return t;
}

// The checkpoint as vsb_model_set_tensor delivers it, and the pool of every weight packed from it
struct Weights {
  std::map<std::string, HostTensor> sd;   // host copies, dropped once the model is finalized
  DevicePool pool;

  const HostTensor& get(const std::string& k) const {
    auto it = sd.find(k);
    if (it == sd.end()) throw Error("missing checkpoint tensor: " + k, kErrState);
    return it->second;
  }
  // tensor k uploaded as it is (fp32); n >= 0: it must hold n values
  float* vec(const std::string& k, int64_t n = -1) {
    const HostTensor& t = get(k);
    VSB_CHECK(n < 0 || t.numel() == n, k + ": expected " + std::to_string(n) + " values");
    return pool.upload(t.data);
  }
  Taps taps(const std::string& k, const std::vector<float>* out_scale = nullptr, const std::vector<float>* in_scale = nullptr) const {
    return conv_taps(get(k), out_scale, in_scale);
  }
  // eval-mode BatchNorm2d folded into the preceding bias-free conv: w' = w*g/sqrt(var+eps), b' = beta - mean*g/sqrt(var+eps)
  void bn_fold(const std::string& bn, std::vector<float>& scale, std::vector<float>& bias) const {
    const HostTensor &g = get(bn + ".weight"), &b = get(bn + ".bias"), &mu = get(bn + ".running_mean"), &var = get(bn + ".running_var");
    const size_t n = g.data.size();
    scale.resize(n); bias.resize(n);
    for (size_t i = 0; i < n; ++i) {
      const float s = g.data[i] / std::sqrt(var.data[i] + 1e-5f);
      scale[i] = s;
      bias[i] = b.data[i] - mu.data[i] * s;
    }
  }

  ConvW with_bias(ConvW cw, const std::vector<float>& bias) {
    cw.bias = bias.empty() ? nullptr : pool.upload(bias);
    return cw;
  }
  // GEMM operand [N][T][C] with rows padded to a multiple of 8 elements (a no-op for every width of the tiny / pixelseal cards).
  // pad_taps: every tap's channel run is zero-padded to a multiple of 8 (gather loaders move 16-byte channel chunks; the
  // activation buffer then has the same padded pixel pitch with ZERO pad channels).
  ConvW gemm(const Taps& t, const std::vector<float>& bias, bool pad_taps = false) {
    const int Cp = pad_taps ? (t.C + 7) / 8 * 8 : t.C;
    ConvW cw;
    cw.N = t.N; cw.K = t.T * Cp; cw.ld = (cw.K + 7) / 8 * 8;
    std::vector<float> p((size_t)t.N * cw.ld, 0.f);
    for (int n = 0; n < t.N; ++n)
      for (int k = 0; k < t.T; ++k)
        for (int c = 0; c < t.C; ++c) p[(size_t)n * cw.ld + (size_t)k * Cp + c] = t(n, k, c);
    cw.w = pool.upload(to_half(p));
    return with_bias(cw, bias);
  }
  // 3x3 conv -> halo-loader layout [N][chunk][tap][cc], chunks zero-padded to kb_per_c*64
  ConvW halo(const Taps& t, const std::vector<float>& bias) {
    VSB_CHECK(t.R == 3 && t.S == 3, "halo conv weight shape");
    const int cc = t.C < 64 ? t.C : 64, kbc = (9 * cc + 63) / 64, Kpad = halo_kpad(t.C, 0);
    std::vector<float> p((size_t)t.N * Kpad, 0.f);
    for (int n = 0; n < t.N; ++n)
      for (int c = 0; c < t.C; ++c)
        for (int k = 0; k < 9; ++k) p[(size_t)n * Kpad + (size_t)(c / cc) * kbc * 64 + k * cc + (c % cc)] = t(n, k, c);
    ConvW cw;
    cw.N = t.N; cw.K = Kpad;
    cw.w = pool.upload(to_half(p));
    return with_bias(cw, bias);
  }
  // 3x3 up-conv as a low-resolution tap GEMM (see ups_gather_ln_kernel): rows n' = tap*Cout + co, K = input channels (zero-padded to
  // Kp columns when Kp > C: the pixel decoder's narrow stage inputs, see Decoder::gemm_k)
  ConvW upconv_taps(const Taps& t, int Kp = 0) {
    VSB_CHECK(t.R == 3 && t.S == 3, "up conv weight shape");
    if (Kp < t.C) Kp = t.C;
    std::vector<float> p((size_t)9 * t.N * Kp, 0.f);
    for (int co = 0; co < t.N; ++co)
      for (int k = 0; k < 9; ++k)
        for (int c = 0; c < t.C; ++c) p[((size_t)k * t.N + co) * Kp + c] = t(co, k, c);
    ConvW cw;
    cw.N = 9 * t.N; cw.K = Kp;
    cw.w = pool.upload(to_half(p));
    return cw;
  }
  // the same up-conv folded for the phase path (conv3_direct_host.cuh, setup_up_phase_direct): rows n = (py*2+px)*Cout + co,
  // K = (ey*3+ex)*Ct + c over the 3x3 LOW-resolution neighbourhood; g[phase][d][e] = weight of low-res offset e-1 in tap d of
  // an output row of that phase (bilinear x2, align_corners=False).  Also the plain fp32 taps for the border fix-up kernel.
  void upconv_phase(const Taps& t, __half** wd_out, float** wk_out) {
    const int Co = t.N, Ct = t.C;
    static const float g[2][3][3] = {{{.75f, .25f, 0.f}, {.25f, .75f, 0.f}, {0.f, .75f, .25f}},
                                     {{.25f, .75f, 0.f}, {0.f, .75f, .25f}, {0.f, .25f, .75f}}};
    std::vector<float> p((size_t)4 * Co * 9 * Ct, 0.f), wk((size_t)9 * Co * Ct);
    for (int co = 0; co < Co; ++co)
      for (int c = 0; c < Ct; ++c)
        for (int dy = 0; dy < 3; ++dy)
          for (int dx = 0; dx < 3; ++dx) {
            const float kv = t(co, dy * 3 + dx, c);
            wk[((size_t)(dy * 3 + dx) * Co + co) * Ct + c] = kv;
            for (int py = 0; py < 2; ++py)
              for (int px = 0; px < 2; ++px)
                for (int ey = 0; ey < 3; ++ey)
                  for (int ex = 0; ex < 3; ++ex) {
                    const float cf = g[py][dy][ey] * g[px][dx][ex];
                    if (cf != 0.f) p[((size_t)((py * 2 + px) * Co + co) * 9 + (ey * 3 + ex)) * Ct + c] += kv * cf;
                  }
          }
    *wd_out = direct_taps(p, 4 * Co, Ct);
    *wk_out = pool.upload(wk);
  }
  // fp32 taps [N][T][C] -> weights in the direct conv's core-matrix layout (pack_direct_weights_kernel); each value is rounded to
  // fp16 once, and the fp16 copy the kernel reads is freed once it is done
  __half* direct_taps(const std::vector<float>& taps, int N, int C, int T = 9) {
    DevicePool tmp;
    __half* wd = pool.alloc_n<__half>(taps.size());
    pack_direct_weights(tmp.upload(to_half(taps)), N, C, wd, 0, T);
    VSB_CUDA(cudaStreamSynchronize(0));
    return wd;
  }
  // stride-1 3x3 / 1x1 conv for the direct conv (conv3_direct.cuh); 8 -> 8 channels (unet_tiny_*) run only on its 8-channel
  // instantiation (KS = 0), through the virtual-tap layout of direct8_weights
  __half* direct(const Taps& t) {
    if (t.C != 8) return direct_taps(t.v, t.N, t.C, t.T);
    VSB_CHECK(t.N == 8, "8-channel conv weight shape");
    return direct_taps(direct8_weights(t.v, t.N, t.R), t.N, 16, t.R * ((t.R + 1) / 2));
  }
  // DBlock.down for the space-to-depth ring conv (conv3_direct_host.cuh, setup_down_s2d_direct)
  __half* down_s2d(const Taps& t) { return direct_taps(s2d_weights(t.v, t.N, t.C), t.N, 4 * t.C); }
};

// one tensor-core GEMM step on packed weights (w_override: another copy of w.w in the same layout)
inline void add_conv(Plan& pl, ConvGemmOp op, const ConvW& w, const std::string& name, int num_sms, const __half* w_override = nullptr) {
  finalize_op(op, w_override ? w_override : w.w, w.N, w.K, w.ld ? w.ld : w.K, num_sms, 0);
  pl.add(name, [op](cudaStream_t st) { launch(op, st); });
  const ConvGemmParams& p = op.p;
  const bool ragged = op.longk ? p.M % kLongM != 0 : (long)p.m_tiles * kBlockM != (long)p.M;
  pl.gemms.push_back(name + "\tM=" + std::to_string(p.M) + "\tN=" + std::to_string(w.N) + "\tK=" + std::to_string(w.K) +
                     "\tblock_n=" + std::to_string(p.block_n) + "\ttma_store=" + std::to_string(p.tma_store) +
                     "\tb_resident=" + std::to_string(p.b_resident) + "\tb_fixed_ntile=" + std::to_string(p.b_fixed_ntile) +
                     "\tkernel=" + (op.longk ? "longk" : "128") + "\tbias_global=" + std::to_string(p.bias_global) +
                     "\tm_tiles=" + (ragged ? "ragged" : "whole"));
}

}  // namespace vsb
