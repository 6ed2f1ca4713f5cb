// The HiDDeN embedder and extractor (modules/hidden.py; models/embedder.py HiddenEmbedder, models/extractor.py HiddenExtractor):
// stacks of ConvBNRelu = 3x3 conv (pad 1, bias) + BatchNorm2d (eval) or GroupNorm(8, C) + ReLU or GELU.  Their rules, kernels,
// packed weights and plans.
//
// Kernels of a layer, by its input and its norm:
//   3 -> C (the first layer, and the image columns of the encoder's concat layer): hidden_c3_kernel on CUDA cores, x = 2 x - 1
//          read from the planar fp32 frames, BatchNorm folded, and for the concat layer the message table added.
//   C -> C: the tensor-core TMA conv (conv_gemm.cuh, existing instantiations only), BatchNorm folded into weights and bias.
//   BatchNorm layers apply the activation in the producer's epilogue.  GroupNorm layers write the pre-norm map (fp16), then
//   hidden_gn_stats_kernel and hidden_norm_act_kernel (statistics, then (y - mu) rstd gamma + beta and the activation).
//   The last layer of each network always ends in hidden_norm_act_kernel (identity scale for BatchNorm), which fuses the encoder's
//   1x1 final_layer (+ tanh) or the decoder's spatial mean.
//
// GroupNorm statistics are deterministic and atomic-free: per tile of kGnTile pixels of one frame, fp64 sums of x and x^2 over each
// group's 8 channels (the fp16 inputs and their squares are exact in fp64), reduced in a fixed order and written with plain stores;
// the apply kernel adds a frame's tile partials in tile order.  With fp64 sums the one-pass variance E[x^2] - mu^2 loses
// log2(mu^2 / var) of fp64's 53 bits: |mu| / sigma = 1e4 still leaves 26 exact bits, beyond what the fp32 apply uses.  A frame's
// statistics depend on its own pixels only, so they do not change with the batch split.
//
// Message folding: the concat [m (K planes of +-1) | enc (C) | x (3)] is never materialised.  Under zero padding a constant plane's
// 3x3 contribution at a pixel depends only on which taps fall inside the map: 9 border cases (interior, 4 edges, 4 corners).
// pack sums the message columns of the weight over the valid taps of each case ([9][C][K]); hidden_msg_table_kernel turns that into
// a per-frame [9][C] fp32 table from the message, and hidden_c3_kernel adds table[case] to the image columns' conv.  That fp16 map
// is the residual of the tensor-core conv over enc: the same sum, reassociated.
#pragma once
#include "pointwise_host.cuh"
#include "weights.cuh"

namespace vsb {

constexpr int kGnTile = 2048;      // pixels per GroupNorm statistics partial
constexpr int kHidPix = 256;       // pixels (threads) per block of the pointwise kernels
constexpr int kHidC = 64;          // the one width the kernels implement

enum : int { HID_OUT16 = 0, HID_OUTC = 1, HID_POOL = 2 };

__device__ __forceinline__ float hid_act(float v, int act) {
  return act == ACT_RELU ? fmaxf(v, 0.f) : (act == ACT_GELU ? gelu_erf(v) : v);
}

// 3 -> 64 3x3 conv over x = 2 imgs - 1 (planar fp32 [B][3][S][S], frame stride fstride), zero padding; one thread per pixel.
// w: [27][64] fp32 (k = c * 9 + r * 3 + s), bias [64] (may be null); table: [B][9][64] added by border case (may be null);
// out: NHWC fp16 [B*S*S][64] after `act`.
__global__ void __launch_bounds__(kHidPix) hidden_c3_kernel(const float* __restrict__ imgs, long fstride, int S,
                                                            const float* __restrict__ w, const float* __restrict__ bias,
                                                            const float* __restrict__ table, int act, __half* __restrict__ out) {
  __shared__ float4 sw[27 * 16];
  __shared__ float4 sb[16];
  for (int i = threadIdx.x; i < 27 * 16; i += blockDim.x) sw[i] = reinterpret_cast<const float4*>(w)[i];
  if (threadIdx.x < 16) sb[threadIdx.x] = bias ? reinterpret_cast<const float4*>(bias)[threadIdx.x] : make_float4(0.f, 0.f, 0.f, 0.f);
  __syncthreads();
  const int b = blockIdx.y;
  const long p = (long)blockIdx.x * kHidPix + threadIdx.x;
  const int y = (int)(p / S), x = (int)(p % S);
  const float* im = imgs + (long)b * fstride;
  float in[27];
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int yy = y + r - 1, xx = x + s - 1;
        const bool ok = yy >= 0 && yy < S && xx >= 0 && xx < S;
        in[c * 9 + r * 3 + s] = ok ? 2.f * __ldg(im + ((long)c * S + yy) * S + xx) - 1.f : 0.f;
      }
  const float4* tb = nullptr;
  if (table) {
    const int cs = (y == 0 ? 0 : (y == S - 1 ? 2 : 1)) * 3 + (x == 0 ? 0 : (x == S - 1 ? 2 : 1));
    tb = reinterpret_cast<const float4*>(table + ((long)b * 9 + cs) * kHidC);
  }
  uint4* o = reinterpret_cast<uint4*>(out + ((long)b * S * S + p) * kHidC);
#pragma unroll
  for (int v = 0; v < 8; ++v) {   // 8 output channels (one 16-byte store) at a time
    float4 a0 = sb[2 * v], a1 = sb[2 * v + 1];
#pragma unroll
    for (int k = 0; k < 27; ++k) {
      const float4 w0 = sw[k * 16 + 2 * v], w1 = sw[k * 16 + 2 * v + 1];
      a0.x = fmaf(w0.x, in[k], a0.x); a0.y = fmaf(w0.y, in[k], a0.y); a0.z = fmaf(w0.z, in[k], a0.z); a0.w = fmaf(w0.w, in[k], a0.w);
      a1.x = fmaf(w1.x, in[k], a1.x); a1.y = fmaf(w1.y, in[k], a1.y); a1.z = fmaf(w1.z, in[k], a1.z); a1.w = fmaf(w1.w, in[k], a1.w);
    }
    if (tb) {
      const float4 t0 = __ldg(tb + 2 * v), t1 = __ldg(tb + 2 * v + 1);
      a0.x += t0.x; a0.y += t0.y; a0.z += t0.z; a0.w += t0.w;
      a1.x += t1.x; a1.y += t1.y; a1.z += t1.z; a1.w += t1.w;
    }
    const float f[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
    __align__(16) __half h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __float2half_rn(hid_act(f[j], act));
    o[v] = *reinterpret_cast<const uint4*>(h);
  }
}

// per-frame message table: table[b][cs][n] = sum_k (2 m[b][k] - 1) wc[cs][n][k]  (fixed order over k)
__global__ void __launch_bounds__(9 * kHidC) hidden_msg_table_kernel(const uint8_t* __restrict__ msgs, int msg_stride, int K,
                                                                     const float* __restrict__ wc, float* __restrict__ table) {
  const int b = blockIdx.x, i = threadIdx.x;   // i = cs * 64 + n
  const uint8_t* m = msgs + (long)b * msg_stride;
  const float* wr = wc + (long)i * K;
  float a = 0.f;
  for (int k = 0; k < K; ++k) a += (m[k] ? 1.f : -1.f) * __ldg(wr + k);
  table[(long)b * 9 * kHidC + i] = a;
}

// GroupNorm(8, 64) partials: part[b][tile][g] = (sum x, sum x^2) in fp64 over the kGnTile pixels of `tile` and the 8 channels of
// group g (one 16-byte vector).  Thread t reads vector g = t & 7 of pixels t / 8 + 32 i.
__global__ void __launch_bounds__(256) hidden_gn_stats_kernel(const __half* __restrict__ y, int hw, double2* __restrict__ part) {
  const int b = blockIdx.y, tile = blockIdx.x, t = threadIdx.x, g = t & 7;
  const uint4* src = reinterpret_cast<const uint4*>(y + ((long)b * hw + (long)tile * kGnTile) * kHidC);
  double s = 0.0, q = 0.0;
  for (int i = t >> 3; i < kGnTile; i += 32) {
    const uint4 u = __ldg(src + (long)i * 8 + g);
    const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const double v = (double)__half2float(h[j]); s += v; q += v * v; }
  }
  // lanes l, l ^ 8, l ^ 16, l ^ 24 share a group
#pragma unroll
  for (int o = 8; o < 32; o <<= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  __shared__ double2 red[8][8];
  if ((t & 31) < 8) red[t >> 5][g] = make_double2(s, q);
  __syncthreads();
  if (t < 8) {
    double2 a = red[0][t];
    for (int w = 1; w < 8; ++w) { a.x += red[w][t].x; a.y += red[w][t].y; }
    part[((long)b * gridDim.x + tile) * 8 + t] = a;
  }
}

// scale / shift of channel c (< 64) of frame b: GroupNorm from the frame's tile partials in tile order, or the identity (part null)
__device__ __forceinline__ void hid_scale_shift(const double2* __restrict__ part, int tiles, int hw, const float* __restrict__ gamma,
                                                const float* __restrict__ beta, int b, int c, float& scale, float& shift) {
  scale = 1.f; shift = 0.f;
  if (!part) return;
  const int g = c >> 3;
  double s = 0.0, q = 0.0;
  for (int i = 0; i < tiles; ++i) { const double2 v = part[((long)b * tiles + i) * 8 + g]; s += v.x; q += v.y; }
  const double n = (double)hw * 8.0, mu = s / n, var = fmax(q / n - mu * mu, 0.0);
  const float rstd = (float)(1.0 / sqrt(var + 1e-5));
  scale = rstd * gamma[c];
  shift = beta[c] - (float)mu * scale;
}

// GroupNorm apply + activation, fp16 map in, fp16 map out.  One thread per 16-byte vector (8 channels: exactly one group), consecutive
// threads on consecutive vectors, so every warp load and store is 512 contiguous bytes; a block covers kGnTile pixels of one frame
// and each thread keeps the one group's 8 scales and shifts in registers.
__global__ void __launch_bounds__(256) hidden_gn_apply_kernel(const __half* __restrict__ y, int hw, const double2* __restrict__ part,
                                                              int tiles, const float* __restrict__ gamma, const float* __restrict__ beta,
                                                              int act, __half* __restrict__ out) {
  __shared__ float sc[kHidC], sh[kHidC];
  const int b = blockIdx.y, t = threadIdx.x;
  if (t < kHidC) hid_scale_shift(part, tiles, hw, gamma, beta, b, t, sc[t], sh[t]);
  __syncthreads();
  const int g = t & 7;   // vector i = t + 256 k holds channels [8 (i & 7), 8 (i & 7) + 8)
  float s8[8], h8[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { s8[j] = sc[g * 8 + j]; h8[j] = sh[g * 8 + j]; }
  const long base = ((long)b * hw + (long)blockIdx.x * kGnTile) * 8;
  const uint4* src = reinterpret_cast<const uint4*>(y) + base;
  uint4* dst = reinterpret_cast<uint4*>(out) + base;
#pragma unroll 4
  for (int i = t; i < kGnTile * 8; i += 256) {
    const uint4 u = __ldg(src + i);
    const __half* h = reinterpret_cast<const __half*>(&u);
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2half_rn(hid_act(fmaf(__half2float(h[j]), s8[j], h8[j]), act));
    dst[i] = *reinterpret_cast<const uint4*>(o);
  }
}

struct HidNormAct {
  const __half* y; int hw;                       // pre-norm map [B*hw][64]
  const double2* part; int tiles;                // GroupNorm partials (nullptr: identity, a folded BatchNorm)
  const float *gamma, *beta;
  int act;
  int mode;                                      // HID_OUTC / HID_POOL (HID_OUT16: hidden_gn_apply_kernel)
  __half* out16;                                 // HID_OUT16
  const float *outc_w, *outc_b; int tanh_; float* delta;   // HID_OUTC: 1x1 conv 64 -> 3 (+ tanh) -> planar fp32 [B][3][hw]
  float* pool_part;                              // HID_POOL: [B][hw / kHidPix][64] block sums
};

// normalisation + activation of a network's last map, fused with its tail (the 1x1 final_layer + tanh, or the spatial mean's block
// sums); one thread per pixel, which needs all 64 channels; a block's pixels belong to one frame
__global__ void __launch_bounds__(kHidPix) hidden_norm_act_kernel(const HidNormAct a) {
  __shared__ float sc[kHidC], sh[kHidC];
  __shared__ float red[kHidPix / 32][kHidC];
  const int b = blockIdx.y, t = threadIdx.x;
  if (t < kHidC) hid_scale_shift(a.part, a.tiles, a.hw, a.gamma, a.beta, b, t, sc[t], sh[t]);
  __syncthreads();
  const long p = (long)blockIdx.x * kHidPix + t;
  const long row = (long)b * a.hw + p;
  const uint4* src = reinterpret_cast<const uint4*>(a.y + row * kHidC);
  float v[kHidC];
#pragma unroll
  for (int q = 0; q < 8; ++q) {
    const uint4 u = __ldg(src + q);
    const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const int c = q * 8 + j; v[c] = hid_act(fmaf(__half2float(h[j]), sc[c], sh[c]), a.act); }
  }
  if (a.mode == HID_OUTC) {
#pragma unroll
    for (int j = 0; j < 3; ++j) {
      float o = __ldg(a.outc_b + j);
#pragma unroll
      for (int c = 0; c < kHidC; ++c) o = fmaf(__ldg(a.outc_w + j * kHidC + c), v[c], o);
      a.delta[((long)b * 3 + j) * a.hw + p] = a.tanh_ ? tanhf(o) : o;
    }
  } else {
    const int lane = t & 31, warp = t >> 5;
#pragma unroll
    for (int c = 0; c < kHidC; ++c) {
      float s = v[c];
#pragma unroll
      for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) red[warp][c] = s;
    }
    __syncthreads();
    if (t < kHidC) {
      float s = red[0][t];
      for (int w = 1; w < kHidPix / 32; ++w) s += red[w][t];
      a.pool_part[((long)b * gridDim.x + blockIdx.x) * kHidC + t] = s;
    }
  }
}

// pooled[b][c] = (sum of the frame's block sums, in block order) / hw
__global__ void hidden_pool_kernel(const float* __restrict__ part, int nblk, int hw, float* __restrict__ pooled) {
  const int b = blockIdx.x, c = threadIdx.x;
  float s = 0.f;
  for (int i = 0; i < nblk; ++i) s += part[((long)b * nblk + i) * kHidC + c];
  pooled[(long)b * kHidC + c] = s / (float)hw;
}

struct Hidden {
  bool on = false;
  bool embedder = false;   // the encoder (embedder) or the decoder (extractor)
  vsb_hidden_desc h{};
  int nbits = 0, nsm = 0;

  // ---- packed weights
  struct Layer { float *w3 = nullptr, *b3 = nullptr; ConvW cw; const float *gamma = nullptr, *beta = nullptr; };
  std::vector<Layer> layers;   // conv_bns / layers
  Layer cat_x;                 // the concat layer: its image columns (hidden_c3_kernel) and its enc columns (cw)
  float* msg_wc = nullptr;     // [9][64][K] message columns summed over the valid taps of each border case
  float *fin_w = nullptr, *fin_b = nullptr;   // final_layer [3][64] / linear [1+K][64]

  bool group() const { return h.norm == 1; }
  int act() const { return h.act == 1 ? ACT_GELU : ACT_RELU; }

  // vsb_model_set_hidden_embedder / _extractor: the rules (no CUDA calls)
  void set(const vsb_hidden_desc& desc, bool emb, const vsb_model_desc& d) {
    VSB_CHECK(desc.num_layers >= 1 && desc.num_layers <= 64, "HiDDeN: 1 to 64 conv layers");
    VSB_CHECK(desc.last_tanh == 0 || desc.last_tanh == 1, "HiDDeN: last_tanh must be 0 or 1");
    VSB_CHECK(emb || desc.last_tanh == 0, "HiDDeN extractor: last_tanh must be 0");
    if (desc.norm != 0 && desc.norm != 1)
      throw Error("HiDDeN: only BatchNorm (0) and GroupNorm (1) are implemented", kErrUnsupported);
    if (desc.act != 0 && desc.act != 1) throw Error("HiDDeN: only ReLU (0) and GELU (1) are implemented", kErrUnsupported);
    if (desc.z_channels != kHidC)
      throw Error("HiDDeN width " + std::to_string(desc.z_channels) + " is not implemented (z_channels 64)", kErrUnsupported);
    VSB_CHECK(d.nbits >= 1, "nbits must be at least 1");
    // the tensor-core conv tiles maps by 128 pixels, the statistics by kGnTile
    VSB_CHECK(d.img_size >= 128 && d.img_size % 128 == 0, "processing size must be a positive multiple of 128");
    h = desc; embedder = emb; nbits = d.nbits; on = true;
  }

  static std::vector<float> ones(int n) { return std::vector<float>(n, 1.f); }
  // ConvBNRelu `key` (".layers.0" conv, ".layers.1" norm): the output scale and bias of the conv with a BatchNorm folded in
  void fold(Weights& ws, const std::string& key, std::vector<float>& s, std::vector<float>& b, Layer& L) const {
    const std::vector<float>& cb = ws.get(key + ".layers.0.bias").data;
    VSB_CHECK((int)cb.size() == kHidC, key + ": conv bias shape");
    if (group()) {
      s = ones(kHidC); b = cb;
      L.gamma = ws.vec(key + ".layers.1.weight", kHidC);
      L.beta = ws.vec(key + ".layers.1.bias", kHidC);
    } else {
      ws.bn_fold(key + ".layers.1", s, b);
      for (int n = 0; n < kHidC; ++n) b[n] += s[n] * cb[n];
    }
  }
  // image columns [c0, c0 + 3) of the 3x3 weight `w` [64][Ct][3][3], times s[n] -> the [27][64] layout of hidden_c3_kernel
  static std::vector<float> c3_weights(const HostTensor& w, int c0, const std::vector<float>& s) {
    const int Ct = (int)w.shape[1];
    std::vector<float> o((size_t)27 * kHidC);
    for (int n = 0; n < kHidC; ++n)
      for (int k = 0; k < 27; ++k) o[(size_t)k * kHidC + n] = s[n] * w.data[((size_t)n * Ct + c0 + k / 9) * 9 + k % 9];
    return o;
  }
  // input channels [c0, c0 + C) of a 3x3 weight as a 4-D tensor
  static HostTensor columns(const HostTensor& w, int c0, int C) {
    const int Ct = (int)w.shape[1];
    HostTensor t; t.shape = {w.shape[0], C, 3, 3};
    t.data.resize((size_t)w.shape[0] * C * 9);
    for (int64_t n = 0; n < w.shape[0]; ++n)
      for (int c = 0; c < C; ++c)
        for (int k = 0; k < 9; ++k) t.data[((size_t)n * C + c) * 9 + k] = w.data[((size_t)n * Ct + c0 + c) * 9 + k];
    return t;
  }
  const HostTensor& conv_w(Weights& ws, const std::string& key, int cin) const {
    const HostTensor& w = ws.get(key + ".layers.0.weight");
    VSB_CHECK(w.shape.size() == 4 && w.shape[0] == kHidC && w.shape[1] == cin && w.shape[2] == 3 && w.shape[3] == 3,
              key + ": expected a [64][" + std::to_string(cin) + "][3][3] conv (in_channels 3, z_channels 64)");
    return w;
  }

  void pack(Weights& ws, int num_sms) {
    nsm = num_sms;
    const std::string P = embedder ? "embedder.hidden_encoder." : "detector.hidden_decoder.";
    const std::string blk = embedder ? "conv_bns." : "layers.";
    std::vector<float> s, b;
    for (int i = 0; i < h.num_layers; ++i) {
      const std::string key = P + blk + std::to_string(i);
      Layer L;
      fold(ws, key, s, b, L);
      const HostTensor& w = conv_w(ws, key, i == 0 ? 3 : kHidC);
      if (i == 0) { L.w3 = ws.pool.upload(c3_weights(w, 0, s)); L.b3 = ws.pool.upload(b); }
      else L.cw = ws.gemm(conv_taps(w, &s), b);
      layers.push_back(L);
    }
    if (embedder) {
      const std::string key = P + "after_concat_layer";
      const int K = nbits;
      fold(ws, key, s, b, cat_x);
      const HostTensor& w = conv_w(ws, key, K + kHidC + 3);
      // channel order of the reference's concat: [m (K) | enc (64) | x (3)]
      cat_x.w3 = ws.pool.upload(c3_weights(w, K + kHidC, s));
      cat_x.cw = ws.gemm(conv_taps(columns(w, K, kHidC), &s), b);
      std::vector<float> wc((size_t)9 * kHidC * K, 0.f);
      for (int cs = 0; cs < 9; ++cs) {
        const int rc = cs / 3, cc = cs % 3;   // 0: first row / column (tap 0 outside), 2: last (tap 2 outside)
        for (int n = 0; n < kHidC; ++n)
          for (int k = 0; k < K; ++k) {
            float a = 0.f;
            for (int r = 0; r < 3; ++r)
              for (int c = 0; c < 3; ++c)
                if (!(rc == 0 && r == 0) && !(rc == 2 && r == 2) && !(cc == 0 && c == 0) && !(cc == 2 && c == 2))
                  a += w.data[((size_t)n * (K + kHidC + 3) + k) * 9 + r * 3 + c];
            wc[((size_t)cs * kHidC + n) * K + k] = s[n] * a;
          }
      }
      msg_wc = ws.pool.upload(wc);
      fin_w = ws.vec(P + "final_layer.weight", 3 * kHidC);
      fin_b = ws.vec(P + "final_layer.bias", 3);
    } else {
      const HostTensor& lw = ws.get(P + "linear.weight");
      VSB_CHECK(lw.shape.size() == 2 && lw.shape[0] == 1 + nbits && lw.shape[1] == kHidC,
                P + "linear.weight: expected [1 + nbits][64] (a pooled HiDDeN decoder)");
      fin_w = ws.vec(P + "linear.weight");
      fin_b = ws.vec(P + "linear.bias", 1 + nbits);
    }
  }

  // GroupNorm statistics of the pre-norm map y, then the normalisation and activation in `mode`; identity scale for BatchNorm
  void add_norm_act(Plan& pl, const std::string& name, const __half* y, int B, int S, const Layer& L, HidNormAct a) const {
    const int hw = S * S, tiles = hw / kGnTile;
    const std::string at = "@" + std::to_string(S);
    a.y = y; a.hw = hw; a.part = nullptr; a.tiles = tiles; a.act = act();
    if (group()) {
      double2* part = pl.pool.alloc_n<double2>((size_t)B * tiles * 8);
      pl.add("hidden.gn_stats" + at, [=](cudaStream_t st) {
        hidden_gn_stats_kernel<<<dim3(tiles, B), 256, 0, st>>>(y, hw, part);
        VSB_CUDA(cudaGetLastError());
      });
      pl.tap(name + ".stats", part, 0, B, tiles, 8, 4, 4);   // fp64 (sum, sum of squares) pairs as four fp32 words each
      a.part = part; a.gamma = L.gamma; a.beta = L.beta;
    }
    if (a.mode == HID_OUT16) {
      VSB_CHECK(group(), "HiDDeN: a BatchNorm layer applies its activation in the conv epilogue");
      const double2* part = a.part;
      const float *g = a.gamma, *be = a.beta;
      const int ac = a.act;
      __half* out = a.out16;
      pl.add("hidden.gn_apply" + at, [=](cudaStream_t st) {
        hidden_gn_apply_kernel<<<dim3(tiles, B), 256, 0, st>>>(y, hw, part, tiles, g, be, ac, out);
        VSB_CUDA(cudaGetLastError());
      });
      return;
    }
    pl.add(std::string(group() ? "hidden.gn_apply" : "hidden.act") + (a.mode == HID_OUTC ? "+outc" : "+pool") + at, [=](cudaStream_t st) {
      hidden_norm_act_kernel<<<dim3(hw / kHidPix, B), kHidPix, 0, st>>>(a);
      VSB_CUDA(cudaGetLastError());
    });
  }

  // the plan of B frames at S x S: the embed plan (-> pl.delta [B][3][S][S]) or the detect plan (-> pl.logits [B][1 + nbits]).
  // keep (test seam, vsb_debug_keep_inputs): copy layers 0 and 1's pre-norm maps (GroupNorm) and outputs aside before later layers
  // overwrite them, as taps <henc|hdec>.{0,1}.pre and <henc|hdec>.{0,1}.
  void build(Plan& pl, int B, int S, bool keep = false) const {
    const long M = (long)B * S * S;
    const int hw = S * S;
    const long fstride = (long)3 * hw;
    const std::string at = "@" + std::to_string(S);
    Plan* plp = &pl;
    const int nl = h.num_layers, a_fused = group() ? ACT_NONE : act();
    __half* pre = pl.pool.alloc_n<__half>(M * kHidC);   // pre-norm map of GroupNorm layers
    __half* bufs[2] = {pl.pool.alloc_n<__half>(M * kHidC), pl.pool.alloc_n<__half>(M * kHidC)};
    const __half* x = nullptr;
    const std::string tp = embedder ? "henc." : "hdec.";
    for (int i = 0; i < nl; ++i) {
      const Layer& L = layers[i];
      const bool last = !embedder && i == nl - 1;
      // where the conv writes: the layer's output (BatchNorm, not last) or the pre-norm map
      const bool direct = !group() && !last;
      __half* out = bufs[i & 1];
      __half* y = direct ? out : pre;
      const int ea = direct ? a_fused : ACT_NONE;
      if (i == 0) {
        const float *w3 = L.w3, *b3 = L.b3;
        pl.add("hidden.conv3x3.3-64" + at, [=](cudaStream_t st) {
          hidden_c3_kernel<<<dim3(hw / kHidPix, B), kHidPix, 0, st>>>(plp->in_imgs, fstride, S, w3, b3, nullptr, ea, y);
          VSB_CUDA(cudaGetLastError());
        });
      } else {
        ConvGemmOp op;
        setup_tma_conv(op, x, B, S, S, kHidC, kHidC, 3, 3, 1);
        op.p.epi = EPI_AFFINE; op.p.act = ea; op.p.bias = L.cw.bias; op.p.out16 = y; op.p.ld_out16 = kHidC;
        vsb::add_conv(pl, op, L.cw, "hidden.conv3x3.64-64" + at, nsm);
      }
      // taps: only buffers that no later step overwrites (the maps ping-pong between two buffers and share one pre-norm map)
      if (last) {
        pl.tap(tp + std::to_string(i) + ".pre", pre, 1, B, S, S, kHidC, kHidC);
        float* pp = pl.pool.alloc_n<float>((size_t)B * (hw / kHidPix) * kHidC);
        HidNormAct a{};
        a.mode = HID_POOL; a.pool_part = pp;
        add_norm_act(pl, tp + std::to_string(i), pre, B, S, L, a);
        float* pooled = pl.pool.alloc_n<float>((size_t)B * kHidC);
        const int nblk = hw / kHidPix, NO = 1 + nbits;
        const float *lw = fin_w, *lb = fin_b;
        float* logits = pl.logits;
        pl.add("hidden.pool+linear", [=](cudaStream_t st) {
          hidden_pool_kernel<<<B, kHidC, 0, st>>>(pp, nblk, hw, pooled);
          head_linear_kernel<<<(int)(((long)B * NO + 7) / 8), 256, 0, st>>>(pooled, lw, lb, B, kHidC, NO, logits);
          VSB_CUDA(cudaGetLastError());
        }, 2);
        pl.tap("head_pooled", pooled, 0, B, 1, 1, kHidC, kHidC);
        return;
      }
      if (group()) {
        HidNormAct a{};
        a.mode = HID_OUT16; a.out16 = out;
        add_norm_act(pl, tp + std::to_string(i), pre, B, S, L, a);
      }
      // the encoder's last map (the concat reads it); the decoder's last two before its pooled layer (its conv reads the second)
      if (embedder ? i == nl - 1 : i >= nl - 3) pl.tap(tp + std::to_string(i), out, 1, B, S, S, kHidC, kHidC);
      if (keep && i < 2) {
        const size_t bytes = (size_t)M * kHidC * sizeof(__half);
        std::vector<std::pair<const __half*, __half*>> cp{{out, pl.pool.alloc_n<__half>(M * kHidC)}};
        pl.tap(tp + std::to_string(i), cp[0].second, 1, B, S, S, kHidC, kHidC);
        if (group()) {
          cp.push_back({pre, pl.pool.alloc_n<__half>(M * kHidC)});
          pl.tap(tp + std::to_string(i) + ".pre", cp[1].second, 1, B, S, S, kHidC, kHidC);
        }
        pl.add("hidden.keep", [=](cudaStream_t st) {
          for (auto& c : cp) VSB_CUDA(cudaMemcpyAsync(c.second, c.first, bytes, cudaMemcpyDeviceToDevice, st));
        }, 0);
      }
      x = out;
    }
    // ---- encoder: message table, image columns + table, enc columns (tensor cores), norm + act + final_layer (+ tanh)
    float* table = pl.pool.alloc_n<float>((size_t)B * 9 * kHidC);
    __half* r = bufs[nl & 1];   // the image columns' conv + message table (the buffer the enc map does not occupy)
    {
      const int K = nbits;
      const float* wc = msg_wc;
      pl.add("hidden.msg_table", [=](cudaStream_t st) {
        hidden_msg_table_kernel<<<B, 9 * kHidC, 0, st>>>(plp->in_msgs, plp->in_msg_stride, K, wc, table);
        VSB_CUDA(cudaGetLastError());
      });
      pl.tap("henc.msg_table", table, 0, B, 9, 1, kHidC, kHidC);
      const float* w3 = cat_x.w3;
      pl.add("hidden.concat_x+msg" + at, [=](cudaStream_t st) {
        hidden_c3_kernel<<<dim3(hw / kHidPix, B), kHidPix, 0, st>>>(plp->in_imgs, fstride, S, w3, nullptr, table, ACT_NONE, r);
        VSB_CUDA(cudaGetLastError());
      });
      pl.tap("henc.cat_x", r, 1, B, S, S, kHidC, kHidC);
    }
    {
      ConvGemmOp op;
      setup_tma_conv(op, x, B, S, S, kHidC, kHidC, 3, 3, 1);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = cat_x.cw.bias; op.p.out16 = pre; op.p.ld_out16 = kHidC;
      op.p.resid16 = r; op.p.ld_res16 = kHidC;
      vsb::add_conv(pl, op, cat_x.cw, "hidden.concat_conv3x3.64-64" + at, nsm);
      pl.tap("henc.cat.pre", pre, 1, B, S, S, kHidC, kHidC);
    }
    pl.delta = pl.pool.alloc_n<float>((size_t)B * 3 * hw);
    HidNormAct a{};
    a.mode = HID_OUTC; a.outc_w = fin_w; a.outc_b = fin_b; a.tanh_ = h.last_tanh; a.delta = pl.delta;
    add_norm_act(pl, "henc.cat", pre, B, S, cat_x, a);
    pl.tap("delta", pl.delta, 0, B, 3, S, S, S);
  }
};

}  // namespace vsb
