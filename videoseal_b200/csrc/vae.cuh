// The VAE embedder (modules/vae.py VAEEncoder / VAEDecoder, modules/msg_processor.py 'binary+concat'; models/embedder.py
// VAEEmbedder, build_embedder 'vae*'): decoder(msg_processor(encoder(2 imgs - 1), msgs)).  Its rules, kernels, packed weights and
// plans.  L levels of widths w[l] = ch * ch_mult[l], maps S / 2^l; a ResnetBlock (cin -> cout) is
//   h = conv1(silu(GN1(x))), out = shortcut(x) + conv2(silu(GN2(h))),  shortcut = x (cin == cout) or the 1x1 nin_shortcut,
// GN = GroupNorm(16, C, eps 1e-6, affine); the mid AttnBlock is x + proj_out(softmax(q k^T / sqrt(C)) v) with q, k, v 1x1 convs
// of GN(x) and one head over the whole (S / 2^(L-1))^2 grid.
//   encoder   conv_in (in_ch -> ch) at S; per level num_res_blocks ResnetBlocks, then (not the last) Downsample = pad (0,1,0,1) +
//             3x3 stride 2; mid ResnetBlock, AttnBlock, ResnetBlock; silu(GN) + conv_out (-> z): the latent
//   message   aux[b] = sum_k E[2k + m_bk] (hidden values), concatenated as `hidden` constant planes after the latent
//   decoder   conv_in (z + hidden -> w[L-1]); mid; per level from the deepest num_res_blocks + 1 ResnetBlocks, then (not level 0)
//             Upsample = nearest x2 + 3x3; silu(GN) + conv_out (-> out_ch), tanh when tanh_out: the delta
//
// Kernels:
//   vae_conv_in_kernel          encoder conv_in on CUDA cores from the planar fp32 frames: x = 2 imgs - 1, or for 1 input channel
//                               x = 2 Y - 1 with the U-Net first layer's Y arithmetic.
//   vae_gn_stats_kernel /       GroupNorm(16) statistics, deterministic and atomic-free as hidden_gn_stats_kernel: fp64 (sum, sum of
//   vae_gn_finalize_kernel      squares) partials per tile of kVaeGnTile pixels of one frame in a fixed order, then per frame and group
//                               a fixed-order reduction to (mean, rstd).  A frame's statistics depend on its own pixels only.
//   vae_gn_apply_kernel         (x - mu) rstd gamma + beta, then SiLU (ResnetBlock, norm_out) or nothing (AttnBlock): the fp16 operand
//                               of the next conv.
//   tensor-core TMA conv        every stride-1 3x3 conv and the 1x1 nin_shortcut / qkv / proj_out GEMMs, bias in the epilogue;
//                               conv2 and proj_out add the shortcut as the fp16 residual of their epilogue.  A map that does
//                               not tile by 128 pixels (a side that is neither 16, 32, 64 nor a multiple of 128: 192 and 96
//                               at 768, three of the four levels at 384 and 640) runs its 3x3 convs on the gather loader.
//   gather conv                 Downsample: stride 2, pad 0 (the loader's bounds test zero-fills the last row and column, which is
//                               the reference's asymmetric pad); Upsample: the gather loader's nearest x2 index mode (pad_mode 2)
//                               reads the low-resolution map, so the up-sampled map is never written and the products are the
//                               reference's.
//   vit_attention_kernel        one head, the whole grid, head dim 64 or 128 (attention.cuh), on the qkv GEMM's [M][3C] rows.
//   conv_out (encoder)          the TMA conv with N padded to 16 writes the fp32 latent [B][hw][16].
//   vae_msg_table_kernel        aux per frame, then table[b][cs][n] = sum_j wc[cs][n][j] aux[b][j]: wc is decoder.conv_in's message
//                               columns summed over the valid taps of each of the 9 zero-padding border cases (HiDDeN's folding),
//                               so the concat [latent | aux planes] is never materialised.
//   vae_dec_conv_in_kernel      decoder conv_in over the fp32 latent on CUDA cores (K = 9 z) + bias + table[case].
//   conv_out (decoder)          the TMA conv with N padded to 16 and the fused 1x1 outc epilogue as the identity on the first out_ch
//                               columns (+ tanh) writes the planar fp32 delta with no extra pass (as DVMark's output layer).
// No float atomics anywhere: imgs_w is bit-identical from run to run and for any split of the frames into sub-batches.
#pragma once
#include "attention_host.cuh"
#include "weights.cuh"

namespace vsb {

constexpr int kVaeGroups = 16;      // GroupNorm(16, C)
constexpr int kVaeGnTile = 256;     // pixels per statistics partial: every level's map (>= 16 x 16) is whole tiles
constexpr int kVaeMaxSize = 768;    // a 64-frame vae_big plan at 768^2 holds ~20 GB of maps (DESIGN row a13g)
constexpr int kVaeMaxZ = 16;        // latent channels: conv_out's N is padded to 16
constexpr int kVaeMaxLevels = 6;
constexpr int kVaeMaxGrid = 96;     // the deepest map's side: the single-head attention runs over at most 96^2 = 9 216 tokens

__device__ __forceinline__ float vae_silu(float v) { return v / (1.f + __expf(-v)); }

// encoder conv_in: CIN = 3 (x = 2 imgs - 1) or 1 (x = 2 Y - 1); planar fp32 [B][3][S][S] in, NHWC fp16 [B*S*S][cout] out.
// w [9 CIN][cout] fp32 (k = c * 9 + r * 3 + s), bias [cout]; one thread per pixel, 8 output channels per 16-byte store.
template <int CIN>
__global__ void __launch_bounds__(256) vae_conv_in_kernel(const float* __restrict__ imgs, long fstride, int S,
                                                          const float* __restrict__ w, const float* __restrict__ bias, int cout,
                                                          __half* __restrict__ out) {
  const int b = blockIdx.y;
  const long p = (long)blockIdx.x * 256 + threadIdx.x;
  const long hw = (long)S * S;
  if (p >= hw) return;
  const int y = (int)(p / S), x = (int)(p % S);
  const float* im = imgs + (long)b * fstride;
  float in[CIN * 9];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int s = 0; s < 3; ++s) {
      const int yy = y + r - 1, xx = x + s - 1;
      const bool ok = yy >= 0 && yy < S && xx >= 0 && xx < S;
      const long o = (long)yy * S + xx;
      if (CIN == 1) {
        float v = 0.f;
        if (ok) {
          const float Y = 0.299f * __ldg(im + o) + 0.587f * __ldg(im + hw + o) + 0.114f * __ldg(im + 2 * hw + o);
          v = 2.f * Y - 1.f;
        }
        in[r * 3 + s] = v;
      } else {
#pragma unroll
        for (int c = 0; c < CIN; ++c) in[c * 9 + r * 3 + s] = ok ? 2.f * __ldg(im + c * hw + o) - 1.f : 0.f;
      }
    }
  uint4* dst = reinterpret_cast<uint4*>(out + ((long)b * hw + p) * cout);
  for (int n0 = 0; n0 < cout; n0 += 8) {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = __ldg(bias + n0 + j);
#pragma unroll
    for (int k = 0; k < CIN * 9; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] = fmaf(__ldg(w + k * cout + n0 + j), in[k], a[j]);
    __align__(16) __half h[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) h[j] = __float2half_rn(a[j]);
    dst[n0 / 8] = *reinterpret_cast<const uint4*>(h);
  }
}

// GroupNorm(16, C) partials, C in {16, 32, 64, 128}: part[b][tile][g] = (sum x, sum x^2) in fp64 over the kVaeGnTile pixels of
// `tile` and the C / 16 channels of group g.  Thread t reads channel vector t % V (V = C / 8) of pixels t / V + k (256 / V); the
// per-thread channel sums meet in shared memory and are added per group in thread order.
__global__ void __launch_bounds__(256) vae_gn_stats_kernel(const __half* __restrict__ y, int hw, int C, double2* __restrict__ part) {
  __shared__ double2 red[256][8];
  const int b = blockIdx.y, tile = blockIdx.x, t = threadIdx.x, V = C / 8, v = t % V;
  const uint4* src = reinterpret_cast<const uint4*>(y + ((long)b * hw + (long)tile * kVaeGnTile) * C);
  double s[8], q[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) { s[j] = 0.0; q[j] = 0.0; }
  for (int i = t / V; i < kVaeGnTile; i += 256 / V) {
    const uint4 u = __ldg(src + (long)i * V + v);
    const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
    for (int j = 0; j < 8; ++j) { const double x = (double)__half2float(h[j]); s[j] += x; q[j] += x * x; }
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) red[t][j] = make_double2(s[j], q[j]);
  __syncthreads();
  if (t < kVaeGroups) {
    const int gs = C / kVaeGroups;
    double2 a = make_double2(0.0, 0.0);
    for (int c = t * gs; c < (t + 1) * gs; ++c)
      for (int tt = c / 8; tt < 256; tt += V) { a.x += red[tt][c % 8].x; a.y += red[tt][c % 8].y; }
    part[((long)b * gridDim.x + tile) * kVaeGroups + t] = a;
  }
}

// stat[b][g] = (mean, 1 / sqrt(var + eps)) of group g of frame b from its `tiles` partials; warp g adds them lane-strided, then in a
// fixed shuffle tree
__global__ void __launch_bounds__(32 * kVaeGroups) vae_gn_finalize_kernel(const double2* __restrict__ part, int tiles, double n,
                                                                          float eps, float2* __restrict__ stat) {
  const int b = blockIdx.x, g = threadIdx.x >> 5, lane = threadIdx.x & 31;
  double s = 0.0, q = 0.0;
  for (int i = lane; i < tiles; i += 32) { const double2 v = part[((long)b * tiles + i) * kVaeGroups + g]; s += v.x; q += v.y; }
#pragma unroll
  for (int o = 16; o; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
  if (lane == 0) {
    const double mu = s / n, var = fmax(q / n - mu * mu, 0.0);
    stat[b * kVaeGroups + g] = make_float2((float)mu, (float)(1.0 / sqrt(var + (double)eps)));
  }
}

// out = act((y - mu) rstd gamma + beta), fp16 NHWC [B][hw][C] in and out; act SiLU (silu = 1) or none.  One 16-byte vector per thread.
__global__ void __launch_bounds__(256) vae_gn_apply_kernel(const __half* __restrict__ y, long hw, int C, const float2* __restrict__ stat,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta, int silu,
                                                           long total, __half* __restrict__ out) {
  const int V = C / 8, gs = C / kVaeGroups;
  for (long i = blockIdx.x * (long)blockDim.x + threadIdx.x; i < total; i += (long)gridDim.x * blockDim.x) {
    const int c8 = (int)(i % V) * 8;
    const int b = (int)(i / ((long)hw * V));
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(y) + i);
    const __half* h = reinterpret_cast<const __half*>(&u);
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c8 + j;
      const float2 st = __ldg(stat + b * kVaeGroups + c / gs);
      const float sc = st.y * __ldg(gamma + c), sh = __ldg(beta + c) - st.x * sc;
      float v = fmaf(__half2float(h[j]), sc, sh);
      if (silu) v = vae_silu(v);
      o[j] = __float2half_rn(v);
    }
    reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(o);
  }
}

// per frame: aux[j] = sum_k E[2k + m_k][j] (fixed order over k), then table[b][i] = sum_j wc[i][j] aux[j] for i = cs * C + n.
// Dynamic shared memory: hidden floats.
__global__ void __launch_bounds__(256) vae_msg_table_kernel(const uint8_t* __restrict__ msgs, int msg_stride, int K, int hidden,
                                                            const float* __restrict__ emb, const float* __restrict__ wc, int C,
                                                            float* __restrict__ table) {
  extern __shared__ float aux[];
  const int b = blockIdx.x;
  const uint8_t* m = msgs + (long)b * msg_stride;
  for (int j = threadIdx.x; j < hidden; j += blockDim.x) {
    float a = 0.f;
    for (int k = 0; k < K; ++k) a += __ldg(emb + (long)(2 * k + (m[k] ? 1 : 0)) * hidden + j);
    aux[j] = a;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 9 * C; i += blockDim.x) {
    const float* wr = wc + (long)i * hidden;
    float a = 0.f;
    for (int j = 0; j < hidden; ++j) a = fmaf(__ldg(wr + j), aux[j], a);
    table[(long)b * 9 * C + i] = a;
  }
}

// decoder conv_in over the latent columns: lat fp32 [B][h*h][kVaeMaxZ] (z used), w [9 z][C] (k = c * 9 + r * 3 + s), bias [C],
// table [B][9][C] (the message planes' contribution by border case) -> NHWC fp16 [B][h*h][C].  One thread per pixel.
__global__ void __launch_bounds__(256) vae_dec_conv_in_kernel(const float* __restrict__ lat, int h, int z, const float* __restrict__ w,
                                                              const float* __restrict__ bias, const float* __restrict__ table, int C,
                                                              __half* __restrict__ out) {
  const int b = blockIdx.y;
  const long hw = (long)h * h, p = (long)blockIdx.x * 256 + threadIdx.x;
  if (p >= hw) return;
  const int y = (int)(p / h), x = (int)(p % h);
  const int cs = (y == 0 ? 0 : (y == h - 1 ? 2 : 1)) * 3 + (x == 0 ? 0 : (x == h - 1 ? 2 : 1));
  const float* tb = table + ((long)b * 9 + cs) * C;
  const float* lb = lat + (long)b * hw * kVaeMaxZ;
  uint4* dst = reinterpret_cast<uint4*>(out + ((long)b * hw + p) * C);
  for (int n0 = 0; n0 < C; n0 += 8) {
    float a[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) a[j] = __ldg(bias + n0 + j);
    for (int r = 0; r < 3; ++r)
      for (int s = 0; s < 3; ++s) {
        const int yy = y + r - 1, xx = x + s - 1;
        if (yy < 0 || yy >= h || xx < 0 || xx >= h) continue;
        const float* lp = lb + ((long)yy * h + xx) * kVaeMaxZ;
        for (int c = 0; c < z; ++c) {
          const float v = __ldg(lp + c);
          const float* wr = w + (long)(c * 9 + r * 3 + s) * C + n0;
#pragma unroll
          for (int j = 0; j < 8; ++j) a[j] = fmaf(__ldg(wr + j), v, a[j]);
        }
      }
    __align__(16) __half o[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) o[j] = __float2half_rn(a[j] + __ldg(tb + n0 + j));
    dst[n0 / 8] = *reinterpret_cast<const uint4*>(o);
  }
}

struct VaeEnc {
  bool on = false;
  vsb_vae_desc v{};
  int nbits = 0, hidden = 0, nsm = 0;

  // ---- packed weights
  struct GN { const float *gamma = nullptr, *beta = nullptr; };
  struct Res { int cin = 0, cout = 0; GN n1, n2; ConvW c1, c2, nin; };
  struct Attn { GN n; ConvW qkv, proj; };
  struct Net { std::vector<std::vector<Res>> lv; std::vector<ConvW> resamp; Res m1, m2; Attn at; GN nout; };
  Net enc, dec;
  float *ci_w = nullptr, *ci_b = nullptr;            // encoder conv_in [9 in_ch][ch]
  ConvW e_out;                                       // encoder conv_out, N padded to 16
  float *dci_w = nullptr, *dci_b = nullptr;          // decoder conv_in latent columns [9 z][C_last]
  float *msg_wc = nullptr, *emb = nullptr;           // [9][C_last][hidden] folded message columns; the embedding table
  ConvW d_out;                                       // decoder conv_out, N padded to 16
  float *id_w = nullptr, *zero_b = nullptr;          // the identity outc [out_ch][16] and its zero bias

  int width(int l) const { return v.ch * v.ch_mult[l]; }
  static bool width_ok(int c) { return c == 16 || c == 32 || c == 64 || c == 128; }

  // vsb_model_set_vae_embedder: the rules (no CUDA calls)
  void set(const vsb_vae_desc& desc, const vsb_model_desc& d) {
    VSB_CHECK(desc.in_ch == 1 || desc.in_ch == 3, "VAE embedder: in_ch must be 1 or 3");
    VSB_CHECK((d.yuv != 0) == (desc.in_ch == 1), "VAE embedder: yuv cards take the Y channel (in_ch 1), the others RGB (in_ch 3)");
    VSB_CHECK(desc.levels >= 1 && desc.levels <= kVaeMaxLevels, "VAE embedder: 1 to 6 levels (len(ch_mult))");
    VSB_CHECK(desc.num_res_blocks >= 1 && desc.num_res_blocks <= 8, "VAE embedder: num_res_blocks must be 1 to 8");
    VSB_CHECK(desc.tanh_out == 0 || desc.tanh_out == 1, "VAE embedder: tanh_out must be 0 or 1");
    VSB_CHECK(desc.z_channels >= 1 && desc.ch >= 1 && desc.out_ch >= 1, "VAE embedder: positive widths");
    VSB_CHECK(d.nbits >= 1 && d.hidden >= 1, "VAE embedder: nbits and hidden must be at least 1");
    if (desc.out_ch != 1 && desc.out_ch != 3)
      throw Error("VAE embedder: out_ch " + std::to_string(desc.out_ch) + " is not implemented (1 or 3)", kErrUnsupported);
    if (desc.z_channels > kVaeMaxZ)
      throw Error("VAE embedder: z_channels " + std::to_string(desc.z_channels) + " is not implemented (at most 16)", kErrUnsupported);
    if (!width_ok(desc.ch)) throw Error("VAE embedder: ch " + std::to_string(desc.ch) + " is not implemented (16, 32, 64 or 128)", kErrUnsupported);
    for (int l = 0; l < desc.levels; ++l) {
      VSB_CHECK(desc.ch_mult[l] >= 1, "VAE embedder: ch_mult must be positive");
      const int w = desc.ch * desc.ch_mult[l];
      if (!width_ok(w))
        throw Error("VAE embedder: level width " + std::to_string(w) + " is not implemented (16, 32, 64 or 128)", kErrUnsupported);
    }
    const int hd = desc.ch * desc.ch_mult[desc.levels - 1];
    if (hd != 64 && hd != 128)
      throw Error("VAE embedder: last-level width (the attention head dim) " + std::to_string(hd) + " is not implemented (64 or 128)",
                  kErrUnsupported);
    // every map tiles the statistics by 256 pixels: the deepest map is at least 16 x 16; the AttnBlock attends over the whole deepest
    // map, which is at most kVaeMaxGrid wide (9 216 tokens, the largest grid the attention was sized and measured for)
    const int S = d.img_size, lowest = S >> (desc.levels - 1);
    if (S < 128 || S % 128 != 0 || S > kVaeMaxSize || (lowest << (desc.levels - 1)) != S || lowest < 16 || lowest % 16 != 0 ||
        lowest > kVaeMaxGrid)
      throw Error("VAE embedder: processing size " + std::to_string(S) + " is not implemented with " + std::to_string(desc.levels) +
                  " levels (a multiple of 128, at most " + std::to_string(kVaeMaxSize) + ", whose deepest map is a multiple of 16 "
                  "pixels wide and at most " + std::to_string(kVaeMaxGrid) + ")", kErrUnsupported);
    v = desc; nbits = d.nbits; hidden = d.hidden; on = true;
  }

  // ---- packing
  static const HostTensor& shaped(Weights& ws, const std::string& k, std::vector<int64_t> shape) {
    const HostTensor& t = ws.get(k);
    std::string want;
    for (auto s : shape) want += "[" + std::to_string(s) + "]";
    VSB_CHECK(t.shape == shape, k + ": expected a " + want + " tensor (VAE embedder)");
    return t;
  }
  static GN gn(Weights& ws, const std::string& k, int C) { return {ws.vec(k + ".weight", C), ws.vec(k + ".bias", C)}; }
  // conv `k` [cout][cin][R][R] with rows zero-padded to cout_pad
  static ConvW conv(Weights& ws, const std::string& k, int cin, int cout, int R, int cout_pad = 0) {
    HostTensor w = shaped(ws, k + ".weight", {cout, cin, R, R});
    const std::vector<float>& b = shaped(ws, k + ".bias", {cout}).data;
    std::vector<float> bias(b);
    if (cout_pad > cout) {
      w.shape[0] = cout_pad;
      w.data.resize((size_t)cout_pad * cin * R * R, 0.f);
      bias.resize(cout_pad, 0.f);
    }
    return ws.gemm(conv_taps(w), bias);
  }
  static Res res(Weights& ws, const std::string& k, int cin, int cout) {
    Res r;
    r.cin = cin; r.cout = cout;
    r.n1 = gn(ws, k + ".norm1", cin);
    r.c1 = conv(ws, k + ".conv1", cin, cout, 3);
    r.n2 = gn(ws, k + ".norm2", cout);
    r.c2 = conv(ws, k + ".conv2", cout, cout, 3);
    if (cin != cout) r.nin = conv(ws, k + ".nin_shortcut", cin, cout, 1);
    return r;
  }
  // AttnBlock: q, k, v as one [3C][C] GEMM (rows q | k | v: vit_attention_kernel's (3, heads = 1, hd) columns), proj_out
  static Attn attn(Weights& ws, const std::string& k, int C) {
    Attn a;
    a.n = gn(ws, k + ".norm", C);
    HostTensor w;
    w.shape = {3 * C, C};
    std::vector<float> b;
    for (const char* m : {".q", ".k", ".v"}) {
      const HostTensor& t = shaped(ws, k + m + ".weight", {C, C, 1, 1});
      w.data.insert(w.data.end(), t.data.begin(), t.data.end());
      const std::vector<float>& tb = shaped(ws, k + m + ".bias", {C}).data;
      b.insert(b.end(), tb.begin(), tb.end());
    }
    a.qkv = ws.gemm(conv_taps(w), b);
    a.proj = conv(ws, k + ".proj_out", C, C, 1);
    return a;
  }

  void pack(Weights& ws, int num_sms) {
    nsm = num_sms;
    const int L = v.levels, nr = v.num_res_blocks, CL = width(L - 1), z = v.z_channels;
    const std::string E = "embedder.encoder.", D = "embedder.decoder.";
    {   // encoder conv_in -> [9 in_ch][ch]
      const HostTensor& w = shaped(ws, E + "conv_in.weight", {v.ch, v.in_ch, 3, 3});
      const int K = 9 * v.in_ch;
      std::vector<float> o((size_t)K * v.ch);
      for (int n = 0; n < v.ch; ++n)
        for (int k = 0; k < K; ++k) o[(size_t)k * v.ch + n] = w.data[(size_t)n * K + k];
      ci_w = ws.pool.upload(o);
      ci_b = ws.vec(E + "conv_in.bias", v.ch);
    }
    int cin = v.ch;
    enc.lv.assign(L, {});
    for (int l = 0; l < L; ++l) {
      for (int i = 0; i < nr; ++i) {
        enc.lv[l].push_back(res(ws, E + "down." + std::to_string(l) + ".block." + std::to_string(i), cin, width(l)));
        cin = width(l);
      }
      if (l != L - 1) enc.resamp.push_back(conv(ws, E + "down." + std::to_string(l) + ".downsample.conv", cin, cin, 3));
    }
    enc.m1 = res(ws, E + "mid.block_1", CL, CL);
    enc.at = attn(ws, E + "mid.attn_1", CL);
    enc.m2 = res(ws, E + "mid.block_2", CL, CL);
    enc.nout = gn(ws, E + "norm_out", CL);
    e_out = conv(ws, E + "conv_out", CL, z, 3, kVaeMaxZ);
    {   // decoder conv_in: latent columns [9 z][CL]; message columns folded per border case [9][CL][hidden]
      const int Ct = z + hidden;
      const HostTensor& w = shaped(ws, D + "conv_in.weight", {CL, Ct, 3, 3});
      std::vector<float> o((size_t)9 * z * CL);
      for (int n = 0; n < CL; ++n)
        for (int k = 0; k < 9 * z; ++k) o[(size_t)k * CL + n] = w.data[(size_t)n * Ct * 9 + k];
      dci_w = ws.pool.upload(o);
      dci_b = ws.vec(D + "conv_in.bias", CL);
      std::vector<float> wc((size_t)9 * CL * hidden, 0.f);
      for (int cs = 0; cs < 9; ++cs) {
        const int rc = cs / 3, cc = cs % 3;   // 0: first row / column (tap 0 outside), 2: last (tap 2 outside)
        for (int n = 0; n < CL; ++n)
          for (int j = 0; j < hidden; ++j) {
            float a = 0.f;
            for (int r = 0; r < 3; ++r)
              for (int c = 0; c < 3; ++c)
                if (!(rc == 0 && r == 0) && !(rc == 2 && r == 2) && !(cc == 0 && c == 0) && !(cc == 2 && c == 2))
                  a += w.data[((size_t)n * Ct + z + j) * 9 + r * 3 + c];
            wc[((size_t)cs * CL + n) * hidden + j] = a;
          }
      }
      msg_wc = ws.pool.upload(wc);
      emb = ws.pool.upload(shaped(ws, "embedder.msg_processor.msg_embeddings.weight", {2 * nbits, hidden}).data);
    }
    dec.m1 = res(ws, D + "mid.block_1", CL, CL);
    dec.at = attn(ws, D + "mid.attn_1", CL);
    dec.m2 = res(ws, D + "mid.block_2", CL, CL);
    dec.lv.assign(L, {});
    dec.resamp.assign(L, ConvW{});
    cin = CL;
    for (int l = L - 1; l >= 0; --l) {
      for (int i = 0; i <= nr; ++i) {
        dec.lv[l].push_back(res(ws, D + "up." + std::to_string(l) + ".block." + std::to_string(i), cin, width(l)));
        cin = width(l);
      }
      if (l != 0) dec.resamp[l] = conv(ws, D + "up." + std::to_string(l) + ".upsample.conv", cin, cin, 3);
    }
    dec.nout = gn(ws, D + "norm_out", v.ch * v.ch_mult[0]);
    d_out = conv(ws, D + "conv_out", v.ch * v.ch_mult[0], v.out_ch, 3, 16);
    std::vector<float> id((size_t)v.out_ch * 16, 0.f);
    for (int o = 0; o < v.out_ch; ++o) id[(size_t)o * 16 + o] = 1.f;
    id_w = ws.pool.upload(id);
    zero_b = ws.pool.upload(std::vector<float>(v.out_ch, 0.f));
  }

  // ---- the embed plan of B frames at S x S -> pl.delta [B][out_ch][S][S].
  // Buffers by lifetime: two maps X / Y that the blocks ping-pong between, the normalised operand A and the conv1 output H (later
  // the nin_shortcut output), each as large as the widest map of any level; the qkv rows of the deepest level; the fp32 latent.
  // keep (test seam, vsb_debug_keep_inputs): every map gets a buffer of its own, so that each step's input stays readable as a tap.
  // Taps (prefix vae.enc / vae.dec): .conv_in, .<blk>.{gn1,conv1,gn2,nin,out} for blk = d<l>.<i> / u<l>.<i> / mid1 / mid2,
  // .attn.{gn,qkv,o,out}, .down<l> / .up<l>, .gn_out, vae.latent, vae.msg_table, delta.
  void build(Plan& pl, int B, int S, bool keep) const {
    const int L = v.levels, CL = width(L - 1);
    long cap = 0;   // elements of the widest map: level l holds widths w[l - 1] / w[l + 1] (resampled inputs) and w[l]
    for (int l = 0; l < L; ++l) {
      int c = std::max(width(l), l == 0 ? v.ch : width(l - 1));
      if (l + 1 < L) c = std::max(c, width(l + 1));
      cap = std::max(cap, (long)(S >> l) * (S >> l) * c);
    }
    cap *= B;
    Plan* plp = &pl;
    const int sms = nsm;
    auto alloc = [&](long n) { return pl.pool.alloc_n<__half>((size_t)n); };
    __half *X = alloc(cap), *Y = alloc(cap), *A = alloc(cap), *H = alloc(cap);
    const int hL = S >> (L - 1);
    const long ML = (long)B * hL * hL;
    __half* QKV = alloc(ML * 3 * CL);
    float* lat = pl.pool.alloc_n<float>((size_t)ML * kVaeMaxZ);
    float* table = pl.pool.alloc_n<float>((size_t)B * 9 * CL);
    pl.delta = pl.pool.alloc_n<float>((size_t)B * v.out_ch * S * S);
    const long maxtiles = (long)S * S / kVaeGnTile;
    double2* part = pl.pool.alloc_n<double2>((size_t)B * maxtiles * kVaeGroups);
    float2* stat = pl.pool.alloc_n<float2>((size_t)B * kVaeGroups);
    auto fresh = [&](__half* shared) { return keep ? alloc(cap) : shared; };
    auto other = [&](const __half* cur) { return keep ? alloc(cap) : (cur == X ? Y : X); };
    auto at = [](int h) { return "@" + std::to_string(h); };
    auto tap16 = [&](const std::string& name, const __half* p, int h, int C) { pl.tap(name, p, 1, B, h, h, C, C); };

    // GroupNorm(16) of x [B][h*h][C] (+ SiLU) -> out
    auto add_gn = [&](const __half* x, int h, int C, const GN& g, bool silu, __half* out) {
      const int hw = h * h, tiles = hw / kVaeGnTile;
      const long total = (long)B * hw * (C / 8);
      const int blocks = (int)std::min<long>((total + 255) / 256, (long)sms * 16);
      const float *ga = g.gamma, *be = g.beta;
      const double n = (double)hw * (C / kVaeGroups);
      pl.add("vae.gn16" + std::string(silu ? ".silu." : ".") + std::to_string(C) + at(h), [=](cudaStream_t st) {
        vae_gn_stats_kernel<<<dim3(tiles, B), 256, 0, st>>>(x, hw, C, part);
        vae_gn_finalize_kernel<<<B, 32 * kVaeGroups, 0, st>>>(part, tiles, n, 1e-6f, stat);
        vae_gn_apply_kernel<<<blocks, 256, 0, st>>>(x, hw, C, stat, ga, be, silu ? 1 : 0, total, out);
        VSB_CUDA(cudaGetLastError());
      }, 3);
    };
    // stride-1 3x3 conv (setup_conv3x3: the 192 and 96 wide maps at 768, 320 / 160 / 80 at 640 and 192 / 96 / 48 at 384 run on
    // the gather loader; not measured) x (cin) -> out (cout) + bias (+ fp16 residual).  Gather-loader steps are named conv3x3g.
    auto add_c3 = [&](const std::string& net, const ConvW& w, const __half* x, int h, int cin, __half* out, const __half* resid) {
      ConvGemmOp op;
      setup_conv3x3(op, x, B, h, cin, cin);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.bias; op.p.out16 = out; op.p.ld_out16 = w.N;
      if (resid) { op.p.resid16 = resid; op.p.ld_res16 = w.N; }
      vsb::add_conv(pl, op, w, net + ".conv3x3" + (op.loader == LD_GATHER_CONV ? "g" : "") + (resid ? "+res." : ".") +
                                   std::to_string(cin) + "-" + std::to_string(w.N) + at(h), sms);
    };
    // 1x1 GEMM over M rows of x (K columns) -> out (pitch N) + bias (+ fp16 residual)
    auto add_gemm = [&](const std::string& name, const ConvW& w, const __half* x, long M, __half* out, const __half* resid) {
      ConvGemmOp op;
      setup_tma_gemm(op, x, M, w.K, w.K);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.bias; op.p.out16 = out; op.p.ld_out16 = w.N;
      if (resid) { op.p.resid16 = resid; op.p.ld_res16 = w.N; }
      vsb::add_conv(pl, op, w, name, sms);
    };
    // ResnetBlock on x at h -> returns its output buffer
    auto add_res = [&](const std::string& net, const std::string& tp, const Res& r, const __half* x, int h) -> __half* {
      __half* a1 = fresh(A);
      add_gn(x, h, r.cin, r.n1, true, a1);
      tap16(tp + ".gn1", a1, h, r.cin);
      __half* h1 = fresh(H);
      add_c3(net, r.c1, a1, h, r.cin, h1, nullptr);
      tap16(tp + ".conv1", h1, h, r.cout);
      __half* a2 = fresh(A);
      add_gn(h1, h, r.cout, r.n2, true, a2);
      tap16(tp + ".gn2", a2, h, r.cout);
      const __half* sc = x;
      if (r.cin != r.cout) {
        __half* s = fresh(H);   // conv1's output is consumed by the second norm
        add_gemm(net + ".nin." + std::to_string(r.cin) + "-" + std::to_string(r.cout) + at(h), r.nin, x, (long)B * h * h, s, nullptr);
        tap16(tp + ".nin", s, h, r.cout);
        sc = s;
      }
      __half* out = other(x);
      add_c3(net, r.c2, a2, h, r.cout, out, sc);
      tap16(tp + ".out", out, h, r.cout);
      return out;
    };
    // AttnBlock at the deepest level
    auto add_attn = [&](const std::string& net, const std::string& tp, const Attn& a, const __half* x) -> __half* {
      const int h = hL, C = CL;
      __half* n = fresh(A);
      add_gn(x, h, C, a.n, false, n);
      tap16(tp + ".gn", n, h, C);
      __half* qkv = keep ? alloc(ML * 3 * C) : QKV;
      add_gemm(net + ".qkv." + std::to_string(C) + at(h), a.qkv, n, ML, qkv, nullptr);
      tap16(tp + ".qkv", qkv, h, 3 * C);
      __half* o = fresh(A);   // the normalised map is consumed by the qkv GEMM
      AttnParams ap{};
      ap.qkv = qkv; ap.out = o; ap.G = h; ap.n = h; ap.heads = 1; ap.E = C; ap.regions = 1;
      ap.scale = (float)(1.0 / std::sqrt((double)C));
      pl.add("vae.attn." + std::to_string(C) + at(h), [=](cudaStream_t st) {
        if (C == 128) launch_vit_attention<128>(ap, B, st);
        else launch_vit_attention<64>(ap, B, st);
      });
      tap16(tp + ".o", o, h, C);
      __half* out = other(x);
      add_gemm(net + ".proj+res." + std::to_string(C) + at(h), a.proj, o, ML, out, x);
      tap16(tp + ".out", out, h, C);
      return out;
    };

    // ---- encoder
    __half* cur = fresh(X);
    {
      const float *w = ci_w, *b = ci_b;
      const int ch = v.ch, cin = v.in_ch;
      const long fstride = 3L * S * S;
      __half* out = cur;
      pl.add("vae.enc.conv_in." + std::to_string(cin) + "-" + std::to_string(ch) + at(S), [=](cudaStream_t st) {
        const dim3 grid((unsigned)(((long)S * S + 255) / 256), B);
        if (cin == 1) vae_conv_in_kernel<1><<<grid, 256, 0, st>>>(plp->in_imgs, fstride, S, w, b, ch, out);
        else vae_conv_in_kernel<3><<<grid, 256, 0, st>>>(plp->in_imgs, fstride, S, w, b, ch, out);
        VSB_CUDA(cudaGetLastError());
      });
      tap16("vae.enc.conv_in", cur, S, ch);
    }
    for (int l = 0; l < L; ++l) {
      const int h = S >> l;
      for (size_t i = 0; i < enc.lv[l].size(); ++i)
        cur = add_res("vae.enc", "vae.enc.d" + std::to_string(l) + "." + std::to_string(i), enc.lv[l][i], cur, h);
      if (l != L - 1) {
        const int C = width(l);
        __half* out = other(cur);
        ConvGemmOp op;
        setup_gather_conv(op, LD_GATHER_CONV, cur, C, C, nullptr, 0, 0, B, h, h, h / 2, h / 2, 3, 3, 2, 0, 0);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = enc.resamp[l].bias; op.p.out16 = out; op.p.ld_out16 = C;
        vsb::add_conv(pl, op, enc.resamp[l], "vae.enc.down." + std::to_string(C) + at(h), sms);
        cur = out;
        tap16("vae.enc.down" + std::to_string(l), cur, h / 2, C);
      }
    }
    cur = add_res("vae.enc", "vae.enc.mid1", enc.m1, cur, hL);
    cur = add_attn("vae.enc", "vae.enc.attn", enc.at, cur);
    cur = add_res("vae.enc", "vae.enc.mid2", enc.m2, cur, hL);
    {
      __half* a = fresh(A);
      add_gn(cur, hL, CL, enc.nout, true, a);
      tap16("vae.enc.gn_out", a, hL, CL);
      ConvGemmOp op;
      setup_conv3x3(op, a, B, hL, CL, CL);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = e_out.bias; op.p.out32 = lat; op.p.ld_out32 = kVaeMaxZ;
      vsb::add_conv(pl, op, e_out, "vae.enc.conv_out" + std::string(op.loader == LD_GATHER_CONV ? "g." : ".") + std::to_string(CL) + "-" +
                                       std::to_string(v.z_channels) + at(hL), sms);
      pl.tap("vae.latent", lat, 0, B, hL, hL, v.z_channels, kVaeMaxZ);
    }
    // ---- message and decoder conv_in
    {
      const int K = nbits, hid = hidden, z = v.z_channels;
      const float *e = emb, *wc = msg_wc, *w = dci_w, *b = dci_b;
      pl.add("vae.msg_table", [=](cudaStream_t st) {
        vae_msg_table_kernel<<<B, 256, (size_t)hid * sizeof(float), st>>>(plp->in_msgs, plp->in_msg_stride, K, hid, e, wc, CL, table);
        VSB_CUDA(cudaGetLastError());
      });
      pl.tap("vae.msg_table", table, 0, B, 9, 1, CL, CL);
      __half* out = fresh(X);
      pl.add("vae.dec.conv_in+msg." + std::to_string(z) + "-" + std::to_string(CL) + at(hL), [=](cudaStream_t st) {
        vae_dec_conv_in_kernel<<<dim3((unsigned)(((long)hL * hL + 255) / 256), B), 256, 0, st>>>(lat, hL, z, w, b, table, CL, out);
        VSB_CUDA(cudaGetLastError());
      });
      cur = out;
      tap16("vae.dec.conv_in", cur, hL, CL);
    }
    // ---- decoder
    cur = add_res("vae.dec", "vae.dec.mid1", dec.m1, cur, hL);
    cur = add_attn("vae.dec", "vae.dec.attn", dec.at, cur);
    cur = add_res("vae.dec", "vae.dec.mid2", dec.m2, cur, hL);
    for (int l = L - 1; l >= 0; --l) {
      const int h = S >> l;
      for (size_t i = 0; i < dec.lv[l].size(); ++i)
        cur = add_res("vae.dec", "vae.dec.u" + std::to_string(l) + "." + std::to_string(i), dec.lv[l][i], cur, h);
      if (l != 0) {
        const int C = width(l);
        __half* out = other(cur);
        ConvGemmOp op;
        setup_gather_conv(op, LD_GATHER_CONV, cur, C, C, nullptr, 0, 0, B, h, h, 2 * h, 2 * h, 3, 3, 1, 1, 2);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = dec.resamp[l].bias; op.p.out16 = out; op.p.ld_out16 = C;
        vsb::add_conv(pl, op, dec.resamp[l], "vae.dec.up." + std::to_string(C) + at(h), sms);
        cur = out;
        tap16("vae.dec.up" + std::to_string(l), cur, 2 * h, C);
      }
    }
    {
      const int C0 = width(0);
      __half* a = fresh(A);
      add_gn(cur, S, C0, dec.nout, true, a);
      tap16("vae.dec.gn_out", a, S, C0);
      // C0 -> out_ch (N padded to 16) + bias, then the fused outc epilogue as the identity (+ tanh) -> planar fp32 delta
      ConvGemmOp op;
      setup_tma_conv(op, a, B, S, S, C0, C0, 3, 3, 1);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = d_out.bias;
      op.p.outc_w = id_w; op.p.outc_b = zero_b; op.p.n_out = v.out_ch; op.p.outc_tanh = v.tanh_out;
      op.p.delta = pl.delta; op.p.hw = S * S;
      vsb::add_conv(pl, op, d_out, "vae.dec.conv_out" + std::string(v.tanh_out ? "+tanh." : ".") + std::to_string(C0) + "-" +
                                       std::to_string(v.out_ch) + at(S), sms);
    }
    pl.tap("delta", pl.delta, 0, B, v.out_ch, S, S, S);
  }
};

}  // namespace vsb
