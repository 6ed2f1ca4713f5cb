// Model assembly: weight folding/packing (host), per-batch execution plans (device buffers + launch lists),
// and the embed / detect drivers behind the C ABI.
#pragma once
#include <cmath>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

#include "../../include/vsb200.h"
#include "attention_host.cuh"
#include "conv_gemm_host.cuh"
#include "conv3_direct_host.cuh"
#include "pointwise_host.cuh"
#include "resize_blend_host.cuh"

namespace vsb {

static int64_t g_launches = 0;

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

struct DebugTensor { const void* ptr; int dtype; /*0 f32, 1 f16*/ int64_t shape[4]; int64_t ld; };

struct Step {
  std::function<void(cudaStream_t)> fn;
  int launches = 1;
  std::string name = "";
};

// optional per-step CUDA-event profile (bench.py roofline leg): name -> (total ms, launches)
struct Profile {
  bool enabled = false;
  std::map<std::string, std::pair<double, long>> acc;
  std::vector<std::pair<std::string, std::pair<cudaEvent_t, cudaEvent_t>>> pending;
  void flush() {
    for (auto& e : pending) {
      float ms = 0.f;
      cudaEventSynchronize(e.second.second);
      cudaEventElapsedTime(&ms, e.second.first, e.second.second);
      auto& a = acc[e.first];
      a.first += ms; a.second += 1;
      cudaEventDestroy(e.second.first); cudaEventDestroy(e.second.second);
    }
    pending.clear();
  }
};
static Profile g_profile;

// runs `fn`, which makes `launches` kernel launches on `st`, under one profile entry `name` when profiling is on
template <class Fn> void prof_scope(const std::string& name, cudaStream_t st, int launches, Fn&& fn) {
  if (!g_profile.enabled) { fn(); g_launches += launches; return; }
  cudaEvent_t a, b;
  cudaEventCreate(&a); cudaEventCreate(&b);
  cudaEventRecord(a, st);
  fn();
  cudaEventRecord(b, st);
  g_launches += launches;
  g_profile.pending.push_back({name, {a, b}});
}

struct Plan {
  DevicePool pool;
  uint64_t last_use = 0;    // LRU stamp of the plan cache
  std::vector<Step> steps;
  std::map<std::string, DebugTensor> dbg;
  // embed plan I/O
  const float* in_imgs = nullptr;  // set per call (pointer slot read by the first kernel's lambda)
  long in_frame_stride = 0;
  const uint8_t* in_msgs = nullptr;
  int in_msg_stride = 0;
  float* x_res = nullptr;   // [B,3,S,S] resized RGB when the input is not at processing size
  float* delta = nullptr;   // [B,CD,S,S]
  float* logits = nullptr;  // [B,1+K]
  float* out_maps = nullptr;  // pixel-wise detect plans: the caller's [B,1+K,P,P] slice, set per call
  void run(cudaStream_t st) {
    for (auto& s : steps) prof_scope(s.name, st, s.launches, [&] { s.fn(st); });
  }
};

// tiling caps of the gather kernels: the pixel decoder's is the opt-in shared memory of one H100 block, the U-Net up-convs' 160 KB
constexpr size_t kPdMaxSmem = 227 * 1024;
constexpr size_t kUpGatherSmem = 160 * 1024;

class Model {
 public:
  vsb_model_desc d;
  std::map<std::string, HostTensor> sd;
  bool finalized = false;
  int device = -1, num_sms = 0;
  std::recursive_mutex mu;   // serialises the C entry points of one handle (vsb200.cu VSB_MODEL_SCOPE)
  DevicePool wpool;
  static constexpr int kMaxBatch = 64;

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
  // extractor
  __half* stem_w16 = nullptr;
  float* stem_wk = nullptr;   // widths > 256 (chunkyseal): fp32 [48][C0] for the CUDA-core stem kernel
  float *stem_b = nullptr, *stem_lnw = nullptr, *stem_lnb = nullptr;
  struct DsW { float* lnw; float* lnb; ConvW conv; };
  std::vector<DsW> ds;
  struct CnBlockW { float* dww; float* dwb; float* lnw; float* lnb; ConvW pw1; float* gamma; ConvW pw2; };
  std::vector<std::vector<CnBlockW>> cn;
  ConvW head_conv;
  float *head_lnw = nullptr, *head_lnb = nullptr, *head_lw = nullptr, *head_lb = nullptr;
  // pixel-wise decoder (vsb_model_set_pixel_decoder; pixel_decoder.py:44-83): stage i = bilinear x pd[i].f, reflect-padded 3x3
  // conv C -> C / f, LayerNorm, GELU; then the 1x1 conv head C_last -> 1 + nbits per pixel
  bool pixelwise = false;
  // geometry and gather kernel (16-byte vectors per thread; tiled when smem > 0) from set_pixel_decoder, weights from finalize
  struct PdStageW { ConvW taps; float* lnw; float* lnb; int f, cin, cout, kin, vpt; size_t smem; };
  std::vector<PdStageW> pd;
  float *pd_hw = nullptr, *pd_hb = nullptr;   // fp32 [1+nbits][C_last], [1+nbits]
  // SAM-ViT extractor (vsb_model_set_vit_extractor; modules/vit.py ImageEncoderViT): replaces the ConvNeXt trunk when `vit`
  bool vit = false;
  vsb_vit_desc vd{};
  ConvW vit_patch;                      // [E][768] fp16, x*2-1 folded: W' = 2W (K order c, r, s); no bias (it is in vit_pos)
  float* vit_pos = nullptr;             // fp32 [grid^2][E]: pos_embed + b - sum(W)
  struct VitBlockW { float *n1w, *n1b, *n2w, *n2b; ConvW qkv, proj, lin1, lin2; __half *rel_h, *rel_w; };
  std::vector<VitBlockW> vit_blk;
  ConvW vit_neck1, vit_neck3;
  float *vit_nln1w = nullptr, *vit_nln1b = nullptr, *vit_nln2w = nullptr, *vit_nln2b = nullptr;

  // grow-only device staging for the host-buffer entry points (no cudaMalloc on the steady-state path)
  struct Staging { void* p = nullptr; size_t cap = 0; };
  Staging staging[8];   // 0-5: host entry points; 6-7: low-resolution attenuation scratch
  void* stage(int slot, size_t bytes) {
    Staging& s = staging[slot];
    if (bytes > s.cap) {
      if (s.p) cudaFree(s.p);
      s.p = nullptr; s.cap = 0;
      VSB_CUDA(cudaMalloc(&s.p, bytes));
      s.cap = bytes;
    }
    return s.p;
  }
  ~Model() {
    for (auto& s : staging) if (s.p) cudaFree(s.p);
    if (s_in) { cudaStreamDestroy(s_in); cudaStreamDestroy(s_cmp); cudaStreamDestroy(s_out); }
    for (auto e : ev_in) cudaEventDestroy(e);
    for (auto e : ev_cmp) cudaEventDestroy(e);
  }

  std::map<int, std::unique_ptr<Plan>> embed_plans, detect_plans;
  std::map<std::tuple<int, int, int, int, int, bool, bool>, std::unique_ptr<ResampleDev>> resamplers;
  Plan* last_plan = nullptr;
  // test seam (vsb_debug_last_dispatch): the variant of the most recent launch of each full-resolution kernel, -1 before the first
  //   resize: MT, GST, vec, toy, OW       blend: 3 (jnd_blend3_kernel) or 2 (jnd_blend2_kernel), VEC, FASTUP, CD, JIN
  int32_t last_resize[5] = {-1, -1, -1, -1, -1};
  int32_t last_blend[5] = {-1, -1, -1, -1, -1};
  // test seam (vsb_debug_keep_inputs): detect plans copy the ConvNeXt residual stream aside where the blocks read it
  bool keep_inputs = false;
  void set_keep_inputs(bool on) {
    keep_inputs = on;
    for (auto& kv : detect_plans) if (kv.second.get() == last_plan) last_plan = nullptr;
    detect_plans.clear();
  }

  explicit Model(const vsb_model_desc& desc) : d(desc) { check_desc(); }

  // ---- the kernel of every U-Net layer at the map width it runs at, chosen once by check_desc.  finalize packs only the weights
  // that kernel reads, and plan building follows them: ConvW::wd (direct ring conv) or ::w (tensor-core GEMM), down_conv[i].wd
  // (space-to-depth ring conv) or .w (gather GEMM), up_phase_w[j] (phase-folded ring conv + border fix) or up_conv[j] (tap GEMM +
  // gather with `vpt` 16-byte channel vectors per thread, tiled when smem > 0).
  struct ResBlockK { bool res, c1, c2; };   // true: the direct ring conv
  struct UpK { bool phase; int vpt; size_t smem; };
  bool inc_k = false;
  std::vector<bool> down_k;
  std::vector<ResBlockK> down_rb_k, up_rb_k;
  ResBlockK bott_rb_k{};
  std::vector<UpK> up_k;

  // vsb_model_create: every rule that depends only on the descriptor, and the U-Net's kernels (no CUDA calls)
  void check_desc() {
    if (d.unet_act != 0 || d.unet_norm != 0) throw Error("unsupported card: only BatchNorm+ReLU U-Nets are implemented on the GPU path", kErrUnsupported);
    VSB_CHECK(d.unet_levels >= 2 && d.unet_levels <= 6, "unet levels");
    VSB_CHECK(d.unet_in_ch == 1 || d.unet_in_ch == 3, "unet in_channels must be 1 or 3");
    VSB_CHECK(d.unet_out_ch >= 1 && d.unet_out_ch <= 3, "unet out_channels must be <= 3");
    VSB_CHECK((d.yuv != 0) == (d.unet_in_ch == 1), "yuv cards use 1 input channel");
    const int S = d.img_size, L = d.unet_levels, zb = d.unet_z[L - 1] + d.hidden;
    const int* z = d.unet_z;
    for (int i = 0; i < L; ++i) {
      // widths the kernels implement: 8 (a leading run of levels, not the last: the direct conv's 8-channel instantiations),
      // 16, 32 and multiples of 64
      const bool ok8 = z[i] == 8 && i < L - 1 && (i == 0 || z[i - 1] == 8);
      if (!(ok8 || z[i] == 16 || z[i] == 32 || (z[i] > 0 && z[i] % 64 == 0)))
        throw Error("U-Net width " + std::to_string(z[i]) + " at level " + std::to_string(i) + " is not implemented (8 in the "
                    "leading levels, 16, 32 or a multiple of 64)", kErrUnsupported);
    }
    // the tensor-core convs tile maps by 128 pixels
    if ((S >> (L - 1)) < 16)
      throw Error("img_size=" + std::to_string(S) + ": the U-Net's " + std::to_string(L) + " levels leave a " +
                  std::to_string(S >> (L - 1)) + "-pixel bottleneck map; at least 16 is implemented", kErrUnsupported);
    // policy, also where the 8-channel rings would still fit: unet_tiny_yuv_quant's first ring to overflow is at 896
    if (z[0] == 8 && S > 768)
      throw Error("img_size=" + std::to_string(S) + ": an 8-channel U-Net runs at processing sizes up to 768", kErrUnsupported);
    VSB_CHECK(S % 128 == 0, "processing size must be a multiple of 128");
    VSB_CHECK(d.hidden % 8 == 0, "hidden must be a multiple of 8");
    if (d.jnd_in_ch != 0 && !((d.jnd_in_ch == 1 || d.jnd_in_ch == 3) && (d.jnd_out_ch == 1 || d.jnd_out_ch == 3)))
      throw Error("JND attenuation: in_channels / out_channels must be 1 or 3 (configs/attenuation.yaml)", kErrUnsupported);
    for (int s = 0; s < 4; ++s) {
      VSB_CHECK(d.ext_dims[s] % 2 == 0, "extractor widths must be even (channel pairs in the depthwise kernel)");
      VSB_CHECK(s == 0 || d.ext_dims[s] >= d.ext_dims[s - 1], "extractor widths must not shrink along the trunk");
    }
    // 8-channel layers have no GEMM path: where their ring does not fit, the model is not implemented
    auto ring8 = [](bool ring, int C, int W) {
      if (C == 8 && !ring)
        throw Error("8-channel layer on a " + std::to_string(W) + "-wide map: the direct conv's ring does not fit (processing size "
                    "too large for an 8-channel U-Net)", kErrUnsupported);
      return ring;
    };
    // ResnetBlock of C channels on a W-wide map; dense_out: its output has pitch C (the last down level writes the concat buffer)
    auto resblock = [&](int C, int W, bool dense_out) {
      return ResBlockK{ring8(conv3_direct_ok(C, C, W, 1), C, W), ring8(conv3_direct_ok(C, C, W), C, W),
                       ring8(dense_out && conv3_direct_ok(C, C, W), C, W)};
    };
    inc_k = ring8(conv3_direct_ok(z[0], z[0], S), z[0], S);
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

  // vsb_model_set_pixel_decoder: the stage rules (include/vsb200.h) and each stage's gather kernel, no CUDA calls.  Stage i maps
  // c -> c / f_i channels on an h-pixel map; the last stage's kernel holds one pixel's channels in registers and the head's weights
  // beside its staged taps.
  void set_pixel_decoder(int n, const int32_t* f, int pw) {
    if (finalized) throw Error("model already finalized", kErrState);
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
    if (!vit && d.ext_stem_stride != 4) throw Error("pixel-wise decoder: needs a ConvNeXt trunk with stem stride 4", kErrUnsupported);
    std::vector<PdStageW> stages;
    int c = trunk_width(), h = trunk_map();
    for (int i = 0; i < n; ++i) {
      const int F = f[i], co = c / F, T = 16 / F;
      const bool last = i + 1 == n;
      if (c % F != 0 || co % 8 != 0 || (last ? co > 32 : pd_vpt(co) == 0) || (i == 0 && pd_gemm_k(c) != c))
        throw Error("pixel decoder: stage " + std::to_string(i) + " (" + std::to_string(c) + " channels / " + std::to_string(F) +
                    ") is not implemented (a trunk width of 16, 32 or >= 64; stage widths multiples of 8 of the form 8 * {1,3} * 2^k, "
                    "the last one at most 32)", kErrUnsupported);
      PdStageW s{};
      s.f = F; s.cin = c; s.cout = co; s.kin = pd_gemm_k(c);
      const size_t tsmem = ups_tile_smem(F, co);
      if (last) {
        s.vpt = co / 8;
        s.smem = tsmem + (size_t)(1 + d.nbits) * (co + 1) * sizeof(float);
        if (h % T != 0 || s.smem > kPdMaxSmem)
          throw Error("pixel-wise head: a " + std::to_string(h) + "-pixel map with " + std::to_string(1 + d.nbits) + " outputs is not implemented", kErrUnsupported);
      } else {
        s.vpt = pd_vpt(co);
        s.smem = h % T == 0 && tsmem <= kPdMaxSmem ? tsmem : 0;
      }
      stages.push_back(s);
      c = co; h *= F;
    }
    pixelwise = true;
    pd = std::move(stages);
  }
  // vsb_model_set_vit_extractor: the ViT rules (include/vsb200.h), no CUDA calls
  void set_vit_extractor(const vsb_vit_desc& v) {
    if (finalized) throw Error("model already finalized", kErrState);
    if (pixelwise) throw Error("vsb_model_set_vit_extractor must come before vsb_model_set_pixel_decoder", kErrState);
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
    const int G = d.img_size / kVitPatch;
    const uint32_t all = v.depth == 32 ? ~0u : (1u << v.depth) - 1u;
    if (v.global_mask != all) {   // some block attends over windows
      if (v.window_size <= 0 || G % v.window_size != 0)
        unsup("a " + std::to_string(G) + "-token grid is not divisible by window_size " + std::to_string(v.window_size) + " (window padding is not implemented)");
      if (v.window_size * v.window_size % kAttnTile != 0)
        unsup("window_size " + std::to_string(v.window_size) + " holds " + std::to_string(v.window_size * v.window_size) + " tokens, not a multiple of 64");
    }
    if (v.global_mask != 0 && G * G > 1024)
      unsup("global attention over " + std::to_string(G * G) + " tokens (img_size " + std::to_string(d.img_size) + ") is not implemented (at most 1024, img_size <= 512)");
    // the kernel stages the 2n - 1 rows of each relative-position table in 64 rows: region sides n <= 32 (global blocks: the cap above)
    if (v.use_rel_pos && v.global_mask != all && v.window_size > kAttnMaxRelSide)
      unsup("relative positions over " + std::to_string(v.window_size) + "-token-wide windows are not implemented (at most " +
            std::to_string(kAttnMaxRelSide) + ")");
    vd = v;
    vit = true;
  }
  int trunk_width() const { return vit ? vd.out_chans : d.ext_dims[3]; }
  // side of the trunk's last feature map: stem k4 / stride st, then three k2 s2 downsampling layers; the ViT's token grid
  int trunk_map() const {
    if (vit) return d.img_size / kVitPatch;
    int h = (d.img_size - 4) / d.ext_stem_stride + 1;
    for (int s = 1; s < 4; ++s) h = (h - 2) / 2 + 1;
    return h;
  }
  // floats vsb_detect writes per frame: 1+nbits logits, or 1+nbits maps of P x P for a pixel-wise model
  size_t detect_out_per_frame() const {
    size_t P = (size_t)trunk_map();
    for (const PdStageW& s : pd) P *= s.f;
    return pixelwise ? (size_t)(1 + d.nbits) * P * P : (size_t)(1 + d.nbits);
  }
  void check_pooled_head(const std::string& what) const {
    if (pixelwise) throw Error(what + ": per-pixel maps of a streamed video are not implemented (use vsb_detect / vsb_detect_host)", kErrUnsupported);
  }
  // K of a pixel-decoder stage GEMM over C input channels: the TMA GEMM loader takes K in {16, 32} or >= 64, narrower widths
  // are zero-padded (in the packed weights and in the pitch of the activation buffer, whose pad channels are zeroed once)
  static int pd_gemm_k(int C) { return (C == 16 || C == 32 || C >= 64) ? C : (C < 16 ? 16 : (C < 32 ? 32 : 64)); }
  // 16-byte channel vectors per gather thread for a non-final stage of C channels: C = 8 * VPT * G, G a power of two <= 32
  static int pd_vpt(int C) {
    for (int v : {1, 3}) {
      if (C % (8 * v)) continue;
      const int g = C / (8 * v);
      if (g <= 32 && (g & (g - 1)) == 0) return v;
    }
    return 0;
  }

  const HostTensor& get(const std::string& k) const {
    auto it = sd.find(k);
    if (it == sd.end()) throw Error("missing checkpoint tensor: " + k, kErrState);
    return it->second;
  }

  // ---------------------------------------------------------------- packing helpers
  static std::vector<__half> to_half(const std::vector<float>& v) {
    std::vector<__half> h(v.size());
    for (size_t i = 0; i < v.size(); ++i) h[i] = __float2half_rn(v[i]);
    return h;
  }
  // conv weight [N][C][R][S] (+ per-output-channel scale, + per-input-channel scale) -> [N][R][S][C]
  // pad_taps: every tap's channel run is zero-padded to a multiple of 8 (gather loaders move 16-byte channel chunks; the
  // activation buffer then has the same padded pixel pitch with ZERO pad channels).  Rows are padded to a multiple of 8
  // elements either way (a no-op for every width of the tiny / pixelseal cards).
  ConvW pack_conv(const std::string& wkey, const std::vector<float>* out_scale, const std::vector<float>& bias,
                  const std::vector<float>* in_scale = nullptr, bool pad_taps = false) {
    const HostTensor& w = get(wkey);
    VSB_CHECK(w.shape.size() == 4 || w.shape.size() == 2, "conv weight rank");
    const int N = (int)w.shape[0], C = (int)w.shape[1];
    const int R = w.shape.size() == 4 ? (int)w.shape[2] : 1, S = w.shape.size() == 4 ? (int)w.shape[3] : 1;
    const int Cp = pad_taps ? (C + 7) / 8 * 8 : C;
    const int K = R * S * Cp, ld = (K + 7) / 8 * 8;
    std::vector<float> p((size_t)N * ld, 0.f);
    for (int n = 0; n < N; ++n)
      for (int c = 0; c < C; ++c)
        for (int r = 0; r < R; ++r)
          for (int s = 0; s < S; ++s) {
            float v = w.data[(((size_t)n * C + c) * R + r) * S + s];
            if (out_scale) v *= (*out_scale)[n];
            if (in_scale) v *= (*in_scale)[c];
            p[(size_t)n * ld + ((size_t)r * S + s) * Cp + c] = v;
          }
    ConvW cw;
    cw.N = N; cw.K = K; cw.ld = ld;
    cw.w = wpool.upload(to_half(p));
    cw.bias = bias.empty() ? nullptr : wpool.upload(bias);
    return cw;
  }
  // 3x3 conv weight [N][C0+C1][3][3] -> halo-loader layout [N][chunk][tap][cc], chunks zero-padded to kb_per_c*64
  ConvW pack_conv_halo(const std::string& wkey, const std::vector<float>* out_scale, const std::vector<float>& bias, int C0, int C1,
                       const std::vector<float>* in_scale = nullptr) {
    const HostTensor& w = get(wkey);
    VSB_CHECK(w.shape.size() == 4 && w.shape[2] == 3 && w.shape[3] == 3 && (int)w.shape[1] == C0 + C1, "halo conv weight shape");
    const int N = (int)w.shape[0], Ct = C0 + C1;
    const int cc = C0 < 64 ? C0 : 64, kbc = (9 * cc + 63) / 64, Kpad = halo_kpad(C0, C1);
    std::vector<float> p((size_t)N * Kpad, 0.f);
    for (int n = 0; n < N; ++n)
      for (int c = 0; c < Ct; ++c)
        for (int t = 0; t < 9; ++t) {
          float v = w.data[((size_t)n * Ct + c) * 9 + t];
          if (out_scale) v *= (*out_scale)[n];
          if (in_scale) v *= (*in_scale)[c];
          p[(size_t)n * Kpad + (size_t)(c / cc) * kbc * 64 + t * cc + (c % cc)] = v;
        }
    ConvW cw;
    cw.N = N; cw.K = Kpad;
    cw.w = wpool.upload(to_half(p));
    cw.bias = bias.empty() ? nullptr : wpool.upload(bias);
    return cw;
  }
  // UBlock up-conv as a low-resolution tap GEMM (see ups_gather_ln_kernel): rows n' = tap*Cout + co, K = concat channels
  // (zero-padded to Kp columns when Kp > Ct: the pixel decoder's narrow stage inputs, see pd_gemm_k)
  ConvW pack_upconv_taps(const std::string& wkey, const std::vector<float>& in_scale, int Kp = 0) {
    const HostTensor& w = get(wkey);
    VSB_CHECK(w.shape.size() == 4 && w.shape[2] == 3 && w.shape[3] == 3, "up conv weight shape");
    const int Co = (int)w.shape[0], Ct = (int)w.shape[1];
    if (Kp < Ct) Kp = Ct;
    std::vector<float> p((size_t)9 * Co * Kp, 0.f);
    for (int co = 0; co < Co; ++co)
      for (int c = 0; c < Ct; ++c)
        for (int t = 0; t < 9; ++t) p[((size_t)t * Co + co) * Kp + c] = w.data[((size_t)co * Ct + c) * 9 + t] * in_scale[c];
    ConvW cw;
    cw.N = 9 * Co; cw.K = Kp;
    cw.w = wpool.upload(to_half(p));
    return cw;
  }
  // the same up-conv folded for the phase path (conv3_direct_host.cuh, setup_up_phase_direct): rows n = (py*2+px)*Cout + co,
  // K = (ey*3+ex)*Ct + c over the 3x3 LOW-resolution neighbourhood; g[phase][d][e] = weight of low-res offset e-1 in tap d of
  // an output row of that phase (bilinear x2, align_corners=False).  Also the plain fp32 taps for the border fix-up kernel.
  void pack_upconv_phase(const std::string& wkey, const std::vector<float>& in_scale, __half** wd_out, float** wk_out) {
    const HostTensor& w = get(wkey);
    const int Co = (int)w.shape[0], Ct = (int)w.shape[1];
    static const float g[2][3][3] = {{{.75f, .25f, 0.f}, {.25f, .75f, 0.f}, {0.f, .75f, .25f}},
                                     {{.25f, .75f, 0.f}, {0.f, .75f, .25f}, {0.f, .25f, .75f}}};
    std::vector<float> p((size_t)4 * Co * 9 * Ct, 0.f), wk((size_t)9 * Co * Ct);
    for (int co = 0; co < Co; ++co)
      for (int c = 0; c < Ct; ++c)
        for (int dy = 0; dy < 3; ++dy)
          for (int dx = 0; dx < 3; ++dx) {
            const float kv = w.data[(((size_t)co * Ct + c) * 3 + dy) * 3 + dx] * in_scale[c];
            wk[((size_t)(dy * 3 + dx) * Co + co) * Ct + c] = kv;
            for (int py = 0; py < 2; ++py)
              for (int px = 0; px < 2; ++px)
                for (int ey = 0; ey < 3; ++ey)
                  for (int ex = 0; ex < 3; ++ex) {
                    const float cf = g[py][dy][ey] * g[px][dx][ex];
                    if (cf != 0.f) p[((size_t)((py * 2 + px) * Co + co) * 9 + (ey * 3 + ex)) * Ct + c] += kv * cf;
                  }
          }
    *wd_out = pack_direct_taps(p, 4 * Co, Ct);
    *wk_out = wpool.upload(wk);
  }
  // conv weight [N][C][R][R] (x out_scale) -> fp32 taps [N][R*R][C] (K order r, s, c)
  std::vector<float> conv_taps(const HostTensor& w, const std::vector<float>* out_scale) const {
    const int N = (int)w.shape[0], C = (int)w.shape[1], T = w.shape.size() == 4 ? (int)(w.shape[2] * w.shape[3]) : 1;
    std::vector<float> t((size_t)N * T * C);
    for (int n = 0; n < N; ++n)
      for (int c = 0; c < C; ++c)
        for (int k = 0; k < T; ++k) {
          float v = w.data[((size_t)n * C + c) * T + k];
          if (out_scale) v *= (*out_scale)[n];
          t[((size_t)n * T + k) * C + c] = v;
        }
    return t;
  }
  // fp32 taps [N][T][C] -> weights in the direct conv's core-matrix layout (pack_direct_weights_kernel); each value is rounded to
  // fp16 once, and the fp16 copy the kernel reads is freed once it is done
  __half* pack_direct_taps(const std::vector<float>& taps, int N, int C, int T = 9) {
    DevicePool tmp;
    __half* wd = wpool.alloc_n<__half>(taps.size());
    pack_direct_weights(tmp.upload(to_half(taps)), N, C, wd, 0, T);
    VSB_CUDA(cudaStreamSynchronize(0));
    return wd;
  }
  // stride-1 3x3 / 1x1 conv weights for the direct conv (conv3_direct.cuh); 8 -> 8 channels (unet_tiny_*) run only on its
  // 8-channel instantiation (KS = 0), through the virtual-tap layout of direct8_weights
  __half* pack_direct(const std::string& wkey, const std::vector<float>* out_scale) {
    const HostTensor& w = get(wkey);
    const int N = (int)w.shape[0], C = (int)w.shape[1], R = w.shape.size() == 4 ? (int)w.shape[2] : 1;
    if (C != 8) return pack_direct_taps(conv_taps(w, out_scale), N, C, R * R);
    VSB_CHECK(N == 8, "8-channel conv weight shape");
    return pack_direct_taps(direct8_weights(conv_taps(w, out_scale), N, R), N, 16, R * ((R + 1) / 2));
  }
  // DBlock.down weights for the space-to-depth ring conv (conv3_direct_host.cuh, setup_down_s2d_direct)
  __half* pack_down_s2d(const std::string& wkey) {
    const HostTensor& w = get(wkey);
    const int N = (int)w.shape[0], Ci = (int)w.shape[1];
    return pack_direct_taps(s2d_weights(conv_taps(w, nullptr), N, Ci), N, 4 * Ci);
  }
  static bool use_halo(int C) { return C <= 16; }
  // U-Net conv (3x3 or 1x1, stride 1) in the layout its kernel reads: the direct ring conv's, or the GEMM's (for 3x3 convs up to 16
  // input channels, the halo loader's)
  ConvW pack_unet_conv(const std::string& wkey, const std::vector<float>* out_scale, const std::vector<float>& bias, bool direct) {
    const HostTensor& w = get(wkey);
    const int C = (int)w.shape[1];
    if (!direct)
      return w.shape.size() == 4 && w.shape[2] == 3 && use_halo(C) ? pack_conv_halo(wkey, out_scale, bias, C, 0) : pack_conv(wkey, out_scale, bias);
    ConvW cw;
    cw.N = (int)w.shape[0];
    cw.wd = pack_direct(wkey, out_scale);
    cw.bias = wpool.upload(bias);
    return cw;
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
  ResBlockW pack_resblock(const std::string& key, const ResBlockK& k) {
    ResBlockW rb;
    std::vector<float> s, b;
    bn_fold(key + ".double_conv.1", s, b);
    rb.c1 = pack_unet_conv(key + ".double_conv.0.weight", &s, b, k.c1);
    bn_fold(key + ".double_conv.4", s, b);
    rb.c2 = pack_unet_conv(key + ".double_conv.3.weight", &s, b, k.c2);
    rb.res = pack_unet_conv(key + ".res_conv.weight", nullptr, get(key + ".res_conv.bias").data, k.res);
    return rb;
  }

  void finalize(int dev) {
    if (finalized) throw Error("model already finalized", kErrState);
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) throw Error("no CUDA device: libvsb200 has no CPU fallback", kErrCuda);
    VSB_CUDA(cudaSetDevice(dev));
    cudaDeviceProp prop;
    VSB_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) throw Error("libvsb200 is built for sm_90a only (found sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ")", kErrUnsupported);
    device = dev;
    num_sms = prop.multiProcessorCount;
    const std::string P = "embedder.unet.";
    const int L = d.unet_levels;
    std::vector<int> z(d.unet_z, d.unet_z + L);
    // ---- inc: first conv on CUDA cores, fp32 weights with BN folded
    {
      std::vector<float> s, b;
      bn_fold(P + "inc.double_conv.1", s, b);
      const HostTensor& w = get(P + "inc.double_conv.0.weight");
      VSB_CHECK((int)w.shape[0] == z[0] && (int)w.shape[1] == d.unet_in_ch, "inc conv shape");
      std::vector<float> w1(w.data);
      const size_t per = (size_t)d.unet_in_ch * 9;
      for (int n = 0; n < z[0]; ++n) for (size_t k = 0; k < per; ++k) w1[n * per + k] *= s[n];
      first_w1 = wpool.upload(w1); first_b1 = wpool.upload(b);
      first_wr = wpool.upload(get(P + "inc.res_conv.weight").data);
      first_br = wpool.upload(get(P + "inc.res_conv.bias").data);
      bn_fold(P + "inc.double_conv.4", s, b);
      inc_c2 = pack_unet_conv(P + "inc.double_conv.3.weight", &s, b, inc_k);
    }
    for (int i = 0; i < L - 1; ++i) {
      const std::string D = P + "downs." + std::to_string(i);
      const std::vector<float>& bias = get(D + ".down.bias").data;
      ConvW dc;
      if (down_k[i]) { dc.wd = pack_down_s2d(D + ".down.weight"); dc.bias = wpool.upload(bias); }
      else dc = pack_conv(D + ".down.weight", nullptr, bias);
      down_conv.push_back(dc);
      down_rb.push_back(pack_resblock(D + ".conv", down_rb_k[i]));
    }
    for (int i = 0; i < d.unet_num_blocks; ++i) bott_rb.push_back(pack_resblock(P + "bottleneck.model." + std::to_string(i), bott_rb_k));
    {
      std::vector<int> zz(z);
      zz[L - 1] += d.hidden;
      int j = 0;
      for (int ii = L - 2; ii >= 0; --ii, ++j) {
        const std::string U = P + "ups." + std::to_string(j);
        // virtual concat (x | skip * 2^-1/2): fold the skip scale into the second half of the input channels
        std::vector<float> in_scale(2 * zz[ii + 1], 1.0f);
        for (int c = zz[ii + 1]; c < 2 * zz[ii + 1]; ++c) in_scale[c] = 0.70710678118654752440f;
        // 8-channel sources go through the gather loader, whose K block is 64: pad K to one block
        up_conv.push_back(up_k[j].phase ? ConvW{} : pack_upconv_taps(U + ".up.upsample_block.2.weight", in_scale, zz[ii + 1] == 8 ? 64 : 0));
        __half* pw = nullptr; float* bw = nullptr;
        if (up_k[j].phase) pack_upconv_phase(U + ".up.upsample_block.2.weight", in_scale, &pw, &bw);
        up_phase_w.push_back(pw); up_border_w.push_back(bw);
        up_lnw.push_back(wpool.upload(get(U + ".up.upsample_block.3.weight").data));
        up_lnb.push_back(wpool.upload(get(U + ".up.upsample_block.3.bias").data));
        up_rb.push_back(pack_resblock(U + ".conv", up_rb_k[j]));
      }
    }
    outc_w = wpool.upload(get(P + "outc.weight").data);  // [n_out][z0][1][1]
    outc_b = wpool.upload(get(P + "outc.bias").data);
    {
      const HostTensor& t = get(P + "msg_processor.msg_embeddings.weight");
      VSB_CHECK((int)t.shape[0] == 2 * d.nbits && (int)t.shape[1] == d.hidden, "message table shape");
      msg_table = wpool.upload(t.data);
    }
    if (vit) finalize_vit();
    else finalize_convnext();
    finalize_head();
    sd.clear();  // host copies no longer needed
    finalized = true;
  }

  // ---- SAM-ViT extractor (modules/vit.py:14-143, :146-210, :302-353, :494-525)
  void finalize_vit() {
    const std::string Q = "detector.image_encoder.";
    const int E = vd.embed_dim, G = d.img_size / kVitPatch;
    auto shape_is = [](const HostTensor& t, std::vector<int64_t> s) { return t.shape == s; };
    auto vec = [&](const std::string& k, int n) {
      const HostTensor& t = get(k);
      VSB_CHECK(t.numel() == n, k + ": expected " + std::to_string(n) + " values");
      return wpool.upload(t.data);
    };
    {
      const HostTensor& w = get(Q + "patch_embed.proj.weight");
      VSB_CHECK(shape_is(w, {E, 3, kVitPatch, kVitPatch}), Q + "patch_embed.proj.weight: expected [embed_dim, 3, 16, 16]");
      const HostTensor& b = get(Q + "patch_embed.proj.bias");
      const HostTensor& pos = get(Q + "pos_embed");
      if (!shape_is(pos, {1, G, G, E}))
        throw Error(Q + "pos_embed: a " + std::to_string(G) + " x " + std::to_string(G) + " grid of " + std::to_string(E) +
                    " is needed at img_size " + std::to_string(d.img_size), kErrInvalid);
      // x*2-1 folded (extractor.py:64): W (2x - 1) + b = (2W) x + (b - sum W)
      std::vector<float> wp(w.data.size()), table((size_t)G * G * E);
      std::vector<double> bias(E);
      for (int e = 0; e < E; ++e) {
        double s = 0.0;
        for (int k = 0; k < 768; ++k) { s += w.data[(size_t)e * 768 + k]; wp[(size_t)e * 768 + k] = 2.f * w.data[(size_t)e * 768 + k]; }
        bias[e] = (double)b.data[e] - s;
      }
      for (int pidx = 0; pidx < G * G; ++pidx)
        for (int e = 0; e < E; ++e) table[(size_t)pidx * E + e] = (float)((double)pos.data[(size_t)pidx * E + e] + bias[e]);
      vit_patch.N = E; vit_patch.K = 768;
      vit_patch.w = wpool.upload(to_half(wp));
      vit_pos = wpool.upload(table);
    }
    for (int i = 0; i < vd.depth; ++i) {
      const std::string B = Q + "blocks." + std::to_string(i) + ".";
      VitBlockW w{};
      w.n1w = vec(B + "norm1.weight", E); w.n1b = vec(B + "norm1.bias", E);
      w.n2w = vec(B + "norm2.weight", E); w.n2b = vec(B + "norm2.bias", E);
      auto lin = [&](const std::string& k, int N, int K, bool bias) {
        VSB_CHECK(shape_is(get(k + ".weight"), {N, K}), k + ".weight: expected [" + std::to_string(N) + ", " + std::to_string(K) + "]");
        return pack_conv(k + ".weight", nullptr, bias ? get(k + ".bias").data : std::vector<float>{});
      };
      w.qkv = lin(B + "attn.qkv", 3 * E, E, vd.qkv_bias != 0);
      w.proj = lin(B + "attn.proj", E, E, true);
      w.lin1 = lin(B + "mlp.lin1", vd.mlp_dim, E, true);
      w.lin2 = lin(B + "mlp.lin2", E, vd.mlp_dim, true);
      if (vd.use_rel_pos) {
        const int n = (vd.global_mask >> i) & 1u ? G : vd.window_size;
        auto rel = [&](const std::string& k) {
          const HostTensor& t = get(k);
          // the reference interpolates a table of another length (vit.py:398-428, for checkpoints of another size): not here
          if (!shape_is(t, {2 * n - 1, kAttnHd}))
            throw Error(k + ": expected [" + std::to_string(2 * n - 1) + ", 64] (2 * " + std::to_string(n) + " - 1 relative positions); "
                        "tables of another length are not interpolated", kErrInvalid);
          VSB_CHECK(n <= kAttnMaxRelSide, k + ": more than 63 relative positions (set_vit_extractor's rule)");
          std::vector<float> p((size_t)kAttnTile * kAttnHd, 0.f);   // zero rows past 2n-1: the kernel reads whole 8-row tiles
          std::copy(t.data.begin(), t.data.end(), p.begin());
          return wpool.upload(to_half(p));
        };
        w.rel_h = rel(B + "attn.rel_pos_h");
        w.rel_w = rel(B + "attn.rel_pos_w");
      }
      vit_blk.push_back(w);
    }
    const int oc = vd.out_chans;
    VSB_CHECK(shape_is(get(Q + "neck.0.weight"), {oc, E, 1, 1}), Q + "neck.0.weight: expected [out_chans, embed_dim, 1, 1]");
    VSB_CHECK(shape_is(get(Q + "neck.2.weight"), {oc, oc, 3, 3}), Q + "neck.2.weight: expected [out_chans, out_chans, 3, 3]");
    vit_neck1 = pack_conv(Q + "neck.0.weight", nullptr, {});
    vit_neck3 = pack_conv(Q + "neck.2.weight", nullptr, {}, nullptr, /*pad_taps=*/true);
    vit_nln1w = vec(Q + "neck.1.weight", oc); vit_nln1b = vec(Q + "neck.1.bias", oc);
    vit_nln2w = vec(Q + "neck.3.weight", oc); vit_nln2b = vec(Q + "neck.3.bias", oc);
  }

  // ---- extractor (ConvNeXt-V2)
  void finalize_convnext() {
    const std::string Q = "detector.convnext.";
    {
      const HostTensor& w = get(Q + "downsample_layers.0.0.weight");  // [C0][3][4][4]
      const int C0 = d.ext_dims[0];
      VSB_CHECK((int)w.shape[0] == C0 && w.shape[1] == 3 && w.shape[2] == 4, "stem shape");
      if (C0 <= 256) {   // tensor-core stem GEMM with the LayerNorm fused in the epilogue (needs the whole row in one N tile)
        std::vector<float> t((size_t)C0 * 64, 0.f);   // GEMM operand [C0][64], K = (c, r, t) zero-padded 48 -> 64
        for (int c = 0; c < C0; ++c) for (int k = 0; k < 48; ++k) t[(size_t)c * 64 + k] = w.data[(size_t)c * 48 + k];
        stem_w16 = wpool.upload(to_half(t));
      } else {           // stem_ln_kernel: [48][C0]
        std::vector<float> t((size_t)48 * C0);
        for (int c = 0; c < C0; ++c) for (int k = 0; k < 48; ++k) t[(size_t)k * C0 + c] = w.data[(size_t)c * 48 + k];
        stem_wk = wpool.upload(t);
      }
      stem_b = wpool.upload(get(Q + "downsample_layers.0.0.bias").data);
      stem_lnw = wpool.upload(get(Q + "downsample_layers.0.1.weight").data);
      stem_lnb = wpool.upload(get(Q + "downsample_layers.0.1.bias").data);
    }
    for (int i = 1; i < 4; ++i) {
      DsW w;
      const std::string K = Q + "downsample_layers." + std::to_string(i);
      w.lnw = wpool.upload(get(K + ".0.weight").data);
      w.lnb = wpool.upload(get(K + ".0.bias").data);
      w.conv = pack_conv(K + ".1.weight", nullptr, get(K + ".1.bias").data, nullptr, /*pad_taps=*/true);
      ds.push_back(w);
    }
    cn.resize(4);
    for (int s = 0; s < 4; ++s) {
      const int C = d.ext_dims[s];
      for (int j = 0; j < d.ext_depths[s]; ++j) {
        const std::string B = Q + "stages." + std::to_string(s) + "." + std::to_string(j) + ".";
        CnBlockW w;
        const HostTensor& dw = get(B + "dwconv.weight");  // [C][1][7][7]
        std::vector<float> t((size_t)49 * C);
        for (int c = 0; c < C; ++c) for (int k = 0; k < 49; ++k) t[(size_t)k * C + c] = dw.data[(size_t)c * 49 + k];
        w.dww = wpool.upload(t);
        w.dwb = wpool.upload(get(B + "dwconv.bias").data);
        w.lnw = wpool.upload(get(B + "norm.weight").data);
        w.lnb = wpool.upload(get(B + "norm.bias").data);
        w.pw1 = pack_conv(B + "pwconv1.weight", nullptr, get(B + "pwconv1.bias").data);
        w.gamma = wpool.upload(get(B + "grn.gamma").data);
        // GRN: gamma*(x*Nx) + beta + x  ==  x*(gamma*Nx + 1) + beta ; beta goes through pwconv2 into its bias
        const HostTensor &w2 = get(B + "pwconv2.weight"), &b2 = get(B + "pwconv2.bias"), &beta = get(B + "grn.beta");
        std::vector<float> bias2(C);
        for (int n = 0; n < C; ++n) {
          double a = b2.data[n];
          for (int k = 0; k < 4 * C; ++k) a += (double)w2.data[(size_t)n * 4 * C + k] * (double)beta.data[k];
          bias2[n] = (float)a;
        }
        w.pw2 = pack_conv(B + "pwconv2.weight", nullptr, bias2);
        cn[s].push_back(w);
      }
    }
  }

  // ---- pixel decoder (pixel_decoder.py:44-83): pooled head or pixel-wise stages
  void finalize_head() {
    if (pixelwise) {
      const std::string D = "detector.pixel_decoder.";
      for (size_t i = 0; i < pd.size(); ++i) {
        const std::string K = D + "output_upscaling." + std::to_string(i) + ".upsample_block.";
        PdStageW& sw = pd[i];
        const HostTensor& w = get(K + "2.weight");
        VSB_CHECK(w.shape.size() == 4 && (int)w.shape[0] == sw.cout && (int)w.shape[1] == sw.cin && w.shape[2] == 3 && w.shape[3] == 3,
                  "pixel decoder stage " + std::to_string(i) + ": weight must be [C/f, C, 3, 3]");
        sw.taps = pack_upconv_taps(K + "2.weight", std::vector<float>(sw.cin, 1.f), sw.kin);
        sw.lnw = wpool.upload(get(K + "3.weight").data);
        sw.lnb = wpool.upload(get(K + "3.bias").data);
      }
      const HostTensor& lw = get(D + "linear.weight");
      VSB_CHECK(lw.shape.size() == 4 && (int)lw.shape[0] == 1 + d.nbits && (int)lw.shape[1] == pd.back().cout && lw.shape[2] == 1 && lw.shape[3] == 1,
                "pixel-wise head: linear.weight must be [1+nbits, C, 1, 1]");
      pd_hw = wpool.upload(lw.data);
      pd_hb = wpool.upload(get(D + "linear.bias").data);
    } else {
      const std::string D = "detector.pixel_decoder.";
      head_conv = pack_conv(D + "output_upscaling.0.upsample_block.2.weight", nullptr, {}, nullptr, /*pad_taps=*/true);
      head_lnw = wpool.upload(get(D + "output_upscaling.0.upsample_block.3.weight").data);
      head_lnb = wpool.upload(get(D + "output_upscaling.0.upsample_block.3.bias").data);
      const HostTensor& lw = get(D + "linear.weight");
      VSB_CHECK((int)lw.shape[0] == 1 + d.nbits, "head linear shape");
      head_lw = wpool.upload(lw.data);
      head_lb = wpool.upload(get(D + "linear.bias").data);
    }
  }

  // ---------------------------------------------------------------- plan building helpers
  static void dbg(Plan& pl, const std::string& name, const void* p, int dtype, int64_t B, int64_t H, int64_t W, int64_t C, int64_t ld) {
    pl.dbg[name] = DebugTensor{p, dtype, {B, H, W, C}, ld};
  }
  void add_conv(Plan& pl, ConvGemmOp op, const ConvW& w, const std::string& name, int block_n = 0, const __half* w_override = nullptr) {
    finalize_op(op, w_override ? w_override : w.w, w.N, w.K, w.ld ? w.ld : w.K, num_sms, block_n);
    pl.steps.push_back(Step{[op](cudaStream_t st) { launch(op, st); }, 1, name});
  }

  // One U-Net conv step, R x R (3: stride 1, zero pad 1; or 1) over x [B,H,W,Cin] (pitch ldx): the direct ring conv when its
  // weights were packed for it (choose_unet), else the tensor-core GEMM.  Epilogue: bias, ReLU (relu), + the fp16 residual
  // `resid` (pitch w.N), output `out` (pitch ld_out; nullptr: not written) and, fuse_outc, the 1x1 outc + tanh into pl.delta.
  void add_unet_conv(Plan& pl, const ConvW& w, int R, const __half* x, int B, int H, int W, int Cin, int ldx, bool relu,
                     const __half* resid, __half* out, int ld_out, bool fuse_outc = false) {
    const int N = w.N;
    const bool direct = w.wd != nullptr;
    VSB_CHECK(!direct || (ldx == Cin && (out == nullptr || ld_out == N)), "direct conv: dense input and output");
    const std::string name = std::string("unet.conv") + (R == 3 ? "3x3" : "1x1") + (direct ? "d" : "") + (fuse_outc ? "+outc." : ".") +
                             std::to_string(Cin) + "-" + std::to_string(N) + "@" + std::to_string(H);
    if (direct) {
      Conv3DirectOp op; setup_conv3_direct(op, x, B, H, W, Cin, N, w.wd, num_sms, R);
      op.p.bias = w.bias; op.p.relu = relu ? 1 : 0; op.p.resid = resid; op.p.out = out;
      if (fuse_outc) {
        op.p.outc_w = outc_w; op.p.outc_b = outc_b; op.p.n_out = d.unet_out_ch; op.p.delta = pl.delta; op.p.outc_tanh = d.unet_last_tanh;
      }
      pl.steps.push_back(Step{[op](cudaStream_t st) { launch_direct(op, st); }, 1, name});
      return;
    }
    // 3x3 up to 16 input channels: on-chip im2col from a shared-memory halo tile (input crosses L2->SM once), one TMA load per tap
    // above; the weight layout follows the same rule (pack_unet_conv)
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
    add_conv(pl, op, w, name);
  }

  // ResnetBlock on NHWC fp16 (modules/unet.py:17-39):  out = relu(conv3'(relu(conv3'(x)))) + (conv1(x) + b)
  // `x` has pixel pitch ldx; output written with pitch ld_out.  If fuse_outc: the 1x1 outc + tanh is fused and the
  // block output itself is not written.
  __half* add_resblock(Plan& pl, const std::string& name, const ResBlockW& w, const __half* x, int B, int H, int W, int Cin, int ldx,
                       __half* out, int ld_out, bool fuse_outc = false) {
    const int Cout = w.c1.N;
    const long M = (long)B * H * W;
    __half* r = pl.pool.alloc_n<__half>(M * Cout);
    __half* h = pl.pool.alloc_n<__half>(M * Cout);
    if (!out && !fuse_outc) { out = pl.pool.alloc_n<__half>(M * Cout); ld_out = Cout; }
    add_unet_conv(pl, w.res, 1, x, B, H, W, Cin, ldx, false, nullptr, r, Cout);
    add_unet_conv(pl, w.c1, 3, x, B, H, W, Cin, ldx, true, nullptr, h, Cout);
    add_unet_conv(pl, w.c2, 3, h, B, H, W, Cout, Cout, true, r, out, ld_out, fuse_outc);
    dbg(pl, name + ".h", h, 1, B, H, W, Cout, Cout);
    dbg(pl, name + ".r", r, 1, B, H, W, Cout, Cout);
    if (out) dbg(pl, name, out, 1, B, H, W, Cout, ld_out);
    return out;
  }

  // Plan cache: one activation arena per distinct batch size, at most `max_plans` per kind (VSB_MAX_PLANS, default 8): a service that sees
  // many different clip / tail lengths would otherwise accumulate up to 64 arenas of up to 2.3 GB each.  The least recently used plan
  // is dropped (its cudaFree calls synchronise the device, so work still in flight on it completes first).
  uint64_t plan_clock = 0;
  int max_plans = [] { const char* e = getenv("VSB_MAX_PLANS"); const int v = e ? atoi(e) : 8; return v < 2 ? 2 : v; }();
  Plan* get_plan(std::map<int, std::unique_ptr<Plan>>& m, int B, void (Model::*build)(Plan&, int)) {
    auto it = m.find(B);
    if (it != m.end()) { it->second->last_use = ++plan_clock; return it->second.get(); }
    std::unique_ptr<Plan> up(new Plan());
    (this->*build)(*up, B);
    Plan* ret = up.get();
    ret->last_use = ++plan_clock;
    m[B] = std::move(up);
    while ((int)m.size() > max_plans) {
      auto victim = m.end();
      for (auto it = m.begin(); it != m.end(); ++it)
        if (it->second.get() != ret && (victim == m.end() || it->second->last_use < victim->second->last_use)) victim = it;
      if (victim == m.end()) break;
      if (victim->second.get() == last_plan) last_plan = nullptr;
      m.erase(victim);
    }
    return ret;
  }
  Plan* get_embed_plan(int B) { return get_plan(embed_plans, B, &Model::build_embed_plan); }
  Plan* get_detect_plan(int B) { return get_plan(detect_plans, B, &Model::build_detect_plan); }

  void build_embed_plan(Plan& pl, int B) {
    const int S = d.img_size, L = d.unet_levels;
    std::vector<int> z(d.unet_z, d.unet_z + L);
    pl.x_res = pl.pool.alloc_n<float>((size_t)B * 3 * S * S);
    dbg(pl, "x_res", pl.x_res, 0, B, 3, S, S, S);
    pl.delta = pl.pool.alloc_n<float>((size_t)B * d.unet_out_ch * S * S);
    Plan* plp = &pl;
    // ---- inc
    const long M0 = (long)B * S * S;
    __half* h1 = pl.pool.alloc_n<__half>(M0 * z[0]);
    __half* r0 = pl.pool.alloc_n<__half>(M0 * z[0]);
    {
      const int Z = z[0], yuv = d.yuv, cin = d.unet_in_ch;
      const float *w1 = first_w1, *b1 = first_b1, *wr = first_wr, *br = first_br;
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_unet_first(plp->in_imgs, B, S, Z, cin, w1, b1, wr, br, h1, r0, yuv, st); }, 1,
                              "unet.first"});
    }
    dbg(pl, "first_h", h1, 1, B, S, S, z[0], z[0]);
    dbg(pl, "first_r", r0, 1, B, S, S, z[0], z[0]);
    std::vector<__half*> skips;  // outputs of inc, downs[0..]
    std::vector<int> skip_ld;
    __half* x = pl.pool.alloc_n<__half>(M0 * z[0]);
    add_unet_conv(pl, inc_c2, 3, h1, B, S, S, z[0], z[0], true, r0, x, z[0]);
    dbg(pl, "inc", x, 1, B, S, S, z[0], z[0]);
    int ldx = z[0], hs = S;
    const int zb = z[L - 1] + d.hidden;
    __half* cat = nullptr;
    for (int i = 0; i < L - 1; ++i) {
      const int ho = hs / 2;
      const long Mo = (long)B * ho * ho;
      __half* dn = pl.pool.alloc_n<__half>(Mo * z[i + 1]);
      if (down_conv[i].wd) {
        Conv3DirectOp op;
        setup_down_s2d_direct(op, x, z[i], B, ho, ho, z[i + 1], down_conv[i].wd, down_conv[i].bias, dn, num_sms);
        pl.steps.push_back(Step{[op](cudaStream_t st) { launch_direct(op, st); }, 1,
                                "unet.down3x3s2d." + std::to_string(z[i]) + "-" + std::to_string(z[i + 1]) + "@" + std::to_string(ho)});
      } else {
        ConvGemmOp op;
        setup_gather_conv(op, LD_GATHER_CONV, x, z[i], ldx, nullptr, 0, 0, B, hs, hs, ho, ho, 3, 3, 2, 1, 0);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = down_conv[i].bias; op.p.out16 = dn; op.p.ld_out16 = z[i + 1];
        add_conv(pl, op, down_conv[i], "unet.down3x3s2." + std::to_string(z[i]) + "-" + std::to_string(z[i + 1]) + "@" + std::to_string(ho));
      }
      dbg(pl, "down" + std::to_string(i) + "_conv", dn, 1, B, ho, ho, z[i + 1], z[i + 1]);
      __half* out = nullptr; int ld_out = 0;
      if (i == L - 2) {  // last level writes straight into the message-concat buffer (channels [0, z))
        cat = pl.pool.alloc_n<__half>(Mo * zb);
        out = cat; ld_out = zb;
      }
      x = add_resblock(pl, "down" + std::to_string(i), down_rb[i], dn, B, ho, ho, z[i + 1], z[i + 1], out, ld_out);
      ldx = (i == L - 2) ? zb : z[i + 1];
      hs = ho;
      skips.push_back(x); skip_ld.push_back(ldx);
    }
    // ---- message channels
    {
      const int K = d.nbits, hidden = d.hidden, hw = hs * hs, coff = z[L - 1];
      const float* table = msg_table;
      pl.steps.push_back(Step{[=](cudaStream_t st) {
        launch_msg_embed(plp->in_msgs, plp->in_msg_stride, table, K, hidden, cat, B, hw, zb, coff, st);
      }, 1, "unet.msg"});
      dbg(pl, "cat", cat, 1, B, hs, hs, zb, zb);
    }
    // ---- bottleneck
    x = cat; ldx = zb;
    for (int i = 0; i < d.unet_num_blocks; ++i) {
      x = add_resblock(pl, "bott" + std::to_string(i), bott_rb[i], x, B, hs, hs, zb, ldx, nullptr, 0);
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
        setup_up_phase_direct(op, x, Cin, skip, Cin, B, hs, hs, up_phase_w[j], up_lnw[j], up_lnb[j], 1e-6f, u, num_sms);
        pl.steps.push_back(Step{[op](cudaStream_t st) { launch_direct(op, st); }, 1,
                                "unet.upphase." + std::to_string(2 * Cin) + "-" + std::to_string(Cout) + "@" + std::to_string(ho)});
        const __half *x0 = x, *x1 = skip;
        const int IH = hs, Ci = Cin, nsm = num_sms;
        const float *wk = up_border_w[j], *lw = up_lnw[j], *lb = up_lnb[j];
        pl.steps.push_back(Step{[=](cudaStream_t st) { launch_up_border_fix(x0, x1, Ci, B, IH, wk, lw, lb, u, nsm, st); }, 1,
                                "unet.upborder." + std::to_string(Cout) + "@" + std::to_string(ho)});
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
        add_conv(pl, op, up_conv[j], "unet.uptap1x1." + std::to_string(2 * Cin) + "-" + std::to_string(9 * Cout) + "@" + std::to_string(hs));
        dbg(pl, "up" + std::to_string(j) + "_taps", ytap, 1, B, hs, hs, 9 * Cout, 9 * Cout);
        // then bilinear x2 + reflect pad + 3x3 tap sum + LayerNorm + ReLU (CUDA cores, memory-bound)
        const int vpt = up_k[j].vpt;
        UpsGather g;
        g.y = ytap; g.B = B; g.IH = hs; g.C = Cout; g.lnw = up_lnw[j]; g.lnb = up_lnb[j]; g.out = u; g.ld_out = Cout; g.num_sms = num_sms;
        g.optin = kUpGatherSmem;
        g.smem = up_k[j].smem;
        pl.steps.push_back(Step{[g, vpt](cudaStream_t st) { launch_unet_upgather(g, vpt, st); }, 1,
                                "unet.upgather." + std::to_string(Cout) + "@" + std::to_string(ho)});
      }
      dbg(pl, "up" + std::to_string(j) + "_conv", u, 1, B, ho, ho, Cout, Cout);
      const bool last = (ii == 0);
      x = add_resblock(pl, "up" + std::to_string(j), up_rb[j], u, B, ho, ho, Cout, Cout, nullptr, 0, /*fuse_outc=*/last);
      ldx = Cout; hs = ho;
    }
    dbg(pl, "delta", pl.delta, 0, B, d.unet_out_ch, S, S, S);
  }

  void build_detect_plan(Plan& pl, int B) {
    Plan* plp = &pl;
    const int S = d.img_size;
    pl.x_res = pl.pool.alloc_n<float>((size_t)B * 3 * S * S);
    dbg(pl, "x_res", pl.x_res, 0, B, 3, S, S, S);
    pl.logits = pl.pool.alloc_n<float>((size_t)B * (1 + d.nbits));
    if (vit) {
      build_vit_trunk(pl, B);
      return;
    }
    const int st_ = d.ext_stem_stride;
    int hs = (S - 4) / st_ + 1;
    int C = d.ext_dims[0];
    // pixel pitch of every NHWC buffer of the trunk: the width rounded up to 8 channels (16-byte fp16 rows for TMA / vector
    // access; the proportional chunkyseal widths 362 / 724 are not multiples of 8).  Pad channels are never read through a
    // TMA map (its K extent is the true width); the buffers the gather loaders read are zeroed once below.
    auto pitch = [](int c) { return (c + 7) / 8 * 8; };
    int Cp = pitch(C);
    float* x = pl.pool.alloc_n<float>((size_t)B * hs * hs * Cp);
    if (stem_wk != nullptr) {
      // widths > 256: CUDA-core stem conv + LayerNorm (one warp per output pixel); the fused-LN GEMM epilogue needs N <= 256
      const int OH = hs, Cc = C, ldo = Cp, nsm = num_sms;
      const float *wk = stem_wk, *sb = stem_b, *lw = stem_lnw, *lb = stem_lnb;
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_stem_ln(plp->in_imgs, B, S, OH, st_, wk, sb, lw, lb, Cc, x, ldo, nsm, st); }, 1,
                              "cnx.stem_ln." + std::to_string(C) + "@" + std::to_string(hs)});
    } else {
      // stem (convnext.py:108-111): im2col of the k4 patches (x = 2*img-1 folded) -> tensor-core GEMM [M,64]x[64,C0] with the
      // conv bias and the channels-first LayerNorm fused into the epilogue, fp32 NHWC output (the residual stream)
      const int OH = hs, nsm = num_sms;
      const long M = (long)B * OH * OH;
      __half* patches = pl.pool.alloc_n<__half>(M * 64);
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_stem_im2col(plp->in_imgs, B, S, OH, st_, patches, nsm, st); }, 1,
                              "cnx.stem_im2col"});
      ConvGemmOp op; setup_tma_gemm(op, patches, M, 64, 64);
      op.p.epi = EPI_LN; op.p.act = ACT_NONE; op.p.bias = stem_b; op.p.ln_w = stem_lnw; op.p.ln_b = stem_lnb; op.p.ln_eps = 1e-6f;
      op.p.out32 = x; op.p.ld_out32 = Cp;
      ConvW sw; sw.w = stem_w16; sw.N = C; sw.K = 64; sw.bias = stem_b;
      add_conv(pl, op, sw, "cnx.stem_gemm." + std::to_string(C) + "@" + std::to_string(hs));
    }
    // keep_inputs (vsb_debug_keep_inputs): the residual stream is updated in place by every block, so the values a stage's first
    // and last blocks read are copied aside as they pass: s{s}_ds after the stem / down conv, s{s}_in before the last block
    auto keep = [&](const std::string& name, const float* src, int h, int c, int cp) {
      const size_t bytes = (size_t)B * h * h * cp * sizeof(float);
      float* dst = pl.pool.alloc_n<float>((size_t)B * h * h * cp);
      pl.steps.push_back(Step{[=](cudaStream_t st) { VSB_CUDA(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st)); }, 0,
                              "dbg.keep." + name});
      dbg(pl, name, dst, 0, B, h, h, c, cp);
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
    {
      int h2 = hs;
      for (int s = 0; s < 4; ++s) {
        if (s > 0) h2 = (h2 - 2) / 2 + 1;
        const long rps = (long)h2 * h2, Ms = (long)B * rps;
        if (rps % 32 != 0) all_part = false;      // every epilogue warp (32 rows) then lies inside one sample, also in a ragged last tile
        part_n = std::max(part_n, (size_t)((Ms + kBlockM - 1) / kBlockM * 4) * 4 * d.ext_dims[s]);
      }
    }
    float* part_buf = all_part ? pl.pool.alloc_n<float>(part_n) : nullptr;
    if (!all_part)
      pl.steps.push_back(Step{[=](cudaStream_t st) { VSB_CUDA(cudaMemsetAsync(stats_all, 0, 2 * stats_n * sizeof(float), st)); }, 0,
                              "cnx.grn_clear"});
    __half* x16 = nullptr;
    for (int s = 0; s < 4; ++s) {
      if (s > 0) {
        const int Cv = d.ext_dims[s - 1], Cvp = Cp, Cn = d.ext_dims[s], Cnp = pitch(Cn);
        const long Mp = (long)B * hs * hs;
        // pad channels stay zero: ln_rows writes [0, Cv)
        __half* xn = Cvp != Cv ? pl.pool.alloc_zeroed<__half>(Mp * Cvp) : pl.pool.alloc_n<__half>(Mp * Cvp);
        {
          const float *lw = ds[s - 1].lnw, *lb = ds[s - 1].lnb, *xin = x;
          const int nsm = num_sms;
          pl.steps.push_back(Step{[=](cudaStream_t st) { launch_ln_rows(xin, Mp, Cv, Cvp, lw, lb, 1e-6f, xn, Cvp, nsm, st); }, 1, "cnx.ln_rows"});
        }
        dbg(pl, "s" + std::to_string(s) + "_ln", xn, 1, B, hs, hs, Cv, Cvp);
        const int ho = (hs - 2) / 2 + 1;   // odd maps (127, 63, 31): the last row / column is dropped, like nn.Conv2d k2 s2
        float* xo = pl.pool.alloc_n<float>((size_t)B * ho * ho * Cnp);
        ConvGemmOp op;
        // K order (r, s, c) with c over the PADDED width: matches pack_conv(..., pad_taps)
        setup_gather_conv(op, LD_GATHER_CONV, xn, Cvp, Cvp, nullptr, 0, 0, B, hs, hs, ho, ho, 2, 2, 2, 0, 0);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = ds[s - 1].conv.bias; op.p.out32 = xo; op.p.ld_out32 = Cnp;
        add_conv(pl, op, ds[s - 1].conv, "cnx.down2x2s2." + std::to_string(Cv) + "-" + std::to_string(Cn) + "@" + std::to_string(ho));
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
      for (int jb = 0; jb < d.ext_depths[s]; ++jb) {
        const CnBlockW& w = cn[s][jb];
        const bool last = jb == d.ext_depths[s] - 1;
        if (keep_inputs && last) {
          if (jb == 0) dbg(pl, ss + "_in", kept_ds, 0, B, hs, hs, C, Cp);
          else keep(ss + "_in", x, hs, C, Cp);
        }
        {
          const DwConvOp op = setup_dwconv(x, B, hs, C, Cp, w.dww, w.dwb, w.lnw, w.lnb, a);
          pl.steps.push_back(Step{[op](cudaStream_t st) { launch_dwconv(op, st); }, 1,
                                  std::string("cnx.dwconv7_ln.") + dw_kind_name(op.kind) + "." + std::to_string(C) + "@" + std::to_string(hs)});
        }
        {
          ConvGemmOp op; setup_tma_gemm(op, a, M, C, Cp);
          op.p.epi = EPI_AFFINE; op.p.act = ACT_GELU; op.p.bias = w.pw1.bias; op.p.out16 = g; op.p.ld_out16 = 4 * C;
          float* stats = all_part ? part_buf : stats_pp[blk_counter & 1];
          ++blk_counter;
          op.p.grn_stats = stats; op.p.rows_per_sample = rows_per_sample; op.p.grn_part = all_part ? 1 : 0;
          add_conv(pl, op, w.pw1, "cnx.pwconv1." + std::to_string(C) + "@" + std::to_string(hs));
        }
        {
          const int K4 = 4 * C, Cc = C, part_rows = all_part ? rows_per_sample / 32 : 0, nsm = num_sms;
          const float* gamma = w.gamma;
          float* stats = all_part ? part_buf : stats_pp[(blk_counter - 1) & 1];
          float* stats_next = all_part ? nullptr : stats_pp[blk_counter & 1];
          // GRN multiplier folded into per-sample copies of W2 (pointwise.cuh K2e: no pass over g at all), or applied to g in place
          const __half* w2 = w.pw2.w;
          pl.steps.push_back(Step{[=](cudaStream_t st) {
            launch_grn(stats, stats_next, gamma, K4, part_rows, B, w2, w2s, Cc, g, rows_per_sample, nsm, st);
          }, 1, (wscale ? "cnx.grn_wscale." : "cnx.grn_apply.") + std::to_string(C) + "@" + std::to_string(hs)});
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
            dbg(pl, "stage3_16", x16, 1, B, hs, hs, C, Cp);
          }
          add_conv(pl, op, w.pw2, "cnx.pwconv2." + std::to_string(C) + "@" + std::to_string(hs), 0, wscale ? w2s : nullptr);
        }
      }
      // a, g and w2s are reused by every block of the stage: after a run they hold the last block's values (g after the in-place
      // GRN where it is applied)
      dbg(pl, ss + "_a", a, 1, B, hs, hs, C, Cp);
      dbg(pl, ss + "_g", g, 1, B, hs, hs, 4 * C, 4 * C);
      if (wscale) dbg(pl, ss + "_w2s", w2s, 1, B, C, 1, 4 * C, 4 * C);
      dbg(pl, "stage" + std::to_string(s), x, 0, B, hs, hs, C, Cp);
    }
    add_head(pl, x16, B, hs, C, Cp, "cnx.");
  }

  // ---- head (pixel_decoder.py:61-83) on the trunk's fp16 NHWC output x16 [B, hs, hs, C] (pixel pitch Cp)
  void add_head(Plan& pl, const __half* x16, int B, int hs, int C, int Cp, const std::string& prefix) {
    if (pixelwise) {
      add_pixel_decoder(pl, x16, B, hs, Cp);
      return;
    }
    const long M = (long)B * hs * hs;
    float* y = pl.pool.alloc_n<float>(M * Cp);
    ConvGemmOp op;
    setup_gather_conv(op, LD_GATHER_CONV, x16, Cp, Cp, nullptr, 0, 0, B, hs, hs, hs, hs, 3, 3, 1, 1, 1);
    op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = y; op.p.ld_out32 = Cp;
    add_conv(pl, op, head_conv, prefix + "head3x3." + std::to_string(C) + "@" + std::to_string(hs));
    dbg(pl, "head_conv", y, 0, B, hs, hs, C, Cp);
    float* pooled = pl.pool.alloc_n<float>((size_t)B * C);
    dbg(pl, "head_pooled", pooled, 0, B, 1, 1, C, C);
    const int P = hs * hs, Cc = C, ldy = Cp, NO = 1 + d.nbits;
    const float *lw = head_lnw, *lb = head_lnb, *hw = head_lw, *hb = head_lb;
    float* logits = pl.logits;
    pl.steps.push_back(Step{[=](cudaStream_t st) { launch_head(y, B, P, Cc, ldy, lw, lb, pooled, hw, hb, NO, logits, st); }, 2,
                            prefix + "head_tail"});
  }

  // SAM-ViT trunk (modules/vit.py:111-143) on the fp32 residual stream x [B*G*G][E] (token rows in raster order), ending in the
  // fp16 [B, G, G, out_chans] map the head reads
  void build_vit_trunk(Plan& pl, int B) {
    Plan* plp = &pl;
    const int S = d.img_size, G = S / kVitPatch, E = vd.embed_dim, H3 = 3 * E, MLP = vd.mlp_dim, oc = vd.out_chans, nsm = num_sms;
    const long M = (long)B * G * G;
    float* x = pl.pool.alloc_n<float>(M * E);
    float* x0 = pl.pool.alloc_n<float>(M * E);         // patch embedding + position table: block 0 reads it, its proj writes x
    __half* xn = pl.pool.alloc_n<__half>(M * E);       // LayerNorm output, the A operand of qkv / lin1
    __half* qkv = pl.pool.alloc_n<__half>(M * H3);
    __half* att = pl.pool.alloc_n<__half>(M * E);
    __half* hid = pl.pool.alloc_n<__half>(M * MLP);
    __half* x16 = pl.pool.alloc_n<__half>(M * E);      // fp16 copy of the last block's output: the neck's A operand
    {
      // patch embed (vit.py:494-525): im2col of the 16 x 16 patches, GEMM into the fp32 stream, + (pos_embed + folded bias)
      __half* patches = pl.pool.alloc_n<__half>(M * 768);
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_vit_patch_im2col(plp->in_imgs, B, S, patches, nsm, st); }, 1, "vit.patch"});
      ConvGemmOp op; setup_tma_gemm(op, patches, M, 768, 768);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = x0; op.p.ld_out32 = E;
      add_conv(pl, op, vit_patch, "vit.patch");
      const float* table = vit_pos;
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_vit_pos_add(x0, M, G * G, E, table, nsm, st); }, 1, "vit.patch"});
      dbg(pl, "vit.embed", x0, 0, B, G, G, E, E);
    }
    for (int i = 0; i < vd.depth; ++i) {
      const VitBlockW& w = vit_blk[i];
      const std::string bi = "vit.blk" + std::to_string(i);
      const bool global = (vd.global_mask >> i) & 1u;
      const float* xin = i == 0 ? x0 : x;   // the block's input stream
      {
        const float *lw = w.n1w, *lb = w.n1b;
        pl.steps.push_back(Step{[=](cudaStream_t st) { launch_ln_rows(xin, M, E, E, lw, lb, 1e-5f, xn, E, nsm, st); }, 1, "vit.ln"});
      }
      {
        ConvGemmOp op; setup_tma_gemm(op, xn, M, E, E);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.qkv.bias; op.p.out16 = qkv; op.p.ld_out16 = H3;
        add_conv(pl, op, w.qkv, "vit.qkv");
      }
      {
        AttnParams ap{};
        ap.qkv = qkv; ap.out = att; ap.rel_h = w.rel_h; ap.rel_w = w.rel_w;
        ap.G = G; ap.n = global ? G : vd.window_size; ap.heads = vd.num_heads; ap.E = E;
        ap.regions = (G / ap.n) * (G / ap.n); ap.scale = 1.0f / std::sqrt((float)kAttnHd);
        pl.steps.push_back(Step{[=](cudaStream_t st) { launch_vit_attention(ap, B, st); }, 1,
                                global ? "vit.attn_global." + std::to_string(G * G) : "vit.attn_win." + std::to_string(ap.n * ap.n)});
      }
      {
        ConvGemmOp op; setup_tma_gemm(op, att, M, E, E);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.proj.bias; op.p.resid32 = xin; op.p.ld_res32 = E;
        op.p.out32 = x; op.p.ld_out32 = E;   // in place after block 0: each element is read and written by the same thread
        add_conv(pl, op, w.proj, "vit.proj");
      }
      {
        const float *lw = w.n2w, *lb = w.n2b;
        pl.steps.push_back(Step{[=](cudaStream_t st) { launch_ln_rows(x, M, E, E, lw, lb, 1e-5f, xn, E, nsm, st); }, 1, "vit.ln"});
      }
      {
        ConvGemmOp op; setup_tma_gemm(op, xn, M, E, E);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_GELU; op.p.bias = w.lin1.bias; op.p.out16 = hid; op.p.ld_out16 = MLP;
        add_conv(pl, op, w.lin1, "vit.lin1");
      }
      {
        ConvGemmOp op; setup_tma_gemm(op, hid, M, MLP, MLP);
        op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.bias = w.lin2.bias; op.p.resid32 = x; op.p.ld_res32 = E;
        op.p.out32 = x; op.p.ld_out32 = E;
        if (i + 1 == vd.depth) { op.p.out16 = x16; op.p.ld_out16 = E; }
        add_conv(pl, op, w.lin2, "vit.lin2");
      }
      // the stream, qkv and att buffers are reused by every block, so they hold the LAST block's values after a run: only its taps
      // exist.  Per-block copies would cost ~0.9 GB per 64-frame 256^2 plan; block k - 1 of a model is compared through the model
      // of depth k built from the same checkpoint prefix (tests/test_vit_gpu.py)
      if (i + 1 == vd.depth) {
        dbg(pl, bi + ".qkv", qkv, 1, B, G, G, H3, H3);
        dbg(pl, bi + ".attn", att, 1, B, G, G, E, E);
        dbg(pl, bi, x, 0, B, G, G, E, E);
      }
    }
    // neck (vit.py:90-109): 1x1 conv, LayerNorm2d, 3x3 conv (zero padding 1), LayerNorm2d; both without bias, eps 1e-6
    float* y = pl.pool.alloc_n<float>(M * oc);
    __half* yn = pl.pool.alloc_n<__half>(M * oc);
    __half* out = pl.pool.alloc_n<__half>(M * oc);
    {
      ConvGemmOp op; setup_tma_gemm(op, x16, M, E, E);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = y; op.p.ld_out32 = oc;
      add_conv(pl, op, vit_neck1, "vit.neck1x1");
      const float *lw = vit_nln1w, *lb = vit_nln1b;
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_ln_rows(y, M, oc, oc, lw, lb, 1e-6f, yn, oc, nsm, st); }, 1, "vit.neck_ln"});
    }
    {
      ConvGemmOp op;
      setup_gather_conv(op, LD_GATHER_CONV, yn, oc, oc, nullptr, 0, 0, B, G, G, G, G, 3, 3, 1, 1, 0);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out32 = y; op.p.ld_out32 = oc;
      add_conv(pl, op, vit_neck3, "vit.neck3x3");
      const float *lw = vit_nln2w, *lb = vit_nln2b;
      pl.steps.push_back(Step{[=](cudaStream_t st) { launch_ln_rows(y, M, oc, oc, lw, lb, 1e-6f, out, oc, nsm, st); }, 1, "vit.neck_ln"});
    }
    dbg(pl, "vit.neck", out, 1, B, G, G, oc, oc);
    add_head(pl, out, B, G, oc, oc, "vit.");
  }

  // Pixel-wise decoder stages.  Each stage is one tensor-core GEMM at the LOW resolution, Y[p, tap*C_out + co] (the tap trick of the
  // U-Net's up-convolutions: bilinear up-sampling, reflection padding and the 3x3 taps are linear, so the channel mixing commutes
  // with the spatial gather), then ups_gather_ln_*_kernel forms each output pixel from 9 taps x 4 bilinear corners + LN + GELU.
  // The last stage's kernel also applies the 1x1 head and writes the 1+K NCHW maps straight into the caller's buffer (plp->out_maps):
  // the full-resolution activation never goes to HBM.
  void add_pixel_decoder(Plan& pl, const __half* x, int B, int h, int ldx) {
    Plan* plp = &pl;
    const int NO = 1 + d.nbits, nsm = num_sms;
    for (size_t i = 0; i < pd.size(); ++i) {
      const PdStageW& s = pd[i];
      const int F = s.f, ho = F * h, Co = s.cout, IH = h;
      const bool last = i + 1 == pd.size();
      const long Mi = (long)B * h * h;
      __half* ytap = pl.pool.alloc_n<__half>(Mi * 9 * Co);
      ConvGemmOp op; setup_tma_gemm(op, x, Mi, s.kin, ldx);
      op.p.epi = EPI_AFFINE; op.p.act = ACT_NONE; op.p.out16 = ytap; op.p.ld_out16 = 9 * Co;
      add_conv(pl, op, s.taps, "pd.uptap1x1." + std::to_string(s.cin) + "-" + std::to_string(9 * Co) + "@" + std::to_string(h));
      dbg(pl, "pd" + std::to_string(i) + "_y", ytap, 1, B, h, h, 9 * Co, 9 * Co);
      UpsGather g;
      g.y = ytap; g.B = B; g.IH = IH; g.C = Co; g.lnw = s.lnw; g.lnb = s.lnb; g.num_sms = nsm; g.optin = kPdMaxSmem;
      g.smem = s.smem;
      const int vpt = s.vpt;
      const std::string tag = std::to_string(Co) + "x" + std::to_string(F) + "@" + std::to_string(ho);
      if (last) {
        g.hw = pd_hw; g.hb = pd_hb; g.NO = NO;
        pl.steps.push_back(Step{[g, F, vpt, plp](cudaStream_t st) mutable { g.maps = plp->out_maps; launch_pd_gather(g, F, vpt, st); }, 1,
                                "pd.gather_head." + tag});
      } else {
        const int ldo = pd_gemm_k(Co);
        // pad channels stay zero: the gather writes [0, Co)
        __half* u = ldo != Co ? pl.pool.alloc_zeroed<__half>((size_t)B * ho * ho * ldo) : pl.pool.alloc_n<__half>((size_t)B * ho * ho * ldo);
        g.out = u; g.ld_out = ldo;
        pl.steps.push_back(Step{[g, F, vpt](cudaStream_t st) { launch_pd_gather(g, F, vpt, st); }, 1,
                                std::string(g.smem ? "pd.upgather." : "pd.upgather_untiled.") + tag});
        dbg(pl, "pd" + std::to_string(i), u, 1, B, ho, ho, Co, ldo);
        x = u; ldx = ldo;
      }
      h = ho;
    }
  }

  ResampleDev* get_resampler(int ih, int iw, int oh, int ow, ResampleMode m) {
    const auto key = std::make_tuple(ih, iw, oh, ow, m.mode, m.align_corners, m.antialias);
    auto it = resamplers.find(key);
    if (it != resamplers.end()) return it->second.get();
    std::unique_ptr<ResampleDev> r(new ResampleDev(ih, iw, oh, ow, m));
    ResampleDev* ret = r.get();
    resamplers[key] = std::move(r);
    return ret;
  }

  // resample `n` frames that are `frame_stride` floats apart to S x S (one launch, also for strided key frames)
  void resize_frames(const float* src, long frame_stride, int n, int H, int W, float* dst, ResampleMode rm, cudaStream_t st) {
    const int S = d.img_size;
    const ResampleDev* r = get_resampler(H, W, S, S, rm);
    for (int i = 0; i < n; i += 16384) {   // gridDim.y limit: split very long frame ranges
      const int m = std::min(16384, n - i);
      prof_scope("pw.resize." + std::to_string(H) + "x" + std::to_string(W) + "@" + std::to_string(m), st, 1, [&] {
        launch_resize(*r, src + (long)i * frame_stride, frame_stride, m, H, W, S, S, dst + (size_t)i * 3 * S * S, last_resize, st);
      });
    }
  }

  void check_ready() const { if (!finalized) throw Error("model not finalized", kErrState); }

  // ---- streaming host path: embed + detect of HOST frames with the PCIe copies overlapped with compute
  cudaStream_t s_in = nullptr, s_cmp = nullptr, s_out = nullptr;
  std::vector<cudaEvent_t> ev_in, ev_cmp;
  // creates the three streams once and at least n (input, compute) event pairs
  void stream_setup(size_t n) {
    if (!s_in) {
      VSB_CUDA(cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking));
      VSB_CUDA(cudaStreamCreateWithFlags(&s_cmp, cudaStreamNonBlocking));
      VSB_CUDA(cudaStreamCreateWithFlags(&s_out, cudaStreamNonBlocking));
    }
    while (ev_in.size() < n) {
      cudaEvent_t a, b;
      VSB_CUDA(cudaEventCreateWithFlags(&a, cudaEventDisableTiming));
      VSB_CUDA(cudaEventCreateWithFlags(&b, cudaEventDisableTiming));
      ev_in.push_back(a); ev_cmp.push_back(b);
    }
  }
  // frames that must stay in one batch: a key frame and its step - 1 followers, or in 'interpolate' mode, where neighbouring keys
  // of one reference chunk are mixed, whole chunks
  static int key_unit(int step, int video_mode, int chunk_keys) {
    return (video_mode == VSB_VIDEO_INTERPOLATE && step > 1) ? step * std::max(1, chunk_keys) : step;
  }
  void embed_detect_host(const float* imgs_h, const uint8_t* msgs_h, int n_msgs, float* imgs_w_h, float* logits_h, int F, int H, int W,
                         int step, int video_mode, int chunk_keys, float scaling_i, float scaling_w, int flags) {
    check_ready();
    const size_t fpx = (size_t)3 * H * W;
    const int NO = 1 + d.nbits;
    float* imgs = (float*)stage(0, (size_t)F * fpx * sizeof(float));
    float* out = (float*)stage(1, (size_t)F * fpx * sizeof(float));
    float* lg = (float*)stage(2, (size_t)F * NO * sizeof(float));
    uint8_t* msgs = (uint8_t*)stage(3, (size_t)n_msgs * d.nbits + 256);
    // Pipeline (three streams): frames travel in SLICES (a short first one, then ~48; multiples of `step`, and of whole reference chunks in
    // 'interpolate' mode where neighbouring keys of one chunk are mixed, so that key-frame groups stay whole); embed() runs per
    // slice as soon as its copy has landed, the D2H of a slice's watermarked frames starts as soon as its embed() is done and
    // runs under the following compute; detect() runs once 64 frames have accumulated (full-size extractor batches) and on the tail.
    // Exposed copies: the first slice in and the last group's logits out.
    // Slice sizes: the FIRST slice's copy is the exposed one, so it is shorter than the rest.  Measured at 64 x 3x256x256 (results
    // bit-identical for every setting): first/rest 32/32 7 165 f/s, 24/40 7 207, 16/48 7 317, 8/56 7 310, 16/24 7 020 -> 16 / 48.
    const int unit = key_unit(step, video_mode, chunk_keys);
    const int sl0 = (16 + unit - 1) / unit * unit, sl1 = (48 + unit - 1) / unit * unit;
    std::vector<std::pair<int, int>> slices;   // (first frame, frames)
    for (int f0 = 0; f0 < F;) {
      const int n = std::min(slices.empty() ? sl0 : sl1, F - f0);
      slices.push_back({f0, n});
      f0 += n;
    }
    const int nsl = (int)slices.size();
    stream_setup(nsl + 1);
    VSB_CUDA(cudaMemcpyAsync(msgs, msgs_h, (size_t)n_msgs * d.nbits, cudaMemcpyHostToDevice, s_in));
    for (int k = 0; k < nsl; ++k) {       // all input copies are queued up front: s_in runs ahead of the compute
      const int f0 = slices[k].first, n = slices[k].second;
      VSB_CUDA(cudaMemcpyAsync(imgs + (size_t)f0 * fpx, imgs_h + (size_t)f0 * fpx, (size_t)n * fpx * sizeof(float), cudaMemcpyHostToDevice, s_in));
      VSB_CUDA(cudaEventRecord(ev_in[k], s_in));
    }
    int g0 = 0;                           // first frame not yet detected
    for (int k = 0; k < nsl; ++k) {
      const int f0 = slices[k].first, n = slices[k].second;
      VSB_CUDA(cudaStreamWaitEvent(s_cmp, ev_in[k], 0));
      const uint8_t* mk = msgs + (n_msgs == 1 ? 0 : (size_t)f0 * d.nbits);
      embed(imgs + (size_t)f0 * fpx, mk, n_msgs == 1 ? 1 : n, out + (size_t)f0 * fpx, nullptr, n, H, W, step, video_mode, chunk_keys, scaling_i,
            scaling_w, flags, s_cmp);
      VSB_CUDA(cudaEventRecord(ev_cmp[k], s_cmp));
      VSB_CUDA(cudaStreamWaitEvent(s_out, ev_cmp[k], 0));
      VSB_CUDA(cudaMemcpyAsync(imgs_w_h + (size_t)f0 * fpx, out + (size_t)f0 * fpx, (size_t)n * fpx * sizeof(float), cudaMemcpyDeviceToHost, s_out));
      if (f0 + n - g0 >= kMaxBatch || k == nsl - 1) {   // a full extractor batch (or the tail) is complete: detect its frames
        const int gn = f0 + n - g0;
        detect(out + (size_t)g0 * fpx, lg + (size_t)g0 * NO, gn, H, W, flags & VSB_FLAG_RESIZE_BITS, s_cmp);
        VSB_CUDA(cudaEventRecord(ev_cmp[nsl], s_cmp));
        VSB_CUDA(cudaStreamWaitEvent(s_out, ev_cmp[nsl], 0));
        VSB_CUDA(cudaMemcpyAsync(logits_h + (size_t)g0 * NO, lg + (size_t)g0 * NO, (size_t)gn * NO * sizeof(float), cudaMemcpyDeviceToHost, s_out));
        g0 = f0 + n;
      }
    }
    VSB_CUDA(cudaStreamSynchronize(s_out));
  }

  // ---- the same streaming scheme with RGB24 frames [F,H,W,3] uint8 on the host (inference_streaming.py:23-33,116-124):
  // out_h == nullptr -> detect only (logits of the input frames); logits_h == nullptr -> embed only; both -> the logits are
  // those of the re-quantised watermarked frames, which is what the reference's detect pass reads back from the encoder
  void frames_host_u8(const uint8_t* in_h, const uint8_t* msgs_h, int n_msgs, uint8_t* out_h, float* logits_h, int F, int H, int W,
                      int step, int video_mode, int chunk_keys, float scaling_i, float scaling_w, int flags) {
    check_ready();
    const bool do_embed = out_h != nullptr, do_detect = logits_h != nullptr;
    VSB_CHECK(do_embed || do_detect, "nothing to do");
    const size_t fpx = (size_t)3 * H * W;
    const long plane = (long)H * W;
    const int NO = 1 + d.nbits;
    float* imgs = (float*)stage(0, (size_t)F * fpx * sizeof(float));
    float* out = do_embed ? (float*)stage(1, (size_t)F * fpx * sizeof(float)) : nullptr;
    float* lg = do_detect ? (float*)stage(2, (size_t)F * NO * sizeof(float)) : nullptr;
    uint8_t* msgs = do_embed ? (uint8_t*)stage(3, (size_t)n_msgs * d.nbits + 256) : nullptr;
    uint8_t* in8 = (uint8_t*)stage(4, (size_t)F * fpx);
    uint8_t* out8 = do_embed ? (uint8_t*)stage(5, (size_t)F * fpx) : nullptr;
    int ch = kMaxBatch;   // one-byte samples: the exposed first/last copies are short, so full 64-frame batches win
    const int unit = key_unit(step, video_mode, chunk_keys);
    if (ch % unit) ch = ((ch + unit - 1) / unit) * unit;
    const int nch = (F + ch - 1) / ch;
    stream_setup(nch);
    if (do_embed) VSB_CUDA(cudaMemcpyAsync(msgs, msgs_h, (size_t)n_msgs * d.nbits, cudaMemcpyHostToDevice, s_in));
    for (int k = 0; k < nch; ++k) {
      const int f0 = k * ch, n = std::min(ch, F - f0);
      VSB_CUDA(cudaMemcpyAsync(in8 + (size_t)f0 * fpx, in_h + (size_t)f0 * fpx, (size_t)n * fpx, cudaMemcpyHostToDevice, s_in));
      VSB_CUDA(cudaEventRecord(ev_in[k], s_in));
      VSB_CUDA(cudaStreamWaitEvent(s_cmp, ev_in[k], 0));
      const long npx = (long)n * plane;
      launch_u8_to_f32(in8 + (size_t)f0 * fpx, imgs + (size_t)f0 * fpx, npx, plane, num_sms, s_cmp);
      g_launches += 1;
      const float* det_in = imgs + (size_t)f0 * fpx;
      if (do_embed) {
        const uint8_t* mk = msgs + (n_msgs == 1 ? 0 : (size_t)f0 * d.nbits);
        embed(imgs + (size_t)f0 * fpx, mk, n_msgs == 1 ? 1 : n, out + (size_t)f0 * fpx, nullptr, n, H, W, step, video_mode, chunk_keys,
              scaling_i, scaling_w, flags, s_cmp);
        launch_f32_to_u8(out + (size_t)f0 * fpx, out8 + (size_t)f0 * fpx, do_detect ? out + (size_t)f0 * fpx : nullptr, npx, plane, num_sms,
                         s_cmp);
        g_launches += 1;
        det_in = out + (size_t)f0 * fpx;
      }
      if (do_detect) detect(det_in, lg + (size_t)f0 * NO, n, H, W, flags & VSB_FLAG_RESIZE_BITS, s_cmp);
      VSB_CUDA(cudaGetLastError());
      VSB_CUDA(cudaEventRecord(ev_cmp[k], s_cmp));
      VSB_CUDA(cudaStreamWaitEvent(s_out, ev_cmp[k], 0));
      if (do_embed) VSB_CUDA(cudaMemcpyAsync(out_h + (size_t)f0 * fpx, out8 + (size_t)f0 * fpx, (size_t)n * fpx, cudaMemcpyDeviceToHost, s_out));
      if (do_detect) VSB_CUDA(cudaMemcpyAsync(logits_h + (size_t)f0 * NO, lg + (size_t)f0 * NO, (size_t)n * NO * sizeof(float), cudaMemcpyDeviceToHost, s_out));
    }
    VSB_CUDA(cudaStreamSynchronize(s_out));
  }

  // U-Net on `n` processing-size RGB frames (contiguous [n,3,S,S]) -> plan->delta
  Plan* run_unet(const float* x, const uint8_t* msgs, int msg_stride, int n, cudaStream_t st) {
    Plan* pl = get_embed_plan(n);
    pl->in_imgs = x;
    pl->in_frame_stride = (long)3 * d.img_size * d.img_size;
    pl->in_msgs = msgs;
    pl->in_msg_stride = msg_stride;
    pl->run(st);
    last_plan = pl;
    return pl;
  }

  void embedder_forward(const float* x, const uint8_t* msgs, int n_msgs, float* delta, int B, cudaStream_t st) {
    check_ready();
    VSB_CHECK(n_msgs == 1 || n_msgs == B, "msgs must be [1,K] or [B,K]");
    const int S = d.img_size;
    for (int b0 = 0; b0 < B; b0 += kMaxBatch) {
      const int n = std::min(kMaxBatch, B - b0);
      Plan* pl = run_unet(x + (size_t)b0 * 3 * S * S, msgs + (n_msgs == 1 ? 0 : (size_t)b0 * d.nbits), n_msgs == 1 ? 0 : d.nbits, n, st);
      VSB_CUDA(cudaMemcpyAsync(delta + (size_t)b0 * d.unet_out_ch * S * S, pl->delta, (size_t)n * d.unet_out_ch * S * S * sizeof(float),
                               cudaMemcpyDeviceToDevice, st));
    }
  }

  void embed(const float* imgs, const uint8_t* msgs, int n_msgs, float* imgs_w, float* preds_w, int F, int H, int W, int step,
             int video_mode, int chunk_keys, float scaling_i, float scaling_w, int flags, cudaStream_t st) {
    check_ready();
    VSB_CHECK(F > 0 && H > 0 && W > 0 && step >= 1, "bad embed shape");
    VSB_CHECK(n_msgs == 1 || (n_msgs == F && step == 1), "msgs must be [1,K], or [F,K] in image mode");
    // 'interpolate' mixes neighbouring key frames inside one reference chunk (videoseal.py:300-331 chunks by chunk_size
    // key frames; :101-113 interpolates within the chunk), so U-Net batches are whole chunks in that mode
    const bool interp = (video_mode == VSB_VIDEO_INTERPOLATE) && step > 1;
    if (interp) VSB_CHECK(chunk_keys >= 1 && chunk_keys <= kMaxBatch, "video_mode='interpolate' needs 1 <= chunk_size <= 64");
    const int kbatch = interp ? (kMaxBatch / chunk_keys) * chunk_keys : kMaxBatch;
    const int bint = interp ? chunk_keys : 0;
    const int S = d.img_size;
    const bool same = (H == S && W == S);
    const ResampleMode rm = same ? ResampleMode() : resample_mode(flags);   // (the flags are read only when a resize happens)
    const bool use_jnd = !(flags & VSB_FLAG_NO_ATTENUATION) && d.jnd_in_ch != 0;
    // channels of hmaps * preds_w (broadcast): what `preds_w` holds and what the low-resolution path hands to the blend
    const int PC = use_jnd ? std::max(d.unet_out_ch, d.jnd_out_ch) : d.unet_out_ch;
    const bool lowres = use_jnd && (flags & VSB_FLAG_LOWRES_ATTN);
    const long fstride = (long)3 * H * W;
    const int nkeys = (F + step - 1) / step;
    ResampleDev* up = same ? nullptr : get_resampler(S, S, H, W, rm);
    for (int k0 = 0; k0 < nkeys; k0 += kbatch) {
      const int nk = std::min(kbatch, nkeys - k0);
      const int f0 = k0 * step, f1 = std::min(F, (k0 + nk) * step);
      const int nf = f1 - f0;
      Plan* pl = get_embed_plan(nk);
      const float* x = imgs + (size_t)f0 * fstride;
      // low-resolution attenuation needs EVERY frame of the chunk at processing size (wam.py:177-180, videoseal.py:321-324):
      // resample them once into a grow-only scratch buffer of the model (no allocation or synchronisation on the steady-state
      // path) and take the key frames from there
      const float* frames_res = x;
      if (lowres && !same) {
        float* fr = (float*)stage(6, (size_t)nf * 3 * S * S * sizeof(float));
        resize_frames(x, fstride, nf, H, W, fr, rm, st);
        frames_res = fr;
      }
      if (!same || step != 1) {
        // key frames -> contiguous processing-size RGB batch
        if (same || lowres) {
          VSB_CUDA(cudaMemcpy2DAsync(pl->x_res, (size_t)3 * S * S * sizeof(float), frames_res, (size_t)step * 3 * S * S * sizeof(float),
                                     (size_t)3 * S * S * sizeof(float), nk, cudaMemcpyDeviceToDevice, st));
        } else {
          resize_frames(x, (long)step * fstride, nk, H, W, pl->x_res, rm, st);
        }
        x = pl->x_res;
      }
      run_unet(x, msgs + (n_msgs == 1 ? 0 : (size_t)k0 * d.nbits), n_msgs == 1 ? 0 : d.nbits, nk, st);
      const float* delta = pl->delta;
      const int balt = (video_mode == VSB_VIDEO_ALTERNATE) ? 1 : 0;
      BlendParams bp;
      memset(&bp, 0, sizeof(bp));
      bp.imgs = imgs + (size_t)f0 * fstride; bp.imgs_w = imgs_w + (size_t)f0 * fstride;
      bp.preds_w = preds_w ? preds_w + (size_t)f0 * PC * H * W : nullptr;
      bp.F = nf; bp.H = H; bp.W = W; bp.PH = S; bp.PW = S; bp.CD = d.unet_out_ch;
      bp.jnd_in = d.jnd_in_ch ? d.jnd_in_ch : 1; bp.jnd_out = d.jnd_out_ch ? d.jnd_out_ch : 1;
      bp.clamp = (flags & VSB_FLAG_CLAMP) ? 1 : 0; bp.identity_resample = same ? 1 : 0;
      bp.scaling_i = scaling_i; bp.scaling_w = scaling_w;
      if (up) bp.tab = up->tab;
      if (lowres) {
        // per-frame attenuated delta at processing size: out[f] = hmap(frames_res[f]) * delta(keys of f); then a plain blend
        float* lowres_buf = (float*)stage(7, (size_t)nf * PC * S * S * sizeof(float));
        VSB_CHECK(nf <= 65535, "too many frames per key-frame batch");
        prof_scope("pw.jnd_lowres@" + std::to_string(nf), st, 1, [&] {
          launch_jnd_lowres(frames_res, delta, lowres_buf, nf, S, S, d.unet_out_ch, step, balt, bint, bp.jnd_in, bp.jnd_out, st);
        });
        bp.delta = lowres_buf; bp.step = 1; bp.alternate = 0; bp.interp_chunk = 0; bp.use_jnd = 0; bp.CD = PC;
      } else {
        bp.delta = delta; bp.step = step; bp.alternate = balt; bp.interp_chunk = bint; bp.use_jnd = use_jnd ? 1 : 0;
      }
      prof_scope(std::string(bp.use_jnd ? "pw.jnd_blend." : "pw.blend.") + std::to_string(bp.H) + "x" + std::to_string(bp.W) + "@" +
                     std::to_string(bp.F) + (bp.preds_w ? "+preds" : ""), st, 1, [&] { launch_blend(bp, up, last_blend, st); });
    }
  }

  void jnd_heatmaps(const float* imgs, float* hmaps, int F, int H, int W, cudaStream_t st) {
    // heat-map only (operator seam, modules/jnd.py:80-108): jnd_lowres_kernel with delta == nullptr writes hmap * 1; hmaps [F, jnd_out, H, W]
    VSB_CHECK(F <= 65535, "too many frames");
    VSB_CHECK(d.jnd_in_ch != 0, "the card has no JND attenuation");
    launch_jnd_lowres(imgs, nullptr, hmaps, F, H, W, 1, 1, 0, 0, d.jnd_in_ch, d.jnd_out_ch, st);
    g_launches += 1;
  }

  void detect(const float* imgs, float* logits, int F, int H, int W, int flags, cudaStream_t st) {
    check_ready();
    VSB_CHECK(F > 0 && H > 0 && W > 0, "bad detect shape");
    const int S = d.img_size;
    const bool same = (H == S && W == S);
    const ResampleMode rm = same ? ResampleMode() : resample_mode(flags);
    const long fstride = (long)3 * H * W;
    const size_t NO = detect_out_per_frame();
    for (int f0 = 0; f0 < F; f0 += kMaxBatch) {
      const int n = std::min(kMaxBatch, F - f0);
      Plan* pl = get_detect_plan(n);
      const float* x = imgs + (size_t)f0 * fstride;
      if (!same) { resize_frames(x, fstride, n, H, W, pl->x_res, rm, st); x = pl->x_res; }
      pl->in_imgs = x;
      pl->out_maps = pixelwise ? logits + (size_t)f0 * NO : nullptr;   // the maps are written in place, at this sub-batch's offset
      pl->run(st);
      last_plan = pl;
      if (!pixelwise)
        VSB_CUDA(cudaMemcpyAsync(logits + (size_t)f0 * NO, pl->logits, (size_t)n * NO * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
  }
};

}  // namespace vsb
