// The model behind the C ABI: the descriptor and the units of its networks (unet.cuh, convnext.cuh / vit_trunk.cuh, decoder.cuh),
// the plan cache, and the embed / detect drivers and host-buffer pipelines.
#pragma once
#include <memory>
#include <mutex>
#include <tuple>

#include "convnext.cuh"
#include "decoder.cuh"
#include "dvmark.cuh"
#include "dvmark_enc.cuh"
#include "hidden.cuh"
#include "resize_blend_host.cuh"
#include "unet.cuh"
#include "vae.cuh"
#include "vit_trunk.cuh"

namespace vsb {

class Model {
 public:
  vsb_model_desc d;
  bool finalized = false;
  int device = -1, num_sms = 0;
  std::recursive_mutex mu;   // serialises the C entry points of one handle (vsb200.cu VSB_MODEL_SCOPE)
  Weights ws;
  static constexpr int kMaxBatch = 64;
  UNet unet;
  ConvNeXt cnx;
  VitTrunk vit;
  Decoder dec;
  Hidden henc, hdec;   // HiDDeN embedder / extractor, in place of the U-Net / the trunk and decoder (vsb_model_set_hidden_*)
  DVMark dvdec;        // DVMark extractor, in place of the trunk and decoder (vsb_model_set_dvmark_extractor)
  DVMarkEnc dvenc;     // DVMark embedder, in place of the U-Net (vsb_model_set_dvmark_embedder)
  VaeEnc vae;          // VAE embedder, in place of the U-Net (vsb_model_set_vae_embedder)

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
  // test seam (vsb_debug_keep_inputs): detect plans (and HiDDeN embed plans) copy buffers that later steps overwrite aside; DVMark
  // and VAE embed plans give every map a buffer of its own
  bool keep_inputs = false;
  void set_keep_inputs(bool on) {
    keep_inputs = on;
    for (auto& kv : detect_plans) if (kv.second.get() == last_plan) last_plan = nullptr;
    detect_plans.clear();
    if (henc.on || dvenc.on || vae.on) {   // HiDDeN, DVMark and VAE embed plans have the seam too (their build)
      for (auto& kv : embed_plans) if (kv.second.get() == last_plan) last_plan = nullptr;
      embed_plans.clear();
    }
  }

  // vsb_model_create: every rule that depends only on the descriptor, and the U-Net's kernels (no CUDA calls)
  // A descriptor with no U-Net levels and 3 input / output channels leaves the embedder to vsb_model_set_hidden_embedder: its U-Net
  // rules are checked at finalize when no HiDDeN embedder was set (so such a descriptor still fails, with the U-Net's message).
  explicit Model(const vsb_model_desc& desc) : d(desc) {
    if (!other_embedder()) unet.check(d);
    if (d.jnd_in_ch != 0 && !((d.jnd_in_ch == 1 || d.jnd_in_ch == 3) && (d.jnd_out_ch == 1 || d.jnd_out_ch == 3)))
      throw Error("JND attenuation: in_channels / out_channels must be 1 or 3 (configs/attenuation.yaml)", kErrUnsupported);
    ConvNeXt::check(d);
    if (!other_embedder()) unet.choose_kernels();
  }
  // no U-Net levels but the embedder's RGB in / out channels: the embedder is set by vsb_model_set_hidden_embedder,
  // vsb_model_set_dvmark_embedder or vsb_model_set_vae_embedder
  bool other_embedder() const { return d.unet_levels == 0 && d.unet_in_ch == 3 && d.unet_out_ch == 3; }
  void check_unfinalized() const { if (finalized) throw Error("model already finalized", kErrState); }
  // channels of the embedder's output delta
  int delta_ch() const { return vae.on ? vae.v.out_ch : ((henc.on || dvenc.on) ? 3 : d.unet_out_ch); }
  // the embedder's 3x3x3 convs mix the key frames of one embedder call (a temporal U-Net or a DVMark embedder)
  bool frame_mixing_embedder() const { return unet.temporal || dvenc.on; }
  void set_hidden_embedder(const vsb_hidden_desc& h) {
    check_unfinalized();
    if (dvenc.on || vae.on) throw Error("vsb_model_set_hidden_embedder: the model already has a DVMark or VAE embedder", kErrState);
    if (!other_embedder())
      throw Error("vsb_model_set_hidden_embedder: the descriptor describes a U-Net (a HiDDeN embedder needs unet_levels 0 and unet_in_ch / "
                  "unet_out_ch 3)", kErrInvalid);
    Hidden e;
    e.set(h, true, d);
    henc = e;
  }
  void set_hidden_extractor(const vsb_hidden_desc& h) {
    check_unfinalized();
    if (vit.on || dec.pixelwise) throw Error("vsb_model_set_hidden_extractor: the model already has a SAM-ViT trunk or a pixel-wise decoder", kErrState);
    for (int s = 0; s < 4; ++s)
      if (d.ext_dims[s] != 0 || d.ext_depths[s] != 0)
        throw Error("vsb_model_set_hidden_extractor: the descriptor also describes a ConvNeXt trunk (ext_dims / ext_depths != 0)", kErrInvalid);
    Hidden e;
    e.set(h, false, d);
    hdec = e;
  }
  void set_dvmark_embedder(int nbits) {
    check_unfinalized();
    if (henc.on || unet.temporal || vae.on)
      throw Error("vsb_model_set_dvmark_embedder: the model already has a HiDDeN or VAE embedder or a temporal U-Net", kErrState);
    if (!other_embedder())
      throw Error("vsb_model_set_dvmark_embedder: the descriptor describes a U-Net (a DVMark embedder needs unet_levels 0 and "
                  "unet_in_ch / unet_out_ch 3)", kErrInvalid);
    DVMarkEnc e;
    e.set(nbits, d);
    dvenc = e;
  }
  void set_vae_embedder(const vsb_vae_desc& v) {
    check_unfinalized();
    if (henc.on || dvenc.on || unet.temporal)
      throw Error("vsb_model_set_vae_embedder: the model already has a HiDDeN or DVMark embedder or a temporal U-Net", kErrState);
    if (!other_embedder())
      throw Error("vsb_model_set_vae_embedder: the descriptor describes a U-Net (a VAE embedder needs unet_levels 0 and "
                  "unet_in_ch / unet_out_ch 3)", kErrInvalid);
    VaeEnc e;
    e.set(v, d);
    vae = e;
  }
  void set_dvmark_extractor(int nbits) {
    check_unfinalized();
    if (vit.on || dec.pixelwise || hdec.on)
      throw Error("vsb_model_set_dvmark_extractor: the model already has a SAM-ViT trunk, a pixel-wise decoder or a HiDDeN extractor", kErrState);
    for (int s = 0; s < 4; ++s)
      if (d.ext_dims[s] != 0 || d.ext_depths[s] != 0)
        throw Error("vsb_model_set_dvmark_extractor: the descriptor also describes a ConvNeXt trunk (ext_dims / ext_depths != 0)", kErrInvalid);
    DVMark e;
    e.set(nbits, d);
    dvdec = e;
  }
  // the entry points that detect slices of a stream cut it on their own boundaries, not on the DVMark extractor's groups
  void check_frame_independent_detect(const std::string& what) const {
    if (dvdec.on)
      throw Error(what + ": a DVMark extractor convolves across the frames of a group, which the streamed slices would split; use "
                  "vsb_detect_grouped", kErrUnsupported);
  }
  void set_tensor(const char* name, const float* data, const int64_t* shape, int ndim) {
    check_unfinalized();
    HostTensor t;
    t.shape.assign(shape, shape + ndim);
    t.data.assign(data, data + t.numel());
    ws.sd[name] = std::move(t);
  }
  void set_pixel_decoder(int n, const int32_t* f, int pw) {
    check_unfinalized();
    if (hdec.on && pw != 0) throw Error("HiDDeN extractor: per-pixel maps (pixelwise) are not implemented", kErrUnsupported);
    if (dvdec.on && pw != 0) throw Error("DVMark extractor: per-pixel maps (pixelwise) are not implemented", kErrUnsupported);
    dec.set(n, f, pw, vit.on || d.ext_stem_stride == 4, d.nbits, [&] { return std::make_pair(trunk_width(), trunk_map()); });
  }
  // the U-Net's rules and kernel choice again, for a temporal U-Net
  void set_unet_temporal(int on) {
    check_unfinalized();
    VSB_CHECK(on == 0 || on == 1, "temporal must be 0 or 1");
    UNet u;
    u.temporal = on != 0;
    u.check(d);
    u.choose_kernels();
    unet = std::move(u);
  }
  void set_vit_extractor(const vsb_vit_desc& v) {
    check_unfinalized();
    if (dec.pixelwise) throw Error("vsb_model_set_vit_extractor must come before vsb_model_set_pixel_decoder", kErrState);
    if (hdec.on || dvdec.on) throw Error("vsb_model_set_vit_extractor: the model already has a HiDDeN or DVMark extractor", kErrState);
    vit.set(v, d.img_size);
  }
  int trunk_width() const { return vit.on ? vit.width() : d.ext_dims[3]; }
  int trunk_map() const { return vit.on ? VitTrunk::map(d.img_size) : ConvNeXt::map(d, 3); }
  // floats vsb_detect writes per frame: 1+nbits logits, or 1+nbits maps of P x P for a pixel-wise model
  size_t detect_out_per_frame() const {
    if (!dec.pixelwise) return 1 + d.nbits;
    const size_t P = (size_t)dec.out_side(trunk_map());
    return (size_t)(1 + d.nbits) * P * P;
  }
  void check_pooled_head(const std::string& what) const {
    if (dec.pixelwise) throw Error(what + ": per-pixel maps of a streamed video are not implemented (use vsb_detect / vsb_detect_host)", kErrUnsupported);
  }

  void finalize(int dev) {
    check_unfinalized();
    int count = 0;
    if (cudaGetDeviceCount(&count) != cudaSuccess || count == 0) throw Error("no CUDA device: libvsb200 has no CPU fallback", kErrCuda);
    VSB_CUDA(cudaSetDevice(dev));
    cudaDeviceProp prop;
    VSB_CUDA(cudaGetDeviceProperties(&prop, dev));
    if (prop.major != 9 || prop.minor != 0) throw Error("libvsb200 is built for sm_90a only (found sm_" + std::to_string(prop.major) + std::to_string(prop.minor) + ")", kErrUnsupported);
    device = dev;
    num_sms = prop.multiProcessorCount;
    if (henc.on) henc.pack(ws, num_sms);
    else if (dvenc.on) dvenc.pack(ws, num_sms);
    else if (vae.on) vae.pack(ws, num_sms);
    else {
      if (other_embedder()) unet.check(d);   // neither a U-Net nor a HiDDeN / DVMark / VAE embedder: the U-Net's rules fail
      unet.pack(ws, num_sms);
    }
    if (hdec.on) hdec.pack(ws, num_sms);
    else if (dvdec.on) dvdec.pack(ws, num_sms);
    else {
      if (vit.on) vit.pack(ws, d.img_size);
      else cnx.pack(ws, d);
      dec.pack(ws, d.nbits);
    }
    ws.sd.clear();  // host copies no longer needed
    finalized = true;
  }

  // Plan cache: one activation arena per distinct batch size, at most `max_plans` per kind (VSB_MAX_PLANS, default 8): a service that sees
  // many different clip / tail lengths would otherwise accumulate up to 64 arenas of up to 2.3 GB each (a temporal U-Net's embed plan
  // holds one more buffer, its time-stacked operand: B * S^2 * temporal_stack_width(z0) fp16 values, 512 MiB at 64 x 256^2 and
  // 4.5 GiB at 64 x 768^2; and its plans are also keyed by the group length; a DVMark detect plan holds three maps, 40 KiB * S^2 in all at
  // 64 frames, and at most 512 MiB of time-stacked operand: 3 GiB at 64 x 256^2, 23 GiB at 64 x 768^2; a DVMark embed plan about 1.9 KiB per
  // processing pixel with the same stack budget: 8.6 GB at 64 x 256^2, 33 GB at 64 x 512^2, DVMarkEnc::build).  The least recently used plan
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
  // embed plans are keyed by B + kPlanGroup * G: the plan of a temporal U-Net or a DVMark embedder also depends on its group length
  // G (0 for the others)
  static constexpr int kPlanGroup = 128;
  void build_embed_plan(Plan& pl, int key) {
    if (!henc.on && !dvenc.on && !vae.on) { unet.build(pl, key % kPlanGroup, key / kPlanGroup); return; }
    const int S = d.img_size, B = key % kPlanGroup;
    pl.x_res = pl.pool.alloc_n<float>((size_t)B * 3 * S * S);
    pl.tap("x_res", pl.x_res, 0, B, 3, S, S, S);
    if (dvenc.on) dvenc.build(pl, B, key / kPlanGroup, S, keep_inputs);
    else if (vae.on) vae.build(pl, B, S, keep_inputs);
    else henc.build(pl, B, S, keep_inputs);
  }
  // detect plans are keyed by B + kPlanGroup * G: a DVMark extractor's plan also depends on its group length G (0 for the others)
  void build_detect_plan(Plan& pl, int key) {
    const int B = key % kPlanGroup, G = key / kPlanGroup;
    const int S = d.img_size;
    pl.x_res = pl.pool.alloc_n<float>((size_t)B * 3 * S * S);
    pl.tap("x_res", pl.x_res, 0, B, 3, S, S, S);
    pl.logits = pl.pool.alloc_n<float>((size_t)B * (1 + d.nbits));
    if (hdec.on) { hdec.build(pl, B, S, keep_inputs); return; }
    if (dvdec.on) { dvdec.build(pl, B, G, S); return; }
    const FeatureMap m = vit.on ? vit.build(pl, B, S, num_sms, keep_inputs) : cnx.build(pl, B, d, num_sms, keep_inputs);
    dec.build(pl, B, m, vit.on ? "vit." : "cnx.", d.nbits, num_sms);
  }
  Plan* get_embed_plan(int B, int G) { return get_plan(embed_plans, B + kPlanGroup * G, &Model::build_embed_plan); }
  // a temporal U-Net or a DVMark embedder convolves across a group of chunk_keys key frames (one reference embedder call), which
  // must fit one sub-batch
  int temporal_group(int chunk_keys) const {
    if (!frame_mixing_embedder()) return 0;
    const std::string what = dvenc.on ? "DVMark embedder" : "temporal U-Net";
    VSB_CHECK(chunk_keys >= 1, "a " + what + " needs chunk_keys >= 1 (key frames per embedder call)");
    if (chunk_keys > kMaxBatch)
      throw Error(what + ": a group of " + std::to_string(chunk_keys) + " frames convolved together (one video chunk, or the "
                  "whole batch in image mode) does not fit one " + std::to_string(kMaxBatch) + "-frame sub-batch; at most " +
                  std::to_string(kMaxBatch) + " are implemented", kErrUnsupported);
    return chunk_keys;
  }
  Plan* get_detect_plan(int B, int G) { return get_plan(detect_plans, B + kPlanGroup * G, &Model::build_detect_plan); }
  // a DVMark extractor convolves across a group of `group` frames (one reference detector call); the other extractors take frames
  // one at a time and ignore it
  int detect_group(int group) const { return dvdec.on ? DVMark::group(group, kMaxBatch) : 0; }


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

  // ---- embed / detect of HOST buffers: one copy in, the device entry point on stream 0, one copy out
  void embed_host(const float* imgs_h, const uint8_t* msgs_h, int n_msgs, float* imgs_w_h, float* preds_w_h, int F, int H, int W, int step,
                  int video_mode, int chunk_keys, float scaling_i, float scaling_w, int flags) {
    check_ready();
    const size_t n = (size_t)F * 3 * H * W;
    const bool use_jnd = !(flags & VSB_FLAG_NO_ATTENUATION) && d.jnd_in_ch != 0;
    const size_t np = (size_t)F * (use_jnd ? std::max(delta_ch(), d.jnd_out_ch) : delta_ch()) * H * W;
    float* imgs = (float*)stage(0, n * sizeof(float));
    float* out = (float*)stage(1, n * sizeof(float));
    float* pw = preds_w_h ? (float*)stage(2, np * sizeof(float)) : nullptr;
    uint8_t* msgs = (uint8_t*)stage(3, (size_t)n_msgs * d.nbits + 256);
    cudaStream_t st = 0;
    VSB_CUDA(cudaMemcpyAsync(imgs, imgs_h, n * sizeof(float), cudaMemcpyHostToDevice, st));
    VSB_CUDA(cudaMemcpyAsync(msgs, msgs_h, (size_t)n_msgs * d.nbits, cudaMemcpyHostToDevice, st));
    embed(imgs, msgs, n_msgs, out, pw, F, H, W, step, video_mode, chunk_keys, scaling_i, scaling_w, flags, st);
    VSB_CUDA(cudaMemcpyAsync(imgs_w_h, out, n * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (pw) VSB_CUDA(cudaMemcpyAsync(preds_w_h, pw, np * sizeof(float), cudaMemcpyDeviceToHost, st));
    VSB_CUDA(cudaStreamSynchronize(st));
  }
  void detect_host(const float* imgs_h, float* logits_h, int F, int H, int W, int group, int flags) {
    check_ready();
    const size_t n = (size_t)F * 3 * H * W;
    const size_t nl = (size_t)F * detect_out_per_frame();
    float* imgs = (float*)stage(0, n * sizeof(float));
    float* lg = (float*)stage(2, nl * sizeof(float));
    cudaStream_t st = 0;
    VSB_CUDA(cudaMemcpyAsync(imgs, imgs_h, n * sizeof(float), cudaMemcpyHostToDevice, st));
    detect(imgs, lg, F, H, W, group, flags, st);
    VSB_CUDA(cudaMemcpyAsync(logits_h, lg, nl * sizeof(float), cudaMemcpyDeviceToHost, st));
    VSB_CUDA(cudaStreamSynchronize(st));
  }

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
  // of one reference chunk are mixed, and for a temporal U-Net or a DVMark embedder, which convolve across them, whole chunks
  int key_unit(int step, int video_mode, int chunk_keys) const {
    if (frame_mixing_embedder()) return step * temporal_group(chunk_keys);
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
        detect(out + (size_t)g0 * fpx, lg + (size_t)g0 * NO, gn, H, W, 0, flags & VSB_FLAG_RESIZE_BITS, s_cmp);
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
      if (do_detect) detect(det_in, lg + (size_t)f0 * NO, n, H, W, 0, flags & VSB_FLAG_RESIZE_BITS, s_cmp);
      VSB_CUDA(cudaGetLastError());
      VSB_CUDA(cudaEventRecord(ev_cmp[k], s_cmp));
      VSB_CUDA(cudaStreamWaitEvent(s_out, ev_cmp[k], 0));
      if (do_embed) VSB_CUDA(cudaMemcpyAsync(out_h + (size_t)f0 * fpx, out8 + (size_t)f0 * fpx, (size_t)n * fpx, cudaMemcpyDeviceToHost, s_out));
      if (do_detect) VSB_CUDA(cudaMemcpyAsync(logits_h + (size_t)f0 * NO, lg + (size_t)f0 * NO, (size_t)n * NO * sizeof(float), cudaMemcpyDeviceToHost, s_out));
    }
    VSB_CUDA(cudaStreamSynchronize(s_out));
  }

  // U-Net on `n` processing-size RGB frames (contiguous [n,3,S,S]), in temporal groups of G (0: a 2-D U-Net) -> plan->delta
  Plan* run_unet(const float* x, const uint8_t* msgs, int msg_stride, int n, int G, cudaStream_t st) {
    Plan* pl = get_embed_plan(n, G);
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
    const int G = temporal_group(B);   // the B frames are one embedder call
    for (int b0 = 0; b0 < B; b0 += kMaxBatch) {
      const int n = std::min(kMaxBatch, B - b0);
      Plan* pl = run_unet(x + (size_t)b0 * 3 * S * S, msgs + (n_msgs == 1 ? 0 : (size_t)b0 * d.nbits), n_msgs == 1 ? 0 : d.nbits, n, G, st);
      VSB_CUDA(cudaMemcpyAsync(delta + (size_t)b0 * delta_ch() * S * S, pl->delta, (size_t)n * delta_ch() * S * S * sizeof(float),
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
    // a temporal U-Net's sub-batches hold whole groups too: its 3x3x3 convs mix the key frames of one chunk
    const int G = temporal_group(chunk_keys);
    const int kbatch = (interp || G) ? (kMaxBatch / chunk_keys) * chunk_keys : kMaxBatch;
    const int bint = interp ? chunk_keys : 0;
    const int S = d.img_size;
    const bool same = (H == S && W == S);
    const ResampleMode rm = same ? ResampleMode() : resample_mode(flags);   // (the flags are read only when a resize happens)
    const bool use_jnd = !(flags & VSB_FLAG_NO_ATTENUATION) && d.jnd_in_ch != 0;
    // channels of hmaps * preds_w (broadcast): what `preds_w` holds and what the low-resolution path hands to the blend
    const int PC = use_jnd ? std::max(delta_ch(), d.jnd_out_ch) : delta_ch();
    const bool lowres = use_jnd && (flags & VSB_FLAG_LOWRES_ATTN);
    const long fstride = (long)3 * H * W;
    const int nkeys = (F + step - 1) / step;
    ResampleDev* up = same ? nullptr : get_resampler(S, S, H, W, rm);
    for (int k0 = 0; k0 < nkeys; k0 += kbatch) {
      const int nk = std::min(kbatch, nkeys - k0);
      const int f0 = k0 * step, f1 = std::min(F, (k0 + nk) * step);
      const int nf = f1 - f0;
      Plan* pl = get_embed_plan(nk, G);
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
      run_unet(x, msgs + (n_msgs == 1 ? 0 : (size_t)k0 * d.nbits), n_msgs == 1 ? 0 : d.nbits, nk, G, st);
      const float* delta = pl->delta;
      const int balt = (video_mode == VSB_VIDEO_ALTERNATE) ? 1 : 0;
      BlendParams bp;
      memset(&bp, 0, sizeof(bp));
      bp.imgs = imgs + (size_t)f0 * fstride; bp.imgs_w = imgs_w + (size_t)f0 * fstride;
      bp.preds_w = preds_w ? preds_w + (size_t)f0 * PC * H * W : nullptr;
      bp.F = nf; bp.H = H; bp.W = W; bp.PH = S; bp.PW = S; bp.CD = delta_ch();
      bp.jnd_in = d.jnd_in_ch ? d.jnd_in_ch : 1; bp.jnd_out = d.jnd_out_ch ? d.jnd_out_ch : 1;
      bp.clamp = (flags & VSB_FLAG_CLAMP) ? 1 : 0; bp.identity_resample = same ? 1 : 0;
      bp.scaling_i = scaling_i; bp.scaling_w = scaling_w;
      if (up) bp.tab = up->tab;
      if (lowres) {
        // per-frame attenuated delta at processing size: out[f] = hmap(frames_res[f]) * delta(keys of f); then a plain blend
        float* lowres_buf = (float*)stage(7, (size_t)nf * PC * S * S * sizeof(float));
        VSB_CHECK(nf <= 65535, "too many frames per key-frame batch");
        prof_scope("pw.jnd_lowres@" + std::to_string(nf), st, 1, [&] {
          launch_jnd_lowres(frames_res, delta, lowres_buf, nf, S, S, delta_ch(), step, balt, bint, bp.jnd_in, bp.jnd_out, st);
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

  // group: frames per DVMark detector call (the last group may be shorter); sub-batches then hold whole groups.  A group longer
  // than the call is the whole call, and a plan's group is at most its frames, so equal computations share one plan.
  void detect(const float* imgs, float* logits, int F, int H, int W, int group, int flags, cudaStream_t st) {
    check_ready();
    VSB_CHECK(F > 0 && H > 0 && W > 0, "bad detect shape");
    const int G = detect_group(std::min(group, F));
    const int batch = G ? (kMaxBatch / G) * G : kMaxBatch;
    const int S = d.img_size;
    const bool same = (H == S && W == S);
    const ResampleMode rm = same ? ResampleMode() : resample_mode(flags);
    const long fstride = (long)3 * H * W;
    const size_t NO = detect_out_per_frame();
    for (int f0 = 0; f0 < F; f0 += batch) {
      const int n = std::min(batch, F - f0);
      Plan* pl = get_detect_plan(n, std::min(G, n));
      const float* x = imgs + (size_t)f0 * fstride;
      if (!same) { resize_frames(x, fstride, n, H, W, pl->x_res, rm, st); x = pl->x_res; }
      pl->in_imgs = x;
      pl->out_maps = dec.pixelwise ? logits + (size_t)f0 * NO : nullptr;   // the maps are written in place, at this sub-batch's offset
      pl->run(st);
      last_plan = pl;
      if (!dec.pixelwise)
        VSB_CUDA(cudaMemcpyAsync(logits + (size_t)f0 * NO, pl->logits, (size_t)n * NO * sizeof(float), cudaMemcpyDeviceToDevice, st));
    }
  }
};

}  // namespace vsb
