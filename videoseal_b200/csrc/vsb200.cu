// libvsb200.so: the single translation unit behind include/vsb200.h.
//   nvcc -std=c++17 -O3 -lineinfo -gencode arch=compute_90a,code=sm_90a -shared -Xcompiler -fPIC vsb200.cu -o libvsb200.so
#include "model.cuh"
#include "quality_host.cuh"
#include "augment_host.cuh"

using namespace vsb;

struct vsb_model {
  Model impl;
  explicit vsb_model(const vsb_model_desc& d) : impl(d) {}
};

static thread_local std::string g_err;

static int fail(const std::exception& e, int code) {
  g_err = e.what();
  return code;
}

static_assert((int)kErrInvalid == (int)VSB_ERR_INVALID && (int)kErrUnsupported == (int)VSB_ERR_UNSUPPORTED && (int)kErrCuda == (int)VSB_ERR_CUDA &&
                  (int)kErrState == (int)VSB_ERR_STATE,
              "status codes of include/vsb200.h");

// Every C entry point that touches the GPU runs on the model's device and restores the caller's current device afterwards (the
// library must not change process-wide state under PyTorch), and holds the model's mutex: plans, scratch buffers and staging
// areas belong to the handle, so calls on ONE handle are serialised (use one handle per thread or stream for concurrency;
// include/vsb200.h "Threading").  The launch and profile counters (g_launches, g_profile) are process-wide, as the handle-less
// vsb_launch_count and vsb_profile_* entry points need.  The guard also records the device for smem_optin (t_device).
struct DeviceGuard {
  int prev = -1, prev_t = t_device;
  explicit DeviceGuard(int dev) {
    if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) { VSB_CUDA(cudaSetDevice(dev)); } else { prev = -1; }
    if (dev >= 0) t_device = dev;
  }
  ~DeviceGuard() { t_device = prev_t; if (prev >= 0) cudaSetDevice(prev); }
};
#define VSB_MODEL_SCOPE(m) std::lock_guard<std::recursive_mutex> _lk((m)->impl.mu); DeviceGuard _dg((m)->impl.device)

#define VSB_API_BEGIN try {
#define VSB_API_END                                                                       \
  }                                                                                       \
  catch (const vsb::Error& e) { return fail(e, e.code); }                                 \
  catch (const std::bad_alloc& e) { return fail(e, VSB_ERR_CUDA); }                       \
  catch (const std::exception& e) { return fail(e, VSB_ERR_INVALID); }

extern "C" {

const char* vsb_last_error(void) { return g_err.c_str(); }
int vsb_version(void) { return 100; }

int vsb_model_create(const vsb_model_desc* desc, vsb_model** out) {
  VSB_API_BEGIN
  VSB_CHECK(desc != nullptr && out != nullptr, "null argument");
  *out = new vsb_model(*desc);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_tensor(vsb_model* m, const char* name, const float* data, const int64_t* shape, int32_t ndim) {
  VSB_API_BEGIN
  VSB_CHECK(m && name && data && (shape || ndim == 0) && ndim >= 0 && ndim <= 5, "bad tensor argument");   // 5: Conv3d weights
  m->impl.set_tensor(name, data, shape, ndim);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_pixel_decoder(vsb_model* m, int32_t n_stages, const int32_t* factors, int32_t pixelwise) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr && (factors != nullptr || n_stages == 0), "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_pixel_decoder(n_stages, factors, pixelwise);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_unet_temporal(vsb_model* m, int32_t on) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_unet_temporal(on);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_vit_extractor(vsb_model* m, const vsb_vit_desc* vit) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr && vit != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_vit_extractor(*vit);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_hidden_embedder(vsb_model* m, const vsb_hidden_desc* h) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr && h != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_hidden_embedder(*h);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_hidden_extractor(vsb_model* m, const vsb_hidden_desc* h) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr && h != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_hidden_extractor(*h);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_dvmark_embedder(vsb_model* m, int32_t nbits) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_dvmark_embedder(nbits);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_vae_embedder(vsb_model* m, const vsb_vae_desc* vae) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr && vae != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_vae_embedder(*vae);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_set_dvmark_extractor(vsb_model* m, int32_t nbits) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr, "null argument");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  m->impl.set_dvmark_extractor(nbits);
  return VSB_OK;
  VSB_API_END
}

int vsb_model_finalize(vsb_model* m, int32_t device) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr, "null model");
  std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
  DeviceGuard dg(device);
  m->impl.finalize(device);
  return VSB_OK;
  VSB_API_END
}

void vsb_model_destroy(vsb_model* m) {
  if (m == nullptr) return;
  try { DeviceGuard dg(m->impl.device); delete m; } catch (...) {}
}

int vsb_embed(vsb_model* m, const float* imgs, const uint8_t* msgs, int32_t n_msgs, float* imgs_w, float* preds_w, int32_t F, int32_t H,
              int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys, float scaling_i, float scaling_w, int32_t flags,
              void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs && msgs && imgs_w, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.embed(imgs, msgs, n_msgs, imgs_w, preds_w, F, H, W, step, video_mode, chunk_keys, scaling_i, scaling_w, flags,
                (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int vsb_embedder_forward(vsb_model* m, const float* x, const uint8_t* msgs, int32_t n_msgs, float* delta, int32_t B, void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(m && x && msgs && delta && B > 0, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.embedder_forward(x, msgs, n_msgs, delta, B, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int vsb_detect(vsb_model* m, const float* imgs, float* logits, int32_t F, int32_t H, int32_t W, int32_t flags, void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs && logits, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.detect(imgs, logits, F, H, W, F, flags, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int vsb_detect_grouped(vsb_model* m, const float* imgs, float* logits, int32_t F, int32_t H, int32_t W, int32_t group, int32_t flags,
                       void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs && logits, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.detect(imgs, logits, F, H, W, group, flags, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int vsb_jnd_heatmaps(vsb_model* m, const float* imgs, float* hmaps, int32_t F, int32_t H, int32_t W, void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs && hmaps, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.jnd_heatmaps(imgs, hmaps, F, H, W, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int vsb_embed_host(vsb_model* m, const float* imgs_h, const uint8_t* msgs_h, int32_t n_msgs, float* imgs_w_h, float* preds_w_h, int32_t F,
                   int32_t H, int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys, float scaling_i, float scaling_w,
                   int32_t flags) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs_h && msgs_h && imgs_w_h, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.embed_host(imgs_h, msgs_h, n_msgs, imgs_w_h, preds_w_h, F, H, W, step, video_mode, chunk_keys, scaling_i, scaling_w, flags);
  return VSB_OK;
  VSB_API_END
}

int vsb_detect_host(vsb_model* m, const float* imgs_h, float* logits_h, int32_t F, int32_t H, int32_t W, int32_t flags) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs_h && logits_h, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.detect_host(imgs_h, logits_h, F, H, W, F, flags);
  return VSB_OK;
  VSB_API_END
}

int vsb_embed_detect_host(vsb_model* m, const float* imgs_h, const uint8_t* msgs_h, int32_t n_msgs, float* imgs_w_h, float* logits_h,
                          int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys, float scaling_i,
                          float scaling_w, int32_t flags) {
  VSB_API_BEGIN
  VSB_CHECK(m && imgs_h && msgs_h && imgs_w_h && logits_h, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.check_pooled_head("vsb_embed_detect_host");
  m->impl.check_frame_independent_detect("vsb_embed_detect_host");
  m->impl.embed_detect_host(imgs_h, msgs_h, n_msgs, imgs_w_h, logits_h, F, H, W, step, video_mode, chunk_keys, scaling_i, scaling_w,
                            flags);
  return VSB_OK;
  VSB_API_END
}

int vsb_frames_host_u8(vsb_model* m, const uint8_t* frames_h, const uint8_t* msgs_h, int32_t n_msgs, uint8_t* frames_w_h, float* logits_h,
                       int32_t F, int32_t H, int32_t W, int32_t step, int32_t video_mode, int32_t chunk_keys, float scaling_i,
                       float scaling_w, int32_t flags) {
  VSB_API_BEGIN
  VSB_CHECK(m && frames_h && (frames_w_h || logits_h) && (msgs_h || !frames_w_h), "null argument");
  VSB_MODEL_SCOPE(m);
  VSB_CHECK(F > 0 && H > 0 && W > 0 && step >= 1, "bad shape");
  if (logits_h) m->impl.check_pooled_head("vsb_frames_host_u8 with logits");
  if (logits_h) m->impl.check_frame_independent_detect("vsb_frames_host_u8 with logits");
  m->impl.frames_host_u8(frames_h, msgs_h, n_msgs, frames_w_h, logits_h, F, H, W, step, video_mode, chunk_keys, scaling_i, scaling_w,
                         flags);
  return VSB_OK;
  VSB_API_END
}

int64_t vsb_launch_count(int32_t reset) {
  const int64_t v = g_launches;
  if (reset) g_launches = 0;
  return v;
}

int64_t vsb_debug_get_tensor(vsb_model* m, const char* name, float* host_out, int64_t capacity, int64_t* shape4) {
  try {
    VSB_CHECK(m && name && shape4, "null argument");
    VSB_MODEL_SCOPE(m);   // before the plan is read: another thread may evict it from the cache
    VSB_CHECK(m->impl.last_plan != nullptr, "no plan has run yet");
    return m->impl.last_plan->read_tap(name, host_out, capacity, shape4);
  } catch (const std::exception& e) { return fail(e, -1); }
}

int vsb_debug_keep_inputs(vsb_model* m, int32_t on) {
  VSB_API_BEGIN
  VSB_CHECK(m != nullptr, "null argument");
  VSB_MODEL_SCOPE(m);
  m->impl.set_keep_inputs(on != 0);
  return VSB_OK;
  VSB_API_END
}

int64_t vsb_debug_plan_gemms(vsb_model* m, char* buf, int64_t capacity) {
  try {
    VSB_CHECK(m != nullptr, "null argument");
    std::lock_guard<std::recursive_mutex> lk(m->impl.mu);   // host state only: no device switch
    VSB_CHECK(m->impl.last_plan != nullptr, "no plan has run yet");
    std::string out;
    for (const std::string& line : m->impl.last_plan->gemms) out += line + "\n";
    if (buf && capacity > (int64_t)out.size()) memcpy(buf, out.c_str(), out.size() + 1);
    return (int64_t)out.size() + 1;
  } catch (const std::exception& e) { return fail(e, -1); }
}

int32_t vsb_debug_last_dispatch(vsb_model* m, int32_t* out, int32_t capacity) {
  try {
    VSB_CHECK(m && out, "null argument");
    VSB_CHECK(capacity >= 10, "dispatch buffer too small");
    std::lock_guard<std::recursive_mutex> lk(m->impl.mu);
    std::copy(m->impl.last_resize, m->impl.last_resize + 5, out);
    std::copy(m->impl.last_blend, m->impl.last_blend + 5, out + 5);
    return 10;
  } catch (const std::exception& e) { return fail(e, -1); }
}

int vsb_debug_conv(const vsb_conv_test* t, void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(t != nullptr, "null argument");
  static int num_sms = 0;
  if (num_sms == 0) {
    int dev = 0;
    VSB_CUDA(cudaGetDevice(&dev));
    VSB_CUDA(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
  }
  if (t->loader == 5) {
    // direct 3x3 conv (conv3_direct.cuh): weights arrive as [N][9*C0] and are re-packed here.  Stride 2 (3x3, pad 1) runs the
    // space-to-depth mode of the model's down convs; 8-channel inputs and stride 2 re-index the weights on the host first.
    const bool s2 = t->stride == 2;
    VSB_CHECK(((t->R == 3 && t->S == 3 && t->pad == 1) || (t->R == 1 && t->S == 1 && t->pad == 0 && !s2)) && (t->stride == 1 || s2) &&
              t->C1 == 0, "direct conv: 3x3 pad 1 or 1x1, stride 1; 3x3 pad 1 stride 2");
    VSB_CHECK(!s2 || (t->IH % 2 == 0 && t->IW % 2 == 0), "direct conv: stride 2 needs an even input map");
    // (scratch buffers, never freed: test-only path; the small pack kernel runs on every call)
    static __half* wpk = nullptr;
    static __half* wtmp = nullptr;
    if (wpk == nullptr) VSB_CUDA(cudaMalloc(&wpk, (size_t)64 * 9 * 64 * sizeof(__half)));
    const int T = t->R * t->S;
    if (s2 || t->C0 == 8) {
      VSB_CHECK((size_t)t->N * 9 * (s2 ? 4 * t->C0 : 16) <= (size_t)64 * 9 * 64, "direct conv: weights too large for the test path");
      if (wtmp == nullptr) VSB_CUDA(cudaMalloc(&wtmp, (size_t)64 * 9 * 64 * sizeof(__half)));
      std::vector<__half> hw((size_t)t->N * T * t->C0);
      VSB_CUDA(cudaMemcpy(hw.data(), t->weights, hw.size() * sizeof(__half), cudaMemcpyDeviceToHost));
      std::vector<float> w(hw.size());
      for (size_t i = 0; i < hw.size(); ++i) w[i] = __half2float(hw[i]);
      const std::vector<__half> vh = to_half(s2 ? s2d_weights(w, t->N, t->C0) : direct8_weights(w, t->N, t->R));
      VSB_CUDA(cudaMemcpy(wtmp, vh.data(), vh.size() * sizeof(__half), cudaMemcpyHostToDevice));
      pack_direct_weights(wtmp, t->N, s2 ? 4 * t->C0 : 16, wpk, (cudaStream_t)stream, s2 ? 9 : t->R * ((t->R + 1) / 2));
    } else {
      pack_direct_weights((const __half*)t->weights, t->N, t->C0, wpk, (cudaStream_t)stream, T);
    }
    Conv3DirectOp dop;
    if (s2) setup_down_s2d_direct(dop, (const __half*)t->src0, t->C0, t->B, t->IH / 2, t->IW / 2, t->N, wpk, t->bias, (__half*)t->out16, num_sms);
    else setup_conv3_direct(dop, (const __half*)t->src0, t->B, t->IH, t->IW, t->C0, t->N, wpk, num_sms, t->R);
    dop.p.relu = t->act == ACT_RELU ? 1 : 0;
    dop.p.bias = t->bias; dop.p.resid = (const __half*)t->resid16; dop.p.out = (__half*)t->out16;
    dop.p.outc_w = t->outc_w; dop.p.outc_b = t->outc_b; dop.p.n_out = t->n_out; dop.p.delta = t->delta; dop.p.outc_tanh = 1;
    launch_direct(dop, (cudaStream_t)stream);
    g_launches += 1;
    return VSB_OK;
  }
  ConvGemmOp op;
  const int Ct = t->C0 + t->C1;
  int K = t->R * t->S * Ct;
  if (t->loader == LD_HALO_CONV3) K = halo_kpad(t->C0, t->C1);  // weights in halo layout
  int OH, OW;
  const int ld0 = t->ld0 ? t->ld0 : t->C0, ld_out = t->ld_out ? t->ld_out : t->N;
  if (t->loader == LD_TMA) {
    OH = t->IH; OW = t->IW;
    if (t->IH == 1 && t->R == 1) setup_tma_gemm(op, (const __half*)t->src0, (long)t->B * t->IW, t->C0, ld0);
    else setup_tma_conv(op, (const __half*)t->src0, t->B, t->IH, t->IW, t->C0, ld0, t->R, t->S, t->pad);
  } else if (t->loader == LD_GATHER_CONV) {
    OH = (t->IH + 2 * t->pad - t->R) / t->stride + 1;
    OW = (t->IW + 2 * t->pad - t->S) / t->stride + 1;
    setup_gather_conv(op, LD_GATHER_CONV, (const __half*)t->src0, t->C0, ld0, (const __half*)t->src1, t->C1, t->C1, t->B, t->IH, t->IW, OH, OW,
                      t->R, t->S, t->stride, t->pad, t->pad_mode);
  } else {
    VSB_CHECK(t->loader == LD_HALO_CONV3, "bad loader");
    OH = t->IH; OW = t->IW;
    setup_halo_conv3(op, (const __half*)t->src0, t->B, t->IH, t->IW, t->C0, t->C0);
  }
  ConvGemmParams& p = op.p;
  p.epi = t->epi; p.act = t->act; p.bias = t->bias;
  p.resid16 = (const __half*)t->resid16; p.ld_res16 = t->N;
  p.resid32 = t->resid32; p.ld_res32 = ld_out;
  p.out16 = (__half*)t->out16; p.ld_out16 = ld_out;
  p.out32 = t->out32; p.ld_out32 = ld_out;
  p.ln_w = t->ln_w; p.ln_b = t->ln_b; p.ln_eps = 1e-6f;
  p.outc_w = t->outc_w; p.outc_b = t->outc_b; p.n_out = t->n_out; p.delta = t->delta; p.hw = OH * OW; p.outc_tanh = 1;
  VSB_CHECK(t->grn_part == 0 || (t->grn_stats != nullptr && t->rows_per_sample > 0 && t->rows_per_sample % 32 == 0),
            "GRN partial rows need rows_per_sample a multiple of 32");
  p.grn_stats = t->grn_stats; p.grn_part = t->grn_part;
  if (t->rows_per_sample) p.rows_per_sample = t->rows_per_sample;
  if (t->w_samples > 1) op.w_samples = t->w_samples;
  VSB_CHECK(t->kernel >= kKernelAuto && t->kernel <= kKernelLongK, "bad kernel selector");
  VSB_CHECK(t->longk_block_n == 0 || t->longk_block_n == 128 || t->longk_block_n == kLongWideN, "bad long-K block_n");
  finalize_op(op, (const __half*)t->weights, t->N, K, t->ldw ? t->ldw : K, num_sms, t->block_n, t->kernel, t->longk_block_n);
  if (t->kernel_ran) *t->kernel_ran = op.longk ? kKernelLongK : kKernel128;
  launch(op, (cudaStream_t)stream);
  g_launches += 1;
  return VSB_OK;
  VSB_API_END
}

int vsb_debug_resample_table(int32_t in, int32_t out, int32_t antialias, int32_t* start, int32_t* cnt, float* weights, int64_t capacity) {
  return vsb_debug_resample_table2(in, out, VSB_RESIZE_BILINEAR, 0, antialias, start, cnt, weights, capacity);
}

int vsb_debug_resample_table2(int32_t in, int32_t out, int32_t mode, int32_t align_corners, int32_t antialias, int32_t* start, int32_t* cnt,
                              float* weights, int64_t capacity) {
  try {
    VSB_CHECK(in > 0 && out > 0 && start && cnt && weights, "bad argument");
    VSB_CHECK(mode >= VSB_RESIZE_BILINEAR && mode <= VSB_RESIZE_AREA && (align_corners | antialias) >= 0 && (align_corners | antialias) <= 1,
              "bad resize mode");
    const ResampleMode m = resample_mode(VSB_FLAG_RESIZE_MODE(mode) | (align_corners ? VSB_FLAG_RESIZE_ALIGN_CORNERS : 0) |
                                         (antialias ? 0 : VSB_FLAG_RESIZE_NO_AA));
    const ResampleHost t = make_resample(in, out, m);
    check_table(t, in);
    VSB_CHECK(capacity >= (int64_t)out * t.maxt, "weights buffer too small");
    for (int i = 0; i < out; ++i) { start[i] = t.start[i]; cnt[i] = t.cnt[i]; }
    for (size_t i = 0; i < t.w.size(); ++i) weights[i] = t.w[i];
    return t.maxt;
  } catch (const std::exception& e) { return fail(e, -1); }
}

int64_t vsb_quality_workspace_bytes(int32_t B, int32_t C, int32_t H, int32_t W, int32_t multiscale) {
  try {
    return (int64_t)quality_layout(B, C, H, W, multiscale != 0).bytes;
  } catch (const vsb::Error& e) { return fail(e, e.code); } catch (const std::exception& e) { return fail(e, VSB_ERR_INVALID); }
}

// device of a CUDA allocation; VSB_ERR_INVALID for host memory
static int device_of(const void* p, const char* what, const char* who = "vsb_ssim") {
  cudaPointerAttributes a;
  const cudaError_t e = cudaPointerGetAttributes(&a, p);
  if (e != cudaSuccess) {
    cudaGetLastError();
    throw Error(std::string(who) + ": cannot query " + what + ": " + cudaGetErrorString(e), kErrCuda);
  }
  if (a.type != cudaMemoryTypeDevice && a.type != cudaMemoryTypeManaged) throw Error(std::string(who) + ": " + what + " is not CUDA device memory");
  return a.device;
}

static void require_sm90(int dev) {
  int major = 0, minor = 0;
  VSB_CUDA(cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev));
  VSB_CUDA(cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev));
  if (major != 9 || minor != 0) throw Error("libvsb200 is built for sm_90a only (found sm_" + std::to_string(major) + std::to_string(minor) + ")", kErrUnsupported);
}

int vsb_ssim(const float* x, const float* y, int32_t B, int32_t C, int32_t H, int32_t W, float data_range, float* ssim_out,
             float* msssim_out, void* workspace, int64_t workspace_bytes, void* stream) {
  VSB_API_BEGIN
  // every rule that needs no device first, so that they hold (and are testable) without a GPU
  VSB_CHECK(x && y && workspace, "vsb_ssim: null argument");
  VSB_CHECK(ssim_out || msssim_out, "vsb_ssim: ssim_out and msssim_out are both NULL");
  VSB_CHECK(std::isfinite(data_range) && data_range > 0.f, "vsb_ssim: data_range must be positive and finite");
  VSB_CHECK(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "vsb_ssim: workspace must be 16-byte aligned");
  const QualityLayout L = quality_layout(B, C, H, W, msssim_out != nullptr);
  VSB_CHECK(workspace_bytes >= (int64_t)L.bytes, "vsb_ssim: workspace smaller than vsb_quality_workspace_bytes()");
  const int dev = device_of(x, "x");
  VSB_CHECK(device_of(y, "y") == dev && device_of(workspace, "workspace") == dev &&
                (!ssim_out || device_of(ssim_out, "ssim_out") == dev) && (!msssim_out || device_of(msssim_out, "msssim_out") == dev),
            "vsb_ssim: x, y, the outputs and the workspace must be on one device");
  DeviceGuard dg(dev);
  require_sm90(dev);
  quality_run(L, x, y, B, C, data_range, ssim_out, msssim_out, (char*)workspace, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

int64_t vsb_augment_workspace_bytes(int32_t op, int32_t B, int32_t H, int32_t W) {
  try {
    return (int64_t)aug_workspace_bytes(op, B, H, W);
  } catch (const vsb::Error& e) { return fail(e, e.code); } catch (const std::exception& e) { return fail(e, VSB_ERR_INVALID); }
}

int vsb_augment(int32_t op, const float* x, float* y, int32_t B, int32_t C, int32_t H, int32_t W, int32_t OH, int32_t OW, const float* params,
                int32_t n_params, const float* aux, void* workspace, int64_t workspace_bytes, void* stream) {
  VSB_API_BEGIN
  VSB_CHECK(x && y, "vsb_augment: null argument");
  aug_check(op, B, C, H, W, OH, OW, params, n_params, aux);
  const size_t need = aug_workspace_bytes(op, B, H, W);
  VSB_CHECK(need == 0 || (workspace && workspace_bytes >= (int64_t)need), "vsb_augment: workspace smaller than vsb_augment_workspace_bytes()");
  VSB_CHECK(reinterpret_cast<uintptr_t>(workspace) % 16 == 0, "vsb_augment: workspace must be 16-byte aligned");
  const char* who = "vsb_augment";
  const int dev = device_of(x, "x", who);
  VSB_CHECK(device_of(y, "y", who) == dev && (!aux || device_of(aux, "aux", who) == dev) && (need == 0 || device_of(workspace, "workspace", who) == dev),
            "vsb_augment: x, y, aux and the workspace must be on one device");
  DeviceGuard dg(dev);
  require_sm90(dev);
  aug_run(op, x, y, B, H, W, OH, OW, params, n_params, aux, (char*)workspace, (cudaStream_t)stream);
  return VSB_OK;
  VSB_API_END
}

}  // extern "C"

// ---- per-step profile (bench.py roofline leg): enable, run some steps, then read "name\ttotal_ms\tcount\n" lines
extern "C" int vsb_profile_enable(int32_t on) {
  g_profile.flush();
  if (on) g_profile.acc.clear();
  g_profile.enabled = on != 0;
  return VSB_OK;
}
extern "C" int64_t vsb_profile_read(char* buf, int64_t capacity) {
  g_profile.flush();
  std::string out;
  for (auto& kv : g_profile.acc) out += kv.first + "\t" + std::to_string(kv.second.first) + "\t" + std::to_string(kv.second.second) + "\n";
  if (buf && capacity > (int64_t)out.size()) memcpy(buf, out.c_str(), out.size() + 1);
  return (int64_t)out.size() + 1;
}
