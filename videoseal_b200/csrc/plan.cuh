// Execution plans (device buffers + launch lists) and the process-wide launch counter and per-step profile every launch goes through.
#pragma once
#include <functional>
#include <map>
#include <string>
#include <utility>
#include <vector>

#include "conv_gemm_host.cuh"

namespace vsb {

static int64_t g_launches = 0;

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

// what a trunk's plan leaves for the decoder: fp16 NHWC [B, h, h, C] with pixel pitch ld
struct FeatureMap { const __half* x16; int h, C, ld; };

struct Plan {
  DevicePool pool;
  uint64_t last_use = 0;    // LRU stamp of the plan cache
  std::vector<Step> steps;
  std::map<std::string, DebugTensor> dbg;
  // host-only record of the variant finalize_op chose for each tensor-core step, one line per add_conv (vsb_debug_plan_gemms)
  std::vector<std::string> gemms;
  // embed plan I/O
  const float* in_imgs = nullptr;  // set per call (pointer slot read by the first kernel's lambda)
  long in_frame_stride = 0;
  const uint8_t* in_msgs = nullptr;
  int in_msg_stride = 0;
  float* x_res = nullptr;   // [B,3,S,S] resized RGB when the input is not at processing size
  float* delta = nullptr;   // [B,CD,S,S]
  float* logits = nullptr;  // [B,1+K]
  float* out_maps = nullptr;  // pixel-wise detect plans: the caller's [B,1+K,P,P] slice, set per call
  // appends a step that makes `launches` kernel launches (0: a copy or memset)
  void add(std::string name, std::function<void(cudaStream_t)> fn, int launches = 1) {
    steps.push_back(Step{std::move(fn), launches, std::move(name)});
  }
  // debug tap (vsb_debug_get_tensor): B x H x W rows of C values, `ld` apart
  void tap(const std::string& name, const void* p, int dtype, int64_t B, int64_t H, int64_t W, int64_t C, int64_t ld) {
    dbg[name] = DebugTensor{p, dtype, {B, H, W, C}, ld};
  }
  // debug tap `name` as fp32 rows without padding, synchronising the device first (host_out == nullptr: its size only)
  int64_t read_tap(const char* name, float* host_out, int64_t capacity, int64_t* shape4) const {
    auto it = dbg.find(name);
    if (it == dbg.end()) throw Error(std::string("unknown debug tensor: ") + name);
    const DebugTensor& t = it->second;
    const int64_t rows = t.shape[0] * t.shape[1] * t.shape[2], C = t.shape[3];
    for (int i = 0; i < 4; ++i) shape4[i] = t.shape[i];
    const int64_t n = rows * C;
    if (host_out == nullptr) return n;
    VSB_CHECK(capacity >= n, "debug buffer too small");
    VSB_CUDA(cudaDeviceSynchronize());
    if (t.dtype == 0) {
      VSB_CUDA(cudaMemcpy2D(host_out, C * sizeof(float), t.ptr, t.ld * sizeof(float), C * sizeof(float), rows, cudaMemcpyDeviceToHost));
    } else {
      std::vector<__half> h((size_t)n);
      VSB_CUDA(cudaMemcpy2D(h.data(), C * sizeof(__half), t.ptr, t.ld * sizeof(__half), C * sizeof(__half), rows, cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < n; ++i) host_out[i] = __half2float(h[i]);
    }
    return n;
  }
  void run(cudaStream_t st) {
    for (auto& s : steps) prof_scope(s.name, st, s.launches, [&] { s.fn(st); });
  }
};

}  // namespace vsb
