// Host side of attention.cuh: grids and shared memory of the SAM-ViT extractor kernels.
#pragma once
#include <algorithm>
#include "attention.cuh"
#include "conv_gemm_host.cuh"

namespace vsb {

inline void launch_vit_patch_im2col(const float* imgs, int B, int S, __half* patches, int num_sms, cudaStream_t st) {
  const int G = S / kVitPatch;
  const long total = (long)B * G * G * 96;
  const int grid = (int)std::min<long>((total + 255) / 256, (long)num_sms * 32);
  vit_patch_im2col_kernel<<<grid, 256, 0, st>>>(imgs, B, S, G, patches);
  VSB_CUDA(cudaGetLastError());
}

inline void launch_vit_pos_add(float* x, long M, int P, int E, const float* table, int num_sms, cudaStream_t st) {
  const long total = M * (E / 4);
  const int grid = (int)std::min<long>((total + 255) / 256, (long)num_sms * 32);
  vit_pos_add_kernel<<<grid, 256, 0, st>>>(x, M, P, E, table);
  VSB_CUDA(cudaGetLastError());
}

// B frames of a G x G token grid, attention over n x n regions (n = G: global); head dim HD (128: no relative positions)
template <int HD = kAttnHd>
inline void launch_vit_attention(AttnParams p, int B, cudaStream_t st) {
  const dim3 grid((unsigned)(B * p.regions * p.heads), (unsigned)(p.n * p.n / kAttnTile));
  const bool rel = p.rel_h != nullptr;
  VSB_CHECK(!rel || p.n <= kAttnMaxRelSide, "attention: relative positions over regions wider than 32 tokens");
  const size_t smem = attn_smem_bytes(rel, HD);
  if constexpr (HD != kAttnHd) {
    VSB_CHECK(!rel, "attention: relative positions need head dim 64");
    smem_optin<vit_attention_kernel<false, HD>>(smem);
    vit_attention_kernel<false, HD><<<grid, 128, smem, st>>>(p);
  } else if (rel) {
    smem_optin<vit_attention_kernel<true>>(smem);
    vit_attention_kernel<true><<<grid, 128, smem, st>>>(p);
  } else {
    smem_optin<vit_attention_kernel<false>>(smem);
    vit_attention_kernel<false><<<grid, 128, smem, st>>>(p);
  }
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
