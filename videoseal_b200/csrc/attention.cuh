// SAM-ViT extractor kernels (modules/vit.py of the reference): the 16 x 16 patch im2col, the periodic position table, and the
// multi-head attention of one window or of the whole token grid with decomposed relative positions.
//
//   K7a vit_patch_im2col_kernel   [B,3,S,S] fp32 -> patches [B*G*G][768] fp16, K order (c, r, s) of the conv weight
//   K7b vit_pos_add_kernel        x[m][e] += table[m mod G*G][e]  (pos_embed + folded patch bias)
//   K7c vit_attention_kernel      softmax((q * scale) k^T + rel_h + rel_w) v for one (frame, region, head, 64 queries)
#pragma once
#include <cstdint>
#include <cuda_fp16.h>

namespace vsb {

constexpr int kVitPatch = 16;
constexpr int kAttnHd = 64;      // head dim of the SAM-ViT heads (the VAE's single head also runs at 128)
constexpr int kAttnTile = 64;    // queries per CTA and keys per online-softmax tile
constexpr int kAttnLds = 72;     // shared row pitch in halves: 36 words, so the 32-bit fragment loads of a warp hit 32 banks
constexpr int kAttnTp = 65;      // row pitch (floats) of the per-warp relative-position products
constexpr int kAttnMaxRelSide = (kAttnTile + 1) / 2;   // with rel-pos: 2n - 1 table rows staged in kAttnTile rows, so n <= 32

// K7a: one thread per 8 consecutive pixels of one patch row of one channel (16-byte fp16 store)
__global__ void __launch_bounds__(256) vit_patch_im2col_kernel(const float* __restrict__ imgs, int B, int S, int G, __half* __restrict__ patches) {
  const long total = (long)B * G * G * 96;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const int chunk = (int)(i % 96);
    const long m = i / 96;
    const int c = chunk >> 5, r = (chunk >> 1) & 15, s0 = (chunk & 1) * 8;
    const int px = (int)(m % G), py = (int)((m / G) % G);
    const long b = m / ((long)G * G);
    const float* src = imgs + ((b * 3 + c) * S + (long)py * kVitPatch + r) * S + (long)px * kVitPatch + s0;
    __align__(16) __half h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(__ldg(src + e));
    *reinterpret_cast<uint4*>(patches + m * 768 + chunk * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

// K7b: E a multiple of 4
__global__ void __launch_bounds__(256) vit_pos_add_kernel(float* __restrict__ x, long M, int P, int E, const float* __restrict__ table) {
  const int E4 = E >> 2;
  const long total = M * E4;
  for (long i = (long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long)gridDim.x * 256) {
    const long m = i / E4;
    const int e4 = (int)(i - m * E4);
    float4* px = reinterpret_cast<float4*>(x + m * E) + e4;
    const float4 t = __ldg(reinterpret_cast<const float4*>(table + (m % P) * E) + e4);
    float4 v = *px;
    v.x += t.x; v.y += t.y; v.z += t.z; v.w += t.w;
    *px = v;
  }
}

struct AttnParams {
  const __half* qkv;           // [B*G*G][3E] rows of the qkv GEMM, columns (3, heads, 64) (vit.py:337)
  __half* out;                 // [B*G*G][E]: head h writes its 64 columns h*64.. of each token's row
  const __half* rel_h;         // [64][64] fp16, rows >= 2n-1 zero (REL only)
  const __half* rel_w;
  int G;                       // token grid side (img_size / 16)
  int n;                       // region side: the window size, or G for global attention; n*n a multiple of 64
  int heads, E;
  int regions;                 // regions per frame, (G / n)^2
  float scale;                 // head_dim^-0.5
};

__device__ __forceinline__ void attn_mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t attn_pack(float lo, float hi) {
  const __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<const uint32_t*>(&h);
}
__device__ __forceinline__ uint32_t ld32(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }

// the q and k tiles have a row pitch of HD + 8 halves at head dim HD, so that the 32-bit fragment loads of a warp hit 32 banks
inline size_t attn_smem_bytes(bool rel, int hd = kAttnHd) {
  return (size_t)2 * kAttnTile * (hd + 8) * sizeof(__half) + (size_t)hd * kAttnLds * sizeof(__half) +
         (rel ? (size_t)2 * kAttnTile * kAttnLds * sizeof(__half) + (size_t)4 * 2 * 16 * kAttnTp * sizeof(float) : 0);
}

// K7c (vit.py:302-353 Attention.forward, :431-470 add_decomposed_rel_pos).  Grid (B * regions * heads, n*n / 64), 4 warps; warp w
// owns queries 16w..16w+15 of the CTA's 64.  Window partition / unpartition (vit.py:356-395) is index arithmetic on the token rows.
// Tensor cores (mma.m16n8k16, fp16 operands, fp32 accumulators) compute q k^T, and with REL q Rh^T / q Rw^T over the 2n-1 table
// rows with the UNSCALED q as in the reference; each score then gathers Th[q, qh-kh+n-1] + Tw[q, qw-kw+n-1].  Softmax in fp32,
// online over 64-key tiles; P is rounded to fp16 for P v and the rows are normalised at the end.  No atomics: a token's output
// depends only on its own region's rows.  HD: head dim, 64 (SAM-ViT; with or without REL) or 128 (the VAE's AttnBlock, no REL); the
// key loop does not bound the token count.
template <bool REL, int HD = kAttnHd>
__global__ void __launch_bounds__(128) vit_attention_kernel(const AttnParams p) {
  static_assert(HD == 64 || (HD == 128 && !REL), "attention: head dim 64, or 128 without relative positions");
  constexpr int LDQ = HD + 8, KS = HD / 16, ND = HD / 8, NDS = HD == 64 ? 3 : 4;   // q / k pitch, k-steps, 8-wide dim tiles (2^NDS)
  extern __shared__ __align__(16) unsigned char attn_smem[];
  __half* sQ = reinterpret_cast<__half*>(attn_smem);   // [64 queries][LDQ]
  __half* sK = sQ + kAttnTile * LDQ;                     // [64 keys][LDQ]
  __half* sVt = sK + kAttnTile * LDQ;                    // [HD dims][72 keys]: v transposed, the B operand of P v
  __half* sRh = sVt + HD * kAttnLds;                     // [64 table rows][72] (REL)
  __half* sRw = sRh + kAttnTile * kAttnLds;
  float* sT = reinterpret_cast<float*>(sRw + kAttnTile * kAttnLds);   // [warp][h/w][16][kAttnTp] (REL)
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n = p.n, T = n * n;
  int idx = blockIdx.x;
  const int head = idx % p.heads;
  idx /= p.heads;
  const int region = idx % p.regions;
  const long frame = idx / p.regions;
  const int per_row = p.G / n;
  const int ry0 = (region / per_row) * n, rx0 = (region % per_row) * n;
  const int q0 = blockIdx.y * kAttnTile;
  const int ld = 3 * p.E;
  auto row_of = [&](int tok) -> long { return (frame * p.G + ry0 + tok / n) * p.G + rx0 + tok % n; };
  const int qcol = head * HD, kcol = p.E + head * HD, vcol = 2 * p.E + head * HD;

  for (int i = threadIdx.x; i < kAttnTile * ND; i += 128) {
    const int r = i >> NDS, c = (i & (ND - 1)) * 8;
    *reinterpret_cast<uint4*>(sQ + r * LDQ + c) = *reinterpret_cast<const uint4*>(p.qkv + row_of(q0 + r) * ld + qcol + c);
    if (REL) {
      *reinterpret_cast<uint4*>(sRh + r * kAttnLds + c) = *reinterpret_cast<const uint4*>(p.rel_h + r * kAttnHd + c);
      *reinterpret_cast<uint4*>(sRw + r * kAttnLds + c) = *reinterpret_cast<const uint4*>(p.rel_w + r * kAttnHd + c);
    }
  }
  __syncthreads();
  uint32_t qa[KS][4];   // A fragments of the warp's 16 query rows over the KS k-steps of the head dim
  {
    const __half* qb = sQ + warp * 16 * LDQ;
#pragma unroll
    for (int kk = 0; kk < KS; ++kk) {
      qa[kk][0] = ld32(qb + g * LDQ + kk * 16 + 2 * t);
      qa[kk][1] = ld32(qb + (g + 8) * LDQ + kk * 16 + 2 * t);
      qa[kk][2] = ld32(qb + g * LDQ + kk * 16 + 8 + 2 * t);
      qa[kk][3] = ld32(qb + (g + 8) * LDQ + kk * 16 + 8 + 2 * t);
    }
  }
  const int qi0 = q0 + warp * 16 + g, qi1 = qi0 + 8;
  const int qh0 = qi0 / n, qw0 = qi0 % n, qh1 = qi1 / n, qw1 = qi1 % n;
  float* sTh = sT + warp * 2 * 16 * kAttnTp;
  float* sTw = sTh + 16 * kAttnTp;
  if (REL) {
    const int nt = (2 * n - 1 + 7) / 8;
    for (int j = 0; j < nt; ++j) {
      float ch[4] = {0.f, 0.f, 0.f, 0.f}, cw[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) {
        const __half* rh = sRh + (j * 8 + g) * kAttnLds + kk * 16 + 2 * t;
        const __half* rw = sRw + (j * 8 + g) * kAttnLds + kk * 16 + 2 * t;
        attn_mma(ch, qa[kk], ld32(rh), ld32(rh + 8));
        attn_mma(cw, qa[kk], ld32(rw), ld32(rw + 8));
      }
      const int c = j * 8 + 2 * t;
      sTh[g * kAttnTp + c] = ch[0]; sTh[g * kAttnTp + c + 1] = ch[1];
      sTh[(g + 8) * kAttnTp + c] = ch[2]; sTh[(g + 8) * kAttnTp + c + 1] = ch[3];
      sTw[g * kAttnTp + c] = cw[0]; sTw[g * kAttnTp + c + 1] = cw[1];
      sTw[(g + 8) * kAttnTp + c] = cw[2]; sTw[(g + 8) * kAttnTp + c + 1] = cw[3];
    }
    __syncwarp();
  }

  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;
  float o[ND][4];
#pragma unroll
  for (int j = 0; j < ND; ++j) o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f;
  for (int k0 = 0; k0 < T; k0 += kAttnTile) {
    __syncthreads();   // every warp is done with the previous key tile
    for (int i = threadIdx.x; i < kAttnTile * ND; i += 128) {
      const int r = i >> NDS, c = (i & (ND - 1)) * 8;
      const __half* src = p.qkv + row_of(k0 + r) * ld;
      *reinterpret_cast<uint4*>(sK + r * LDQ + c) = *reinterpret_cast<const uint4*>(src + kcol + c);
      __align__(16) __half v[8];
      *reinterpret_cast<uint4*>(v) = *reinterpret_cast<const uint4*>(src + vcol + c);
#pragma unroll
      for (int e = 0; e < 8; ++e) sVt[(c + e) * kAttnLds + r] = v[e];
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f;
      const __half* kb = sK + (j * 8 + g) * LDQ + 2 * t;
#pragma unroll
      for (int kk = 0; kk < KS; ++kk) attn_mma(s[j], qa[kk], ld32(kb + kk * 16), ld32(kb + kk * 16 + 8));
    }
    float mx0 = m0, mx1 = m1;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        // == (q * scale) k^T exactly when scale is a power of two (head dim 64); the VAE scales the product (vae.py AttnBlock)
        float v = s[j][e] * p.scale;
        if (REL) {
          const int key = k0 + j * 8 + 2 * t + (e & 1), kh = key / n, kw = key % n;
          const int r = e < 2 ? g : g + 8, qh = e < 2 ? qh0 : qh1, qw = e < 2 ? qw0 : qw1;
          v += sTh[r * kAttnTp + qh - kh + n - 1] + sTw[r * kAttnTp + qw - kw + n - 1];
        }
        s[j][e] = v;
      }
      mx0 = fmaxf(mx0, fmaxf(s[j][0], s[j][1]));
      mx1 = fmaxf(mx1, fmaxf(s[j][2], s[j][3]));
    }
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 1));
    mx0 = fmaxf(mx0, __shfl_xor_sync(0xffffffffu, mx0, 2));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 1));
    mx1 = fmaxf(mx1, __shfl_xor_sync(0xffffffffu, mx1, 2));
    const float a0 = expf(m0 - mx0), a1 = expf(m1 - mx1);   // 0 on the first tile
    m0 = mx0; m1 = mx1;
    l0 *= a0; l1 *= a1;
#pragma unroll
    for (int j = 0; j < ND; ++j) { o[j][0] *= a0; o[j][1] *= a0; o[j][2] *= a1; o[j][3] *= a1; }
    uint32_t pa[4][4];   // P as the A operand of P v: the accumulator layout of two key n-tiles is one k-step's A fragment
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = expf(s[j][0] - m0), p1 = expf(s[j][1] - m0), p2 = expf(s[j][2] - m1), p3 = expf(s[j][3] - m1);
      l0 += p0 + p1; l1 += p2 + p3;
      pa[j >> 1][(j & 1) * 2 + 0] = attn_pack(p0, p1);
      pa[j >> 1][(j & 1) * 2 + 1] = attn_pack(p2, p3);
    }
#pragma unroll
    for (int jd = 0; jd < ND; ++jd) {
      const __half* vb = sVt + (jd * 8 + g) * kAttnLds + 2 * t;
#pragma unroll
      for (int kk = 0; kk < 4; ++kk) attn_mma(o[jd], pa[kk], ld32(vb + kk * 16), ld32(vb + kk * 16 + 8));
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1);
  l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = 1.0f / l0, i1 = 1.0f / l1;
  __half* out0 = p.out + row_of(qi0) * p.E + head * HD + 2 * t;
  __half* out1 = p.out + row_of(qi1) * p.E + head * HD + 2 * t;
#pragma unroll
  for (int jd = 0; jd < ND; ++jd) {
    *reinterpret_cast<__half2*>(out0 + jd * 8) = __floats2half2_rn(o[jd][0] * i0, o[jd][1] * i0);
    *reinterpret_cast<__half2*>(out1 + jd * 8) = __floats2half2_rn(o[jd][2] * i1, o[jd][3] * i1);
  }
}

}  // namespace vsb
