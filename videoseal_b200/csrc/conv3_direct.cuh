// 3x3 stride-1 zero-padded convolution for the narrow, high-resolution layers of the U-Net (modules/unet.py:17-39, the
// ResnetBlock convs at 16@256^2, 32@128^2, 64@64^2): "direct" implicit GEMM, no im2col anywhere.
//
// Idea.  Number the zero-padded input of the whole batch as ONE linear sequence of positions with row pitch `rw`
// (rw >= W + 2, multiple of 8):   P = (b*(H+2) + yy)*rw + xx,  yy = y+1, xx = x+1.   Number the outputs on the same grid,
// Q = (b*(H+2) + y)*rw + x.  Then tap (r, s) of output Q reads input P = Q + r*rw + s: a pure shift, the same for every
// output.  Shared memory holds a ring of padded input rows, split in PLANES of 8 channels (16 bytes per position), which
// is exactly the wgmma no-swizzle K-major canonical layout: 8 consecutive positions x 16 B form one core matrix,
// SBO = 128 B to the next 8 positions, LBO = plane stride to the next 8 channels.  A tile of 128 consecutive outputs
// therefore needs, per tap and 16 input channels, two m64 wgmma whose A descriptors simply point at
// ring + (Q0 + 64h + r*rw + s)*16 B.  The input crosses L2->SM once (16-byte cp.async per position and plane, zero fill = the
// conv padding, also between images), nothing is copied inside shared memory, and the 2/(H+2) + (rw-W)/rw junk outputs
// (pad rows / pad columns) are computed and dropped in the epilogue.
//
// Roles: warps 0, 2 = row producers, warps 4.. = MMA + epilogue sets (one warpgroup each; a set owns every kD3EpiSets-th
// tile, issues its wgmma and runs its epilogue, so the sets overlap each other's MMAs and epilogues).  Weights (<= 72 KB)
// stay resident in shared memory in the same core-matrix layout.  Epilogue: + folded-BN bias, ReLU, + residual, fp16 NHWC store, optionally the
// fused 1x1 `outc` + tanh of the last block (unet.py:191-197).
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>
#include "ptx.cuh"

namespace vsb {

constexpr int kD3MaxRing = 32;    // row_full barriers (ring rows)
constexpr int kD3TileBars = 64;   // tile_done barrier ring
constexpr int kD3EpiSets = 3;
constexpr int kD3Threads = 128 + kD3EpiSets * 128;
constexpr int kD3XposeOff = 2048;     // per epilogue warp: [32 rows][kD3XposePitch] fp32 fragment -> row transpose buffer
constexpr int kD3XposePitch = 20;     // 16 columns + 4: conflict-free float4 row reads
constexpr int kD3HeaderBytes = kD3XposeOff + kD3EpiSets * 4 * 32 * kD3XposePitch * 4;

struct Conv3DirectParams {
  int B, H, W, C, N, R;     // R = 3 (3x3, zero pad 1) or 1 (1x1)
  int rw, hp;               // linear row pitch in positions (>= W + R - 1, multiple of 8); H + R - 1
  int n_tiles;              // ceil(B*hp*rw / 128)
  int ring_rows, mirror_rows;
  uint32_t plane_stride;    // bytes between 8-channel planes of the ring
  uint32_t w_off, ring_off; // offsets from the 1024-aligned dynamic smem base
  uint32_t w_bytes;
  FastDiv fd_rw, fd_hp;
  const __half* x;          // input, dense NHWC fp16
  const __half* wpk;        // weights in core-matrix layout (pack_direct_weights_kernel)
  const float* bias;
  const __half* resid; __half* out;
  const float* outc_w; const float* outc_b; float* delta; int n_out, outc_tanh;
  int relu;                 // 1: ReLU after the bias (before the residual)
  // up-conv phase mode (UP template flag): second source for the virtual channel concat [x | x2] (planes0 planes come
  // from x), replicate instead of zero padding, epilogue = per-phase LayerNorm + ReLU + pixel shuffle to [B,2H,2W,16]
  const __half* x2; int planes0; int replicate;
  const float* ln_w; const float* ln_b; float ln_eps;
  int s2d;                  // stride-2 mode (S2): x is [B,2H,2W,C/4]
};

struct D3Header {
  uint64_t row_full[kD3MaxRing];
  uint64_t tile_done[kD3TileBars];
  float bias[64];
  float ocw[3][64];
};
static_assert(sizeof(D3Header) <= kD3XposeOff, "direct conv header");

// [N][T*C] (k = tap*C + c, T = 9 or 1 taps) fp16  ->  [tap][C/16][k-half][N/8][8 rows][8 halves]
__global__ void pack_direct_weights_kernel(const __half* __restrict__ w, int N, int C, int T, __half* __restrict__ out) {
  const int total = N * T * C;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
    const int n = i / (T * C), k = i - n * T * C;
    const int tap = k / C, c = k - tap * C;
    const int kk = c >> 4, kh = (c >> 3) & 1, k8 = c & 7;
    const long o = ((((long)(tap * (C >> 4) + kk) * 2 + kh) * (N >> 3) + (n >> 3)) * 8 + (n & 7)) * 8 + k8;
    out[o] = w[i];
  }
}

// MODE 0: plain conv; MODE 1 ("UP"): phase-folded up-conv (two sources, replicate padding, LN + pixel-shuffle epilogue);
// MODE 2 ("S2"): stride-2 3x3 conv, pad 1, as a 2x2-tap conv over the space-to-depth view of the input (C = 4*C_in planes
// gathered by the producers straight from the [B,2H,2W,C_in] tensor; taps with an offset of +1 have no weights and are skipped).
// KS = C / 16 k16 steps per tap; KS = 0 is the 8-channel input (C = 8, one plane, MODE 0 only): a k16 MMA then covers two
// horizontally adjacent taps, and the weights are packed as (R * ceil(R/2)) virtual 16-channel taps (direct8_weights).
// N = 8 (m64n8k16) takes C = 8 in MODE 0 or C = 32 (4 x 8) in MODE 2.
template <int N, int KS, int R, int MODE>
__global__ void __launch_bounds__(kD3Threads, 1) conv3_direct_kernel(const Conv3DirectParams p) {
  constexpr bool UP = MODE == 1, S2 = MODE == 2;
  extern __shared__ uint8_t d3_smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(d3_smem_raw) + 1023) & ~(uintptr_t)1023);
  D3Header* hd = reinterpret_cast<D3Header*>(smem);
  uint8_t* wsm = smem + p.w_off;
  uint8_t* ring = smem + p.ring_off;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int NR = p.ring_rows, rw = p.rw;

  // this CTA's contiguous range of 128-output tiles and the padded input rows they read
  const int per = p.n_tiles / (int)gridDim.x, rem = p.n_tiles - per * (int)gridDim.x;
  const int t0 = (int)blockIdx.x * per + min((int)blockIdx.x, rem);
  const int nt = per + ((int)blockIdx.x < rem ? 1 : 0);
  const int t1 = t0 + nt;
  const int row_lo = p.fd_rw.div(128 * t0);
  const int row_hi = p.fd_rw.div(128 * t1 - 1 + (R - 1)) + (R - 1);   // last position read: 128*t1 - 1 + (R-1)*rw + (R-1)

  if (threadIdx.x == 0) {
    for (int i = 0; i < kD3MaxRing; ++i) mbar_init(&hd->row_full[i], 32);   // 32 cp.async arrivals (one producer warp per row)
    for (int i = 0; i < kD3TileBars; ++i) mbar_init(&hd->tile_done[i], 4);   // the 4 warps of the set that computed the tile
    fence_barrier_init();
  }
  {
    const uint4* src = reinterpret_cast<const uint4*>(p.wpk);
    uint4* dst = reinterpret_cast<uint4*>(wsm);
    for (int i = threadIdx.x; i < (int)(p.w_bytes >> 4); i += blockDim.x) dst[i] = __ldg(src + i);
    if (threadIdx.x < N) {
      hd->bias[threadIdx.x] = p.bias ? __ldg(p.bias + threadIdx.x) : 0.f;
      for (int o = 0; o < 3; ++o) hd->ocw[o][threadIdx.x] = (p.outc_w && o < p.n_out) ? __ldg(p.outc_w + o * N + threadIdx.x) : 0.f;
      if (UP && threadIdx.x < 16) { hd->ocw[0][threadIdx.x] = __ldg(p.ln_w + threadIdx.x); hd->ocw[1][threadIdx.x] = __ldg(p.ln_b + threadIdx.x); }
    }
  }
  fence_proxy_async_smem();   // weights were written through the generic proxy, wgmma reads them through the async proxy
  __syncthreads();
  // so far only weights / bias / LN parameters were read: the resident-weight copy overlaps the predecessor's tail
  pdl_launch_dependents();
  pdl_wait();

  if (warp == 0 || warp == 2) {
    // ================================================================= producers (warps 0 and 2): one padded input row per
    // ring slot, 16-byte cp.async per (position, plane) with zero fill for the padding.  (A TMA box with a 16-byte inner
    // extent does the same split, but every 16-byte line is its own request and the TMA unit's request window, not
    // bandwidth, then bounds the kernel.)
    const int pw = warp >> 1;
    const int planes = p.C >> 3, pshift = KS == 0 ? 0 : (planes == 2 ? 1 : (planes == 4 ? 2 : 3));
    int tiles_conf = 0;
    int slot = pw;   // NR >= 8 > 2 producers
    for (int k = pw; k <= row_hi - row_lo && nt > 0; k += 2, slot = slot + 2 >= NR ? slot + 2 - NR : slot + 2) {
      const int gi = row_lo + k;
      if (k >= NR) {
        // the slot still holds row gi - NR: wait for the last tile that reads it
        int need = (((gi - NR + 1) * rw - 1) >> 7);
        need = min(need, t1 - 1) - t0;
        while (tiles_conf <= need) {
          mbar_wait(&hd->tile_done[tiles_conf % kD3TileBars], (uint32_t)(tiles_conf / kD3TileBars) & 1u);
          ++tiles_conf;
        }
      }
      const int b = p.fd_hp.div(gi), yy = gi - b * p.hp;
      constexpr int PAD = (R - 1) / 2;
      const bool mir = slot < p.mirror_rows;
      uint8_t* base0 = ring + (size_t)slot * rw * 16;
      // each lane keeps one plane and walks the positions (32 / planes of them per warp pass): the per-copy address math is
      // one 32-bit multiply-add on a per-row lane pointer
      const int pl = lane & (planes - 1), xstep = 32 >> pshift;
      uint8_t* lane_dst = base0 + (size_t)pl * p.plane_stride;
      if (UP) {
        // two sources (virtual concat along channels), replicate padding: clamp the coordinates instead of zero-filling
        const bool rvalid = b < p.B;
        const int yc = min(max(yy - PAD, 0), p.H - 1);
        const int planes1 = planes - p.planes0;
        const bool first = pl < p.planes0;
        const int lstride = (first ? p.planes0 : planes1) * 8;
        const __half* lane_src = first ? p.x + ((long)b * p.H + yc) * p.W * (p.planes0 * 8) + pl * 8
                                       : p.x2 + ((long)b * p.H + yc) * p.W * (planes1 * 8) + (pl - p.planes0) * 8;
        for (int xx = lane >> pshift; xx < rw; xx += xstep) {
          const int xc = min(max(xx - PAD, 0), p.W - 1);
          const __half* src = rvalid ? lane_src + xc * lstride : p.x;
          uint8_t* dst = lane_dst + xx * 16;
          cp_async16_zfill(dst, src, rvalid ? 16u : 0u);
          if (mir) cp_async16_zfill(dst + (size_t)NR * rw * 16, src, rvalid ? 16u : 0u);
        }
      } else if (S2) {
        // plane = (dy, dx, 8-channel group) of the 2x2 input block under low-res position (Y, X) = (yy - 1, xx - 1)
        const int cin = p.C >> 2, pc = cin >> 3;
        const int sub = pl / pc, c8 = pl - sub * pc, dy = sub >> 1, dx = sub & 1;
        const bool rvalid = b < p.B && yy >= PAD && yy < p.H + PAD;
        const __half* lane_src = p.x + (((long)b * 2 * p.H + 2 * (yy - PAD) + dy) * (2 * p.W) + dx) * cin + c8 * 8 - PAD * 2 * cin;
        for (int xx = lane >> pshift; xx < rw; xx += xstep) {
          const bool ok = rvalid && (unsigned)(xx - PAD) < (unsigned)p.W;
          const __half* src = ok ? lane_src + xx * 2 * cin : p.x;
          uint8_t* dst = lane_dst + xx * 16;
          cp_async16_zfill(dst, src, ok ? 16u : 0u);
          if (mir) cp_async16_zfill(dst + (size_t)NR * rw * 16, src, ok ? 16u : 0u);
        }
      } else {
        const bool rvalid = b < p.B && yy >= PAD && yy < p.H + PAD;
        const __half* lane_src = p.x + ((long)b * p.H + (yy - PAD)) * p.W * p.C + pl * 8 - PAD * p.C;
        for (int xx = lane >> pshift; xx < rw; xx += xstep) {
          const bool ok = rvalid && (unsigned)(xx - PAD) < (unsigned)p.W;
          const __half* src = ok ? lane_src + xx * p.C : p.x;
          uint8_t* dst = lane_dst + xx * 16;
          cp_async16_zfill(dst, src, ok ? 16u : 0u);
          if (mir) cp_async16_zfill(dst + (size_t)NR * rw * 16, src, ok ? 16u : 0u);
        }
      }
      cp_async_mbar_arrive_noinc(&hd->row_full[slot]);
    }
  } else if (warp >= 4) {
    // ================================================================= MMA + epilogue sets.  Set e takes tiles e, e + kD3EpiSets, ...
    // Its 128 threads issue the tile's MMAs as two m64 wgmma (rows [64h, 64h + 64)); the thread's scalar work is strength-reduced:
    // positions advance incrementally and the 64-bit descriptors differ only in the 14-bit address field (one position = 16 B =
    // one unit of addr>>4).  Warp `quad` then holds tile rows 16*quad + (0..15) and 64 + 16*quad + (0..15) and gives lane l the
    // row `row` below: one output position per thread.
    const int e = (warp - 4) >> 2, quad = warp & 3;
    const int row = 16 * quad + (lane & 15) + 64 * (lane >> 4);
    float* xp = reinterpret_cast<float*>(smem + kD3XposeOff) + (size_t)(warp - 4) * 32 * kD3XposePitch;
    // no-swizzle K-major descriptors: LBO = byte distance between the two core matrices along K (next 8 channels), SBO = byte
    // distance between consecutive 8-row groups (next 8 positions / output channels)
    // (KS = 0, one 8-channel plane: LBO = 16 B, so the second core matrix along K is the NEXT position, i.e. tap (r, s + 1))
    const uint32_t a_lbo = KS == 0 ? 16u : p.plane_stride, a_sbo = 128u;
    const uint32_t b_lbo = (uint32_t)N * 16u, b_sbo = 128u;
    const uint32_t a_lo = (((a_lbo >> 4) & 0x3FFFu) << 16) + (smem_u32(ring) >> 4);
    const uint32_t b_lo = (((b_lbo >> 4) & 0x3FFFu) << 16) + (smem_u32(wsm) >> 4);
    const uint64_t a_hi = (uint64_t)((a_sbo >> 4) & 0x3FFFu) << 32;
    const uint64_t b_hi = (uint64_t)((b_sbo >> 4) & 0x3FFFu) << 32;
    const uint32_t kk_step = (2u * p.plane_stride) >> 4;
    const int rows_total = row_hi - row_lo;
    int x0 = 128 * t0 - row_lo * rw, slot0 = 0, g0 = 0;   // first output position of the tile: (ring slot, column), relative row
    int xn = x0 + 127 + (R - 1), gn = 0;                  // last input position of tap (0, R-1): row (relative), column
    while (xn >= rw) { xn -= rw; ++gn; }
    auto advance = [&](int tiles) {
      for (int k = 0; k < tiles; ++k) {
        x0 += 128;
        while (x0 >= rw) { x0 -= rw; ++g0; if (++slot0 == NR) slot0 = 0; }
        xn += 128;
        while (xn >= rw) { xn -= rw; ++gn; }
      }
    };
    advance(e);
    int rows_conf = 0;
    // Coordinates and the residual row of a tile depend on nothing the MMAs produce, so they are fetched early: for
    // N <= 32 one whole tile ahead (the global-load latency hides behind the previous tile's epilogue), for N = 64 (128
    // bytes per thread) just before the wait for the accumulator.
    constexpr bool kDeep = N <= 32;
    struct Where { bool valid; int b, y, x; long pix; };
    auto locate = [&](int i) {
      Where w;
      const int q = 128 * (t0 + i) + row;
      const int g = p.fd_rw.div(q);
      w.x = q - g * rw;
      w.b = p.fd_hp.div(g);
      w.y = g - w.b * p.hp;
      w.valid = i < nt && w.x < p.W && w.y < p.H && w.b < p.B;
      w.pix = w.valid ? ((long)w.b * p.H + w.y) * p.W + w.x : 0;
      return w;
    };
    auto fetch = [&](const Where& w, uint4 (&r)[N / 8]) {
      if (p.resid != nullptr && w.valid) {
        const uint4* rp = reinterpret_cast<const uint4*>(p.resid + w.pix * N);
#pragma unroll
        for (int j = 0; j < N / 8; ++j) r[j] = __ldg(rp + j);
      } else {
#pragma unroll
        for (int j = 0; j < N / 8; ++j) r[j] = make_uint4(0u, 0u, 0u, 0u);
      }
    };
    Where cur = locate(e), nxt = cur;
    uint4 rr[N / 8], rn[kDeep ? N / 8 : 1];
    if (kDeep) fetch(cur, rr);
    for (int i = e; i < nt; i += kD3EpiSets) {
      if constexpr (kDeep) {
        nxt = locate(i + kD3EpiSets);
        fetch(nxt, rn);
      } else {
        cur = locate(i);
        fetch(cur, rr);
      }
      const bool valid = cur.valid;
      const long pix = cur.pix;
      const int b = cur.b, y = cur.y, x = cur.x;
      // rows of the ring this tile reads: [g0, need].  Each is waited for by its own (slot, parity), so a set never waits on
      // a row that only other sets' tiles read (the producer may already have refilled that slot)
      {
        const int need = min(rows_total, gn + (R - 1));
        for (int k = max(rows_conf, g0); k <= need; ++k) mbar_wait(&hd->row_full[k % NR], (uint32_t)(k / NR) & 1u);
        rows_conf = max(rows_conf, need + 1);
      }
      fence_proxy_async_smem();   // rows were written by cp.async (generic proxy); wgmma reads through the async proxy
      float acc[2][N / 2];
      {
        int s1 = slot0 + 1; if (s1 >= NR) s1 -= NR;
        int s2 = s1 + 1; if (s2 >= NR) s2 -= NR;
        const uint32_t arow[3] = {a_lo + (uint32_t)(slot0 * rw + x0), a_lo + (uint32_t)(s1 * rw + x0), a_lo + (uint32_t)(s2 * rw + x0)};
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
        wgmma_fence();
        if constexpr (KS == 0) {
          // C = 8: per kernel row, taps (r, 0) + (r, 1) in one k16 MMA and (r, 2) + a zero-weight (r, 3) in the next (1x1: the
          // tap and a zero-weight neighbour).  The neighbour of a valid output is always in its own padded row (rw >= W + R).
#pragma unroll
          for (int h = 0; h < 2; ++h) {
#pragma unroll
            for (int r = 0; r < R; ++r) {
#pragma unroll
              for (int t = 0; t < (R + 1) / 2; ++t) {
                const uint64_t adesc = a_hi | (uint64_t)(arow[r] + (uint32_t)(64 * h + 2 * t));
                const uint64_t bdesc = b_hi | (uint64_t)(b_lo + (uint32_t)((r * ((R + 1) / 2) + t) * 2 * N));
                Wgmma<N>::mma(acc[h], adesc, bdesc, (r | t) != 0 ? 1u : 0u);
              }
            }
          }
        } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int r = 0; r < (S2 ? 2 : R); ++r) {
#pragma unroll
            for (int s = 0; s < (S2 ? 2 : R); ++s) {
#pragma unroll
              for (int kk = 0; kk < KS; ++kk) {
                const uint64_t adesc = a_hi | (uint64_t)(arow[r] + (uint32_t)(64 * h + s) + (uint32_t)kk * kk_step);
                const uint64_t bdesc = b_hi | (uint64_t)(b_lo + (uint32_t)(((r * R + s) * KS + kk) * 2 * N));
                Wgmma<N>::mma(acc[h], adesc, bdesc, (r | s | kk) != 0 ? 1u : 0u);
              }
            }
          }
        }
        }
        wgmma_commit();
        wgmma_wait<0>();
        wgmma_fence_regs(acc[0]);
        wgmma_fence_regs(acc[1]);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&hd->tile_done[i & (kD3TileBars - 1)]);   // this warp's reads of the ring are complete
      advance(kD3EpiSets);
      if constexpr (N == 8) {
        // m64n8 fragments -> one row (8 columns) per lane; + bias, ReLU, + residual, one 16-byte store, optional fused outc + tanh
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 0; j < 4; j += 2) {
            const int lr = (lane >> 2) + 8 * (j >> 1) + 16 * h, lc = 2 * (lane & 3);
            *reinterpret_cast<float2*>(xp + lr * kD3XposePitch + lc) = make_float2(acc[h][j], acc[h][j + 1]);
          }
        }
        __syncwarp();
        float f[8];
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          const float4 t = *reinterpret_cast<const float4*>(xp + lane * kD3XposePitch + 4 * u);
          const float4 bq = *reinterpret_cast<const float4*>(&hd->bias[4 * u]);
          f[4 * u + 0] = t.x + bq.x; f[4 * u + 1] = t.y + bq.y; f[4 * u + 2] = t.z + bq.z; f[4 * u + 3] = t.w + bq.w;
        }
        __syncwarp();
        if (valid) {
          if (p.relu) {
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
          }
          if (p.resid != nullptr) {
            __align__(16) __half hr[8];
            *reinterpret_cast<uint4*>(hr) = rr[0];
#pragma unroll
            for (int j = 0; j < 8; ++j) f[j] += __half2float(hr[j]);
          }
          if (p.out != nullptr) {
            __align__(16) __half2 h2[4];
#pragma unroll
            for (int j = 0; j < 4; ++j)
              h2[j] = __floats2half2_rn(fminf(fmaxf(f[2 * j], -65504.f), 65504.f), fminf(fmaxf(f[2 * j + 1], -65504.f), 65504.f));
            *reinterpret_cast<uint4*>(p.out + pix * 8) = *reinterpret_cast<const uint4*>(h2);
          }
          if (p.outc_w != nullptr) {
            const long hw = (long)p.H * p.W;
            const long o0 = (long)b * p.n_out * hw + (long)y * p.W + x;
#pragma unroll
            for (int o = 0; o < 3; ++o) {
              if (o < p.n_out) {
                float d = 0.f;
#pragma unroll
                for (int j = 0; j < 8; ++j) d += f[j] * hd->ocw[o][j];
                d += __ldg(p.outc_b + o);
                if (p.outc_tanh) d = tanhf(d);
                p.delta[o0 + o * hw] = d;
              }
            }
          }
        }
      } else {
      // fragments -> one row per lane, 16 columns at a time
      uint32_t v[N / 16][16];
#pragma unroll
      for (int c = 0; c < N / 16; ++c) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int j = 8 * c; j < 8 * c + 8; j += 2) {
            const int lr = (lane >> 2) + 8 * ((j >> 1) & 1) + 16 * h, lc = 8 * ((j >> 2) - 2 * c) + 2 * (lane & 3);
            *reinterpret_cast<float2*>(xp + lr * kD3XposePitch + lc) = make_float2(acc[h][j], acc[h][j + 1]);
          }
        }
        __syncwarp();
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float4 t = *reinterpret_cast<const float4*>(xp + lane * kD3XposePitch + 4 * u);
          v[c][4 * u] = __float_as_uint(t.x); v[c][4 * u + 1] = __float_as_uint(t.y);
          v[c][4 * u + 2] = __float_as_uint(t.z); v[c][4 * u + 3] = __float_as_uint(t.w);
        }
        __syncwarp();
      }
      if (UP) {
        // accumulator columns = (phase py*2+px, co): per phase a LayerNorm over the 16 channels (biased variance,
        // modules/common.py:150-155), ReLU, and the pixel shuffle to (2y+py, 2x+px)
        if (valid) {
#pragma unroll
          for (int c = 0; c < N / 16; ++c) {
            float f[16];
            float sum = 0.f;
#pragma unroll
            for (int j = 0; j < 16; ++j) { f[j] = __uint_as_float(v[c][j]); sum += f[j]; }
            const float mean = sum * (1.f / 16.f);
            float var = 0.f;
#pragma unroll
            for (int j = 0; j < 16; ++j) { const float dd = f[j] - mean; var += dd * dd; }
            const float rstd = 1.0f / sqrtf(var * (1.f / 16.f) + p.ln_eps);
            __align__(16) __half2 h2[8];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
              const float a = fmaxf((f[2 * j] - mean) * rstd * hd->ocw[0][2 * j] + hd->ocw[1][2 * j], 0.f);
              const float bb = fmaxf((f[2 * j + 1] - mean) * rstd * hd->ocw[0][2 * j + 1] + hd->ocw[1][2 * j + 1], 0.f);
              h2[j] = __floats2half2_rn(fminf(a, 65504.f), fminf(bb, 65504.f));
            }
            const long opix = ((long)b * 2 * p.H + 2 * y + (c >> 1)) * (2 * p.W) + 2 * x + (c & 1);
            uint4* op = reinterpret_cast<uint4*>(p.out + opix * 16);
            op[0] = reinterpret_cast<const uint4*>(h2)[0];
            op[1] = reinterpret_cast<const uint4*>(h2)[1];
          }
        }
      } else if (valid) {
      float dot0 = 0.f, dot1 = 0.f, dot2 = 0.f;
      const float lo = p.relu ? 0.f : -3.0e38f;
#pragma unroll
      for (int c = 0; c < N / 16; ++c) {
        float f[16];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const float4 bq = *reinterpret_cast<const float4*>(&hd->bias[c * 16 + 4 * u]);
          f[4 * u + 0] = fmaxf(__uint_as_float(v[c][4 * u + 0]) + bq.x, lo);
          f[4 * u + 1] = fmaxf(__uint_as_float(v[c][4 * u + 1]) + bq.y, lo);
          f[4 * u + 2] = fmaxf(__uint_as_float(v[c][4 * u + 2]) + bq.z, lo);
          f[4 * u + 3] = fmaxf(__uint_as_float(v[c][4 * u + 3]) + bq.w, lo);
        }
        if (p.resid != nullptr) {
          __align__(16) __half h[16];
          reinterpret_cast<uint4*>(h)[0] = rr[2 * c];
          reinterpret_cast<uint4*>(h)[1] = rr[2 * c + 1];
#pragma unroll
          for (int j = 0; j < 16; ++j) f[j] += __half2float(h[j]);
        }
        if (p.outc_w != nullptr) {
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            dot0 += f[j] * hd->ocw[0][c * 16 + j];
            dot1 += f[j] * hd->ocw[1][c * 16 + j];
            dot2 += f[j] * hd->ocw[2][c * 16 + j];
          }
        }
        if (p.out != nullptr) {
          __align__(16) __half2 h2[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const float a = fminf(fmaxf(f[2 * j], -65504.f), 65504.f), bb = fminf(fmaxf(f[2 * j + 1], -65504.f), 65504.f);
            h2[j] = __floats2half2_rn(a, bb);
          }
          uint4* op = reinterpret_cast<uint4*>(p.out + pix * N + c * 16);
          op[0] = reinterpret_cast<const uint4*>(h2)[0];
          op[1] = reinterpret_cast<const uint4*>(h2)[1];
        }
      }
      if (p.outc_w != nullptr) {
        const long hw = (long)p.H * p.W;
        const long o0 = (long)b * p.n_out * hw + (long)y * p.W + x;
        const float dd[3] = {dot0, dot1, dot2};
#pragma unroll
        for (int o = 0; o < 3; ++o) {
          if (o < p.n_out) {
            float d = dd[o] + __ldg(p.outc_b + o);
            if (p.outc_tanh) d = tanhf(d);
            p.delta[o0 + o * hw] = d;
          }
        }
      }
      }  // valid
      }  // N > 8
      if constexpr (kDeep) {
        cur = nxt;
#pragma unroll
        for (int j = 0; j < N / 8; ++j) rr[j] = rn[j];
      }
    }
  }

  __syncthreads();
}

}  // namespace vsb
