// K4 v3: depthwise 7x7 (pad 3, bias) + channels-last LayerNorm (eps 1e-6) -> fp16   (modules/convnext.py:30-31,42-45)
//
// Register-rolling walk down the rows, fed by a TMA ring:
//   * a block owns a band of NS*SX output columns of one image and walks R output rows; a thread owns one channel pair and a strip
//     of SX columns.  Its 49 weights (packed fp32 pairs) stay in registers; every input row is read ONCE (SX+6 64-bit shared loads)
//     and feeds the 7 output rows it overlaps: 7 x SX accumulators in a statically rotated register ring (slot = (row phase + j + 1)
//     mod 7), 49*SX FMA pairs per input row against SX+6 loads -- the tap loop is >90 % FMA-pipe instructions.
//   * one producer warp streams the input rows of the band into a shared-memory ring with cp.async.bulk.tensor (4-D fp32 map of the
//     NHWC residual stream, box = [channels, NS*SX+6 pixels, 1 row]): out-of-image columns are zero-filled by the TMA unit (the
//     conv padding costs nothing), rows above / below the image are skipped on both sides, and the copy of row i+k is in flight
//     while row i is consumed -- the strip kernels re-load a 7 x 14 window per 8 outputs straight from L1/L2 and stall on every
//     one of them.
//   * a finished output row is normalised in registers: the per-pixel sums over the channel pairs are reduced with a halving
//     butterfly over 16-lane segments, combined across the segments through a few floats of shared memory (one named barrier of the
//     compute warps per row, double-buffered partials), one-pass variance.
// Requires dense x / out (pixel pitch C), H % R == 0, W % (NS*SX) == 0, (NS * C/2) % 32 == 0, C <= 256 (one TMA box per row).
#pragma once
#include <type_traits>
#include "ptx.cuh"

namespace vsb {


__device__ __forceinline__ void dw_bar_sync(int nthreads) { asm volatile("bar.sync 3, %0;" ::"r"(nthreads) : "memory"); }

template <int C, int NS, int SX, int kDwRingSlots>
__global__ void __launch_bounds__(NS * C / 2 + 32, 1)
dwconv7_ln_ring_kernel(const __grid_constant__ CUtensorMap tmX, int B, int H, int W, const float* __restrict__ wdw /*[49][C]*/,
                       const float* __restrict__ bdw, const float* __restrict__ lnw, const float* __restrict__ lnb,
                       __half* __restrict__ out, int R) {
  constexpr int C2 = C / 2, KSEG = C2 / 16, NV = 2 * SX;      // 16-lane segments per strip; values per thread in the row reduction
  constexpr int BW = NS * SX + 6;                              // band width in pixels incl. the halo
  constexpr int SLOT = BW * C;                                 // floats per ring slot, layout [BW][C]
  constexpr int NCOMP = NS * C2;                               // compute threads
  static_assert(NCOMP % 32 == 0 && C2 % 16 == 0 && (SX == 2 || SX == 4) && C <= 256, "shape");
  extern __shared__ __align__(128) float dwr_smem[];
  float* ring = dwr_smem;                                                            // [kDwRingSlots][SLOT]
  float* part = ring + kDwRingSlots * SLOT;                                          // [2][NS][KSEG][NV]
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(part + 2 * NS * KSEG * NV);       // [slots] | empty [slots]
  uint64_t* empty_bar = full_bar + kDwRingSlots;

  const int cgroups = W / (NS * SX), rgroups = H / R;
  const int cg = blockIdx.x % cgroups;
  const int t = blockIdx.x / cgroups;
  const int rg = t % rgroups, b = t / rgroups;
  const int xb = cg * NS * SX, y0 = rg * R;
  const int nsteps = R + 6;                          // input rows y0 - 3 ... y0 + R + 2

  if (threadIdx.x == 0) {
    for (int s = 0; s < kDwRingSlots; ++s) { mbar_init(&full_bar[s], 1u); mbar_init(&empty_bar[s], (uint32_t)(NCOMP / 32)); }
    fence_barrier_init();
    tma_prefetch_desc(&tmX);
  }
  __syncthreads();
  pdl_launch_dependents();
  pdl_wait();

  if (threadIdx.x >= NCOMP) {
    // ------------------------------------------------------------------ producer warp
    if (threadIdx.x == NCOMP) {
      int q = 0;
      for (int i = 0; i < nsteps; ++i) {
        const int iy = y0 - 3 + i;
        if ((unsigned)iy >= (unsigned)H) continue;
        const int slot = q % kDwRingSlots;
        mbar_wait(&empty_bar[slot], (((uint32_t)(q / kDwRingSlots)) & 1u) ^ 1u);
        mbar_arrive_expect_tx(&full_bar[slot], (uint32_t)(SLOT * sizeof(float)));
        tma_load_4d(&tmX, &full_bar[slot], ring + (size_t)slot * SLOT, 0, xb - 3, iy, b);
        ++q;
      }
    }
    return;
  }

  // -------------------------------------------------------------------- compute threads
  const int s = threadIdx.x / C2, cp = threadIdx.x - s * C2, c = cp * 2;
  const int lane = threadIdx.x & 31, seg = cp >> 4;
  const int x0 = xb + s * SX;
  // this thread's pixels inside a slot: pixel (s*SX + u) of the band, channel c  ->  [pixel][C]
  const int soff = (s * SX) * C + c;

  float2 wt[49];
#pragma unroll
  for (int k = 0; k < 49; ++k) wt[k] = __ldg(reinterpret_cast<const float2*>(wdw + k * C + c));
  const float2 bias = __ldg(reinterpret_cast<const float2*>(bdw + c));
  const float2 lg = __ldg(reinterpret_cast<const float2*>(lnw + c)), lb = __ldg(reinterpret_cast<const float2*>(lnb + c));

  float2 acc[7][SX];
  float2 cur[SX + 6];
  float2 fin[SX];                                    // the output row that completed in the current step (emitted outside the step body)
  int q = 0;                                         // valid input rows consumed so far (ring sequence number)
  int emitted = 0;                                   // rows emitted so far -> partial-sum buffer parity

  // one step = one input row i (iy = y0 - 3 + i); PH = i mod 7 is a compile-time constant inside the 7-fold unrolled body so that
  // every accumulator index below is static.  Output row o = i + j - 6 (kernel row 6 - j) lives in slot (PH + j + 1) % 7.
  auto step = [&](auto ph_tag, int i) {
    constexpr int PH = decltype(ph_tag)::value;
    const int iy = y0 - 3 + i;
    const bool rowok = (unsigned)iy < (unsigned)H;
    if (rowok) {
      const int slot = q % kDwRingSlots;
      mbar_wait(&full_bar[slot], ((uint32_t)(q / kDwRingSlots)) & 1u);
      const float* rp = ring + (size_t)slot * SLOT + soff;
#pragma unroll
      for (int u = 0; u < SX + 6; ++u) cur[u] = *reinterpret_cast<const float2*>(rp + u * C);
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty_bar[slot]);  // the row now lives in this warp's registers
      ++q;
    }
    {   // j = 6: output row o = i starts here (kernel row 0): initialise its slot
      constexpr int SL = (PH + 7) % 7;
      if (rowok && i < R) {
#pragma unroll
        for (int p = 0; p < SX; ++p) acc[SL][p] = f2fma(cur[p], wt[0], bias);
#pragma unroll
        for (int k = 1; k < 7; ++k) {
          const float2 wk = wt[k];
#pragma unroll
          for (int p = 0; p < SX; ++p) acc[SL][p] = f2fma(cur[p + k], wk, acc[SL][p]);
        }
      } else {
#pragma unroll
        for (int p = 0; p < SX; ++p) acc[SL][p] = bias;
      }
    }
    if (rowok) {
      // output rows o = i + j - 6 (kernel row 6 - j), j = 0..5.  Tap index k is the OUTER loop: consecutive FFMA2 then belong to
      // different accumulators (6 x SX independent chains) instead of walking one 7-long dependent chain (ncu of the first version:
      // 29 % of the stall samples were fixed-latency "wait" between back-to-back dependent FFMA2 at < 2 warps per scheduler)
      if (i >= 6 && i < R) {                           // steady state: all six rows are live
#pragma unroll
        for (int k = 0; k < 7; ++k)
#pragma unroll
          for (int j = 0; j < 6; ++j) {
            const float2 wk = wt[(6 - j) * 7 + k];
#pragma unroll
            for (int p = 0; p < SX; ++p) acc[(PH + j + 1) % 7][p] = f2fma(cur[p + k], wk, acc[(PH + j + 1) % 7][p]);
          }
      } else {
#pragma unroll
        for (int j = 0; j < 6; ++j) {
          const int o = i + j - 6;
          if (o >= 0 && o < R) {
#pragma unroll
            for (int k = 0; k < 7; ++k) {
              const float2 wk = wt[(6 - j) * 7 + k];
#pragma unroll
              for (int p = 0; p < SX; ++p) acc[(PH + j + 1) % 7][p] = f2fma(cur[p + k], wk, acc[(PH + j + 1) % 7][p]);
            }
          }
        }
      }
    }
    if (i >= 6) {                                    // j = 0: output row i - 6 has now seen its last input row
      constexpr int SL = (PH + 1) % 7;
#pragma unroll
      for (int p = 0; p < SX; ++p) fin[p] = acc[SL][p];
    }
  };
  auto emit = [&](int o) {
    {
      float v[NV];
#pragma unroll
      for (int p = 0; p < SX; ++p) {
        const float2 a = fin[p];
        v[2 * p] = a.x + a.y;
        v[2 * p + 1] = fmaf(a.x, a.x, a.y * a.y);
      }
      // halving butterfly over the 16 lanes of the segment, then plain butterflies: lane l ends with value index
      // (bits of l from 8 downwards, one per halving) summed over the 16 lanes
      int idx;
      if (NV == 8) {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const float send = (lane & 8) ? v[k] : v[k + 4];
          const float keep = (lane & 8) ? v[k + 4] : v[k];
          v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const float send = (lane & 4) ? v[k] : v[k + 2];
          const float keep = (lane & 4) ? v[k + 2] : v[k];
          v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
        {
          const float send = (lane & 2) ? v[0] : v[1];
          const float keep = (lane & 2) ? v[1] : v[0];
          v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 2);
        }
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
        idx = ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
      } else {
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          const float send = (lane & 8) ? v[k] : v[k + 2];
          const float keep = (lane & 8) ? v[k + 2] : v[k];
          v[k] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
        }
        {
          const float send = (lane & 4) ? v[0] : v[1];
          const float keep = (lane & 4) ? v[1] : v[0];
          v[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
        }
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], 2);
        v[0] += __shfl_xor_sync(0xffffffffu, v[0], 1);
        idx = ((lane >> 3) & 1) * 2 + ((lane >> 2) & 1);
      }
      const int buf = emitted & 1;
      const bool writer = NV == 8 ? ((lane & 1) == 0) : ((lane & 3) == 0);
      if (writer) part[((buf * NS + s) * KSEG + seg) * NV + idx] = v[0];
      dw_bar_sync(NCOMP);     // one barrier per emitted row: the other buffer is only rewritten after the NEXT barrier
      float tot[NV];
#pragma unroll
      for (int k = 0; k < NV; ++k) tot[k] = 0.f;
#pragma unroll
      for (int g = 0; g < KSEG; ++g) {
        const float4* pp = reinterpret_cast<const float4*>(part + ((buf * NS + s) * KSEG + g) * NV);
#pragma unroll
        for (int k4 = 0; k4 < NV / 4; ++k4) {
          const float4 t4 = pp[k4];
          tot[4 * k4] += t4.x; tot[4 * k4 + 1] += t4.y; tot[4 * k4 + 2] += t4.z; tot[4 * k4 + 3] += t4.w;
        }
      }
      __half* dst = out + (((long)b * H + (y0 + o)) * W + x0) * C + c;
#pragma unroll
      for (int p = 0; p < SX; ++p) {
        const float mean = tot[2 * p] * (1.0f / (float)C);
        const float var = fmaxf(tot[2 * p + 1] * (1.0f / (float)C) - mean * mean, 0.f);
        const float rstd = rsqrtf(var + 1e-6f);
        const float sx = rstd * lg.x, sy = rstd * lg.y;
        const float2 a = fin[p];
        *reinterpret_cast<__half2*>(dst + p * C) = __floats2half2_rn(fmaf(a.x, sx, fmaf(-mean, sx, lb.x)), fmaf(a.y, sy, fmaf(-mean, sy, lb.y)));
      }
      ++emitted;
    }
  };
  // one call site for the emission (its ~300 instructions exist once; the 7 phase-specialised step bodies are loads + FFMA2 only: the
  // first version inlined the emission 7 times and lost 10 % of its issue slots to instruction-cache misses)
  int ph = 0;
  for (int i = 0; i < nsteps; ++i) {
    switch (ph) {
      case 0: step(std::integral_constant<int, 0>{}, i); break;
      case 1: step(std::integral_constant<int, 1>{}, i); break;
      case 2: step(std::integral_constant<int, 2>{}, i); break;
      case 3: step(std::integral_constant<int, 3>{}, i); break;
      case 4: step(std::integral_constant<int, 4>{}, i); break;
      case 5: step(std::integral_constant<int, 5>{}, i); break;
      default: step(std::integral_constant<int, 6>{}, i); break;
    }
    ph = ph == 6 ? 0 : ph + 1;
    if (i >= 6) emit(i - 6);
  }
}

template <int C, int NS, int SX, int kDwRingSlots> constexpr size_t dw_ring_smem() {
  return (size_t)(kDwRingSlots * (NS * SX + 6) * C + 2 * NS * (C / 32) * 2 * SX) * sizeof(float) + 2 * kDwRingSlots * sizeof(uint64_t) + 128;
}

}  // namespace vsb
