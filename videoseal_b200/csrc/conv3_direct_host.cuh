// Host side of conv3_direct.cuh: geometry, tensor map, shared-memory plan, launch.
#pragma once
#include <vector>
#include "conv3_direct.cuh"
#include "conv_gemm_host.cuh"

namespace vsb {

struct Conv3DirectOp {
  Conv3DirectParams p;
  int grid = 0;
  size_t smem = 0;
  Conv3DirectOp() { memset(&p, 0, sizeof(p)); }
};

// padded row pitch in positions: W + R - 1, plus one column for the 8-channel kernel (its second K core matrix reads the
// position after each tap), rounded up to 8
inline int conv3_direct_pitch(int W, int R, int C) { return (W + R - 1 + (C == 8 ? 1 : 0) + 7) / 8 * 8; }
// bytes of the resident weights: R*R taps of C channels, or for C = 8 R*ceil(R/2) virtual taps of 16 (direct8_weights)
inline size_t conv3_direct_wbytes(int C, int N, int R) {
  return C == 8 ? (size_t)N * R * ((R + 1) / 2) * 16 * 2 : (size_t)N * R * R * C * 2;
}
// channel counts with a kernel instantiation (launch_direct): plain C, N in {16, 32, 64} or 8 -> 8; stride-2 (space-to-depth,
// C = 4 x C_in) 16 -> 32 and 8 -> 8
inline bool conv3_direct_channels(int C, int N, bool s2d) {
  if (s2d) return (C == 64 && N == 32) || (C == 32 && N == 8);
  return ((C == 16 || C == 32 || C == 64) && (N == 16 || N == 32 || N == 64)) || (C == 8 && N == 8);
}
// ring rows that fit next to the resident weights for a W-wide map (0 = channel counts not supported)
inline int conv3_direct_ring_rows(int C, int N, int W, int R = 3, bool s2d = false) {
  if (!conv3_direct_channels(C, N, s2d)) return 0;
  const int rw = conv3_direct_pitch(W, R, C);
  const uint32_t w_pad = ((uint32_t)conv3_direct_wbytes(C, N, R) + 1023u) & ~1023u;
  const size_t budget = 227 * 1024 - 1024 /*alignment slack*/ - kD3HeaderBytes - w_pad;
  int rows = (int)(budget / ((size_t)C * 2 * rw)) - (128 / rw + 1);
  rows = std::min(rows, kD3MaxRing);
  rows = std::min(rows, (kD3TileBars - 16) * 128 / rw);   // tiles in flight must stay below the tile_done barrier ring
  return rows;
}
// Fewest ring rows that are safe.  The kD3EpiSets sets work on consecutive tiles at the same time, and a set waits for ring row k
// on (slot k % NR, parity of k / NR), which is only sound once row k - NR has landed; the producer refills a slot only after the
// tiles that read its previous row are done.  So the ring must hold every row that kD3EpiSets consecutive tiles read
// (ceil((kD3EpiSets*128 + R - 1) / rw) + R - 1) plus one; two more rows keep loads ahead of the MMAs.
inline int conv3_direct_min_rows(int W, int R = 3, int C = 16) {
  const int rw = conv3_direct_pitch(W, R, C);
  return (kD3EpiSets * 128 + R - 1 + rw - 1) / rw + R + 2;
}
// R x R conv C -> N over a dense W-wide map: a kernel instantiation exists and its ring fits
inline bool conv3_direct_ok(int C, int N, int W, int R = 3) {
  return W % 8 == 0 && conv3_direct_ring_rows(C, N, W, R) >= conv3_direct_min_rows(W, R, C);
}
// stride-2 conv Cin -> N through the space-to-depth ring (setup_down_s2d_direct) on an output map W wide
inline bool conv3_direct_s2d_ok(int Cin, int N, int W) {
  return W % 8 == 0 && conv3_direct_ring_rows(4 * Cin, N, W, 3, true) >= conv3_direct_min_rows(W, 3, 4 * Cin);
}

// x: dense NHWC fp16 [B,H,W,C]; wpk: weights in core-matrix layout (pack_direct_weights_kernel), N*9*C halves
inline void setup_conv3_direct(Conv3DirectOp& op, const __half* x, int B, int H, int W, int C, int N, const __half* wpk, int num_sms,
                               int R = 3, bool s2d = false) {
  Conv3DirectParams& p = op.p;
  VSB_CHECK(R == 3 || R == 1, "direct conv: 3x3 or 1x1 only");
  VSB_CHECK(conv3_direct_ring_rows(C, N, W, R, s2d) > 0, "direct conv3: unsupported channel counts");
  p.B = B; p.H = H; p.W = W; p.C = C; p.N = N; p.R = R;
  p.relu = 1;
  p.rw = conv3_direct_pitch(W, R, C);
  p.hp = H + R - 1;
  const long positions = (long)B * p.hp * p.rw;
  VSB_CHECK(positions + 3L * p.rw < (1L << 31) - 1024, "direct conv3: batch too large for 32-bit positions");
  p.n_tiles = (int)((positions + 127) / 128);
  p.mirror_rows = 128 / p.rw + 1;
  p.w_bytes = (uint32_t)conv3_direct_wbytes(C, N, R);
  const uint32_t w_pad = (p.w_bytes + 1023u) & ~1023u;
  const int rows = conv3_direct_ring_rows(C, N, W, R, s2d);
  VSB_CHECK(rows >= conv3_direct_min_rows(W, R, C), "direct conv3: shared-memory ring too small");
  p.ring_rows = rows;
  p.plane_stride = (uint32_t)((size_t)(rows + p.mirror_rows) * p.rw * 16);
  p.w_off = kD3HeaderBytes;
  p.ring_off = kD3HeaderBytes + w_pad;
  op.smem = 1024 + (size_t)p.ring_off + (size_t)(C / 8) * p.plane_stride;
  p.fd_rw = make_fastdiv(p.rw);
  p.fd_hp = make_fastdiv(p.hp);
  p.wpk = wpk;
  p.x = x;
  VSB_CHECK((reinterpret_cast<uintptr_t>(x) & 15) == 0, "direct conv3: input must be 16-byte aligned");
  op.grid = std::min(num_sms, p.n_tiles);
}

template <int N, int KS, int R, int MODE = 0>
inline void launch_direct_nkr(const Conv3DirectOp& op, cudaStream_t st) {
  smem_optin<conv3_direct_kernel<N, KS, R, MODE>>(227 * 1024);
  launch_pdl(conv3_direct_kernel<N, KS, R, MODE>, dim3(op.grid), dim3(kD3Threads), op.smem, st, op.p);
  VSB_CUDA(cudaGetLastError());
}
template <int N, int KS>
inline void launch_direct_nk(const Conv3DirectOp& op, cudaStream_t st) {
  if (op.p.R == 3) launch_direct_nkr<N, KS, 3>(op, st);
  else launch_direct_nkr<N, KS, 1>(op, st);
}
template <int N>
inline void launch_direct_n(const Conv3DirectOp& op, cudaStream_t st) {
  if (op.p.C == 16) launch_direct_nk<N, 1>(op, st);
  else if (op.p.C == 32) launch_direct_nk<N, 2>(op, st);
  else launch_direct_nk<N, 4>(op, st);
}

inline void launch_direct(const Conv3DirectOp& op, cudaStream_t st) {
  VSB_CHECK(op.smem <= 227 * 1024, "direct conv3: shared-memory plan too large");
  if (op.p.x2 != nullptr) {   // up-conv phase mode: 64 input channels (two sources), 4 phases x 16 output channels
    VSB_CHECK(op.p.N == 64 && op.p.C == 64 && op.p.R == 3, "up-phase direct conv: C = 64, N = 4 x 16 only");
    launch_direct_nkr<64, 4, 3, 1>(op, st);
    return;
  }
  if (op.p.s2d) {             // stride-2 conv through the space-to-depth view: C = 4 x C_in input channels
    VSB_CHECK(op.p.R == 3 && ((op.p.N == 32 && op.p.C == 64) || (op.p.N == 8 && op.p.C == 32)),
              "stride-2 direct conv: 16 -> 32 or 8 -> 8 channels only");
    if (op.p.N == 32) launch_direct_nkr<32, 4, 3, 2>(op, st);
    else launch_direct_nkr<8, 2, 3, 2>(op, st);
    return;
  }
  if (op.p.C == 8 || op.p.N == 8) {   // 8-channel layers: one input plane, m64n8 output
    VSB_CHECK(op.p.C == 8 && op.p.N == 8, "direct conv: 8-channel layers are 8 -> 8 only");
    if (op.p.R == 3) launch_direct_nkr<8, 0, 3>(op, st);
    else launch_direct_nkr<8, 0, 1>(op, st);
    return;
  }
  if (op.p.N == 16) launch_direct_n<16>(op, st);
  else if (op.p.N == 32) launch_direct_n<32>(op, st);
  else launch_direct_n<64>(op, st);
}

// UBlock up-conv (bilinear x2 -> reflect pad -> conv3x3 -> LN -> ReLU, modules/common.py:45-52 + unet.py:187-190) as ONE 3x3 conv
// on the LOW-resolution grid with 4 x 16 output columns (one group per output phase (oy&1, ox&1)) and replicate padding:
// away from the image border the bilinear weights depend only on the phase, so they fold into the conv weights
// (Weights::upconv_phase).  The outermost output rows/columns (reflect padding of the up-sampled map) do not follow the
// phase pattern and are recomputed exactly by up_border_fix_kernel afterwards.
inline void setup_up_phase_direct(Conv3DirectOp& op, const __half* x0, int C0, const __half* x1, int C1, int B, int H, int W,
                                  const __half* wpk, const float* ln_w, const float* ln_b, float eps, __half* out, int num_sms) {
  VSB_CHECK(C0 % 8 == 0 && C1 % 8 == 0 && C0 + C1 == 64, "up-phase direct conv: 64 input channels in two sources");
  setup_conv3_direct(op, x0, B, H, W, 64, 64, wpk, num_sms, 3);
  op.p.x2 = x1; op.p.planes0 = C0 / 8; op.p.replicate = 1;
  op.p.ln_w = ln_w; op.p.ln_b = ln_b; op.p.ln_eps = eps;
  op.p.out = out; op.p.relu = 0;
  VSB_CHECK((reinterpret_cast<uintptr_t>(x1) & 15) == 0, "direct conv3: input must be 16-byte aligned");
}

// DBlock.down (unet.py:75: 3x3, stride 2, pad 1, bias) on x [B,2H,2W,Cin] -> [B,H,W,N]: output (Y,X), tap r reads input row
// 2Y + r - 1 = row (Y-1, dy=1), (Y, dy=0), (Y, dy=1) of the space-to-depth view, i.e. a conv with offsets {-1, 0} only.
// wpk: weights re-indexed to [N][(ey,ex)][(dy,dx,c)] (Weights::down_s2d) in the direct layout.
inline void setup_down_s2d_direct(Conv3DirectOp& op, const __half* x, int Cin, int B, int H, int W, int N, const __half* wpk,
                                  const float* bias, __half* out, int num_sms) {
  setup_conv3_direct(op, x, B, H, W, 4 * Cin, N, wpk, num_sms, 3, /*s2d=*/true);
  op.p.s2d = 1; op.p.bias = bias; op.p.out = out; op.p.relu = 0;
}

// Host re-indexing for the 8-channel kernel (KS = 0): w [N][R][R][8] (K order r, s, c)  ->  [N][R*ceil(R/2)][16] virtual taps
// (r, t) whose channels 0-7 are tap (r, 2t) and 8-15 tap (r, 2t + 1), zero where 2t + 1 = R; then pack_direct_weights with C = 16
// and T = R*ceil(R/2).
inline std::vector<float> direct8_weights(const std::vector<float>& w, int N, int R) {
  const int H = (R + 1) / 2;
  std::vector<float> o((size_t)N * R * H * 16, 0.f);
  for (int n = 0; n < N; ++n)
    for (int r = 0; r < R; ++r)
      for (int s = 0; s < R; ++s)
        for (int c = 0; c < 8; ++c) o[(((size_t)n * R + r) * H + s / 2) * 16 + (s & 1) * 8 + c] = w[(((size_t)n * R + r) * R + s) * 8 + c];
  return o;
}
// stride-2 3x3 weights w [N][3][3][Ci] (K order r, s, c) -> the space-to-depth layout of setup_down_s2d_direct:
// K = (ey*3+ex)*4Ci + (dy*2+dx)*Ci + c with tap r -> (ey, dy) = (0,1), (1,0), (1,1)
inline std::vector<float> s2d_weights(const std::vector<float>& w, int N, int Ci) {
  static const int E[3] = {0, 1, 1}, D[3] = {1, 0, 1};
  const int Cs = 4 * Ci;
  std::vector<float> p((size_t)N * 9 * Cs, 0.f);
  for (int n = 0; n < N; ++n)
    for (int r = 0; r < 3; ++r)
      for (int s2 = 0; s2 < 3; ++s2)
        for (int c = 0; c < Ci; ++c)
          p[((size_t)n * 9 + (E[r] * 3 + E[s2])) * Cs + (D[r] * 2 + D[s2]) * Ci + c] = w[(((size_t)n * 3 + r) * 3 + s2) * Ci + c];
  return p;
}

// [N][9*C] fp16 on the device -> a new buffer in the direct layout
inline void pack_direct_weights(const __half* w, int N, int C, __half* out, cudaStream_t st, int T = 9) {
  pack_direct_weights_kernel<<<32, 256, 0, st>>>(w, N, C, T, out);
  VSB_CUDA(cudaGetLastError());
}

}  // namespace vsb
