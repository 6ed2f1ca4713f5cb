"""Float64 references and forward error bounds for every kernel of the ConvNeXt-V2 detect plan (trunk + pooled head), judged one
kernel at a time.

Each step's inputs are the plan's debug taps (exact fp16 / fp32 values, or the caller's fp32 frames for the stem), so a step is
compared against float64 arithmetic on exactly what the kernel read.  The residual stream is updated in place by every block, so
the stage inputs come from the copies `vsb_debug_keep_inputs` adds: s{s}_ds (after the stem / down conv) and s{s}_in (before the
stage's last block); a, g and the scaled W2 hold the last block's values.  The references are built from `oracle/restate.py`
(`layernorm_cf`, the dwconv / LayerNorm / pwconv1 / GELU / GRN / pwconv2 order of `convnext_block`, the stem, down and head of
`convnext_extractor_forward`) on the state dict cast to float64.

Error bounds reuse tests/unet_kernels.py: u = 2^-11, u32 = 2^-24, K22 = 2^-22, the convolution-epilogue form
c u A + K 2^-22 A (+ 1/2 ulp_fp16 where the output is fp16), A = |W| * |x| + |b| (+ |resid|), and the first-order LayerNorm
propagation `ln_tol` (two-pass fp32 statistics, fallback to the output range when rho >= 1/4, which the GPU test forbids).

* Stem GEMM + LN (C0 <= 256).  The patches 2x - 1 are formed in fp32 (|err| <= 2^-25) and rounded to fp16, the weights are rounded
  to fp16: c = 2 (the u^2 cross term is far inside the K22 term), K = 64 + 8 (48 products, zero-padded to 64), plus 2^-25 sum|W|.
  The epilogue LayerNorm is ONE-pass: var = sum(x^2) / N - mean^2 in fp32.  On top of ln_tol, the cancellation of that difference:
  |D var| <= 2 ((C + 9) u32 (E[x^2] + 2 |mean| mean|x|) + u32 var), which moves the output by |g| |x_hat| |D var| / (2 sigma^2).
  fp32 output, no rounding term.
* `stem_ln_kernel` (C0 > 256): fp32 operands, c = 0, K = 48 + 8, the 2^-25 sum|W| term, two-pass LN.
* `ln_rows`: ln_tol with no input error, then 1/2 ulp_fp16.
* k2s2 down conv (gather loader): c = 1, K = 4 Cp + 8 with Cp the width padded to 8 (the gather runs K over the padded width against
  zero weight columns), fp32 output.
* dwconv7 + LN: a 49-tap fp32 FMA chain from the bias, c = 0, K = 49 + 8; ln_tol; 1/2 ulp_fp16.
* pwconv1 + GELU (stages that fold GRN into the weights, where g is the GELU output itself): e = u A + (C + 8) K22 A before the
  activation; |gelu'| <= 1.13; the packed `gelu_erf_p` differs from the exact GELU by <= 1.0e-6 (conv_gemm.cuh), ex2.approx adds
  <= 2^-22 relative to 0.5 |x| e <= 0.6e-6, so 4e-6 absolute plus 4 u32 |x| for the fp32 arithmetic; saturating fp16 output
  (1/2 ulp, nothing reaches 65504 here).
* GRN weight fold: the multiplier m = gamma Gx / (mean_k Gx + 1e-6) + 1 is taken in float64 from the fp16 g the tap holds.  The
  kernel sums the squares of the PRE-rounding fp32 values, so ||.|| moves by at most u ||g|| (+ sqrt(P) 2^-25 for subnormals), and
  the fp32 sum of P squares (per-warp butterflies, then P/32 partial rows or float atomics) by (P/32 + 16) u32 relative.  The mean
  over K adds (K + 8) u32, the reciprocal and products 3 u32, gamma Nx + 1 two roundings.  The reference w2s = W2 m uses the float64
  W2: the fp16 rounding of W2 adds 1/2 ulp_fp16(|W2|) (m + Dm) (absolute: small weights are fp16 subnormals), the fp32 product
  u32, then the fp16 rounding of w2s.
* pwconv1 + GELU + GRN apply (composite, stages that apply GRN to g in place): the pwconv1 bound d1 before the fp16 rounding; the
  kernel's norm is taken from values within d1 of the float64 h, so |Gx' - Gx| <= ||d1||_2 (triangle inequality) plus the summation
  term; then the multiplier as above, |fp16(h') m' - h m| <= d16 (m + Dm) + |h| Dm with d16 = d1 + 1/2 ulp, the fp32 product and
  the second fp16 rounding.
* pwconv2 + fp32 residual: c = 0 on the per-sample w2s (exact fp16 operands read from the tap), c = 1 on W2, K = 4C + 8; the host
  folds GRN beta into the bias in float64 and rounds it to fp32 once (u32 |bias|).  fp32 output.  At stage 3 the epilogue also
  writes stage3_16 = fp16(stage3): 1/2 ulp of the fp32 value.
* head 3x3 (reflect padding, no bias): c = 1, K = 9 Cp + 8, fp32 output.
* head pool: ln_tol on the fp32 head conv, `erff` GELU (1.13 d + 4 u32 (|v| + |gelu|)), the mean over P pixels in 8 per-warp rows
  ((P / 8 + 16) u32 of the mean of |gelu|), u32 for the division.
* head linear: a C-term fp32 dot product per lane stride + butterfly + bias, (C / 32 + 8) K22 A.

A ratio err / tol above 1 is a bug to find, never a reason to raise a constant.  Each step family also has mutations: a reference
with one deliberate defect that the GPU output must violate.  A mutation's footprint is None (anywhere), "last_frame", an int w:
the w outermost rows / columns of every map, or "tile_edge": the 3 outermost rows / columns of every 16 x 16 tile (the pixel
decoder's tiled gathers, tests/pd_kernels.py).
"""
from __future__ import annotations

import math
from typing import Callable, Dict, List

import torch
import torch.nn.functional as F

from oracle import restate
from tests.unet_kernels import K22, U16, U32, Check, half_ulp16, ln_tol

Q = "detector.convnext."
D = "detector.pixel_decoder."
GELU_D = 1.13            # max |gelu'|
GELU_ABS = 4e-6          # gelu_erf_p / erff against the exact GELU, with the ex2.approx term and margin
SUB = 2.0 ** -25         # fp32 rounding of 2x - 1, and half the fp16 subnormal spacing


def pitch(c: int) -> int:
    """pixel pitch of the trunk's NHWC buffers: the width rounded up to 8 channels"""
    return (c + 7) // 8 * 8


def r16(v: torch.Tensor) -> torch.Tensor:
    return v.half().to(v.dtype)


class Trunk:
    """float64 parameters of one ConvNeXt extractor with its pooled head; `blk(s)` is the key of stage s's last block"""

    def __init__(self, sd: Dict[str, torch.Tensor], spec: dict, device="cpu"):
        self.spec, self.cn = spec, spec["convnext"]
        self.sd = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items()
                   if v.is_floating_point() and (k.startswith(Q) or k.startswith(D))}
        self.dims, self.depths, self.stride = self.cn["dims"], self.cn["depths"], self.cn["stem_stride"]

    def blk(self, s: int, j: int = -1) -> str:
        return Q + f"stages.{s}.{self.depths[s] - 1 if j < 0 else j}."

    def w1(self, s):
        k = self.blk(s)
        return self.sd[k + "pwconv1.weight"][:, :, None, None], self.sd[k + "pwconv1.bias"]

    def w2(self, s):
        return self.sd[self.blk(s) + "pwconv2.weight"]

    def bias2(self, s, beta=True):
        """pwconv2's bias with GRN beta folded in, in float64 (ConvNeXt::pack then rounds it to fp32 once)"""
        k = self.blk(s)
        b = self.sd[k + "pwconv2.bias"]
        return b + self.w2(s) @ self.sd[k + "grn.beta"].reshape(-1) if beta else b

    def gamma(self, s):
        return self.sd[self.blk(s) + "grn.gamma"].reshape(-1)


# ---------------------------------------------------------------------------------------------------------------- helpers
def frame_border(h: int, w: int, width: int, device) -> torch.Tensor:
    m = torch.zeros(h, w, dtype=torch.bool, device=device)
    m[:width, :] = m[-width:, :] = m[:, :width] = m[:, -width:] = True
    return m


def tile_edge(h: int, w: int, device) -> torch.Tensor:
    """the 3 outermost rows / columns of every 16 x 16 output tile: the pixels whose bilinear corners (factor 2 or 4) reach into
    the one-pixel halo of the tile's low-resolution taps"""
    r, c = torch.arange(h, device=device) % 16, torch.arange(w, device=device) % 16
    er, ec = (r < 3) | (r >= 13), (c < 3) | (c >= 13)
    return er[:, None] | ec[None, :]


def outside(v: torch.Tensor, where) -> int:
    """violations of a mutation that lie off its footprint"""
    if where == "last_frame":
        return int(v[:-1].sum())
    if where == "tile_edge":
        return int((v & ~tile_edge(v.shape[-2], v.shape[-1], v.device)).sum())
    if isinstance(where, int):
        return int((v & ~frame_border(v.shape[-2], v.shape[-1], where, v.device)).sum())
    return 0


def shift1(x: torch.Tensor) -> torch.Tensor:
    """the map moved by one pixel down-right (zero filled): a sampling grid with the phase +1"""
    return F.pad(x, (0, 1, 0, 1))[:, :, 1:, 1:]


def drop_last_kblock(w: torch.Tensor, cp: int) -> torch.Tensor:
    """w [N, C, R, S] with the GEMM's last 64-wide K block zeroed.  K runs over (r, s, c) with c padded to cp (the gather loaders);
    cp = C for the TMA GEMMs, whose last block is partial when 64 does not divide C"""
    n, c, r, s = w.shape
    wp = F.pad(w.permute(0, 2, 3, 1), (0, cp - c)).reshape(n, r * s * cp).clone()
    k = wp.shape[1]
    wp[:, 64 * ((k - 1) // 64):] = 0
    return wp.reshape(n, r, s, cp)[..., :c].permute(0, 3, 1, 2)


def grn_mult(h: torch.Tensor, gamma: torch.Tensor):
    """GRN multiplier (common.py:166-169 with beta split off): Gx = ||h||_2 over the map per (frame, channel); [B, K]"""
    Gx = h.pow(2).sum((2, 3)).sqrt()
    mean = Gx.mean(1, keepdim=True)
    return gamma * Gx / (mean + 1e-6) + 1, Gx, mean


def grn_mult_err(Gx, mean, dG, gamma, P: int):
    """bound on |m' - m| given |Gx' - Gx| <= dG (see the module docstring)"""
    K = Gx.shape[1]
    dG = dG + (P / 32 + 16) * U32 * Gx
    dmean = dG.mean(1, keepdim=True) + (K + 8) * U32 * mean
    den = mean + 1e-6
    Nx = Gx / den
    dNx = dG / den + Gx * dmean / den ** 2 + 3 * U32 * Nx
    return gamma.abs() * dNx + 2 * U32 * (gamma.abs() * Nx + 1)


def conv1x1(x, w, b=None):
    return F.conv2d(x, w if w.dim() == 4 else w[:, :, None, None], b)


# ---------------------------------------------------------------------------------------------------------------- the plan
def plan_checks(tr: Trunk, tap: Callable[[str], torch.Tensor], has_tap: Callable[[str], bool], imgs: torch.Tensor,
                logits: torch.Tensor):
    """Yields one Check per kernel of the detect plan.  tap(name) -> float64 debug tap of the sub-batch whose frames are `imgs`
    [B, 3, S, S] (NCHW maps; s{s}_w2s [B, C, 4C]; head_pooled [B, C]); `logits` [B, 1 + K] are that sub-batch's outputs."""
    sd, dims = tr.sd, tr.dims
    # ---- stem
    x = 2 * imgs.to(torch.float64) - 1
    w, b = sd[Q + "downsample_layers.0.0.weight"], sd[Q + "downsample_layers.0.0.bias"]
    lw, lb = sd[Q + "downsample_layers.0.1.weight"], sd[Q + "downsample_layers.0.1.bias"]
    gemm = dims[0] <= 256
    stem = lambda xx: F.conv2d(xx, w, b, stride=tr.stride)
    pre = stem(x)
    A = F.conv2d(x.abs(), w.abs(), b.abs(), stride=tr.stride)
    e = ((2 * U16 + 72 * K22) if gemm else 56 * K22) * A + SUB * w.abs().sum((1, 2, 3))[None, :, None, None]
    ref, d, fb = ln_tol(pre, e, lw, lb)
    if gemm:   # one-pass statistics: the cancellation of E[x^2] - mean^2
        C = pre.shape[1]
        mu, var = pre.mean(1, keepdim=True), pre.var(1, unbiased=False, keepdim=True)
        dvar = 2 * ((C + 9) * U32 * (pre.pow(2).mean(1, keepdim=True) + 2 * mu.abs() * pre.abs().mean(1, keepdim=True)) + U32 * var)
        d = d + lw.abs()[None, :, None, None] * ((pre - mu) / torch.sqrt(var + 1e-6)).abs() * dvar / (2 * (var + 1e-6))
    ln = lambda p: restate.layernorm_cf(p, lw, lb)
    yield Check("stem GEMM + LN (one-pass)" if gemm else "stem_ln_kernel", tap("s0_ds"), ref, d,
                [("stem phase +1", ln(stem(shift1(x))), None), ("x instead of 2x - 1", ln(stem(imgs.to(torch.float64))), None)],
                fallback=fb)
    del x, pre, A, e, ref, d
    for s in range(4):
        C = dims[s]
        if s > 0:
            # ---- ln_rows: stage{s-1} -> s{s}_ln
            lw, lb = sd[Q + f"downsample_layers.{s}.0.weight"], sd[Q + f"downsample_layers.{s}.0.bias"]
            xs = tap(f"stage{s - 1}")
            ref, d, fb = ln_tol(xs, torch.zeros_like(xs), lw, lb)
            yield Check(f"s{s} ln_rows", tap(f"s{s}_ln"), ref, d + half_ulp16(ref.abs() + d),
                        [("LayerNorm affine dropped", restate.layernorm_cf(xs, torch.ones_like(lw), torch.zeros_like(lb)), None)],
                        fallback=fb)
            del xs, ref, d
            # ---- k2s2 down conv: s{s}_ln -> s{s}_ds
            xn = tap(f"s{s}_ln")
            w, b = sd[Q + f"downsample_layers.{s}.1.weight"], sd[Q + f"downsample_layers.{s}.1.bias"]
            ref = F.conv2d(xn, w, b, stride=2)
            A = F.conv2d(xn.abs(), w.abs(), b.abs(), stride=2)
            yield Check(f"s{s} down2x2s2", tap(f"s{s}_ds"), ref, (U16 + (4 * pitch(dims[s - 1]) + 8) * K22) * A,
                        [("k2s2 phase +1", F.conv2d(shift1(xn), w, b, stride=2), None),
                         ("last K block dropped", F.conv2d(xn, drop_last_kblock(w, pitch(dims[s - 1])), b, stride=2), None)])
            del xn, ref, A
        k = tr.blk(s)
        xin = tap(f"s{s}_in")
        # ---- dwconv7 + LN: s{s}_in -> s{s}_a
        dw, db, lw, lb = sd[k + "dwconv.weight"], sd[k + "dwconv.bias"], sd[k + "norm.weight"], sd[k + "norm.bias"]
        dwc = lambda xx, ww=dw: F.conv2d(xx, ww, db, padding=3, groups=C)
        pre = dwc(xin)
        e = 57 * K22 * F.conv2d(xin.abs(), dw.abs(), db.abs(), padding=3, groups=C)
        ref, d, fb = ln_tol(pre, e, lw, lb)
        ln = lambda p: restate.layernorm_cf(p, lw, lb)
        yield Check(f"s{s} dwconv7_ln", tap(f"s{s}_a"), ref, d + half_ulp16(ref.abs() + d),
                    [("pad zero->replicate", ln(F.conv2d(F.pad(xin, (3,) * 4, mode="replicate"), dw, db, groups=C)), 3),
                     ("7x7 kernel flipped", ln(dwc(xin, dw.flip(2, 3))), None)], fallback=fb)
        del pre, e, ref, d
        # ---- pwconv1 + GELU (+ GRN): s{s}_a -> s{s}_g
        a = tap(f"s{s}_a")
        w1, b1 = tr.w1(s)
        pre = conv1x1(a, w1, b1)
        e1 = (U16 + (C + 8) * K22) * conv1x1(a.abs(), w1.abs(), b1.abs())
        d1 = GELU_D * e1 + GELU_ABS + 4 * U32 * pre.abs()
        h = F.gelu(pre)
        h_drop = F.gelu(conv1x1(a, drop_last_kblock(w1, C), b1))
        del e1
        gam = tr.gamma(s)[None, :]
        P = h.shape[2] * h.shape[3]
        fold = has_tap(f"s{s}_w2s")
        W2 = tr.w2(s)
        if fold:
            yield Check(f"s{s} pwconv1_gelu", tap(f"s{s}_g"), h, d1 + half_ulp16(h.abs() + d1),
                        [("last K block dropped", h_drop, None)])
            # ---- GRN weight fold: s{s}_g, W2 -> s{s}_w2s
            g = tap(f"s{s}_g")
            m, Gx, mean = grn_mult(g, gam)
            dG = U16 * 1.01 * Gx + math.sqrt(P) * SUB
            dm = grn_mult_err(Gx, mean, dG, gam, P)
            ref = W2[None] * m[:, None, :]
            pre_t = W2.abs()[None] * dm[:, None, :] + half_ulp16(W2.abs())[None] * (m + dm)[:, None, :] + U32 * ref.abs()
            m0 = m.clone()
            m0[-1] = m[0]
            yield Check(f"s{s} grn_wscale", tap(f"s{s}_w2s"), ref, pre_t + half_ulp16(ref.abs() + pre_t),
                        [("last frame with frame 0's statistics", W2[None] * m0[:, None, :], "last_frame"),
                         ("GRN without the + x term", W2[None] * (m - 1)[:, None, :], None)])
            del g, ref, pre_t
        else:
            # ---- composite pwconv1 + GELU + GRN apply
            m, Gx, mean = grn_mult(h, gam)
            dm = grn_mult_err(Gx, mean, d1.pow(2).sum((2, 3)).sqrt(), gam, P)
            ref = h * m[:, :, None, None]
            d16 = d1 + half_ulp16(h.abs() + d1)
            mm, dmm = m[:, :, None, None], dm[:, :, None, None]
            pre_t = d16 * (mm.abs() + dmm) + h.abs() * dmm
            pre_t = pre_t + U32 * (ref.abs() + pre_t)
            m0 = m.clone()
            m0[-1] = m[0]
            Gc = h.pow(2).sum(1, keepdim=True).sqrt()      # the norm over the channels, normalised by its spatial mean
            msp = gam[:, :, None, None] * Gc / (Gc.mean((2, 3), keepdim=True) + 1e-6) + 1
            yield Check(f"s{s} pwconv1_gelu_grn_apply", tap(f"s{s}_g"), ref, pre_t + half_ulp16(ref.abs() + pre_t),
                        [("last frame with frame 0's statistics", h * m0[:, :, None, None], "last_frame"),
                         ("GRN over the spatial axes instead of the channels", h * msp, None),
                         ("last K block dropped", h_drop * grn_mult(h_drop, gam)[0][:, :, None, None], None)])
            del ref, pre_t, d16
        del a, pre, h, h_drop, d1
        # ---- pwconv2 + fp32 residual: s{s}_g (+ s{s}_w2s), s{s}_in -> stage{s}
        g = tap(f"s{s}_g")
        b2, b2n = tr.bias2(s), tr.bias2(s, beta=False)
        bb = lambda v: v[None, :, None, None]
        if fold:
            ws = tap(f"s{s}_w2s")
            mix = lambda ww, gg=g: torch.einsum("bnk,bkhw->bnhw", ww, gg)
            ref = xin + mix(ws) + bb(b2)
            tol = (4 * C + 8) * K22 * (xin.abs() + mix(ws.abs(), g.abs()) + bb(b2.abs())) + U32 * bb(b2.abs())
            ws0 = ws.clone()
            ws0[-1] = ws[0]
            wsd = ws.clone()
            wsd[:, :, 64 * ((4 * C - 1) // 64):] = 0
            muts = [("last frame with frame 0's W2", xin + mix(ws0) + bb(b2), "last_frame"),
                    ("GRN beta not folded into the bias", xin + mix(ws) + bb(b2n), None),
                    ("last K block dropped", xin + mix(wsd) + bb(b2), None)]
            del ws, ws0, wsd
        else:
            ref = xin + conv1x1(g, W2, b2)
            Ag = conv1x1(g.abs(), W2.abs())
            tol = U16 * Ag + (4 * C + 8) * K22 * (xin.abs() + Ag + bb(b2.abs())) + U32 * bb(b2.abs())
            muts = [("GRN beta not folded into the bias", xin + conv1x1(g, W2, b2n), None),
                    ("last K block dropped", xin + conv1x1(g, drop_last_kblock(W2[:, :, None, None], 4 * C), b2), None)]
        yield Check(f"s{s} pwconv2_resid", tap(f"stage{s}"), ref, tol, muts)
        del g, ref, tol, muts
        if s == 3:
            st = tap("stage3")
            yield Check("s3 pwconv2 fp16 copy", tap("stage3_16"), st, half_ulp16(st.abs()), [("the block input instead", xin, None)])
        del xin
    yield from head_checks(sd, tap("stage3_16"), tap, logits)


def head_checks(sd: Dict[str, torch.Tensor], x16: torch.Tensor, tap: Callable[[str], torch.Tensor], logits: torch.Tensor):
    """the pooled head (decoder.cuh add_head) on the fp16 trunk map x16 [B, C, h, h]: head3x3, head_pool, head_linear; tap(name)
    -> head_conv [B, C, h, h] / head_pooled [B, C] (float64)"""
    # ---- head 3x3, reflect padding: x16 -> head_conv
    C = x16.shape[1]
    w = sd[D + "output_upscaling.0.upsample_block.2.weight"]
    rp = lambda v: F.pad(v, (1, 1, 1, 1), mode="reflect")
    ref = F.conv2d(rp(x16), w)
    tol = (U16 + (9 * pitch(C) + 8) * K22) * F.conv2d(rp(x16.abs()), w.abs())
    yield Check("head3x3 (reflect)", tap("head_conv"), ref, tol,
                [("pad reflect->zero", F.conv2d(x16, w, padding=1), 1)])
    del x16, ref, tol
    # ---- head pool: head_conv -> head_pooled
    y = tap("head_conv")
    lw, lb = sd[D + "output_upscaling.0.upsample_block.3.weight"], sd[D + "output_upscaling.0.upsample_block.3.bias"]
    v, d, fb = ln_tol(y, torch.zeros_like(y), lw, lb)
    gv = F.gelu(v)
    dg = GELU_D * d + 4 * U32 * (v.abs() + gv.abs())
    P = y.shape[2] * y.shape[3]
    ref = gv.mean((2, 3))
    tol = dg.mean((2, 3)) + (P / 8 + 16) * U32 * gv.abs().mean((2, 3)) + U32 * ref.abs()
    yield Check("head_pool (LN + GELU + mean)", tap("head_pooled"), ref, tol,
                [("LayerNorm affine dropped", F.gelu(restate.layernorm_cf(y, torch.ones_like(lw), torch.zeros_like(lb))).mean((2, 3)),
                  None)], fallback=fb)
    del y, v, d, gv, dg
    # ---- head linear: head_pooled -> logits
    p = tap("head_pooled")
    lw, lb = sd[D + "linear.weight"].reshape(-1, C), sd[D + "linear.bias"]
    ref = p @ lw.T + lb
    tol = (C / 32 + 8) * K22 * (p.abs() @ lw.abs().T + lb.abs())
    yield Check("head_linear", logits.to(ref.dtype), ref, tol, [("bias dropped", p @ lw.T, None)])


def judge(ck: Check) -> dict:
    """max err / tol, NaN check, and for each mutation how often (and where) the output leaves the bound"""
    got = ck.got.to(ck.ref.dtype)
    nan = bool(torch.isnan(got).any())
    ratio = ((got - ck.ref).abs() / ck.tol).max().item()
    res = {"step": ck.step, "ratio": ratio, "nan": nan, "fallback": ck.fallback, "mutations": []}
    for name, mref, where in ck.mutations:
        v = (got - mref).abs() > ck.tol
        res["mutations"].append({"name": name, "violations": int(v.sum()), "outside": outside(v, where), "where": where})
    return res


def family(step: str) -> str:
    """step name -> family: the stage prefix dropped"""
    return step.split(" ", 1)[1] if step[:1] == "s" and step[1:2].isdigit() else step


# ---------------------------------------------------------------------------------------------------------------- CPU chains
def one_pass_ln(x: torch.Tensor, g: torch.Tensor, b: torch.Tensor, eps: float = 1e-6) -> torch.Tensor:
    """channels-first LayerNorm from sum(x) and sum(x^2), var = E[x^2] - mean^2 clamped at 0 (the stem GEMM's epilogue)"""
    mu = x.mean(1, keepdim=True)
    var = ((x * x).mean(1, keepdim=True) - mu * mu).clamp_min(0)
    return g[:, None, None] * (x - mu) / torch.sqrt(var + eps) + b[:, None, None]


def chain(tr: Trunk, imgs: torch.Tensor, fold: List[bool], emulate: bool = False) -> Dict[str, torch.Tensor]:
    """every tap of the detect plan for frames `imgs`, computed step by step, `fold[s]`: stage s folds GRN into W2, and the
    logits (float64 tensors).  emulate=False: float64, the blocks before each stage's last one through restate.convnext_block.
    emulate=True: the kernels' precision: every convolution, LayerNorm, GELU and sum in fp32 (the stem GEMM's LayerNorm one-pass),
    fp16 rounding of the operands and outputs the kernels round, GRN statistics of the pre-rounding values, the folded bias
    computed in float64 and rounded to fp32.  Its fp32 sums run in ATen's order, not the kernels', so they exercise the K 2^-22
    terms of the bounds without reproducing the kernels' exact values."""
    dt = torch.float32 if emulate else torch.float64
    sd = {k: v.to(dt) for k, v in tr.sd.items()}
    dims = tr.dims
    t: Dict[str, torch.Tensor] = {}
    h16 = r16 if emulate else (lambda v: v)
    x = 2 * imgs.to(dt) - 1
    w0, b0 = sd[Q + "downsample_layers.0.0.weight"], sd[Q + "downsample_layers.0.0.bias"]
    ln0 = restate.layernorm_cf
    if emulate and dims[0] <= 256:
        x, w0, ln0 = r16(x), r16(w0), one_pass_ln
    x = ln0(F.conv2d(x, w0, b0, stride=tr.stride), sd[Q + "downsample_layers.0.1.weight"], sd[Q + "downsample_layers.0.1.bias"])
    for s in range(4):
        C = dims[s]
        if s > 0:
            t[f"s{s}_ln"] = h16(restate.layernorm_cf(x, sd[Q + f"downsample_layers.{s}.0.weight"], sd[Q + f"downsample_layers.{s}.0.bias"]))
            x = F.conv2d(t[f"s{s}_ln"], h16(sd[Q + f"downsample_layers.{s}.1.weight"]), sd[Q + f"downsample_layers.{s}.1.bias"], stride=2)
        t[f"s{s}_ds"] = x
        for j in range(tr.depths[s]):
            k = tr.blk(s, j)
            if j == tr.depths[s] - 1:
                t[f"s{s}_in"] = x
            if not emulate and j < tr.depths[s] - 1:
                x = restate.convnext_block(sd, k, x)
                continue
            a = h16(restate.layernorm_cf(F.conv2d(x, sd[k + "dwconv.weight"], sd[k + "dwconv.bias"], padding=3, groups=C),
                                         sd[k + "norm.weight"], sd[k + "norm.bias"]))
            h = F.gelu(conv1x1(a, h16(sd[k + "pwconv1.weight"]), sd[k + "pwconv1.bias"]))
            m = grn_mult(h, sd[k + "grn.gamma"].reshape(1, -1))[0]       # from the pre-rounding values
            g = h16(h)
            W2 = sd[k + "pwconv2.weight"]
            b2 = (tr.sd[k + "pwconv2.bias"] + tr.sd[k + "pwconv2.weight"] @ tr.sd[k + "grn.beta"].reshape(-1)).to(dt)
            if fold[s]:
                w2s = h16(h16(W2)[None] * m[:, None, :])
                y = torch.einsum("bnk,bkhw->bnhw", w2s, g)
            else:
                w2s = None
                g = h16(g * m[:, :, None, None])
                y = conv1x1(g, h16(W2))
            x = x + (y + b2[None, :, None, None])
            if j == tr.depths[s] - 1:
                t[f"s{s}_a"], t[f"s{s}_g"] = a, g
                if w2s is not None:
                    t[f"s{s}_w2s"] = w2s
        t[f"stage{s}"] = x
    t["stage3_16"] = h16(x)
    t["head_conv"] = F.conv2d(F.pad(t["stage3_16"], (1, 1, 1, 1), mode="reflect"), h16(sd[D + "output_upscaling.0.upsample_block.2.weight"]))
    v = restate.layernorm_cf(t["head_conv"], sd[D + "output_upscaling.0.upsample_block.3.weight"],
                             sd[D + "output_upscaling.0.upsample_block.3.bias"])
    t["head_pooled"] = F.gelu(v).mean((2, 3))
    t["logits"] = t["head_pooled"] @ sd[D + "linear.weight"].reshape(-1, dims[3]).T + sd[D + "linear.bias"]
    return {n: v.to(torch.float64) for n, v in t.items()}
