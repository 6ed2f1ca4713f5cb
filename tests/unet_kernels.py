"""Float64 references and forward error bounds for every kernel the U-Net embed plan launches, judged one kernel at a time.

Each step's inputs are the plan's own debug taps (exact fp16 values, or the caller's fp32 frames for `unet.first`), so a step
is compared against float64 arithmetic on exactly what the kernel read and errors never accumulate from step to step.  The
references are built from `oracle/restate.py` (BatchNorm as `_norm`, `layernorm_cf`, `msg_embed`, the luma row of `rgb_to_y`,
the bilinear / reflect / conv order of `upsample_block`), in float64, on the state dict cast to float64.

Error bounds (u = 2^-11 is the fp16 unit roundoff, u32 = 2^-24 the fp32 one; `*` is the step's own convolution, taken in
float64 on absolute values):

* Convolution epilogues (resblock 3x3 / 1x1, stride-2 down conv, up tap GEMM).  With `W` the BN-folded float64 weight,
  A = |W| * |x| + |b| (+ |resid| where the epilogue adds one), the computed value differs from the float64 one by
      |D| <= c u A  +  K 2^-22 A  +  1/2 ulp_fp16(|ref| + c u A + K 2^-22 A).
  c = 1 counts the single fp16 rounding of each weight (BN fold, skip scale 2^-1/2 and the phase fold are done in fp32 on the
  host and rounded once); the operands are exact fp16 taps.  K = (number of products) + 8 covers the fp32 tensor-core
  accumulation (each partial sum is within 2^-23 of its exact value, counted with a 2x margin as 2^-22), the fp32 bias /
  residual adds and the fp32 fold of BN into the weight (about 4 u32 per weight).  ReLU is 1-Lipschitz; the last term is the
  rounding of the output to fp16, taken at the largest value the computed result can have (subnormals: 2^-25).
* `unet.first` runs in fp32 on fp32 frames (no fp16 weights): c = 0, K = 9 C_in + 16, with A = |W| * (|x| + 1) + |b| so
  that the absolute fp32 error of the luma / 2x - 1 preprocessing (<= 8 u32) is covered too.
* Bilinear gather + LayerNorm (`unet.upgather`).  Each tap's four-corner mix is one packed fp16 multiply and three packed
  fma: four roundings, each at most u times the running partial sum, which is at most T = sum_corners w |y| (all w >= 0),
  plus 2^-25 each where the partial sum is subnormal; the nine taps add in fp32.  Per channel, before the norm,
      e_c = (4 u + 9 u32) G(|y|)_c + 36 2^-25,      G = the gather (bilinear x2, reflect pad, 9-tap sum),
  since G applied to |y| is exactly the sum of the T's.  The phase-folded up-conv (`unet.upphase`) has e_c = c u A_c +
  K 2^-22 A_c with A = the up-conv of |[x | skip 2^-1/2]| with |W| (bilinear weights are >= 0, so the folded phase weights
  are bounded by it), c = 1 inside and c = 0 on the border pixels that `unet.upborder` recomputes in fp32.
* LayerNorm (eps 1e-6, biased variance) then propagates e to first order with the float64 sigma and x_hat of the reference:
      |D y_c| <= |g_c| / sigma (e_c + mean(e) + |x_hat_c| mean(|x_hat| e)) / (1 - 2 rho)^2,   rho = max(e) / sigma,
  where the factor 1 / (1 - 2 rho)^2 bounds the change of sigma itself (|sigma' - sigma| <= 2 max(e)); it is applied while
  rho < 1/4 and otherwise the bound is the output range 2 |g_c| sqrt(C), on which the check cannot fail: the fraction of
  pixels on that fallback is reported per step and the GPU tests require it to be zero.  The fp32 norm adds C u32 mean|a| / sigma to the
  shift, (C + 6) u32 |x_hat_c| to the scale and 2 u32 (|g x_hat| + |beta|) to the affine.  ReLU is 1-Lipschitz; then the
  fp16 output rounding as above.
* Message channels: an fp32 sum of K table rows, |D| <= K u32 sum|rows| + 1/2 ulp_fp16.
* `delta` (the last block's second conv with the 1x1 outc + tanh fused, all in fp32): the block output before rounding is
  within e = u A + K 2^-22 A, so |D delta_o| <= sum_c |w_oc| e_c + (C + 8) 2^-22 (sum_c |w_oc| |blk_c| + |b_o|) + 2^-21
  (tanhf), using |tanh'| <= 1.

A ratio err / tol above 1 is a bug to find, never a reason to raise c.  Each step family also has mutations: a reference
with one deliberate defect that the GPU output must violate, proving the bound is tight enough to see it.
"""
from __future__ import annotations

import math
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional

import torch
import torch.nn.functional as F

from oracle import restate

U16 = 2.0 ** -11
U32 = 2.0 ** -24
K22 = 2.0 ** -22
SUB16 = 2.0 ** -25           # half the spacing of fp16 subnormals
SQ = 2.0 ** -0.5
P = "embedder.unet."


def half_ulp16(v: torch.Tensor) -> torch.Tensor:
    """half the fp16 spacing at |value| v (v >= 0)"""
    e = torch.floor(torch.log2(v.clamp_min(2.0 ** -14)))
    return torch.where(v < 2.0 ** -14, torch.full_like(v, SUB16), torch.exp2(e - 11))


def border_mask(h: int, w: int, device) -> torch.Tensor:
    m = torch.zeros(h, w, dtype=torch.bool, device=device)
    m[0, :] = m[-1, :] = m[:, 0] = m[:, -1] = True
    return m


@dataclass
class Check:
    """one kernel output against its float64 reference: |got - ref| <= tol everywhere; each mutation must break that"""
    step: str
    got: torch.Tensor
    ref: torch.Tensor
    tol: torch.Tensor
    mutations: List[tuple] = field(default_factory=list)   # (name, mutated ref, where: None | "border" | "last_frame")
    fallback: float = 0.0   # LayerNorm steps: fraction of pixels whose bound is the output range (rho >= 1/4), where it cannot fail


class Net:
    """float64 parameters of one U-Net embedder, BatchNorm folded the way the plan folds it"""

    def __init__(self, sd: Dict[str, torch.Tensor], spec: dict, device="cpu"):
        self.spec, self.u = spec, spec["unet"]
        self.sd = {k: v.to(device=device, dtype=torch.float64) for k, v in sd.items() if v.is_floating_point()}
        self.L = len(self.u["mults"])
        self.z = [self.u["z_channels"] * m for m in self.u["mults"]]
        self.zb = self.z[-1] + spec["hidden"]

    def bn_conv(self, block: str, i: int):
        """conv `block`.double_conv.i (i = 0, 3) with the eval-mode BatchNorm at i + 1 folded in: (W', b') in float64"""
        bn = f"{block}.double_conv.{i + 1}"
        s = self.sd[bn + ".weight"] / torch.sqrt(self.sd[bn + ".running_var"] + 1e-5)
        b = self.sd[bn + ".bias"] - self.sd[bn + ".running_mean"] * s
        return self.sd[f"{block}.double_conv.{i}.weight"] * s[:, None, None, None], b


# ---------------------------------------------------------------------------------------------------------------- conv steps
def conv_check(step, got, x, w, b, *, relu=False, resid=None, stride=1, pad=1, c=1, mut_pad=True, mut_shift=False,
               extra_mut: Optional[Callable] = None) -> Check:
    """got = [relu](conv(x, w) + b) [+ resid] with zero padding `pad` and `stride`; x exact operands (float64)"""
    def run(xx, pad_mode="zeros", shift=False):
        if shift:     # stride-2 sampling grid moved by one pixel: centres 2i + 1 instead of 2i
            xx = F.pad(xx, (1, 1, 1, 1))[:, :, 1:, 1:]
            y = F.conv2d(xx, w, b, stride=stride)
        elif pad_mode == "replicate":
            y = F.conv2d(F.pad(xx, (pad,) * 4, mode="replicate"), w, b, stride=stride)
        else:
            y = F.conv2d(xx, w, b, stride=stride, padding=pad)
        if relu:
            y = F.relu(y)
        return y + resid if resid is not None else y
    ref = run(x)
    A = F.conv2d(x.abs(), w.abs(), b.abs() if b is not None else None, stride=stride, padding=pad)
    if resid is not None:
        A = A + resid.abs()
    K = w.shape[1] * w.shape[2] * w.shape[3] + 8
    pre = (c * U16 + K * K22) * A
    ck = Check(step, got, ref, pre + half_ulp16(ref.abs() + pre))
    if mut_pad and pad > 0:
        ck.mutations.append(("pad zero->replicate", run(x, "replicate"), "border"))
    if mut_shift:
        ck.mutations.append(("stride-2 phase +1", run(x, shift=True), None))
    if extra_mut is not None:
        ck.mutations.extend(extra_mut(run))
    return ck


def ln_tol(pre: torch.Tensor, e: torch.Tensor, g: torch.Tensor, beta: torch.Tensor, eps: float = 1e-6):
    """(LayerNorm(pre) reference, bound on |D LN| for a pre-norm error <= e per channel, fraction of pixels on the output-range
    fallback); channels dim 1"""
    C = pre.shape[1]
    mu = pre.mean(1, keepdim=True)
    sig = torch.sqrt((pre - mu).pow(2).mean(1, keepdim=True) + eps)
    xh = (pre - mu) / sig
    e = e + C * U32 * pre.abs().mean(1, keepdim=True)
    first = (e + e.mean(1, keepdim=True) + xh.abs() * (xh.abs() * e).mean(1, keepdim=True)) / sig
    rho = e.amax(1, keepdim=True) / sig
    gg, bb = g.abs()[None, :, None, None], beta.abs()[None, :, None, None]
    d = gg * (first / (1 - 2 * rho.clamp_max(0.25)) ** 2 + (C + 6) * U32 * xh.abs()) + 2 * U32 * (gg * xh.abs() + bb)
    d = torch.where(rho < 0.25, d, 2 * gg * math.sqrt(C))
    ref = restate.layernorm_cf(pre, g, beta, eps)
    return ref, d, (rho >= 0.25).double().mean().item()


def ln_relu_check(step, got, pre, e, g, beta, muts) -> Check:
    ref, d, fb = ln_tol(pre, e, g, beta)
    ref = F.relu(ref)
    ck = Check(step, got, ref, d + half_ulp16(ref.abs() + d), fallback=fb)
    for name, mpre, where in muts:
        ck.mutations.append((name, F.relu(restate.layernorm_cf(mpre, g, beta, 1e-6)), where))
    return ck


def gather(y: torch.Tensor, C: int, align_corners=False, pad="reflect", f: int = 2) -> torch.Tensor:
    """y [B, 9 C, h, w] (tap-major channels, tap = 3 r + s) -> sum_taps shift(pad(bilinear_xf(y_tap))), [B, C, f h, f w]"""
    B, _, h, w = y.shape
    out = torch.zeros(B, C, f * h, f * w, dtype=y.dtype, device=y.device)
    for t in range(9):
        r, s = divmod(t, 3)
        u = F.interpolate(y[:, t * C:(t + 1) * C], scale_factor=f, mode="bilinear", align_corners=align_corners)
        out += F.pad(u, (1, 1, 1, 1), mode=pad)[:, :, r:r + f * h, s:s + f * w]
    return out


def up_pre(xcat: torch.Tensor, w: torch.Tensor, align_corners=False, pad="reflect") -> torch.Tensor:
    """the up-conv of restate.upsample_block before its LayerNorm"""
    u = F.interpolate(xcat, scale_factor=2, mode="bilinear", align_corners=align_corners)
    return F.conv2d(F.pad(u, (1, 1, 1, 1), mode=pad), w)


def tap_weight(w: torch.Tensor) -> torch.Tensor:
    """[Cout, Ct, 3, 3] -> the tap GEMM's [9 Cout, Ct, 1, 1], rows tap * Cout + co"""
    co, ct = w.shape[:2]
    return w.permute(2, 3, 0, 1).reshape(9 * co, ct, 1, 1)


def phase_pre(xcat: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """the phase decomposition of up_pre: per output phase (py, px) a 3x3 conv over the replicate-padded LOW-resolution map
    with the bilinear weights folded into the taps.  Equals up_pre except on the outermost output rows / columns."""
    g = torch.tensor([[[.75, .25, 0.], [.25, .75, 0.], [0., .75, .25]],
                      [[.25, .75, 0.], [0., .75, .25], [0., .25, .75]]], dtype=w.dtype, device=w.device)   # [phase][d][e]
    B, _, h, wd = xcat.shape
    xp = F.pad(xcat, (1, 1, 1, 1), mode="replicate")
    out = torch.empty(B, w.shape[0], 2 * h, 2 * wd, dtype=w.dtype, device=w.device)
    for py in range(2):
        for px in range(2):
            wp = torch.einsum("ocde,dy,ex->ocyx", w, g[py], g[px])
            out[:, :, py::2, px::2] = F.conv2d(xp, wp)
    return out


# ---------------------------------------------------------------------------------------------------------------- the plan
def first_input(net: Net, imgs: torch.Tensor, luma=(0.299, 0.587, 0.114), swap_rb=False) -> torch.Tensor:
    """embedder.py:23 x * 2 - 1 on the luma row of restate.rgb_to_y (yuv cards) or on RGB"""
    x = imgs.to(torch.float64)
    if swap_rb:
        x = x[:, [2, 1, 0]]
    if net.spec["yuv"]:
        x = luma[0] * x[:, 0:1] + luma[1] * x[:, 1:2] + luma[2] * x[:, 2:3]
    return 2 * x - 1


def plan_checks(net: Net, tap: Callable[[str], torch.Tensor], imgs: torch.Tensor, msgs: torch.Tensor, has_tap: Callable[[str], bool]):
    """Yields one Check per kernel of the embed plan.  tap(name) -> NCHW float64 debug tap of the sub-batch whose frames are
    `imgs` [B, 3, S, S] and messages `msgs` [B, K]."""
    sd, L, z, zb = net.sd, net.L, net.z, net.zb
    cin = net.u["in_channels"]
    # unet.first: fp32 conv + folded BN + ReLU, and the fp32 1x1 residual conv
    x = first_input(net, imgs)
    w1, b1 = net.bn_conv(P + "inc", 0)
    wr, br = sd[P + "inc.res_conv.weight"], sd[P + "inc.res_conv.bias"]
    colour = [("BT.709 luma", first_input(net, imgs, luma=(0.2126, 0.7152, 0.0722)))] if net.spec["yuv"] else \
             [("R/B swapped", first_input(net, imgs, swap_rb=True))]

    def first(step, got, w, b, relu, pad):
        A = F.conv2d(x.abs() + 1, w.abs(), b.abs(), padding=pad)
        ref = F.conv2d(x, w, b, padding=pad)
        if relu:
            ref = F.relu(ref)
        pre = (9 * cin + 16) * K22 * A
        ck = Check(step, got, ref, pre + half_ulp16(ref.abs() + pre))
        for name, xm in colour:
            m = F.conv2d(xm, w, b, padding=pad)
            ck.mutations.append((name, F.relu(m) if relu else m, None))
        if pad:
            m = F.conv2d(F.pad(x, (1, 1, 1, 1), mode="replicate"), w, b)
            ck.mutations.append(("pad zero->replicate", F.relu(m) if relu else m, "border"))
        return ck
    yield first("unet.first h1", tap("first_h"), w1, b1, True, 1)
    yield first("unet.first r0", tap("first_r"), wr, br, False, 0)
    del x

    def resblock(name, key, xin, out_got, fuse_outc=False):
        wres, bres = sd[key + ".res_conv.weight"], sd[key + ".res_conv.bias"]
        yield conv_check(f"{name}.r (1x1)", tap(name + ".r"), xin, wres, bres, pad=0)
        wa, ba = net.bn_conv(key, 0)
        yield conv_check(f"{name}.h (3x3)", tap(name + ".h"), xin, wa, ba, relu=True)
        h, r = tap(name + ".h"), tap(name + ".r")
        wb, bb = net.bn_conv(key, 3)
        if not fuse_outc:
            yield conv_check(f"{name} (3x3 + resid)", out_got(), h, wb, bb, relu=True, resid=r)
            return
        # last block: the 3x3 conv's fp32 output goes through the fused 1x1 outc (+ tanh) into delta
        blk = F.relu(F.conv2d(h, wb, bb, padding=1)) + r
        A = F.conv2d(h.abs(), wb.abs(), bb.abs(), padding=1) + r.abs()
        e = (U16 + (wb.shape[1] * 9 + 8) * K22) * A
        ow, ob = sd[P + "outc.weight"], sd[P + "outc.bias"]

        def outc(v, bias=True):
            o = F.conv2d(v, ow, ob if bias else None)
            return torch.tanh(o) if net.u["last_tanh"] else o
        tol = F.conv2d(e, ow.abs()) + (ow.shape[1] + 8) * K22 * F.conv2d(blk.abs(), ow.abs(), ob.abs()) + 2.0 ** -21
        yield Check(f"{name} (3x3 + resid) + outc -> delta", out_got(), outc(blk), tol, [("outc bias dropped", outc(blk, False), None)])

    yield conv_check("inc (3x3 + resid)", tap("inc"), tap("first_h"), *net.bn_conv(P + "inc", 3), relu=True, resid=tap("first_r"))
    prev = "inc"
    for i in range(L - 1):
        yield conv_check(f"down{i}_conv (3x3 s2)", tap(f"down{i}_conv"), tap(prev), sd[P + f"downs.{i}.down.weight"],
                         sd[P + f"downs.{i}.down.bias"], stride=2, mut_pad=False, mut_shift=True)
        out = (lambda: tap("cat")[:, :z[-1]]) if i == L - 2 else (lambda n=f"down{i}": tap(n))
        yield from resblock(f"down{i}", P + f"downs.{i}.conv", tap(f"down{i}_conv"), out)
        prev = f"down{i}"
    # message channels of the bottleneck concat
    table = sd[P + "msg_processor.msg_embeddings.weight"].cpu()
    hs = imgs.shape[-1] >> (L - 1)
    msgs = msgs.cpu()
    emb = lambda t, m: restate.msg_embed({P + "msg_processor.msg_embeddings.weight": t}, net.spec, m)
    mref, msum = emb(table, msgs), emb(table.abs(), msgs)
    flip = msgs.clone()
    flip[-1, 0] = 1 - flip[-1, 0]
    mflip = emb(table, flip)
    K = msgs.shape[1]
    bc = lambda v: v.to(imgs.device)[:, :, None, None].expand(-1, -1, hs, hs)
    pre = K * U32 * msum
    yield Check("msg channels", tap("cat")[:, z[-1]:], bc(mref), bc(pre + half_ulp16(mref.abs() + pre)),
                [("bit 0 of the last frame flipped", bc(mflip), "last_frame")])
    prev = "cat"
    for i in range(net.u["num_blocks"]):
        yield from resblock(f"bott{i}", P + f"bottleneck.model.{i}", tap(prev), lambda n=f"bott{i}": tap(n))
        prev = f"bott{i}"
    zz = list(z)
    zz[-1] = zb
    for j, ii in enumerate(reversed(range(L - 1))):
        cin_, cout = zz[ii + 1], zz[ii]
        U = P + f"ups.{j}.up.upsample_block."
        w, lg, lb = sd[U + "2.weight"], sd[U + "3.weight"], sd[U + "3.bias"]
        xs = tap(prev)
        skip = tap("cat") if j == 0 else tap(f"down{L - 2 - j}")
        xcat = torch.cat([xs, skip * SQ], 1)
        x1 = torch.cat([xs, skip], 1)
        del xs, skip
        if has_tap(f"up{j}_taps"):
            wt = tap_weight(w)
            ref = F.conv2d(xcat, wt)
            A = F.conv2d(xcat.abs(), wt.abs())
            pre = (U16 + (2 * cin_ + 8) * K22) * A
            yield Check(f"up{j}_taps (tap GEMM {2 * cin_}->{9 * cout})", tap(f"up{j}_taps"), ref, pre + half_ulp16(ref.abs() + pre),
                        [("skip scale 1", F.conv2d(x1, wt), None)])
            del ref, A, pre
            y = tap(f"up{j}_taps")
            e = (4 * U16 + 9 * U32) * gather(y.abs(), cout) + 36 * SUB16
            yield ln_relu_check(f"up{j}_conv (gather + LN {cout})", tap(f"up{j}_conv"), gather(y, cout), e, lg, lb,
                                [("align_corners=True", gather(y, cout, align_corners=True), None),
                                 ("pad reflect->replicate", gather(y, cout, pad="replicate"), "border")])
            del y, e
        else:   # phase-folded up-conv + fp32 border fix-up, one unit
            A = up_pre(xcat.abs(), w.abs())
            cmask = (~border_mask(A.shape[-2], A.shape[-1], A.device)).to(A.dtype)
            e = (cmask * U16 + (9 * 2 * cin_ + 8 + 36) * K22) * A
            del A
            yield ln_relu_check(f"up{j}_conv (phase + border {2 * cin_}->{cout})", tap(f"up{j}_conv"), up_pre(xcat, w), e, lg, lb,
                                [("skip scale 1", up_pre(x1, w), None),
                                 ("align_corners=True", up_pre(xcat, w, align_corners=True), None),
                                 ("pad reflect->replicate", up_pre(xcat, w, pad="replicate"), "border")])
        del xcat, x1
        last = ii == 0
        yield from resblock(f"up{j}", P + f"ups.{j}.conv", tap(f"up{j}_conv"),
                            (lambda: tap("delta")) if last else (lambda n=f"up{j}": tap(n)), fuse_outc=last)
        prev = f"up{j}"


def judge(ck: Check) -> dict:
    """max err / tol, NaN check, and for each mutation whether (and where) the GPU output leaves the bound"""
    got = ck.got.to(ck.ref.dtype)
    nan = bool(torch.isnan(got).any())
    ratio = ((got - ck.ref).abs() / ck.tol).max().item()
    res = {"step": ck.step, "ratio": ratio, "nan": nan, "fallback": ck.fallback, "mutations": []}
    for name, mref, where in ck.mutations:
        v = (got - mref).abs() > ck.tol
        n = int(v.sum())
        if where == "border":
            inside = int((v & ~border_mask(v.shape[-2], v.shape[-1], v.device)).sum())
        elif where == "last_frame":
            inside = int(v[:-1].sum())
        else:
            inside = 0
        res["mutations"].append({"name": name, "violations": n, "outside": inside, "where": where})
    return res
