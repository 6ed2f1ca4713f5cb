"""Float64 references and forward error bounds for every kernel of the SAM-ViT detect plan (patch embedding, the last block, the
neck and the pooled head), judged one kernel at a time.

Each step's inputs are the plan's debug taps (exact fp16 / fp32 values, or the caller's fp32 frames for the im2col), so a step is
compared against float64 arithmetic on exactly what the kernel read.  The plan reuses one residual stream, one LayerNorm buffer and
one neck buffer, so the values the last block L and the neck read from a buffer a later step overwrites come from the copies
`vsb_debug_keep_inputs` adds: vit.blk{L}.in, .ln1, .mid and vit.neck1x1.  The references are built from `oracle/restate.py`
(`_vit_block`'s LayerNorm / qkv / attention / proj / MLP order, `layernorm_cf`, the neck and head of `sam_extractor_forward`) and the
attention restatement below, on the state dict cast to float64.  Taps are token rows [B, G, G, C] (float64).

Error bounds reuse tests/unet_kernels.py and tests/cnx_kernels.py: u = 2^-11, u32 = 2^-24, K22 = 2^-22, the GEMM-epilogue form
    |D| <= |a| * r16(W) + K 2^-22 A (+ 1/2 ulp_fp16(|ref| + ...) where the output is fp16),   A = |a| * |W| + |b| (+ |resid|),
with r16(W) = 1/2 ulp_fp16(|W|) the rounding of each weight to fp16 (exact for normal and subnormal weights alike, where the
c u A form of the other suites misses the subnormal ones), K = (number of products) + 8 for the fp32 tensor-core accumulation and
the fp32 bias / residual adds, and the first-order LayerNorm propagation `ln_tol` (two-pass fp32 statistics; the GPU test forbids
its output-range fallback).

* `vit_patch_im2col_kernel`: bit-exact.  Each patch row is fp16 of the frame's pixels in the weight's K order (c, r, s).
* patch GEMM + `vit_pos_add_kernel` (composite): the host folds x * 2 - 1 into W' = 2W (exact in fp32, one fp16 rounding) and the
  table T = pos_embed + b - sum(W) (float64, rounded to fp32 once: u32 |T|).  The GEMM adds 768 products into fp32, the table add
  is one more fp32 rounding: |p| * r16(2W) + (768 + 8) K22 (|p| * |2W| + |T|) + u32 |T|.  fp32 output.
* `ln_rows` (LayerNorm 1 / 2 of the block with eps 1e-5, both neck LayerNorms with eps 1e-6): ln_tol with no input error, then
  1/2 ulp_fp16.
* qkv (with or without bias), lin1 + erf GELU: fp16 outputs; GELU as in tests/cnx_kernels.py (|gelu'| <= 1.13, 4e-6 absolute for
  the packed gelu_erf_p and ex2.approx, 4 u32 |x|).
* attention: `attention_bound` below on the qkv tap (fp16 P, fp32 scores over 64 products, fp16 output).
* proj + in-place fp32 residual: K = E + 8 on A = |att| * |Wp| + |bp| + |in|, against vit.blk{L}.mid.
* lin2 + in-place fp32 residual: K = mlp_dim + 8 on A = |hid| * |W2| + |b2| + |mid|, against vit.blk{L}.
* vit.x16: the same epilogue writes fp16 of the fp32 stream value it stores: bit-exact.
* neck 1x1 (no bias): K = E + 8, fp32 output.
* neck 3x3 (zero padding 1, gather loader over M = B G G rows, K in (r, s, c) order): K = 9 out_chans + 8, fp32 output.  Judged on
  every element, so frame borders and 128-row tiles that straddle two frames are covered.
* pooled head: `cnx_kernels.head_checks` on vit.neck.

A ratio err / tol above 1 is a bug to find, never a reason to raise a constant.  Each step family has mutations (a reference with
one deliberate defect that the GPU output must violate).  Footprints as in tests/cnx_kernels.py: None (anywhere), "last_frame", or
an int w (the w outermost rows / columns of every map).  Left out on purpose:
* the LayerNorm eps swap 1e-5 <-> 1e-6: at the unit-scale variance of these rows it moves sigma by ~5e-6 relative, far inside
  1/2 ulp_fp16 (2.4e-4 relative), so it is structurally invisible;
* the attention window shift where a frame holds one region and there are no relative positions (a relabelling of the keys);
* "bias dropped" on the bias-less qkv epilogue; there the checkpoint's unused qkv bias added is the mutation instead.
* the tanh-approximate GELU in lin1: it differs from the erf GELU by at most 4.7e-4 (at x = 2.7), below 1/2 ulp_fp16 of the
  output wherever |x| < 2.5, and fp16 resolves it only for pre-activations below about -2.5, more than four standard deviations
  of these lin1 rows: no row of the 64-frame batch reaches one (measured on an H100), nor does the 2-frame emulation.
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F

from oracle import restate
from tests import cnx_kernels as ck
from tests.cnx_kernels import GELU_ABS, GELU_D, r16
from tests.unet_kernels import K22, U32, Check, half_ulp16, ln_tol

Q = "detector.image_encoder."
PATCH = 16
EXACT = 1e-300          # the bound of a bit-exact step: any difference leaves it

# name: (encoder overrides of the videoseal_0.0 card's sam_small block, processing size, frames on the GPU); global_attn_indexes
# picks the kind of the last block, the one under test
_TINY = {"embed_dim": 192, "num_heads": 3, "out_chans": 192}       # the reference's sam_tiny widths
_BASE = {"embed_dim": 768, "num_heads": 12, "out_chans": 768}      # the reference's sam_base widths
CONFIGS = {
    "small_256_b3": ({"depth": 2, "global_attn_indexes": [0]}, 256, 3),                # last block windowed + rel-pos
    "small_256_b64": ({"depth": 2, "global_attn_indexes": [1]}, 256, 64),              # production batch, last block global
    "small_256_b70": ({"depth": 1, "global_attn_indexes": []}, 256, 70),               # taps of the 6-frame second sub-batch
    "tiny_256_b4": ({**_TINY, "depth": 2, "global_attn_indexes": [1]}, 256, 4),        # block_n 96, 3 heads, LN over 192
    "base_256_b3": ({**_BASE, "depth": 2, "global_attn_indexes": [1]}, 256, 3),        # 12 heads, lin2 K = 3072, LN over 768
    "small_128_b3": ({"depth": 1, "global_attn_indexes": []}, 128, 3),                 # ragged M, one window per frame, 8 x 8 map
    "small_384_b3": ({"depth": 2, "global_attn_indexes": [1]}, 384, 3),                # 576 tokens, 47-row table, straddling tiles
    "small_512_b2": ({"depth": 2, "global_attn_indexes": [1]}, 512, 2),                # 1024 tokens, n = 32
    "win40_640_b2": ({"depth": 1, "window_size": 40, "global_attn_indexes": [], "use_rel_pos": False}, 640, 2),
    "nobias_norel_256_b3": ({"depth": 1, "global_attn_indexes": [], "qkv_bias": False, "use_rel_pos": False}, 256, 3),
    "e448_256_b3": ({"embed_dim": 448, "num_heads": 7, "out_chans": 320, "depth": 1, "global_attn_indexes": []}, 256, 3),
}


class Vit:
    """float64 parameters of one SAM-ViT extractor with its pooled head; L is the last block"""

    def __init__(self, sd: Dict[str, torch.Tensor], spec: dict, device="cpu"):
        self.spec, v = spec, spec["vit"]
        self.sd = {k: t.to(device=device, dtype=torch.float64) for k, t in sd.items()
                   if t.is_floating_point() and (k.startswith(Q) or k.startswith(ck.D))}
        self.E, self.depth, self.heads = int(v["embed_dim"]), int(v["depth"]), int(v["num_heads"])
        self.mlp, self.oc, self.window = int(self.E * float(v["mlp_ratio"])), int(v["out_chans"]), int(v["window_size"])
        self.glob = [int(i) for i in v["global_attn_indexes"]]    # the card's encoder block (restate / vit_oracle spec)
        self.rel, self.qkv_bias = bool(v.get("use_rel_pos", False)), bool(v.get("qkv_bias", True))
        self.G = int(spec["img_size"]) // PATCH
        self.L = self.depth - 1

    def blk(self, i: int = -1) -> str:
        return Q + f"blocks.{self.L if i < 0 else i}."

    def n(self, i: int = -1) -> int:
        """side of the attention regions of block i"""
        return self.G if (self.L if i < 0 else i) in self.glob else self.window

    def rel_tables(self, i: int = -1, rounded: bool = True):
        k = self.blk(i) + "attn.rel_pos_"
        if not self.rel:
            return None, None
        return tuple(r16(self.sd[k + a]) if rounded else self.sd[k + a] for a in "hw")

    def qkv_b(self) -> Optional[torch.Tensor]:
        return self.sd[self.blk() + "attn.qkv.bias"] if self.qkv_bias else None


# ---------------------------------------------------------------------------------------------------------------- helpers
def patches_of(imgs: torch.Tensor) -> torch.Tensor:
    """[B, 3, S, S] -> [B, G, G, 768] im2col rows in the weight's K order (c, r, s)"""
    B, _, S, _ = imgs.shape
    G = S // PATCH
    return imgs.reshape(B, 3, G, PATCH, G, PATCH).permute(0, 2, 4, 1, 3, 5).reshape(B, G, G, 3 * PATCH * PATCH)


def lin(a: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor] = None) -> torch.Tensor:
    y = a @ w.T
    return y if b is None else y + b


def gemm_tol(a: torch.Tensor, w: torch.Tensor, b: Optional[torch.Tensor] = None, resid: Optional[torch.Tensor] = None):
    """fp16 rounding of the weights plus the fp32 accumulation of K products, the bias and the residual (module docstring)"""
    A = lin(a.abs(), w.abs(), None if b is None else b.abs())
    if resid is not None:
        A = A + resid.abs()
    return lin(a.abs(), half_ulp16(w.abs())) + (w.shape[1] + 8) * K22 * A


def nchw(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 3, 1, 2)


def nhwc(t: torch.Tensor) -> torch.Tensor:
    return t.permute(0, 2, 3, 1)


def ln_rows_check(step, got, x, w, b, eps, muts) -> Check:
    """ln_rows on rows x [B, G, G, C] -> fp16; muts: (name, (w, b, unbiased)) LayerNorms of x with other parameters"""
    ref, d, fb = ln_tol(nchw(x), torch.zeros_like(nchw(x)), w, b, eps)
    ref, d = nhwc(ref), nhwc(d)
    mr = []
    for name, (mw, mb, unbiased) in muts:
        mu = x.mean(-1, keepdim=True)
        var = x.var(-1, unbiased=unbiased, keepdim=True)
        mr.append((name, (x - mu) / torch.sqrt(var + eps) * mw + mb, None))
    return Check(step, got, ref, d + half_ulp16(ref.abs() + d), mr, fallback=fb)


def last_frame_from_first(t: torch.Tensor) -> torch.Tensor:
    m = t.clone()
    m[-1] = t[0]
    return m


# ---------------------------------------------------------------------------------------------------------------- attention
def attention_f64(qkv, heads, n, G, rel_h, rel_w, mutate=None):
    """float64 restatement of vit.py:302-353 + :431-470 on the qkv rows [B, G, G, 3E] of one block (window partition by index);
    rel_h / rel_w: the fp16-rounded tables or None.  Returns (out [B, G, G, E], A [B, G, G, E]) with A = sum_k p |v| / sum_k p,
    and the per-row score error scale S_err [B, G, G, heads] for the bound.  mutate: "shift" (windows one token to the right),
    "scaled" (relative terms from the scaled q), "transpose" (the h / w tables swapped), "reverse" (offsets k - q, not q - k)."""
    B, E = qkv.shape[0], qkv.shape[-1] // 3
    hd = E // heads
    shift = 1 if mutate == "shift" else 0     # windows placed one token to the right (with wrap-around)
    x = qkv.double().roll(-shift, dims=2).reshape(B, G // n, n, G // n, n, 3, heads, hd).permute(5, 0, 1, 3, 6, 2, 4, 7)
    x = x.reshape(3, -1, n * n, hd)           # [3, B*win*heads, T, hd]
    q, k, v = x[0], x[1], x[2]
    scale = hd ** -0.5
    s = (q * scale) @ k.transpose(-1, -2)
    serr = (q.abs() * scale) @ k.abs().transpose(-1, -2)
    if rel_h is not None:
        ar = torch.arange(n, device=qkv.device)
        idx = ar[:, None] - ar[None, :] + n - 1
        if mutate == "reverse":
            idx = (n - 1) - (ar[:, None] - ar[None, :])
        Rh, Rw = rel_h.double()[idx], rel_w.double()[idx]      # [n, n, hd]
        if mutate == "transpose":
            Rh, Rw = Rw, Rh
        rq = (q * scale if mutate == "scaled" else q).reshape(-1, n, n, hd)
        rh = torch.einsum("bhwc,hkc->bhwk", rq, Rh)
        rw = torch.einsum("bhwc,wkc->bhwk", rq, Rw)
        s = (s.view(-1, n, n, n, n) + rh[:, :, :, :, None] + rw[:, :, :, None, :]).view(-1, n * n, n * n)
        aq = q.abs().reshape(-1, n, n, hd)
        eh = torch.einsum("bhwc,hkc->bhwk", aq, Rh.abs())
        ew = torch.einsum("bhwc,wkc->bhwk", aq, Rw.abs())
        serr = (serr.view(-1, n, n, n, n) + eh[:, :, :, :, None] + ew[:, :, :, None, :]).view(-1, n * n, n * n)
    p = torch.softmax(s, dim=-1)
    o = p @ v
    a = p @ v.abs()
    se = serr.amax(dim=-1, keepdim=True).expand(-1, -1, hd)

    def back(t):   # [B*win*heads, T, hd] -> [B, G, G, E]
        return t.reshape(B, G // n, G // n, heads, n, n, hd).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, G, G, E).roll(shift, dims=2)
    return back(o), back(a), back(se)


def attention_bound(ref, a, se):
    """per element: fp16 rounding of the output (2^-11 |o|); fp16 rounding of P (2^-11 per p, so 2^-11 sum p|v| / sum p); the fp32
    score accumulation over 64 products (<= 64 * 2^-24 of the sum of |terms|, twice: it moves a p and the normaliser); fp32 exp,
    sums and division (a few ulps of A)"""
    u16, u32 = 2.0 ** -11, 2.0 ** -24
    return u16 * ref.abs() + (u16 + 2 * 64 * u32 * se + 16 * u32) * a + 1e-7


def attention_emulated(qkv, heads, n, G, rel_h, rel_w):
    """the attention kernel's precision: fp32 scores and softmax, P rounded to fp16 before P V, fp32 normaliser, fp16 output"""
    B, E = qkv.shape[0], qkv.shape[-1] // 3
    hd = E // heads
    x = qkv.float().reshape(B, G // n, n, G // n, n, 3, heads, hd).permute(5, 0, 1, 3, 6, 2, 4, 7).reshape(3, -1, n * n, hd)
    q, k, v = x[0], x[1], x[2]
    s = (q * hd ** -0.5) @ k.transpose(-1, -2)
    if rel_h is not None:
        ar = torch.arange(n, device=qkv.device)
        idx = ar[:, None] - ar[None, :] + n - 1
        rq = q.reshape(-1, n, n, hd)
        rh = torch.einsum("bhwc,hkc->bhwk", rq, rel_h.float()[idx])
        rw = torch.einsum("bhwc,wkc->bhwk", rq, rel_w.float()[idx])
        s = (s.view(-1, n, n, n, n) + rh[:, :, :, :, None] + rw[:, :, :, None, :]).view(-1, n * n, n * n)
    p = torch.exp(s - s.amax(-1, keepdim=True))
    o = (r16(p) @ v) / p.sum(-1, keepdim=True)
    o = o.reshape(B, G // n, G // n, heads, n, n, hd).permute(0, 1, 4, 2, 5, 3, 6).reshape(B, G, G, E)
    return r16(o)


# ---------------------------------------------------------------------------------------------------------------- the plan
def plan_checks(vt: Vit, tap: Callable[[str], torch.Tensor], imgs: torch.Tensor, logits: torch.Tensor):
    """Yields one Check per kernel of the ViT detect plan.  tap(name) -> float64 debug tap [B, G, G, C] of the sub-batch whose
    frames are `imgs` [B, 3, S, S] (head_pooled [B, 1, 1, C]); `logits` [B, 1 + K] are that sub-batch's outputs."""
    sd, E, G = vt.sd, vt.E, vt.G
    bi = f"vit.blk{vt.L}"
    k = vt.blk()
    # ---- im2col: frames -> vit.patches
    x = imgs.to(torch.float64)
    ref = patches_of(r16(x))
    shp = ref.shape[:3] + (3, PATCH, PATCH)
    yield Check("vit_patch_im2col", tap("vit.patches"), ref, torch.full_like(ref, EXACT),
                [("(r, s) transposed in a patch", ref.reshape(shp).transpose(-1, -2).reshape(ref.shape), None),
                 ("channels reversed", ref.reshape(shp).flip(3).reshape(ref.shape), None),
                 ("last frame from frame 0's pixels", last_frame_from_first(ref), "last_frame")])
    del x, ref
    # ---- patch GEMM + position table: vit.patches -> vit.embed
    p = tap("vit.patches")
    W = sd[Q + "patch_embed.proj.weight"].reshape(E, -1)
    b, pe = sd[Q + "patch_embed.proj.bias"], sd[Q + "pos_embed"][0]
    table = pe + (b - W.sum(1))
    emb = lambda pp, t: lin(pp, 2 * W) + t
    ref = emb(p, table)
    tol = gemm_tol(p, 2 * W) + 776 * K22 * table.abs() + U32 * table.abs()
    yield Check("patch_gemm_pos_add", tap("vit.embed"), ref, tol,
                [("x * 2 - 1 fold dropped (b, not b - sum W)", emb(p, pe + b), None),
                 ("pos table transposed (py <-> px)", emb(p, pe.transpose(0, 1) + (b - W.sum(1))), None),
                 ("pos row shifted by one token", emb(p, table.reshape(G * G, E).roll(1, 0).reshape(G, G, E)), None),
                 ("last frame from frame 0's patches", last_frame_from_first(ref), "last_frame")])
    del p, ref, tol, table
    # ---- LayerNorm 1: vit.blk{L}.in -> .ln1
    n1, n2 = (sd[k + "norm1.weight"], sd[k + "norm1.bias"]), (sd[k + "norm2.weight"], sd[k + "norm2.bias"])
    xin = tap(bi + ".in")
    yield ln_rows_check("ln1", tap(bi + ".ln1"), xin, *n1, 1e-5,
                        [("norm1 / norm2 parameters swapped", (*n2, False)), ("unbiased variance", (*n1, True))])
    # ---- qkv: .ln1 -> .qkv
    a = tap(bi + ".ln1")
    Wq, bq = sd[k + "attn.qkv.weight"], vt.qkv_b()
    ref = lin(a, Wq, bq)
    pre = gemm_tol(a, Wq, bq)
    h = vt.heads
    muts = [("columns (heads, 3, 64) instead of (3, heads, 64)",
             ref.reshape(*ref.shape[:3], 3, h, 64).transpose(3, 4).reshape(ref.shape), None)]
    muts.append(("bias dropped", lin(a, Wq), None) if bq is not None
                else ("the checkpoint's unused bias added", lin(a, Wq, sd[k + "attn.qkv.bias"]), None))
    yield Check("qkv", tap(bi + ".qkv"), ref, pre + half_ulp16(ref.abs() + pre), muts)
    del a, ref, pre, muts
    # ---- attention: .qkv -> .attn
    qkv = tap(bi + ".qkv")
    n = vt.n()
    rel = vt.rel_tables()
    ref, A, se = attention_f64(qkv, h, n, G, *rel)
    muts = (["shift"] if n < G or vt.rel else []) + (["scaled", "transpose", "reverse"] if vt.rel else [])
    yield Check("attention", tap(bi + ".attn"), ref, attention_bound(ref, A, se),
                [(m, attention_f64(qkv, h, n, G, *rel, mutate=m)[0], None) for m in muts])
    del qkv, ref, A, se
    # ---- proj + in-place fp32 residual: .attn, .in -> .mid
    att = tap(bi + ".attn")
    Wp, bp = sd[k + "attn.proj.weight"], sd[k + "attn.proj.bias"]
    ref = xin + lin(att, Wp, bp)
    yield Check("proj_resid", tap(bi + ".mid"), ref, gemm_tol(att, Wp, bp, xin), [("residual dropped", lin(att, Wp, bp), None)])
    del att, ref
    # ---- LayerNorm 2: .mid -> .ln2
    mid = tap(bi + ".mid")
    yield ln_rows_check("ln2", tap(bi + ".ln2"), mid, *n2, 1e-5,
                        [("norm1 / norm2 parameters swapped", (*n1, False)), ("unbiased variance", (*n2, True))])
    # ---- lin1 + GELU: .ln2 -> .hid
    a = tap(bi + ".ln2")
    W1, b1 = sd[k + "mlp.lin1.weight"], sd[k + "mlp.lin1.bias"]
    pre = lin(a, W1, b1)
    d1 = GELU_D * gemm_tol(a, W1, b1) + GELU_ABS + 4 * U32 * pre.abs()
    ref = F.gelu(pre)
    yield Check("lin1_gelu", tap(bi + ".hid"), ref, d1 + half_ulp16(ref.abs() + d1),
                [("bias dropped", F.gelu(lin(a, W1)), None),
                 ("last K block dropped", F.gelu(lin(a, ck.drop_last_kblock(W1[:, :, None, None], E)[:, :, 0, 0], b1)), None)])
    del a, pre, d1, ref
    # ---- lin2 + in-place fp32 residual: .hid, .mid -> vit.blk{L}; its fp16 copy vit.x16
    hid = tap(bi + ".hid")
    W2, b2 = sd[k + "mlp.lin2.weight"], sd[k + "mlp.lin2.bias"]
    ref = mid + lin(hid, W2, b2)
    yield Check("lin2_resid", tap(bi), ref, gemm_tol(hid, W2, b2, mid),
                [("residual dropped", lin(hid, W2, b2), None), ("residual from .in instead of .mid", xin + lin(hid, W2, b2), None)])
    del hid, ref, xin
    out = tap(bi)
    yield Check("x16 copy", tap("vit.x16"), r16(out), torch.full_like(out, EXACT), [("fp16 of .mid instead", r16(mid), None)])
    del out, mid
    # ---- neck 1x1 (no bias): vit.x16 -> vit.neck1x1
    x16 = tap("vit.x16")
    Wn = sd[Q + "neck.0.weight"][:, :, 0, 0]
    yield Check("neck1x1", tap("vit.neck1x1"), lin(x16, Wn), gemm_tol(x16, Wn),
                [("last K block dropped", lin(x16, ck.drop_last_kblock(Wn[:, :, None, None], E)[:, :, 0, 0]), None)])
    del x16
    # ---- neck LayerNorm 1: vit.neck1x1 -> vit.neck_ln1
    l1, l2 = (sd[Q + "neck.1.weight"], sd[Q + "neck.1.bias"]), (sd[Q + "neck.3.weight"], sd[Q + "neck.3.bias"])
    yield ln_rows_check("neck_ln1", tap("vit.neck_ln1"), tap("vit.neck1x1"), *l1, 1e-6,
                        [("neck.1 / neck.3 parameters swapped", (*l2, False)), ("unbiased variance", (*l1, True))])
    # ---- neck 3x3, zero padding 1: vit.neck_ln1 -> vit.neck3x3 (judged channels-first: the border footprint is spatial)
    yn = nchw(tap("vit.neck_ln1"))
    W3 = sd[Q + "neck.2.weight"]
    ref = F.conv2d(yn, W3, padding=1)
    tol = F.conv2d(yn.abs(), half_ulp16(W3.abs()), padding=1) + (9 * vt.oc + 8) * K22 * F.conv2d(yn.abs(), W3.abs(), padding=1)
    yield Check("neck3x3", nchw(tap("vit.neck3x3")), ref, tol,
                [("pad zero->reflect", F.conv2d(F.pad(yn, (1, 1, 1, 1), mode="reflect"), W3), 1),
                 ("kh <-> kw", F.conv2d(yn, W3.transpose(2, 3), padding=1), None)])
    del yn, ref, tol
    # ---- neck LayerNorm 2: vit.neck3x3 -> vit.neck
    yield ln_rows_check("neck_ln2", tap("vit.neck"), tap("vit.neck3x3"), *l2, 1e-6,
                        [("neck.1 / neck.3 parameters swapped", (*l1, False)), ("unbiased variance", (*l2, True))])
    # ---- the pooled head on vit.neck
    htap = lambda name: tap(name)[:, 0, 0, :] if name == "head_pooled" else nchw(tap(name))
    yield from ck.head_checks(sd, nchw(tap("vit.neck")), htap, logits)


def family(step: str) -> str:
    return step


# ---------------------------------------------------------------------------------------------------------------- CPU chains
def mm32(a: torch.Tensor, w: torch.Tensor) -> torch.Tensor:
    """a [..., K] @ w[N, K]^T in fp32, accumulated one 64-wide K block after the other (the kernels' K-block order)"""
    acc = None
    for k0 in range(0, a.shape[-1], 64):
        part = a[..., k0:k0 + 64] @ w[:, k0:k0 + 64].T
        acc = part if acc is None else acc + part
    return acc


def chain(vt: Vit, imgs: torch.Tensor, emulate: bool = False) -> Dict[str, torch.Tensor]:
    """every tap of the ViT detect plan for frames `imgs` and the logits (float64 tensors, tap layouts).  emulate=False: float64,
    the blocks before the last through restate._vit_block.  emulate=True: the kernels' precision: fp16 operands (pixels, weights,
    LayerNorm outputs, qkv, attention output, hidden rows, the neck's fp16 maps), fp32 GEMM accumulation in 64-wide K blocks (the
    3x3 over its (r, s, c) im2col), fp32 LayerNorm / GELU / attention softmax with P rounded to fp16, the position table formed in
    float64 and rounded to fp32 once."""
    dt = torch.float32 if emulate else torch.float64
    sd = {k: v.to(dt) for k, v in vt.sd.items()}
    h16 = r16 if emulate else (lambda v: v)
    mm = (lambda a, w: mm32(a, r16(w))) if emulate else (lambda a, w: a @ w.T)
    E, G, L = vt.E, vt.G, vt.L
    t: Dict[str, torch.Tensor] = {}
    bi = f"vit.blk{L}"
    t["vit.patches"] = patches_of(h16(imgs.to(dt)))
    W = vt.sd[Q + "patch_embed.proj.weight"].reshape(E, -1)
    table = (vt.sd[Q + "pos_embed"][0] + vt.sd[Q + "patch_embed.proj.bias"] - W.sum(1)).to(dt)
    x = mm(t["vit.patches"], (2 * W).to(dt)) + table
    t["vit.embed"] = x
    for i in range(L):
        x = restate._vit_block(sd, vt.blk(i), x, vt.heads, 0 if i in vt.glob else vt.window, vt.rel)
    k = vt.blk()
    ln = lambda v, w, b, eps: F.layer_norm(v, (v.shape[-1],), sd[w], sd[b], eps)
    t[bi + ".in"] = x
    t[bi + ".ln1"] = a = h16(ln(x, k + "norm1.weight", k + "norm1.bias", 1e-5))
    q = mm(a, sd[k + "attn.qkv.weight"])
    if vt.qkv_bias:
        q = q + sd[k + "attn.qkv.bias"]
    t[bi + ".qkv"] = q = h16(q)
    if emulate:
        att = attention_emulated(q, vt.heads, vt.n(), G, *vt.rel_tables())
    else:
        att = attention_f64(q, vt.heads, vt.n(), G, *vt.rel_tables(rounded=False))[0]
    t[bi + ".attn"] = att
    x = x + (mm(att, sd[k + "attn.proj.weight"]) + sd[k + "attn.proj.bias"])
    t[bi + ".mid"] = x
    t[bi + ".ln2"] = a = h16(ln(x, k + "norm2.weight", k + "norm2.bias", 1e-5))
    t[bi + ".hid"] = hid = h16(F.gelu(mm(a, sd[k + "mlp.lin1.weight"]) + sd[k + "mlp.lin1.bias"]))
    x = x + (mm(hid, sd[k + "mlp.lin2.weight"]) + sd[k + "mlp.lin2.bias"])
    t[bi] = x
    t["vit.x16"] = x16 = h16(x)
    t["vit.neck1x1"] = y = mm(x16, sd[Q + "neck.0.weight"][:, :, 0, 0])
    t["vit.neck_ln1"] = yn = h16(ln(y, Q + "neck.1.weight", Q + "neck.1.bias", 1e-6))
    W3 = sd[Q + "neck.2.weight"]
    if emulate:   # the gather loader's K order (r, s, c)
        cols = F.pad(nchw(yn), (1, 1, 1, 1))
        cols = torch.stack([cols[:, :, r:r + G, s:s + G] for r in range(3) for s in range(3)], 1)   # [B, 9, C, G, G]
        cols = cols.permute(0, 3, 4, 1, 2).reshape(*yn.shape[:3], -1)
        y3 = mm(cols, W3.permute(0, 2, 3, 1).reshape(W3.shape[0], -1))
    else:
        y3 = nhwc(F.conv2d(nchw(yn), W3, padding=1))
    t["vit.neck3x3"] = y3
    t["vit.neck"] = h16(ln(y3, Q + "neck.3.weight", Q + "neck.3.bias", 1e-6))
    D = ck.D
    hc = F.conv2d(F.pad(nchw(t["vit.neck"]), (1, 1, 1, 1), mode="reflect"), h16(sd[D + "output_upscaling.0.upsample_block.2.weight"]))
    t["head_conv"] = nhwc(hc)
    v = restate.layernorm_cf(hc, sd[D + "output_upscaling.0.upsample_block.3.weight"], sd[D + "output_upscaling.0.upsample_block.3.bias"])
    pooled = F.gelu(v).mean((2, 3))
    t["head_pooled"] = pooled[:, None, None, :]
    t["logits"] = pooled @ sd[D + "linear.weight"].reshape(-1, vt.oc).T + sd[D + "linear.bias"]
    return {n: v.to(torch.float64) for n, v in t.items()}
