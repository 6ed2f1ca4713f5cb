"""Float64 references and forward error bounds for every kernel of the pixel-wise decoder (Decoder::add_pixel_decoder), judged one
kernel at a time.

Each stage i is a tap GEMM at the low resolution, y = x W_tap (`pd.uptap1x1`, debug tap pd{i}_y [B, h, h, 9 Co], tap-major
channels tap * Co + co), then a gather kernel that forms every output pixel from 9 taps x 4 bilinear corners, LayerNorm and GELU
(`pd.upgather` tiled, `pd.upgather_untiled`, fp16 output pd{i}), or, at the last stage, the same gather with the 1x1 head fused,
writing the caller's fp32 maps (`pd.gather_head`).  Stage 0 reads the trunk's fp16 output (stage3_16, or vit.neck for a SAM-ViT),
stage i > 0 reads pd{i-1}.  So every step is compared against float64 arithmetic on exactly what its kernel read.  The references
restate modules/common.py:45-52 through oracle/restate.py (`layernorm_cf`) and the tap form of tests/unet_kernels.py (`gather`,
`tap_weight`): bilinear x F with align_corners=False, ReflectionPad2d(1), the 3x3 conv without bias, LayerNorm eps 1e-6, GELU.

Error bounds (u = 2^-11, u32 = 2^-24, K22 = 2^-22, as in tests/unet_kernels.py):

* `pd.uptap1x1` (TMA GEMM, fp16 weights rounded once on the host, fp32 accumulation, no bias, fp16 output):
  c u A + K 2^-22 A + 1/2 ulp_fp16, A = |W_tap| |x|, K = C_in + 8.  A stage whose input is narrower than its GEMM K (48 channels
  at K = 64, Decoder::gemm_k) runs over zero pad columns: the reference uses the C_in real channels only, so pad columns that
  did not read as zero would break the bound.
* The gather's four-corner mix of each tap is one packed fp16 multiply and three packed fma, each rounding at most u times the
  running partial sum (all corner weights are >= 0, so the partial sums are at most T = sum_corners w |y|), plus 2^-25 where a
  partial sum is subnormal; the nine taps add in fp32.  The corner weights are products of two 1-D weights that are multiples of
  1/4 (factor 2) or 1/8 (factor 4), so they are multiples of 1/64 and exact in fp16.  Per channel, before the norm,
      e_c = (4 u + 9 u32) G_F(|y|)_c + 36 2^-25,      G_F = the gather (bilinear x F, reflect pad, 9-tap sum),
  since G_F applied to |y| is exactly the sum of the T's.  Then `ln_tol` (first-order LayerNorm propagation, fallback to the
  output range when rho >= 1/4, which the GPU tests forbid), then the `erff` GELU, 1.13 d + 4 u32 (|v| + |gelu(v)|) as for the
  ConvNeXt head pool (tests/cnx_kernels.py), then the fp16 output rounding.
* `pd.gather_head`: the gather, LayerNorm and GELU stay in fp32 registers (d_c as above, no rounding), then the 1x1 head in fp32
  with two accumulators (the bias in the first):  sum_c |w_oc| d_c + (C + 1) 2^-22 (sum_c |w_oc| (|g_c| + d_c) + |b_o|).

A ratio err / tol above 1 is a bug to find, never a reason to raise a constant.  Mutations (footprints as in tests/cnx_kernels.py):
the GEMM's taps transposed (r <-> s) and its last input channel dropped; the gather's align_corners=True, its bilinear phase moved
by one output pixel, reflect -> zero padding and, for the fp16 gathers at factor 2, reflect -> replicate padding (both on the
image border), and, for the tiled kernels, the staged taps clamped at the tile's edge instead of the image's (the tile-edge
pixels); the head's bias dropped, the weights of two channels swapped, two output planes swapped, and the last frame's maps
replaced by the frame before (the sub-batch offset of the maps).  Replicate padding is no defect at factor 4, where up-sampled rows
0 and 1 both equal input row 0, and at the head it moves the maps by less than the bound, which sums the LayerNorm bound over
the channels (at most 0.4 of it on the CPU cases of tests/test_pd_kernels_cpu.py).
"""
from __future__ import annotations

from typing import Callable, Dict, Sequence

import torch
import torch.nn.functional as F

from oracle import restate
from tests.cnx_kernels import GELU_D, r16, shift1
from tests.unet_kernels import K22, SUB16, U16, U32, Check, gather, half_ulp16, ln_tol, tap_weight

D = "detector.pixel_decoder."

# The configurations the GPU tests run: name -> (extractor, upscale stages, processing size, frames, nbits, ConvNeXt dims or None for
# the preset's).  ConvNeXt trunks at depth 1 (the trunk is not under test here).  Together they reach every gather instantiation
# of launch_pd_gather that a loadable model can dispatch: the eight fused heads (F 2 / 4 x VPT 1..4), the tiled (F, VPT) pairs
# (2, 1), (2, 3), (4, 1), (4, 3) and the untiled (2, 1), (2, 3), (4, 3).  Untiled F4/VPT1 cannot be dispatched: processing sizes
# are multiples of 128, so every map is a multiple of 4 pixels, and 256 channels (VPT 1, G 32) stage in 166 KB.
CONFIGS = {
    "tiny256_b70": ("convnext_tiny_pw", [4, 4, 2], 256, 70, 256, None),   # 192, 48, 24: tiled F4/VPT3 (G 8, G 2), K 48 padded to
                                                                           # 64, head F2/VPT3; maps of the 6-frame sub-batch at 64
    "tiny256_424": ("convnext_tiny_pw", [4, 2, 4], 256, 3, 256, None),    # 192, 96, 24: tiled F2/VPT3, head F4/VPT3 (257 outputs)
    "tiny384_b5": ("convnext_tiny_pw", [2, 4, 4], 384, 5, 256, None),     # 384, 96, 24: untiled F2/VPT3 on the 12-pixel map
    "wide256": ("convnext_tiny_pw", [4, 4, 4], 256, 2, 32, [96, 192, 384, 1536]),     # 384, 96, 24: untiled F4/VPT3 (the tile
                                                                                       # would take 243 KB), 512^2 maps
    "base256_442": ("convnext_base_pw", [4, 4, 2], 256, 2, 256, None),    # 256, 64, 32: tiled F4/VPT1 (G 32, G 8), head F2/VPT4
    "base256_424": ("convnext_base_pw", [4, 2, 4], 256, 2, 256, None),    # 256, 128, 32: tiled F2/VPT1 (G 16), head F4/VPT4
    "base256_444": ("convnext_base_pw", [4, 4, 4], 256, 2, 32, None),     # 256, 64, 16: head F4/VPT2, 512^2 maps
    "base256_4424": ("convnext_base_pw", [4, 4, 2, 4], 256, 2, 32, None),  # ..., 32, 8: tiled F2/VPT1 (G 4), head F4/VPT1, 1024^2
    "base256_4442": ("convnext_base_pw", [4, 4, 4, 2], 256, 2, 32, None),  # ..., 16, 8: F4 gather at 16 channels (G 2), head F2/VPT1
    "narrow384_244": ("convnext_tiny_pw", [2, 4, 4], 384, 3, 32, [96, 192, 256, 256]),    # 128, 32, 8: untiled F2/VPT1 on the
                                                                                           # 12-pixel map
    "vit256_422": ("vit", [4, 2, 2], 256, 3, 256, None),                  # out_chans 256 -> 64, 32, 16: input vit.neck, head F2/VPT2
}


def config_card(name: str) -> dict:
    """the model card of a CONFIGS entry"""
    from tests import pixelwise_oracle as pw
    from tests import vit_oracle as vo
    from tests.util import apply_overrides, load_card
    ext, stages, S, _, nbits, dims = CONFIGS[name]
    if ext == "vit":
        card = vo.vit_card(True, S, {"out_chans": 256, "depth": 1}, stages)
    else:
        card = apply_overrides(pw.preset_card(ext, load_card("videoseal_1.0")), {"depths": [1, 1, 1, 1]})
        card["extractor"]["params"]["pixel_decoder"]["upscale_stages"] = list(stages)
        card["args"]["img_size_proc"] = S
        if dims:
            card["extractor"]["params"]["encoder"]["dims"] = list(dims)
    card["args"]["nbits"] = nbits
    return card


def stage_weights(sd: Dict[str, torch.Tensor], i: int):
    k = D + f"output_upscaling.{i}.upsample_block."
    return sd[k + "2.weight"], sd[k + "3.weight"], sd[k + "3.bias"]


def act(pre: torch.Tensor, g: torch.Tensor, b: torch.Tensor) -> torch.Tensor:
    return F.gelu(restate.layernorm_cf(pre, g, b))


def tile_clamped(y: torch.Tensor, C: int, f: int) -> torch.Tensor:
    """gather(y) as a tiled kernel would compute it if its staged taps were clamped at the tile's edge instead of the image's: each
    16 x 16 output tile sees the halo row / column of its T x T low-resolution tile (T = 16 / f) replaced by the tile's own edge.
    Tiles two apart have disjoint halos, so the four (row, column) parities of the tiles each take one gather."""
    B, _, h, w = y.shape
    T = 16 // f

    def idx(n, parity):
        i = torch.arange(n, device=y.device)
        for t in range(parity, n // T, 2):
            if t > 0:
                i[t * T - 1] = t * T
            if (t + 1) * T < n:
                i[(t + 1) * T] = (t + 1) * T - 1
        return i
    out = torch.empty(B, C, f * h, f * w, dtype=y.dtype, device=y.device)
    par_r = (torch.arange(f * h, device=y.device) // 16) % 2
    par_c = (torch.arange(f * w, device=y.device) // 16) % 2
    for pr in range(2):
        for pc in range(2):
            g = gather(y[:, :, idx(h, pr)][:, :, :, idx(w, pc)], C, f=f)
            m = (par_r[:, None] == pr) & (par_c[None, :] == pc)
            out[..., m] = g[..., m]
    return out


def plan_checks(sd: Dict[str, torch.Tensor], stages: Sequence[int], x0: torch.Tensor, tap: Callable[[str], torch.Tensor],
                maps: torch.Tensor, tiled: Sequence[bool]):
    """Yields one Check per kernel of the pixel decoder.  sd: float64 state dict; x0: the stage-0 input [B, C, h, h] (exact fp16
    values); tap(name) -> NCHW float64 debug tap of the same sub-batch; maps [B, 1 + K, P, P]: that sub-batch's output;
    tiled[i]: stage i ran the tiled gather (the head always does)."""
    x = x0
    n = len(stages)
    for i, f in enumerate(stages):
        w, lg, lb = stage_weights(sd, i)
        Co, cin, h = w.shape[0], x.shape[1], x.shape[-1]
        wt = tap_weight(w)
        ref = F.conv2d(x, wt)
        pre = (U16 + (cin + 8) * K22) * F.conv2d(x.abs(), wt.abs())
        yield Check(f"pd{i} uptap1x1 {cin}-{9 * Co}@{h}", tap(f"pd{i}_y"), ref, pre + half_ulp16(ref.abs() + pre),
                    [("taps transposed (r <-> s)", F.conv2d(x, tap_weight(w.transpose(2, 3))), None),
                     ("last input channel dropped", F.conv2d(x[:, :-1], wt[:, :-1]), None)])
        del ref, pre
        y = tap(f"pd{i}_y")
        pre = gather(y, Co, f=f)
        e = (4 * U16 + 9 * U32) * gather(y.abs(), Co, f=f) + 36 * SUB16
        v, d, fb = ln_tol(pre, e, lg, lb)
        del e
        g = F.gelu(v)
        dg = GELU_D * d + 4 * U32 * (v.abs() + g.abs())
        del v, d
        muts = [("align_corners=True", gather(y, Co, align_corners=True, f=f), None), ("bilinear phase +1", shift1(pre), None),
                ("pad reflect->zero", gather(y, Co, pad="constant", f=f), 1)]
        if f == 2 and i + 1 < n:   # see the module docstring
            muts.append(("pad reflect->replicate", gather(y, Co, pad="replicate", f=f), 1))
        if tiled[i]:
            muts.append(("taps clamped at the tile's edge", tile_clamped(y, Co, f), "tile_edge"))
        del y, pre
        tag = f"{Co}x{f}@{f * h}"
        if i + 1 < n:
            yield Check(f"pd{i} {'upgather' if tiled[i] else 'upgather_untiled'} {tag}", tap(f"pd{i}"), g,
                        dg + half_ulp16(g.abs() + dg), [(m, act(p, lg, lb), wh) for m, p, wh in muts], fallback=fb)
            del g, dg, muts
            x = tap(f"pd{i}")
            continue
        hw, hb = sd[D + "linear.weight"], sd[D + "linear.bias"]
        head = lambda gg, ww=hw, bb=hb: F.conv2d(gg, ww, bb)   # noqa: E731
        ref = head(g)
        tol = F.conv2d(dg, hw.abs()) + (Co + 1) * K22 * F.conv2d(g.abs() + dg, hw.abs(), hb.abs())
        hm = [(m, head(act(p, lg, lb)), wh) for m, p, wh in muts]
        del muts
        hm.append(("head bias dropped", head(g, hw, None), None))
        wsw = hw.clone()
        wsw[:, [0, 1]] = hw[:, [1, 0]]
        hm.append(("head weights of channels 0 and 1 swapped", head(g, wsw), None))
        hm.append(("output planes 0 and 1 swapped", ref[:, [1, 0] + list(range(2, ref.shape[1]))], None))
        prev = ref.clone()
        prev[-1] = ref[-2]
        hm.append(("last frame's maps from the frame before", prev, "last_frame"))
        yield Check(f"pd{i} gather_head {tag}", maps, ref, tol, hm, fallback=fb)


def family(step: str) -> str:
    """step name -> family: the stage prefix and the geometry dropped (pd.upgather, pd.gather_head, ...)"""
    return "pd." + step.split(" ")[1]


# ---------------------------------------------------------------------------------------------------------------- CPU chains
def chain(sd: Dict[str, torch.Tensor], stages: Sequence[int], x0: torch.Tensor) -> Dict[str, torch.Tensor]:
    """every tap of the pixel decoder in float64 from the stage-0 input x0, and the maps"""
    t, x = {}, x0
    for i, f in enumerate(stages):
        w, lg, lb = stage_weights(sd, i)
        t[f"pd{i}_y"] = F.conv2d(x, tap_weight(w))
        x = t[f"pd{i}"] = act(gather(t[f"pd{i}_y"], w.shape[0], f=f), lg, lb)
    t["maps"] = F.conv2d(x, sd[D + "linear.weight"], sd[D + "linear.bias"])
    return t


def src_table(n_out: int, n_in: int, f: int, r: int):
    """ups_gather_ln_{tiled_,}kernel's bilinear sources along one axis: for each output coordinate o, the rows (a, b) and the weight
    of a that tap offset r (0..2) reads after reflecting o + r - 1 into the up-sampled map (align_corners=False, clamped at 0)"""
    u = torch.arange(n_out) + r - 1
    u = torch.where(u < 0, -u, u)
    u = torch.where(u >= n_out, 2 * n_out - 2 - u, u)
    if f == 2:
        i, odd = u // 2, u % 2 == 1
        a = torch.where(odd, i, (i - 1).clamp_min(0))
        b = torch.where(odd, (i + 1).clamp_max(n_in - 1), i)
        wa = torch.where(odd, 0.75, 0.25)
    else:
        i, p = u // 4, u % 4
        lo = p < 2
        a = torch.where(lo, (i - 1).clamp_min(0), i)
        b = torch.where(lo, i, (i + 1).clamp_max(n_in - 1))
        wa = torch.where(lo, (3 - 2 * p) / 8, (11 - 2 * p) / 8)
    return a, b, wa.to(torch.float64)


def kernel_gather(y: torch.Tensor, C: int, f: int) -> torch.Tensor:
    """the gather in the kernel's precision and order: per tap, __hmul2 then three __hfma2 over the corners (w11, w10, w01, w00),
    each fma computed exactly in float64 and rounded once to fp16 (exact fma semantics: the products of 1/64-multiples and fp16
    values and their sums are exact in float64), the nine taps summed in fp32 in (r, s) order.  y: fp16 values; fp32 result."""
    B, _, h, w = y.shape
    acc = torch.zeros(B, C, f * h, f * w, dtype=torch.float32)
    for r in range(3):
        ya, yb, wy = src_table(f * h, h, f, r)
        for s in range(3):
            xa, xb, wx = src_table(f * w, w, f, s)
            Y = y[:, (3 * r + s) * C:(3 * r + s + 1) * C]
            at = lambda ii, jj: Y[:, :, ii][:, :, :, jj]   # noqa: E731
            Wy, Wx = wy[:, None], wx[None, :]
            t = r16((1 - Wy) * (1 - Wx) * at(yb, xb))
            t = r16((1 - Wy) * Wx * at(yb, xa) + t)
            t = r16(Wy * (1 - Wx) * at(ya, xb) + t)
            t = r16(Wy * Wx * at(ya, xa) + t)
            acc = acc + t.float()
    return acc


def emulate(sd: Dict[str, torch.Tensor], stages: Sequence[int], x0: torch.Tensor) -> Dict[str, torch.Tensor]:
    """every tap of the pixel decoder in the kernels' precision from the fp16 stage-0 input x0: fp16 weights and fp32 accumulation
    in the GEMM (ATen's order), fp16 taps, kernel_gather, LayerNorm and GELU in fp32, fp16 stage outputs, the head in fp32"""
    s32 = {k: v.float() for k, v in sd.items() if k.startswith(D)}
    t, x = {}, x0
    for i, f in enumerate(stages):
        w, lg, lb = stage_weights(s32, i)
        y = r16(F.conv2d(x.float(), r16(tap_weight(w))).double())
        t[f"pd{i}_y"] = y
        g = act(kernel_gather(y, w.shape[0], f), lg, lb)
        if i + 1 < len(stages):
            x = t[f"pd{i}"] = r16(g.double())
        else:
            t["maps"] = F.conv2d(g, s32[D + "linear.weight"], s32[D + "linear.bias"]).double()
    return t
