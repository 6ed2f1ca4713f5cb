"""Per-step float64 references, rounding bounds and mutations of the VAE embedder's plan (csrc/vae.cuh), and an fp16 emulation of the
whole plan: the same data flow as tests/vae_oracle.vae_forward, with every value rounded where the plan rounds it.

Where the plan rounds (`Plan16`):
  - maps it stores in fp16: the encoder conv_in output, every GroupNorm output, every conv / GEMM output of the fp16 stream (conv1,
    nin_shortcut, the resampling convs, qkv, the attention output) and the ResnetBlock / AttnBlock outputs;
  - the weights of every tensor-core conv / GEMM (fp16); the CUDA-core input convs keep fp32 weights;
  - the attention probabilities P (fp16 operand of P v);
  - not rounded to fp16: the latent (fp32), the pre-tanh output and the delta (fp32), and the maps named in `keep32` (the plan keeps
    those in fp32).

The GPU tests judge each step on the exact inputs it read (plan taps); the CPU tests run the same judges on the emulation's inputs, so
that the bounds are exercised, and every mutation has to leave them, without a GPU."""
from typing import Callable, Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from tests import vae_oracle as vo

U16 = 2.0 ** -11      # fp16 unit roundoff
U32 = 2.0 ** -24
SUB = 2.0 ** -25      # half the spacing of fp16 subnormals: the rounding of a value near zero
E, D = vo.E, vo.D


def r16(t: Tensor) -> Tensor:
    return t.to(torch.float16).to(t.dtype)


class Plan16:
    """the plan's roundings for vae_forward_emulated; keep32: tap names (see vae_oracle.vae_forward) the plan keeps in fp32"""

    def __init__(self, keep32=()):
        self.keep32 = set(keep32)

    def store(self, name: str, t: Tensor) -> Tensor:
        return t if any(name.endswith(k) for k in self.keep32) else r16(t)

    @staticmethod
    def weight(w: Tensor) -> Tensor:
        return r16(w)


def _conv(sd, key, x, stride=1, pad=1, tc=True):
    w = sd[key + ".weight"]
    w = r16(w) if tc else w
    return F.conv2d(x, w, sd[key + ".bias"], stride=stride, padding=pad if w.shape[-1] == 3 else 0)


def vae_forward_emulated(sd, v: dict, x: Tensor, msgs: Tensor, plan: Plan16, taps: Optional[dict] = None) -> Tensor:
    """vae_oracle.vae_forward with the plan's roundings (float64 arithmetic between them)"""
    t = taps if taps is not None else {}
    st = plan.store
    L, nr = len(v["ch_mult"]), v["num_res_blocks"]

    def gn(key, h, silu, name):
        return st(name, vo.gn(sd, key, h, silu))

    def res(key, h, tp):
        a1 = t[tp + ".gn1"] = gn(key + ".norm1", h, True, tp + ".gn1")
        c1 = t[tp + ".conv1"] = st(tp + ".conv1", _conv(sd, key + ".conv1", a1))
        a2 = t[tp + ".gn2"] = gn(key + ".norm2", c1, True, tp + ".gn2")
        sc = h
        if key + ".nin_shortcut.weight" in sd:
            sc = t[tp + ".nin"] = st(tp + ".nin", _conv(sd, key + ".nin_shortcut", h))
        out = t[tp + ".out"] = st(tp + ".out", sc + _conv(sd, key + ".conv2", a2))
        return out

    def attn(key, h, tp):
        B, C, hh, ww = h.shape
        n = t[tp + ".gn"] = gn(key + ".norm", h, False, tp + ".gn")
        qkv = [st(tp + ".qkv", _conv(sd, key + "." + m, n)).reshape(B, C, hh * ww) for m in ("q", "k", "v")]
        t[tp + ".qkv"] = torch.cat(qkv, 1).reshape(B, 3 * C, hh, ww)
        q, k, vv = qkv
        p = r16(torch.softmax(torch.bmm(q.permute(0, 2, 1), k) * C ** -0.5, dim=2))
        o = t[tp + ".o"] = st(tp + ".o", torch.bmm(vv, p.permute(0, 2, 1)).reshape(B, C, hh, ww))
        out = t[tp + ".out"] = st(tp + ".out", h + _conv(sd, key + ".proj_out", o))
        return out

    h = t["vae.enc.conv_in"] = st("vae.enc.conv_in", _conv(sd, E + "conv_in", 2 * x - 1, tc=False))
    for l in range(L):
        for i in range(nr):
            h = res(E + f"down.{l}.block.{i}", h, f"vae.enc.d{l}.{i}")
        if l != L - 1:
            h = t[f"vae.enc.down{l}"] = st(f"vae.enc.down{l}", _conv(sd, E + f"down.{l}.downsample.conv", F.pad(h, (0, 1, 0, 1)), 2, 0))
    h = res(E + "mid.block_1", h, "vae.enc.mid1")
    h = attn(E + "mid.attn_1", h, "vae.enc.attn")
    h = res(E + "mid.block_2", h, "vae.enc.mid2")
    a = t["vae.enc.gn_out"] = gn(E + "norm_out", h, True, "vae.enc.gn_out")
    lat = t["vae.latent"] = _conv(sd, E + "conv_out", a)
    ax = vo.aux(sd, msgs, x.dtype)
    z = torch.cat([lat, ax[:, :, None, None].expand(-1, -1, *lat.shape[-2:])], 1)
    h = t["vae.dec.conv_in"] = st("vae.dec.conv_in", _conv(sd, D + "conv_in", z, tc=False))
    h = res(D + "mid.block_1", h, "vae.dec.mid1")
    h = attn(D + "mid.attn_1", h, "vae.dec.attn")
    h = res(D + "mid.block_2", h, "vae.dec.mid2")
    for l in reversed(range(L)):
        for i in range(nr + 1):
            h = res(D + f"up.{l}.block.{i}", h, f"vae.dec.u{l}.{i}")
        if l != 0:
            h = t[f"vae.dec.up{l}"] = st(f"vae.dec.up{l}", _conv(sd, D + f"up.{l}.upsample.conv", F.interpolate(h, scale_factor=2.0)))
    a = t["vae.dec.gn_out"] = gn(D + "norm_out", h, True, "vae.dec.gn_out")
    d = _conv(sd, D + "conv_out", a)
    d = t["delta"] = torch.tanh(d) if v["tanh_out"] else d
    return d


# ---------------------------------------------------------------------------------------------------------------------------------
# per-step references, bounds and mutations


BORDER_ONLY = ("replicate_border",)   # mutations that differ from the reference on the one-pixel border of the map only


def judge(name: str, got: Tensor, ref: Tensor, bound: Tensor, mutants: Dict[str, Tensor]) -> float:
    """|got - ref| <= bound everywhere; every mutant leaves the bound somewhere, and a BORDER_ONLY mutant nowhere but on the border"""
    q = (got - ref).abs() / bound
    r = q.max().item()
    if r > 1.0:
        i = int(q.reshape(-1).argmax())
        raise AssertionError((name, r, "got", got.reshape(-1)[i].item(), "ref", ref.reshape(-1)[i].item(), "bound",
                              bound.reshape(-1)[i].item(), "index", i, "shape", tuple(got.shape)))
    for mname, mut in mutants.items():
        out = (got - mut).abs() > bound
        assert bool(out.any()), (name, mname, ((got - mut).abs() / bound).max().item())
        if mname in BORDER_ONLY:
            inside = int(out[..., 1:-1, 1:-1].sum())
            assert inside == 0, (name, mname, inside, "violations off the one-pixel border")
    return r


def conv_ref(sd, key, inp, stride=1, pad=1, w=None, bias=True):
    ww = sd[key + ".weight"] if w is None else w
    return F.conv2d(inp, ww, sd[key + ".bias"] if bias else None, stride=stride, padding=pad if ww.shape[-1] == 3 else 0)


def conv3_mutants(sd, key, inp, add=0.0, post=None, w=None):
    """mutations of a stride-1 zero-padded 3x3 conv of inp (+ add, then post): the (r, s) taps transposed, and replicate instead of
    zero padding (which moves the one-pixel border only)"""
    ww = sd[key + ".weight"] if w is None else w
    post = post or (lambda u: u)
    return {"taps_transposed": post(add + F.conv2d(inp, ww.transpose(-1, -2), sd[key + ".bias"], padding=1)),
            "replicate_border": post(add + F.conv2d(F.pad(inp, (1, 1, 1, 1), mode="replicate"), ww, sd[key + ".bias"]))}


def nearest_shifted(x: Tensor) -> Tensor:
    """a wrong nearest x2 up-sample: output row / column i reads source (i + 1) // 2, clamped to the map"""
    h, w = x.shape[-2:]
    ri = ((torch.arange(2 * h, device=x.device) + 1) // 2).clamp(max=h - 1)
    ci = ((torch.arange(2 * w, device=x.device) + 1) // 2).clamp(max=w - 1)
    return x[..., ri, :][..., ci]


def conv_bound(sd, key, inp, ref, fp16_w=True, stride=1, pad=1, out16=True):
    """fp16 weights (2^-11 each, tensor-core convs) and fp32 sums (K 2^-24) times sum |x| |w|, plus the output rounding"""
    w = sd[key + ".weight"]
    mag = conv_ref(sd, key, inp.abs(), stride, pad, w.abs(), bias=False) + sd[key + ".bias"].abs().view(1, -1, 1, 1)
    b = ((U16 if fp16_w else 0.0) + w[0].numel() * U32) * mag
    return b + (U16 * ref.abs() + SUB if out16 else 1e-30)


def gn_step(x: Tensor, gamma: Tensor, beta: Tensor, silu: bool, got: Tensor, eps_mutant: bool = False):
    """GroupNorm(16, eps 1e-6) (+ SiLU) of the fp16 map x: statistics in fp64 (exact to far below the bound), the affine
    fmaf(x, rstd gamma, beta - mu rstd gamma) in fp32: a few 2^-24 of |x sc|, |mu sc| and |beta|, SiLU with __expf (relative 2^-21
    on the exponential: |silu'| <= 1.1 times 2^-21 |v|), one fp16 rounding.  Mutations: interleaved groups, GELU for SiLU, eps 1e-5,
    and (statistics of) the neighbouring frame.  eps 1e-5 only moves the result where a group's variance is within a few
    orders of 1e-6, so that mutation is judged on such inputs (eps_mutant)."""
    pre = F.group_norm(x, 16, gamma, beta, 1e-6)
    ref = F.silu(pre) if silu else pre
    act = (lambda u: F.silu(u)) if silu else (lambda u: u)
    B, C = x.shape[:2]
    xg = x.reshape(B, 16, -1)
    rstd = (xg.var(dim=2, unbiased=False) + 1e-6).rsqrt().repeat_interleave(C // 16, 1).view(B, C, 1, 1)
    sc = rstd * gamma.view(1, -1, 1, 1)
    mu = xg.mean(2).repeat_interleave(C // 16, 1).view(B, C, 1, 1)
    # the fp32 rounding of rstd, mu, sc = rstd gamma, mu sc, sh = beta - mu sc and the fma each carry 2^-24 of their operands: near
    # pre = 0 the cancellation in sh leaves |mu sc| and |beta| (not |sh|) as the scale of the absolute error
    mag = (x * sc).abs() + (mu * sc).abs() + beta.abs().view(1, -1, 1, 1)
    bound = U16 * ref.abs() + 4 * U32 * (mag + pre.abs()) + (2 ** -20 * pre.abs() if silu else 0.0) + SUB
    perm = torch.arange(C, device=x.device).view(C // 16, 16).t().reshape(-1)
    inv = torch.argsort(perm)
    # with one channel per group (C = 16) contiguous and interleaved groups are the same groups
    mutants = {"interleaved_groups": act(F.group_norm(x[:, perm], 16, gamma[perm], beta[perm], 1e-6)[:, inv])} if C > 16 else {}
    if eps_mutant:   # only where a group's variance is small enough for eps to matter (small_variance_map, a flat frame)
        mutants["eps_1e-5"] = act(F.group_norm(x, 16, gamma, beta, 1e-5))
    if silu:
        mutants["gelu"] = F.gelu(pre)
    if B > 1:
        mutants["neighbour_frame_stats"] = act(_gn_with_stats(x, torch.roll(x, 1, 0), gamma, beta))
    return got, ref, bound, mutants


def _gn_with_stats(x, s, gamma, beta):
    """x normalised with the group statistics of s"""
    B, C = x.shape[:2]
    sg = s.reshape(B, 16, -1)
    mu = sg.mean(2).repeat_interleave(C // 16, 1).view(B, C, 1, 1)
    rstd = (sg.var(dim=2, unbiased=False) + 1e-6).rsqrt().repeat_interleave(C // 16, 1).view(B, C, 1, 1)
    return (x - mu) * rstd * gamma.view(1, -1, 1, 1) + beta.view(1, -1, 1, 1)


def small_variance_map(B: int, C: int, h: int, seed: int, device=None) -> Tensor:
    """an fp16 map whose groups have variance ~1e-5 around a mean of ~1e-2: there eps 1e-5 against 1e-6 changes rstd by ~40 %,
    far outside the bound, while the fp16 inputs still resolve the spread (spacing 2^-17 near 1e-2)"""
    g = torch.Generator().manual_seed(seed)
    x = 1e-2 * (1 + torch.rand(B, C, 1, 1, generator=g)) + 3e-3 * torch.randn(B, C, h, h, generator=g)
    return r16(x.double()).to(device)


def attn_step(qkv: Tensor, got: Tensor):
    """softmax(q k^T / sqrt(C)) v from the fp16 qkv rows: fp32 scores and exponentials, P rounded to fp16 (2^-11 relative), fp32
    accumulation, one fp16 rounding of the output.  Mutations: no 1/sqrt(C), softmax over queries, k and v swapped, and the last
    tile of 64 keys left out of the softmax and the sum."""
    B, C3, hh, ww = qkv.shape
    C = C3 // 3
    q, k, v = (qkv[:, i * C:(i + 1) * C].reshape(B, C, hh * ww) for i in range(3))
    sc = torch.bmm(q.permute(0, 2, 1), k)
    p = torch.softmax(sc * C ** -0.5, dim=2)

    def of(pp, vv):
        return torch.bmm(vv, pp.permute(0, 2, 1)).reshape(B, C, hh, ww)
    o = of(p, v)
    # P's fp16 rounding and the exp / score error (|s| 2^-22 relative, scores up to |q||k|): 3 x 2^-11 of sum p |v|
    bound = 3 * U16 * of(p, v.abs()) + U16 * o.abs() + SUB
    return got, o, bound, {"no_scale": of(torch.softmax(sc, 2), v), "softmax_over_queries": of(torch.softmax(sc * C ** -0.5, 1), v),
                           "k_v_swapped": of(torch.softmax(torch.bmm(q.permute(0, 2, 1), v) * C ** -0.5, 2), k),
                           "last_key_tile_dropped": of(torch.softmax(sc[:, :, :-64] * C ** -0.5, 2), v[:, :, :-64])}


def steps(sd, v: dict, x: Tensor, msgs: Tensor, t, delta: Tensor, eps_steps=()):
    """every checked step of one plan, judged on the inputs `t[name]` (taps, NCHW float64; a dict or a lazy getter): yields
    (name, got, ref, bound, mutants).  x: the frames' embedder input in [0, 1] ([B, in_ch, S, S]; Y for yuv presets).  eps_steps:
    GroupNorm steps (tap names) whose input has small-variance groups, judged with the eps 1e-5 mutation too"""
    L, nr = len(v["ch_mult"]), v["num_res_blocks"]
    xin = 2 * x - 1
    ref = conv_ref(sd, E + "conv_in", xin)
    yield ("conv_in",) + (t["vae.enc.conv_in"], ref, conv_bound(sd, E + "conv_in", xin, ref, fp16_w=False),
                          conv3_mutants(sd, E + "conv_in", xin))
    # every ResnetBlock: both norms, conv1, the shortcut, conv2 + residual
    blocks = [(E + f"down.{l}.block.{i}", f"vae.enc.d{l}.{i}") for l in range(L) for i in range(nr)]
    blocks += [(E + "mid.block_1", "vae.enc.mid1"), (E + "mid.block_2", "vae.enc.mid2"), (D + "mid.block_1", "vae.dec.mid1"),
               (D + "mid.block_2", "vae.dec.mid2")]
    blocks += [(D + f"up.{l}.block.{i}", f"vae.dec.u{l}.{i}") for l in reversed(range(L)) for i in range(nr + 1)]
    prev = {}
    order = ["vae.enc.conv_in"]
    for l in range(L):
        order += [f"vae.enc.d{l}.{i}.out" for i in range(nr)] + ([f"vae.enc.down{l}"] if l != L - 1 else [])
    order += ["vae.enc.mid1.out", "vae.enc.attn.out", "vae.enc.mid2.out"]
    dorder = ["vae.dec.conv_in", "vae.dec.mid1.out", "vae.dec.attn.out", "vae.dec.mid2.out"]
    for l in reversed(range(L)):
        dorder += [f"vae.dec.u{l}.{i}.out" for i in range(nr + 1)] + ([f"vae.dec.up{l}"] if l != 0 else [])
    for seq in (order, dorder):
        for a, b in zip(seq, seq[1:]):
            prev[b] = a
    for key, tp in blocks:
        xb = t[prev[tp + ".out"]]
        yield (tp + ".gn1",) + gn_step(xb, sd[key + ".norm1.weight"], sd[key + ".norm1.bias"], True, t[tp + ".gn1"],
                                            tp + ".gn1" in eps_steps)
        a1 = t[tp + ".gn1"]
        ref = conv_ref(sd, key + ".conv1", a1)
        yield (tp + ".conv1",) + (t[tp + ".conv1"], ref, conv_bound(sd, key + ".conv1", a1, ref), conv3_mutants(sd, key + ".conv1", a1))
        yield (tp + ".gn2",) + gn_step(t[tp + ".conv1"], sd[key + ".norm2.weight"], sd[key + ".norm2.bias"], True, t[tp + ".gn2"])
        sc = xb
        if key + ".nin_shortcut.weight" in sd:
            ref = conv_ref(sd, key + ".nin_shortcut", xb)
            yield (tp + ".nin",) + (t[tp + ".nin"], ref, conv_bound(sd, key + ".nin_shortcut", xb, ref), {})
            sc = t[tp + ".nin"]
        a2 = t[tp + ".gn2"]
        body = conv_ref(sd, key + ".conv2", a2)
        ref = sc + body
        yield (tp + ".out",) + (t[tp + ".out"], ref, conv_bound(sd, key + ".conv2", a2, ref),
                                {"missing_shortcut": body, **conv3_mutants(sd, key + ".conv2", a2, add=sc)})
    # resampling
    for l in range(L - 1):
        xd = t[f"vae.enc.d{l}.{nr - 1}.out"]
        xp = F.pad(xd, (0, 1, 0, 1))
        ref = conv_ref(sd, E + f"down.{l}.downsample.conv", xp, 2, 0)
        wd = sd[E + f"down.{l}.downsample.conv.weight"]
        yield (f"down{l}",) + (t[f"vae.enc.down{l}"], ref, conv_bound(sd, E + f"down.{l}.downsample.conv", xp, ref, stride=2, pad=0),
                           {"symmetric_pad": conv_ref(sd, E + f"down.{l}.downsample.conv", xd, 2, 1),
                            "taps_transposed": conv_ref(sd, E + f"down.{l}.downsample.conv", xp, 2, 0, w=wd.transpose(-1, -2))})
    for l in range(1, L):
        xu = t[f"vae.dec.u{l}.{nr}.out"]
        up = F.interpolate(xu, scale_factor=2.0, mode="nearest")
        ref = conv_ref(sd, D + f"up.{l}.upsample.conv", up)
        yield (f"up{l}",) + (t[f"vae.dec.up{l}"], ref, conv_bound(sd, D + f"up.{l}.upsample.conv", up, ref),
                         {"bilinear": conv_ref(sd, D + f"up.{l}.upsample.conv",
                                               F.interpolate(xu, scale_factor=2.0, mode="bilinear", align_corners=False)),
                          "nearest_shifted": conv_ref(sd, D + f"up.{l}.upsample.conv", nearest_shifted(xu)),
                          **conv3_mutants(sd, D + f"up.{l}.upsample.conv", up)})
    # the AttnBlocks: norm (no activation), qkv, attention, proj_out + residual
    for P, tp, xin_name in ((E, "vae.enc.attn", "vae.enc.mid1.out"), (D, "vae.dec.attn", "vae.dec.mid1.out")):
        key = P + "mid.attn_1"
        xa = t[xin_name]
        yield (tp + ".gn",) + gn_step(xa, sd[key + ".norm.weight"], sd[key + ".norm.bias"], False, t[tp + ".gn"])
        n = t[tp + ".gn"]
        w3 = torch.cat([sd[key + "." + m + ".weight"] for m in ("q", "k", "v")])
        b3 = torch.cat([sd[key + "." + m + ".bias"] for m in ("q", "k", "v")])
        qref = F.conv2d(n, w3, b3)
        qb = (U16 + n.shape[1] * U32) * (F.conv2d(n.abs(), w3.abs()) + b3.abs().view(1, -1, 1, 1)) + U16 * qref.abs() + SUB
        yield (tp + ".qkv",) + (t[tp + ".qkv"], qref, qb, {})
        yield (tp + ".attn",) + attn_step(t[tp + ".qkv"], t[tp + ".o"])
        o = t[tp + ".o"]
        body = conv_ref(sd, key + ".proj_out", o)
        ref = xa + body
        yield (tp + ".out",) + (t[tp + ".out"], ref, conv_bound(sd, key + ".proj_out", o, ref), {"missing_residual": body})
    # latent (fp32 output), the decoder conv_in with the message planes' border cases, the output conv + tanh
    for P, tp in ((E, "vae.enc"), (D, "vae.dec")):
        key = P + "norm_out"
        src = t["vae.enc.mid2.out"] if P == E else t[f"vae.dec.u0.{nr}.out"]
        yield (tp + ".gn_out",) + gn_step(src, sd[key + ".weight"], sd[key + ".bias"], True, t[tp + ".gn_out"])
    ga = t["vae.enc.gn_out"]
    ref = conv_ref(sd, E + "conv_out", ga)
    yield ("latent",) + (t["vae.latent"], ref, conv_bound(sd, E + "conv_out", ga, ref, out16=False), conv3_mutants(sd, E + "conv_out", ga))
    lat = t["vae.latent"]
    K = msgs.shape[1]
    ax = vo.aux(sd, msgs.long(), torch.float64)
    z = lat.shape[1]
    zfull = torch.cat([lat, ax[:, :, None, None].expand(-1, -1, *lat.shape[-2:])], 1)
    ref = conv_ref(sd, D + "conv_in", zfull)
    wl = sd[D + "conv_in.weight"]
    interior = conv_ref(sd, D + "conv_in", lat, w=wl[:, :z], bias=False) + sd[D + "conv_in.bias"].view(1, -1, 1, 1) + \
        torch.einsum("bj,nj->bn", ax, wl[:, z:].sum(dim=(2, 3)))[:, :, None, None]
    pm = (2 * msgs.long() - 1).double()
    pm_planes = torch.cat([lat, pm[:, :, None, None].expand(-1, -1, *lat.shape[-2:])], 1)
    yield ("dec.conv_in",) + (t["vae.dec.conv_in"], ref, conv_bound(sd, D + "conv_in", zfull, ref, fp16_w=False),
                          {"border_as_interior": interior,
                           "pm1_planes": F.conv2d(pm_planes[:, :z + K], wl[:, :z + K], sd[D + "conv_in.bias"], padding=1)})
    go = t["vae.dec.gn_out"]
    pre = conv_ref(sd, D + "conv_out", go)
    ob = conv_bound(sd, D + "conv_out", go, pre, out16=False) + 4 * U32
    fin = torch.tanh(pre) if v["tanh_out"] else pre
    yield ("out",) + (delta, fin, ob, {**({"tanh_ignored": pre} if v["tanh_out"] else {}),
                                       **conv3_mutants(sd, D + "conv_out", go, post=torch.tanh if v["tanh_out"] else None)})


def run_steps(sd, v, x, msgs, t, delta, log: Optional[Callable[[str], None]] = None, eps_steps=()) -> Dict[str, float]:
    """judge every step; returns name -> err / bound"""
    res = {}
    for name, got, ref, bound, mut in steps(sd, v, x, msgs, t, delta, eps_steps):
        res[name] = judge(name, got, ref, bound, mut)
        if log:
            log(f"  {name:22s} err/bound {res[name]:.3f} " +
                " ".join(f"{k}:rejected" + (" (border only)" if k in BORDER_ONLY else "") for k in mut))
    return res
