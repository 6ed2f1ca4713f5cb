"""Per-step float64 references, bounds and mutations of the HiDDeN plans (csrc/hidden.cuh), shared by the CPU test (on an fp16
emulation of every step) and the GPU test (on the plan's own taps).

Each step is judged on its own input as the plan stored it: ref = the step in float64, err / tol <= 1 on every element.  Bounds:
  conv (3 -> 64 on CUDA cores, fp32 weights)         2^-11 |ref| + 1e-5 (|W| * |x|) + 1e-6      (fp16 output; fp32 sums)
  conv (64 -> 64, tensor cores, fp16 weights)          2^-11 |ref| + 2^-10 (|W| * |x|) + 1e-6     (fp16 weights and output)
  GroupNorm partials (fp64 sums of fp16 values)        1e-12 (1 + |ref|)
  GroupNorm apply + activation (fp16 out)              2^-11 |ref| + 1e-5 (1 + |ref|)            (fp32 scale / shift, GELU polynomial)
  message table, pooled mean, linear (fp32)            1e-5 (1 + |ref|)
  image columns + table (fp16 out)                     2^-11 |ref| + 1e-5 (1 + |W| * |x|)
  norm + act + final_layer (+ tanh) (fp32 out)         1e-4 (1 + |ref|)
Every mutation below must leave the bound of each step that has it:
  interleaved  GroupNorm groups of channels c = g (mod 8) instead of the contiguous [8g, 8g + 8)      stats, apply, +outc, +pool
  frame0       the last frame normalised with frame 0's statistics                                    apply, +outc, +pool
  msg01        messages as {0, 1} planes instead of 2 m - 1                                           table, image columns + table
  order        the concat read as [enc | m | x] instead of [m | enc | x]                              table, concat conv
  border       the top-left corner case given the interior's table row                                table, image columns + table
  x01          the image as x instead of 2 x - 1                                                      first conv, image columns
  tanh         tanh dropped (last_tanh) or added (no last_tanh)                                       +outc
  nobias       the linear head's bias dropped                                                         linear
Dropped: unbiased variance.  n / (n - 1) - 1 = 1.9e-6 for a group of 8 x 256^2 values (7.6e-6 at 128^2, the smallest map), far
below the fp16 output's 2^-11 = 4.9e-4: no fp16 map can show it.
"""
from typing import Dict

import torch
import torch.nn.functional as F

U = 2.0 ** -11
TILE = 2048


def folded(sd, key, norm):
    """conv weight and bias with an eval BatchNorm folded in (float64), or the conv's own for GroupNorm"""
    w, b = sd[key + ".layers.0.weight"].double(), sd[key + ".layers.0.bias"].double()
    if norm == "batch":
        s = sd[key + ".layers.1.weight"].double() / torch.sqrt(sd[key + ".layers.1.running_var"].double() + 1e-5)
        return w * s[:, None, None, None], (b - sd[key + ".layers.1.running_mean"].double()) * s + sd[key + ".layers.1.bias"].double()
    return w, b


def act(kind, z):
    return F.relu(z) if kind == "relu" else F.gelu(z)


def _perm(interleaved):
    """channel order that puts each GroupNorm group's channels next to each other"""
    return torch.arange(64).reshape(8, 8).t().reshape(-1) if interleaved else torch.arange(64)


def gn(sd, key, y, interleaved=False, frame0=False):
    p = _perm(interleaved)
    inv = torch.argsort(p)
    z = F.group_norm(y[:, p], 8, None, None, 1e-5)[:, inv]
    if frame0:   # the last frame with frame 0's statistics
        yy = torch.cat([y[:1], y[-1:]])[:, p]
        g = yy.reshape(2, 8, -1)
        mu, var = g[0].mean(dim=1), g[0].var(dim=1, unbiased=False)
        last = (g[1] - mu[:, None]) / torch.sqrt(var[:, None] + 1e-5)
        z = z.clone()
        z[-1] = last.reshape(yy.shape[1:])[inv]
    return z * sd[key + ".layers.1.weight"].double()[:, None, None] + sd[key + ".layers.1.bias"].double()[:, None, None]


def norm_act(sd, key, h, y, mut=None):
    if h["normalization"] == "batch":
        return act(h["activation"], y)
    return act(h["activation"], gn(sd, key, y, mut == "interleaved", mut == "frame0"))


def stats(pre, interleaved=False):
    """[B, tiles, 8, 2] fp64 (sum, sum of squares) per tile of TILE pixels and group"""
    B = pre.shape[0]
    pix = pre.permute(0, 2, 3, 1)[..., _perm(interleaved)].reshape(B, -1, TILE, 8, 8)
    return torch.stack([pix.sum(dim=(2, 4)), (pix * pix).sum(dim=(2, 4))], dim=-1)


def _conv_tol(ref, mag, tc):
    return U * ref.abs() + (2 * U if tc else 1e-5) * mag + 1e-6


def _msg_part(w, m, K, S, planes01=False, order=False):
    planes = (m.double() if planes01 else 2 * m.double() - 1)[:, :, None, None].expand(-1, -1, S, S)
    wm = w[:, 64:64 + K] if order else w[:, :K]
    return F.conv2d(planes, wm, None, padding=1)


def _table(mp, S, border=False):
    rows = [0, 1, S - 1]
    t = torch.stack([mp[:, :, r, c] for r in rows for c in rows], dim=1)
    if border:
        t = t.clone()
        t[:, 0] = t[:, 4]
    return t


class Judge:
    """collects err / tol per step and, per mutation, the smallest err / tol over the steps that have it (must exceed 1)"""

    def __init__(self):
        self.worst: Dict[str, float] = {}
        self.mutations: Dict[str, float] = {}

    def __call__(self, step, got, ref, tol, muts=None):
        got = got.double()
        r = ((got - ref).abs() / tol).max().item()
        self.worst[step] = max(self.worst.get(step, 0.0), r)
        assert r <= 1.0, (step, r)
        for name, mref in (muts or {}).items():
            rm = ((got - mref).abs() / tol).max().item()
            key = f"{name}@{step}"
            self.mutations[key] = min(self.mutations.get(key, float("inf")), rm)
            assert rm > 1.0, (key, rm)


def check_encoder(sd, spec, x, m, taps, J: Judge, early: bool = True):
    """taps (NCHW float tensors; stats [B, tiles, 8, 2] fp64; msg_table [B, 9, 64]; delta [B, 3, S, S]) of one embed plan"""
    h, K = spec["hidden_encoder"], spec["nbits"]
    P = "embedder.hidden_encoder."
    S = x.shape[-1]
    xin = 2 * x.double() - 1
    grp = h["normalization"] == "group"
    nl = h["num_blocks"]
    if early:
        _check_early(sd, h, P + "conv_bns.", "henc.", x, taps, J)
    key = P + "after_concat_layer"
    w, b = folded(sd, key, h["normalization"])
    wx = w[:, K + 64:]
    mp = _msg_part(w, m, K, S)
    J("msg_table", taps["henc.msg_table"], _table(mp, S), 1e-5 * (1 + _table(mp, S).abs()),
      {"msg01": _table(_msg_part(w, m, K, S, planes01=True), S), "order": _table(_msg_part(w, m, K, S, order=True), S),
       "border": _table(mp, S, border=True)})

    def cx_ref(xx, mpp, border=False):
        full = F.conv2d(xx, wx, None, padding=1) + mpp
        if border:
            full = full.clone()
            full[:, :, 0, 0] = full[:, :, 0, 0] - mpp[:, :, 0, 0] + mpp[:, :, 1, 1]
        return full
    ref = cx_ref(xin, mp)
    J("concat_x+msg", taps["henc.cat_x"], ref, U * ref.abs() + 1e-5 * (1 + F.conv2d(xin.abs(), wx.abs(), None, padding=1)),
      {"x01": cx_ref(x.double(), mp), "msg01": cx_ref(xin, _msg_part(w, m, K, S, planes01=True)), "border": cx_ref(xin, mp, True)})
    enc, cx = taps[f"henc.{nl - 1}"].double(), taps["henc.cat_x"].double()
    ref = F.conv2d(enc, w[:, K:K + 64], b, padding=1) + cx
    mag = F.conv2d(enc.abs(), w[:, K:K + 64].abs(), b.abs(), padding=1) + cx.abs()
    J("concat_conv", taps["henc.cat.pre"], ref, _conv_tol(ref, mag, True),
      {"order": F.conv2d(enc, w[:, :64], b, padding=1) + cx})
    pre = taps["henc.cat.pre"].double()
    if grp:
        J("gn_stats", taps["henc.cat.stats"], stats(pre), 1e-12 * (1 + stats(pre).abs()), {"interleaved": stats(pre, True)})

    def outc(mut=None):
        y = F.conv2d(norm_act(sd, key, h, pre, mut), sd[P + "final_layer.weight"].double(), sd[P + "final_layer.bias"].double())
        tanh = h["last_tanh"] != (mut == "tanh")
        return torch.tanh(y) if tanh else y
    ref = outc()
    muts = {"tanh": outc("tanh")}
    if grp:
        muts.update(interleaved=outc("interleaved"), frame0=outc("frame0"))
    J("norm_act+outc", taps["delta"], ref, 1e-4 * (1 + ref.abs()), muts)


def check_decoder(sd, spec, x, taps, logits, J: Judge, early: bool = True):
    h, K = spec["hidden_decoder"], spec["nbits"]
    P = "detector.hidden_decoder."
    grp = h["normalization"] == "group"
    L = h["num_blocks"]
    if early:
        _check_early(sd, h, P + "layers.", "hdec.", x, taps, J)
    key = P + f"layers.{L}"
    w, b = folded(sd, key, h["normalization"])
    prev = taps[f"hdec.{L - 1}"].double()
    ref = F.conv2d(prev, w, b, padding=1)
    J("conv64", taps[f"hdec.{L}.pre"], ref, _conv_tol(ref, F.conv2d(prev.abs(), w.abs(), b.abs(), padding=1), True))
    pre = taps[f"hdec.{L}.pre"].double()
    if grp:
        J("gn_stats", taps[f"hdec.{L}.stats"], stats(pre), 1e-12 * (1 + stats(pre).abs()), {"interleaved": stats(pre, True)})
    ref = norm_act(sd, key, h, pre).mean(dim=(2, 3))
    muts = {"interleaved": norm_act(sd, key, h, pre, "interleaved").mean(dim=(2, 3)),
            "frame0": norm_act(sd, key, h, pre, "frame0").mean(dim=(2, 3))} if grp else {}
    J("norm_act+pool", taps["head_pooled"], ref, 1e-5 * (1 + ref.abs()), muts)
    pooled = taps["head_pooled"].double()
    lw, lb = sd[P + "linear.weight"].double(), sd[P + "linear.bias"].double()
    ref = F.linear(pooled, lw, lb)
    J("linear", logits, ref, 1e-5 * (1 + ref.abs()), {"nobias": F.linear(pooled, lw)})


def _check_early(sd, h, stem, tp, x, taps, J):
    """the first layer (3 -> 64 on CUDA cores), its GroupNorm partials and apply, and the second layer's 64 -> 64 conv, on the copies
    the debug seam keeps"""
    grp = h["normalization"] == "group"
    xin = 2 * x.double() - 1
    for i in (0, 1):
        key = stem + str(i)
        w, b = folded(sd, key, h["normalization"])
        inp = xin if i == 0 else taps[tp + "0"].double()

        def conv(xx):
            y = F.conv2d(xx, w, b, padding=1)
            return y if grp else act(h["activation"], y)
        ref = conv(inp)
        tol = _conv_tol(ref, F.conv2d(inp.abs(), w.abs(), b.abs(), padding=1), i > 0)
        muts = {"x01": conv(x.double())} if i == 0 else {}
        J("conv3-64" if i == 0 else "conv64", taps[tp + str(i) + (".pre" if grp else "")], ref, tol, muts)
        if grp:
            pre = taps[tp + str(i) + ".pre"].double()
            J("gn_stats", taps[tp + str(i) + ".stats"], stats(pre), 1e-12 * (1 + stats(pre).abs()), {"interleaved": stats(pre, True)})
            ref = norm_act(sd, key, h, pre)
            J("gn_apply", taps[tp + str(i)], ref, U * ref.abs() + 1e-5 * (1 + ref.abs()),
              {"interleaved": norm_act(sd, key, h, pre, "interleaved"), "frame0": norm_act(sd, key, h, pre, "frame0")})


# ------------------------------------------------------------------------------------------------- fp16 emulation (CPU test)
def _h(t):
    return t.to(torch.float16).to(torch.float32)


def _emu_stats(pre32):
    return stats(pre32.double())


def _emu_norm_act(sd, key, h, pre32):
    """the kernel's arithmetic: fp64 statistics, fp32 scale / shift, fp32 activation"""
    if h["normalization"] == "batch":
        return act(h["activation"], pre32)
    st = _emu_stats(pre32).sum(dim=1)   # [B, 8, 2]
    n = pre32.shape[-1] * pre32.shape[-2] * 8
    mu = st[..., 0] / n
    var = (st[..., 1] / n - mu * mu).clamp(min=0)
    rstd = (1.0 / torch.sqrt(var + 1e-5)).float()
    g, bb = sd[key + ".layers.1.weight"].float(), sd[key + ".layers.1.bias"].float()
    scale = rstd.repeat_interleave(8, dim=1) * g
    shift = bb - mu.float().repeat_interleave(8, dim=1) * scale
    return act(h["activation"], pre32 * scale[:, :, None, None] + shift[:, :, None, None])


def emulate(sd, spec, x, m, decoder: bool):
    """taps of one plan as the kernels compute them: fp16 maps and tensor-core weights, fp32 arithmetic, fp64 statistics"""
    h = spec["hidden_decoder" if decoder else "hidden_encoder"]
    stem, tp = ("detector.hidden_decoder.layers.", "hdec.") if decoder else ("embedder.hidden_encoder.conv_bns.", "henc.")
    grp = h["normalization"] == "group"
    nl = h["num_blocks"] + (1 if decoder else 0)
    taps = {}
    xin = (2 * x - 1).float()
    cur = None
    for i in range(nl):
        key = stem + str(i)
        w, b = folded(sd, key, h["normalization"])
        last = decoder and i == nl - 1
        y = F.conv2d(xin if i == 0 else cur, (w.float() if i == 0 else _h(w.float())), b.float(), padding=1)
        if grp or last:
            pre = _h(y)
            taps[f"{tp}{i}.pre"] = pre
            if grp:
                taps[f"{tp}{i}.stats"] = _emu_stats(pre)
            if last:
                taps["head_pooled"] = _emu_norm_act(sd, key, h, pre).mean(dim=(2, 3))
                P = "detector.hidden_decoder."
                taps["logits"] = F.linear(taps["head_pooled"], sd[P + "linear.weight"].float(), sd[P + "linear.bias"].float())
                return taps
            cur = _h(_emu_norm_act(sd, key, h, pre))
        else:
            cur = _h(act(h["activation"], y))
        taps[f"{tp}{i}"] = cur
    K, S = spec["nbits"], x.shape[-1]
    P = "embedder.hidden_encoder."
    key = P + "after_concat_layer"
    w, b = folded(sd, key, h["normalization"])
    mp = _msg_part(w, m, K, S).float()
    taps["henc.msg_table"] = _table(mp, S)
    tab_map = torch.empty_like(mp)
    rows = [0, 1, S - 1]
    for ri, r in enumerate(rows):
        for ci, c in enumerate(rows):
            rs = slice(r, r + 1) if ri != 1 else slice(1, S - 1)
            cs = slice(c, c + 1) if ci != 1 else slice(1, S - 1)
            tab_map[:, :, rs, cs] = taps["henc.msg_table"][:, ri * 3 + ci][:, :, None, None]
    cx = _h(F.conv2d(xin, w[:, K + 64:].float(), None, padding=1) + tab_map)
    taps["henc.cat_x"] = cx
    pre = _h(F.conv2d(cur, _h(w[:, K:K + 64].float()), b.float(), padding=1) + cx)
    taps["henc.cat.pre"] = pre
    if grp:
        taps["henc.cat.stats"] = _emu_stats(pre)
    d = F.conv2d(_emu_norm_act(sd, key, h, pre), sd[P + "final_layer.weight"].float(), sd[P + "final_layer.bias"].float())
    taps["delta"] = torch.tanh(d) if h["last_tanh"] else d
    return taps
