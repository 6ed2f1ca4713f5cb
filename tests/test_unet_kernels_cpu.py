"""The per-kernel float64 references and error bounds of tests/unet_kernels.py, checked without a GPU: chained, they reproduce
restate.unet_forward; each bound covers an fp16 emulation of its step; each mutation moves the reference by more than the bound."""
import pytest
import torch
import torch.nn.functional as F

from oracle import restate
from tests import unet_kernels as uk
from tests import unet_tiny as ut
from tests.util import apply_overrides, load_card

P = uk.P
S = 128
EMBEDDERS = ["videoseal_1.0", "pixelseal", "chunkyseal", "unet_tiny_yuv_quant"]


def _net(name: str):
    card = ut.tiny_card() if name == "unet_tiny_yuv_quant" else load_card(name)
    card = apply_overrides(card, {"num_blocks": 1})
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, seed=1234)
    return uk.Net(sd, spec), spec, sd


def _inputs(spec, B=1, seed=0):
    g = torch.Generator().manual_seed(seed)
    return torch.rand(B, 3, S, S, generator=g, dtype=torch.float64), torch.randint(0, 2, (B, spec["nbits"]), generator=g)


def _gather16(y: torch.Tensor, C: int) -> torch.Tensor:
    """ups_gather_ln_kernel's pre-norm sum in fp16 emulation: each tap's four-corner mix w11 p11 -> + w10 p10 -> + w01 p01 ->
    + w00 p00 rounded to fp16 after every packed op, the nine taps summed exactly"""
    B, _, h, w = y.shape
    OH, OW = 2 * h, 2 * w

    def src(n, lo):   # rows of the reflect-padded x2 map: (a, b, weight of a)
        u = torch.arange(-1, 2 * n + 1).abs()
        u = torch.where(u >= 2 * n, 4 * n - 2 - u, u)
        i = u // 2
        odd = (u % 2) == 1
        a = torch.where(odd, i, (i - 1).clamp_min(0))
        b = torch.where(odd, (i + 1).clamp_max(n - 1), i)
        return a, b, torch.where(odd, 0.75, 0.25).to(torch.float64)
    ya, yb, wy = src(h, 0)
    xa, xb, wx = src(w, 0)
    r16 = lambda v: v.half().to(torch.float64)
    out = torch.zeros(B, C, OH, OW, dtype=torch.float64)
    for t in range(9):
        r, s = divmod(t, 3)
        yt = y[:, t * C:(t + 1) * C]
        Ya, Yb, Wy = ya[r:r + OH], yb[r:r + OH], wy[r:r + OH][:, None]
        Xa, Xb, Wx = xa[s:s + OW], xb[s:s + OW], wx[s:s + OW][None, :]
        pk = lambda rows, cols: yt[:, :, rows][:, :, :, cols]
        m = r16((1 - Wy) * (1 - Wx) * pk(Yb, Xb))
        m = r16((1 - Wy) * Wx * pk(Yb, Xa) + m)
        m = r16(Wy * (1 - Wx) * pk(Ya, Xb) + m)
        m = r16(Wy * Wx * pk(Ya, Xa) + m)
        out += m
    return out


def _chain(net: uk.Net, imgs, msgs, fp16=False):
    """every debug tap of the embed plan, computed step by step.  fp16=False: float64 through restate's own functions
    (BatchNorm unfolded, upsample_block); fp16=True: the kernels' roundings emulated (BN-folded weights and the skip-scaled
    tap weights rounded to fp16, every fp16 output rounded, the gather's packed mixes rounded)."""
    sd, spec, u = net.sd, net.spec, net.u
    act, norm = u["activation"], u["normalization"]
    r16 = (lambda v: v.half().to(torch.float64)) if fp16 else (lambda v: v)
    taps = {}

    def conv(x, key, i):
        if fp16:
            w, b = net.bn_conv(key, i)
            return F.conv2d(x, r16(w), b, padding=1)
        return restate._norm(sd, f"{key}.double_conv.{i + 1}", norm, F.conv2d(x, sd[f"{key}.double_conv.{i}.weight"], None, padding=1))

    def resblock(name, key, x, out=True):
        taps[name + ".r"] = r16(F.conv2d(x, r16(sd[key + ".res_conv.weight"]), sd[key + ".res_conv.bias"]))
        taps[name + ".h"] = r16(F.relu(conv(x, key, 0)))
        y = F.relu(conv(taps[name + ".h"], key, 3)) + taps[name + ".r"]
        if out:
            taps[name] = r16(y)
        return y

    wf, bf = net.bn_conv(P + "inc", 0)
    wr, br = sd[P + "inc.res_conv.weight"], sd[P + "inc.res_conv.bias"]
    if fp16:   # unet_first_kernel: float32 frames, luma and 2x - 1, float32 weights and sums, fp16 outputs
        f32 = lambda v: v.to(torch.float32)
        x = f32(imgs)
        x = 2 * (0.299 * x[:, 0:1] + 0.587 * x[:, 1:2] + 0.114 * x[:, 2:3]) - 1 if spec["yuv"] else 2 * x - 1
        taps["first_h"] = r16(F.relu(F.conv2d(x, f32(wf), f32(bf), padding=1)).double())
        taps["first_r"] = r16(F.conv2d(x, f32(wr), f32(br)).double())
    else:
        x = uk.first_input(net, imgs)
        taps["first_h"] = F.relu(F.conv2d(x, wf, bf, padding=1))
        taps["first_r"] = F.conv2d(x, wr, br)
    h = F.relu(conv(taps["first_h"], P + "inc", 3)) + taps["first_r"]
    taps["inc"] = r16(h)
    prev = taps["inc"]
    skips = []
    for i in range(net.L - 1):
        taps[f"down{i}_conv"] = r16(F.conv2d(prev, r16(sd[P + f"downs.{i}.down.weight"]), sd[P + f"downs.{i}.down.bias"], stride=2, padding=1))
        prev = resblock(f"down{i}", P + f"downs.{i}.conv", taps[f"down{i}_conv"])
        prev = taps[f"down{i}"]
        skips.append(prev)
    m = restate.msg_embed({P + "msg_processor.msg_embeddings.weight": sd[P + "msg_processor.msg_embeddings.weight"]}, spec, msgs)
    m = r16(m[:, :, None, None].expand(-1, -1, prev.shape[-2], prev.shape[-1]))
    taps["cat"] = torch.cat([prev, m], 1)
    x = taps["cat"]
    for i in range(u["num_blocks"]):
        resblock(f"bott{i}", P + f"bottleneck.model.{i}", x)
        x = taps[f"bott{i}"]
    for j in range(net.L - 1):
        skip = taps["cat"] if j == 0 else skips[net.L - 2 - j]
        xcat = torch.cat([x, skip * uk.SQ], 1)
        U = P + f"ups.{j}.up.upsample_block."
        w = sd[U + "2.weight"]
        cout = w.shape[0]
        if fp16:
            ws = torch.cat([w[:, :x.shape[1]], w[:, x.shape[1]:] * uk.SQ], 1)   # skip scale folded before the rounding
            taps[f"up{j}_taps"] = r16(F.conv2d(torch.cat([x, skip], 1), r16(uk.tap_weight(ws))))
            pre = _gather16(taps[f"up{j}_taps"], cout)
            taps[f"up{j}_conv"] = r16(F.relu(restate.layernorm_cf(pre, sd[U + "3.weight"], sd[U + "3.bias"])))
        else:
            taps[f"up{j}_taps"] = F.conv2d(xcat, uk.tap_weight(w))
            taps[f"up{j}_conv"] = restate.upsample_block(sd, P + f"ups.{j}.up", xcat, act)
        last = j == net.L - 2
        y = resblock(f"up{j}", P + f"ups.{j}.conv", taps[f"up{j}_conv"], out=not last)
        if last:
            o = F.conv2d(y, sd[P + "outc.weight"], sd[P + "outc.bias"])
            taps["delta"] = torch.tanh(o) if u["last_tanh"] else o
        else:
            x = taps[f"up{j}"]
    return taps


@pytest.fixture(scope="module", params=EMBEDDERS)
def case(request):
    torch.manual_seed(0)
    net, spec, sd = _net(request.param)
    imgs, msgs = _inputs(spec)
    return request.param, net, spec, sd, imgs, msgs


@pytest.mark.parametrize("gather_path", [True, False], ids=["tapgemm+gather", "phase"])
def test_chained_references_reproduce_unet_forward(case, gather_path):
    """each step's reference, fed the float64 output of the step before, reproduces that output; the chain ends at
    restate.unet_forward in float64"""
    name, net, spec, sd, imgs, msgs = case
    taps = _chain(net, imgs, msgs)
    # restate.rgb_to_y multiplies by a float32 matrix: hand unet_forward the float64 luma row instead
    ref = restate.unet_forward(net.sd, spec, (uk.first_input(net, imgs) + 1) / 2 if spec["yuv"] else imgs, msgs)
    assert (taps["delta"] - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    worst = 0.0
    for ck in uk.plan_checks(net, lambda n: taps[n], imgs, msgs, lambda n: gather_path and n in taps):
        rel = ((ck.got - ck.ref).abs().max() / ck.ref.abs().max().clamp_min(1e-30)).item()
        worst = max(worst, rel)
        assert rel <= 1e-12, (ck.step, rel)
    print(f"[{name} {'gather' if gather_path else 'phase'}] chained references: max relative difference {worst:.2e}")


def test_phase_decomposition_matches_upsample_block_inside_and_needs_the_border_fix():
    """the phase-folded up-conv (replicate-padded low-resolution 3x3 per output phase) equals upsample_block's conv on every
    pixel but the outermost rows / columns, which up_border_fix_kernel recomputes"""
    g = torch.Generator().manual_seed(3)
    x = torch.randn(2, 64, 16, 16, generator=g, dtype=torch.float64)
    w = torch.randn(16, 64, 3, 3, generator=g, dtype=torch.float64)
    a, b = uk.up_pre(x, w), uk.phase_pre(x, w)
    border = uk.border_mask(32, 32, "cpu")
    d = (a - b).abs()
    assert d[..., ~border].max().item() <= 1e-12 * a.abs().max().item()
    assert (d[..., border].amax(0).amax(0) > 1e-6).float().mean().item() > 0.9


def test_bounds_cover_fp16_emulation(case):
    """every step's bound holds for an emulation of its kernel's fp16 roundings; the ratio shows how loose each bound is"""
    name, net, spec, sd, imgs, msgs = case
    taps = _chain(net, imgs, msgs, fp16=True)
    worst = {}
    for ck in uk.plan_checks(net, lambda n: taps[n], imgs, msgs, lambda n: n in taps):
        r = uk.judge(ck)
        assert not r["nan"] and r["ratio"] <= 1.0, (ck.step, r["ratio"])
        fam = ck.step.split(" ", 1)[1] if " " in ck.step else ck.step
        worst[fam] = max(worst.get(fam, 0.0), r["ratio"])
    for fam, r in sorted(worst.items()):
        print(f"[{name}] emulated err / bound {r:.3f}  {fam}")


def test_mutations_move_the_reference_beyond_the_bound(case):
    """each deliberate defect changes the float64 reference by more than the step's bound (so they are not no-ops), on
    border pixels only / the last frame only where that is the defect's footprint"""
    name, net, spec, sd, imgs, msgs = case
    imgs, msgs = _inputs(spec, B=2, seed=1)
    taps = _chain(net, imgs, msgs)
    seen = set()
    # the phase-folded up-conv exists only for [x 32 | skip 32] -> 16 channels (UNet::check): other levels keep the tap GEMM
    phase_ok = lambda n: taps[n].shape[1] == 9 * 16
    for gather_path in (True, False):
        for ck in uk.plan_checks(net, lambda n: taps[n], imgs, msgs, lambda n: n in taps and (gather_path or not phase_ok(n))):
            for mname, mref, where in ck.mutations:
                v = (mref - ck.ref).abs() > ck.tol
                assert v.any(), (ck.step, mname)
                if where == "border":
                    assert not (v & ~uk.border_mask(v.shape[-2], v.shape[-1], "cpu")).any(), (ck.step, mname)
                elif where == "last_frame":
                    assert not v[:-1].any(), (ck.step, mname)
                seen.add(mname)
    print(f"[{name}] mutations detected: {sorted(seen)}")
    expect = {"pad zero->replicate", "stride-2 phase +1", "skip scale 1", "align_corners=True", "pad reflect->replicate",
              "bit 0 of the last frame flipped", "outc bias dropped", "BT.709 luma" if spec["yuv"] else "R/B swapped"}
    assert expect <= seen, expect - seen
