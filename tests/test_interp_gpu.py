"""Every interpolation mode at the two resize sites, on the GPU, against float64 references (the companion of test_fullres_gpu.py,
whose helpers this imports):

  a. the resize to processing size (`x_res` tap) for every (mode, align_corners, antialias), with the compiled variant pinned;
  b. the delta up-scale inside the blend kernels (imgs_w / preds_w from the `delta` tap), including the 4-tap (bicubic) variants;
  c. end to end against tests/golden/interp.pt, written by tests/make_golden_interp.py from the unmodified reference;
  d. no dict, or the default dict, gives what the mode bits 0 give, bit for bit.

Float64 operators.  Anti-aliased and area resizes: F.interpolate of a double identity.  Nearest: fp32 F.interpolate of the identity
(0 / 1 weights: exact).  Plain bilinear with align_corners=True and plain bicubic: ATen's fp32 source coordinate and fp32 weights
(emulated in numpy float32, in the order the library's tables evaluate them), applied in float64; test_interp_cpu.py holds the
tables to ATen itself.
"""
import functools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.test_e2e_gpu import LOGIT_RTOL, PIX_TOL, logits_ok
from tests.test_fullres_gpu import (BAND_FRAC, EPS, JND_CFG, TOL_IW, TOL_PW, _embed_raw, _min_err, configured, dispatch, frames,
                                    hmap_candidates, pair, video_deltas64)  # noqa: F401 - pair is a fixture
from videoseal_b200 import _lib

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CL, LR = _lib.FLAG_CLAMP, _lib.FLAG_LOWRES_ATTN
# (mode, align_corners, antialias) as the reference's dicts give them (None: not in the dict)
MODES = [("bilinear", False, True), ("bilinear", False, False), ("bilinear", True, True), ("bilinear", True, False),
         ("bicubic", False, True), ("bicubic", False, False), ("bicubic", True, True), ("bicubic", True, False),
         ("nearest", None, False), ("area", None, False)]


def idict(m):
    d = {"mode": m[0], "antialias": m[2]}
    if m[1] is not None:
        d["align_corners"] = m[1]
    return d


def mflags(m):
    return (_lib.RESIZE_MODES[m[0]] << _lib.FLAG_RESIZE_MODE_SHIFT) | (_lib.FLAG_RESIZE_ALIGN_CORNERS if m[1] else 0) | \
        (0 if m[2] else _lib.FLAG_RESIZE_NO_AA)


def _mid(m):
    return f"{m[0]}-ac{int(bool(m[1]))}-aa{int(m[2])}"


def _keys32(t):
    """Keys cubic coefficients (A = -0.75) of fp32 t in fp32, evaluated as aten/src/ATen/native/UpSample.h writes them"""
    f = np.float32
    A = f(-0.75)

    def c1(x):
        return ((A + f(2)) * x - (A + f(3))) * x * x + f(1)

    def c2(x):
        return ((A * x - f(5) * A) * x + f(8) * A) * x - f(4) * A
    return [c2(t + f(1)), c1(t), c1(f(1) - t), c2(f(1) - t + f(1))]


@functools.lru_cache(maxsize=None)
def op64(n_in: int, n_out: int, m: tuple) -> torch.Tensor:
    """[n_out, n_in] float64 operator of F.interpolate(size=n_out, **idict(m)) along one axis"""
    mode, ac, aa = m
    if n_in == n_out:
        return torch.eye(n_in, dtype=torch.float64)
    if mode == "bilinear" and not ac and not (aa and n_in > n_out):
        from tests.test_fullres_gpu import resample_matrix          # plain half-pixel bilinear (the parent's reference)
        return resample_matrix(n_in, n_out, False)
    if aa or mode in ("area", "nearest") or (mode == "bilinear" and not ac):
        dt = torch.float32 if mode == "nearest" else torch.float64
        eye = torch.eye(n_in, dtype=dt).reshape(n_in, 1, 1, n_in)
        kw = {} if ac is None else {"align_corners": ac}
        return F.interpolate(eye, size=(1, n_out), mode=mode, antialias=aa, **kw).reshape(n_in, n_out).t().double().contiguous()
    f = np.float32
    scale = f(n_in - 1) / f(n_out - 1) if ac else f(n_in) / f(n_out)
    opm = np.zeros((n_out, n_in))
    for i in range(n_out):
        src = f(scale * f(i)) if ac else f(np.float64(scale) * (i + 0.5) - 0.5)     # one fused multiply-add
        x0 = min(int(np.floor(src)), n_in - 1)
        t = min(max(f(src - f(x0)), f(0)), f(1))
        if mode == "bilinear":
            x1 = x0 + (1 if x0 < n_in - 1 else 0)
            opm[i, x0] += np.float64(f(1) - t)
            opm[i, x1] += np.float64(t) if x1 != x0 else 0.0
            continue
        w = np.zeros(n_in, dtype=np.float32)
        for j, c in enumerate(_keys32(t)):
            w[max(min(x0 - 1 + j, n_in - 1), 0)] += c
        opm[i] = w
    return torch.from_numpy(opm)


def resize64(x: torch.Tensor, oh: int, ow: int, m, absolute=False) -> torch.Tensor:
    my, mx = op64(x.shape[-2], oh, m), op64(x.shape[-1], ow, m)
    if absolute:
        my, mx = my.abs(), mx.abs()
    return torch.matmul(torch.matmul(my, x.double()), mx.t())


def taps_and_sum(n_in, n_out, m):
    op = op64(n_in, n_out, m)
    return int((op != 0).sum(1).max()), float(op.abs().sum(1).max())


# ----------------------------------------------------------------------------------------------------- a. resize
# (W, H): 1080p, 4K, 854 x 480 and 1366 x 768 (4-byte cp.async path), 176 x 144 (up-scale); S = 256
RESIZE_GEOMS = [(1920, 1080), (3840, 2160), (854, 480), (1366, 768), (176, 144)]


def _want_mt(maxt):
    return 2 if maxt <= 2 else (8 if maxt <= 8 else 0)


@pytest.mark.parametrize("m", MODES, ids=_mid)
@pytest.mark.parametrize("W,H", RESIZE_GEOMS, ids=lambda v: str(v))
def test_resize_matches_float64(pair, W, H, m):
    """x_res of detect against the float64 resize.  Bound: (taps_x + taps_y + 2) * 2^-23 * sum|w_x| * sum|w_y| (one rounding per
    tap and pass; the Keys and cubic filters have negative lobes).  The resize variant (MT from the table's width) is pinned."""
    x = frames(2, H, W, seed=W + H)
    with configured(pair) as model:
        model.detect((1 - x).cuda(), is_video=True, interpolation=idict(m))
        model.detect(x.cuda(), is_video=True, interpolation=idict(m))
        rs, _ = dispatch(model)
        got = model.debug_tensor("x_res").double()
    tx, sx = taps_and_sum(W, 256, m)
    ty, sy = taps_and_sum(H, 256, m)
    buf = np.zeros(256 * 64, dtype=np.float32)
    idx = np.zeros(256, dtype=np.int32)
    maxt = _lib.lib().vsb_debug_resample_table2(W, 256, _lib.RESIZE_MODES[m[0]], int(bool(m[1])), int(m[2]), idx.ctypes.data,
                                                idx.ctypes.data, buf.ctypes.data, buf.size)
    assert rs[0] == _want_mt(maxt) and rs[2] == (1 if W % 4 == 0 else 0) and rs[4] == 256, rs
    ref = resize64(x, 256, 256, m)
    tol = (tx + ty + 2) * EPS * sx * sy
    err = (got - ref).abs().max().item()
    print(f"[resize] {_mid(m)} {W}x{H}: variant {rs}, max|x_res - float64| = {err:.2e} (bound {tol:.2e})")
    assert err <= tol, (err, tol)


# ----------------------------------------------------------------------------------------------------- b. blend
BIC = ("bicubic", False, True)
BICN = ("bicubic", False, False)
# (id, mode, jnd, W, H, F, step, video mode, chunk, flags, expected blend dispatch (kernel, VEC, FASTUP, CD, JIN))
BLEND_CASES = [
    ("bicubic-aa-1080p", BIC, "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 4, 1, 1)),
    ("bicubic-noaa-1080p", BICN, "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 4, 1, 1)),
    ("bicubic-aa-4k", BIC, "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, CL, (3, 4, 4, 1, 1)),
    ("bicubic-noaa-4k-noclamp", BICN, "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, 0, (3, 4, 4, 1, 1)),
    ("bicubic-ac-aa-1080p", ("bicubic", True, True), "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 4, 1, 1)),
    ("bicubic-ac-noaa-4k", ("bicubic", True, False), "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, CL, (3, 4, 4, 1, 1)),
    ("bilinear-ac-aa-1080p", ("bilinear", True, True), "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("bilinear-ac-noaa-4k", ("bilinear", True, False), "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("nearest-1080p", ("nearest", None, False), "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("nearest-4k", ("nearest", None, False), "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("area-1080p", ("area", None, False), "jnd_1_1", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("area-4k", ("area", None, False), "jnd_1_1", 3840, 2160, 1, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("bicubic-jnd_3_3-1080p", BIC, "jnd_3_3", 1920, 1080, 2, 1, "repeat", 32, CL, (3, 4, 4, 1, 3)),
    ("bicubic-scalar-854x480", BIC, "jnd_1_1", 854, 480, 2, 1, "repeat", 32, CL, (2, 1, 4, 1, 1)),
    ("bicubic-scalar-1366x768-jnd_3_1", BICN, "jnd_3_1", 1366, 768, 2, 1, "repeat", 32, CL, (2, 1, 4, 1, 3)),
    ("bicubic-small-176x144", BIC, "jnd_1_1", 176, 144, 2, 1, "repeat", 32, CL, (2, 4, 0, 1, 1)),
    ("bicubic-lowres-720p", BIC, "jnd_1_1", 1280, 720, 2, 1, "repeat", 32, CL | LR, (3, 4, 4, 1, 1)),
    ("bicubic-lowres-720p-jnd_3_3", BIC, "jnd_3_3", 1280, 720, 2, 1, "repeat", 32, CL | LR, (3, 4, 4, 3, 1)),
    ("bicubic-repeat-1080p", BIC, "jnd_1_1", 1920, 1080, 10, 4, "repeat", 2, CL, (3, 4, 4, 1, 1)),
    ("bicubic-interpolate-1080p", BIC, "jnd_1_1", 1920, 1080, 14, 4, "interpolate", 2, CL, (3, 4, 4, 1, 1)),
    ("bicubic-interpolate-1366x768", BICN, "jnd_1_1", 1366, 768, 14, 4, "interpolate", 2, CL, (2, 1, 4, 1, 1)),
]


@pytest.mark.parametrize("case", BLEND_CASES, ids=[c[0] for c in BLEND_CASES])
def test_blend_matches_float64(pair, case):
    """imgs_w and preds_w against the float64 blend of (frames, delta tap), as test_fullres_gpu.py::test_blend_matches_float64 with
    the delta up-scaled by the mode's operator; the bounds TOL_PW / TOL_IW scale with sum|w_x| * sum|w_y|.  With
    lowres_attenuation a band pixel's two branches span an interval at processing size; its up-scale is bounded through |weights|
    (bicubic weights can be negative)."""
    name, m, jnd, W, H, F_, step, mode, chunk, flags, want = case
    jin, jout = JND_CFG[jnd]
    lowres = bool(flags & LR)
    pc = max(1, jout)
    x = frames(F_, H, W, seed=BLEND_CASES.index(case) + 100)
    sx, sy = taps_and_sum(256, W, m)[1], taps_and_sum(256, H, m)[1]
    tol_pw, tol_iw = TOL_PW * sx * sy, TOL_IW * sx * sy
    with configured(pair, jnd=jnd) as model:
        iw, pw, dkeys = _embed_raw(model, x.cuda(), step, mode, chunk, flags | mflags(m), pc)
        assert dispatch(model)[1] == want, dispatch(model)
        assert not torch.isnan(iw).any() and not torch.isnan(pw).any(), "an output pixel was not written"
        dS = video_deltas64(dkeys, F_, step, mode, chunk)
        x64 = x.double()
        if not lowres:
            cands, nband, npx = hmap_candidates(x, jin, jout)
            dup = resize64(dS, H, W, m)
            e_pw = e_iw = None
            for h in cands:
                p = h * dup
                i = x64 + 0.2 * p
                if flags & CL:
                    i = i.clamp(0, 1)
                e_pw = _min_err(pw.double(), [p], e_pw)
                e_iw = _min_err(iw.double(), [i], e_iw)
            e_pw, e_iw = e_pw.max().item(), e_iw.max().item()
        else:
            xr = model.debug_tensor("x_res")
            hc, nband, npx = hmap_candidates(xr, jin, jout)
            att = torch.stack([h * dS for h in hc])
            mid, rad = (att.max(0).values + att.min(0).values) / 2, (att.max(0).values - att.min(0).values) / 2
            c, r = resize64(mid, H, W, m), resize64(rad, H, W, m, absolute=True)
            lo, hi = c - r, c + r
            e_pw = torch.maximum(lo - pw.double(), pw.double() - hi).clamp_min(0).max().item()
            ilo, ihi = x64 + 0.2 * lo, x64 + 0.2 * hi
            if flags & CL:
                ilo, ihi = ilo.clamp(0, 1), ihi.clamp(0, 1)
            e_iw = torch.maximum(ilo - iw.double(), iw.double() - ihi).clamp_min(0).max().item()
    print(f"[blend] {name}: dispatch {want}, max err preds_w {e_pw:.2e} (bound {tol_pw:.1e}), imgs_w {e_iw:.2e} (bound {tol_iw:.1e}); "
          f"band pixels {nband} of {npx}")
    assert nband <= BAND_FRAC * npx, (nband, npx)
    assert e_pw <= tol_pw and e_iw <= tol_iw, (e_pw, e_iw)


def test_blend_matrix_reaches_the_4tap_variants():
    """the cases above run the 4-tap up-scale of both blend kernels (TMA-fed and per-thread, both vector widths, one- and
    three-channel delta, both heat-map input counts), and bilinear, nearest and area up-scales stay on the <= 2-tap paths"""
    seen = {c[-1] for c in BLEND_CASES}
    assert {(k, v) for k, v, fu, _, _ in seen if fu == 4} == {(3, 4), (2, 1)}
    assert {cd for _, _, fu, cd, _ in seen if fu == 4} == {1, 3} and {j for _, _, fu, _, j in seen if fu == 4} == {1, 3}
    assert all(c[-1][2] in (1, 0) for c in BLEND_CASES if c[1][0] != "bicubic")


# ----------------------------------------------------------------------------------------------------- c. end to end
@pytest.fixture(scope="module")
def golden():
    return torch.load(os.path.join(ROOT, "tests", "golden", "interp.pt"), weights_only=False)


def test_e2e_matches_the_reference(golden):
    """embed / detect / extract_message with every dict of tests/golden/interp.pt against the unmodified reference's outputs: imgs_w
    and preds_w within PIX_TOL, logits within the logits contract, no flipped bit where the reference's margin is clear"""
    from tests.util import make_model_pair
    from tests.make_golden_interp import TINY, inputs, sub
    model, orc, spec = make_model_pair("videoseal_1.0", seed=golden["seed"], tiny=TINY)
    model.step_size, model.chunk_size, model.video_mode = golden["step"], golden["chunk"], "repeat"
    imgs, clip = inputs()
    msgs_i, msgs_v = golden["msgs_img"], golden["msgs_vid"]
    for key, r in golden["dicts"].items():
        interp = r["interpolation"]
        out = model.embed(imgs.cuda(), msgs_i, is_video=False, interpolation=interp)
        e_img = (sub(out["imgs_w"].cpu()) - r["img_imgs_w"]).abs().max().item()
        e_pw = (sub(out["preds_w"].cpu()) - r["img_preds_w"]).abs().max().item()
        vid = model.embed(clip.cuda(), msgs_v, is_video=True, interpolation=interp)
        e_vid = (sub(vid["imgs_w"].cpu()) - r["vid_imgs_w"]).abs().max().item()
        det = model.detect(vid["imgs_w"], is_video=True, interpolation=interp)["preds"].cpu()
        rel, flips, unsure = logits_ok(det, r["vid_preds"])
        bits = model.extract_message(vid["imgs_w"], interpolation=interp).cpu()
        agg = r["vid_preds"][:, 1:].mean(0)
        sure = agg.abs() > 1e-2 * agg.abs().max()
        print(f"[e2e] {key}: imgs_w {e_img:.2e}, preds_w {e_pw:.2e}, video imgs_w {e_vid:.2e}; logits rel {rel:.2e}, flips {flips}")
        assert e_img <= PIX_TOL and e_pw <= PIX_TOL and e_vid <= PIX_TOL, (key, e_img, e_pw, e_vid)
        assert rel <= LOGIT_RTOL and flips == 0, (key, rel, flips, unsure)
        assert (bits[0][sure] == r["extract_bits"][0][sure]).all(), key


# ----------------------------------------------------------------------------------------------------- d. defaults
def test_default_dict_is_mode_zero(pair):
    """embed without a dict, with the explicit default dict, and straight through the C ABI with mode bits 0: bit-identical;
    the same for detect and for extract_message's default dict"""
    x = frames(2, 1080, 1920, seed=5)
    msgs = torch.randint(0, 2, (2, pair[2]["nbits"]), generator=torch.Generator().manual_seed(5))
    with configured(pair) as model:
        a = model.embed(x.cuda(), msgs, is_video=False)
        b = model.embed(x.cuda(), msgs, is_video=False, interpolation={"mode": "bilinear", "align_corners": False, "antialias": True})
        assert torch.equal(a["imgs_w"], b["imgs_w"]) and torch.equal(a["preds_w"], b["preds_w"])
        xc, mm = x.cuda(), model._msgs_u8(msgs)
        iw, pw = torch.empty_like(xc), torch.empty_like(a["preds_w"])
        _lib.check(_lib.lib().vsb_embed(model._handle(), xc.data_ptr(), mm.data_ptr(), 2, iw.data_ptr(), pw.data_ptr(), 2, 1080, 1920, 1,
                                        0, 32, float(model.blender.scaling_i), float(model.blender.scaling_w), CL, model._stream()))
        torch.cuda.synchronize()
        assert torch.equal(a["imgs_w"], iw) and torch.equal(a["preds_w"], pw)
        d0 = model.detect(x.cuda(), is_video=True)["preds"]
        d1 = model.detect(x.cuda(), is_video=True, interpolation={"mode": "bilinear", "align_corners": False, "antialias": True})["preds"]
        out = torch.empty_like(d0)
        _lib.check(_lib.lib().vsb_detect(model._handle(), xc.data_ptr(), out.data_ptr(), 2, 1080, 1920, 0, model._stream()))
        torch.cuda.synchronize()
        assert torch.equal(d0, d1) and torch.equal(d0, out)
        n0 = model.detect(x.cuda(), is_video=True, interpolation={"mode": "bilinear", "align_corners": False, "antialias": False})["preds"]
        _lib.check(_lib.lib().vsb_detect(model._handle(), xc.data_ptr(), out.data_ptr(), 2, 1080, 1920, _lib.FLAG_RESIZE_NO_AA,
                                         model._stream()))
        torch.cuda.synchronize()
        assert torch.equal(n0, out)
        assert torch.equal(model.extract_message(x.cuda()), model.extract_message(
            x.cuda(), interpolation={"mode": "bilinear", "align_corners": False, "antialias": False}))


def test_c_abi_rejects_nearest_with_antialias(pair):
    """the host entry points validate the resize bits as F.interpolate does, only when a resize happens"""
    model = pair[0]
    x = torch.rand(1, 3, 300, 320).cuda()
    out = torch.empty(1, 1 + pair[2]["nbits"]).cuda()
    bad = _lib.RESIZE_MODES["nearest"] << _lib.FLAG_RESIZE_MODE_SHIFT      # antialias on (NO_AA clear)
    assert _lib.lib().vsb_detect(model._handle(), x.data_ptr(), out.data_ptr(), 1, 300, 320, bad, model._stream()) == -1
    S = model.img_size
    xs = torch.rand(1, 3, S, S).cuda()
    assert _lib.lib().vsb_detect(model._handle(), xs.data_ptr(), out.data_ptr(), 1, S, S, bad, model._stream()) == 0
