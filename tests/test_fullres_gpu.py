"""The two full-resolution kernels every frame passes, at real video geometries, against float64 references.

  resize_sep_kernel<MT, GST>        input -> processing size S (the U-Net's and the extractor's input)
  jnd_blend3_kernel / jnd_blend2_kernel   JND heat-map x up-sampled delta, blend, clamp

The end-to-end contract (imgs_w <= 1e-3 of the oracle) cannot see a few-percent error in the watermark term
scaling_w * hmap * delta (<= 0.2 * 0.13), nor a wrong resize tap once two networks and fp16 rounding sit behind it, so these
tests read the kernels' outputs directly: the `x_res` debug tap (the last resize of a call) and, for the blend, `imgs_w` /
`preds_w` of vsb_embed computed from the `delta` tap.  vsb_debug_last_dispatch tells which compiled variant ran.

References (float64):
  resize   F.interpolate on double tensors for anti-aliased down-scales; plain bilinear (no antialias, or up-scaling) from the
           fp32-rounded source coordinate, as ATen's fp32 kernels and the library's tables compute it (test_cpu_library.py
           checks the tables against ATen).  Both are applied as separable [n_out, n_in] operators.
  JND      modules/jnd.py:63-108 (oracle/restate.py:jnd_heatmaps) in float64.
  blend    models/videoseal.py:80-118 video modes, wam.py:183-201 and blender.py:61-68, in float64.

JND branch band.  The luminance-adaptation term is discontinuous at la0 = 127 (17 (1 - sqrt(la0/127 + 1e-5)) ~ 0 below,
3/128 (la0 - 127) + 3 = 3 above): a pixel whose la0 lies within fp32 rounding of 127 may take either side on the GPU, in the
fp32 oracle and in float64 alike, and moves the heat-map by up to 0.012.  Pixels with |la0_64 - 127| <= BAND (5e-4, ~64 fp32
ulps at 127; the kernels' la0 is within ~3e-5 of float64) are counted, must be a small fraction, and are checked against the
reference's value under either branch (per channel for the jnd_3_* configurations).  Flat u8 grey frames sit exactly on the
boundary; there the kernels must take the branch the fp32 reference takes (test_heatmaps_flat_grey_take_the_reference_branch).
"""
import contextlib
import ctypes as C
import functools
import itertools
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import restate
from tests.test_e2e_gpu import LOGIT_RTOL, PIX_TOL, logits_ok
from tests.util import make_model_pair
from videoseal_b200 import _lib

pytestmark = pytest.mark.gpu

TINY = {"num_blocks": 1, "depths": [1, 1, 1, 1]}
EPS = 2.0 ** -23
BAND = 5e-4
NOAA = {"mode": "bilinear", "align_corners": False, "antialias": False}
NAN = float("nan")
JND_CFG = {"jnd_1_1": (1, 1), "jnd_1_3": (1, 3), "jnd_3_1": (3, 1), "jnd_3_3": (3, 3)}

# Blend bounds, from the kernels' arithmetic (|delta| <= 1: tanh output; hmap <= ~0.15; scaling_w = 0.2, scaling_i = 1):
#  * delta up-sampling: <= 2 taps per axis with fp32 weights, 6 roundings: <= 6 * 2^-24 ~ 3.6e-7 (the anti-aliased down-scale of
#    a frame smaller than S: (maxt_x + maxt_y + 2) * 2^-24 <= 7.2e-7);
#  * heat-map: L = 255 Y in fp32 (1 rounding of <= 255), the 5x5 / Sobel sums as separable fp32 sums (la0 within ~3e-5 of
#    float64 in the worst case, which moves `lo` / `hi` by <= 2e-6 away from la0 ~ 0 and by 7e-7 on the `hi` side), and the
#    SFU's sqrt / lg2 / ex2 / rcp .approx (relative ~2^-22 each: <= 17 * 2^-22 on `lo`, <= 3 * 2^-22 * cm on cm <= 40):
#    together <= ~4e-5 before the final / 255, i.e. <= 1.6e-7 on hmap;
#  * preds_w = hmap * delta: <= 1.6e-7 + 0.15 * 7.2e-7 + 2^-24 < 3e-7;   imgs_w = fma(scaling_i, x, scaling_w * preds_w):
#    one rounding of a value <= 1.2 (1.2 * 2^-24) + 0.2 * 3e-7 < 1.5e-7.
# Both bounds below keep a factor of ~3 over that sum, and are 1000x tighter than the end-to-end PIX_TOL.
TOL_PW = 1e-6
TOL_IW = 5e-7
TOL_HM = 5e-7          # vsb_jnd_heatmaps (jnd_lowres_kernel): the heat-map part of the above
BAND_FRAC = 2e-3       # random frames: ~4e-5 of the pixels fall in the band (la0 has a std of ~11 grey levels around 127)


# ----------------------------------------------------------------------------------------------------- float64 references
def maxt(n_in, n_out, aa):
    return 2 * int(np.ceil(n_in / n_out)) + 1 if aa and n_in > n_out else 2


@functools.lru_cache(maxsize=None)
def resample_matrix(n_in: int, n_out: int, aa: bool) -> torch.Tensor:
    """[n_out, n_in] float64 operator of F.interpolate(mode='bilinear', align_corners=False) along one axis"""
    if n_in == n_out:
        return torch.eye(n_in, dtype=torch.float64)
    if aa and n_in > n_out:
        eye = torch.eye(n_in, dtype=torch.float64).reshape(n_in, 1, 1, n_in)
        return F.interpolate(eye, size=(1, n_out), mode="bilinear", align_corners=False, antialias=True).reshape(n_in, n_out).t().contiguous()
    # area_pixel_compute_source_index in fp32: one rounding of scale * (i + 0.5) - 0.5 (exact in float64, then rounded)
    scale = np.float64(np.float32(n_in / n_out))
    src = (scale * (np.arange(n_out) + 0.5) - 0.5).astype(np.float32).astype(np.float64)
    src = np.maximum(src, 0.0)
    x0 = np.minimum(src.astype(np.int64), n_in - 1)
    x1 = np.minimum(x0 + 1, n_in - 1)
    l1 = np.clip(src - x0, 0.0, 1.0)
    m = np.zeros((n_out, n_in))
    np.add.at(m, (np.arange(n_out), x0), 1.0 - l1)
    np.add.at(m, (np.arange(n_out), x1), l1)
    return torch.from_numpy(m)


def resize64(x: torch.Tensor, oh: int, ow: int, aa: bool) -> torch.Tensor:
    """[..., H, W] -> [..., oh, ow] float64"""
    my = resample_matrix(x.shape[-2], oh, aa)
    mx = resample_matrix(x.shape[-1], ow, aa)
    return torch.matmul(torch.matmul(my, x.double()), mx.t())


_KL = restate._K_L.double()
_KX = restate._K_X.double()
_KY = restate._K_Y.double()


def jnd_parts64(imgs: torch.Tensor, jin: int):
    """modules/jnd.py:63-108 in float64 per input channel, before the channel mixing: (la0, hmap with the low branch, hmap with
    the high branch), each [F, jin, H, W] and already / 255"""
    x = 255.0 * imgs.double()
    if jin == 1:
        x = 0.299 * x[:, 0:1] + 0.587 * x[:, 1:2] + 0.114 * x[:, 2:3]
    la0 = F.conv2d(x, _KL.repeat(jin, 1, 1, 1), padding=2, groups=jin) / 32
    gx = F.conv2d(x, _KX.repeat(jin, 1, 1, 1), padding=1, groups=jin)
    gy = F.conv2d(x, _KY.repeat(jin, 1, 1, 1), padding=1, groups=jin)
    g2 = gx * gx + gy * gy
    cm = 0.117 * (16 * g2 ** 1.2 / (g2 + 26 ** 2))

    def h(la):
        return torch.clamp_min(la + cm - 0.3 * torch.minimum(la, cm), 0) / 255

    return la0, h(17 * (1 - torch.sqrt(la0 / 127 + 1e-5))), h(3 / 128 * (la0 - 127) + 3)


def la0_fp32(imgs: torch.Tensor, jin: int) -> torch.Tensor:
    """la0 as the fp32 reference computes it (oracle/restate.py:jnd_heatmaps): decides the branch on flat grey frames"""
    x = 255 * imgs.float()
    if jin == 1:
        x = 0.299 * x[:, 0:1] + 0.587 * x[:, 1:2] + 0.114 * x[:, 2:3]
    return F.conv2d(x, restate._K_L.repeat(jin, 1, 1, 1), padding=2, groups=jin) / 32


def mix_channels(h: torch.Tensor, jin: int, jout: int) -> torch.Tensor:
    if jin == 1 and jout == 3:
        return h.repeat(1, 3, 1, 1)
    if jin == 3 and jout == 1:
        return torch.sum(h / 3, dim=1, keepdim=True)
    return h


def hmap_candidates(imgs, jin, jout, fp32_branch=False):
    """The heat-maps [F, jout, H, W] a correct kernel may produce: the nominal one, plus, for every combination of branches of the
    in-band channels, the one with those channels on the other side.  Returns (candidates, band pixel count, pixel count)."""
    la0, lo, hi = jnd_parts64(imgs, jin)
    low = (la0_fp32(imgs, jin).double() if fp32_branch else la0) <= 127
    nominal, other = torch.where(low, lo, hi), torch.where(low, hi, lo)
    band = torch.zeros_like(low) if fp32_branch else (la0 - 127).abs() <= BAND
    nband = int(band.any(1).sum())
    if nband == 0:
        return [mix_channels(nominal, jin, jout)], 0, band[:, 0].numel()
    cands = []
    for bits in itertools.product([False, True], repeat=jin):
        flip = band & torch.tensor(bits).view(1, jin, 1, 1)
        cands.append(mix_channels(torch.where(flip, other, nominal), jin, jout))
    return cands, nband, band[:, 0].numel()


def video_deltas64(keys: torch.Tensor, F_: int, step: int, mode: str, chunk_keys: int) -> torch.Tensor:
    """models/videoseal.py:80-118 and :300-331 (oracle/restate.py:apply_video_mode per chunk) in float64: the delta of every frame"""
    out = torch.zeros((F_,) + keys.shape[1:], dtype=torch.float64)
    nkeys = keys.shape[0]
    for f in range(F_):
        k, ph = divmod(f, step)
        if mode == "repeat" or step == 1:
            out[f] = keys[k]
        elif mode == "alternate":
            if ph == 0:
                out[f] = keys[k]
        else:
            c0 = k // chunk_keys * chunk_keys
            last = min(c0 + chunk_keys, nkeys) - 1            # the chunk's last key stands alone
            if k < last:
                a = 1.0 - ph / (step - 1)
                out[f] = a * keys[k] + (1 - a) * keys[k + 1]
            else:
                out[f] = keys[k]
    return out


# ----------------------------------------------------------------------------------------------------- model handling
@pytest.fixture(scope="module")
def pair():
    return make_model_pair("videoseal_1.0", tiny=TINY)


@contextlib.contextmanager
def configured(pair, S=256, jnd="jnd_1_1", step=None, chunk=None, mode=None):
    """the model (and its oracle) at processing size S with a JND configuration and video settings, restored afterwards"""
    model, orc, spec = pair
    old = (model.img_size, model.step_size, model.chunk_size, model.video_mode)
    jin, jout = JND_CFG[jnd]
    try:
        model.img_size = orc.img_size = S
        model.attenuation = types.SimpleNamespace(in_channels=jin, out_channels=jout)
        orc.attenuation = jnd
        if step is not None:
            model.step_size = orc.step_size = step
        if chunk is not None:
            model.chunk_size = orc.chunk_size = chunk
        if mode is not None:
            model.video_mode = orc.video_mode = mode
        yield model
    finally:
        model.img_size = orc.img_size = spec["img_size"]
        model.attenuation = types.SimpleNamespace(in_channels=1, out_channels=1)
        orc.attenuation = "jnd_1_1"
        model.step_size, model.chunk_size, model.video_mode = old[1:]
        orc.step_size, orc.chunk_size, orc.video_mode = old[1:]


def dispatch(model):
    buf = (C.c_int32 * 10)()
    assert _lib.lib().vsb_debug_last_dispatch(model._handle(), buf, 10) == 10, _lib.lib().vsb_last_error()
    return tuple(buf[:5]), tuple(buf[5:])


def test_last_dispatch_seam_rejects_a_short_buffer(pair):
    model = pair[0]
    buf = (C.c_int32 * 10)()
    assert _lib.lib().vsb_debug_last_dispatch(model._handle(), buf, 9) < 0


def frames(F_, H, W, seed):
    """random frames, and in slot 1 (when F_ > 1) a dark frame with single bright rows and columns on the borders, around the
    middle and on the first staging-round boundaries (rows 1..8 cover GST = 1, 2 and 4 rounds)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(F_, 3, H, W, generator=g)
    if F_ > 1:
        s = torch.full((3, H, W), 0.05)
        for r in {0, 1, 2, 3, 4, 7, 8, H // 2, H - 2, H - 1}:
            s[:, min(r, H - 1)] = 1.0
        for c in {0, 1, 3, 4, 255, 256, W // 2, W - 2, W - 1}:
            s[:, :, min(c, W - 1)] = 1.0
        x[1] = s
    return x


# ----------------------------------------------------------------------------------------------------- a. resize
# (W, H, S, antialias, expected (MT, GST, vec))
RESIZE_CASES = [
    (1920, 1080, 256, True, (0, 2, 1)),
    (1080, 1920, 256, True, (0, 2, 1)),
    (3840, 2160, 256, True, (0, 1, 1)),
    (3840, 2160, 256, False, (2, 1, 1)),
    (1920, 1080, 256, False, (2, 2, 1)),
    (1280, 720, 256, True, (0, 2, 1)),
    (854, 480, 256, True, (0, 4, 0)),
    (1366, 768, 256, True, (0, 2, 0)),
    (1024, 576, 256, True, (0, 4, 1)),
    (1025, 577, 256, True, (0, 2, 0)),
    (2048, 1152, 256, True, (0, 2, 1)),
    (2049, 1153, 256, True, (0, 1, 0)),
    (768, 432, 256, True, (8, 4, 1)),
    (769, 433, 256, True, (0, 4, 0)),
    (1280, 720, 512, True, (8, 2, 1)),
    (2304, 1296, 768, True, (8, 1, 1)),
    (1920, 1080, 128, True, (0, 2, 1)),
    (1920, 1080, 384, True, (0, 2, 1)),
    (176, 144, 256, True, (2, 4, 1)),
    (16384, 16, 256, True, (0, 1, 1)),      # the widest frame whose staging ring fits in shared memory (~194 KB)
]


def _rid(c):
    return f"{c[0]}x{c[1]}-S{c[2]}-{'aa' if c[3] else 'noaa'}"


def _check_x_res(model, ref_frames, S, aa, tag):
    got = model.debug_tensor("x_res").double()
    ref = resize64(ref_frames, S, S, aa)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    tol = (maxt(ref_frames.shape[-1], S, aa) + maxt(ref_frames.shape[-2], S, aa) + 2) * EPS
    err = (got - ref).abs().max().item()
    print(f"[resize] {tag}: max|x_res - float64| = {err:.2e} (bound {tol:.2e})")
    assert err <= tol, (tag, err, tol)


@pytest.mark.parametrize("case", RESIZE_CASES, ids=_rid)
def test_resize_matches_float64(pair, case):
    """x_res of detect (contiguous frames) and of video embed (key frames `step` frames apart, ragged last group) against the
    float64 resize.  A different input runs through the same plan first, so an output the kernel never wrote shows up as stale
    data.  Bound: (maxt_x + maxt_y + 2) * 2^-23 on inputs in [0, 1] (one rounding per tap and per pass)."""
    W, H, S, aa, want = case
    kw = {} if aa else {"interpolation": NOAA}
    x = frames(2, H, W, seed=W + H + S)
    vid = frames(10, H, W, seed=W * H)                      # key frames 0, 4, 8; the last group has 2 frames
    with configured(pair, S=S, step=4, chunk=32, mode="repeat") as model:
        model.detect((1 - x).cuda(), is_video=True, **kw)
        model.detect(x.cuda(), is_video=True, **kw)
        rs, _ = dispatch(model)
        assert rs[:3] == want and rs[4] == S, rs
        _check_x_res(model, x, S, aa, _rid(case) + " detect")
        if S & (S - 1):
            return      # the U-Net's tensor-core convolutions tile every map by 128 pixels: it runs at S = 128 * 2^k only
        model.embed((1 - vid).cuda(), is_video=True, **kw)
        model.embed(vid.cuda(), is_video=True, **kw)
        assert dispatch(model)[0][:3] == want
        _check_x_res(model, vid[::4], S, aa, _rid(case) + " embed keys")


def test_resize_and_blend_variant_coverage(pair):
    """every compiled resize variant and both blend kernels run at the geometries above: all 9 (MT, GST) instantiations, both
    copy paths, fewer than 8 output rows per block, output widths above 256 and not a multiple of 256; blend3 / blend2 with both
    vector widths, both delta paths and both heat-map input counts.  A dispatch change that moves a case off its variant fails here."""
    seen_rs, seen_bl = set(), set()
    for W, H, S, aa, _ in RESIZE_CASES:
        with configured(pair, S=S) as model:
            model.detect(torch.rand(1, 3, H, W).cuda(), is_video=True, **({} if aa else {"interpolation": NOAA}))
            seen_rs.add(dispatch(model)[0])
    for W, H, jnd in [(1920, 1080, "jnd_1_1"), (854, 480, "jnd_1_1"), (176, 144, "jnd_1_1"), (1920, 1080, "jnd_3_3"), (854, 480, "jnd_3_1")]:
        with configured(pair, jnd=jnd) as model:
            model.embed(torch.rand(1, 3, H, W).cuda(), is_video=False)
            seen_bl.add(dispatch(model)[1])
    print("[coverage] resize (MT, GST, vec, toy, OW):", sorted(seen_rs))
    print("[coverage] blend (kernel, VEC, FASTUP, CD, JIN):", sorted(seen_bl))
    assert {(r[0], r[1]) for r in seen_rs} == {(mt, g) for mt in (2, 8, 0) for g in (4, 2, 1)}
    assert {r[2] for r in seen_rs} == {0, 1}
    assert min(r[3] for r in seen_rs) < 8
    assert any(r[4] > 256 for r in seen_rs) and any(r[4] % 256 != 0 for r in seen_rs)
    assert {b[0] for b in seen_bl} == {2, 3} and {b[1] for b in seen_bl} == {1, 4}
    assert {b[2] for b in seen_bl} == {0, 1} and {b[4] for b in seen_bl} == {1, 3}


# ----------------------------------------------------------------------------------------------------- b. blend
def _embed_raw(model, imgs, step, mode, chunk, flags, pc, scaling_w=0.2):
    """vsb_embed straight through the C ABI into NaN-filled outputs; returns (imgs_w, preds_w, delta keys) on the CPU"""
    F_, _, H, W = imgs.shape
    nmsg = F_ if step == 1 else 1
    msgs = torch.randint(0, 2, (nmsg, model.spec["nbits"]), generator=torch.Generator().manual_seed(F_ + H)).to(torch.uint8).cuda()
    iw = torch.full_like(imgs, NAN)
    pw = torch.full((F_, pc, H, W), NAN, device=imgs.device)
    _lib.check(_lib.lib().vsb_embed(model._handle(), imgs.data_ptr(), msgs.data_ptr(), nmsg, iw.data_ptr(), pw.data_ptr(), F_, H, W, step,
                                    _lib.VIDEO_MODES[mode], chunk, 1.0, scaling_w, flags, model._stream()))
    torch.cuda.synchronize()
    return iw.cpu(), pw.cpu(), model.debug_tensor("delta").double()


# (id, jnd, W, H, S, F, step, mode, chunk keys, flags, expected blend dispatch (kernel, VEC, FASTUP, CD, JIN) with CD = 1)
CL, LR, NA, NOAAF = _lib.FLAG_CLAMP, _lib.FLAG_LOWRES_ATTN, _lib.FLAG_NO_ATTENUATION, _lib.FLAG_RESIZE_NO_AA
BLEND_CASES = [
    ("image-1080p", "jnd_1_1", 1920, 1080, 256, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("image-4k", "jnd_1_1", 3840, 2160, 256, 1, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("repeat-1080x1920", "jnd_1_1", 1080, 1920, 256, 10, 4, "repeat", 2, CL, (3, 4, 1, 1, 1)),
    ("alternate-1080p", "jnd_1_1", 1920, 1080, 256, 10, 4, "alternate", 2, CL, (3, 4, 1, 1, 1)),
    ("interpolate-1080p", "jnd_1_1", 1920, 1080, 256, 14, 4, "interpolate", 2, CL, (3, 4, 1, 1, 1)),
    ("interpolate-720p-S512", "jnd_1_1", 1280, 720, 512, 10, 4, "interpolate", 2, CL, (3, 4, 1, 1, 1)),
    ("jnd_1_3-1080p", "jnd_1_3", 1920, 1080, 256, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("jnd_3_1-1080p", "jnd_3_1", 1920, 1080, 256, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 3)),
    ("jnd_3_3-1080p", "jnd_3_3", 1920, 1080, 256, 2, 1, "repeat", 32, CL, (3, 4, 1, 1, 3)),
    ("no-attenuation-1080p", "jnd_1_1", 1920, 1080, 256, 2, 1, "repeat", 32, CL | NA, (3, 4, 1, 1, 1)),
    ("no-aa-4k", "jnd_1_1", 3840, 2160, 256, 1, 1, "repeat", 32, CL | NOAAF, (3, 4, 1, 1, 1)),
    ("no-clamp-1080p", "jnd_1_1", 1920, 1080, 256, 2, 1, "repeat", 32, 0, (3, 4, 1, 1, 1)),
    ("identity-256", "jnd_1_1", 256, 256, 256, 3, 1, "repeat", 32, CL, (3, 4, 1, 1, 1)),
    ("identity-512-repeat", "jnd_3_3", 512, 512, 512, 6, 4, "repeat", 32, CL, (3, 4, 1, 1, 3)),
    ("scalar-854x480", "jnd_1_1", 854, 480, 256, 2, 1, "repeat", 32, CL, (2, 1, 1, 1, 1)),
    ("scalar-1366x768-alternate", "jnd_1_1", 1366, 768, 256, 10, 4, "alternate", 2, CL, (2, 1, 1, 1, 1)),
    ("scalar-854x480-jnd_3_1", "jnd_3_1", 854, 480, 256, 2, 1, "repeat", 32, CL, (2, 1, 1, 1, 3)),
    ("downscaled-delta-176x144", "jnd_1_1", 176, 144, 256, 2, 1, "repeat", 32, CL, (2, 4, 0, 1, 1)),
    ("downscaled-delta-176x144-no-aa", "jnd_1_1", 176, 144, 256, 2, 1, "repeat", 32, CL | NOAAF, (2, 4, 0, 1, 1)),
    ("downscaled-delta-854x480-S512", "jnd_3_3", 854, 480, 512, 2, 1, "repeat", 32, CL, (2, 1, 0, 1, 3)),
    ("lowres-720p", "jnd_1_1", 1280, 720, 256, 2, 1, "repeat", 32, CL | LR, (3, 4, 1, 1, 1)),
    ("lowres-720p-jnd_3_3", "jnd_3_3", 1280, 720, 256, 2, 1, "repeat", 32, CL | LR, (3, 4, 1, 3, 1)),
    ("lowres-1366x768-jnd_3_1", "jnd_3_1", 1366, 768, 256, 2, 1, "repeat", 32, CL | LR, (2, 1, 1, 1, 1)),
]


def _min_err(got, cands, err=None):
    """elementwise distance of `got` to the nearest candidate (and to what `err` already holds)"""
    for c in cands:
        e = (got - c).abs()
        err = e if err is None else torch.minimum(err, e)
    return err


@pytest.mark.parametrize("case", BLEND_CASES, ids=[c[0] for c in BLEND_CASES])
def test_blend_matches_float64(pair, case):
    """imgs_w and preds_w of the blend kernels against the float64 blend of (frames, delta tap): TOL_IW / TOL_PW (derived above)
    outside the JND branch band, either branch inside it.  With lowres_attenuation the heat-map is taken at processing size from
    the resized frames (the x_res tap in image mode) and the attenuated delta is up-sampled; a band pixel there spreads over the
    output pixels its taps reach, so those are checked against the interval spanned by the two branches (the weights are >= 0)."""
    name, jnd, W, H, S, F_, step, mode, chunk, flags, want = case
    jin, jout = JND_CFG[jnd]
    use_jnd = not flags & NA
    lowres = use_jnd and bool(flags & LR)
    aa = not flags & NOAAF
    pc = max(1, jout) if use_jnd else 1
    x = frames(F_, H, W, seed=BLEND_CASES.index(case))
    with configured(pair, S=S, jnd=jnd) as model:
        iw, pw, dkeys = _embed_raw(model, x.cuda(), step, mode, chunk, flags, pc)
        assert dispatch(model)[1] == want, dispatch(model)
        assert not torch.isnan(iw).any() and not torch.isnan(pw).any(), "an output pixel was not written"
        assert dkeys.shape[0] == (F_ + step - 1) // step
        dS = video_deltas64(dkeys, F_, step, mode, chunk)                     # [F, 1, S, S]
        x64 = x.double()
        if not use_jnd:
            cands, nband, npx = [torch.ones(F_, 1, H, W, dtype=torch.float64)], 0, F_ * H * W
        elif not lowres:
            cands, nband, npx = hmap_candidates(x, jin, jout)
        if not lowres:
            dup = resize64(dS, H, W, aa)
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
            xr = model.debug_tensor("x_res")                                  # every frame is a key frame in image mode
            hc, nband, npx = hmap_candidates(xr, jin, jout)
            att = torch.stack([h * dS for h in hc])                           # [cands, F, PC, S, S]
            lo, hi = resize64(att.min(0).values, H, W, aa), resize64(att.max(0).values, H, W, aa)
            e_pw = torch.maximum(lo - pw.double(), pw.double() - hi).clamp_min(0).max().item()
            ilo, ihi = x64 + 0.2 * lo, x64 + 0.2 * hi
            if flags & CL:
                ilo, ihi = ilo.clamp(0, 1), ihi.clamp(0, 1)
            e_iw = torch.maximum(ilo - iw.double(), iw.double() - ihi).clamp_min(0).max().item()
    print(f"[blend] {name}: max err preds_w {e_pw:.2e}, imgs_w {e_iw:.2e}; branch-band pixels {nband} of {npx}")
    assert nband <= BAND_FRAC * npx, (nband, npx)
    assert e_pw <= TOL_PW and e_iw <= TOL_IW, (e_pw, e_iw)


# ----------------------------------------------------------------------------------------------------- c. heat-maps
@pytest.mark.parametrize("jnd,H,W", [("jnd_1_1", 1080, 1920), ("jnd_1_1", 2160, 3840), ("jnd_1_1", 201, 333), ("jnd_1_1", 769, 1366),
                                     ("jnd_1_3", 1080, 1920), ("jnd_3_1", 1080, 1920), ("jnd_3_3", 1080, 1920), ("jnd_3_3", 201, 333)])
def test_heatmaps_match_float64(pair, jnd, H, W):
    """the vsb_jnd_heatmaps seam against float64 modules/jnd.py, TOL_HM outside the branch band, either branch inside"""
    jin, jout = JND_CFG[jnd]
    x = frames(2, H, W, seed=H * W)
    with configured(pair, jnd=jnd) as model:
        got = model.attenuation.heatmaps(x.cuda()).cpu().double()
    cands, nband, npx = hmap_candidates(x, jin, jout)
    err = _min_err(got, cands).max().item()
    print(f"[heatmap] {jnd} {W}x{H}: max err {err:.2e}; branch-band pixels {nband} of {npx}")
    assert got.shape == cands[0].shape
    assert nband <= BAND_FRAC * npx and err <= TOL_HM, (nband, err)


def grey_frames(H, W):
    """flat u8 grey 126, 127, 128, and 127 with +-1 texture, as x = u8 / 255 like a decoded video frame"""
    g = torch.Generator().manual_seed(3)
    u8 = torch.stack([torch.full((3, H, W), 126), torch.full((3, H, W), 127), torch.full((3, H, W), 128),
                      127 + torch.randint(-1, 2, (1, H, W), generator=g).repeat(3, 1, 1)])
    return u8.float() / 255.0


@pytest.mark.parametrize("jnd", ["jnd_1_1", "jnd_3_3"])
def test_heatmaps_flat_grey_take_the_reference_branch(pair, jnd):
    """grey 127 lies exactly on the branch point: exact arithmetic (and the fp32 reference) give la0 = 127 and the low branch
    (heat-map 0 away from the borders), while one fp32 rounding upwards would give the high branch (0.0119, 0.6 grey levels of
    watermark amplitude at scaling_w = 0.2).  The flat frames must follow the fp32 reference's branch decision with no band; the
    textured frame, where many pixels have la0 exactly 127 in exact arithmetic, follows the band rule.  Checked for the heat-map
    seam and for the blend kernels' own heat-map (preds_w = hmap * delta with the luminance computed by lum255)."""
    jin, jout = JND_CFG[jnd]
    H, W = 264, 520             # >= S in both directions: the TMA-fed kernel takes the 4-aligned width
    x = grey_frames(H, W)
    flat, tex = x[:3], x[3:]
    with configured(pair, jnd=jnd) as model:
        got = model.attenuation.heatmaps(x.cuda()).cpu().double()
        for W_, kind in [(W, 3), (W - 2, 2)]:             # TMA-fed and scalar blend kernels
            xs = x[..., :W_].contiguous()
            iw, pw, dkeys = _embed_raw(model, xs.cuda(), 1, "repeat", 32, CL, jout)
            assert dispatch(model)[1][0] == kind
            dup = resize64(dkeys, H, W_, True)
            hf, _, _ = hmap_candidates(xs[:3], jin, jout, fp32_branch=True)
            e_flat = (pw[:3].double() - hf[0] * dup[:3]).abs().max().item()
            ht, nb, npx = hmap_candidates(xs[3:], jin, jout)
            e_tex = _min_err(pw[3:].double(), [h * dup[3:] for h in ht]).max().item()
            print(f"[grey] {jnd} blend{kind}: flat max err {e_flat:.2e}; textured {e_tex:.2e}, band pixels {nb} of {npx}")
            assert e_flat <= TOL_PW and e_tex <= TOL_PW, (kind, e_flat, e_tex)
    hf, _, _ = hmap_candidates(flat, jin, jout, fp32_branch=True)
    e_flat = (got[:3] - hf[0]).abs().max().item()
    assert hf[0][1, :, 8:-8, 8:-8].abs().max().item() == 0.0          # grey 127: low branch, no texture -> 0
    assert hf[0][2, :, 8:-8, 8:-8].min().item() > 0.011               # grey 128: high branch
    ht, nb, npx = hmap_candidates(tex, jin, jout)
    e_tex = _min_err(got[3:], ht).max().item()
    print(f"[grey] {jnd} heat-map seam: flat max err {e_flat:.2e}; textured {e_tex:.2e}, band pixels {nb} of {npx}")
    assert e_flat <= TOL_HM and e_tex <= TOL_HM, (e_flat, e_tex)


# ----------------------------------------------------------------------------------------------------- d. end to end
def _band_mask(imgs, jin, S=None, aa=True):
    """output pixels whose JND branch is uncertain: la0 within BAND of 127 at full resolution, or (lowres_attenuation) at
    processing size, spread by the up-sampling taps"""
    if S is None:
        la0 = jnd_parts64(imgs, jin)[0]
        return ((la0 - 127).abs() <= BAND).any(1, keepdim=True)
    la0 = jnd_parts64(resize64(imgs, S, S, aa), jin)[0]
    b = ((la0 - 127).abs() <= BAND).any(1, keepdim=True).double()
    return resize64(b, imgs.shape[-2], imgs.shape[-1], aa) != 0


def _check_imgs_w(got, ref, band, tag):
    """PIX_TOL outside the band; inside it the two branches differ by up to scaling_w * 0.012 * |delta|"""
    err = (got - ref).abs()
    band = band.expand_as(err)
    e_out = err[~band].max().item()
    e_in = err[band].max().item() if band.any() else 0.0
    nb = int(band[:, 0].sum())
    print(f"[e2e] {tag}: max|imgs_w - oracle| {e_out:.2e} outside the band, {e_in:.2e} on its {nb} pixels")
    assert e_out <= PIX_TOL and e_in <= PIX_TOL + 0.2 * 0.0125, (e_out, e_in)
    assert nb <= BAND_FRAC * band[:, 0].numel()


@pytest.mark.parametrize("B,H,W", [(2, 1080, 1920), (1, 2160, 3840)])
def test_e2e_images_at_video_resolutions(pair, B, H, W):
    model, orc, spec = pair
    g = torch.Generator().manual_seed(H)
    imgs = torch.rand(B, 3, H, W, generator=g)
    msgs = torch.randint(0, 2, (B, spec["nbits"]), generator=g)
    with torch.no_grad():
        ref = orc.embed(imgs, msgs, is_video=False)
        ref_det = orc.detect(ref["imgs_w"], is_video=False)["preds"]
    out = model.embed(imgs.cuda(), msgs, is_video=False)
    _check_imgs_w(out["imgs_w"].cpu(), ref["imgs_w"], _band_mask(imgs, 1), f"image {W}x{H}")
    rel, flips, unsure = logits_ok(model.detect(out["imgs_w"], is_video=False)["preds"].cpu(), ref_det)
    assert rel <= LOGIT_RTOL and flips == 0, (rel, flips, unsure)


@pytest.mark.parametrize("mode", ["repeat", "alternate", "interpolate"])
@pytest.mark.parametrize("W,H", [(1080, 1920), (854, 480)])
def test_e2e_video_at_video_resolutions(pair, mode, W, H):
    model, orc, spec = pair
    g = torch.Generator().manual_seed(W + H)
    vid = torch.rand(10, 3, H, W, generator=g)
    msgs = torch.randint(0, 2, (1, spec["nbits"]), generator=g)
    with configured(pair, step=4, chunk=2, mode=mode):
        with torch.no_grad():
            ref = orc.embed(vid, msgs, is_video=True)
            ref_det = orc.detect(ref["imgs_w"], is_video=True)["preds"]
        out = model.embed(vid.cuda(), msgs, is_video=True)
        _check_imgs_w(out["imgs_w"].cpu(), ref["imgs_w"], _band_mask(vid, 1), f"video {mode} {W}x{H}")
        rel, flips, unsure = logits_ok(model.detect(out["imgs_w"], is_video=True)["preds"].cpu(), ref_det)
        assert rel <= LOGIT_RTOL and flips == 0, (rel, flips, unsure)


def test_e2e_lowres_attenuation_720p(pair):
    model, orc, spec = pair
    g = torch.Generator().manual_seed(720)
    imgs = torch.rand(2, 3, 720, 1280, generator=g)
    msgs = torch.randint(0, 2, (2, spec["nbits"]), generator=g)
    with torch.no_grad():
        ref = orc.embed(imgs, msgs, is_video=False, lowres_attenuation=True)
    out = model.embed(imgs.cuda(), msgs, is_video=False, lowres_attenuation=True)
    _check_imgs_w(out["imgs_w"].cpu(), ref["imgs_w"], _band_mask(imgs, 1, S=256), "lowres 1280x720")


def test_e2e_extract_message_1080p(pair):
    """extract_message resizes without antialias (videoseal.py:394): the plain-bilinear <2, 2> resize at 1080p"""
    model, orc, spec = pair
    g = torch.Generator().manual_seed(1080)
    vid = torch.rand(6, 3, 1080, 1920, generator=g)
    with torch.no_grad():
        ref_det = orc.detect(vid, is_video=True, interpolation=NOAA)["preds"]
        ref_msg = orc.extract_message(vid)
    det = model.detect(vid.cuda(), is_video=True, interpolation=NOAA)["preds"].cpu()
    assert dispatch(model)[0][:2] == (2, 2)
    rel, flips, unsure = logits_ok(det, ref_det)
    assert rel <= LOGIT_RTOL and flips == 0, (rel, flips, unsure)
    agg = ref_det[:, 1:].mean(0)
    sure = agg.abs() > 1e-2 * agg.abs().max()
    assert (model.extract_message(vid.cuda()).cpu()[0][sure] == ref_msg[0][sure]).all()


def test_u8_streaming_entry_1080p(pair):
    """the RGB24 streaming entry (vsb_frames_host_u8) on 40 frames of 1080p: bit-identical to the same arithmetic through the
    fp32 API, as test_e2e_gpu.py::test_u8_streaming_clip_entry checks at a small size"""
    from videoseal_b200.streaming import embed_video_clip
    model, orc, spec = pair
    g = torch.Generator().manual_seed(40)
    clip = torch.randint(0, 256, (40, 1080, 1920, 3), dtype=torch.uint8, generator=g).numpy()
    msgs = torch.randint(0, 2, (1, spec["nbits"]), generator=g)
    with configured(pair, step=4):
        out = embed_video_clip(model, clip, msgs)
        # u8 / 255 on the CPU: a CUDA tensor divided by a Python scalar is multiplied by its reciprocal (not correctly rounded)
        x = torch.from_numpy(clip).permute(0, 3, 1, 2).float() / 255.0
        ref32 = model.embed(x.cuda(), msgs, is_video=True, lowres_attenuation=True)["imgs_w"]
        ref_u8 = (ref32 * 255.0).byte().permute(0, 2, 3, 1).cpu().numpy()
    assert out.shape == clip.shape and np.array_equal(out, ref_u8)


# ----------------------------------------------------------------------------------------------------- e. limits
def test_frame_too_wide_for_the_resize_kernel_is_unsupported(pair):
    """the resize kernel stages whole input rows in shared memory: 16384 columns fit (~194 KB; detect and embed in the resize
    cases above, where embed up-samples the delta to that width through the blend's table), 20000 do not and must fail with
    VSB_ERR_UNSUPPORTED and a message instead of launching"""
    model = pair[0]
    with pytest.raises(NotImplementedError, match="too wide"):
        model.detect(torch.rand(1, 3, 16, 20000).cuda(), is_video=True)
    with pytest.raises(NotImplementedError, match="too wide"):
        model.embed(torch.rand(1, 3, 16, 20000).cuda(), is_video=False)
