"""Every interpolation mode of the reference's `interpolation` dict without a GPU: the host-built resample tables against ATen's
F.interpolate, the validation and encoding of the dict (model.resize_flags), and the evaluation CLIs' options.

Tables.  vsb_debug_resample_table2 exports the separable table one axis uses; applied to the identity it must equal
F.interpolate of the identity.  The anti-aliased and area tables are computed in double and rounded once to fp32 (a weight <= ~1.1:
<= 6.6e-8), so they are held to float64 ATen at 1e-7.  Nearest tables must select the same source index as fp32 ATen, exactly.
Plain bilinear (align_corners=True) and plain bicubic take their source coordinate and weights in fp32, as ATen's fp32 kernels do,
so they are held to fp32 ATen with the bound derived at TOL_PLAIN below.
"""
import itertools
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from videoseal_b200 import _lib
from videoseal_b200.model import resize_flags

# the geometries of test_cpu_library.py::test_resample_tables_match_aten_interpolate, then video sizes <-> 256, a 176 x 144 frame
# up to 256, 257 -> 256 and 256 -> 768
GEOMS = sorted({(768, 256), (300, 256), (480, 256), (257, 256), (200, 256), (256, 768), (256, 300), (17, 256), (1080, 256), (769, 256),
                (1920, 256), (2160, 256), (3840, 256), (1280, 256), (1920, 384), (3840, 128), (256, 1920), (256, 2160), (512, 1080),
                (256, 1080), (256, 3840), (176, 256), (144, 256)})
# (mode, align_corners, antialias): every combination F.interpolate accepts (None: align_corners not given)
MODES = [("bilinear", ac, aa) for ac in (False, True) for aa in (False, True)] + \
        [("bicubic", ac, aa) for ac in (False, True) for aa in (False, True)] + [("nearest", None, False), ("area", None, False)]
EPS24 = 2.0 ** -24
# Plain bilinear / bicubic: the table and ATen compute the same fp32 source coordinate (one fused multiply-add, or one multiply with
# align_corners), so they differ only in how the weights are evaluated.  A Keys coefficient is a Horner cubic whose intermediates
# stay below 8 (|A| = 0.75, t + 1 <= 2): each of its <= 6 roundings is <= 2^-22, 6 * 2^-22 per coefficient and evaluation; the two
# evaluations may round differently (compilers contract differently), and a folded edge tap sums two coefficients: 4 * 6 * 2^-22.
# Bilinear weights (1 - t, t) are one rounding each: covered.
TOL_PLAIN = 4 * 6 * 2.0 ** -22


def table2(lib, n_in, n_out, mode, ac, aa):
    start = np.zeros(n_out, dtype=np.int32)
    cnt = np.zeros(n_out, dtype=np.int32)
    cap = n_out * 256
    w = np.zeros(cap, dtype=np.float32)
    maxt = lib.vsb_debug_resample_table2(n_in, n_out, _lib.RESIZE_MODES[mode], int(bool(ac)), int(aa), start.ctypes.data,
                                         cnt.ctypes.data, w.ctypes.data, cap)
    assert maxt > 0, lib.vsb_last_error()
    return maxt, start, cnt, w[: n_out * maxt].reshape(n_out, maxt)


def operator(n_in, maxt, start, cnt, w):
    n_out = len(start)
    op = np.zeros((n_out, n_in), dtype=np.float64)
    for o in range(n_out):
        assert 0 <= start[o] and start[o] + cnt[o] <= n_in and 1 <= cnt[o] <= maxt
        assert o == 0 or (start[o] >= start[o - 1] and start[o] + cnt[o] >= start[o - 1] + cnt[o - 1])   # taps never move back
        op[o, start[o]:start[o] + cnt[o]] = w[o, :cnt[o]]
    return op


def aten(n_in, n_out, mode, ac, aa, dt):
    eye = torch.eye(n_in, dtype=dt).reshape(1, n_in, 1, n_in)          # n_in "channels", each a one-hot row of width n_in
    kw = {} if ac is None else {"align_corners": ac}
    return F.interpolate(eye, size=(1, n_out), mode=mode, antialias=aa, **kw).reshape(n_in, n_out).t().double().numpy()


@pytest.mark.parametrize("mode,ac,aa", [m for m in MODES if not (m[0] == "bilinear" and m[1] is False)],
                         ids=lambda v: str(v))
@pytest.mark.parametrize("n_in,n_out", GEOMS, ids=lambda v: str(v))
def test_tables_match_aten(built_lib, n_in, n_out, mode, ac, aa):
    """(bilinear with align_corners=False is the table test_cpu_library.py checks; here its export must equal the old one)"""
    maxt, start, cnt, w = table2(built_lib, n_in, n_out, mode, ac, aa)
    op = operator(n_in, maxt, start, cnt, w)
    assert maxt == cnt.max()                                            # tables are packed to their widest output
    if mode == "nearest":
        ref = aten(n_in, n_out, mode, ac, aa, torch.float32)
        assert maxt == 1 and np.array_equal(op, ref)
        return
    exact = aa or mode == "area"
    ref = aten(n_in, n_out, mode, ac, aa, torch.float64 if exact else torch.float32)
    err = np.abs(op - ref).max()
    assert err <= (1e-7 if exact else TOL_PLAIN), err
    if mode == "bicubic" and not aa:
        assert maxt <= 4
    if mode == "bicubic" and n_out >= n_in:
        assert maxt <= 4                                                # bicubic up-scales: the blend's 4-tap path
    if mode in ("area", "bilinear") and n_out >= n_in:
        assert maxt <= 2                                                # the blend's <= 2-tap path


@pytest.mark.parametrize("n_in,n_out", GEOMS, ids=lambda v: str(v))
@pytest.mark.parametrize("aa", [False, True])
def test_bilinear_tables_are_the_old_export(built_lib, n_in, n_out, aa):
    """mode bilinear, align_corners=False through the new export: bit-identical to vsb_debug_resample_table"""
    maxt, start, cnt, w = table2(built_lib, n_in, n_out, "bilinear", False, aa)
    s1 = np.zeros(n_out, dtype=np.int32)
    c1 = np.zeros(n_out, dtype=np.int32)
    w1 = np.zeros(n_out * 256, dtype=np.float32)
    m1 = built_lib.vsb_debug_resample_table(n_in, n_out, int(aa), s1.ctypes.data, c1.ctypes.data, w1.ctypes.data, n_out * 256)
    assert m1 == maxt and np.array_equal(s1, start) and np.array_equal(c1, cnt)
    assert w1[: n_out * maxt].tobytes() == w.tobytes()


def test_resample_table2_rejects_what_interpolate_rejects(built_lib):
    buf = np.zeros(4096, dtype=np.float32)
    idx = np.zeros(256, dtype=np.int32)
    for mode, ac, aa in [("nearest", 1, 0), ("nearest", 0, 1), ("area", 1, 0), ("area", 0, 1)]:
        assert built_lib.vsb_debug_resample_table2(300, 256, _lib.RESIZE_MODES[mode], ac, aa, idx.ctypes.data, idx.ctypes.data,
                                                   buf.ctypes.data, buf.size) < 0
    assert built_lib.vsb_debug_resample_table2(300, 256, 4, 0, 0, idx.ctypes.data, idx.ctypes.data, buf.ctypes.data, buf.size) < 0


# ------------------------------------------------------------------------------------------------------------ the dict
DICT_GRID = [dict(zip(("mode", "align_corners", "antialias"), v)) for v in
             itertools.product(["bilinear", "bicubic", "nearest", "area", "nearest-exact", "linear", "trilinear", "foo"],
                               [None, False, True], [False, True])]
DICT_GRID += [{}, {"mode": "bicubic"}, {"antialias": True}, {"align_corners": False}, {"mode": "bilinear", "scale_factor": 2.0},
              {"mode": "bilinear", "scale_factor": None}, {"mode": "bicubic", "recompute_scale_factor": True},
              {"mode": "bicubic", "recompute_scale_factor": False}, {"mode": "bilinear", "size": 4}, {"mode": "area", "foo": 1}]
DICT_GRID = [{k: v for k, v in d.items() if v is not None or k != "align_corners" or i % 2} for i, d in enumerate(DICT_GRID)]


@pytest.mark.parametrize("interp", DICT_GRID, ids=lambda d: ",".join(f"{k}={v}" for k, v in d.items()) or "empty")
def test_dict_raises_what_interpolate_raises(interp):
    """resize_flags raises the exception type F.interpolate raises on a CPU tensor (none when it accepts the dict), except
    'nearest-exact', which is not implemented (NotImplementedError); with no resize nothing is raised"""
    x = torch.rand(1, 3, 8, 8)
    try:
        F.interpolate(x, size=(4, 4), **interp)
        want = None
    except Exception as e:   # noqa: BLE001 - the type is what is compared
        want = type(e)
    if want is None and interp.get("mode", "nearest") == "nearest-exact":
        want = NotImplementedError
    if want is None:
        f = resize_flags(interp, True)
        mode = interp.get("mode", "nearest")
        assert f >> _lib.FLAG_RESIZE_MODE_SHIFT == _lib.RESIZE_MODES[mode]
        assert bool(f & _lib.FLAG_RESIZE_ALIGN_CORNERS) == bool(interp.get("align_corners"))
        assert bool(f & _lib.FLAG_RESIZE_NO_AA) == (not interp.get("antialias", False))
    else:
        with pytest.raises(want):
            resize_flags(interp, True)
    assert resize_flags(interp, False) == 0


def test_default_dicts_encode_as_before():
    """the defaults of embed / detect and of extract_message: mode bits 0, as the flags were before modes existed"""
    assert resize_flags({"mode": "bilinear", "align_corners": False, "antialias": True}, True) == 0
    assert resize_flags({"mode": "bilinear", "align_corners": False, "antialias": False}, True) == _lib.FLAG_RESIZE_NO_AA
    assert resize_flags({"mode": "bicubic", "align_corners": True, "antialias": True}, True) == (1 << 5) | 16
    assert resize_flags({"mode": "area", "antialias": False}, True) == (3 << 5) | 8


def test_embed_and_detect_validate_before_any_device_work():
    """a rejected dict raises from embed / detect / extract_message on a CPU model (before the missing GPU would), and only when
    the frames are resized"""
    from tests.util import synthetic_card_on_disk
    import videoseal_b200
    cpath, spec, _ = synthetic_card_on_disk("videoseal_1.0", 0, {"num_blocks": 1, "depths": [1, 1, 1, 1]})
    model = videoseal_b200.load(cpath)
    S = spec["img_size"]
    bad = {"mode": "nearest", "align_corners": False, "antialias": False}     # what the reference CLIs build for --interpolation_mode nearest
    x = torch.rand(1, 3, S + 8, S)
    with pytest.raises(ValueError, match="align_corners"):
        model.embed(x, is_video=True, interpolation=bad)
    with pytest.raises(ValueError, match="align_corners"):
        model.detect(x, is_video=True, interpolation=bad)
    with pytest.raises(ValueError, match="align_corners"):
        model.extract_message(x, interpolation=bad)
    with pytest.raises(NotImplementedError, match="nearest-exact"):
        model.detect(x, is_video=True, interpolation={"mode": "nearest-exact"})
    same = torch.rand(1, 3, S, S)
    for call in (lambda: model.embed(same, is_video=True, interpolation=bad), lambda: model.detect(same, is_video=True, interpolation=bad)):
        with pytest.raises(RuntimeError, match="H100"):                 # the dict passes; the CPU model then refuses to run
            call()
    # image-mode detect drops `interpolation` as the reference does (videoseal.py:374)
    with pytest.raises(RuntimeError, match="H100"):
        model.detect(x, is_video=False, interpolation=bad)


# ------------------------------------------------------------------------------------------------------------ the CLIs
class _FakeModel:
    def __init__(self):
        self.blender = type("B", (), {"scaling_w": 0.2})()

    def eval(self):
        return self

    def to(self, device):
        return self


@pytest.mark.parametrize("argv,want", [
    ([], {"mode": "bilinear", "align_corners": False, "antialias": True}),
    (["--interpolation_mode", "bicubic", "--interpolation_antialias", "false"], {"mode": "bicubic", "align_corners": False, "antialias": False}),
    (["--interpolation_mode", "bilinear", "--interpolation_align_corners", "true"], {"mode": "bilinear", "align_corners": True, "antialias": True}),
    (["--interpolation_mode", "nearest", "--interpolation_antialias", "false"], {"mode": "nearest", "align_corners": False, "antialias": False}),
    (["--interpolation_mode", "area"], {"mode": "area", "align_corners": False, "antialias": True}),
])
def test_cli_interpolation_dicts(monkeypatch, tmp_path, argv, want):
    """evals.full and evals.speed parse --interpolation_mode / _align_corners / _antialias into the reference's dict (all three keys,
    evals/full.py:345-349, evals/speed.py:215-219) and hand it to the evaluation"""
    from videoseal_b200 import cfg
    from videoseal_b200.evals import full, speed
    got = {}
    monkeypatch.setattr(cfg, "setup_model_from_checkpoint", lambda ck: _FakeModel())

    def fake_evaluate(model, dataset, is_video, output_dir, num_frames, video_aggregation, **kw):
        got["full"] = kw["interpolation"]
        return [{"psnr": 0.0}]

    monkeypatch.setattr(full, "evaluate", fake_evaluate)
    full.main(["--checkpoint", "x", "--output_dir", str(tmp_path)] + argv)

    def fake_test_speed(self, model, dataset, is_video, num_frames, video_aggregation, lowres_attenuation, interpolation, *a):
        got["speed"] = interpolation
        return {}

    monkeypatch.setattr(speed.SpeedTester, "test_speed", fake_test_speed)
    speed.main(["--checkpoint", "x", "--output_dir", str(tmp_path)] + argv)
    assert got["full"] == want and got["speed"] == want
    with pytest.raises(SystemExit):
        speed.main(["--checkpoint", "x", "--interpolation_mode", "nearest-exact"])


# ------------------------------------------------------------------------------------------------------------ the golden fixture
def test_restatement_matches_the_reference_fixture():
    """oracle/restate.py with every dict of tests/golden/interp.pt reproduces the unmodified reference's outputs stored there
    (tests/make_golden_interp.py asserted the same against the reference itself when it wrote them)"""
    from oracle import restate
    from tests.make_golden_interp import DICTS, TINY, inputs, sub
    from tests.util import apply_overrides, load_card
    gold = torch.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "interp.pt"), weights_only=False)
    assert set(gold["dicts"]) == set(DICTS)
    spec = restate.spec_from_card(apply_overrides(load_card("videoseal_1.0"), TINY))
    orc = restate.OracleModel(spec, restate.synth_state_dict(spec, seed=gold["seed"]))
    orc.step_size, orc.chunk_size = gold["step"], gold["chunk"]
    imgs, clip = inputs()
    for key, r in gold["dicts"].items():
        interp = r["interpolation"]
        with torch.no_grad():
            e = orc.embed(imgs, gold["msgs_img"], is_video=False, interpolation=interp)
            v = orc.embed(clip, gold["msgs_vid"], is_video=True, interpolation=interp)
            p = orc.detect(v["imgs_w"], is_video=True, interpolation=interp)["preds"]
            b = orc.extract_message(v["imgs_w"], interpolation=interp)
        assert torch.equal(sub(e["imgs_w"]), r["img_imgs_w"]) and torch.equal(sub(e["preds_w"]), r["img_preds_w"]), key
        assert torch.equal(sub(v["imgs_w"]), r["vid_imgs_w"]) and torch.equal(p, r["vid_preds"]), key
        assert torch.equal(b, r["extract_bits"]), key
