"""Host side of the temporal video attacks, without a GPU: the frame tables and random draws equal the reference's
(tests/golden/augment_video.pt), the column names and the codec-free video list equal the reference's, op 11 of the C ABI checks
its arguments before any CUDA call, and CPU tensors raise."""
import ctypes as C
import os
import random
import re

import pytest
import torch

from videoseal_b200 import _lib
from videoseal_b200 import augmentation as A

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment_video.pt")
CODEC = re.compile(r"^\(?(H264|H264rgb|H265|VP9|AV1)[_)]")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _params(case) -> tuple:
    """The forward's parameters of a fixture call, after the class's (frames, mask)"""
    if case["kind"] == "kw":
        return tuple(case["arg"].values())
    if case["kind"] == "strength":
        return case["arg"] if isinstance(case["arg"], tuple) else (case["arg"],)
    return ()


def test_frame_tables_equal_the_reference(golden):
    n = 0
    for case in golden["cases"]:
        if case["cls"] == "WindowAveraging":
            continue
        T = case["T"]
        aug = getattr(A, case["cls"])(**case["ctor"])
        random.seed(case["seed"])
        idx = aug.get_indices(T, *_params(case))
        got = list(range(T)) if idx is None else idx.tolist()
        assert got == case["index"], case
        # SpeedChange and TemporalReorder move the mask with the frames; DropFrame returns it unchanged, as the reference does
        assert case["mask_index"] == (list(range(T)) if case["cls"] == "DropFrame" else got), case
        n += 1
    assert n > 200


def test_window_parameters_follow_the_reference_draws(golden):
    for case in golden["cases"]:
        if case["cls"] != "WindowAveraging":
            continue
        aug = A.WindowAveraging(**case["ctor"])
        random.seed(case["seed"])
        p = aug.get_params(case["T"], *_params(case))
        # the reference returns its input exactly when the clip has at most min_window_size frames
        assert (p is None) == (case["T"] <= aug.min_window_size), case
    for seed, d in golden["draws"].items():
        random.seed(seed)
        assert A.SpeedChange().get_random_speed() == d["speed"]
        assert A.TemporalReorder().get_random_chunk_size() == d["chunk"]
        assert A.WindowAveraging().get_random_window_size() == d["window"]
        assert A.WindowAveraging().get_random_alpha() == d["alpha"]
        assert random.random() == d["state_after"]
        random.seed(seed)    # forward draws the window, then alpha
        w, alpha = A.WindowAveraging().get_params(72)
        random.seed(seed)
        assert (w, alpha) == (A.WindowAveraging().get_random_window_size(), A.WindowAveraging().get_random_alpha())


def test_column_names_equal_the_reference(golden):
    for name, keys in golden["keys"].items():
        aug = getattr(A, name)()
        assert str(aug) == golden["reprs"][name]
        strengths = {"SpeedChange": [0.5, 2.0], "WindowAveraging": [(3, 1.0)], "DropFrame": [0.2, 0.5], "TemporalReorder": [(4, 0.7)]}
        assert [A.column_key(aug, s) for s in strengths[name]] == keys
    assert A.column_key(A.SpeedChange(), 0.5) == "SpeedChange(min_speed=0.5_max_speed=1.5)_0.5"


def test_codec_free_video_list(golden):
    augs = A.get_codec_free_video_augs()
    names = [A.column_key(a, s) for a, ss in augs for s in ss]
    kept = [n for n in golden["video_names"] if not CODEC.match(n)]
    temporal = [k for name in ("SpeedChange", "WindowAveraging", "DropFrame", "TemporalReorder") for k in golden["keys"][name]]
    assert names == kept + temporal
    assert len(kept) == 19 and len(golden["video_names"]) - len(kept) == 17
    assert not A._has_codec(augs)
    assert [type(a).__name__ for a, _ in augs[-4:]] == ["SpeedChange", "WindowAveraging", "DropFrame", "TemporalReorder"]
    assert [s for _, s in augs[-4:]] == [[0.5, 2.0], [(3, 1.0)], [0.2, 0.5], [(4, 0.7)]]
    # the reference's video list itself still raises here
    with pytest.raises(NotImplementedError):
        A.get_validation_augs(is_video=True)


def _call(op, B=72, Cc=3, H=24, W=40, OH=24, OW=40, params=(3, 0.7, 0.3), n=None):
    L = _lib.lib()
    p = (C.c_float * max(len(params), 1))(*params)
    # fake, never dereferenced device pointers: every rule below is checked before any CUDA call
    return L.vsb_augment(op, C.c_void_p(256), C.c_void_p(512), B, Cc, H, W, OH, OW, p, len(params) if n is None else n, None,
                         None, 0, None)


def test_op_11_checks_its_arguments():
    L = _lib.lib()
    op = A.OPS["window_avg"]
    assert op == 11
    assert L.vsb_augment_workspace_bytes(op, 72, 1080, 1920) == 0
    assert L.vsb_augment_workspace_bytes(12, 72, 24, 40) < 0
    bad = [dict(params=(0, 0.5, 0.5)), dict(params=(-3, 0.5, 0.5)), dict(params=(2.5, 0.5, 0.5)),
           dict(params=(float("nan"), 0.5, 0.5)), dict(params=(3, float("nan"), 0.5)), dict(params=(3, float("inf"), float("-inf"))),
           dict(params=(3, 0.5, float("nan"))), dict(B=0), dict(Cc=4), dict(Cc=1), dict(OH=12), dict(params=(3, 0.5)),
           dict(params=(3, 0.5, 0.5), n=0)]
    for kw in bad:
        assert _call(op, **kw) == -1, (kw, L.vsb_last_error())
    for window in (18, 19, 1000):
        assert _call(op, params=(window, 0.5, 0.5)) == -2, window
        assert "at most 17 frames" in L.vsb_last_error().decode()
    with pytest.raises(NotImplementedError, match="at most 17 frames"):
        _lib.check(_call(op, params=(18, 0.5, 0.5)))


def test_cpu_tensors_raise():
    x = torch.zeros(8, 3, 8, 8)
    for aug, s in ((A.SpeedChange(), 0.5), (A.TemporalReorder(), (2, 1.0)), (A.WindowAveraging(), (3, 0.5)), (A.DropFrame(), 0.5)):
        with pytest.raises(RuntimeError, match="CUDA"):
            aug(x, None, s)
    with pytest.raises(RuntimeError, match="CUDA"):
        A.Sequential(A.DropFrame(), A.Crop(), A.Brightness())(x, None, (0.2, 0.71, 0.5))


def test_codec_free_flag_needs_a_video_bank_run():
    from videoseal_b200.evals import full
    for argv in (["--codec_free_video", "True"], ["--codec_free_video", "True", "--is_video", "True"],
                 ["--codec_free_video", "True", "--only_identity", "False"],
                 ["--codec_free_video", "True", "--is_video", "True", "--only_identity", "False", "--only_combined", "True"]):
        with pytest.raises(SystemExit):
            full.main(["--checkpoint", "x"] + argv)
