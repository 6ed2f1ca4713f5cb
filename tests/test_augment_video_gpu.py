"""The temporal video attacks on the GPU: every class against the reference's outputs (tests/golden/augment_video.pt), the window
kernel (vsb_augment op 11) on every pixel of 72 x 3 x 1080 x 1920 clips against a float64 restatement, and the codec-free video
rows of evals.full.

Bound of the window kernel.  Output i is fl(fl(a_keep x_i) + fl(a_avg fl(s / n))), s the fp32 sum of the window's n frames in
frame order.  With u = 2^-24 and M the largest |x| in the window, the sum is off by at most (n - 1) u n M, the mean by
(n - 1) u M + u M, and the two products and the add by u each of their operands, so
    |y - y64| <= (n + 4) u M (|a_keep| + |a_avg|)   (first order; 1 % on top covers the rest)
against y64 = a_keep x_i + a_avg mean64, where a_keep and a_avg are the fp32 factors the kernel multiplies with.  Two mutated
restatements must leave this bound: the half-open window x[i - h : i + h] (a frame short) and a running add / subtract sum over
the clip, which carries the rounding of a bright frame into windows that no longer hold it."""
import os
import random

import pytest
import torch

from videoseal_b200 import augmentation as A

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment_video.pt")
U = 2.0 ** -24
REINDEX = ("SpeedChange", "TemporalReorder", "DropFrame")


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def _call(aug, x, m, case):
    random.seed(case["seed"])
    if case["kind"] == "kw":
        return aug.forward(x, m, **case["arg"])
    if case["kind"] == "strength":
        return aug(x, m, case["arg"])
    return aug(x, m)


def test_every_class_matches_the_reference(golden):
    for case in golden["cases"]:
        T = case["T"]
        x = (golden["clips"][T].float() / 255).cuda()
        m = torch.arange(T, dtype=torch.float32, device="cuda").view(T, 1, 1, 1).expand(T, 1, *x.shape[-2:]).contiguous()
        aug = getattr(A, case["cls"])(**case["ctor"])
        y, ym = _call(aug, x, m, case)
        if case["cls"] in REINDEX:
            idx = torch.tensor(case["index"], device="cuda")
            assert torch.equal(y, x[idx]), case
            assert torch.equal(ym, m[torch.tensor(case["mask_index"], device="cuda")]), case
        else:
            # the same fp32 operations in the same order as the reference's torch.mean and blend: equal, not merely close
            assert torch.equal(y[..., ::6, ::8].cpu(), case["out"]), case
            assert ym is m


# ---------------------------------------------------------------- the window kernel against float64
def _factors(alpha):
    return A._f32(alpha), A._f32(1 - alpha)


def _restated(x, window, alpha, half_open=False):
    """float64 y64 and the per-element bound; half_open drops the window's last frame (a mutant)"""
    T = x.shape[0]
    h = min(window, T) // 2
    a_avg, a_keep = _factors(alpha)
    x64 = x.double()
    s = torch.zeros_like(x64)
    big = torch.zeros_like(x)
    hi = h - 1 if half_open else h
    for k in range(-h, hi + 1):          # frame i + k into output i
        lo_o, hi_o = max(0, -k), T - max(0, k)
        if hi_o > lo_o:
            s[lo_o:hi_o] += x64[lo_o + k:hi_o + k]
            big[lo_o:hi_o] = torch.maximum(big[lo_o:hi_o], x[lo_o + k:hi_o + k].abs())
    i = torch.arange(T, device=x.device)
    n = (torch.clamp(i + hi + 1, max=T) - torch.clamp(i - h, min=0)).double().view(T, 1, 1, 1)
    y64 = a_keep * x64 + a_avg * (s / n)
    bound = ((n + 4) * U * (abs(a_keep) + abs(a_avg)) * 1.01) * big.double()
    return y64, bound


def _running_sum(x, window, alpha):
    """the mutant that slides one fp32 sum along the clip (add the entering frame, subtract the leaving one)"""
    T = x.shape[0]
    h = min(window, T) // 2
    a_avg, a_keep = _factors(alpha)
    y = torch.empty_like(x)
    s = torch.zeros_like(x[0])
    for j in range(min(T, h + 1)):
        s = s + x[j]
    for i in range(T):
        if i > 0:
            if i + h < T:
                s = s + x[i + h]
            if i - h - 1 >= 0:
                s = s - x[i - h - 1]
        n = min(T, i + h + 1) - max(0, i - h)
        y[i] = a_keep * x[i] + a_avg * (s / n)
    return y


def _window(x, window, alpha):
    a_avg, a_keep = _factors(alpha)
    return A.apply("window_avg", x, None, (window, a_avg, a_keep))


def _clip(T, seed, H=1080, W=1920):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.rand(T, 3, H, W, device="cuda", generator=g)


@pytest.mark.parametrize("T", [1, 2, 3, 5, 72])
def test_window_kernel_on_every_pixel_against_float64(T):
    x = _clip(T, 100 + T)
    for window in (1, 2, 3, 4, 5, 8, 17):
        for alpha in (0.0, 0.3, 0.7, 1.0):
            y = _window(x, window, alpha)
            y64, bound = _restated(x, window, alpha)
            err = (y.double() - y64).abs()
            ratio = (err / bound.clamp_min(1e-300)).max().item()
            print(f"T={T:2d} window={window:2d}{' (> T)' if window > T else ''} alpha={alpha}: max err {err.max().item():.2e}, "
                  f"max err / bound {ratio:.3f}")
            assert ratio <= 1.0, (T, window, alpha, ratio)
            del y, y64, bound, err
    torch.cuda.empty_cache()


def test_the_bound_rejects_both_mutants():
    """On a clip with one bright frame: the kernel stays inside the bound, the half-open window and the running sum do not."""
    x = _clip(72, 7)
    x[10] += 4096.0
    for window, alpha in ((3, 1.0), (5, 0.7), (17, 0.3)):
        y64, bound = _restated(x, window, alpha)
        ok = ((_window(x, window, alpha).double() - y64).abs() / bound).max().item()
        half = ((_restated(x, window, alpha, half_open=True)[0] - y64).abs() / bound).max().item()
        run = ((_running_sum(x, window, alpha).double() - y64).abs() / bound).max().item()
        print(f"window={window} alpha={alpha}: err / bound: kernel {ok:.3f}, half-open {half:.3g}, running sum {run:.3g}")
        assert ok <= 1.0 and half > 1.0 and run > 1.0, (window, ok, half, run)
        del y64, bound
    torch.cuda.empty_cache()


def test_windows_wider_than_17_frames_are_rejected():
    x = _clip(72, 3, 64, 96)
    with pytest.raises(NotImplementedError, match="at most 17 frames"):
        _window(x, 18, 0.5)
    with pytest.raises(NotImplementedError, match="at most 17 frames"):
        A.WindowAveraging()(x, None, (18, 0.5))
    # min(window, T) is what counts: 18 on a 12-frame clip is a 12-frame window, and the class clamps any window first
    y = _window(x[:12], 18, 0.5)
    y64, bound = _restated(x[:12], 18, 0.5)
    assert ((y.double() - y64).abs() <= bound).all()
    assert torch.equal(A.WindowAveraging()(x[:12], None, (18, 0.5))[0], y)
    assert torch.equal(A.WindowAveraging()(x[:12], None, (2 ** 40, 0.5))[0], y)


def test_unaligned_frames_take_the_scalar_path():
    """3 H W not a multiple of 4: frames are not 16-byte aligned, so the kernel reads one float per thread"""
    x = _clip(9, 4, 45, 61)
    for window in (2, 5, 9):
        y64, bound = _restated(x, window, 0.7)
        assert ((_window(x, window, 0.7).double() - y64).abs() <= bound).all(), window


def _abi_window(x, y, window, alpha):
    """op 11 through the C ABI on caller-chosen x and y pointers"""
    import ctypes as C
    from videoseal_b200 import _lib
    a_avg, a_keep = _factors(alpha)
    T, _, H, W = x.shape
    p = (C.c_float * 3)(window, a_avg, a_keep)
    _lib.check(_lib.lib().vsb_augment(A.OPS["window_avg"], x.data_ptr(), y.data_ptr(), T, 3, H, W, H, W, p, 3, None, None, 0,
                                      torch.cuda.current_stream().cuda_stream))


def test_pointers_off_16_byte_alignment_take_the_scalar_path():
    """A contiguous fp32 view may start 4 bytes into its storage: 3 H W is a multiple of 4 here, but x or y is not 16-byte
    aligned, so the kernel must not go wide"""
    T, H, W = 9, 48, 64
    n = T * 3 * H * W
    src = _clip(1, 8, 1, n + 1).view(-1)
    x = src[1:n + 1].view(T, 3, H, W)
    assert x.is_contiguous() and x.data_ptr() % 16 == 4
    for window in (2, 5, 9):
        y64, bound = _restated(x, window, 0.7)
        y = _window(x, window, 0.7)                       # misaligned x, aligned y
        assert ((y.double() - y64).abs() <= bound).all(), window
        assert torch.equal(_window(x.clone(), window, 0.7), y)   # the 16-byte path computes the same values
        out = torch.empty(n + 3, device="cuda")
        for off in (1, 2, 3):                             # aligned x, misaligned y; then both misaligned
            xa = x.clone()
            ya = out[off:off + n].view(T, 3, H, W)
            _abi_window(xa, ya, window, 0.7)
            assert torch.equal(ya, y), (window, off)
            _abi_window(x, ya, window, 0.7)
            assert torch.equal(ya, y), (window, off)


def test_masks_move_with_their_frames():
    T, H, W = 13, 32, 48
    t = torch.arange(T, dtype=torch.float32, device="cuda").view(T, 1, 1, 1)
    x, m = t.expand(T, 3, H, W).contiguous(), t.expand(T, 1, H, W).contiguous()   # frame t holds t
    for aug, s in ((A.SpeedChange(), 0.5), (A.SpeedChange(), 2.0), (A.TemporalReorder(), (3, 1.0)), (A.TemporalReorder(), None)):
        random.seed(4)
        y, ym = aug(x, m, s)
        assert torch.equal(y[:, :1], ym), (aug, s)
    y, ym = A.SpeedChange()(x, m, 0.5)
    assert y.shape[0] == 26
    random.seed(4)
    y, ym = A.DropFrame()(x, m, 0.5)
    assert ym is m and not torch.equal(y, x)          # the reference returns the mask unchanged
    _, ym = A.WindowAveraging()(x, m, (3, 0.7))
    assert ym is m


def test_sequential_dropframe_crop_brightness():
    x = _clip(8, 5, 72, 96)
    random.seed(9)
    torch.manual_seed(9)
    y, _ = A.Sequential(A.DropFrame(), A.Crop(), A.Brightness())(x, None, (0.5, 0.71, 0.5))
    random.seed(9)
    torch.manual_seed(9)
    idx = A.DropFrame().get_indices(8, 0.5)
    i, j, th, tw = A.Crop().get_params(72, 96, 0.71)
    want = (x[idx.cuda(), :, i:i + th, j:j + tw] * 0.5).clamp(0, 1)
    assert y.shape == (8, 3, th, tw) and torch.equal(y, want)


def test_runs_are_deterministic():
    x = _clip(72, 6)
    a = _window(x, 5, 0.3)
    assert torch.equal(a, _window(x, 5, 0.3))
    del a
    for aug in (A.SpeedChange(), A.TemporalReorder(), A.DropFrame(), A.WindowAveraging()):
        outs = []
        for _ in range(2):
            random.seed(12)
            outs.append(aug(x[:20], None)[0])
        assert torch.equal(*outs), aug


def _eval_model():
    import videoseal_b200
    from tests.util import synthetic_card_on_disk
    card, spec, _ = synthetic_card_on_disk("videoseal_1.0")
    return videoseal_b200.load(card).eval().to("cuda"), spec


def test_evaluate_writes_the_codec_free_video_columns(tmp_path):
    import csv
    from videoseal_b200.evals import full, speed
    model, _ = _eval_model()
    augs = A.get_codec_free_video_augs() + [(A.WindowAveraging(), [(3, 0.0)])]
    items = list(speed.synthetic_items(1, True, 16, 256, 256, "cuda", seed=3))
    random.seed(0)
    rows = full.evaluate(model, items, is_video=True, output_dir=str(tmp_path), num_frames=16, validation_augs=augs)
    with open(tmp_path / "metrics.csv") as f:
        header = next(csv.reader(f))
    keys = [A.column_key(a, s) for a, ss in augs for s in ss]
    for stat in ("bit_acc", "pvalue", "log_pvalue", "capacity"):
        assert [c[len(stat) + 1:] for c in header if c.startswith(stat + "_")] == keys, stat
    assert keys[-1] == "WindowAveraging(min_window=2_max_window=5)_(3_0.0)"
    assert "SpeedChange(min_speed=0.5_max_speed=1.5)_0.5" in keys
    assert "TemporalReorder(min_chunk_size=2_max_chunk_size=5_reorder_prob=0.5)_(4_0.7)" in keys
    for stat in ("bit_acc", "pvalue", "log_pvalue", "capacity"):
        assert rows[0][f"{stat}_{keys[-1]}"] == rows[0][f"{stat}_Identity_0"], stat
    for k in keys:
        assert 0.0 <= rows[0][f"bit_acc_{k}"] <= 1.0, k


def test_dvmark_extractor_reads_a_changed_frame_count():
    """A DVMark extractor mixes the frames of each detector call; a clip slowed to twice its length is detected in the
    reference's chunks of the new length."""
    from tests import dvmark_oracle as dv
    from videoseal_b200 import cfg
    from videoseal_b200.model import Videoseal
    card = dv.card("hidden", img_size=256, nbits=96)
    model = Videoseal(cfg.spec_from_card(card))
    sd = dv.synth_state_dict(dv.spec_from_card(card), dv.SEED)
    model.load_state_dict(sd)
    model = model.to("cuda")
    model.chunk_size = 4
    x = torch.rand(7, 3, 256, 256, generator=torch.Generator().manual_seed(2)).cuda()
    slow, _ = A.SpeedChange()(x, None, 0.5)
    assert slow.shape[0] == 14                   # chunks of 4, 4, 4 and 2 frames
    ref = dv.grouped({k: v.to("cuda", torch.float64) for k, v in sd.items()}, slow.double(), 4)
    got = model.detect(slow, is_video=True)["preds"]
    rel = ((got.double() - ref).abs().max() / ref.abs().max()).item()
    assert rel <= 1e-2, rel
    mean = ref[:, 1:].mean(dim=0)
    sure = mean.abs() > 2e-2 * ref.abs().max()
    bits = model.extract_message(slow)[0]
    assert torch.equal(bits[sure].cpu(), (mean > 0)[sure].cpu())
