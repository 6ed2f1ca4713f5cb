"""The validation augmentation kernels (csrc/augment.cuh) against the reference's outputs (tests/golden/augment.pt), PIL and
torchvision, and the augmented rows of evals.full on the GPU.

Bounds: flip, crop, rotate (nearest, with torchvision's fp32 grid arithmetic) and JPEG (integer libjpeg arithmetic) are exact.
Brightness and grayscale round like torch and are exact too.  The rest differ only in summation order: contrast's mean (fp64
partials against torch's fp32 mean, ~1e-7), the blur (separable taps against the 2-D product kernel, a few ulp of values <= 1),
hue (division and fmod in fp32, identical operations; 1e-6 covers a changed branch at a max == channel tie), perspective
(identical grid arithmetic, bilinear weights in the same order).  1e-5 absolute covers each with a margin of 10x or more.
Against live torchvision at larger sizes the perspective grid's 3-term products come from the host's BLAS, whose rounding can
differ by an ulp of |grid| <= 2 from the fixture machine's; one ulp moves a bilinear sample by max(H, W) * 2^-24 pixel, and
values in [0, 1] change by at most that much per pixel moved, so that comparison allows 8 such ulps on top of 1e-5."""
import io
import os

import numpy as np
import pytest
import torch
from PIL import Image

from videoseal_b200 import augmentation as A

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment.pt")
EXACT = ("HorizontalFlip", "Crop", "Rotate", "JPEG", "Grayscale", "Brightness", "Identity", "(JPEG_Crop_Brightness)")
TOL = 1e-5


@pytest.fixture(scope="module")
def golden():
    return torch.load(GOLDEN, weights_only=False)


def test_every_image_strength_matches_the_reference(golden):
    x = golden["inputs"]["45x61"].cuda()
    worst = {}
    for aug, strengths in A.get_validation_augs(is_video=False):
        for s in strengths:
            key = A.column_key(aug, s)
            torch.manual_seed(golden["seed"])
            y, _ = aug(x.clone(), None, s)
            want = golden["outputs"][key]
            got = y[..., ::3, ::3].cpu()
            assert got.shape == want.shape, key
            err = (got - want).abs().max().item()
            worst[key] = err
            if key.startswith(EXACT):
                assert err == 0.0, (key, err)
            else:
                assert err <= TOL, (key, err)
    print("max |err| per op:", {k: f"{v:.1e}" for k, v in worst.items() if v})


def _pil(u8: np.ndarray, q: int) -> np.ndarray:
    b = io.BytesIO()
    Image.fromarray(u8).save(b, format="JPEG", quality=q)
    b.seek(0)
    return np.asarray(Image.open(b))


@pytest.mark.parametrize("shape", [(45, 61), (72, 88), (256, 256), (131, 257), (1080, 1920)])
def test_jpeg_is_bit_exact_against_pil(shape, golden):
    g = torch.Generator().manual_seed(shape[0])
    x = torch.rand(2, 3, *shape, generator=g)
    x[1, :, : shape[0] // 2] = 0.5       # a flat half: DC-only blocks
    for q in (40, 50, 60, 70, 80, 90):
        y = A.apply("jpeg", x.cuda(), None, (q,)).cpu()
        for b in range(2):
            u8 = x[b].mul(255).byte().permute(1, 2, 0).numpy()
            want = torch.from_numpy(_pil(u8, q).copy()).permute(2, 0, 1).float() / 255
            passthrough = (want - x[b]) + x[b]
            assert torch.equal(y[b], passthrough), (shape, q, b)
            assert int((y[b] * 255).round().to(torch.uint8).ne(want.mul(255).round().to(torch.uint8)).sum()) == 0


@pytest.mark.parametrize("shape", [(256, 256), (720, 1280)])
def test_geometric_ops_equal_torchvision(shape):
    F = pytest.importorskip("torchvision.transforms.functional")
    x = torch.rand(2, 3, *shape, generator=torch.Generator().manual_seed(9))
    xc = x.cuda()
    assert torch.equal(A.HorizontalFlip()(xc, None, 0)[0].cpu(), F.hflip(x))
    torch.manual_seed(3)
    i, j, h, w = A.Crop().get_params(*shape, 0.55)
    assert torch.equal(A.apply("crop_flip", xc, (h, w), (i, j, 0)).cpu(), F.crop(x, i, j, h, w))
    for angle in (5, 30, 90):
        assert torch.equal(A.rotate(A.rotate(xc, angle // 90 * 90, expand=True), angle % 90).cpu(),
                           F.rotate(F.rotate(x, angle // 90 * 90, expand=True), angle % 90)), angle
    torch.manual_seed(4)
    start, end = A.Perspective.get_perspective_params(shape[1], shape[0], 0.5)
    assert (A.perspective(xc, start, end).cpu() - F.perspective(x, start, end)).abs().max() <= TOL + 8 * max(shape) * 2.0 ** -24
    for k in (3, 17):
        assert (A.GaussianBlur()(xc, None, k)[0].cpu() - F.gaussian_blur(x, k)).abs().max() <= TOL
    out = (int(0.55 * shape[0]), int(0.55 * shape[1]))
    # the embedder's resize kernel, judged against float64 (torch's fp32 CPU path has errors of its own at this scale)
    want = torch.nn.functional.interpolate(x.double(), size=out, mode="bilinear", align_corners=False, antialias=True)
    assert (A.Resize()(xc, None, 0.55)[0].cpu().double() - want).abs().max() <= TOL
    assert (A.Saturation()(xc, None, 1.5)[0].cpu() - F.adjust_saturation(x, 1.5)).abs().max() <= TOL


def test_masks_follow_the_geometric_ops():
    x = torch.rand(1, 3, 40, 56, generator=torch.Generator().manual_seed(2)).cuda()
    m = torch.ones(1, 1, 40, 56, device="cuda")
    torch.manual_seed(1)
    _, mc = A.Crop()(x, m, 0.5)
    assert mc.shape == (1, 1, 20, 28) and bool((mc == 1).all())
    _, mr = A.Rotate()(x, m, 45)
    assert mr.shape == (1, 1, 40, 56) and 0 < float(mr.mean()) < 1


def _eval_model():
    import videoseal_b200
    from tests.util import synthetic_card_on_disk
    card, spec, _ = synthetic_card_on_disk("videoseal_1.0")
    return videoseal_b200.load(card).eval().to("cuda"), spec


def test_evaluate_writes_the_reference_columns(tmp_path, golden):
    import csv
    from videoseal_b200.evals import full, speed
    F = pytest.importorskip("torchvision.transforms.functional")
    model, spec = _eval_model()
    items = list(speed.synthetic_items(2, False, 1, 300, 280, "cuda", seed=5))
    torch.manual_seed(77)
    base = full.evaluate(model, items, is_video=False, output_dir=str(tmp_path / "id"))
    torch.manual_seed(77)
    rows = full.evaluate(model, items, is_video=False, output_dir=str(tmp_path / "all"), only_identity=False)
    names = golden["names"][(False, False, False)]
    with open(tmp_path / "all" / "metrics.csv") as f:
        header = next(csv.reader(f))
    groups = [c[len("bit_acc_"):] for c in header if c.startswith("bit_acc_")]
    assert groups == names
    # the first item only: embed draws each item's message from the global generator, and the crops draw from it before the next
    # item, in the reference as here
    for r0, r in zip(base[:1], rows[:1]):
        for k in ("bit_acc_Identity_0", "pvalue_Identity_0", "capacity_Identity_0", "psnr"):
            assert r0[k] == r[k], k
    # each group against model.detect on imgs_w augmented by torchvision / PIL (the first item: its message is the first draw
    # after the seed; the crops draw from the same generator before the next item's message)
    torch.manual_seed(77)
    for it, (x, _) in enumerate(items[:1]):
        out = model.embed(x.unsqueeze(0), is_video=False)
        imgs_w, msgs = out["imgs_w"], out["msgs"].cpu()
        cpu = imgs_w.cpu()
        u8 = cpu[0].clamp(0, 1).mul(255).byte().permute(1, 2, 0).numpy()
        refs = {"HorizontalFlip_0": F.hflip(cpu), "Brightness_0.5": F.adjust_brightness(cpu, 0.5),
                "JPEG_60": (torch.from_numpy(_pil(u8, 60).copy()).permute(2, 0, 1)[None].float() / 255 - cpu.clamp(0, 1)) + cpu.clamp(0, 1),
                "Rotate_10": F.rotate(F.rotate(cpu, 0, expand=True), 10)}
        for key, ref in refs.items():
            logits = model.detect(ref.cuda(), is_video=False)["preds"][:, 1:].cpu()
            acc = ((logits > 0) == msgs.bool()).float().mean().item()
            unsure = int((logits.abs() <= 1e-2 * logits.abs().max()).sum())
            assert abs(rows[it][f"bit_acc_{key}"] - acc) <= (unsure + 0.5) / spec["nbits"], key


def test_evaluate_video_with_an_explicit_list(tmp_path):
    from videoseal_b200.evals import full, speed
    model, _ = _eval_model()
    augs = [(A.Identity(), [0]), (A.HorizontalFlip(), [0]), (A.Crop(), [0.71]), (A.Brightness(), [0.5]), (A.JPEG(), [40])]
    items = list(speed.synthetic_items(1, True, 6, 256, 256, "cuda", seed=3))
    rows = full.evaluate(model, items, is_video=True, output_dir=str(tmp_path), num_frames=6, validation_augs=augs)
    for key in ("HorizontalFlip_0", "Crop_0.71", "Brightness_0.5", "JPEG_40"):
        assert 0.0 <= rows[0][f"bit_acc_{key}"] <= 1.0
