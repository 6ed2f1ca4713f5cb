"""Every validation-augmentation kernel (csrc/augment.cuh) on every pixel, against the reference's own outputs
(tests/golden/augment_full.pt), the torchvision / PIL oracle (tests/augment_oracle.py) and the float64 references with derived
bounds of tests/augment_kernels.py, at the frame sizes the evaluation meets: 1080p, 720p batches, odd dataset sizes and 4K, on
random and structured inputs; the smallest legal blur images and every JPEG size up to 19 x 19; batch independence and
determinism; one call above 2^31 elements; the profile names of each configuration; and the masks of the geometric ops.  Each
family's bound is printed as the largest err / bound, and every mutation of tests/augment_kernels.py must be told apart."""
import ctypes as C
import os
import time

import pytest
import torch
import torchvision.transforms as T

from tests import augment_kernels as ak
from videoseal_b200 import _lib
from videoseal_b200 import augmentation as A

pytestmark = pytest.mark.gpu

CLASSES = {"flip": A.HorizontalFlip, "crop": A.Crop, "rotate": A.Rotate, "resize": A.Resize, "perspective": A.Perspective,
           "brightness": A.Brightness, "contrast": A.Contrast, "saturation": A.Saturation, "hue": A.Hue, "grayscale": A.Grayscale,
           "jpeg": A.JPEG, "blur": A.GaussianBlur}
KEY_FAMILY = {"HorizontalFlip": "flip", "Crop": "crop", "Rotate": "rotate", "Resize": "resize", "Perspective": "perspective",
              "Brightness": "brightness", "Contrast": "contrast", "Saturation": "saturation", "Hue": "hue", "Grayscale": "grayscale",
              "JPEG": "jpeg", "GaussianBlur": "blur"}
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "augment_full.pt")
TOL = 1e-5          # the fixture contract of the non-exact ops
WORST = {}


def gpu(fam, x, s, seed, mask=None):
    """one evaluation cell on the GPU: (image, mask) on the CPU"""
    torch.manual_seed(seed)
    y, m = CLASSES[fam]()(x.cuda(), None if mask is None else mask.cuda(), s)
    return y.cpu(), (None if m is None else m.cpu())


def note(fam, r, tag):
    assert r <= 1.0, (fam, tag, r)
    WORST[fam] = max(WORST.get(fam, 0.0), r)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nmax err / bound per family:", {k: f"{v:.3f}" for k, v in sorted(WORST.items())})


# ----------------------------------------------------------------------------------------------------- the full-pixel fixture
def test_every_strength_on_every_pixel_of_the_fixture():
    g = torch.load(GOLDEN, weights_only=False)
    x = g["input"]
    cells = [(A.column_key(a, s), a, s) for a, ss in A.get_validation_augs(is_video=False) for s in ss]
    cells += [(f"Saturation_{s}", A.Saturation(), s) for s in (0.5, 1.5)]
    assert [k for k, _, _ in cells] == list(g["outputs"])
    for key, aug, s in cells:
        torch.manual_seed(g["seed"])
        y = aug(x.cuda(), None, s)[0].cpu()
        want = g["outputs"][key]
        assert y.shape == want.shape, key
        fam = KEY_FAMILY.get(key.split("_")[0])
        if fam is None or fam in ak.EXACT or key.startswith("(JPEG"):
            assert torch.equal(y, want), key
        else:
            assert (y - want).abs().max().item() <= TOL, key
            note(fam, ak.judge(fam, x, y, s, g["seed"]), "fixture " + key)


# ----------------------------------------------------------------------------------------------------- real geometries
def _ends(v):
    return [v[0], v[len(v) // 2], v[-1]]


# Every strength where the float64 references stay cheap; the extreme strengths and the middle one at 1080p and above.
GEOMETRIES = {   # name: (H, W, image kinds, strengths per family, require every mutation to be told apart)
    "1080p": (1080, 1920, ("random",), {f: _ends(v) for f, v in ak.STRENGTHS.items()}, False),
    "720p_x3": (720, 1280, ("random", "ties", "checker"), {f: _ends(v) for f, v in ak.STRENGTHS.items()}, False),
    "427x640_x2": (427, 640, ("random", "vramp"), ak.STRENGTHS, True),
    "375x500": (375, 500, ("random",), ak.STRENGTHS, False),
    "structured_375x500": (375, 500, ak.KINDS, ak.STRENGTHS, True),
    "4k": (2160, 3840, ("random",), {f: _ends(v) for f, v in ak.STRENGTHS.items()}, False),
}


@pytest.mark.parametrize("geom", list(GEOMETRIES))
def test_real_geometries_against_float64_and_the_oracle(geom):
    H, W, kinds, strengths, mutations = GEOMETRIES[geom]
    x = ak.batch(kinds, H, W, seed=H + W)
    t0, bands, caught = time.time(), [], {}
    for fam in ak.FAMILIES:
        for s in strengths[fam]:
            y, _ = gpu(fam, x, s, seed=11)
            note(fam, ak.judge(fam, x, y, s, 11, caught=caught if mutations else None, band=bands), f"{geom} {fam} {s}")
    if "random" in kinds and len(kinds) == 1:
        nb, n = map(sum, zip(*bands))
        assert nb <= 1e-3 * n, (geom, nb, n)      # random pixels rarely sit on a sector boundary (~5e-5 of them)
    if mutations:
        for fam, muts in ak.MUTATIONS.items():
            assert caught.get(fam, set()) == set(muts), (geom, fam, caught.get(fam))
    print(f"[{geom}] {time.time() - t0:.1f} s")


# ----------------------------------------------------------------------------------------------------- edges
def test_crop_and_resize_at_1_return_their_input():
    x = torch.rand(2, 3, 375, 500, device="cuda")
    assert A.Resize()(x, None, 1.0)[0] is x
    torch.manual_seed(0)
    assert torch.equal(A.Crop()(x, None, 1.0)[0], x)


@pytest.mark.parametrize("k", [3, 5, 9, 13, 17])
def test_blur_at_the_smallest_legal_images(k):
    n = k // 2 + 1                                  # reflect padding needs k / 2 <= size - 1
    for H, W in ((n, n), (n, 3 * k), (2 * k, n)):
        x = ak.batch(("random", "checker"), H, W, seed=k)
        y, _ = gpu("blur", x, k, 0)
        note("blur", ak.judge("blur", x, y, k, 0), f"blur {k} at {H}x{W}")
    with pytest.raises(RuntimeError):
        A.apply("blur", torch.rand(1, 3, n - 1, n - 1, device="cuda"), None, A.gaussian_taps(k))


def test_jpeg_at_every_size_up_to_19_and_on_strips():
    sizes = [(h, w) for h in range(1, 20) for w in range(1, 20)] + [(1, 1920), (1080, 1), (1, 17), (17, 1), (2, 1921)]
    for h, w in sizes:
        x = ak.batch(("random", "hramp"), h, w, seed=h * 31 + w)
        for q in ((40, 90) if h * w < 400 else (40, 60, 80)):
            y, _ = gpu("jpeg", x, q, 0)
            assert ak.judge("jpeg", x, y, q, 0) == 0.0, (h, w, q)


# ----------------------------------------------------------------------------------------------------- batches
def test_an_image_alone_and_in_a_batch_of_three_are_bit_identical():
    x = ak.batch(("checker", "random", "ties"), 427, 640, seed=5)
    for fam in ak.FAMILIES:
        for s in ak.STRENGTHS[fam]:
            y3, _ = gpu(fam, x, s, 3)
            y1, _ = gpu(fam, x[1:2], s, 3)
            again, _ = gpu(fam, x, s, 3)
            assert torch.equal(y3[1:2], y1), (fam, s)
            assert torch.equal(y3, again), (fam, s)


def test_one_call_above_2_pow_31_elements():
    B, H, W = 346, 1080, 1920
    assert B * 3 * H * W > 2 ** 31
    torch.cuda.reset_peak_memory_stats()
    x = torch.rand(B, 3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    ends = x[[0, B - 1]].cpu()
    t0 = time.time()
    for fam, s in (("flip", 0), ("crop", 0.71), ("contrast", 0.5), ("rotate", 10), ("jpeg", 40)):
        torch.manual_seed(2)
        y = CLASSES[fam]()(x, None, s)[0]
        got = y[[0, B - 1]].cpu()
        del y
        for i in range(2):
            if fam == "crop":       # the window drawn for the whole batch
                torch.manual_seed(2)
                i0, j0, th, tw = T.RandomCrop.get_params(x[:1], output_size=(int(s * H), int(s * W)))
                assert torch.equal(got[i:i + 1], ends[i:i + 1, :, i0:i0 + th, j0:j0 + tw]), fam
            else:
                note(fam, ak.judge(fam, ends[i:i + 1], got[i:i + 1], s, 2), f"2^31 {fam} frame {i}")
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    del x
    torch.cuda.empty_cache()
    print(f"[2^31] {B}x3x{H}x{W}: {time.time() - t0:.1f} s, peak {peak:.1f} GiB")


# ----------------------------------------------------------------------------------------------------- dispatch
def _profiled(fn):
    L = _lib.lib()
    L.vsb_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    return {r.split("\t")[0] for r in buf.value.decode().splitlines() if r}


DISPATCH = {   # (family, strength, H, W): the profile names of one call on one image
    ("flip", 0, 1080, 1920): "crop_flip@1x1080x1920",
    ("crop", 0.71, 1080, 1920): "crop_flip@1x1080x1920",
    ("rotate", 10, 1080, 1920): "grid_nearest@1x1080x1920",
    ("rotate", 90, 1080, 1920): "grid_nearest@1x1080x1920 grid_nearest@1x1920x1080",
    ("perspective", 0.5, 1080, 1920): "grid_bilinear@1x1080x1920",
    ("brightness", 0.5, 1080, 1920): "color0@1x1080x1920",
    ("contrast", 0.5, 1080, 1920): "gray_sum@1x1080x1920 color1@1x1080x1920",
    ("saturation", 1.5, 1080, 1920): "color2@1x1080x1920",
    ("hue", 0.2, 1080, 1920): "color3@1x1080x1920",
    ("grayscale", -1, 1080, 1920): "color4@1x1080x1920",
    ("blur", 17, 1080, 1920): "blur_h@1x1080x1920 blur_v@1x1080x1920",
    ("jpeg", 40, 1080, 1920): "jpeg_mcu@1x1080x1920 jpeg_rgb@1x1080x1920",
    ("resize", 0.32, 1080, 1920): "resize.mt0g2@1x1080x1920",      # 9 taps per column, 2 rows per staging round
    ("resize", 0.71, 1080, 1920): "resize.mt8g2@1x1080x1920",      # 5 taps
    ("resize", 0.32, 2160, 3840): "resize.mt0g1@1x2160x3840",
    ("resize", 0.55, 375, 500): "resize.mt8g4@1x375x500",
}


@pytest.mark.parametrize("cfg", list(DISPATCH), ids=lambda c: f"{c[0]}{c[1]}@{c[2]}x{c[3]}")
def test_profile_names_pin_the_dispatch(cfg):
    fam, s, H, W = cfg
    x = torch.rand(1, 3, H, W, device="cuda")
    names = _profiled(lambda: (torch.manual_seed(0), CLASSES[fam]()(x, None, s)))
    assert names == {"aug." + n for n in DISPATCH[cfg].split()}, (cfg, names)


# ----------------------------------------------------------------------------------------------------- masks
@pytest.mark.parametrize("fam", ["flip", "crop", "rotate", "resize", "perspective"])
def test_masks_follow_the_image_as_the_oracle_masks_do(fam):
    H, W = 427, 640
    x = ak.batch(("random", "checker"), H, W, seed=3)
    m = (torch.rand(2, 1, H // 8 + 1, W // 8 + 1, generator=torch.Generator().manual_seed(4)) > 0.5).float()
    m = m.repeat_interleave(8, 2).repeat_interleave(8, 3)[..., :H, :W].contiguous()
    for s in ak.STRENGTHS[fam]:
        y, ym = gpu(fam, x, s, 9, mask=m)
        torch.manual_seed(9)
        _, om = ak.oracle_class(fam)()(x.clone(), m.clone(), s)
        assert ym.shape == om.shape and ym.shape[1] == 1, (fam, s, ym.shape, om.shape)
        m3 = m.expand(-1, 3, -1, -1).contiguous()
        note(fam, ak.judge(fam, m3, ym.expand(-1, 3, -1, -1), s, 9, oracle_out=om.expand(-1, 3, -1, -1)), f"mask {fam} {s}")
        note(fam, ak.judge(fam, x, y, s, 9), f"image with mask {fam} {s}")
