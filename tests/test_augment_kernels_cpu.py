"""The references of tests/augment_kernels.py and the oracle of tests/augment_oracle.py, checked without a GPU: the oracle gives
the reference's own pixels (tests/golden/augment.pt, every third pixel of one image; tests/golden/augment_full.pt, every pixel of
a batch of two); each derived bound covers an fp32 emulation of its kernel in the kernel's operation order; every mutation of
every family leaves its bound on the structured inputs the GPU tests use, at reduced sizes."""
import os

import pytest
import torch

from tests import augment_kernels as ak
from tests import augment_oracle as AO

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")


def test_oracle_equals_the_sampled_fixture():
    g = torch.load(os.path.join(GOLDEN, "augment.pt"), weights_only=False)
    x = g["inputs"]["45x61"]
    for aug, strengths in AO.image_augs():
        for s in strengths:
            key = AO.column_key(aug, s)
            y, _ = AO.run(aug, x, s, g["seed"])
            assert torch.equal(y[..., ::3, ::3], g["outputs"][key]), key


def test_oracle_equals_the_full_fixture():
    g = torch.load(os.path.join(GOLDEN, "augment_full.pt"), weights_only=False)
    x = g["input"]
    assert x.shape == (2, 3, 19, 29) and not torch.equal(x[0], x[1])
    cells = [(AO.column_key(a, s), a, s) for a, ss in AO.image_augs() for s in ss]
    cells += [(f"Saturation_{s}", AO.Saturation(), s) for s in (0.5, 1.5)]
    assert [k for k, _, _ in cells] == list(g["outputs"])
    for key, aug, s in cells:
        y, _ = AO.run(aug, x, s, g["seed"])
        assert torch.equal(y, g["outputs"][key]), key


def test_resize_at_full_size_returns_its_input():
    x = torch.rand(1, 3, 19, 29)
    assert AO.Resize()(x, None, 1.0)[0] is x


# reduced-size stand-ins of the GPU geometries: odd sizes, a non-square frame, two images per batch at least
SIZES = [(2, 37, 53), (3, 24, 40)]


@pytest.mark.parametrize("fam", ak.FAMILIES)
def test_bounds_cover_the_fp32_emulation_and_catch_every_mutation(fam):
    caught, worst = {}, 0.0
    for (B, H, W), kinds in zip(SIZES, [("random", "ties"), ("primaries", "hramp", "checker")]):
        x = ak.batch(kinds, H, W, seed=H)
        for s in ak.STRENGTHS[fam]:
            got = ak.emulate(fam, x, s, seed=7)
            r = ak.judge(fam, x, got, s, seed=7, caught=caught)
            assert r <= 1.0, (fam, s, (B, H, W), r)
            worst = max(worst, r)
    print(f"[{fam}] max err / bound of the fp32 emulation: {worst:.3f}")
    assert caught.get(fam, set()) == set(ak.MUTATIONS.get(fam, ())), (fam, caught)


def test_blur_padding_mutations_differ_on_the_border_only():
    x = ak.batch(("random",), 20, 27)
    for k in (3, 17):
        ref, tol = ak.blur_ref(x, k)
        inner = ~ak.border(20, 27, k // 2)
        for m in ("zero_pad", "replicate_pad"):
            mut = ak.blur_ref(x, k, m)[0]
            assert torch.equal(mut[..., inner], ref[..., inner]) or (mut - ref)[..., inner].abs().max() <= 1e-15, (k, m)
            assert ak.outside(mut, ref, tol)[..., ~inner].any(), (k, m)
