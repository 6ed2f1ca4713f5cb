"""Writes tests/golden/augment_full.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_augment_full

Runs the UNMODIFIED reference augmentation classes on one batch of two different images of odd size (2 x 3 x 19 x 29: two JPEG
MCUs per axis with partial last ones, an odd chroma height and width, room for the 17-tap blur's reflect padding, a non-square
frame for Rotate 90's expand), reseeding the global generator before each call, and stores every pixel of every strength of the
image validation list, of the video list's Saturation strengths and of the three Sequential rows (~0.9 MB of fp32).  Then checks
that tests/augment_oracle.py gives the same pixels on the same inputs and prints the largest |oracle - reference| per op: 0
everywhere, except where the host BLAS rounds perspective's grid products differently from the reference's call (none on the
machine that wrote the fixture)."""
import os

import torch

from oracle import ref_import
from tests import augment_oracle as AO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "augment_full.pt")
SHAPE = (2, 3, 19, 29)
SEED = 4321
SATURATION = (0.5, 1.5)         # get_validation_augs(is_video=True)'s Saturation strengths


def inputs() -> torch.Tensor:
    """image 0 uniform noise; image 1 smooth colour ramps with a few hue-tie pixels (r == g, g == b, r == g == b) and exact 0 / 1"""
    g = torch.Generator().manual_seed(11)
    x = torch.rand(*SHAPE, generator=g)
    H, W = SHAPE[-2:]
    yy = torch.linspace(0, 1, H)[:, None].expand(H, W)
    xx = torch.linspace(0, 1, W)[None, :].expand(H, W)
    x[1] = torch.stack([xx, yy, 0.5 * (xx + yy)]) + 0.05 * torch.rand(3, H, W, generator=g)
    x[1, :, 3, :] = x[1, 0:1, 3, :]                       # r == g == b
    x[1, 1, 5, :] = x[1, 0, 5, :]                         # r == g
    x[1, 2, 7, :] = x[1, 1, 7, :]                         # g == b
    x[1, :, 9, :4] = torch.tensor([1.0, 0.0, 0.0])[:, None]
    return x.clamp(0, 1)


def cells(A):
    """[(key, augmentation, strength)] of the image list and the video list's Saturation row"""
    out = [(AO.column_key(a, s), a, s) for a, ss in A.get_validation_augs(is_video=False) for s in ss]
    return out + [(f"Saturation_{s}", A.Saturation(), s) for s in SATURATION]


def main():
    ref_import.install_stubs()
    import videoseal.augmentation as A
    x = inputs()
    outs = {}
    for key, aug, s in cells(A):
        torch.manual_seed(SEED)
        outs[key] = aug(x.clone(), None, s)[0].clone()
    mine = {AO.column_key(a, s): (a, s) for a, ss in AO.image_augs() for s in ss}
    mine.update({f"Saturation_{s}": (AO.Saturation(), s) for s in SATURATION})
    assert list(mine) == list(outs), "augment_oracle's list differs from the reference's"
    worst = {}
    for key, (aug, s) in mine.items():
        y, _ = AO.run(aug, x, s, SEED)
        assert y.shape == outs[key].shape, key
        worst[key] = (y - outs[key]).abs().max().item()
    torch.save({"seed": SEED, "input": x, "outputs": outs}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1024:.0f} KB, {len(outs)} outputs")
    print(f"max |oracle - reference| = {max(worst.values()):.3e}; nonzero: {({k: v for k, v in worst.items() if v})}")


if __name__ == "__main__":
    main()
