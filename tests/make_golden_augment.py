"""Writes tests/golden/augment.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_augment

Runs the UNMODIFIED reference augmentation classes (videoseal/augmentation) on seeded inputs at every strength of the image
validation list, reseeding the global generator before each call, and stores every third row and column of each output (the full
tensors would be several MB).  Also stores PIL's JPEG round trip (uint8) at q = 40..90, the reference's random parameter draws for
fixed seeds, and the column names of every validation list."""
import io
import os

import numpy as np
import torch
from PIL import Image

from oracle import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "augment.pt")
SIZES = {"45x61": (45, 61), "72x88": (72, 88)}
QUALITIES = (40, 50, 60, 70, 80, 90)
SEED = 1234


def inputs():
    g = torch.Generator().manual_seed(5)
    return {k: torch.rand(1, 3, h, w, generator=g) for k, (h, w) in SIZES.items()}


def pil_jpeg(u8: np.ndarray, q: int) -> np.ndarray:
    b = io.BytesIO()
    Image.fromarray(u8).save(b, format="JPEG", quality=q)
    b.seek(0)
    return np.asarray(Image.open(b))


def column_names(A, is_video, only_identity, only_combined):
    augs = A.get_validation_augs(is_video=is_video, only_identity=only_identity, only_combined=only_combined)
    return [(str(a) + f"_{s}").replace(", ", "_") for a, ss in augs for s in ss]


def main():
    ref_import.install_stubs()
    import torchvision.transforms as T
    import videoseal.augmentation as A
    imgs = inputs()
    outs = {}
    for aug, strengths in A.get_validation_augs(is_video=False):
        for s in strengths:
            torch.manual_seed(SEED)
            y, _ = aug(imgs["45x61"].clone(), None, s)
            outs[(str(aug) + f"_{s}").replace(", ", "_")] = y[..., ::3, ::3].clone()
    jpeg = {}
    for k, x in imgs.items():
        u8 = x[0].mul(255).byte().permute(1, 2, 0).numpy()
        for q in QUALITIES:
            jpeg[(k, q)] = torch.from_numpy(pil_jpeg(u8, q).copy())
    draws = {}
    for seed in (0, 1, 2):
        torch.manual_seed(seed)
        d = {"crop": T.RandomCrop.get_params(imgs["72x88"], output_size=(int(0.71 * 72), int(0.71 * 88)))}
        d["crop_random"] = A.Crop(0.5, 0.9).forward(imgs["72x88"], None)[0].shape[-2:]
        d["perspective"] = A.Perspective.get_perspective_params(88, 72, 0.5)
        d["perspective_scale"] = A.Perspective(0.1, 0.8).get_random_distortion_scale()
        d["rotate"] = A.Rotate(5, 45).get_random_angle()
        d["resize"] = A.Resize(0.5, 0.9).get_random_size(72, 88)
        d["brightness"] = A.Brightness(0.5, 1.5).get_random_factor()
        d["jpeg"] = A.JPEG(40, 90).get_random_quality()
        d["blur"] = A.GaussianBlur(3, 17).get_random_kernel_size()
        draws[seed] = d
    names = {}
    for is_video in (False, True):
        for oi, oc in ((True, False), (False, True), (False, False)):
            names[(is_video, oi, oc)] = column_names(A, is_video, oi, oc)
    torch.save({"seed": SEED, "inputs": imgs, "outputs": outs, "jpeg": jpeg, "draws": draws, "names": names}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1024:.0f} KB, {len(outs)} outputs")


if __name__ == "__main__":
    main()
