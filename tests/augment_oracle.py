"""The reference's image validation augmentations (videoseal/augmentation/geometric.py, valuemetric.py, sequential.py) restated
on the CPU through the torchvision / PIL calls they make, with their random draws (torch.randint / torch.rand on the global CPU
generator) in the same order, so that one seed gives the reference's parameters and its pixels.

This is the CPU oracle of tests/test_augment_kernels_gpu.py at sizes no fixture holds (torchvision and PIL are all it needs);
tests/test_augment_kernels_cpu.py checks it against the reference's own outputs (tests/golden/augment.pt, augment_full.pt).
Every class has `forward(image, mask, strength) -> (image, mask)` on [B, 3, H, W] fp32 images and [B, 1, H, W] masks."""
from __future__ import annotations

import io

import torch
import torchvision.transforms as T
import torchvision.transforms.functional as F
from PIL import Image


def _randint(lo: int, hi: int) -> int:
    return torch.randint(lo, hi, size=(1,)).item()


def _uniform(lo: float, hi: float) -> float:
    return torch.rand(1).item() * (hi - lo) + lo


def _size(lo, hi, h, w):
    return _randint(int(lo * h), int(hi * h) + 1), _randint(int(lo * w), int(hi * w) + 1)


class Identity:
    def __call__(self, image, mask=None, *args):
        return image, mask

    def __repr__(self):
        return "Identity"


class HorizontalFlip(Identity):
    def __call__(self, image, mask=None, *args):
        return F.hflip(image), (F.hflip(mask) if mask is not None else None)

    def __repr__(self):
        return "HorizontalFlip"


class Rotate(Identity):
    """base_angle = angle // 90 * 90 first with expand=True, the rest without (nearest, zero fill)"""

    def __init__(self, min_angle=None, max_angle=None, do90=False):
        self.min_angle, self.max_angle = min_angle, max_angle
        self.base_angles = torch.tensor([-90, 0, 0, 90]) if do90 else torch.tensor([0])

    def get_random_angle(self):
        base = self.base_angles[torch.randint(0, len(self.base_angles), size=(1,))].item()
        return base + _randint(self.min_angle, self.max_angle + 1)

    def __call__(self, image, mask=None, angle=None):
        angle = angle or self.get_random_angle()
        base = angle // 90 * 90
        rest = angle - base

        def rot(t):
            return None if t is None else F.rotate(F.rotate(t, base, expand=True), rest)
        return rot(image), rot(mask)

    def __repr__(self):
        return "Rotate"


class Resize(Identity):
    """F.resize(antialias=True); torchvision returns its input unchanged when the size does not change"""

    def __init__(self, min_size=None, max_size=None):
        self.min_size, self.max_size = min_size, max_size

    def __call__(self, image, mask=None, size=None):
        h, w = image.shape[-2:]
        out = _size(self.min_size, self.max_size, h, w) if size is None else (int(size * h), int(size * w))
        rs = lambda t: None if t is None else F.resize(t, list(out), antialias=True)  # noqa: E731
        return rs(image), rs(mask)

    def __repr__(self):
        return "Resize"


class Crop(Identity):
    def __init__(self, min_size=None, max_size=None):
        self.min_size, self.max_size = min_size, max_size

    def __call__(self, image, mask=None, size=None):
        h, w = image.shape[-2:]
        out = _size(self.min_size, self.max_size, h, w) if size is None else (int(size * h), int(size * w))
        i, j, th, tw = T.RandomCrop.get_params(image, output_size=out)
        cr = lambda t: None if t is None else F.crop(t, i, j, th, tw)  # noqa: E731
        return cr(image), cr(mask)

    def __repr__(self):
        return "Crop"


def perspective_params(width: int, height: int, scale: float):
    """(startpoints, endpoints): eight randint draws, corner by corner (x then y), as the reference makes them"""
    dw, dh = int(scale * (width // 2)), int(scale * (height // 2))
    tl = [_randint(0, dw + 1), _randint(0, dh + 1)]
    tr = [_randint(width - dw - 1, width), _randint(0, dh + 1)]
    br = [_randint(width - dw - 1, width), _randint(height - dh - 1, height)]
    bl = [_randint(0, dw + 1), _randint(height - dh - 1, height)]
    return [[0, 0], [width - 1, 0], [width - 1, height - 1], [0, height - 1]], [tl, tr, br, bl]


class Perspective(Identity):
    def __init__(self, min_distortion_scale=None, max_distortion_scale=None):
        self.lo, self.hi = min_distortion_scale, max_distortion_scale

    def __call__(self, image, mask=None, distortion_scale=None):
        scale = distortion_scale or self.lo + torch.rand(1).item() * (self.hi - self.lo)
        start, end = perspective_params(image.shape[-1], image.shape[-2], scale)
        pe = lambda t: None if t is None else F.perspective(t, start, end)  # noqa: E731
        return pe(image), pe(mask)

    def __repr__(self):
        return "Perspective"


class _Factor(Identity):
    fn = None
    name = ""

    def __init__(self, min_factor=None, max_factor=None):
        self.min_factor, self.max_factor = min_factor, max_factor

    def __call__(self, image, mask=None, factor=None):
        factor = _uniform(self.min_factor, self.max_factor) if factor is None else factor
        return type(self).fn(image, factor), mask

    def __repr__(self):
        return self.name


class Brightness(_Factor):
    fn, name = F.adjust_brightness, "Brightness"


class Contrast(_Factor):
    fn, name = F.adjust_contrast, "Contrast"


class Saturation(_Factor):
    fn, name = F.adjust_saturation, "Saturation"


class Hue(_Factor):
    fn, name = F.adjust_hue, "Hue"


class Grayscale(Identity):
    """the reference's own BT.601 weights, not rgb_to_grayscale's 0.2989"""

    def __call__(self, image, mask=None, *args):
        g = 0.299 * image[:, 0:1] + 0.587 * image[:, 1:2] + 0.114 * image[:, 2:3]
        return g.expand_as(image), mask

    def __repr__(self):
        return "Grayscale"


def pil_jpeg(image: torch.Tensor, quality: int) -> torch.Tensor:
    """[3, H, W] in [0, 1] -> ToPILImage, PIL JPEG save at `quality`, decode, ToTensor"""
    b = io.BytesIO()
    T.ToPILImage()(image).save(b, format="JPEG", quality=quality)
    b.seek(0)
    return T.ToTensor()(Image.open(b))


class JPEG(Identity):
    """the pass-through form: (jpeg(x) - x) + x on the clamped image, one image at a time"""

    def __init__(self, min_quality=None, max_quality=None):
        self.min_quality, self.max_quality = min_quality, max_quality

    def __call__(self, image, mask=None, quality=None):
        quality = quality or _randint(self.min_quality, self.max_quality + 1)
        image = torch.clamp(image, 0, 1)
        for i in range(image.shape[0]):
            image[i] = (pil_jpeg(image[i], quality) - image[i]) + image[i]
        return image, mask

    def __repr__(self):
        return "JPEG"


class GaussianBlur(Identity):
    def __init__(self, min_kernel_size=None, max_kernel_size=None):
        self.min_kernel_size, self.max_kernel_size = min_kernel_size, max_kernel_size

    def __call__(self, image, mask=None, kernel_size=None):
        if not kernel_size:
            kernel_size = _randint(self.min_kernel_size, self.max_kernel_size + 1)
            kernel_size += kernel_size % 2 == 0
        return F.gaussian_blur(image, kernel_size), mask

    def __repr__(self):
        return "GaussianBlur"


class Sequential(Identity):
    def __init__(self, *transforms):
        self.transforms = transforms

    def __call__(self, image, mask, args):
        args = args + (None,) * (len(self.transforms) - len(args))
        for t, a in zip(self.transforms, args):
            image, mask = t(image, mask, a)
        return image, mask

    def __repr__(self):
        return f"{self.transforms}".replace(", ", "_")


STEPS = (0.32, 0.45, 0.55, 0.63, 0.71, 0.77, 0.84, 0.89, 0.95, 1.00)


def image_augs() -> list:
    """get_validation_augs(is_video=False): (augmentation, strengths) in the evaluation's column order"""
    return [
        (Identity(), [0]), (HorizontalFlip(), [0]), (Rotate(), [5, 10, 30, 45, 90]), (Resize(), list(STEPS)), (Crop(), list(STEPS)),
        (Perspective(), [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8]),
        (Brightness(), [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0]),
        (Contrast(), [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0]),
        (Hue(), [-0.4, -0.3, -0.2, -0.1, 0.0, 0.1, 0.2, 0.3, 0.4, 0.5]),
        (Grayscale(), [-1]), (JPEG(), [40, 50, 60, 70, 80, 90]), (GaussianBlur(), [3, 5, 9, 13, 17]),
    ] + [(Sequential(JPEG(), Crop(), Brightness()), [(q, 0.71, 0.5)]) for q in (40, 60, 80)]


def column_key(aug, strength) -> str:
    return (str(aug) + f"_{strength}").replace(", ", "_")


def run(aug, x: torch.Tensor, strength, seed: int, mask: torch.Tensor | None = None):
    """one evaluation cell: reseed the global generator, then aug(x.clone(), mask, strength)"""
    torch.manual_seed(seed)
    return aug(x.clone(), None if mask is None else mask.clone(), strength)
