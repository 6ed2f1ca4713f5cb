"""The reference's validation augmentations (videoseal/augmentation/__init__.py, geometric.py, valuemetric.py, sequential.py, and
the temporal attacks of video.py) on the GPU.  Each class has the reference's `forward(image, mask, strength) -> (image, mask)`
and `__repr__`, so that the evaluation's column names match; random draws (crop offsets, sizes, angles, perspective endpoints,
factors) make the reference's torch.randint / torch.rand calls on the global CPU generator in the same order, so a seed gives the
same parameters.  The pixels are computed by libvsb200's vsb_augment kernels (csrc/augment.cuh) on CUDA tensors; CPU tensors
raise, as everywhere in this package.  Masks ([B, 1, H, W]) go through the geometric ops.  The video codecs (H264, H264rgb, H265,
VP9, AV1) need ffmpeg and raise NotImplementedError.

The temporal attacks take a clip [T, 3, H, W] and draw from Python's `random` module in the reference's order, so that
random.seed(s) gives the reference's parameters.  SpeedChange, TemporalReorder and DropFrame re-index frames: the index table is
built on the host with the reference's arithmetic and applied on the device with index_select, so the frame count may change
(speed 0.5 doubles it).  WindowAveraging blends each frame with the mean of its temporal window in vsb_augment's window kernel.
Masks move with the frames of SpeedChange and TemporalReorder; DropFrame and WindowAveraging return the mask unchanged, as the
reference does.  A tuple strength is unpacked into the forward's parameters in order: (window_size, alpha) and (chunk_size, swap_probability), as
the reference's commented-out video rows mean them."""
from __future__ import annotations

import ctypes as C
import math
import random

import torch

from .. import _lib

OPS = {"crop_flip": 0, "grid_nearest": 1, "grid_bilinear": 2, "brightness": 3, "contrast": 4, "saturation": 5, "hue": 6,
       "grayscale": 7, "blur": 8, "jpeg": 9, "resize": 10, "window_avg": 11}


def _require_cuda(x: torch.Tensor):
    if not x.is_cuda:
        raise RuntimeError("videoseal_b200.augmentation runs on CUDA tensors only (no CPU fallback)")


def apply(op: str, x: torch.Tensor, out_hw=None, params=(), aux: torch.Tensor | None = None) -> torch.Tensor:
    """One vsb_augment call on a CUDA fp32 [B, 3, H, W] tensor; returns [B, 3, OH, OW]."""
    _require_cuda(x)
    if x.dim() != 4 or x.shape[1] != 3:
        raise ValueError(f"expected a [B, 3, H, W] tensor, got {tuple(x.shape)}")
    x = x.float().contiguous()
    B, _, H, W = x.shape
    OH, OW = out_hw if out_hw is not None else (H, W)
    y = torch.empty(B, 3, OH, OW, device=x.device, dtype=torch.float32)
    L = _lib.lib()
    code = OPS[op]
    nbytes = L.vsb_augment_workspace_bytes(code, B, H, W)
    if nbytes < 0:
        _lib.check(nbytes)
    ws = torch.empty(max(nbytes, 1), dtype=torch.uint8, device=x.device)
    p = (C.c_float * max(len(params), 1))(*[float(v) for v in params])
    if aux is not None:
        aux = aux.to(device=x.device, dtype=torch.float32).contiguous()
    stream = torch.cuda.current_stream(x.device).cuda_stream
    with torch.cuda.device(x.device):
        _lib.check(L.vsb_augment(code, x.data_ptr(), y.data_ptr(), B, 3, H, W, OH, OW, p, len(params),
                                 aux.data_ptr() if aux is not None else None, ws.data_ptr(), nbytes, stream))
    return y


def _apply_mask(op, mask, *a, **kw):
    """Run a geometric op on a [B, 1, H, W] mask through its 3-channel kernel."""
    if mask is None:
        return None
    return apply(op, mask.expand(-1, 3, -1, -1), *a, **kw)[:, :1]


# ---------------------------------------------------------------- torchvision's parameter arithmetic (host side)
def inverse_affine_matrix(angle: float) -> list:
    """torchvision's _get_inverse_affine_matrix for a rotation by `angle` about the centre (F.rotate passes -angle)."""
    rot = math.radians(angle)
    a, b, c, d = math.cos(rot), -math.sin(rot), math.sin(rot), math.cos(rot)
    return [d, -b, 0.0, -c, a, 0.0]


def affine_output_size(matrix: list, w: int, h: int):
    """torchvision's _compute_affine_output_size (F.rotate with expand=True), in its fp32 arithmetic."""
    pts = torch.tensor([[-0.5 * w, -0.5 * h, 1.0], [-0.5 * w, 0.5 * h, 1.0], [0.5 * w, 0.5 * h, 1.0], [0.5 * w, -0.5 * h, 1.0]])
    theta = torch.tensor(matrix, dtype=torch.float).view(2, 3)
    new_pts = torch.matmul(pts, theta.T)
    min_vals, _ = new_pts.min(dim=0)
    max_vals, _ = new_pts.max(dim=0)
    min_vals += torch.tensor((w * 0.5, h * 0.5))
    max_vals += torch.tensor((w * 0.5, h * 0.5))
    tol = 1e-4
    cmax = torch.ceil((max_vals / tol).trunc_() * tol)
    cmin = torch.floor((min_vals / tol).trunc_() * tol)
    size = cmax - cmin
    return int(size[0]), int(size[1])


def perspective_coeffs(startpoints, endpoints) -> list:
    """torchvision's _get_perspective_coeffs: float64 least squares, rounded to fp32."""
    a = torch.zeros(8, 8, dtype=torch.float64)
    for i, (p1, p2) in enumerate(zip(endpoints, startpoints)):
        a[2 * i, :] = torch.tensor([p1[0], p1[1], 1, 0, 0, 0, -p2[0] * p1[0], -p2[0] * p1[1]])
        a[2 * i + 1, :] = torch.tensor([0, 0, 0, p1[0], p1[1], 1, -p2[1] * p1[0], -p2[1] * p1[1]])
    b = torch.tensor(startpoints, dtype=torch.float64).view(8)
    return torch.linalg.lstsq(a, b, driver="gels").solution.to(torch.float32).tolist()


def _rescaled(theta6, sx: float, sy: float) -> list:
    """theta [2][3] -> theta^T / [sx, sy] as [3][2], in fp32 (torchvision's rescaled_theta)."""
    t = torch.tensor(theta6, dtype=torch.float32).reshape(1, 2, 3)
    return (t.transpose(1, 2) / torch.tensor([sx, sy], dtype=torch.float32)).reshape(6).tolist()


def _linspace_pair(ow: int, oh: int, x0: float, x1: float, y0: float, y1: float) -> torch.Tensor:
    return torch.cat([torch.linspace(x0, x1, steps=ow), torch.linspace(y0, y1, steps=oh)])


def rotate(x: torch.Tensor, angle: float, expand: bool = False) -> torch.Tensor:
    """F.rotate(x, angle, expand=expand): nearest, zero fill."""
    H, W = x.shape[-2:]
    m = inverse_affine_matrix(-angle)
    ow, oh = affine_output_size(m, W, H) if expand else (W, H)
    params = _rescaled(m, 0.5 * W, 0.5 * H) + [0.0, 0.0, 0.0]
    aux = _linspace_pair(ow, oh, -ow * 0.5 + 0.5, ow * 0.5 + 0.5 - 1, -oh * 0.5 + 0.5, oh * 0.5 + 0.5 - 1)
    return apply("grid_nearest", x, (oh, ow), params, aux)


def perspective(x: torch.Tensor, startpoints, endpoints) -> torch.Tensor:
    """F.perspective(x, startpoints, endpoints): bilinear, zero fill."""
    H, W = x.shape[-2:]
    c = perspective_coeffs(startpoints, endpoints)
    params = _rescaled(c[:6], 0.5 * W, 0.5 * H) + [c[6], c[7], 1.0]
    aux = _linspace_pair(W, H, 0.5, W * 1.0 + 0.5 - 1.0, 0.5, H * 1.0 + 0.5 - 1.0)
    return apply("grid_bilinear", x, (H, W), params, aux)


def gaussian_taps(k: int) -> list:
    """The 1-D kernel F.gaussian_blur(img, k) builds (sigma = 0.3 ((k - 1) / 2 - 1) + 0.8), in fp32."""
    sigma = 0.3 * ((k - 1) * 0.5 - 1) + 0.8
    half = (k - 1) * 0.5
    xs = torch.linspace(-half, half, steps=k, dtype=torch.float32)
    pdf = torch.exp(-0.5 * (xs / sigma).pow(2))
    return (pdf / pdf.sum()).tolist()


def _f32(v: float) -> float:
    return float(torch.tensor(float(v), dtype=torch.float32))


def _blend(op: str, x: torch.Tensor, factor: float) -> torch.Tensor:
    if factor < 0:
        raise ValueError(f"{op} factor ({factor}) is not non-negative.")
    return apply(op, x, None, (_f32(factor), _f32(1.0 - float(factor))))


def _randint(lo: int, hi: int) -> int:
    return torch.randint(lo, hi, size=(1,)).item()


# ---------------------------------------------------------------- the reference's classes
class _Aug:
    name = ""

    def __call__(self, image, mask=None, *args):
        return self.forward(image, mask, *args)

    def __repr__(self):
        return self.name


class Identity(_Aug):
    name = "Identity"

    def forward(self, image, mask=None, *args, **kwargs):
        return image, mask


class HorizontalFlip(_Aug):
    name = "HorizontalFlip"

    def forward(self, image, mask=None, *args, **kwargs):
        H, W = image.shape[-2:]
        return apply("crop_flip", image, (H, W), (0, 0, 1)), _apply_mask("crop_flip", mask, (H, W), (0, 0, 1))


class Rotate(_Aug):
    name = "Rotate"

    def __init__(self, min_angle=None, max_angle=None, do90=False):
        self.min_angle, self.max_angle = min_angle, max_angle
        self.base_angles = torch.tensor([-90, 0, 0, 90]) if do90 else torch.tensor([0])

    def get_random_angle(self):
        if self.min_angle is None or self.max_angle is None:
            raise ValueError("min_angle and max_angle must be provided")
        base_angle = self.base_angles[torch.randint(0, len(self.base_angles), size=(1,))].item()
        return base_angle + _randint(self.min_angle, self.max_angle + 1)

    def forward(self, image, mask=None, angle=None):
        angle = angle or self.get_random_angle()
        base_angle = angle // 90 * 90
        angle = angle - base_angle
        image = rotate(rotate(image, base_angle, expand=True), angle)
        if mask is not None:
            mask = rotate(rotate(mask.expand(-1, 3, -1, -1), base_angle, expand=True), angle)[:, :1]
        return image, mask


def _random_size(lo, hi, h, w):
    if lo is None or hi is None:
        raise ValueError("min_size and max_size must be provided")
    return _randint(int(lo * h), int(hi * h) + 1), _randint(int(lo * w), int(hi * w) + 1)


class Resize(_Aug):
    name = "Resize"

    def __init__(self, min_size=None, max_size=None):
        self.min_size, self.max_size = min_size, max_size

    def forward(self, image, mask=None, size=None):
        h, w = image.shape[-2:]
        out = _random_size(self.min_size, self.max_size, h, w) if size is None else (int(size * h), int(size * w))
        if tuple(out) == (h, w):     # F.resize returns its input when the size does not change
            return image, mask
        return apply("resize", image, out), _apply_mask("resize", mask, out)


class Crop(_Aug):
    name = "Crop"

    def __init__(self, min_size=None, max_size=None):
        self.min_size, self.max_size = min_size, max_size

    def get_params(self, h, w, size=None):
        """(i, j, th, tw) as the reference draws them: its size rule, then RandomCrop.get_params."""
        th, tw = _random_size(self.min_size, self.max_size, h, w) if size is None else (int(size * h), int(size * w))
        if h < th or w < tw:
            raise ValueError(f"Required crop size {(th, tw)} is larger than input image size {(h, w)}")
        i, j = (0, 0) if (th, tw) == (h, w) else (_randint(0, h - th + 1), _randint(0, w - tw + 1))
        return i, j, th, tw

    def forward(self, image, mask=None, size=None):
        i, j, th, tw = self.get_params(*image.shape[-2:], size)
        return apply("crop_flip", image, (th, tw), (i, j, 0)), _apply_mask("crop_flip", mask, (th, tw), (i, j, 0))


class Perspective(_Aug):
    name = "Perspective"

    def __init__(self, min_distortion_scale=None, max_distortion_scale=None):
        self.min_distortion_scale, self.max_distortion_scale = min_distortion_scale, max_distortion_scale

    def get_random_distortion_scale(self):
        if self.min_distortion_scale is None or self.max_distortion_scale is None:
            raise ValueError("min_distortion_scale and max_distortion_scale must be provided")
        return self.min_distortion_scale + torch.rand(1).item() * (self.max_distortion_scale - self.min_distortion_scale)

    @staticmethod
    def get_perspective_params(width, height, distortion_scale):
        hh, hw = height // 2, width // 2
        dw, dh = int(distortion_scale * hw), int(distortion_scale * hh)
        topleft = [_randint(0, dw + 1), _randint(0, dh + 1)]
        topright = [_randint(width - dw - 1, width), _randint(0, dh + 1)]
        botright = [_randint(width - dw - 1, width), _randint(height - dh - 1, height)]
        botleft = [_randint(0, dw + 1), _randint(height - dh - 1, height)]
        startpoints = [[0, 0], [width - 1, 0], [width - 1, height - 1], [0, height - 1]]
        return startpoints, [topleft, topright, botright, botleft]

    def forward(self, image, mask=None, distortion_scale=None):
        distortion_scale = distortion_scale or self.get_random_distortion_scale()
        start, end = self.get_perspective_params(image.shape[-1], image.shape[-2], distortion_scale)
        image = perspective(image, start, end)
        if mask is not None:
            mask = perspective(mask.expand(-1, 3, -1, -1), start, end)[:, :1]
        return image, mask


class _Factor(_Aug):
    def __init__(self, min_factor=None, max_factor=None):
        self.min_factor, self.max_factor = min_factor, max_factor

    def get_random_factor(self):
        if self.min_factor is None or self.max_factor is None:
            raise ValueError("min_factor and max_factor must be provided")
        return torch.rand(1).item() * (self.max_factor - self.min_factor) + self.min_factor

    def forward(self, image, mask, factor=None):
        factor = self.get_random_factor() if factor is None else factor
        return self._op(image, factor), mask


class Brightness(_Factor):
    name = "Brightness"

    def _op(self, x, f):
        return _blend("brightness", x, f)


class Contrast(_Factor):
    name = "Contrast"

    def _op(self, x, f):
        return _blend("contrast", x, f)


class Saturation(_Factor):
    name = "Saturation"

    def _op(self, x, f):
        return _blend("saturation", x, f)


class Hue(_Factor):
    name = "Hue"

    def _op(self, x, f):
        if not -0.5 <= f <= 0.5:
            raise ValueError(f"hue_factor ({f}) is not in [-0.5, 0.5].")
        return apply("hue", x, None, (f,))


class Grayscale(_Aug):
    name = "Grayscale"

    def forward(self, image, mask, *args, **kwargs):
        return apply("grayscale", image), mask


class JPEG(_Aug):
    name = "JPEG"

    def __init__(self, min_quality=None, max_quality=None, passthrough=True):
        self.min_quality, self.max_quality, self.passthrough = min_quality, max_quality, passthrough

    def get_random_quality(self):
        if self.min_quality is None or self.max_quality is None:
            raise ValueError("Quality range must be specified")
        return _randint(self.min_quality, self.max_quality + 1)

    def forward(self, image, mask, quality=None):
        quality = quality or self.get_random_quality()
        if not self.passthrough:
            raise NotImplementedError("JPEG(passthrough=False) is not implemented; the validation lists use the pass-through")
        return apply("jpeg", image, None, (quality,)), mask


class GaussianBlur(_Aug):
    name = "GaussianBlur"

    def __init__(self, min_kernel_size=None, max_kernel_size=None):
        self.min_kernel_size, self.max_kernel_size = min_kernel_size, max_kernel_size

    def get_random_kernel_size(self):
        if self.min_kernel_size is None or self.max_kernel_size is None:
            raise ValueError("Kernel size range must be specified")
        k = _randint(self.min_kernel_size, self.max_kernel_size + 1)
        return k + 1 if k % 2 == 0 else k

    def forward(self, image, mask, kernel_size=None):
        kernel_size = kernel_size or self.get_random_kernel_size()
        return apply("blur", image, None, gaussian_taps(int(kernel_size))), mask


class Sequential(_Aug):
    def __init__(self, *transforms):
        self.transforms = transforms

    def forward(self, image, mask, args):
        args = args + (None,) * (len(self.transforms) - len(args))
        for t, a in zip(self.transforms, args):
            image, mask = t(image, mask, a)
        return image, mask

    def __repr__(self):
        return f"{self.transforms}".replace(", ", "_")


class _Codec(_Aug):
    def forward(self, *args, **kwargs):
        raise NotImplementedError(f"{self.name} needs ffmpeg video compression, which this package does not implement; "
                                  "pass an explicit list of image augmentations instead")


class H264(_Codec):
    name = "H264"


class H264rgb(_Codec):
    name = "H264rgb"


class H265(_Codec):
    name = "H265"


class VP9(_Codec):
    name = "VP9"


class AV1(_Codec):
    name = "AV1"


class _Temporal(_Aug):
    """A clip [T, 3, H, W] in, a clip out; a tuple strength fills the forward's parameters in order."""

    def __call__(self, frames, mask=None, *args):
        if len(args) == 1 and isinstance(args[0], tuple):
            args = args[0]
        return self.forward(frames, mask, *args)


def _reindex(frames, mask, idx):
    """frames[idx] and mask[idx] on the device; idx None returns both unchanged"""
    if idx is None:
        return frames, mask
    idx = idx.to(frames.device)
    return frames.index_select(0, idx), (mask.index_select(0, idx) if mask is not None else None)


class SpeedChange(_Temporal):
    def __init__(self, min_speed=0.5, max_speed=1.5):
        self.min_speed, self.max_speed = min_speed, max_speed

    def get_random_speed(self):
        if self.min_speed is None or self.max_speed is None:
            raise ValueError("min_speed and max_speed must be provided")
        return random.uniform(self.min_speed, self.max_speed)

    def get_indices(self, num_frames: int, speed_factor=None):
        """The frame table of forward (video.py:292-307), or None where the reference returns its input: an fp32 linspace,
        rounded and clamped; a speed-up keeps its first num_frames entries."""
        speed_factor = speed_factor if speed_factor is not None else self.get_random_speed()
        if speed_factor == 1.0:
            return None
        if speed_factor < 1.0:
            return torch.linspace(0, num_frames - 1, int(num_frames / speed_factor)).round().long().clamp(0, num_frames - 1)
        idx = torch.linspace(0, num_frames - 1, int(num_frames * speed_factor))
        return idx[:num_frames].round().long().clamp(0, num_frames - 1)

    def forward(self, frames, mask=None, speed_factor=None, *args, **kwargs):
        _require_cuda(frames)
        return _reindex(frames, mask, self.get_indices(frames.shape[0], speed_factor))

    def __repr__(self):
        return f"SpeedChange(min_speed={self.min_speed}, max_speed={self.max_speed})"


class TemporalReorder(_Temporal):
    def __init__(self, min_chunk_size=2, max_chunk_size=5, reorder_prob=0.5):
        self.min_chunk_size, self.max_chunk_size, self.reorder_prob = min_chunk_size, max_chunk_size, reorder_prob

    def get_random_chunk_size(self):
        if self.min_chunk_size is None or self.max_chunk_size is None:
            raise ValueError("min_chunk_size and max_chunk_size must be provided")
        return random.randint(self.min_chunk_size, self.max_chunk_size)

    def get_indices(self, num_frames: int, chunk_size=None, swap_probability=None):
        """The frame table of forward (video.py:352-405), or None where the reference returns its input: one random.random() per
        chunk pair swaps the pair; the frames after the last whole chunk stay."""
        chunk_size = chunk_size if chunk_size is not None else self.get_random_chunk_size()
        swap_probability = swap_probability if swap_probability is not None else self.reorder_prob
        if num_frames < chunk_size * 2:
            return None
        num_chunks = num_frames // chunk_size
        order = list(range(num_chunks))
        for i in range(0, num_chunks - 1, 2):
            if random.random() < swap_probability and i + 1 < num_chunks:
                order[i], order[i + 1] = order[i + 1], order[i]
        usable = num_chunks * chunk_size
        return torch.tensor([c * chunk_size + k for c in order for k in range(chunk_size)] + list(range(usable, num_frames)))

    def forward(self, frames, mask=None, chunk_size=None, swap_probability=None, *args, **kwargs):
        _require_cuda(frames)
        return _reindex(frames, mask, self.get_indices(frames.shape[0], chunk_size, swap_probability))

    def __repr__(self):
        return (f"TemporalReorder(min_chunk_size={self.min_chunk_size}, max_chunk_size={self.max_chunk_size}, "
                f"reorder_prob={self.reorder_prob})")


class WindowAveraging(_Temporal):
    def __init__(self, min_window_size=2, max_window_size=5, min_alpha=0.3, max_alpha=0.7):
        self.min_window_size, self.max_window_size = min_window_size, max_window_size
        self.min_alpha, self.max_alpha = min_alpha, max_alpha

    def get_random_window_size(self):
        if self.min_window_size is None or self.max_window_size is None:
            raise ValueError("min_window_size and max_window_size must be provided")
        return random.randint(self.min_window_size, self.max_window_size)

    def get_random_alpha(self):
        if self.min_alpha is None or self.max_alpha is None:
            raise ValueError("min_alpha and max_alpha must be provided")
        return random.uniform(self.min_alpha, self.max_alpha)

    def get_params(self, num_frames: int, window_size=None, alpha=None):
        """(min(window_size, num_frames), alpha) as forward draws them (video.py:455-464), or None where the reference returns its
        input: a clip of at most min_window_size frames, the class's minimum and not the given window."""
        if num_frames <= self.min_window_size:
            return None
        window_size = window_size if window_size is not None else self.get_random_window_size()
        alpha = alpha if alpha is not None else self.get_random_alpha()
        if window_size != int(window_size):
            raise ValueError(f"window_size ({window_size}) must be an integer")
        return min(int(window_size), num_frames), alpha      # video.py:463

    def forward(self, frames, mask=None, window_size=None, alpha=None, *args, **kwargs):
        _require_cuda(frames)
        p = self.get_params(frames.shape[0], window_size, alpha)
        if p is None:
            return frames, mask
        # the blend factors round as torch rounds the Python scalars
        return apply("window_avg", frames, None, (p[0], _f32(p[1]), _f32(1 - p[1]))), mask

    def __repr__(self):
        return f"WindowAveraging(min_window={self.min_window_size}, max_window={self.max_window_size})"


class DropFrame(_Temporal):
    def __init__(self, drop_frame_prob=0.125):
        self.drop_frame_prob = drop_frame_prob

    def get_random_drop_prob(self):
        return self.drop_frame_prob

    def get_indices(self, num_frames: int, drop_prob=None):
        """The frame table of forward (video.py:516-525): one random.random() per frame, and one more for the direction of each
        dropped frame's neighbour, which wraps."""
        drop_prob = drop_prob if drop_prob is not None else self.drop_frame_prob
        idx = list(range(num_frames))
        for i in range(num_frames):
            if random.random() >= drop_prob:
                continue
            idx[i] = (i + (-1 if random.random() < 0.5 else 1)) % num_frames
        return torch.tensor(idx)

    def forward(self, frames, mask=None, drop_prob=None, *args, **kwargs):
        """The mask comes back unchanged, as in the reference."""
        _require_cuda(frames)
        return _reindex(frames, None, self.get_indices(frames.shape[0], drop_prob))[0], mask

    def __repr__(self):
        return f"DropFrame(prob={self.drop_frame_prob})"


def _has_codec(augs) -> bool:
    return any(isinstance(a, _Codec) or (isinstance(a, Sequential) and _has_codec([(t, None) for t in a.transforms])) for a, _ in augs)


def _video_augs() -> list:
    """The reference's full video validation list (augmentation/__init__.py:76-105)."""
    return [
        (Identity(), [0]), (HorizontalFlip(), [0]), (Rotate(), [10, 90]), (Resize(), [0.55, 0.71]), (Crop(), [0.55, 0.71]),
        (Perspective(), [0.5]), (Brightness(), [0.5, 1.5]), (Contrast(), [0.5, 1.5]), (Saturation(), [0.5, 1.5]), (Hue(), [0.25]),
        (Grayscale(), [-1]), (JPEG(), [40]), (GaussianBlur(), [9]), (H264(), [23, 30, 40, 50]), (H264rgb(), [23, 30, 40, 50]),
        (H265(), [23, 30, 40, 50]), (VP9(), [-1]),
    ] + [(Sequential(H264(), Crop(), Brightness()), [(crf, 0.71, 0.5)]) for crf in (23, 30, 40, 50)]


def get_validation_augs(is_video: bool = False, only_identity: bool = False, only_combined: bool = False) -> list:
    """The reference's lists (augmentation/__init__.py:get_validation_augs).  Every non-identity video list holds a codec,
    so it raises NotImplementedError here; pass an explicit list to evals.full.evaluate instead."""
    if only_identity:
        augs = [(Identity(), [0])]
    elif only_combined:
        if is_video:
            augs = [(Identity(), [0]), (Sequential(H264(), Crop(), Brightness()), [(30, 0.71, 0.5)]),
                    (Sequential(H264(), Crop(), Brightness()), [(40, 0.71, 0.5)])]
        else:
            augs = [(Identity(), [0]), (Sequential(JPEG(), Crop(), Brightness()), [(40, 0.71, 0.5)])]
    elif is_video:
        augs = _video_augs()
    else:
        augs = [
            (Identity(), [0]), (HorizontalFlip(), [0]), (Rotate(), [5, 10, 30, 45, 90]),
            (Resize(), [0.32, 0.45, 0.55, 0.63, 0.71, 0.77, 0.84, 0.89, 0.95, 1.00]),
            (Crop(), [0.32, 0.45, 0.55, 0.63, 0.71, 0.77, 0.84, 0.89, 0.95, 1.00]),
            (Perspective(), [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8]),
            (Brightness(), [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0]),
            (Contrast(), [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0]),
            (Hue(), [-0.4, -0.3, -0.2, -0.1, 0.0, 0.1, 0.2, 0.3, 0.4, 0.5]),
            (Grayscale(), [-1]), (JPEG(), [40, 50, 60, 70, 80, 90]), (GaussianBlur(), [3, 5, 9, 13, 17]),
        ] + [(Sequential(JPEG(), Crop(), Brightness()), [(q, 0.71, 0.5)]) for q in (40, 60, 80)]
    if _has_codec(augs):
        raise NotImplementedError("this validation list holds video codecs (H264 / H265 / VP9), which need ffmpeg; "
                                  "pass an explicit list of augmentations instead")
    return augs


def get_codec_free_video_augs() -> list:
    """The reference's video validation list without its codec rows and codec Sequentials, followed by the four temporal attacks
    with the strengths of the list's commented-out block (augmentation/__init__.py:100-104)."""
    return [(a, s) for a, s in _video_augs() if not _has_codec([(a, s)])] + [
        (SpeedChange(), [0.5, 2.0]), (WindowAveraging(), [(3, 1.0)]), (DropFrame(), [0.2, 0.5]), (TemporalReorder(), [(4, 0.7)])]


def column_key(aug, strength) -> str:
    """The evaluation's column suffix for one (augmentation, strength): evals/full.py:199-200."""
    return (str(aug) + f"_{strength}").replace(", ", "_")
