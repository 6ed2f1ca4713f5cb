"""Float64 references, derived error bounds and mutations for every validation-augmentation kernel (csrc/augment.cuh), judged on
every pixel of the kernel's output.  u = 2^-24 (fp32 unit roundoff); inputs lie in [0, 1], so every colour term is >= 0.

  family        kernel(s)                                     compared with                              bound
  crop / flip   aug_gather_kernel                             the oracle (F.crop, F.hflip)               exact
  rotate        aug_grid_kernel<true>                         the oracle (F.rotate, nearest)             exact
  brightness    aug_color_kernel                              the oracle (adjust_brightness)             exact
  grayscale     aug_color_kernel                              the oracle (0.299 / 0.587 / 0.114)         exact
  jpeg          jpeg_mcu_kernel + jpeg_rgb_kernel             the oracle (PIL)                           0 differing bytes
  contrast      aug_gray_sum_kernel + aug_color_kernel        float64 clamp(f x + f1 o), o = per-image   2u (|f x| + |f1 o|) + |f1| 4u o
                                                              float64 mean of the fp32-weighted gray
  saturation    aug_color_kernel                              the same, o = the pixel's float64 gray     2u (|f x| + |f1 o|) + |f1| 3u o
  hue           aug_color_kernel                              float64 _rgb2hsv, shift, _hsv2rgb          (54 cr + 6 v) u
  blur          aug_blur_h_kernel + aug_blur_v_kernel         float64 separable conv, fp32 taps, reflect 2 k u (|w| (x) |w|) * x
  perspective   aug_grid_kernel<false>                        float64 bilinear at the float64 grid of    R (ex + ey) + 8 u M
                                                              the same fp32 coefficients
  resize        resize_sep_kernel                             float64 F.interpolate(antialias=True)      (maxt_x + maxt_y + 2) 2^-23

Derivations.
* contrast / saturation: f and f1 = 1 - f are the fp32 numbers the kernel takes (torch rounds the Python scalars the same way).
  The fp32 gray (0.2989 r + 0.587 g) + 0.114 b is three products and two sums of non-negative terms: within 3u of its float64
  value.  Contrast's mean sums those grays in fp64 (error ~HW 2^-53, far below u) and rounds once to fp32: |m - o| <= 4u o.  The
  blend rounds f x, f1 m and their sum: 2u (|f x| + |f1 o|) + |f1| |m - o|; the clamp cannot increase a difference.
* hue: cr = max - min is rounded once, rc / gc / bc = (max - c) / cr within 3u, the raw hue (bc - gc, 2 + rc - bc or 4 + gc - rc,
  |.| <= 5) within 12u, h = fmod(h / 6 + 1, 1) + shift, wrapped, within 8u, h6 = 6 h within 54u.  _hsv2rgb is continuous and
  periodic in h (neighbouring sectors agree at their boundary), with slope v s = cr per unit of h6, so a sector boundary or the
  wrap at 1 does not break the bound: the outputs v, p = v (1 - s), q = v (1 - s f), t = v (1 - s (1 - f)) are within
  54u cr + 6u v.  Channel ties (max == two channels) are exact comparisons of the same fp32 inputs on both sides.
* blur: each pass is a k-term fma chain of non-negative terms: within k u of its float64 value (gamma_k), and the vertical pass
  reads the rounded horizontal result: 2 k u (|w| (x) |w|) * x to first order.
* perspective: x t0, then fma(y, t2, .), then + t4 is within 3u A of float64 (A = |x t0| + |y t2| + |t4|), the denominator
  within 3u D (D = |x p0| + |y p1| + 1); the quotient q, q - 1, + 1, * (W / 2) and - 0.5 add one rounding each:
      ex = (W / 2) u (3 (A + |q| D) / |den| + 4 |q| + 1) + u |ix|,   and ey likewise.
  A sample moves by at most the local range R of its 4 x 4 zero-padded neighbourhood per pixel of grid error; the bilinear
  weights and the four-term sum add <= 8u M, M the neighbourhood's largest value.
* resize: tests/test_fullres_gpu.py's bound for the tap counts of the two axes.

Mutations (each must leave its bound on the inputs the tests use): contrast: the batch's mean instead of each image's, the mean of
the 0.299 luma, f and 1 - f swapped; saturation: the 0.299 gray; hue: the shift negated, the shift not wrapped (h + shift used as
is, the sector clamped to 0..5), sectors 1 and 5 exchanged; blur: zero and replicate padding (on the border only), sigma of
k + 1; perspective: align_corners=True, start and end points swapped, the denominator dropped; resize: antialias off; crop: the
offset moved one row or one column; rotate: the angle negated, the centre moved half a pixel; grayscale: torchvision's 0.2989.
"""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F

U = 2.0 ** -24


def f32(v: float) -> float:
    return float(torch.tensor(float(v), dtype=torch.float32))


TV_GRAY = tuple(f32(c) for c in (0.2989, 0.587, 0.114))
BT601 = tuple(f32(c) for c in (0.299, 0.587, 0.114))


# ------------------------------------------------------------------------------------------------------------- inputs
def pattern(kind: str, H: int, W: int, seed: int = 0) -> torch.Tensor:
    """[3, H, W] fp32 in [0, 1]: random, flat grey, primaries / secondaries, channel ties, ramps, checkerboard"""
    g = torch.Generator().manual_seed(seed)
    yy = torch.arange(H, dtype=torch.float32)[:, None].expand(H, W)
    xx = torch.arange(W, dtype=torch.float32)[None, :].expand(H, W)
    if kind == "random":
        return torch.rand(3, H, W, generator=g)
    if kind == "grey":
        return torch.full((3, H, W), 0.5)
    if kind == "primaries":       # black, the three primaries, the three secondaries and white in vertical bands
        cols = torch.tensor([[0, 0, 0], [1, 0, 0], [0, 1, 0], [0, 0, 1], [1, 1, 0], [0, 1, 1], [1, 0, 1], [1, 1, 1]], dtype=torch.float32)
        return cols[(xx * 8 / W).long().clamp(max=7)].permute(2, 0, 1).contiguous()
    if kind == "ties":            # random levels with two or three equal channels, cycling r == g, g == b, r == b, r == g == b
        x = torch.rand(3, H, W, generator=g)
        m = (xx + yy).long() % 4
        x[1] = torch.where(m == 0, x[0], x[1])
        x[2] = torch.where(m == 1, x[1], x[2])
        x[2] = torch.where(m == 2, x[0], x[2])
        x[1] = torch.where(m == 3, x[0], x[1])
        x[2] = torch.where(m == 3, x[0], x[2])
        return x
    if kind == "hramp":
        r = xx / max(W - 1, 1)
        return torch.stack([r, 1 - r, 0.5 * r + 0.25])
    if kind == "vramp":
        r = yy / max(H - 1, 1)
        return torch.stack([r, r * r, 1 - r])
    if kind == "checker":
        c = ((xx + yy).long() % 2).float()
        return torch.stack([c, 1 - c, 0.25 + 0.5 * c])
    raise ValueError(kind)


KINDS = ("random", "grey", "primaries", "ties", "hramp", "vramp", "checker")


def batch(kinds, H: int, W: int, seed: int = 0) -> torch.Tensor:
    return torch.stack([pattern(k, H, W, seed + i) for i, k in enumerate(kinds)])


# ------------------------------------------------------------------------------------------------------------- judging
def ratio(got: torch.Tensor, ref: torch.Tensor, tol: torch.Tensor) -> float:
    """max |got - ref| / tol (0 / 0 counts as 0: an exact bound)"""
    d = (got.double() - ref.double()).abs()
    tol = torch.as_tensor(tol, dtype=torch.float64).expand_as(d)
    over = torch.where(tol > 0, d / tol.clamp_min(1e-300), torch.where(d > 0, torch.full_like(d, math.inf), torch.zeros_like(d)))
    return over.max().item() if over.numel() else 0.0


def outside(got: torch.Tensor, ref: torch.Tensor, tol) -> torch.Tensor:
    """[..., H, W] bool: where |got - ref| exceeds tol"""
    d = (got.double() - ref.double()).abs()
    return d > torch.as_tensor(tol, dtype=torch.float64)


def border(H: int, W: int, width: int) -> torch.Tensor:
    m = torch.zeros(H, W, dtype=torch.bool)
    m[:width], m[-width:], m[:, :width], m[:, -width:] = True, True, True, True
    return m


# ------------------------------------------------------------------------------------------------------------- colour
def gray64(x: torch.Tensor, w=TV_GRAY) -> torch.Tensor:
    x = x.double()
    return w[0] * x[:, 0:1] + w[1] * x[:, 1:2] + w[2] * x[:, 2:3]


def contrast_ref(x: torch.Tensor, factor: float, mutation: str | None = None):
    """(float64 reference, bound) of Contrast(factor) on [B, 3, H, W]"""
    f, f1 = f32(factor), f32(1.0 - factor)
    if mutation == "swap":
        f, f1 = f1, f
    g = gray64(x, BT601 if mutation == "luma_0.299" else TV_GRAY)
    o = g.mean(dim=(1, 2, 3), keepdim=True)
    if mutation == "batch_mean":
        o = o.mean(dim=0, keepdim=True).expand_as(o)
    xd = x.double()
    ref = (f * xd + f1 * o).clamp(0, 1)
    tol = 2 * U * ((f * xd).abs() + (f1 * o).abs()) + abs(f1) * 4 * U * o
    return ref, tol


def saturation_ref(x: torch.Tensor, factor: float, mutation: str | None = None):
    f, f1 = f32(factor), f32(1.0 - factor)
    o = gray64(x, BT601 if mutation == "gray_0.299" else TV_GRAY)
    xd = x.double()
    ref = (f * xd + f1 * o).clamp(0, 1)
    tol = 2 * U * ((f * xd).abs() + (f1 * o).abs()) + abs(f1) * 3 * U * o
    return ref, tol


def hsv64(x: torch.Tensor):
    """float64 _rgb2hsv of [B, 3, H, W]: (h in [0, 1), s, v, cr)"""
    x = x.double()
    r, g, b = x.unbind(1)
    maxc, minc = x.max(1).values, x.min(1).values
    eqc = maxc == minc
    cr = maxc - minc
    one = torch.ones_like(maxc)
    s = cr / torch.where(eqc, one, maxc)
    crd = torch.where(eqc, one, cr)
    rc, gc, bc = (maxc - r) / crd, (maxc - g) / crd, (maxc - b) / crd
    h = (maxc == r) * (bc - gc) + ((maxc == g) & (maxc != r)) * (2.0 + rc - bc) + ((maxc != g) & (maxc != r)) * (4.0 + gc - rc)
    return torch.fmod(h / 6.0 + 1.0, 1.0), s, maxc, cr


def hue_ref(x: torch.Tensor, shift: float, mutation: str | None = None):
    """(float64 reference, bound, h6) of Hue(shift); h6 = 6 h after the shift, for the sector-boundary band"""
    h, s, v, cr = hsv64(x)
    sh = f32(shift)
    if mutation == "negated":
        sh = -sh
    h = h + sh
    if mutation != "unwrapped":
        h = torch.remainder(h, 1.0)
    h6 = h * 6.0
    fi = torch.floor(h6)
    fr = h6 - fi
    i = fi.clamp(0, 5).long() if mutation == "unwrapped" else torch.remainder(fi, 6).long()
    p = (v * (1 - s)).clamp(0, 1)
    q = (v * (1 - s * fr)).clamp(0, 1)
    t = (v * (1 - s * (1 - fr))).clamp(0, 1)
    table = [(v, t, p), (q, v, p), (p, v, t), (p, q, v), (t, p, v), (v, p, q)]
    if mutation == "sectors_1_5":
        table[1], table[5] = table[5], table[1]
    out = torch.zeros_like(x, dtype=torch.float64)
    for k, (a, b_, c) in enumerate(table):
        m = i == k
        out[:, 0] = torch.where(m, a, out[:, 0])
        out[:, 1] = torch.where(m, b_, out[:, 1])
        out[:, 2] = torch.where(m, c, out[:, 2])
    tol = ((54 * cr + 6 * v) * U).unsqueeze(1)
    return out, tol, h6


HUE_BAND = 64 * 6 * U          # |h6 - nearest integer| within this: a sector boundary the fp32 hue may land on either side of


def hue_band(x: torch.Tensor, h6: torch.Tensor) -> torch.Tensor:
    """[B, H, W] bool: pixels at a sector boundary (h6 within HUE_BAND of an integer, not grey) or with two or three equal channels"""
    x = x.double()
    mx = x.max(1).values
    ties = (x == mx.unsqueeze(1)).sum(1) >= 2
    grey = x.max(1).values == x.min(1).values
    return ((h6 - h6.round()).abs() <= HUE_BAND) & ~grey | ties


def brightness_ref(x: torch.Tensor, factor: float) -> torch.Tensor:
    return (x * f32(factor)).clamp(0, 1)


def grayscale_ref(x: torch.Tensor, mutation: str | None = None) -> torch.Tensor:
    w = TV_GRAY if mutation == "tv_0.2989" else BT601
    g = w[0] * x[:, 0:1] + w[1] * x[:, 1:2] + w[2] * x[:, 2:3]       # fp32, in the reference's order
    return g.expand_as(x).contiguous()


# ------------------------------------------------------------------------------------------------------------- blur
def taps(k: int, sigma_k: int | None = None) -> list:
    """the fp32 1-D Gaussian F.gaussian_blur builds for k taps (sigma of sigma_k, default k)"""
    sk = k if sigma_k is None else sigma_k
    sigma = 0.3 * ((sk - 1) * 0.5 - 1) + 0.8
    half = (k - 1) * 0.5
    xs = torch.linspace(-half, half, steps=k, dtype=torch.float32)
    pdf = torch.exp(-0.5 * (xs / sigma).pow(2))
    return (pdf / pdf.sum()).tolist()


def _sep64(x: torch.Tensor, w: list, mode: str) -> torch.Tensor:
    k = len(w)
    p = k // 2
    C = x.shape[1]
    wt = torch.tensor(w, dtype=torch.float64)
    xp = F.pad(x.double(), [p, p, p, p], mode=mode) if mode != "constant" else F.pad(x.double(), [p, p, p, p])
    y = F.conv2d(xp, wt.view(1, 1, 1, k).expand(C, 1, 1, k), groups=C)
    return F.conv2d(y, wt.view(1, 1, k, 1).expand(C, 1, k, 1), groups=C)


def blur_ref(x: torch.Tensor, k: int, mutation: str | None = None):
    """(float64 reference, bound) of GaussianBlur(k)"""
    w = taps(k, k + 1 if mutation == "sigma_k+1" else None)
    mode = {"zero_pad": "constant", "replicate_pad": "replicate"}.get(mutation, "reflect")
    ref = _sep64(x, w, mode)
    tol = 2 * k * U * _sep64(x.abs(), [abs(v) for v in taps(k)], "reflect")
    return ref, tol


def blur_emulation(x: torch.Tensor, k: int) -> torch.Tensor:
    """aug_blur_h_kernel then aug_blur_v_kernel in fp32: a fma chain per output over the reflect-padded taps, tap 0 first"""
    w = [f32(v) for v in taps(k)]
    p = k // 2

    def fma_pass(t, dim):
        n = t.shape[dim]
        idx = torch.arange(-p, n + p)
        idx = torch.where(idx < 0, -idx, torch.where(idx >= n, 2 * n - 2 - idx, idx))
        tp = t.index_select(dim, idx)
        acc = torch.zeros_like(t)
        for j in range(k):
            acc = (w[j] * tp.narrow(dim, j, n).double() + acc.double()).float()   # fma: exact product, one rounding
        return acc
    return fma_pass(fma_pass(x.float(), 3), 2)


# ------------------------------------------------------------------------------------------------------------- perspective
def perspective_grid64(H: int, W: int, start, end, mutation: str | None = None):
    """float64 (ix, iy, ex, ey) [H, W]: the sample position of every output pixel from the kernel's fp32 coefficients, and the
    bound on the kernel's fp32 error in it"""
    from videoseal_b200 import augmentation as A
    if mutation == "swapped":
        start, end = end, start
    c = A.perspective_coeffs(start, end)
    t = A._rescaled(c[:6], 0.5 * W, 0.5 * H)
    p0, p1 = (0.0, 0.0) if mutation == "no_den" else (c[6], c[7])
    xs = torch.linspace(0.5, W * 1.0 + 0.5 - 1.0, steps=W).double()[None, :].expand(H, W)
    ys = torch.linspace(0.5, H * 1.0 + 0.5 - 1.0, steps=H).double()[:, None].expand(H, W)
    den = xs * p0 + ys * p1 + 1.0
    D = (xs * p0).abs() + (ys * p1).abs() + 1.0
    out = []
    for (a, b, cc), n in (((t[0], t[2], t[4]), W), ((t[1], t[3], t[5]), H)):
        num = xs * a + ys * b + cc
        A_ = (xs * a).abs() + (ys * b).abs() + abs(cc)
        q = num / den
        g = q - 1.0
        i = (g + 1.0) * (n / 2) - 0.5 if mutation != "align_corners" else (g + 1.0) / 2 * (n - 1)
        e = (n / 2) * U * (3 * (A_ + q.abs() * D) / den.abs() + 4 * q.abs() + 1) + U * i.abs()
        out += [i, e]
    return out[0], out[2], out[1], out[3]


def bilinear64(x: torch.Tensor, ix: torch.Tensor, iy: torch.Tensor) -> torch.Tensor:
    """float64 grid_sample (bilinear, zero padding) of [B, C, H, W] at pixel coordinates ix, iy [OH, OW]"""
    x = x.double()
    B, C, H, W = x.shape
    x0, y0 = torch.floor(ix), torch.floor(iy)
    wx, wy = ix - x0, iy - y0
    out = torch.zeros(B, C, *ix.shape, dtype=torch.float64)
    for dy, dx, w in ((0, 0, (1 - wy) * (1 - wx)), (0, 1, (1 - wy) * wx), (1, 0, wy * (1 - wx)), (1, 1, wy * wx)):
        cx, cy = (x0 + dx).long(), (y0 + dy).long()
        ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
        v = x[:, :, cy.clamp(0, H - 1), cx.clamp(0, W - 1)]
        out += torch.where(ok, w, torch.zeros_like(w)) * v * ok
    return out


def _local(x: torch.Tensor, ix: torch.Tensor, iy: torch.Tensor):
    """(range, max) of the zero-padded 4 x 4 neighbourhood rows floor(iy) - 1 .. + 2, columns floor(ix) - 1 .. + 2"""
    x = x.double()
    H, W = x.shape[-2:]
    xp = F.pad(x, [2, 2, 2, 2])
    mx = F.max_pool2d(xp, 4, stride=1)
    mn = -F.max_pool2d(-xp, 4, stride=1)
    r = (torch.floor(iy) + 1).clamp(0, H).long()
    c = (torch.floor(ix) + 1).clamp(0, W).long()
    return (mx - mn)[:, :, r, c], mx[:, :, r, c]


def perspective_ref(x: torch.Tensor, start, end, mutation: str | None = None):
    """(float64 reference, bound) of F.perspective(x, start, end)"""
    H, W = x.shape[-2:]
    ix, iy, ex, ey = perspective_grid64(H, W, start, end, mutation)
    ref = bilinear64(x, ix, iy)
    ix0, iy0, ex0, ey0 = perspective_grid64(H, W, start, end) if mutation else (ix, iy, ex, ey)
    R, M = _local(x, ix0, iy0)
    return ref, R * (ex0 + ey0) + 8 * U * M


def perspective_emulation(x: torch.Tensor, start, end) -> torch.Tensor:
    """aug_grid_kernel<false> in fp32, operation for operation (the fma rounded once through float64)"""
    from videoseal_b200 import augmentation as A
    H, W = x.shape[-2:]
    c = A.perspective_coeffs(start, end)
    t = A._rescaled(c[:6], 0.5 * W, 0.5 * H)
    xs = torch.linspace(0.5, W * 1.0 + 0.5 - 1.0, steps=W)[None, :].expand(H, W)
    ys = torch.linspace(0.5, H * 1.0 + 0.5 - 1.0, steps=H)[:, None].expand(H, W)

    def dot3(a, b, cc):
        return ((ys.double() * b + (xs * f32(a)).double()).float() + f32(cc))
    den = dot3(c[6], c[7], 1.0)
    gx, gy = dot3(t[0], t[2], t[4]) / den - 1.0, dot3(t[1], t[3], t[5]) / den - 1.0
    ix = (gx + 1.0) * f32(0.5 * W) - 0.5
    iy = (gy + 1.0) * f32(0.5 * H) - 0.5
    x0, y0 = torch.floor(ix), torch.floor(iy)
    wx, wy = ix - x0, iy - y0
    ex, sy = 1.0 - wx, 1.0 - wy
    w4 = [sy * ex, sy * wx, wy * ex, wy * wx]
    acc = None
    for q, (dy, dx) in enumerate(((0, 0), (0, 1), (1, 0), (1, 1))):
        cx, cy = (x0 + dx).long(), (y0 + dy).long()
        ok = (cx >= 0) & (cx < W) & (cy >= 0) & (cy < H)
        v = torch.where(ok, x[:, :, cy.clamp(0, H - 1), cx.clamp(0, W - 1)], torch.zeros(()))
        term = v * w4[q]
        acc = term if acc is None else acc + term
    return acc


# ------------------------------------------------------------------------------------------------------------- resize
def resize_ref(x: torch.Tensor, oh: int, ow: int, antialias: bool = True):
    """(float64 reference, bound) of Resize to (oh, ow)"""
    from tests.test_fullres_gpu import maxt, resize64
    H, W = x.shape[-2:]
    tol = (maxt(W, ow, True) + maxt(H, oh, True) + 2) * 2.0 ** -23
    return resize64(x, oh, ow, antialias), tol


# ------------------------------------------------------------------------------------------------------------- exact families
def rotate_mutated(x: torch.Tensor, angle: int, mutation: str) -> torch.Tensor:
    """Rotate(angle) with both turns negated, or with the centre of the second (expand=False) turn moved half a pixel right;
    the latter needs angle % 90 != 0"""
    import torchvision.transforms.functional as TF
    base = angle // 90 * 90
    rest = angle - base
    if mutation == "negated":
        return TF.rotate(TF.rotate(x, -base, expand=True), -rest)
    assert mutation == "centre+0.5" and rest != 0, (angle, mutation)
    y = TF.rotate(x, base, expand=True)
    h, w = y.shape[-2:]
    return TF.rotate(y, rest, center=[w * 0.5 + 0.5, h * 0.5])


MUTATIONS = {
    "contrast": ("batch_mean", "luma_0.299", "swap"),
    "saturation": ("gray_0.299",),
    "hue": ("negated", "unwrapped", "sectors_1_5"),
    "blur": ("zero_pad", "replicate_pad", "sigma_k+1"),
    "perspective": ("align_corners", "swapped", "no_den"),
    "resize": ("no_antialias",),
    "crop": ("row+1", "col+1"),
    "rotate": ("negated", "centre+0.5"),
    "grayscale": ("tv_0.2989",),
}


# ------------------------------------------------------------------------------------------------------------- one cell
FAMILIES = ("flip", "crop", "rotate", "resize", "perspective", "brightness", "contrast", "saturation", "hue", "grayscale", "jpeg",
            "blur")
EXACT = ("flip", "crop", "rotate", "brightness", "grayscale", "jpeg")


def oracle_class(fam: str):
    from tests import augment_oracle as AO
    return {"flip": AO.HorizontalFlip, "crop": AO.Crop, "rotate": AO.Rotate, "resize": AO.Resize, "perspective": AO.Perspective,
            "brightness": AO.Brightness, "contrast": AO.Contrast, "saturation": AO.Saturation, "hue": AO.Hue,
            "grayscale": AO.Grayscale, "jpeg": AO.JPEG, "blur": AO.GaussianBlur}[fam]


def oracle(fam: str, x: torch.Tensor, s, seed: int) -> torch.Tensor:
    torch.manual_seed(seed)
    return oracle_class(fam)()(x.clone(), None, s)[0]


def _contrast_emulation(x: torch.Tensor, factor: float, per_pixel: bool) -> torch.Tensor:
    """aug_gray_sum_kernel + aug_color_kernel in fp32: fp32 gray, fp64 sum rounded once to the fp32 mean, then the blend"""
    c = TV_GRAY
    g = (c[0] * x[:, 0:1] + c[1] * x[:, 1:2]) + c[2] * x[:, 2:3]
    o = g if per_pixel else (g.double().sum(dim=(1, 2, 3), keepdim=True) / g[0].numel()).float()
    return (f32(factor) * x + f32(1.0 - factor) * o).clamp(0, 1)


def emulate(fam: str, x: torch.Tensor, s, seed: int) -> torch.Tensor:
    """fp32 emulation of the kernels of one cell in their operation order (the oracle where torchvision already computes so)"""
    if fam in ("contrast", "saturation"):
        return _contrast_emulation(x, s, fam == "saturation")
    if fam == "blur":
        return blur_emulation(x, s)
    if fam == "perspective":
        from tests import augment_oracle as AO
        torch.manual_seed(seed)
        return perspective_emulation(x, *AO.perspective_params(x.shape[-1], x.shape[-2], s))
    if fam == "resize" and int(s * x.shape[-2]) != x.shape[-2]:
        return resize_emulation(x, int(s * x.shape[-2]), int(s * x.shape[-1]))
    return oracle(fam, x, s, seed)


def resample_table(n_in: int, n_out: int):
    """(start [n_out], weights [n_out, maxt] fp32, zero past each row's count) of the library's host-built resample table"""
    import ctypes as C
    import numpy as np
    from videoseal_b200 import _lib
    start, cnt = np.zeros(n_out, np.int32), np.zeros(n_out, np.int32)
    w = np.zeros(n_out * 64, np.float32)
    maxt = _lib.lib().vsb_debug_resample_table(n_in, n_out, 1, start.ctypes.data_as(C.c_void_p), cnt.ctypes.data_as(C.c_void_p),
                                               w.ctypes.data_as(C.c_void_p), w.size)
    assert maxt > 0
    w = torch.from_numpy(w[: n_out * maxt].reshape(n_out, maxt).copy())
    w[torch.arange(maxt)[None, :] >= torch.from_numpy(cnt)[:, None]] = 0
    return torch.from_numpy(start).long(), w


def resize_emulation(x: torch.Tensor, oh: int, ow: int) -> torch.Tensor:
    """the resize kernel's arithmetic in fp32: the library's fp32 tables, rows then columns, each a fp32 sum of fp32 products"""
    def one_axis(t, dim, n_out):
        start, w = resample_table(t.shape[dim], n_out)
        n_in = t.shape[dim]
        acc = None
        for k in range(w.shape[1]):
            v = t.index_select(dim, (start + k).clamp(max=n_in - 1))
            wk = w[:, k].view([-1 if d == dim % t.dim() else 1 for d in range(t.dim())])
            acc = v * wk if acc is None else acc + v * wk
        return acc
    return one_axis(one_axis(x.float(), 2, oh), 3, ow)


def judge(fam: str, x: torch.Tensor, got: torch.Tensor, s, seed: int, caught: dict | None = None, oracle_out=None,
          band: list | None = None) -> float:
    """err / bound of one cell's output `got` (CPU) on input x; with `caught`, records there each mutation of the family that the
    bound tells apart from `got`.  Exact families return 0 or inf.  Hue also requires the pixels of its branch band to equal
    torchvision (`oracle_out`, else computed) exactly, and appends (band pixels, pixels) to `band`."""
    from tests import augment_oracle as AO
    import torchvision.transforms as T
    import torchvision.transforms.functional as TF
    H, W = x.shape[-2:]
    muts = {}
    tol = 0.0
    mut = caught is not None
    if fam in EXACT:
        ref = oracle(fam, x, s, seed) if oracle_out is None else oracle_out
        if fam == "crop":
            torch.manual_seed(seed)
            i, j, th, tw = T.RandomCrop.get_params(x, output_size=(int(s * H), int(s * W)))
            if mut and th < H:
                muts["row+1"] = TF.crop(x, i + 1 if i + th < H else i - 1, j, th, tw)
            if mut and tw < W:
                muts["col+1"] = TF.crop(x, i, j + 1 if j + tw < W else j - 1, th, tw)
        elif fam == "rotate" and mut:
            muts["negated"] = rotate_mutated(x, s, "negated")
            if s % 90:
                muts["centre+0.5"] = rotate_mutated(x, s, "centre+0.5")
        elif fam == "grayscale" and mut:
            muts["tv_0.2989"] = grayscale_ref(x, "tv_0.2989")
    elif fam == "contrast":
        ref, tol = contrast_ref(x, s)
        muts = {m: contrast_ref(x, s, m)[0] for m in MUTATIONS[fam] if mut}
    elif fam == "saturation":
        ref, tol = saturation_ref(x, s)
        muts = {m: saturation_ref(x, s, m)[0] for m in MUTATIONS[fam] if mut}
    elif fam == "hue":
        ref, tol, h6 = hue_ref(x, s)
        muts = {m: hue_ref(x, s, m)[0] for m in MUTATIONS[fam] if mut}
        bd = hue_band(x, h6)
        if band is not None:
            band.append((int(bd.sum()), bd.numel()))
        bd = bd.unsqueeze(1).expand_as(got)
        tv = AO.Hue()(x.clone(), None, s)[0] if oracle_out is None else oracle_out
        if not torch.equal(got[bd], tv[bd]):
            return math.inf
    elif fam == "blur":
        ref, tol = blur_ref(x, s)
        muts = {m: blur_ref(x, s, m)[0] for m in MUTATIONS[fam] if mut}
        edge = border(H, W, s // 2)
        for m in ("zero_pad", "replicate_pad"):     # border-only defects: caught on the border, and nowhere else
            if m in muts and outside(got, muts[m], tol)[..., ~edge].any():
                muts.pop(m)
    elif fam == "perspective":
        torch.manual_seed(seed)
        start, end = AO.perspective_params(W, H, s)
        ref, tol = perspective_ref(x, start, end)
        muts = {m: perspective_ref(x, start, end, m)[0] for m in MUTATIONS[fam] if mut}
    elif fam == "resize":
        oh, ow = int(s * H), int(s * W)
        if (oh, ow) == (H, W):
            ref = x
        else:
            ref, tol = resize_ref(x, oh, ow)
            if mut:
                muts["no_antialias"] = resize_ref(x, oh, ow, antialias=False)[0]
    else:
        raise ValueError(fam)
    assert got.shape == ref.shape, (fam, s, tuple(got.shape), tuple(ref.shape))
    if caught is not None:
        for m, r in muts.items():
            if r.shape == got.shape and outside(got, r, tol).any():
                caught.setdefault(fam, set()).add(m)
    return ratio(got, ref, tol)


# every strength of the image validation list per family, and the video list's Saturation strengths
STRENGTHS = {
    "flip": [0], "crop": [0.32, 0.45, 0.55, 0.63, 0.71, 0.77, 0.84, 0.89, 0.95, 1.00], "rotate": [5, 10, 30, 45, 90],
    "resize": [0.32, 0.45, 0.55, 0.63, 0.71, 0.77, 0.84, 0.89, 0.95, 1.00], "perspective": [0.1, 0.2, 0.3, 0.4, 0.5, 0.6, 0.7, 0.8],
    "brightness": [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0], "contrast": [0.1, 0.25, 0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0],
    "saturation": [0.5, 1.5], "hue": [-0.4, -0.3, -0.2, -0.1, 0.0, 0.1, 0.2, 0.3, 0.4, 0.5], "grayscale": [-1],
    "jpeg": [40, 50, 60, 70, 80, 90], "blur": [3, 5, 9, 13, 17],
}
