"""Integer restatement of the JPEG round trip that `utils/image.py:jpeg_compress` performs through PIL (libjpeg-turbo): baseline
4:2:0, accurate integer ("islow") DCT, fancy (triangle) chroma upsampling.  Huffman coding is lossless and left out.  Written
from the algorithm (ITU-T T.81 Annex K tables, the IJG quality rule, the 13-bit fixed-point LL&M DCT) in numpy int64; the
GPU kernels in csrc/augment.cuh follow the same steps, and tests/test_augment_cpu.py checks this file against PIL itself."""
from __future__ import annotations

import numpy as np

# ITU-T T.81 Annex K.1, natural (row-major) order
STD_LUMA = np.array([
    16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
    14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
    49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99], np.int64)
STD_CHROMA = np.array([
    17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
    47, 66, 99, 99, 99, 99, 99, 99] + [99] * 32, np.int64)


def quant_table(base: np.ndarray, quality: int) -> np.ndarray:
    """IJG quality scaling with baseline clamping to 1..255."""
    q = min(max(int(quality), 1), 100)
    scale = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((base * scale + 50) // 100, 1, 255)


def _fix(x: float) -> int:
    return int(x * 65536 + 0.5)


def rgb_to_ycc(rgb: np.ndarray):
    r, g, b = (rgb[..., i].astype(np.int64) for i in range(3))
    half, off = 1 << 15, 128 << 16
    y = (_fix(0.299) * r + _fix(0.587) * g + _fix(0.114) * b + half) >> 16
    cb = (-_fix(0.16874) * r - _fix(0.33126) * g + _fix(0.5) * b + off + half - 1) >> 16
    cr = (_fix(0.5) * r - _fix(0.41869) * g - _fix(0.08131) * b + off + half - 1) >> 16
    return y, cb, cr


def ycc_to_rgb(y, cb, cr) -> np.ndarray:
    half = 1 << 15
    x_cb, x_cr = cb - 128, cr - 128
    r = y + ((_fix(1.402) * x_cr + half) >> 16)
    g = y + ((-_fix(0.34414) * x_cb + half - _fix(0.71414) * x_cr) >> 16)
    b = y + ((_fix(1.772) * x_cb + half) >> 16)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def downsample_h2v2(p: np.ndarray) -> np.ndarray:
    """2x2 box average with libjpeg's ordered-dither bias 1, 2, 1, 2 ... along each output row."""
    s = p[0::2, 0::2] + p[0::2, 1::2] + p[1::2, 0::2] + p[1::2, 1::2]
    bias = np.where(np.arange(s.shape[1]) % 2 == 0, 1, 2)
    return (s + bias) >> 2


C = dict(c0298=2446, c0390=3196, c0541=4433, c0765=6270, c0899=7373, c1175=9633, c1501=12299, c1847=15137, c1961=16069,
         c2053=16819, c2562=20995, c3072=25172)


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _fdct_1d(d, pass1: bool):
    """One pass of the islow forward DCT along the last axis (8 samples)."""
    t0, t7 = d[..., 0] + d[..., 7], d[..., 0] - d[..., 7]
    t1, t6 = d[..., 1] + d[..., 6], d[..., 1] - d[..., 6]
    t2, t5 = d[..., 2] + d[..., 5], d[..., 2] - d[..., 5]
    t3, t4 = d[..., 3] + d[..., 4], d[..., 3] - d[..., 4]
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    out = [None] * 8
    sh = 13 - 2 if pass1 else 13 + 2
    if pass1:
        out[0], out[4] = (t10 + t11) << 2, (t10 - t11) << 2
    else:
        out[0], out[4] = _descale(t10 + t11, 2), _descale(t10 - t11, 2)
    z1 = (t12 + t13) * C["c0541"]
    out[2] = _descale(z1 + t13 * C["c0765"], sh)
    out[6] = _descale(z1 - t12 * C["c1847"], sh)
    z1, z2, z3, z4 = t4 + t7, t5 + t6, t4 + t6, t5 + t7
    z5 = (z3 + z4) * C["c1175"]
    t4, t5, t6, t7 = t4 * C["c0298"], t5 * C["c2053"], t6 * C["c3072"], t7 * C["c1501"]
    z1, z2, z3, z4 = -z1 * C["c0899"], -z2 * C["c2562"], -z3 * C["c1961"] + z5, -z4 * C["c0390"] + z5
    out[7] = _descale(t4 + z1 + z3, sh)
    out[5] = _descale(t5 + z2 + z4, sh)
    out[3] = _descale(t6 + z2 + z3, sh)
    out[1] = _descale(t7 + z1 + z4, sh)
    return np.stack(out, -1)


def fdct(blocks: np.ndarray) -> np.ndarray:
    """[..., 8, 8] level-shifted samples -> DCT coefficients scaled by 8."""
    rows = _fdct_1d(blocks, True)
    return np.swapaxes(_fdct_1d(np.swapaxes(rows, -1, -2), False), -1, -2)


def _idct_1d(d, pass1: bool):
    """One pass of the islow inverse DCT along the last axis."""
    z2, z3 = d[..., 2], d[..., 6]
    z1 = (z2 + z3) * C["c0541"]
    t2, t3 = z1 - z3 * C["c1847"], z1 + z2 * C["c0765"]
    t0, t1 = (d[..., 0] + d[..., 4]) << 13, (d[..., 0] - d[..., 4]) << 13
    t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
    t0, t1, t2, t3 = d[..., 7], d[..., 5], d[..., 3], d[..., 1]
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * C["c1175"]
    t0, t1, t2, t3 = t0 * C["c0298"], t1 * C["c2053"], t2 * C["c3072"], t3 * C["c1501"]
    z1, z2, z3, z4 = -z1 * C["c0899"], -z2 * C["c2562"], -z3 * C["c1961"] + z5, -z4 * C["c0390"] + z5
    t0, t1, t2, t3 = t0 + z1 + z3, t1 + z2 + z4, t2 + z2 + z3, t3 + z1 + z4
    sh = 13 - 2 if pass1 else 13 + 2 + 3
    return np.stack([_descale(t10 + t3, sh), _descale(t11 + t2, sh), _descale(t12 + t1, sh), _descale(t13 + t0, sh),
                     _descale(t13 - t0, sh), _descale(t12 - t1, sh), _descale(t11 - t2, sh), _descale(t10 - t3, sh)], -1)


def range_limit(v):
    """libjpeg's post-IDCT table: clamp(v + 128, 0, 255) for |v| <= 512, wrapping on the low ten bits beyond."""
    x = v & 1023
    return np.where(x < 128, x + 128, np.where(x < 512, 255, np.where(x < 896, 0, x - 896)))


def idct(coef: np.ndarray) -> np.ndarray:
    """[..., 8, 8] dequantised coefficients -> samples 0..255 (columns first, then rows)."""
    cols = np.swapaxes(_idct_1d(np.swapaxes(coef, -1, -2), True), -1, -2)
    return range_limit(_idct_1d(cols, False))


def quantize(coef: np.ndarray, q: np.ndarray) -> np.ndarray:
    """libjpeg-turbo's quantiser: division by 8q through a 16-bit reciprocal, rounding half away from zero."""
    out = np.empty_like(coef)
    for i in range(64):
        d = int(q[i]) * 8
        b = d.bit_length() - 1
        r = 16 + b
        fq, fr, c = (1 << r) // d, (1 << r) % d, d // 2
        if fr == 0:
            fq >>= 1
            r -= 1
        elif fr <= d // 2:
            c += 1
        else:
            fq += 1
        t = coef[..., i // 8, i % 8]
        out[..., i // 8, i % 8] = np.sign(t) * (((np.abs(t) + c) * fq) >> r)
    return out


def _blocks(p: np.ndarray) -> np.ndarray:
    h, w = p.shape
    return p.reshape(h // 8, 8, w // 8, 8).swapaxes(1, 2)


def _unblocks(b: np.ndarray) -> np.ndarray:
    n, m = b.shape[:2]
    return b.swapaxes(1, 2).reshape(n * 8, m * 8)


def _codec(plane: np.ndarray, q: np.ndarray) -> np.ndarray:
    qq = q.reshape(8, 8)
    return _unblocks(idct(quantize(fdct(_blocks(plane) - 128), q) * qq))


def upsample_h2v2_fancy(p: np.ndarray, h: int, w: int) -> np.ndarray:
    """Triangle-filter 2x upsampling of the first (ceil(h/2), ceil(w/2)) samples, edges replicated, cropped to (h, w);
    plain 2x2 replication when ceil(w/2) <= 2."""
    ch, cw = (h + 1) // 2, (w + 1) // 2
    p = p[:ch, :cw]
    if cw <= 2:   # libjpeg-turbo replicates instead when the downsampled width is at most 2
        return np.repeat(np.repeat(p, 2, 0), 2, 1)[:h, :w]
    up = np.concatenate([p[:1], p[:-1]], 0)
    dn = np.concatenate([p[1:], p[-1:]], 0)
    cols = np.stack([3 * p + up, 3 * p + dn], 1).reshape(2 * ch, cw)     # rows 2r (upper) and 2r+1 (lower)
    left = np.concatenate([cols[:, :1], cols[:, :-1]], 1)
    right = np.concatenate([cols[:, 1:], cols[:, -1:]], 1)
    out = np.stack([(3 * cols + left + 8) >> 4, (3 * cols + right + 7) >> 4], 2).reshape(2 * ch, 2 * cw)
    return out[:h, :w]


def jpeg_roundtrip(rgb: np.ndarray, quality: int) -> np.ndarray:
    """uint8 [H, W, 3] -> uint8 [H, W, 3]: what PIL's save(format='JPEG', quality=q) followed by a decode returns."""
    h, w = rgb.shape[:2]
    hp, wp = -(-h // 16) * 16, -(-w // 16) * 16
    # columns are replicated at full resolution up to whole MCUs; rows only up to an even count before the chroma is
    # downsampled, after which the last downsampled chroma row is replicated (libjpeg pads the bottom after downsampling)
    y, cb, cr = rgb_to_ycc(np.pad(rgb, ((0, hp - h), (0, wp - w), (0, 0)), mode="edge"))
    he = h + (h & 1)

    def chroma(p):
        d = downsample_h2v2(np.pad(p[:h], ((0, he - h), (0, 0)), mode="edge"))
        return np.pad(d, ((0, hp // 2 - he // 2), (0, 0)), mode="edge")

    ql, qc = quant_table(STD_LUMA, quality), quant_table(STD_CHROMA, quality)
    y = _codec(y, ql)[:h, :w]
    cb = upsample_h2v2_fancy(_codec(chroma(cb), qc), h, w)
    cr = upsample_h2v2_fancy(_codec(chroma(cr), qc), h, w)
    return ycc_to_rgb(y, cb, cr)
