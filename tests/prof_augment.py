"""Device time of each validation augmentation kernel at 16 x 3 x 1080 x 1920 fp32 (CUDA events over repeated calls, after a
warm-up), with the bytes each op must move and the fraction of the H100 SXM data-sheet 3.35 TB/s that gives.

    python -m tests.prof_augment [out.json]
"""
import json
import subprocess
import sys

import torch

from videoseal_b200 import augmentation as A

B, H, W = 16, 1080, 1920
PEAK = 3.35e12


def cases(x):
    n = B * 3 * H * W * 4
    ch, cw = int(0.71 * H), int(0.71 * W)
    return [
        ("hflip", lambda: A.HorizontalFlip()(x, None, 0), 2 * n),
        ("crop 0.71", lambda: A.apply("crop_flip", x, (ch, cw), (10, 20, 0)), 2 * B * 3 * ch * cw * 4),
        ("rotate 10 (nearest)", lambda: A.rotate(x, 10), 2 * n),
        ("perspective 0.5 (bilinear)", lambda: A.Perspective()(x, None, 0.5), 2 * n),
        ("resize 0.71", lambda: A.apply("resize", x, (ch, cw)), n + B * 3 * ch * cw * 4),
        ("brightness", lambda: A.Brightness()(x, None, 0.5), 2 * n),
        ("contrast", lambda: A.Contrast()(x, None, 0.5), 3 * n),
        ("hue", lambda: A.Hue()(x, None, 0.25), 2 * n),
        ("grayscale", lambda: A.Grayscale()(x, None, -1), 2 * n),
        ("blur 17", lambda: A.GaussianBlur()(x, None, 17), 4 * n),
        ("jpeg 60", lambda: A.JPEG()(x, None, 60), 3 * n + B * H * W * 3),
    ]


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    x = torch.rand(B, 3, H, W, device="cuda")
    rows = []
    for name, fn, nbytes in cases(x):
        for _ in range(3):
            fn()
        torch.cuda.synchronize()
        reps = 20
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(reps):
            fn()
        b.record()
        torch.cuda.synchronize()
        ms = a.elapsed_time(b) / reps
        rows.append({"op": name, "ms": ms, "bytes": nbytes, "frac_peak_bw": nbytes / (ms * 1e-3) / PEAK})
        print(f"{name:28s} {ms:8.3f} ms  {nbytes / 1e9:6.2f} GB  {rows[-1]['frac_peak_bw'] * 100:5.1f} % of 3.35 TB/s", flush=True)
    print("gpu:", gpu)
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump({"gpu": gpu, "shape": [B, 3, H, W], "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
