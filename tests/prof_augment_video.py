"""Device time of the temporal window-averaging kernel (vsb_augment op 11) on 72-frame clips at 1080p and 2160p, windows 3 and 5,
with CUDA events over repeated calls after a warm-up.  Each call must read the clip once and write it once, T 3 H W 4 bytes each
(3.58 GB per call at 72 x 1080p); the rate is reported against the H100 SXM data-sheet HBM bandwidth of 3.35 TB/s, beside the
card's name and power limit.

    python -m tests.prof_augment_video [out.json]
"""
import json
import subprocess
import sys

import torch

from videoseal_b200 import augmentation as A

T = 72
SIZES = ((1080, 1920), (2160, 3840))
WINDOWS = (3, 5)
PEAK = 3.35e12


def main():
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu, flush=True)
    rows = []
    for H, W in SIZES:
        x = torch.rand(T, 3, H, W, device="cuda")
        nbytes = 2 * T * 3 * H * W * 4
        for window in WINDOWS:
            def fn():
                return A.apply("window_avg", x, None, (window, A._f32(0.5), A._f32(0.5)))
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
            gbs = nbytes / (ms * 1e-3) / 1e9
            rows.append({"T": T, "H": H, "W": W, "window": window, "ms": ms, "bytes": nbytes, "GB/s": gbs,
                         "frac_peak_bw": gbs * 1e9 / PEAK})
            print(f"{T} x 3 x {H} x {W} window {window}: {ms:7.3f} ms  {nbytes / 1e9:5.2f} GB  {gbs:7.0f} GB/s  "
                  f"{rows[-1]['frac_peak_bw'] * 100:5.1f} % of 3.35 TB/s", flush=True)
        del x
        torch.cuda.empty_cache()
    if len(sys.argv) > 1:
        with open(sys.argv[1], "w") as f:
            json.dump({"gpu": gpu, "rows": rows}, f, indent=1)


if __name__ == "__main__":
    main()
