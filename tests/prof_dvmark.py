"""Timing of the DVMark extractor: detect() of 64 x 3x256x256 frames in video mode, two chunks of 32 frames (videoseal_1.0's args with
the `dvmark` extractor and 96 bits, synthetic checkpoint).

    python tests/prof_dvmark.py [--iters N]

Prints the GPU name and power limit, the device-event time per call after 3 warm-up calls, then, from a separate profiled pass, every
DVMark step's time per call (all its launches) with its TFLOP/s: 2 MACs of the 3x3x3 convs (layer1 K = 81, layer2 and layer3
K = 27 x 128 over the map each runs on).
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

B, S, K = 64, 256, 96
PX = B * S * S
FLOPS = {   # step -> flops per call
    "dvmark.conv3x3x3.3-128": 2 * PX * 128 * 81,
    "dvmark.conv3x3x3.128-128": 2 * PX * 128 * 27 * 128,
    "dvmark.conv3x3x3.128-256": 2 * (PX // 4) * 256 * 27 * 128,
}


def timed(fn, iters):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def profile(fn, calls=3):
    from videoseal_b200 import _lib
    L = _lib.lib()
    fn()
    torch.cuda.synchronize()
    L.vsb_profile_enable(1)
    for _ in range(calls):
        fn()
    torch.cuda.synchronize()
    buf = C.create_string_buffer(1 << 16)
    L.vsb_profile_read(buf, len(buf))
    L.vsb_profile_enable(0)
    rows = {}
    for line in buf.value.decode().splitlines():
        name, ms, n = line.split("\t")
        if name.startswith("dvmark."):
            rows[name] = (float(ms) / calls, int(n) // calls)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from tests.test_dvmark_gpu import _model
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip())
    model, _ = _model(S, K)
    model.chunk_size = 32
    x = torch.rand(B, 3, S, S, device="cuda")
    det = lambda: model.detect(x, is_video=True)   # noqa: E731
    print(f"dvmark detect {timed(det, args.iters):.3f} ms per {B} x {S}^2 call (two chunks of 32 frames)")
    for name, (ms, n) in sorted(profile(det).items()):
        fl = FLOPS.get(name.split("@")[0], 0)
        print(f"  {name:44s} {ms:8.3f} ms x{n:<3d}" + (f" {fl / ms / 1e9:8.1f} TFLOP/s" if fl else ""))


if __name__ == "__main__":
    main()
