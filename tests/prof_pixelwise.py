"""Timing of the pixel-wise extractor: detect() of 64 x 3x256x256 frames with convnext_tiny_pw (nbits 256, synthetic checkpoint).

    python tests/prof_pixelwise.py [--iters N] [--preset convnext_tiny_pw]

Prints the GPU name and power limit, the device-event time per detect() call after a warm-up, then (in separate calls) the
per-step CUDA-event profile of the library (vsb_profile_enable), with the bytes the head writes per second against the H100 SXM's
3.35 TB/s and the achieved FLOP/s of the stage GEMMs, both computed from the shapes.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests import pixelwise_oracle as pw  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--preset", default="convnext_tiny_pw")
    ap.add_argument("--batch", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    model, _, spec = pw.model_pair(a.preset, device="cuda")
    B, S, NO = a.batch, spec["img_size"], 1 + spec["nbits"]
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
    for _ in range(3):
        model.detect(x, is_video=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(a.iters):
        model.detect(x, is_video=False)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / a.iters
    print(f"detect {B} x 3x{S}x{S} {a.preset}: {ms:.3f} ms per call = {B / ms * 1e3:.0f} frames/s (device events, {a.iters} calls)")

    from videoseal_b200 import _lib
    L = _lib.lib()
    calls = 3
    L.vsb_profile_enable(1)
    for _ in range(calls):
        model.detect(x, is_video=False)
    torch.cuda.synchronize()
    n = L.vsb_profile_read(None, 0)
    buf = C.create_string_buffer(int(n) + 16)
    L.vsb_profile_read(buf, len(buf))
    L.vsb_profile_enable(0)
    # each row: a step name's total time over the profiled calls and its number of launches; trunk step names repeat once per
    # block, so the time per detect() call is total / calls
    rows = []
    for line in buf.value.decode().splitlines():
        name, tms, cnt = line.split("\t")
        rows.append((name, float(tms) / calls, int(cnt) // calls))
    tot = sum(r[1] for r in rows)
    print(f"per-step profile (ms per detect() call, all steps: {tot:.3f} ms):")
    # shapes of the stages: trunk map S/32, widths C, C/f, ...
    h, c = S // 32, spec["convnext"]["dims"][-1]
    stage = {}
    for f in spec["pixel_decoder"]["upscale_stages"]:
        stage[f"pd.uptap1x1.{c}-{9 * (c // f)}@{h}"] = 2.0 * B * h * h * c * 9 * (c // f)   # FLOPs of the low-resolution tap GEMM
        h, c = h * f, c // f
    for name, t, cnt in sorted(rows, key=lambda r: -r[1]):
        extra = ""
        if name in stage:
            extra = f"  {stage[name] / (t * 1e-3) / 1e12:.1f} TFLOP/s ({stage[name] / 1e9:.1f} GFLOP)"
        if name.startswith("pd.gather_head"):
            by = 4.0 * B * NO * h * h
            extra = (f"  writes {by / 1e9:.2f} GB -> {by / (t * 1e-3) / 1e12:.2f} TB/s = {by / (t * 1e-3) / 3.35e12 * 100:.0f}% of 3.35 TB/s; "
                     f"head {2.0 * B * NO * c * h * h / (t * 1e-3) / 1e12:.1f} TFLOP/s fp32")
        print(f"  {name:40s} {t:8.3f} ms ({cnt} per call){extra}")


if __name__ == "__main__":
    main()
