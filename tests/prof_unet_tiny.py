"""Timing of the unet_tiny_yuv_quant embedder against videoseal_1.0's U-Net: embed() of 64 x 3x256x256 frames in image mode
(synthetic checkpoints, nbits 256, JND attenuation as in the card).

    python tests/prof_unet_tiny.py [--iters N] [--batch B]

Prints the GPU name and power limit, the device-event time per embed() call of each model after a warm-up, then (in separate
calls) the per-step CUDA-event profile of the library (vsb_profile_enable) of the tiny embedder.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests import unet_tiny as ut  # noqa: E402
from tests.util import make_model_pair  # noqa: E402


def time_embed(model, x, m, iters):
    for _ in range(3):
        model.embed(x, m, is_video=False)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        model.embed(x, m, is_video=False)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    B, S = a.batch, 256
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
    tiny, _, spec = ut.model_pair(device="cuda")
    m = torch.randint(0, 2, (B, spec["nbits"]), generator=torch.Generator().manual_seed(1))
    v1, _, _ = make_model_pair("videoseal_1.0", device="cuda")
    for name, model in (("unet_tiny_yuv_quant", tiny), ("videoseal_1.0", v1)):
        ms = time_embed(model, x, m, a.iters)
        print(f"embed {B} x 3x{S}x{S} {name}: {ms:.3f} ms per call = {B / ms * 1e3:.0f} frames/s (device events, {a.iters} calls)")
    v1._release()

    from videoseal_b200 import _lib
    L = _lib.lib()
    calls = 3
    L.vsb_profile_enable(1)
    for _ in range(calls):
        tiny.embed(x, m, is_video=False)
    torch.cuda.synchronize()
    n = L.vsb_profile_read(None, 0)
    buf = C.create_string_buffer(int(n) + 16)
    L.vsb_profile_read(buf, len(buf))
    L.vsb_profile_enable(0)
    # each row: a step name's total time over the profiled calls and its number of launches (names repeat once per block)
    rows = []
    for line in buf.value.decode().splitlines():
        name, tms, cnt = line.split("\t")
        rows.append((name, float(tms) / calls, int(cnt) // calls))
    print(f"per-step profile of unet_tiny_yuv_quant embed (ms per call, all steps: {sum(r[1] for r in rows):.3f} ms):")
    for name, t, cnt in sorted(rows, key=lambda r: -r[1]):
        print(f"  {name:40s} {t:8.3f} ms ({cnt} per call)")
    tiny._release()


if __name__ == "__main__":
    main()
