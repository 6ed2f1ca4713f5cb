"""Timing of the temporal unet_small2_yuv_quant_conv3d embedder against its 2-D twin unet_small2_yuv_quant (videoseal_1.0's U-Net):
embed() of 64 x 3x256x256 frames in image mode (one 64-frame time axis; synthetic checkpoints, JND attenuation as in the card).

    python tests/prof_temporal.py [--iters N]

Prints the GPU name and power limit, the device-event time per embed() call of each model after a warm-up (the two alternate,
`--rounds` times, in one process), then, from a separate profiled pass, every temporal step's time per call and the achieved
TFLOP/s of the 3x3x3 convs: 2 * M * N * 27 * C flops (M = 64 * H * W output pixels; the zero channels that pad the stacked operand
to the TMA conv's K block are not counted).
"""
import argparse
import ctypes as C
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests import temporal_oracle as to  # noqa: E402


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


def profile(model, x, m, calls=3):
    from videoseal_b200 import _lib
    L = _lib.lib()
    L.vsb_profile_enable(1)
    for _ in range(calls):
        model.embed(x, m, is_video=False)
    torch.cuda.synchronize()
    n = L.vsb_profile_read(None, 0)
    buf = C.create_string_buffer(int(n) + 16)
    L.vsb_profile_read(buf, len(buf))
    L.vsb_profile_enable(0)
    rows = []
    for line in buf.value.decode().splitlines():
        name, tms, cnt = line.split("\t")
        rows.append((name, float(tms) / calls, int(cnt) // calls))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    B, S = 64, 256
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(0)).cuda()
    t3, _, spec = to.model_pair("unet_small2_yuv_quant_conv3d", device="cuda")
    t2, _, _ = to.model_pair("unet_small2_yuv_quant", device="cuda")
    m = torch.randint(0, 2, (B, spec["nbits"]), generator=torch.Generator().manual_seed(1))
    times = {"unet_small2_yuv_quant_conv3d": [], "unet_small2_yuv_quant": []}
    for _ in range(a.rounds):
        for name, model in (("unet_small2_yuv_quant_conv3d", t3), ("unet_small2_yuv_quant", t2)):
            times[name].append(time_embed(model, x, m, a.iters))
    for name, ts in times.items():
        print(f"embed {B} x 3x{S}x{S} {name}: " + " / ".join(f"{t:.3f}" for t in ts) + f" ms per call (device events, {a.iters} "
              f"calls per round); best {B / min(ts) * 1e3:.0f} frames/s")
    print(f"ratio temporal / 2-D (best of {a.rounds}): {min(times['unet_small2_yuv_quant_conv3d']) / min(times['unet_small2_yuv_quant']):.2f}")
    t2._release()

    rows = profile(t3, x, m)
    print(f"per-step profile of unet_small2_yuv_quant_conv3d embed (ms per call, all steps: {sum(r[1] for r in rows):.3f} ms):")
    for name, t, cnt in sorted(rows, key=lambda r: -r[1]):
        extra = ""
        g = re.match(r"unet\.conv3x3x3(\+outc)?\.(\d+)-(\d+)@(\d+)", name)
        if g:
            c, n, h = int(g.group(2)), int(g.group(3)), int(g.group(4))
            flops = 2.0 * B * h * h * n * 27 * c * cnt
            extra = f"  {flops / (t * 1e-3) / 1e12:6.1f} TFLOP/s"
        print(f"  {name:40s} {t:8.3f} ms ({cnt} per call){extra}")
    t3._release()


if __name__ == "__main__":
    main()
