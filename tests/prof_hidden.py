"""Timing of the HiDDeN presets: embed() and detect() of 64 x 3x256x256 frames in image mode (hidden + hidden and
hidden_orig + hidden_orig cards on videoseal_1.0's args, synthetic checkpoints, JND attenuation as in the card).

    python tests/prof_hidden.py [--iters N]

Prints the GPU name and power limit, the device-event time per call after a warm-up, then, from a separate profiled pass, every
step's time per call (all its launches) and, per launch, with its share of the H100 SXM data-sheet roofline (989 TFLOP/s dense fp16, 3.35 TB/s): the larger of
flops / peak and bytes / bandwidth over the step's time.  Flops count 2 MACs of the 3x3 convs (K = 27 or 576, N = 64); bytes
count each step's compulsory reads and writes of its activations (fp16 maps of 128 B per pixel, fp32 frames of 12 B per pixel).
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

B, S = 64, 256
PX = B * S * S
# step -> (flops, bytes) per call
MODEL = {
    "hidden.conv3x3.3-64": (2 * PX * 64 * 27, PX * (12 + 128)),
    "hidden.conv3x3.64-64": (2 * PX * 64 * 576, PX * 256),
    "hidden.concat_x+msg": (2 * PX * 64 * 27, PX * (12 + 128)),
    "hidden.concat_conv3x3.64-64": (2 * PX * 64 * 576, PX * 384),
    "hidden.gn_stats": (0, PX * 128),
    "hidden.gn_apply": (0, PX * 256),
    "hidden.act+outc": (2 * PX * 3 * 64, PX * (128 + 12)),
    "hidden.gn_apply+outc": (2 * PX * 3 * 64, PX * (128 + 12)),
    "hidden.act+pool": (0, PX * 128),
    "hidden.gn_apply+pool": (0, PX * 128),
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
        if name.startswith("hidden."):
            rows[name] = (float(ms) / calls, int(n) // calls)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    args = ap.parse_args()
    from tests.test_hidden_gpu import _load
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip())
    for preset in ("hidden", "hidden_orig"):
        model, _, spec, _ = _load(preset, preset)
        x = torch.rand(B, 3, S, S, device="cuda")
        m = torch.randint(0, 2, (B, spec["nbits"]))
        emb = lambda: model.embed(x, m, is_video=False)  # noqa: E731
        det = lambda: model.detect(x, is_video=False)    # noqa: E731
        print(f"{preset}: embed {timed(emb, args.iters):.3f} ms, detect {timed(det, args.iters):.3f} ms per {B} x {S}^2 call")
        for what, fn in (("embed", emb), ("detect", det)):
            for name, (ms, n) in sorted(profile(fn).items()):
                base = name.split("@")[0]
                fl, by = MODEL.get(base, (0, 0))
                ms1 = ms / max(n, 1)   # per launch: the model counts one launch
                frac = max(fl / 989e12, by / 3.35e12) / (ms1 * 1e-3) if ms1 > 0 else 0.0
                bound = "tensor" if fl / 989e12 >= by / 3.35e12 else "HBM"
                print(f"  {what:6s} {name:36s} {ms:8.3f} ms x{n:<3d} {fl / ms1 / 1e9 if ms1 else 0:8.1f} TFLOP/s "
                      f"{by / ms1 / 1e9 if ms1 else 0:6.2f} TB/s  {100 * frac:5.1f}% of the {bound} roofline" if fl or by else
                      f"  {what:6s} {name:36s} {ms:8.3f} ms x{n:<3d}")


if __name__ == "__main__":
    main()
