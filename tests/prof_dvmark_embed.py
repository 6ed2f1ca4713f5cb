"""Timing of the DVMark embedder: embed() of 64 x 3x256x256 frames in video mode, step_size 1, two chunks of 32 key frames (the
`dvmark` embedder and extractor with 96 bits, synthetic checkpoint).

    python tests/prof_dvmark_embed.py [--iters N]

Prints the GPU name and power limit, the device-event time per call after 3 warm-up calls, then, from a separate profiled pass, every
DVMark embedder step's time per call (all its launches) with the TFLOP/s of the convs: 2 MACs per tap, input and output channel
over the map each runs on (7 274 304 + 10 368 K MACs per processing pixel in all).
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests.prof_dvmark import timed  # noqa: E402

B, S, K = 64, 256, 96
PX = B * S * S
P1, P2 = (64 + K + 7) // 8 * 8, (128 + K + 7) // 8 * 8


def flops() -> dict:
    """step name (without @size) -> flops per call, counted with the reference's channel counts (64 + K, 128 + K), not the padded
    pitches"""
    f = {"dvmark_enc.conv1x3x3.3-64": 2 * PX * 64 * 27, "dvmark_enc.conv1x3x3.64-64": 2 * 2 * PX * 64 * 9 * 64}
    full = [(64, 64), (P1, 256, 64 + K), (256, 128), (128, 128), (384, 256), (256, 128)]
    for c in full:
        cin, n = c[0], c[1]
        f[f"dvmark_enc.conv3x3x3.{cin}-{n}"] = f.get(f"dvmark_enc.conv3x3x3.{cin}-{n}", 0) + 2 * PX * n * 27 * (c[2] if len(c) > 2 else cin)
    for cin, n, real in ((P2, 512, 128 + K), (512, 256, 512), (256, 256, 256)):
        f[f"dvmark_enc.conv3x3x3.{cin}-{n}"] = f.get(f"dvmark_enc.conv3x3x3.{cin}-{n}", 0) + 2 * (PX // 4) * n * 27 * real
    f["dvmark_enc.conv3x3x3+tanh.128-3"] = 2 * PX * 3 * 27 * 128
    return f


def profile(fn, calls=3):
    """step name -> (ms per call, launches per call) of the DVMark embedder's steps, from the library's per-step event profile"""
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
        if name.startswith(("dvmark_enc.", "pw.")):
            rows[name] = (float(ms) / calls, int(n) // calls)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from tests.test_dvmark_embed_gpu import _model
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip())
    model, _ = _model(S, K)
    model.chunk_size, model.step_size = 32, 1
    x = torch.rand(B, 3, S, S, device="cuda")
    m = torch.randint(0, 2, (1, K))
    emb = lambda: model.embed(x, m, is_video=True)   # noqa: E731
    ms = timed(emb, args.iters)
    total = 2 * PX * (7274304 + 10368 * K)
    print(f"dvmark embed {ms:.2f} ms per {B} x {S}^2 call (two chunks of 32 key frames), {total / 1e12:.2f} TFLOP counted, "
          f"{total / ms / 1e9:.1f} TFLOP/s end to end")
    f = flops()
    # the conv rows sum the 3x3x3 convs of equal shape (emb_layer1.2 and emb_layer3.2 are both 256 -> 128 at S)
    for name, (t, n) in sorted(profile(emb).items()):
        fl = f.get(name.split("@")[0], 0)
        print(f"  {name:48s} {t:8.3f} ms x{n:<3d}" + (f" {fl / t / 1e9:8.1f} TFLOP/s" if fl else ""))
    assert abs(sum(f.values()) - total) <= 1e-6 * total, (sum(f.values()), total)


if __name__ == "__main__":
    main()
