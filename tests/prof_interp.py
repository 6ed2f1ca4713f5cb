"""Device time of the resize and blend kernels for every interpolation mode, from the library's CUDA-event profile
(vsb_profile_enable / vsb_profile_read: one event pair around each kernel launch).

    python tests/prof_interp.py [out.json]      (the rows are printed; given a path, also written there as JSON)

  resize  64 x 1080p -> 256 and 16 x 4K -> 256 (detect, video mode), per (mode, align_corners, antialias)
  blend   256 -> 1080p (16 images) and 256 -> 4K (4 images) (embed, image mode, jnd_1_1, preds_w written), bilinear against bicubic
          (the 4-tap path), with the bytes the kernel must move (frames in, imgs_w and preds_w out, the delta keys in) over the
          H100 SXM data-sheet HBM3 bandwidth of 3.35 TB/s

Prints the card's name, power limit and maximum SM clock beside the numbers.  Each row is the best of 3 rounds of 10 calls."""
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ctypes as C  # noqa: E402

import torch  # noqa: E402

from tests.util import make_model_pair  # noqa: E402
from videoseal_b200 import _lib  # noqa: E402

HBM = 3.35e12
MODES = [("bilinear", False, True), ("bilinear", False, False), ("bilinear", True, False), ("bicubic", False, True),
         ("bicubic", False, False), ("nearest", None, False), ("area", None, False)]


def idict(m):
    d = {"mode": m[0], "antialias": m[2]}
    if m[1] is not None:
        d["align_corners"] = m[1]
    return d


def profiled(fn, prefix):
    """best per-call device time (ms) of the profiled steps whose name starts with `prefix`, over 3 rounds of 10 calls"""
    L = _lib.lib()
    fn()
    torch.cuda.synchronize()
    best = None
    for _ in range(3):
        L.vsb_profile_enable(1)
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 20)
        L.vsb_profile_read(buf, len(buf))
        L.vsb_profile_enable(0)
        tot = cnt = 0
        for line in buf.value.decode().splitlines():
            name, ms, n = line.split("\t")
            if name.startswith(prefix):
                tot, cnt = tot + float(ms), cnt + int(n)
        assert cnt > 0, (prefix, buf.value.decode()[:500])
        best = tot / cnt if best is None else min(best, tot / cnt)
    return best


def main():
    out_path = sys.argv[1] if len(sys.argv) > 1 else None
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    model, _, spec = make_model_pair("videoseal_1.0", tiny={"num_blocks": 1, "depths": [1, 1, 1, 1]})
    S = spec["img_size"]
    rows = {"card": q, "resize": [], "blend": []}
    for n, H, W in [(64, 1080, 1920), (16, 2160, 3840)]:
        x = torch.rand(n, 3, H, W, device="cuda")
        for m in MODES:
            ms = profiled(lambda: model.detect(x, is_video=True, interpolation=idict(m)), f"pw.resize.{H}x{W}@")
            nbytes = (n * 3 * H * W + n * 3 * S * S) * 4
            r = {"frames": f"{n}x{H}x{W}", "mode": idict(m), "ms": round(ms, 4), "GB/s": round(nbytes / ms / 1e6, 1),
                 "of_3.35TB/s": round(nbytes / ms / 1e-3 / HBM, 3)}
            rows["resize"].append(r)
            print("[resize]", r)
        del x
    for n, H, W in [(16, 1080, 1920), (4, 2160, 3840)]:
        x = torch.rand(n, 3, H, W, device="cuda")
        msgs = torch.randint(0, 2, (n, spec["nbits"]))
        for m in [("bilinear", False, True), ("bicubic", False, True), ("bicubic", False, False)]:
            ms = profiled(lambda: model.embed(x, msgs, is_video=False, interpolation=idict(m)), f"pw.jnd_blend.{H}x{W}@")
            nbytes = (n * H * W * (3 + 3 + 1) + n * S * S) * 4
            r = {"frames": f"{n}x{H}x{W}", "mode": idict(m), "ms": round(ms, 4), "GB/s": round(nbytes / ms / 1e6, 1),
                 "of_3.35TB/s": round(nbytes / ms / 1e-3 / HBM, 3)}
            rows["blend"].append(r)
            print("[blend]", r)
        del x
    if out_path:                                  # optional: the rows as JSON
        os.makedirs(os.path.dirname(out_path) or ".", exist_ok=True)
        json.dump(rows, open(out_path, "w"), indent=1)
        print("->", out_path)


if __name__ == "__main__":
    main()
