"""Timing of the SAM-ViT extractors: detect() of 64 x 3x256x256 frames with sam_small and sam_small_pw (synthetic checkpoints).

    python tests/prof_vit.py [--iters N] [--batch B]

Prints the GPU name and power limit, the device-event time per detect() call after a warm-up, the achieved TFLOP/s of the whole
call from the FLOP counts below, then (in separate calls) the per-step CUDA-event profile of the library (vsb_profile_enable) with
the TFLOP/s of each ViT step.  One 256^2 frame is ~13.1 GFLOP: blocks 11.5 (attention 0.60 of it), neck 0.76, head 0.68, patch
embed 0.15.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests import vit_oracle as vo  # noqa: E402


def step_flops(spec) -> dict:
    """FLOPs per frame of each profile step name (multiply-add = 2)"""
    v = spec["vit"]
    G = spec["img_size"] // 16
    T, E, M, oc, heads = G * G, v["embed_dim"], v["mlp_dim"], v["out_chans"], v["num_heads"]
    f = {"vit.patch": 2.0 * T * 768 * E, "vit.qkv": 0.0, "vit.proj": 0.0, "vit.lin1": 0.0, "vit.lin2": 0.0,
         "vit.neck1x1": 2.0 * T * E * oc, f"vit.neck3x3": 2.0 * T * 9 * oc * oc}
    for i in range(v["depth"]):
        f["vit.qkv"] += 2.0 * T * E * 3 * E
        f["vit.proj"] += 2.0 * T * E * E
        f["vit.lin1"] += 2.0 * T * E * M
        f["vit.lin2"] += 2.0 * T * M * E
        n = G if i in v["global_attn_indexes"] else v["window_size"]
        name = f"vit.attn_global.{T}" if n == G else f"vit.attn_win.{n * n}"
        # q k^T and P v over the n^2 keys of the token's region, + q Rh^T and q Rw^T over the 2n - 1 table rows
        per_query = 2.0 * 2 * n * n * 64 + (2.0 * 2 * (2 * n - 1) * 64 if v["use_rel_pos"] else 0.0)
        f[name] = f.get(name, 0.0) + per_query * T * heads
    if not spec["pixel_decoder"]["pixelwise"]:
        f[f"vit.head3x3.{oc}@{G}"] = 2.0 * T * 9 * oc * oc
    return f


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--batch", type=int, default=64)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("needs a GPU")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    print("gpu:", torch.cuda.get_device_name(0), "|", q.stdout.strip())
    from videoseal_b200 import _lib
    L = _lib.lib()
    for pixelwise in (False, True):
        preset = "sam_small_pw" if pixelwise else "sam_small"
        model, _, spec = vo.model_pair(pixelwise, device="cuda")
        B, S = a.batch, spec["img_size"]
        fl = step_flops(model.spec)
        total = sum(fl.values())
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
        print(f"detect {B} x 3x{S}x{S} {preset}: {ms:.3f} ms per call = {B / ms * 1e3:.0f} frames/s (device events, {a.iters} calls); "
              f"{total / 1e9:.2f} GFLOP per frame (trunk{'' if pixelwise else ' + head conv'}) -> {B * total / (ms * 1e-3) / 1e12:.1f} TFLOP/s")
        calls = 3
        L.vsb_profile_enable(1)
        for _ in range(calls):
            model.detect(x, is_video=False)
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
        L.vsb_profile_enable(0)
        rows = []
        for line in buf.value.decode().splitlines():
            name, tms, cnt = line.split("\t")
            rows.append((name, float(tms) / calls, int(cnt) // calls))
        print(f"  per-step profile (ms per detect() call, all steps: {sum(r[1] for r in rows):.3f} ms):")
        for name, t, cnt in sorted(rows, key=lambda r: -r[1]):
            extra = f"  {B * fl[name] / (t * 1e-3) / 1e12:6.1f} TFLOP/s ({fl[name] / 1e9:.3f} GFLOP per frame)" if name in fl else ""
            print(f"    {name:36s} {t:8.3f} ms ({cnt} per call){extra}")
        model._release()


if __name__ == "__main__":
    main()
