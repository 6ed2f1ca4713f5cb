"""Time the 128-row and the 256-row (long-K) tensor-core kernels on the same buffers, alternating them in one process.
   python tests/prof_longk.py [--launches 200] [--rounds 4]
Shapes: the videoseal_1.0 bottleneck conv (p_conv3_bott of tests/prof_cases.py) and the pixelseal / chunkyseal bottleneck convs.
Every launch of a round is under one pair of device events; the input rotates over enough buffers to exceed the 50 MB L2.  Needs
a GPU: there is no fallback."""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tests import conv_longk_cases as cc
from tests.prof_cases import BIG
from videoseal_b200 import _lib

_BOTT = BIG["p_conv3_bott"]
SHAPES = {
    "videoseal_1.0 384-384@32 x64": dict({k: _BOTT[k] for k in ("B", "IH", "IW", "C0", "N", "R", "pad", "act", "resid16")}),
    "pixelseal 512-512@32 x32": cc.CASES["pixelseal"],
    "chunkyseal 2560-2560@32 x16": cc.CASES["chunky"],
}
L2_BYTES = 50 << 20


def l2_to_smem_bytes(cfg, tile_m):
    """operand bytes the TMA loads of one launch bring from L2: per tile and K block one [tile_m x 64] A and one [128 x 64] B tile"""
    M, N, K = cfg["B"] * cfg["IH"] * cfg["IW"], cfg["N"], cfg["R"] * cfg["R"] * cfg["C0"]
    bn = 128
    return (M // tile_m) * (N // bn) * (K // 64) * (tile_m + bn) * 64 * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=4)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_longk: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    for label, cfg in SHAPES.items():
        B, H, W, Cin, N = cfg["B"], cfg["IH"], cfg["IW"], cfg["C0"], cfg["N"]
        K = cfg["R"] * cfg["R"] * Cin
        M = B * H * W
        nbuf = max(2, L2_BYTES // (M * Cin * 2) + 2)
        op = cc.make_op(cfg, n_inputs=nbuf)
        tests, out, ran = op["tests"], op["out"], op["ran"]
        lib = _lib.lib()

        def run(kernel, n):
            for i in range(n):
                t = tests[i % nbuf]
                t.kernel = kernel
                _lib.check(lib.vsb_debug_conv(C.byref(t), None))
            assert ran.value == kernel

        outs = {}
        for kernel in (cc.K_128, cc.K_LONGK):      # warm-up, and the two kernels agree on buffer 0
            run(kernel, nbuf * 3)
            run(kernel, 1)
            torch.cuda.synchronize()
            outs[kernel] = out.clone()
        same = torch.equal(outs[cc.K_128], outs[cc.K_LONGK])
        flop = 2.0 * M * N * K
        print(f"{label}: M={M} N={N} K={K}, {nbuf} input buffers, outputs bit-identical: {same}")
        us = {cc.K_128: [], cc.K_LONGK: []}
        for _ in range(a.rounds):
            for kernel in (cc.K_128, cc.K_LONGK):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(kernel, a.launches)
                e1.record()
                torch.cuda.synchronize()
                us[kernel].append(1000.0 * e0.elapsed_time(e1) / a.launches)
        for kernel, name, tile_m in ((cc.K_128, "128-row", 128), (cc.K_LONGK, "256-row long-K", 256)):
            v = us[kernel]
            best = min(v)
            print(f"  {name:15s} us/launch per round {[round(x, 1) for x in v]}  best {best:.1f} us = {flop / best / 1e6:.0f} TFLOP/s, "
                  f"L2->smem {l2_to_smem_bytes(cfg, tile_m) / 1e9:.2f} GB/launch", flush=True)
        del op, tests


if __name__ == "__main__":
    main()
