"""Time the long-K tensor-core kernel at 256 x 128 and 256 x 192 tiles on the same buffers, alternating them in one process.
   python tests/prof_longk_wide.py [--launches 200] [--rounds 3]
Shapes: the videoseal_1.0 bottleneck conv (p_conv3_bott of tests/prof_cases.py) and the temporal bottleneck conv over the stacked
operand (K = 9 * 1152).  Every launch of a round is under one pair of device events; the input rotates over enough buffers to exceed
the 50 MB L2.  Needs a GPU: there is no fallback."""
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
    "temporal 1152-384@32 x64": dict(B=64, IH=32, IW=32, C0=1152, N=384, R=3, pad=1, act=1, resid16=True),
}
L2_BYTES = 50 << 20
WIDTHS = (128, 192)


def l2_to_smem_bytes(cfg, bn):
    """operand bytes the TMA loads of one launch bring from L2: per 256 x bn tile and K block one [256 x 64] A and one [bn x 64] B"""
    M, N, K = cfg["B"] * cfg["IH"] * cfg["IW"], cfg["N"], cfg["R"] * cfg["R"] * cfg["C0"]
    return (M // 256) * (N // bn) * (K // 64) * (256 + bn) * 64 * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_longk_wide: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    lib = _lib.lib()
    for label, cfg in SHAPES.items():
        M, N, K = cfg["B"] * cfg["IH"] * cfg["IW"], cfg["N"], cfg["R"] * cfg["R"] * cfg["C0"]
        nbuf = max(2, L2_BYTES // (M * cfg["C0"] * 2) + 2)
        op = cc.make_op(cfg, n_inputs=nbuf)
        tests, out, ran = op["tests"], op["out"], op["ran"]

        def run(bn, n):
            for i in range(n):
                t = tests[i % nbuf]
                t.kernel, t.longk_block_n = cc.K_LONGK, bn
                _lib.check(lib.vsb_debug_conv(C.byref(t), None))
            assert ran.value == cc.K_LONGK

        outs = {}
        for bn in WIDTHS:      # warm-up, and the two widths agree on buffer 0
            run(bn, nbuf * 3)
            run(bn, 1)
            torch.cuda.synchronize()
            outs[bn] = out.clone()
        same = torch.equal(outs[128], outs[192])
        flop = 2.0 * M * N * K
        print(f"{label}: M={M} N={N} K={K}, {nbuf} input buffers, outputs bit-identical: {same}")
        us = {bn: [] for bn in WIDTHS}
        for _ in range(a.rounds):
            for bn in WIDTHS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                run(bn, a.launches)
                e1.record()
                torch.cuda.synchronize()
                us[bn].append(1000.0 * e0.elapsed_time(e1) / a.launches)
        for bn in WIDTHS:
            v = us[bn]
            best = min(v)
            print(f"  256 x {bn}  us/launch per round {[round(x, 1) for x in v]}  best {best:.1f} us = {flop / best / 1e6:.0f} TFLOP/s, "
                  f"L2->smem {l2_to_smem_bytes(cfg, bn) / 1e9:.2f} GB/launch", flush=True)
        del op, tests


if __name__ == "__main__":
    main()
