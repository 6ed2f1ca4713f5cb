"""Time the 128-row and the 256-row (long-K) tensor-core kernels on the ConvNeXt pointwise GEMMs of the videoseal_1.0 detector at
64 frames of 256^2, both forced on the same buffers and alternated in one process.
   python tests/prof_longk_cnx.py [--launches 100] [--rounds 3]
Reports, per shape and kernel, the best round's us per launch, TFLOP/s, and the share of the op's floor: the larger of its HBM bytes
(fp16 input and g, fp32 GRN partial rows or residual stream read + write, weights) at 3.35 TB/s and its FLOPs at 989 TFLOP/s (H100
SXM data sheet).  The input rotates over enough buffers to exceed the 50 MB L2.  Needs a GPU: there is no fallback."""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from tests import conv_longk_cnx_cases as cc
from videoseal_b200 import _lib

SHAPES = ["pw1_s0", "pw2_s0", "pw1_s1", "pw2_s1", "pw1_s2", "pw2_s2", "pw1_s3", "pw2_s3"]
L2_BYTES = 50 << 20
HBM_BPS, TENSOR_FLOPS = 3.35e12, 989e12


def floor_bytes(cfg):
    M, K, N = cfg["M"], cfg["K"], cfg["N"]
    w = cfg.get("w_samples", 1) * N * K * 2
    if cfg["kind"] == "pw1":
        return M * K * 2 + M * N * 2 + (M // 32) * N * 4 + w
    return M * K * 2 + 2 * M * N * 4 + w + (M * N * 2 if cfg.get("x16") else 0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--launches", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("prof_longk_cnx: no CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print("card:", q.stdout.strip(), flush=True)
    lib = _lib.lib()
    for name in SHAPES:
        cfg = dict(cc.CASES[name])
        M, K, N = cfg["M"], cfg["K"], cfg["N"]
        nbuf = max(2, L2_BYTES // (M * K * 2) + 2)
        op = cc.make_op(cfg, n_inputs=nbuf)
        tests, ran = op["tests"], op["ran"]

        def launch(kernel, n):
            for i in range(n):
                t = tests[i % nbuf]
                t.kernel = kernel
                _lib.check(lib.vsb_debug_conv(C.byref(t), None))
            assert ran.value == kernel

        for kernel in (cc.K_128, cc.K_LONGK):      # warm-up
            launch(kernel, nbuf * 2)
        torch.cuda.synchronize()
        flop = 2.0 * M * N * K
        fb = floor_bytes(cfg)
        floor_us = max(fb / HBM_BPS, flop / TENSOR_FLOPS) * 1e6
        bound = "HBM" if fb / HBM_BPS >= flop / TENSOR_FLOPS else "FLOP"
        print(f"{name} ({cfg['kind']}): M={M} K={K} N={N} w_samples={cfg.get('w_samples', 1)}, {nbuf} input buffers, "
              f"floor {floor_us:.1f} us ({bound}: {fb / 1e6:.0f} MB, {flop / 1e9:.0f} GFLOP), library picks "
              f"{'256-row' if cfg['ran'] == cc.K_LONGK else '128-row'}")
        us = {cc.K_128: [], cc.K_LONGK: []}
        for _ in range(a.rounds):
            for kernel in (cc.K_128, cc.K_LONGK):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                launch(kernel, a.launches)
                e1.record()
                torch.cuda.synchronize()
                us[kernel].append(1000.0 * e0.elapsed_time(e1) / a.launches)
        for kernel, label in ((cc.K_128, "128-row"), (cc.K_LONGK, "256-row long-K")):
            v = us[kernel]
            best = min(v)
            print(f"  {label:15s} us/launch per round {[round(x, 1) for x in v]}  best {best:.1f} us = {flop / best / 1e6:.0f} TFLOP/s, "
                  f"{floor_us / best:.0%} of floor", flush=True)
        del op, tests


if __name__ == "__main__":
    main()
