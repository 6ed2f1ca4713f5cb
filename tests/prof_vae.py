"""Timing of the VAE embedder: embed() of 64 x 3x256x256 frames in image mode for each preset, and of vae_small at 512 and 768
(16 frames there), 32 bits, synthetic checkpoint, the convnext extractor of videoseal_1.0.

    python tests/prof_vae.py [--iters N]

Prints the GPU name and power limit, then per case the device-event time per embed() call after 3 warm-up calls, the counted work
per frame (2 FLOP per MAC of every conv and GEMM; 4 C T^2 for the two products of each AttnBlock, encoder and decoder: 8 C T^2)
and the achieved rate, and, from a separate profiled pass, the attention steps' share of the call.
"""
import argparse
import ctypes as C
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from tests.prof_dvmark import timed  # noqa: E402

K = 32


def counted(v: dict, S: int, hidden: int):
    """(conv + GEMM FLOP, attention FLOP) per frame of the VAE at S x S"""
    w = [v["ch"] * m for m in v["ch_mult"]]
    L, nr, z = len(w), v["num_res_blocks"], v["z_channels"]
    conv = 0

    def c3(cin, cout, h, k=9):
        return 2 * h * h * cin * cout * k

    def res(cin, cout, h):
        return c3(cin, cout, h) + c3(cout, cout, h) + (c3(cin, cout, h, 1) if cin != cout else 0)

    hL = S >> (L - 1)
    CL = w[-1]
    conv += c3(v["in_channels"], v["ch"], S)
    cin = v["ch"]
    for l in range(L):
        for _ in range(nr):
            conv += res(cin, w[l], S >> l)
            cin = w[l]
        if l != L - 1:
            conv += c3(cin, cin, S >> (l + 1))
    mid = 2 * res(CL, CL, hL) + c3(CL, 3 * CL, hL, 1) + c3(CL, CL, hL, 1)
    conv += mid + c3(CL, z, hL)
    conv += c3(z + hidden, CL, hL) + mid
    cin = CL
    for l in reversed(range(L)):
        for _ in range(nr + 1):
            conv += res(cin, w[l], S >> l)
            cin = w[l]
        if l != 0:
            conv += c3(cin, cin, S >> (l - 1))
    conv += c3(cin, v["out_ch"], S)
    T = hL * hL
    return conv, 2 * 4 * CL * T * T


def profile(fn, calls=3):
    """step name -> ms per call of the VAE's steps, from the library's per-step event profile"""
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
        name, ms, _ = line.split("\t")
        if name.startswith("vae."):
            rows[name] = float(ms) / calls
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    from tests import vae_oracle as vo
    from tests.test_vae_gpu import _model
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    print("GPU:", q.stdout.strip())
    cases = [(p, 256, 64) for p in vo.PRESETS] + [("vae_small", 512, 16), ("vae_small", 768, 16)]
    for preset, S, B in cases:
        model, _ = _model(preset, S, K)
        x = torch.rand(B, 3, S, S, device="cuda")
        m = torch.randint(0, 2, (B, K))
        emb = lambda: model.embed(x, m, is_video=False)   # noqa: E731
        ms = timed(emb, args.iters)
        cf, af = counted(model.spec["vae_encoder"], S, model.spec["hidden"])
        rows = profile(emb)
        att = sum(t for n, t in rows.items() if n.startswith("vae.attn."))
        vae_ms = sum(rows.values())
        print(f"{preset:14s} {B:2d} x {S}^2: embed {ms:8.2f} ms, {cf / 1e9:6.1f} + {af / 1e9:5.1f} GFLOP per frame (conv + attention), "
              f"{B * (cf + af) / ms / 1e9:6.1f} TFLOP/s end to end; attention {att:.2f} ms ({100 * att / ms:.1f} % of embed, "
              f"{B * af / max(att, 1e-9) / 1e9:.1f} TFLOP/s); all VAE steps {vae_ms:.2f} ms")
        del model
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
