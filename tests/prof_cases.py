"""Launch a few representative conv/GEMM ops at BASELINE configs[1] sizes (for ncu captures and quick timing).
   python tests/prof_cases.py [names...]"""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from tests import conv_cases as cc

BIG = {
    "p_conv1_c16":  dict(loader=cc.LD_TMA, B=64, IH=256, IW=256, C0=16, N=16, R=1, S=1, bias=True, out="f16"),
    "p_conv3_c16":  dict(loader=cc.LD_TMA, B=64, IH=256, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_conv3_bott": dict(loader=cc.LD_TMA, B=64, IH=32, IW=32, C0=384, N=384, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_halo3_c16":  dict(loader=cc.LD_HALO, B=64, IH=256, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_direct_c16": dict(loader=cc.LD_DIRECT, B=64, IH=256, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_direct_c32": dict(loader=cc.LD_DIRECT, B=64, IH=128, IW=128, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_direct_c64": dict(loader=cc.LD_DIRECT, B=64, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_direct1_c16": dict(loader=cc.LD_DIRECT, B=64, IH=256, IW=256, C0=16, N=16, R=1, S=1, bias=True, out="f16"),
    "p_halo3_c32":  dict(loader=cc.LD_HALO, B=64, IH=128, IW=128, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_conv3_c32":  dict(loader=cc.LD_TMA, B=64, IH=128, IW=128, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_halo3_c64":  dict(loader=cc.LD_HALO, B=64, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_conv3_c64":  dict(loader=cc.LD_TMA, B=64, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_halo3_bott": dict(loader=cc.LD_HALO, B=64, IH=32, IW=32, C0=384, N=384, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "p_conv1_bott": dict(loader=cc.LD_TMA, B=64, IH=32, IW=32, C0=384, N=384, R=1, S=1, bias=True, out="f16"),
    "p_pw1_96":     dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 4096, C0=96, N=384, R=1, S=1, bias=True, act=2, grn=True, rps=4096, out="f16"),
    "p_pw1_384":    dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 256, C0=384, N=1536, R=1, S=1, bias=True, act=2, grn=True, rps=256, out="f16"),
    "p_pw2_384":    dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 256, C0=1536, N=384, R=1, S=1, bias=True, resid32=True, out="f32"),
    "p_pw2_96t":    dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 4096, C0=384, N=96, R=1, S=1, bias=True, resid32=True, out="f32"),
    "p_pw2_192t":   dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 1024, C0=768, N=192, R=1, S=1, bias=True, resid32=True, out="f32"),
    "p_uptap_128":  dict(loader=cc.LD_TMA, B=1, IH=1, IW=64 * 4096, C0=128, N=288, R=1, S=1, out="f16"),
    "p_down_16_32": dict(loader=cc.LD_GCONV, B=64, IH=256, IW=256, C0=16, N=32, R=3, S=3, stride=2, pad=1, bias=True, out="f16"),
}
cc.CASES.update(BIG)

if __name__ == "__main__":
    iters = 0
    args = sys.argv[1:]
    if args and args[0] == "--time":
        iters = 10
        args = args[1:]
    names = args or list(BIG)
    for n in names:
        torch.cuda.synchronize()
        t0 = time.time()
        r = cc.run_case(n, time_iters=iters)
        # re-launch for timing: run_case again under CUDA events (includes input generation only outside events? no -> use ncu/bench for exact)
        print(n, {k: (round(v, 5) if isinstance(v, float) else v) for k, v in r.items() if k in ("ok", "out_maxerr", "delta_maxerr", "stats_relerr", "us", "tflops")}, f"{time.time()-t0:.2f}s", flush=True)
