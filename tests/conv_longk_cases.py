"""Unit cases for the 256-row long-K tensor-core kernel (conv_gemm_longk_kernel) through vsb_debug_conv, against the fp32 PyTorch
reference of tests/conv_cases.py on the same fp16-rounded operands.  Every case names the kernel the library must select for the op
by itself (`ran`); `kernel` forces one, `same_as` re-runs the op on the other kernel and asks for the same bits.
Used by tests/test_conv_longk_gpu.py and tests/prof_longk.py."""
import ctypes as C
import math

import torch

from tests.conv_cases import LD_TMA, reference
from videoseal_b200 import _lib

K_AUTO, K_128, K_LONGK = 0, 1, 2      # vsb_conv_test.kernel / kernel_ran: the 128-row kernel, the 256-row long-K kernel

CASES = {
    # the two convs of a videoseal_1.0 bottleneck ResnetBlock at 64 frames, and the same op without activation
    "bott_relu": dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, ran=K_LONGK),
    "bott_res":  dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),
    "bott_none": dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1, resid16=True, ran=K_LONGK),
    "n256":      dict(B=80, IH=32, IW=32, C0=256, N=256, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),     # two N tiles
    "n320":      dict(B=72, IH=32, IW=32, C0=320, N=320, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),     # block_n 80
    "gemm":      dict(B=1, IH=1, IW=64 * 256, C0=1536, N=768, R=1, ran=K_LONGK),                            # plain 2-D GEMM form
    "map16":     dict(B=96, IH=16, IW=16, C0=384, N=384, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),     # one tile per image
    "map64":     dict(B=16, IH=64, IW=64, C0=256, N=256, R=3, pad=1, act=1, ran=K_LONGK),                   # tile = 4 rows x 64
    "pixelseal": dict(B=32, IH=32, IW=32, C0=512, N=512, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),     # four N tiles
    # 360 K blocks: the 4-stage ring wraps its phase 45 times per tile
    "chunky":    dict(B=16, IH=32, IW=32, C0=2560, N=2560, R=3, pad=1, act=1, resid16=True, ran=K_LONGK),
    "small_b":   dict(B=4, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, resid16=True, ran=K_128),        # too few tiles: 128-row kernel
    "vs_128":    dict(B=8, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, resid16=True, kernel=K_LONGK, ran=K_LONGK, same_as=K_128),
}


def make_op(cfg, seed=0, n_inputs=1):
    """Operands of one case on the GPU and a vsb_conv_test per input buffer (all share weights, bias, residual and output)."""
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(seed)
    B, IH, IW, C0, N, R = cfg["B"], cfg["IH"], cfg["IW"], cfg["C0"], cfg["N"], cfg["R"]
    K = R * R * C0
    xs = [torch.randn(B, IH, IW, C0, generator=g).half().to(dev) for _ in range(n_inputs)]
    w = (torch.randn(N, R, R, C0, generator=g) / math.sqrt(K)).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    resid = torch.randn(B, IH, IW, N, generator=g).half().to(dev) if cfg.get("resid16") else None
    out = torch.full((B, IH, IW, N), float("nan"), dtype=torch.float16, device=dev)
    ran = C.c_int32(0)
    tests = []
    for x in xs:
        t = _lib.ConvTest()
        t.loader, t.B, t.IH, t.IW, t.C0, t.C1 = LD_TMA, B, IH, IW, C0, 0
        t.R, t.S, t.stride, t.pad, t.N, t.act = R, R, 1, cfg.get("pad", 0), N, cfg.get("act", 0)
        t.src0, t.weights, t.bias = x.data_ptr(), w.data_ptr(), bias.data_ptr()
        t.resid16 = resid.data_ptr() if resid is not None else None
        t.out16 = out.data_ptr()
        t.kernel, t.kernel_ran = cfg.get("kernel", K_AUTO), C.pointer(ran)
        tests.append(t)
    return dict(xs=xs, w=w, bias=bias, resid=resid, out=out, ran=ran, tests=tests)


def run_case(name, seed=0):
    cfg = CASES[name]
    op = make_op(cfg, seed)
    t, out, ran = op["tests"][0], op["out"], op["ran"]
    _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
    torch.cuda.synchronize()
    res = {"kernel_ran": ran.value}
    ref, _ = reference(dict(cfg, S=cfg["R"]), op["xs"][0], None, op["w"], op["bias"], op["resid"], None, None)
    got = out.float().permute(0, 3, 1, 2)
    res["nan"] = int(torch.isnan(got).sum().item())
    res["out_maxerr"] = (got - ref).abs().max().item()
    res["out_ref_max"] = ref.abs().max().item()
    res["ok"] = bool(res["nan"] == 0 and res["out_maxerr"] <= 2e-2 * max(1.0, res["out_ref_max"]) and ran.value == cfg["ran"])
    if "same_as" in cfg:       # the other kernel forced on the same operands must give the same bits
        first = out.clone()
        out.fill_(float("nan"))
        t.kernel = cfg["same_as"]
        _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
        torch.cuda.synchronize()
        res["bit_identical"] = bool(ran.value == cfg["same_as"] and torch.equal(first, out))
        res["ok"] = bool(res["ok"] and res["bit_identical"])
    return res
