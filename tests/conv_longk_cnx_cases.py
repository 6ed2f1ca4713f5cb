"""The ConvNeXt pointwise GEMMs (pwconv1: bias + GELU + fp16 g + GRN partial rows; pwconv2: fp32 residual stream += g W2^T + bias,
per-sample weights at stages 0-1) as single ops through vsb_debug_conv, at the videoseal_1.0 detector's shapes.  Every case names
the kernel the library must select by itself (`ran`); the op is then re-run on the forced 128-row kernel for a bit comparison.
Used by tests/test_conv_longk_cnx_gpu.py and tests/prof_longk_cnx.py."""
import ctypes as C
import math

import torch
import torch.nn.functional as F

from tests.conv_cases import LD_TMA
from tests.conv_longk_cases import K_AUTO, K_128, K_LONGK
from videoseal_b200 import _lib


def _pw1(B, hs, C0, ran, M=None):
    return dict(kind="pw1", M=M or B * hs * hs, K=C0, N=4 * C0, rps=hs * hs, ran=ran)


def _pw2(B, hs, C0, ran, wscale, x16=False):
    return dict(kind="pw2", M=B * hs * hs, K=4 * C0, N=C0, rps=hs * hs, w_samples=B if wscale else 1, x16=x16, ran=ran)


# stage s of the tiny trunk at 64 frames of 256^2: C = 96 << s on a (64 >> s)^2 map; pwconv2 folds the GRN multiplier into per-sample
# weights at stages 0-1.  Stages 2-3's pwconv2 have 192 / 96 tiles of 256 rows (fewer than two per SM) and stage 0's a 6-block main
# loop: the 128-row kernel.
CASES = {
    "pw1_s0": _pw1(64, 64, 96, K_LONGK),         # K = 96: two K blocks, the second half zero-filled by TMA
    "pw1_s1": _pw1(64, 32, 192, K_LONGK),
    "pw1_s2": _pw1(64, 16, 384, K_LONGK),
    "pw1_s3": _pw1(64, 8, 768, K_LONGK),
    "pw2_s0": _pw2(64, 64, 96, K_128, True),     # K = 384: 6 K blocks, too short for the fp32-stream epilogue
    "pw2_s1": _pw2(64, 32, 192, K_LONGK, True),  # block_n 96, two N tiles
    "pw2_s2": _pw2(64, 16, 384, K_128, False),
    "pw2_s3": _pw2(64, 8, 768, K_128, False, x16=True),
    # a 70-frame sub-batch, and a GEMM whose rows do not fill the last 256-row tile (the 128-row kernel)
    "pw1_s0_b70": _pw1(70, 64, 96, K_LONGK),
    "pw2_s1_b70": _pw2(70, 32, 192, K_LONGK, True),
    "pw2_s0_longk": dict(_pw2(64, 64, 96, K_LONGK, True), kernel=K_LONGK),       # block_n 96, one N tile, forced
    "pw1_s1_ragged": _pw1(64, 32, 192, K_128, M=64 * 32 * 32 + 128),
    # the fp16 copy of the last stage-3 block's output, forced onto the 256-row kernel
    "pw2_s3_x16_longk": dict(_pw2(64, 8, 768, K_LONGK, False, x16=True), kernel=K_LONGK),
}


def part_rows(M):
    """rows of the GRN partial buffer the 128-row kernel addresses: 4 per 128-row tile"""
    return (M + 127) // 128 * 4


def make_op(cfg, seed=0, n_inputs=1):
    """Operands of one case on the GPU and a vsb_conv_test per input buffer (all share weights, bias and outputs)."""
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(seed)
    M, K, N, ws = cfg["M"], cfg["K"], cfg["N"], cfg.get("w_samples", 1)
    xs = [torch.randn(M, K, generator=g).half().to(dev) for _ in range(n_inputs)]
    w = (torch.randn(ws, N, K, generator=g) / math.sqrt(K)).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev)
    op = dict(xs=xs, w=w, bias=bias, ran=C.c_int32(0))
    if cfg["kind"] == "pw1":
        op["g"] = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev)
        op["part"] = torch.full((part_rows(M), N), float("nan"), device=dev)
    else:
        op["x0"] = torch.randn(M, N, generator=g).to(dev)
        op["x"] = op["x0"].clone()
        op["x16"] = torch.full((M, N), float("nan"), dtype=torch.float16, device=dev) if cfg.get("x16") else None
    tests = []
    for x in xs:
        t = _lib.ConvTest()
        t.loader, t.B, t.IH, t.IW, t.C0, t.C1 = LD_TMA, 1, 1, M, K, 0
        t.R, t.S, t.stride, t.pad, t.N = 1, 1, 1, 0, N
        t.src0, t.weights, t.bias = x.data_ptr(), w.data_ptr(), bias.data_ptr()
        t.rows_per_sample = cfg["rps"]
        if cfg["kind"] == "pw1":
            t.act = 2
            t.out16, t.grn_stats, t.grn_part = op["g"].data_ptr(), op["part"].data_ptr(), 1
        else:
            t.resid32 = t.out32 = op["x"].data_ptr()      # in place, like the residual stream
            t.out16 = op["x16"].data_ptr() if op["x16"] is not None else None
            t.w_samples = ws
        t.kernel, t.kernel_ran = cfg.get("kernel", K_AUTO), C.pointer(op["ran"])
        tests.append(t)
    op["tests"] = tests
    return op


def reference(cfg, op):
    """fp32 (pw1: g, fp64 partial rows of the result's own squares) reference of the op on the same fp16 operands"""
    M, N, rps = cfg["M"], cfg["N"], cfg["rps"]
    x, w, bias = op["xs"][0].float(), op["w"].float(), op["bias"]
    if cfg["kind"] == "pw1":
        return F.gelu(x @ w[0].t() + bias)
    if w.shape[0] == 1:
        return op["x0"] + x @ w[0].t() + bias
    xs = x.reshape(w.shape[0], rps, -1)
    return op["x0"] + torch.bmm(xs, w.transpose(1, 2)).reshape(M, N) + bias


def run(op, kernel=None):
    t = op["tests"][0]
    if kernel is not None:
        t.kernel = kernel
    _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
    torch.cuda.synchronize()
    return op["ran"].value


def outputs(cfg, op):
    if cfg["kind"] == "pw1":
        return {"g": op["g"].clone(), "part": op["part"][: cfg["M"] // 32].clone()}
    out = {"x": op["x"].clone()}
    if op["x16"] is not None:
        out["x16"] = op["x16"].clone()
    return out


def reset(cfg, op):
    if cfg["kind"] == "pw1":
        op["g"].fill_(float("nan"))
        op["part"].fill_(float("nan"))
    else:
        op["x"].copy_(op["x0"])
        if op["x16"] is not None:
            op["x16"].fill_(float("nan"))


def run_case(name, seed=0):
    cfg = CASES[name]
    op = make_op(cfg, seed)
    res = {"kernel_ran": run(op)}
    got = outputs(cfg, op)
    ref = reference(cfg, op)
    main = got["g"].float() if cfg["kind"] == "pw1" else got["x"]
    res["nan"] = int(torch.isnan(main).sum().item())
    res["out_maxerr"] = (main - ref).abs().max().item()
    res["out_ref_max"] = ref.abs().max().item()
    tol = (2e-2 if cfg["kind"] == "pw1" else 5e-3) * max(1.0, res["out_ref_max"])
    ok = res["nan"] == 0 and res["out_maxerr"] <= tol and res["kernel_ran"] == cfg["ran"]
    if cfg["kind"] == "pw1":
        sq = got["g"].double().pow(2).reshape(cfg["M"] // 32, 32, cfg["N"]).sum(1)
        res["part_relerr"] = ((got["part"].double() - sq).abs() / (sq + 1e-3)).max().item()
        ok = ok and res["part_relerr"] <= 2e-2
    elif "x16" in got:
        res["x16_maxerr"] = (got["x16"].float() - got["x"]).abs().max().item()
        ok = ok and res["x16_maxerr"] <= 1e-2 * max(1.0, res["out_ref_max"])
    if res["kernel_ran"] == K_LONGK:
        # the 128-row kernel forced on the same operands gives the same bits in every output
        reset(cfg, op)
        assert run(op, K_128) == K_128
        other = outputs(cfg, op)
        res["bit_identical"] = {k: bool(torch.equal(got[k], other[k])) for k in got}
        ok = ok and all(res["bit_identical"].values())
    res["ok"] = bool(ok)
    return res
