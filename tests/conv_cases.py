"""Unit cases for the wgmma conv/GEMM kernels (vsb_debug_conv) against a plain PyTorch fp32 reference of the same op
computed from the same fp16-rounded operands.  Used by tests/test_conv_gemm_gpu.py and tests/gpu_diag.py."""
import ctypes as C
import math

import torch
import torch.nn.functional as F

from videoseal_b200 import _lib

LD_TMA, LD_GCONV, LD_HALO, LD_DIRECT = 0, 1, 4, 5

CASES = {
    # name: dict(loader, B, IH, IW, C0, C1, R, S, stride, pad, pad_mode, N, extras...)
    "gemm_basic":      dict(loader=LD_TMA, B=1, IH=1, IW=256, C0=128, N=64, R=1, S=1, out="f32"),
    "gemm_tails":      dict(loader=LD_TMA, B=1, IH=1, IW=300, C0=96, N=384, R=1, S=1, bias=True, out="f32"),
    "gemm_n96":        dict(loader=LD_TMA, B=1, IH=1, IW=512, C0=384, N=96, R=1, S=1, bias=True, out="f16"),
    "conv3_c64":       dict(loader=LD_TMA, B=2, IH=32, IW=32, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "conv3_c16_sw32":  dict(loader=LD_TMA, B=1, IH=128, IW=128, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "conv3_c32_sw64":  dict(loader=LD_TMA, B=1, IH=64, IW=64, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "conv1_c128":      dict(loader=LD_TMA, B=2, IH=32, IW=32, C0=128, N=128, R=1, S=1, bias=True, out="f16"),
    "conv3_w256":      dict(loader=LD_TMA, B=1, IH=8, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "conv3_bott":      dict(loader=LD_TMA, B=24, IH=32, IW=32, C0=384, N=384, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "outc":            dict(loader=LD_TMA, B=1, IH=128, IW=128, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=1, out="none"),
    "outc3":           dict(loader=LD_TMA, B=1, IH=128, IW=128, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=3, out="none"),
    "halo_c64":        dict(loader=LD_HALO, B=2, IH=32, IW=32, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "halo_c16":        dict(loader=LD_HALO, B=1, IH=128, IW=128, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "halo_c32":        dict(loader=LD_HALO, B=3, IH=64, IW=64, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "halo_bott":       dict(loader=LD_HALO, B=24, IH=32, IW=32, C0=384, N=384, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "halo_outc":       dict(loader=LD_HALO, B=2, IH=128, IW=128, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=1, out="none"),
    "halo_outc3":      dict(loader=LD_HALO, B=1, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=3, out="none"),
    # direct 3x3 (conv3_direct.cuh): ring of padded rows in 8-channel planes, one MMA per tap straight from the ring
    "direct_c16_w64":  dict(loader=LD_DIRECT, B=2, IH=64, IW=64, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "direct_c16_w256": dict(loader=LD_DIRECT, B=2, IH=24, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "direct_c32":      dict(loader=LD_DIRECT, B=3, IH=48, IW=128, C0=32, N=32, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "direct_c64":      dict(loader=LD_DIRECT, B=2, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "direct_c32_n16":  dict(loader=LD_DIRECT, B=1, IH=32, IW=96, C0=32, N=16, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "direct_outc":     dict(loader=LD_DIRECT, B=2, IH=32, IW=256, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=1, out="none"),
    "direct_outc3":    dict(loader=LD_DIRECT, B=1, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, resid16=True, n_out=3, out="none"),
    "direct1_c16":     dict(loader=LD_DIRECT, B=2, IH=40, IW=256, C0=16, N=16, R=1, S=1, bias=True, out="f16"),
    "direct1_c32":     dict(loader=LD_DIRECT, B=3, IH=128, IW=128, C0=32, N=32, R=1, S=1, bias=True, out="f16"),
    "direct1_c64":     dict(loader=LD_DIRECT, B=70, IH=64, IW=64, C0=64, N=64, R=1, S=1, bias=True, out="f16"),
    "direct1_wrap":    dict(loader=LD_DIRECT, B=96, IH=128, IW=128, C0=16, N=16, R=1, S=1, bias=True, act=1, out="f16"),
    "direct_ringwrap": dict(loader=LD_DIRECT, B=96, IH=128, IW=128, C0=16, N=16, R=3, S=3, pad=1, bias=True, act=1, resid16=True, out="f16"),
    "direct_wrap_c64": dict(loader=LD_DIRECT, B=80, IH=64, IW=64, C0=64, N=64, R=3, S=3, pad=1, bias=True, act=1, out="f16"),
    "gconv_s2":        dict(loader=LD_GCONV, B=2, IH=64, IW=64, C0=16, N=32, R=3, S=3, stride=2, pad=1, bias=True, out="f16"),
    "gconv_patch":     dict(loader=LD_GCONV, B=2, IH=16, IW=16, C0=96, N=192, R=2, S=2, stride=2, pad=0, bias=True, out="f32"),
    "gconv_reflect":   dict(loader=LD_GCONV, B=3, IH=8, IW=8, C0=64, N=64, R=3, S=3, stride=1, pad=1, pad_mode=1, out="f32"),
    "gconv_odd":       dict(loader=LD_GCONV, B=1, IH=15, IW=15, C0=72, N=40, R=3, S=3, stride=1, pad=1, pad_mode=1, out="f32"),
    "gelu_grn":        dict(loader=LD_TMA, B=1, IH=1, IW=512, C0=96, N=384, R=1, S=1, bias=True, act=2, grn=True, rps=256, out="f16"),
    "gelu_grn_rag":    dict(loader=LD_TMA, B=1, IH=1, IW=450, C0=96, N=384, R=1, S=1, bias=True, act=2, grn=True, rps=225, out="f16"),
    # chunkyseal's proportional trunk: widths 362 / 724 / 1448 (not multiples of 8 / 16) in rows padded to 8 elements, odd maps
    "chunky_pw1":      dict(loader=LD_TMA, B=1, IH=1, IW=1922, C0=362, ld0=368, ldw=368, N=1448, R=1, S=1, bias=True, act=2, grn=True, rps=961, out="f16"),
    "chunky_pw2":      dict(loader=LD_TMA, B=1, IH=1, IW=1922, C0=1448, N=362, ld_out=368, R=1, S=1, bias=True, resid32=True, out="f32"),
    "chunky_ds":       dict(loader=LD_GCONV, B=2, IH=31, IW=31, C0=368, N=724, ld_out=728, R=2, S=2, stride=2, pad=0, bias=True, out="f32"),
}


def halo_layout(w, C0, C1):
    """[N, 3, 3, C0+C1] (tap-major) -> the halo loaders' [N][chunk][tap][cc] layout, chunks zero-padded to kb_per_c*64"""
    N, Ct = w.shape[0], C0 + C1
    cc = min(C0, 64)
    kbc = (9 * cc + 63) // 64
    nchunks = Ct // cc
    out = torch.zeros(N, nchunks, kbc * 64, dtype=w.dtype, device=w.device)
    wc = w.reshape(N, 9, nchunks, cc).permute(0, 2, 1, 3).reshape(N, nchunks, 9 * cc)
    out[:, :, :9 * cc] = wc
    return out.reshape(N, nchunks * kbc * 64).contiguous()


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def reference(cfg, x0, x1, w, bias, resid, lnw, lnb):
    """fp32 torch reference on the GPU. x0/x1 NHWC fp16; w [N, R, S, Ct] fp16."""
    xin = x0.float().permute(0, 3, 1, 2)
    if x1 is not None:
        xin = torch.cat([xin, x1.float().permute(0, 3, 1, 2)], dim=1)
    wt = w.float().permute(0, 3, 1, 2).contiguous()          # [N, Ct, R, S]
    pad = cfg.get("pad", 0)
    if cfg.get("pad_mode", 0) == 1 and pad:
        xin = F.pad(xin, (pad,) * 4, mode="reflect")
        pad = 0
    y = F.conv2d(xin, wt, stride=cfg.get("stride", 1), padding=pad)
    if cfg.get("epi", 0) == 1:
        u = y.mean(1, keepdim=True)
        s = (y - u).pow(2).mean(1, keepdim=True)
        y = (y - u) / torch.sqrt(s + 1e-6) * lnw[None, :, None, None] + lnb[None, :, None, None]
    elif bias is not None:
        y = y + bias[None, :, None, None]
    act = cfg.get("act", 0)
    if act == 1:
        y = F.relu(y)
    elif act == 2:
        y = F.gelu(y)
    pre_resid = y
    if resid is not None:
        y = y + resid.float().permute(0, 3, 1, 2)
    return y, pre_resid


def run_case(name, seed=0, verbose=False, time_iters=0):
    cfg = dict(CASES[name])
    dev = "cuda"
    g = torch.Generator(device="cpu").manual_seed(seed)
    B, IH, IW, C0, C1, N = cfg["B"], cfg["IH"], cfg["IW"], cfg["C0"], cfg.get("C1", 0), cfg["N"]
    R, S = cfg["R"], cfg["S"]
    Ct = C0 + C1
    K = R * S * Ct
    ld0, ldw, ld_out = cfg.get("ld0", 0), cfg.get("ldw", 0), cfg.get("ld_out", 0)
    x0 = (torch.randn(B, IH, IW, C0, generator=g)).half().to(dev)
    x1 = (torch.randn(B, IH, IW, C1, generator=g)).half().to(dev) if C1 else None
    w = (torch.randn(N, R, S, Ct, generator=g) / math.sqrt(K)).half().to(dev)
    bias = torch.randn(N, generator=g).to(dev) if cfg.get("bias") else None
    lnw = (1 + 0.1 * torch.randn(N, generator=g)).to(dev) if cfg.get("epi", 0) == 1 else None
    lnb = (0.1 * torch.randn(N, generator=g)).to(dev) if cfg.get("epi", 0) == 1 else None
    ld = cfg["loader"]
    if ld == LD_GCONV:
        st, pad = cfg.get("stride", 1), cfg.get("pad", 0)
        OH, OW = (IH + 2 * pad - R) // st + 1, (IW + 2 * pad - S) // st + 1
    else:
        OH, OW = IH, IW
    M = B * OH * OW
    resid16 = torch.randn(B, OH, OW, N, generator=g).half().to(dev) if cfg.get("resid16") else None
    resid32 = torch.randn(B, OH, OW, N, generator=g).to(dev) if cfg.get("resid32") else None
    out16 = torch.full((B, OH, OW, N), float("nan"), dtype=torch.float16, device=dev) if cfg["out"] == "f16" else None
    out32 = None
    if cfg["out"] == "f32":
        out32 = resid32.clone() if resid32 is not None else torch.full((B, OH, OW, N), float("nan"), device=dev)
    # padded pitches: the operands live in wider rows whose pad columns hold a sentinel the kernel must neither read nor write
    SENT = 1000.0
    x0_p = w_p = out32_p = None
    if ld0:
        x0_p = torch.full((B, IH, IW, ld0), SENT, dtype=torch.float16, device=dev)
        x0_p[..., :C0] = x0
    if ld_out:
        assert out32 is not None
        out32_p = torch.full((B, OH, OW, ld_out), SENT, device=dev)
        out32_p[..., :N] = out32
    n_out = cfg.get("n_out", 0)
    outc_w = (torch.randn(n_out, N, generator=g) / math.sqrt(N)).to(dev) if n_out else None
    outc_b = (0.1 * torch.randn(n_out, generator=g)).to(dev) if n_out else None
    delta = torch.full((B, n_out, OH, OW), float("nan"), device=dev) if n_out else None
    nsamp = (M + cfg.get("rps", M) - 1) // cfg.get("rps", M) if cfg.get("grn") else 0
    stats = torch.zeros(nsamp, N, device=dev) if cfg.get("grn") else None

    t = _lib.ConvTest()
    t.loader, t.B, t.IH, t.IW, t.C0, t.C1 = ld, B, IH, IW, C0, C1
    t.R, t.S, t.stride, t.pad, t.pad_mode = R, S, cfg.get("stride", 1), cfg.get("pad", 0), cfg.get("pad_mode", 0)
    t.N, t.epi, t.act, t.rows_per_sample, t.block_n = N, cfg.get("epi", 0), cfg.get("act", 0), cfg.get("rps", 0), cfg.get("block_n", 0)
    w_dev = halo_layout(w, C0, C1) if ld == LD_HALO else w
    if ldw:
        w_p = torch.full((N, ldw), SENT, dtype=torch.float16, device=dev)
        w_p[:, :K] = w.reshape(N, K)
        w_dev = w_p
    t.ld0, t.ldw, t.ld_out = ld0, ldw, ld_out
    t.src0, t.src1, t.weights = _ptr(x0_p if ld0 else x0), _ptr(x1), _ptr(w_dev)
    t.bias, t.resid16 = _ptr(bias), _ptr(resid16)
    if ld_out:
        out32_true, out32 = out32, out32_p
    t.resid32 = _ptr(out32) if resid32 is not None else None     # in place, like the ConvNeXt residual stream
    t.ln_w, t.ln_b = _ptr(lnw), _ptr(lnb)
    t.outc_w, t.outc_b, t.n_out = _ptr(outc_w), _ptr(outc_b), n_out
    t.out16, t.out32, t.delta, t.grn_stats = _ptr(out16), _ptr(out32), _ptr(delta), _ptr(stats)
    _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
    torch.cuda.synchronize()
    timing = None
    if time_iters:
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        keep = out32 is not None and resid32 is not None
        e0.record()
        for _ in range(time_iters):
            _lib.lib().vsb_debug_conv(C.byref(t), None)
        e1.record()
        torch.cuda.synchronize()
        timing = 1000.0 * e0.elapsed_time(e1) / time_iters
        if keep:                  # in-place residual accumulates across launches: redo one clean launch
            out32.copy_(resid32)
        if stats is not None:
            stats.zero_()
        if keep or stats is not None:
            _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
            torch.cuda.synchronize()

    resid = resid16 if resid16 is not None else resid32
    ref, pre = reference(cfg, x0, x1, w, bias, resid, lnw, lnb)
    res = {}
    if ld_out:
        res["pad_untouched"] = bool((out32[..., N:] == SENT).all())
        out32 = out32[..., :N]
    if timing is not None:
        res["us"] = timing
        res["tflops"] = 2.0 * M * N * K / (timing * 1e-6) / 1e12
    scale_ref = ref.abs().max().item()
    if out16 is not None or out32 is not None:
        got = (out16 if out16 is not None else out32).float().permute(0, 3, 1, 2)
        err = (got - ref).abs()
        res["out_maxerr"] = err.max().item() if not torch.isnan(got).any() else float("nan")
        res["out_ref_max"] = scale_ref
        res["nan"] = int(torch.isnan(got).sum().item())
        tol = 2e-2 * max(1.0, scale_ref) if out16 is not None else 5e-3 * max(1.0, scale_ref)
        res["ok"] = bool(res["nan"] == 0 and res["out_maxerr"] <= tol and res.get("pad_untouched", True))
        if verbose and not res["ok"]:
            e = torch.nan_to_num(err, nan=1e9)
            res["err_by_col"] = e.amax(dim=(0, 2, 3))[: min(N, 64)].tolist()
            eb = e.amax(dim=1).reshape(-1)
            res["err_by_row_first256"] = eb[:256].tolist()
    if delta is not None:
        dref = torch.tanh(torch.einsum("bnhw,on->bohw", ref, outc_w) + outc_b[None, :, None, None])
        res["delta_maxerr"] = (delta - dref).abs().max().item()
        res["ok"] = bool(res.get("ok", True) and res["delta_maxerr"] <= 2e-2 and not torch.isnan(delta).any())
    if stats is not None:
        rps = cfg["rps"]
        gsq = (out16.float() ** 2).reshape(M, N)
        sref = torch.stack([gsq[i * rps:(i + 1) * rps].sum(0) for i in range(nsamp)])
        res["stats_relerr"] = ((stats - sref).abs() / (sref.abs() + 1e-3)).max().item()
        res["ok"] = bool(res.get("ok", True) and res["stats_relerr"] <= 2e-2)
    return res
