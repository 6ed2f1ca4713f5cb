"""GPU parity of the 256 x 192 tiles of the long-K tensor-core kernel (conv_gemm_longk_kernel<192, ·>), one op at a time through the
C ABI (vsb_debug_conv).  Each case runs the same operands three times: on the long-K kernel forced to 192-wide and to 128-wide tiles,
and on the 128-row kernel; the three outputs must be bit-identical (same K order per output, same epilogue arithmetic).  The
192-wide output is also judged against a float64 PyTorch reference on the same fp16-rounded operands, with the bound of
tests/conv_longk_cases.py."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests.conv_longk_cases import K_128, K_LONGK, make_op

pytestmark = pytest.mark.gpu

CASES = {
    # the bottleneck 3x3 convs of videoseal_1.0 at 64 frames: 384 -> 384 @32^2, with and without the fp16 residual
    "x64_relu_res": dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, resid16=True),
    "x64_none":     dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1),
    # the temporal bottleneck: the 3x3 conv over the stacked [x(t-1) | x(t) | x(t+1)] operand, K = 9 * 1152
    "temporal":     dict(B=64, IH=32, IW=32, C0=1152, N=384, R=3, pad=1, act=1, resid16=True),
    # 72 frames: 576 tiles of 256 x 192 on 132 SMs, a partial last wave
    "x72_relu_res": dict(B=72, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1, resid16=True),
    "x64_relu":     dict(B=64, IH=32, IW=32, C0=384, N=384, R=3, pad=1, act=1),
}


def _run(op, kernel, longk_bn):
    t, out, ran = op["tests"][0], op["out"], op["ran"]
    out.fill_(float("nan"))
    t.kernel, t.longk_block_n = kernel, longk_bn
    from videoseal_b200 import _lib
    _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
    torch.cuda.synchronize()
    assert ran.value == kernel
    return out.clone()


def _reference64(cfg, op):
    """bias -> ReLU -> + residual over the float64 convolution of the fp16 operands, NCHW"""
    y = F.conv2d(op["xs"][0].double().permute(0, 3, 1, 2), op["w"].double().permute(0, 3, 1, 2), padding=cfg.get("pad", 0))
    y = y + op["bias"].double()[None, :, None, None]
    if cfg.get("act", 0) == 1:
        y = F.relu(y)
    if op["resid"] is not None:
        y = y + op["resid"].double().permute(0, 3, 1, 2)
    return y


@pytest.mark.parametrize("name", list(CASES))
def test_conv_longk_wide(built_lib, name):
    cfg = CASES[name]
    op = make_op(cfg)
    wide = _run(op, K_LONGK, 192)
    narrow = _run(op, K_LONGK, 128)
    row128 = _run(op, K_128, 0)
    assert torch.equal(wide, narrow), "long-K 192 vs 128 wide"
    assert torch.equal(wide, row128), "long-K 192 wide vs the 128-row kernel"
    ref = _reference64(cfg, op)
    got = wide.double().permute(0, 3, 1, 2)
    assert int(torch.isnan(got).sum().item()) == 0
    err, ref_max = (got - ref).abs().max().item(), ref.abs().max().item()
    assert err <= 2e-2 * max(1.0, ref_max), (err, ref_max)
