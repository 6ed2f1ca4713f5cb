"""The 8-channel, five-level unet_tiny_yuv_quant embedder on the GPU (synthetic checkpoint, seed 1234): the 8-channel direct-conv
kernels against fp32 references, embed() against the CPU oracle and the reference's fixture, the U-Net's intermediate maps, and
which kernels ran.  Prints the measured errors."""
import ctypes as C
import math
import os
from unittest import mock

import pytest
import torch
import torch.nn.functional as F

from oracle import restate
from tests import conv_cases as cc
from tests import unet_tiny as ut

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny.pt"), weights_only=False)
PIX_TOL, PW_TOL = 1e-3, 5e-3      # the bounds of test_e2e_gpu.py: imgs_w, and preds_w (the unscaled delta)


@pytest.fixture(scope="module")
def tiny():
    model, orc, spec = ut.model_pair()
    yield model, orc, spec
    model._release()


# ------------------------------------------------------------------ kernels (vsb_debug_conv)
D8 = dict(loader=cc.LD_DIRECT, C0=8, N=8, bias=True, out="f16")
CONV8 = {
    "d8_relu_w128":   dict(D8, B=3, IH=40, IW=128, R=3, S=3, pad=1, act=1),
    "d8_resid_w256":  dict(D8, B=2, IH=24, IW=256, R=3, S=3, pad=1, act=1, resid16=True),
    "d8_w768":        dict(D8, B=2, IH=12, IW=768, R=3, S=3, pad=1, act=1, resid16=True),
    "d8_noact_w64":   dict(D8, B=5, IH=64, IW=64, R=3, S=3, pad=1),
    "d8_ringwrap":    dict(D8, B=48, IH=128, IW=128, R=3, S=3, pad=1, act=1, resid16=True),
    "d8_outc":        dict(D8, B=2, IH=32, IW=256, R=3, S=3, pad=1, act=1, resid16=True, n_out=1, out="none"),
    "d8_outc3":       dict(D8, B=3, IH=16, IW=128, R=3, S=3, pad=1, act=1, resid16=True, n_out=3, out="none"),
    "d8_1x1_w128":    dict(D8, B=3, IH=64, IW=128, R=1, S=1),
    "d8_1x1_w768":    dict(D8, B=2, IH=16, IW=768, R=1, S=1),
    "d8_1x1_wrap":    dict(D8, B=64, IH=128, IW=128, R=1, S=1, act=1),
    # the tap GEMM of an up block with 8-channel sources: 1x1 gathered conv over [x 8 | skip 8] -> 9 x 8 taps
    "tap_8_8":        dict(loader=cc.LD_GCONV, B=3, IH=128, IW=128, C0=8, C1=8, N=72, R=1, S=1, stride=1, pad=0, out="f16"),
    # the stride-2 8 -> 16 down conv (gather loader with C = 8)
    "gdown_8_16":     dict(loader=cc.LD_GCONV, B=2, IH=128, IW=128, C0=8, N=16, R=3, S=3, stride=2, pad=1, bias=True, out="f16"),
}


@pytest.mark.parametrize("name", sorted(CONV8))
def test_conv_8ch(name):
    with mock.patch.dict(cc.CASES, {name: CONV8[name]}):
        r = cc.run_case(name, verbose=True)
    print(f"[{name}] {r}")
    assert r["ok"], r


@pytest.mark.parametrize("B,IH,IW,act", [(2, 256, 256, 0), (3, 128, 128, 0), (1, 768, 768, 0), (64, 64, 64, 1)])
def test_down_s2d_8_8(B, IH, IW, act):
    """stride-2 3x3 conv 8 -> 8 through the space-to-depth ring (vsb_debug_conv loader 5 with stride 2)"""
    g = torch.Generator().manual_seed(B * 7 + IW)
    x = torch.randn(B, IH, IW, 8, generator=g).half().cuda()
    w = (torch.randn(8, 3, 3, 8, generator=g) / math.sqrt(72)).half().cuda()
    bias = torch.randn(8, generator=g).cuda()
    OH, OW = IH // 2, IW // 2
    out = torch.full((B, OH, OW, 8), float("nan"), dtype=torch.float16, device="cuda")
    from videoseal_b200 import _lib
    t = _lib.ConvTest()
    t.loader, t.B, t.IH, t.IW, t.C0, t.C1 = cc.LD_DIRECT, B, IH, IW, 8, 0
    t.R, t.S, t.stride, t.pad, t.N, t.act = 3, 3, 2, 1, 8, act
    t.src0, t.weights, t.bias, t.out16 = C.c_void_p(x.data_ptr()), C.c_void_p(w.data_ptr()), C.c_void_p(bias.data_ptr()), C.c_void_p(out.data_ptr())
    _lib.check(_lib.lib().vsb_debug_conv(C.byref(t), None))
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.float().permute(0, 3, 1, 2), stride=2, padding=1) + bias[None, :, None, None]
    if act:
        ref = F.relu(ref)
    err = (out.float().permute(0, 3, 1, 2) - ref).abs().max().item()
    print(f"[s2d 8-8 B={B} {IH}x{IW} act={act}] max err {err:.3e} (|ref|max {ref.abs().max().item():.2f})")
    assert not torch.isnan(out).any() and err <= 2e-2 * max(1.0, ref.abs().max().item()), err


# ------------------------------------------------------------------ end to end
def _img_case(tiny, B, H, W, seed, check_detect=False):
    model, orc, spec = tiny
    g = torch.Generator().manual_seed(seed)
    imgs = torch.rand(B, 3, H, W, generator=g)
    msgs = torch.randint(0, 2, (B, spec["nbits"]), generator=g)
    with torch.no_grad():
        ref = orc.embed(imgs, msgs, is_video=False)
    out = model.embed(imgs.cuda(), msgs, is_video=False)
    e_img = (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()
    e_pw = (out["preds_w"].cpu() - ref["preds_w"]).abs().max().item()
    print(f"[embed {B}x{H}x{W} S={spec['img_size'] if model.img_size is None else model.img_size}] imgs_w {e_img:.3e}, preds_w {e_pw:.3e}")
    assert e_img <= PIX_TOL and e_pw <= PW_TOL, (e_img, e_pw)
    return imgs, msgs, out, ref


def test_embed_64_frames_256(tiny):
    _img_case(tiny, 64, 256, 256, 0)


def test_embed_768_input(tiny):
    _img_case(tiny, 2, 768, 768, 1)


def test_embed_at_processing_size_512():
    model, orc, spec = ut.model_pair(img_size=512)
    try:
        assert model.img_size == 512
        _img_case((model, orc, spec), 2, 512, 512, 2)
        _img_case((model, orc, spec), 1, 600, 720, 3)
    finally:
        model._release()


def test_intermediate_maps_against_oracle(tiny):
    """debug taps of the embed plan (NHWC) against the oracle's U-Net taps (NCHW)"""
    model, orc, spec = tiny
    g = torch.Generator().manual_seed(4)
    imgs = torch.rand(2, 3, 256, 256, generator=g)
    msgs = torch.randint(0, 2, (2, spec["nbits"]), generator=g)
    taps = {}
    with torch.no_grad():
        y = 0.299 * imgs[:, :1] + 0.587 * imgs[:, 1:2] + 0.114 * imgs[:, 2:3]      # unet_forward applies 2y - 1 itself
        restate.unet_forward(orc.sd, orc.spec, y, msgs, taps)
        u = orc.spec["unet"]
        taps["inc"] = restate.resnet_block(orc.sd, "embedder.unet.inc", 2 * y - 1, u["activation"], u["normalization"])
        d_ref = orc.embedder(imgs, msgs)
    d = model.embedder(imgs.cuda(), msgs).cpu()
    e = (d - d_ref).abs().max().item()
    print(f"[taps] delta {e:.3e}")
    assert e <= PW_TOL
    names = ["down0", "down1", "down2", "down3"] + [f"bott{i}" for i in range(4)] + \
            [f"up{j}{s}" for j in range(4) for s in ("_conv", "")]
    names = ["inc"] + names
    for n in names:
        if n == "up3":   # the last block's output is consumed by the fused outc + tanh and never written
            continue
        got = model.debug_tensor(n).permute(0, 3, 1, 2)
        r = taps[n].float()
        if n == "down3":   # written into the bottleneck concat buffer: the first z channels
            r = r[:, :got.shape[1]]
        got = got[:, :r.shape[1]]
        rel = ((got - r).abs().max() / r.abs().max().clamp_min(1e-6)).item()
        print(f"[taps] {n:9s} {tuple(r.shape)} max|d| / max|ref| = {rel:.2e}")
        assert rel <= 1e-2, (n, rel)


@pytest.mark.parametrize("case", sorted(GOLDEN["cases"]))
def test_against_reference_fixture(tiny, case):
    model, orc, spec = tiny
    c = GOLDEN["cases"][case]
    from tests.make_golden_unet_tiny import cases
    x, m, is_video, mode, chunk = cases(spec["nbits"])[case]
    old = (model.chunk_size, model.video_mode)
    try:
        model.chunk_size, model.video_mode = chunk, mode
        out = model.embed(x.cuda(), m, is_video=is_video)
    finally:
        model.chunk_size, model.video_mode = old
    e_img = (ut.sample(out["imgs_w"].cpu()) - c["imgs_w_s"]).abs().max().item()
    print(f"[fixture {case}] imgs_w {e_img:.3e}", end="")
    assert e_img <= PIX_TOL, e_img
    if "preds_w" in out:
        e_pw = (ut.sample(out["preds_w"].cpu()) - c["preds_w_s"]).abs().max().item()
        print(f", preds_w {e_pw:.3e}", end="")
        assert e_pw <= PW_TOL, e_pw
    print()


@pytest.mark.parametrize("mode", ["repeat", "alternate", "interpolate"])
def test_video_step4_ragged_chunk(tiny, mode):
    model, orc, spec = tiny
    g = torch.Generator().manual_seed(5)
    vid = torch.rand(11, 3, 272, 304, generator=g)
    msgs = torch.randint(0, 2, (1, spec["nbits"]), generator=g)
    old = (model.chunk_size, model.step_size, model.video_mode)
    try:
        model.chunk_size = orc.chunk_size = 8        # 11 frames: a full chunk and a ragged one of 3
        model.step_size = orc.step_size = 4
        model.video_mode = orc.video_mode = mode
        with torch.no_grad():
            ref = orc.embed(vid, msgs, is_video=True)
        out = model.embed(vid.cuda(), msgs, is_video=True)
        e = (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()
        print(f"[video {mode}] imgs_w {e:.3e}")
        assert e <= PIX_TOL, e
    finally:
        model.chunk_size, model.step_size, model.video_mode = old
        orc.chunk_size, orc.step_size, orc.video_mode = old


def test_detect_and_extract_on_product_output(tiny):
    model, orc, spec = tiny
    imgs, msgs, out, ref = _img_case(tiny, 4, 256, 256, 6)
    with torch.no_grad():
        ref_det = orc.detect(out["imgs_w"].cpu(), is_video=False)["preds"]
        ref_msg = orc.extract_message(out["imgs_w"].cpu(), aggregation="avg")
    det = model.detect(out["imgs_w"], is_video=False)["preds"].cpu()
    scale = ref_det.abs().max()
    e = ((det - ref_det).abs().max() / scale).item()
    print(f"[detect on embed output] max|d| / max|ref| = {e:.2e}")
    assert e <= 1.5e-3
    got = model.extract_message(out["imgs_w"], aggregation="avg").cpu()
    agg = ref_det[:, 1:].mean(0)
    sure = agg.abs() > 1e-2 * agg.abs().max()
    assert got.shape == ref_msg.shape and (got[0][sure] == ref_msg[0][sure]).all()


def test_repeated_calls_and_batch_split_are_bit_identical(tiny):
    model, orc, spec = tiny
    g = torch.Generator().manual_seed(7)
    a = torch.rand(64, 3, 256, 256, generator=g).cuda()
    b = torch.rand(3, 3, 256, 256, generator=g).cuda()
    msgs = torch.randint(0, 2, (64, spec["nbits"]), generator=g)
    w1 = model.embed(a, msgs, is_video=False)["imgs_w"].clone()
    model.embed(b, msgs[:3], is_video=False)
    w2 = model.embed(a, msgs, is_video=False)["imgs_w"]
    assert torch.equal(w1, w2)
    h = torch.cat([model.embed(a[:32], msgs[:32], is_video=False)["imgs_w"],
                   model.embed(a[32:], msgs[32:], is_video=False)["imgs_w"]])
    assert torch.equal(w1, h)


def test_profile_names_show_the_8_channel_kernels(tiny):
    """every 8-channel layer runs on the 8-channel direct kernels, and the s2d / phase-folded paths run at this net's sizes"""
    model, orc, spec = tiny
    from videoseal_b200 import _lib
    L = _lib.lib()
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(8)).cuda()
    m = torch.randint(0, 2, (2, spec["nbits"]))
    model.embed(x, m, is_video=False)
    L.vsb_profile_enable(1)
    try:
        model.embed(x, m, is_video=False)
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    names = {line.split("\t")[0] for line in buf.value.decode().splitlines()}
    unet = sorted(n for n in names if n.startswith("unet."))
    print("[profile]", unet)
    expect = {"unet.first", "unet.conv3x3d.8-8@256", "unet.conv1x1d.8-8@128", "unet.conv3x3d.8-8@128",
              "unet.down3x3s2d.8-8@128", "unet.down3x3s2.8-16@64", "unet.down3x3s2d.16-32@32",
              "unet.uptap1x1.16-72@128", "unet.upgather.8@256", "unet.conv3x3d+outc.8-8@256", "unet.conv1x1d.8-8@256",
              "unet.upphase.64-16@64", "unet.upborder.16@64", "unet.uptap1x1.32-72@64", "unet.upgather.8@128"}
    assert expect <= names, sorted(expect - names)
    # every conv with 8 output channels is a direct-kernel step (the tensor-core GEMMs tile N by at least 16)
    assert not [n for n in unet if "-8@" in n and not any(k in n for k in ("conv3x3d", "conv1x1d", "down3x3s2d"))]
