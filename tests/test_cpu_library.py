"""CPU-side checks: the C-ABI library builds/loads and exports every symbol include/vsb200.h declares; the host logic
(card parsing, API surface) works and fails loudly without a GPU."""
import re
import os

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_exports_match_header(built_lib):
    hdr = open(os.path.join(ROOT, "include", "vsb200.h")).read()
    declared = set(re.findall(r"\b(vsb_[a-z_0-9]+)\s*\(", hdr))
    declared -= {"vsb_model", "vsb_model_desc", "vsb_conv_test", "vsb_status", "vsb_video_mode", "vsb_flags"}
    assert declared, "no declarations parsed"
    for sym in sorted(declared):
        assert hasattr(built_lib, sym), f"libvsb200.so does not export {sym}"
    from videoseal_b200 import _lib
    assert set(_lib.EXPORTS) == declared


def test_desc_struct_layout_matches_header():
    from videoseal_b200 import _lib
    import ctypes as C
    # 4 + 3 + 6 + 4 + 8 + 1 + 2 = 28 int32 fields in vsb_model_desc
    assert C.sizeof(_lib.ModelDesc) == 28 * 4


@pytest.mark.parametrize("card", ["videoseal_1.0", "pixelseal", "chunkyseal"])
def test_card_parsing_matches_oracle_spec(built_lib, card):
    from tests.util import load_card
    from oracle import restate
    from videoseal_b200 import cfg
    c = load_card(card)
    a, b = cfg.spec_from_card(c), restate.spec_from_card(c)
    assert a["nbits"] == b["nbits"] and a["hidden"] == b["hidden"] and a["img_size"] == b["img_size"]
    assert a["unet"]["z"] == [b["unet"]["z_channels"] * m for m in b["unet"]["mults"]]
    assert a["convnext"]["dims"] == b["convnext"]["dims"] and a["convnext"]["depths"] == b["convnext"]["depths"]
    assert a["yuv"] == b["yuv"] and a["step_size"] == b["step_size"] and a["chunk_size"] == b["chunk_size"]


def test_load_and_fail_loudly_without_gpu(built_lib):
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    import videoseal_b200
    from tests.util import synthetic_card_on_disk
    cpath, spec, _ = synthetic_card_on_disk("videoseal_1.0", tiny={"num_blocks": 1, "depths": [1, 1, 1, 1]})
    model = videoseal_b200.load(cpath).eval()
    assert model.get_random_msg(3).shape == (3, spec["nbits"])
    assert model.blender.scaling_w == pytest.approx(0.2) and model.step_size == 4 and model.chunk_size == 32
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.embed(torch.rand(1, 3, 256, 256), is_video=False)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model.detect(torch.rand(1, 3, 256, 256))


def test_unsupported_card_features_raise_at_load():
    from tests.util import load_card
    from videoseal_b200 import cfg
    c = load_card("videoseal_1.0")
    c["args"]["blending_method"] = "multiplicative"
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(c)
    c = load_card("videoseal_1.0")
    c["extractor"]["model"] = "sam_small"
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(c)


@pytest.mark.parametrize("n_in,n_out,aa", [(768, 256, True), (300, 256, True), (480, 256, True), (257, 256, True), (200, 256, True),
                                            (256, 768, True), (256, 768, False), (256, 300, False), (17, 256, False), (1080, 256, False),
                                            # anti-aliased down-scales above 3x (maxt 9 .. 61: resize_sep_kernel's any-tap-count path)
                                            (769, 256, True), (1080, 256, True), (1920, 256, True), (2160, 256, True), (3840, 256, True),
                                            (1280, 256, True), (1920, 384, True), (3840, 128, True),
                                            # large up-scales (the delta of the blend at 1080p / 4K)
                                            (256, 1920, True), (256, 2160, False), (512, 1080, True)])
def test_resample_tables_match_aten_interpolate(built_lib, n_in, n_out, aa):
    """the host-built separable tables of the resize kernels (resize_blend_host.cuh:make_resample) against F.interpolate applied to the
    identity: every output sample's tap positions and weights (wam.py:163,184,224 call sites; bilinear, align_corners=False).
    Anti-aliased down-scales are computed in double and rounded once to fp32, so they are held to float64 ATen; the plain
    bilinear tables take their source coordinate in fp32 (as ATen's fp32 kernels do), so they are held to fp32 ATen."""
    import ctypes as C
    import numpy as np
    import torch.nn.functional as F
    start = np.zeros(n_out, dtype=np.int32)
    cnt = np.zeros(n_out, dtype=np.int32)
    cap = n_out * 64
    w = np.zeros(cap, dtype=np.float32)
    maxt = built_lib.vsb_debug_resample_table(n_in, n_out, int(aa), start.ctypes.data, cnt.ctypes.data, w.ctypes.data, cap)
    assert maxt > 0, built_lib.vsb_last_error()
    w = w[: n_out * maxt].reshape(n_out, maxt)
    op = np.zeros((n_out, n_in), dtype=np.float64)
    for o in range(n_out):
        assert 0 <= start[o] and start[o] + cnt[o] <= n_in and 1 <= cnt[o] <= maxt
        op[o, start[o]:start[o] + cnt[o]] = w[o, :cnt[o]]
    down_aa = aa and n_in > n_out
    assert (maxt == 2 * int(np.ceil(n_in / n_out)) + 1) if down_aa else maxt == 2
    dt = torch.float64 if down_aa else torch.float32
    eye = torch.eye(n_in, dtype=dt).reshape(1, n_in, 1, n_in)          # n_in "channels", each a one-hot row of width n_in
    ref = F.interpolate(eye, size=(1, n_out), mode="bilinear", align_corners=False, antialias=aa)
    ref = ref.reshape(n_in, n_out).t().double().numpy()
    # up-scaling with antialias=True: ATen routes it through its anti-aliasing code (triangle filter of support 1 == plain bilinear
    # mathematically), whose source coordinate is rounded once more than the plain kernel's: half a float ulp of a coordinate < 512
    # (7.6e-6 at 256 -> 1920 and 512 -> 1080).  Anti-aliased down-scales: one fp32 rounding of a weight <= 1 (measured <= 1.5e-8).
    tol = 1e-7 if down_aa else (8e-6 if aa and n_out > n_in else 2e-6)
    assert np.abs(op - ref).max() < tol
    assert np.allclose(op.sum(1), 1.0, atol=1e-5)


def test_gelu_polynomial_constants_match_exact_erf_gelu():
    """conv_gemm.cuh computes nn.GELU (exact erf, modules/convnext.py:33) as max(x,0) - 0.5|x| 2^Q(|x|) with ONE SFU op; the
    constants are parsed from the header and the formula is evaluated in fp32 here against torch's exact GELU"""
    import re
    import torch
    src = open(os.path.join(ROOT, "videoseal_b200", "csrc", "conv_gemm.cuh")).read()
    q = [float(re.search(rf"kGeluQ{i} = (-?[0-9.eE+-]+)f", src).group(1)) for i in range(5)]
    x = torch.linspace(-30, 30, 2_000_001, dtype=torch.float32)
    ax = x.abs()
    p = torch.full_like(ax, q[4])
    for k in (3, 2, 1, 0):
        p = p * ax + q[k]
    got = x.clamp_min(0) - 0.5 * ax * torch.exp2(p * ax)
    ref = torch.nn.functional.gelu(x.double()).float()
    assert (got - ref).abs().max().item() <= 2e-6
