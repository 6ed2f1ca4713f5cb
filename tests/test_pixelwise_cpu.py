"""Pixel-wise ConvNeXt extractors (modules/pixel_decoder.py pixelwise=True) without a GPU: the oracle against the reference's
fixture, preset / card resolution, load-time rejections, and the C setter's error codes on a host-only handle."""
import argparse
import ctypes as C
import os

import pytest
import torch

from tests import pixelwise_oracle as pw
from tests.util import load_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "pixelwise.pt"), weights_only=False)


@pytest.mark.parametrize("preset", pw.PRESETS)
def test_oracle_reproduces_reference_fixture(preset):
    res = GOLDEN["presets"][preset]
    spec = res["spec"]
    assert spec == pw.spec_from_card(pw.preset_card(preset, load_card("videoseal_1.0")))
    orc = pw.OracleModel(spec, pw.synth_state_dict(spec, GOLDEN["seed"]))
    orc.chunk_size = 2
    for name, case in res["cases"].items():
        if name == "extract":
            continue
        assert case["oracle_vs_ref"] == 0.0
        x = torch.rand(*case["shape"], generator=torch.Generator().manual_seed(case["gen_seed"]))
        with torch.no_grad():
            maps = orc.detect(x, is_video=case["is_video"])["preds"]
        assert maps.shape == (case["shape"][0], 1 + spec["nbits"], 256, 256)
        torch.testing.assert_close(pw.sample(maps), case["maps_s"], rtol=0, atol=1e-5)
        assert maps.double().abs().mean().item() == pytest.approx(case["stats"]["all"]["absmean"], rel=1e-6)
        assert maps[:, :1].double().mean().item() == pytest.approx(case["stats"]["det"]["mean"], rel=1e-5, abs=1e-7)
    vid = res["cases"]["vid"]
    x = torch.rand(*vid["shape"], generator=torch.Generator().manual_seed(vid["gen_seed"]))
    for agg, a in res["cases"]["extract"].items():
        assert a["oracle_vs_ref"] == 0
        with torch.no_grad():
            bits = orc.extract_message(x, aggregation=agg)
        assert bits.shape == (1, spec["nbits"], 256, 256)
        # sub-margin pixels (|decoded| ~ 0) may flip between thread counts; the fixture pins all but a handful
        assert abs(int(bits.sum()) - a["ones"]) <= 8, agg
        assert (bits[:, ::8, ::16, ::16] != a["bits_s"]).sum().item() <= 1, agg


@pytest.mark.parametrize("preset,dims,widths", [("convnext_tiny_pw", [96, 192, 384, 768], [768, 192, 48, 24]),
                                                ("convnext_base_pw", [128, 256, 512, 1024], [1024, 256, 64, 32])])
def test_training_checkpoint_naming_preset_resolves(built_lib, tmp_path, preset, dims, widths):
    from videoseal_b200 import cfg
    card = load_card("videoseal_1.0")
    args = argparse.Namespace(**card["args"], embedder_model="unet_small2_yuv_quant", extractor_model=preset)
    path = tmp_path / "ckpt.pth"
    torch.save({"model": {}, "args": args}, path)
    spec = cfg.spec_from_card(cfg.get_config_from_checkpoint(str(path)))
    assert spec["pixel_decoder"] == {"pixelwise": True, "upscale_stages": [4, 4, 2]}
    assert spec["convnext"]["dims"] == dims and spec["convnext"]["stem_stride"] == 4
    c, got = dims[-1], [dims[-1]]
    for f in spec["pixel_decoder"]["upscale_stages"]:
        c //= f
        got.append(c)
    assert got == widths
    # the product's synthetic checkpoints carry the same keys and shapes as the oracle's
    from videoseal_b200 import synth
    sd, ref = synth.synth_state_dict(spec), pw.synth_state_dict(pw.spec_from_card(pw.preset_card(preset, card)))
    shapes = lambda d: {k: tuple(v.shape) for k, v in d.items() if k.startswith("detector.")}  # noqa: E731
    assert shapes(sd) == shapes(ref)


def _pd_card(**pd):
    card = pw.preset_card("convnext_tiny_pw", load_card("videoseal_1.0"))
    card["extractor"]["params"]["pixel_decoder"].update(pd)
    return card


@pytest.mark.parametrize("change", [
    {"pixelwise": False, "upscale_stages": [4, 4, 2]},   # pooled decoder with upscale stages
    {"pixelwise": False, "upscale_stages": [2]},
    {"sigmoid_output": True},
    {"upscale_stages": [4, 3, 2]},                       # factor other than 2 / 4
    {"upscale_stages": []},
    {"upscale_type": "nearest"},                         # same weights as bilinear, other arithmetic
    {"upscale_type": "conv"},
    {"upscale_type": "pixelshuffle"},
    {"upscale_stages": [2, 2, 2]},                       # last stage 96 channels: more than 32
    {"upscale_stages": [4, 4, 4, 2]},                    # 768 -> 192 -> 48 -> 12: not a multiple of 8
])
def test_rejected_pixel_decoders_raise_at_load(built_lib, change):
    from videoseal_b200 import cfg
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(_pd_card(**change))


def test_pixel_decoder_width_and_size_rules_at_load(built_lib):
    from videoseal_b200 import cfg
    card = _pd_card(upscale_type="bilinear")
    assert cfg.spec_from_card(card)["pixel_decoder"]["upscale_stages"] == [4, 4, 2]
    card = _pd_card(upscale_stages=[2, 4, 4])                # 768 -> 384 -> 96 -> 24, accepted also at img_size 384
    card["args"]["img_size_proc"] = 384
    assert cfg.spec_from_card(card)["img_size"] == 384
    card = _pd_card()                                         # 640 -> 160: a middle width outside 8 * {1, 3} * 2^k
    card["extractor"]["params"]["encoder"]["dims"] = [80, 160, 320, 640]
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)
    card = _pd_card()                                         # head weights of 2049 outputs do not fit beside the taps
    card["args"]["nbits"] = 2048
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)


def test_pixelwise_on_chunkyseal_trunk_raises_at_load():
    from videoseal_b200 import cfg
    card = load_card("chunkyseal")
    card["extractor"]["params"]["pixel_decoder"] = {"pixelwise": True, "upscale_stages": [4, 4, 2], "sigmoid_output": False}
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)
    card = _pd_card()
    card["extractor"]["params"]["encoder"]["stem_stride"] = 2
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)


def test_existing_cards_keep_pooled_decoder(built_lib):
    from videoseal_b200 import cfg
    for name in ("videoseal_1.0", "pixelseal", "chunkyseal"):
        assert cfg.spec_from_card(load_card(name))["pixel_decoder"] == {"pixelwise": False, "upscale_stages": [1]}


def test_set_pixel_decoder_error_codes_on_a_valid_descriptor(built_lib):
    from videoseal_b200 import _lib, cfg
    from videoseal_b200.model import native_desc
    L = _lib.lib()
    h = C.c_void_p()
    z = _lib.ModelDesc()                          # a mostly zero descriptor (no U-Net levels, no trunk) is no model
    z.nbits, z.img_size, z.ext_stem_stride = 256, 256, 4
    assert L.vsb_model_create(C.byref(z), C.byref(h)) == -1 and h.value is None
    d = native_desc(cfg.spec_from_card(load_card("videoseal_1.0")))   # 256 bits, S = 256, a 768-wide trunk with stem stride 4
    assert L.vsb_model_create(C.byref(d), C.byref(h)) == 0

    def call(factors, pixelwise, n=None):
        arr = (C.c_int32 * max(1, len(factors)))(*factors)
        return L.vsb_model_set_pixel_decoder(h, len(factors) if n is None else n, arr, pixelwise)
    try:
        assert call([4, 4, 2], 1) == 0
        assert call([2, 2, 2, 2, 2], 1) == 0
        assert call([1], 0) == 0                  # back to the pooled head
        assert call([4, 3, 2], 1) == -2           # VSB_ERR_UNSUPPORTED
        assert call([8], 1) == -2
        assert call([4, 4, 2], 0) == -2           # pooled decoder with stages
        assert call([0, 4], 1) == -1              # VSB_ERR_INVALID
        assert call([4], 2) == -1
        assert call([], 1, n=0) == -1
        assert call([2] * 9, 1) == -1
    finally:
        L.vsb_model_destroy(h)
    d.ext_stem_stride = 2                         # chunkyseal's trunk
    assert L.vsb_model_create(C.byref(d), C.byref(h)) == 0
    try:
        assert call([4, 4, 2], 1) == -2
    finally:
        L.vsb_model_destroy(h)


def test_set_pixel_decoder_before_the_trunk_has_a_map(built_lib):
    """A SAM-ViT spec leaves the ConvNeXt stem stride at 0 (unused); before vsb_model_set_vit_extractor the decoder rules must
    still answer with a status, deciding pooled vs pixel-wise and the stem rule before they ask for the trunk's map."""
    from videoseal_b200 import _lib, cfg
    from videoseal_b200.model import native_desc
    L = _lib.lib()
    h = C.c_void_p()
    d = native_desc(cfg.spec_from_card(load_card("videoseal_1.0")))
    d.ext_stem_stride = 0
    assert L.vsb_model_create(C.byref(d), C.byref(h)) == 0
    try:
        assert L.vsb_model_set_pixel_decoder(h, 1, (C.c_int32 * 1)(1), 0) == 0
        assert L.vsb_model_set_pixel_decoder(h, 3, (C.c_int32 * 3)(4, 4, 2), 1) == -2
        assert "needs a ConvNeXt trunk with stem stride 4" in L.vsb_last_error().decode()
    finally:
        L.vsb_model_destroy(h)
