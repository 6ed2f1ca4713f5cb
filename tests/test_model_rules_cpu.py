"""The load-time geometry rules of libvsb200 without a GPU: each rule accepts on one side of its edge and rejects on the other,
through vsb_model_create / vsb_model_set_pixel_decoder (the C ABI) and through cfg.spec_from_card (its dry run of the same two
calls).  Rejections are VSB_ERR_UNSUPPORTED (NotImplementedError) except the processing-size pitch, a VSB_ERR_INVALID."""
import ctypes as C
import math

import pytest

from tests import pixelwise_oracle as pw
from tests import unet_tiny as ut
from tests.util import load_card

OK, UNSUPPORTED, INVALID = 0, -2, -1


def _card(z=None, img_size=None, nbits=None, dims=None, stages=None, tiny=False):
    """videoseal_1.0 (or its unet_tiny_yuv_quant variant), a pixel-wise convnext_tiny_pw extractor when `stages` is given"""
    card = ut.tiny_card() if tiny else load_card("videoseal_1.0")
    if stages is not None:
        card = pw.preset_card("convnext_tiny_pw", card)
        card["extractor"]["params"]["pixel_decoder"]["upscale_stages"] = stages
    u = card["embedder"]["params"]["unet"]
    if z is not None:
        g = math.gcd(*z)
        u["z_channels"], u["z_channels_mults"] = g, [c // g for c in z]
    if img_size is not None:
        card["args"]["img_size_proc"] = img_size
    if nbits is not None:
        card["args"]["nbits"] = nbits
    if dims is not None:
        card["extractor"]["params"]["encoder"]["dims"] = dims
    return card


def _native_rc(spec):
    """status of vsb_model_create, then of vsb_model_set_pixel_decoder for a pixel-wise spec"""
    from videoseal_b200 import _lib
    from videoseal_b200.model import native_desc
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.vsb_model_create(C.byref(native_desc(spec)), C.byref(h))
    if rc != OK:
        return rc
    try:
        f = spec["pixel_decoder"]["upscale_stages"]
        return L.vsb_model_set_pixel_decoder(h, len(f), (C.c_int32 * len(f))(*f), 1) if spec["pixel_decoder"]["pixelwise"] else OK
    finally:
        L.vsb_model_destroy(h)


def _check(monkeypatch, card, want, hidden=None):
    from videoseal_b200 import cfg, model
    with monkeypatch.context() as m:   # the spec the card describes, before the dry run judges it
        m.setattr(model, "check_native", lambda spec: None)
        spec = cfg.spec_from_card(card)
    if hidden is not None:
        spec["hidden"] = hidden
    assert _native_rc(spec) == want
    if hidden is not None:
        return
    if want == OK:
        assert cfg.spec_from_card(card) == spec
    else:
        with pytest.raises(NotImplementedError if want == UNSUPPORTED else RuntimeError):
            cfg.spec_from_card(card)


@pytest.mark.parametrize("z,want", [
    ([16, 32, 64, 128], OK), ([32, 64, 128, 256], OK), ([64, 128, 256, 512], OK), ([16, 16, 16, 16], OK),
    ([24, 48, 96, 192], UNSUPPORTED),                 # 24: neither 8, 16, 32 nor a multiple of 64
    ([16, 32, 96, 128], UNSUPPORTED),
    ([8, 16, 32, 64], OK),                            # 8 in a leading run of levels
    ([16, 8, 32, 64], UNSUPPORTED),                   # ... but not after a wider level
    ([8, 8, 8, 8], UNSUPPORTED),                      # ... nor at the last level
    ([16, 32, 128, 256], OK),                         # up-conv gathers: 8 * 2^k outputs up to 256 with one vector per thread,
    ([16, 32, 192, 256], UNSUPPORTED),                # 192 = 8 * 24 is no power-of-two thread group
    ([16, 32, 512, 1024], OK),                        # 512: two vectors per thread
    ([16, 64, 1024, 1024], UNSUPPORTED),              # 1024: 64 threads per pixel
])
def test_unet_widths(built_lib, monkeypatch, z, want):
    _check(monkeypatch, _card(z=z), want)


@pytest.mark.parametrize("z,img_size,want", [
    ([16, 32, 64, 128], 128, OK),                     # 4 levels: a 16-pixel bottleneck
    ([16, 16, 32, 64, 128], 256, OK),                 # 5 levels: 16 pixels at 256 ...
    ([16, 16, 32, 64, 128], 128, UNSUPPORTED),        # ... 8 at 128
    ([16, 32, 64, 128], 384, OK),
    ([16, 32, 64, 128], 320, INVALID),                # not a multiple of 128
    ([16, 32, 64, 128], 2048, OK),
])
def test_bottleneck_and_processing_size(built_lib, monkeypatch, z, img_size, want):
    _check(monkeypatch, _card(z=z, img_size=img_size), want)


@pytest.mark.parametrize("tiny", [True, False])
@pytest.mark.parametrize("img_size,want", [(512, OK), (768, OK), (896, UNSUPPORTED), (1024, UNSUPPORTED)])
def test_8_channel_unets_run_up_to_768(built_lib, monkeypatch, tiny, img_size, want):
    """unet_tiny_yuv_quant (z = [8, 8, 16, 32, 64]) and z = [8, 16, 32, 64, 128], whose rings would still fit at 896"""
    card = _card(img_size=img_size, tiny=True) if tiny else _card(z=[8, 16, 32, 64, 128], img_size=img_size)
    _check(monkeypatch, card, want)


@pytest.mark.parametrize("dims_last,stages,want", [
    (16, [2], OK), (32, [2], OK), (64, [2], OK), (96, [4], OK),    # the first stage GEMM takes 16, 32 or >= 64 channels
    (48, [2], UNSUPPORTED), (24, [2, 2], UNSUPPORTED),
    (512, [2, 4, 4], OK),                             # middle stage 256 = 8 * 32
    (1024, [2, 4, 4, 2], UNSUPPORTED),                # 512 = 8 * 64
    (768, [2, 4, 4], OK),                             # 384 = 8 * 3 * 16, 96 = 8 * 3 * 4
    (640, [2, 4, 4], UNSUPPORTED),                    # 320 = 8 * 40
    (768, [4, 4, 2], OK), (768, [2, 2, 2], UNSUPPORTED),   # the last stage holds at most 32 channels
    (768, [4, 4, 4, 2], UNSUPPORTED),                 # 12: not a multiple of 8
])
def test_pixel_decoder_stage_widths(built_lib, monkeypatch, dims_last, stages, want):
    dims = [min(d, dims_last) for d in (96, 192, 384)] + [dims_last]
    _check(monkeypatch, _card(dims=dims, stages=stages), want)


@pytest.mark.parametrize("img_size,want", [(256, OK), (512, OK), (384, UNSUPPORTED), (640, UNSUPPORTED)])
def test_last_stage_tiles_its_map(built_lib, monkeypatch, img_size, want):
    """one factor-2 stage on the img_size / 32 trunk map: the head kernel's 16-pixel output tiles need a multiple of 8"""
    _check(monkeypatch, _card(dims=[64, 64, 64, 64], stages=[2], img_size=img_size), want)


@pytest.mark.parametrize("nbits,hidden,want", [(1888, None, OK), (1896, None, UNSUPPORTED),
                                               (1891, 256, OK), (1892, 256, UNSUPPORTED)])
def test_head_weights_fit_beside_the_staged_taps(built_lib, monkeypatch, nbits, hidden, want):
    """convnext_tiny_pw's last stage (48 -> 24, factor 2): 10^2 * 9 * 24 fp16 taps (43 200 B) + (1 + nbits) * 25 fp32 head weights
    in 227 KB of shared memory, so at most 1891 bits"""
    _check(monkeypatch, _card(nbits=nbits, stages=[4, 4, 2]), want, hidden)
