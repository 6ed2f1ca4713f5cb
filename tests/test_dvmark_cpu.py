"""The DVMark extractor without a GPU: the float64 oracle against the reference's logits (tests/golden/dvmark.pt), loading of cards and
training checkpoints paired with each embedder family, the load-time rules at their edges through spec_from_card and the C ABI, the
detect groups (frames of different groups never interact), and the entry points that refuse a DVMark extractor."""
import ctypes as C
import os

import pytest
import torch

from tests import dvmark_oracle as dv
from tests.util import tmpdir
from videoseal_b200 import _lib, cfg, dist
from videoseal_b200.model import Videoseal, _create, native_desc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dvmark.pt")
UNSUP, INVALID, STATE = -2, -1, -4


@pytest.mark.parametrize("K", [8, 32])
def test_oracle_matches_golden(K):
    from tests.make_golden_dvmark import S, cases
    g = torch.load(GOLDEN, weights_only=False)
    assert g["seed"] == dv.SEED
    res = g["nbits"][K]
    spec = dv.spec_from_card(dv.card("unet", img_size=S, nbits=K))
    assert spec == res["spec"]
    sd = {k: v.double() for k, v in dv.synth_state_dict(spec, dv.SEED).items()}
    for name, (x, is_video) in cases().items():
        ref = res["cases"][name]["logits"].double()
        o = dv.grouped(sd, x.double(), 2 if is_video else x.shape[0])
        assert o.shape == (x.shape[0], 1 + K)
        # the reference ran in fp32: its rounding, not the oracle's, sets the bound
        assert ((o - ref).abs().max() / ref.abs().max()).item() <= 1e-5, name


@pytest.mark.parametrize("emb", dv.EMBEDDERS)
def test_card_and_training_checkpoint_load(emb):
    card = dv.card(emb)
    spec = cfg.spec_from_card(card)
    assert spec["dvmark_decoder"] == {"nbits": spec["nbits"]} and not spec["pixel_decoder"]["pixelwise"]
    assert "convnext" not in spec and "vit" not in spec and "hidden_decoder" not in spec
    model = Videoseal(spec)
    assert model.dvmark and not model.pixelwise
    # a training checkpoint whose args name the presets loads through the package's configs
    emb_model = "unet_small2_yuv_quant" if emb == "unet" else emb
    args = dict(card["args"], embedder_model=emb_model, extractor_model="dvmark")
    sd = dv.synth_state_dict(dv.spec_from_card(dv.card(emb_model)), dv.SEED)
    path = tmpdir() / f"train_{emb_model}_dvmark.pth"
    torch.save({"model": sd, "args": args}, path)
    m = cfg.setup_model_from_checkpoint(str(path))
    assert m.dvmark and m.spec["dvmark_decoder"]["nbits"] == spec["nbits"]
    assert m.state_dict()["detector.layers.layer4.weight"].shape == (1 + spec["nbits"], 256, 3, 3, 3)


@pytest.mark.parametrize("S,ok", [(128, True), (192, False), (256, True), (320, False), (384, True)])
def test_size_rule(S, ok):
    """every embedder already needs a multiple of 128 and says so first (RuntimeError); the DVMark setter's own refusal
    (NotImplementedError, VSB_ERR_UNSUPPORTED) is pinned by test_c_abi_rules"""
    card = dv.card("hidden", img_size=S)
    if ok:
        cfg.spec_from_card(card)
    else:
        with pytest.raises((NotImplementedError, RuntimeError), match="multiple of 128"):
            cfg.spec_from_card(card)


@pytest.mark.parametrize("K", [1, 2, 96, 256])
def test_any_nbits_loads(K):
    assert cfg.spec_from_card(dv.card("hidden", nbits=K))["dvmark_decoder"]["nbits"] == K


@pytest.mark.parametrize("is_video,frames,size,ok", [
    (True, 100, 64, True), (True, 100, 65, False), (True, 20, 65, True), (True, 65, 65, False), (False, 64, 8, True),
    (False, 65, 8, False), (False, 200, 8, False), (True, 200, 8, True)])
def test_group_rule(is_video, frames, size, ok):
    """a detector call (a chunk of chunk_size frames in video mode, so at most the clip; the whole batch in image mode) holds at
    most 64 frames"""
    model = Videoseal(cfg.spec_from_card(dv.card("unet")))
    model.chunk_size = size
    if ok:
        assert model._detect_group(is_video, frames) == (min(size, frames) if is_video else frames)
    else:
        with pytest.raises(NotImplementedError, match="at most 64"):
            model._detect_group(is_video, frames)


def test_group_rule_only_binds_dvmark():
    model = Videoseal(cfg.spec_from_card(dv.ho.card("unet", "convnext")))
    assert model._detect_group(False, 200) == 200


def _rc(spec, nbits=None, tweak=None):
    """status of vsb_model_create + vsb_model_set_dvmark_extractor with the descriptor changed by `tweak`"""
    L = _lib.lib()
    d = native_desc(spec)
    if tweak:
        tweak(d)
    h = C.c_void_p()
    rc = L.vsb_model_create(C.byref(d), C.byref(h))
    if rc != 0:
        return rc
    rc = L.vsb_model_set_dvmark_extractor(h, d.nbits if nbits is None else nbits)
    L.vsb_model_destroy(h)
    return rc


def test_c_abi_rules():
    spec = cfg.spec_from_card(dv.card("hidden"))
    assert _rc(spec) == 0

    def t(field, value):
        return lambda d: setattr(d, field, value)
    assert _rc(spec, tweak=t("img_size", 128)) == 0
    assert _rc(spec, tweak=t("img_size", 192)) == UNSUP
    assert _rc(spec, tweak=t("img_size", 384)) == 0
    assert _rc(spec, tweak=t("nbits", 1)) == 0
    assert _rc(spec, nbits=0) == INVALID
    assert _rc(spec, nbits=spec["nbits"] + 1) == INVALID

    def with_cnx(d):
        d.ext_dims[0] = 96
    assert _rc(spec, tweak=with_cnx) == INVALID
    # call order: a DVMark extractor after a SAM-ViT trunk, and a SAM-ViT trunk after it
    L = _lib.lib()
    h = _create(cfg.spec_from_card(dv.ho.card("hidden", "sam")))
    assert L.vsb_model_set_dvmark_extractor(h, spec["nbits"]) == STATE
    L.vsb_model_destroy(h)
    h = _create(spec)
    from videoseal_b200.model import native_vit_desc
    sam = cfg.spec_from_card(dv.ho.card("hidden", "sam"))
    assert L.vsb_model_set_vit_extractor(h, C.byref(native_vit_desc(sam["vit"]))) == STATE
    assert L.vsb_model_set_pixel_decoder(h, 1, (C.c_int32 * 1)(2), 1) == UNSUP
    L.vsb_model_destroy(h)


def test_streaming_entry_points_refuse_dvmark():
    """vsb_embed_detect_host and vsb_frames_host_u8 with logits cut the frames on slices of their own: they refuse a DVMark
    extractor before reading any buffer (on a handle that is not even finalized)"""
    L = _lib.lib()
    spec = cfg.spec_from_card(dv.card("unet"))
    h = _create(spec)
    buf = (C.c_float * 16)()
    u8 = (C.c_uint8 * 16)()
    rc = L.vsb_embed_detect_host(h, buf, u8, 1, buf, buf, 1, 4, 4, 1, 0, 1, 1.0, 0.2, 0)
    assert rc == UNSUP and "DVMark" in L.vsb_last_error().decode()
    rc = L.vsb_frames_host_u8(h, u8, u8, 1, None, buf, 1, 4, 4, 1, 0, 1, 1.0, 0.2, 0)
    assert rc == UNSUP and "DVMark" in L.vsb_last_error().decode()
    L.vsb_model_destroy(h)


def test_shards_hold_whole_detect_chunks():
    model = Videoseal(cfg.spec_from_card(dv.card("unet")))
    model.step_size, model.chunk_size = 4, 6
    assert dist.shard_unit(model) == 12
    model.chunk_size = 8
    assert dist.shard_unit(model) == 8
    other = Videoseal(cfg.spec_from_card(dv.ho.card("unet", "convnext")))
    other.step_size, other.chunk_size = 4, 6
    assert dist.shard_unit(other) == 4


def test_groups_never_interact():
    """frames of different detector calls do not see each other; frames of one call do"""
    spec = dv.spec_from_card(dv.card("unet", img_size=32, nbits=4))
    sd = {k: v.double() for k, v in dv.synth_state_dict(spec, dv.SEED).items()}
    x = torch.rand(5, 3, 32, 32, generator=torch.Generator().manual_seed(8), dtype=torch.float64)
    y = x.clone()
    y[2] = 1 - y[2]                        # a frame of the second group of 2
    a, b = dv.grouped(sd, x, 2), dv.grouped(sd, y, 2)
    assert torch.equal(a[:2], b[:2]) and torch.equal(a[4:], b[4:])
    assert (a[3] - b[3]).abs().max() > 1e-6
    # one call over all five frames mixes them
    assert (dv.grouped(sd, x, 5)[1] - dv.grouped(sd, y, 5)[1]).abs().max() > 1e-6
    # each group is the reference's call on its frames alone
    assert torch.equal(a[2:4], dv.decoder_forward(sd, x[2:4]))
