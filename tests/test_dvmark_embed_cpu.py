"""The DVMark embedder without a GPU: the float64 oracle against the reference's imgs_w (tests/golden/dvmark_embed.pt) and the spread
of its delta, loading of cards and training checkpoints paired with each extractor family, the load-time rules at their edges
through spec_from_card and the C ABI, and the whole-chunk units of dist.shard_unit and the 64-frame group cap."""
import ctypes as C
import os

import pytest
import torch

from tests import dvmark_enc_oracle as de
from tests import hidden_oracle as ho
from tests.util import tmpdir
from videoseal_b200 import _lib, cfg, dist
from videoseal_b200.model import Videoseal, _create, native_desc, native_hidden_desc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "dvmark_embed.pt")
UNSUP, INVALID, STATE = -2, -1, -4


@pytest.mark.parametrize("K", [8, 32])
def test_oracle_matches_golden(K):
    from tests.make_golden_dvmark_embed import CHUNK, STEP, S, cases
    g = torch.load(GOLDEN, weights_only=False)
    assert g["seed"] == de.SEED
    res = g["nbits"][K]
    spec = de.spec_from_card(de.card("dvmark", img_size=S, nbits=K))
    assert spec == res["spec"]
    orc = de.EncOracle(spec, de.synth_state_dict(spec, de.SEED))
    orc.chunk_size, orc.step_size = CHUNK, STEP
    for name, (x, m, is_video) in cases(K).items():
        assert torch.equal(m, res["cases"][name]["msgs"])
        o = orc.embed(x, m, is_video=is_video)["imgs_w"]
        # the reference ran in fp32: its rounding, not the oracle's, sets the bound
        assert (ho.sample(o) - res["cases"][name]["imgs_w"]).abs().max().item() <= 1e-5, name


def test_delta_spread():
    """the synthetic checkpoint's delta is neither saturated nor vanishing, so parity cannot pass vacuously"""
    spec = de.spec_from_card(de.card("dvmark", img_size=128, nbits=32))
    sd = {k: v.double() for k, v in de.synth_state_dict(spec, de.SEED).items() if k.startswith(de.P)}
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    m = torch.randint(0, 2, (2, 32), generator=torch.Generator().manual_seed(2))
    d = de.encoder_forward(sd, x, m)
    assert 0.05 <= d.std().item() <= 0.9 and d.abs().max().item() < 0.99
    # the message changes the delta
    assert (de.encoder_forward(sd, x, 1 - m) - d).abs().max().item() > 1e-2


@pytest.mark.parametrize("ext", de.EXTRACTORS)
def test_card_and_training_checkpoint_load(ext):
    card = de.card(ext)
    spec = cfg.spec_from_card(card)
    assert spec["dvmark_encoder"] == {"nbits": spec["nbits"]} and not spec["yuv"] and "unet" not in spec
    model = Videoseal(spec)
    assert model.temporal and model.dvmark == (ext == "dvmark")
    ext_model = {"convnext": "convnext_tiny", "sam": None}.get(ext, ext)
    if ext_model is None:
        return   # the package has no SAM-ViT extractor preset; the card above loads
    args = dict(card["args"], embedder_model="dvmark", extractor_model=ext_model)
    sd = de.synth_state_dict(de.spec_from_card(card), de.SEED)
    path = tmpdir() / f"train_dvmark_{ext_model}.pth"
    torch.save({"model": sd, "args": args}, path)
    m = cfg.setup_model_from_checkpoint(str(path))
    assert m.temporal and m.spec["dvmark_encoder"]["nbits"] == spec["nbits"]
    assert m.state_dict()["embedder.unet.emb_layer3.4.weight"].shape == (3, 128, 3, 3, 3)


@pytest.mark.parametrize("S,ok", [(128, True), (192, False), (384, True), (512, True), (640, False)])
def test_size_rule(S, ok):
    card = de.card("dvmark", img_size=S)
    if ok:
        cfg.spec_from_card(card)
    else:
        with pytest.raises((NotImplementedError, RuntimeError), match="multiple of 128|at most 512"):
            cfg.spec_from_card(card)


@pytest.mark.parametrize("K", [1, 30, 256])
def test_any_nbits_loads(K):
    assert cfg.spec_from_card(de.card("dvmark", nbits=K))["dvmark_encoder"]["nbits"] == K


def _rc(spec, nbits=None, tweak=None):
    """status of vsb_model_create + vsb_model_set_dvmark_embedder with the descriptor changed by `tweak`"""
    L = _lib.lib()
    d = native_desc(spec)
    if tweak:
        tweak(d)
    h = C.c_void_p()
    rc = L.vsb_model_create(C.byref(d), C.byref(h))
    if rc != 0:
        return rc
    rc = L.vsb_model_set_dvmark_embedder(h, d.nbits if nbits is None else nbits)
    L.vsb_model_destroy(h)
    return rc


def test_c_abi_rules():
    spec = cfg.spec_from_card(de.card("hidden"))

    def t(field, value):
        return lambda d: setattr(d, field, value)
    assert _rc(spec) == 0
    for S, want in ((128, 0), (192, UNSUP), (384, 0), (512, 0), (640, UNSUP)):
        assert _rc(spec, tweak=t("img_size", S)) == want, S
    assert _rc(spec, tweak=t("nbits", 1)) == 0
    assert _rc(spec, nbits=0) == INVALID
    assert _rc(spec, nbits=spec["nbits"] + 1) == INVALID
    L = _lib.lib()
    h = _create(cfg.spec_from_card(ho.card("unet", "hidden")))       # the descriptor describes a U-Net
    assert L.vsb_model_set_dvmark_embedder(h, spec["nbits"]) == INVALID
    L.vsb_model_destroy(h)
    # another embedder first: a HiDDeN embedder, then a DVMark one, and the other way round
    hspec = cfg.spec_from_card(ho.card("hidden", "hidden"))
    h = _create(hspec)
    assert L.vsb_model_set_dvmark_embedder(h, hspec["nbits"]) == STATE
    L.vsb_model_destroy(h)
    h = _create(spec)
    assert L.vsb_model_set_hidden_embedder(h, C.byref(native_hidden_desc(hspec["hidden_encoder"], True))) == STATE
    assert "DVMark" in L.vsb_last_error().decode()
    L.vsb_model_destroy(h)
    # a temporal U-Net's descriptor describes a U-Net (VSB_ERR_INVALID comes after the state check)
    from tests import temporal_oracle as to
    tspec = cfg.spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d"))
    h = _create(tspec)
    assert L.vsb_model_set_dvmark_embedder(h, tspec["nbits"]) == STATE
    L.vsb_model_destroy(h)


def test_shard_and_key_units_hold_whole_chunks():
    model = Videoseal(cfg.spec_from_card(de.card("convnext")))
    model.step_size, model.chunk_size = 4, 6
    assert dist.shard_unit(model) == 24
    both = Videoseal(cfg.spec_from_card(de.card("dvmark")))
    both.step_size, both.chunk_size = 4, 6
    assert dist.shard_unit(both) == 24
    # the 64-frame cap names the DVMark embedder
    model.chunk_size = 65
    with pytest.raises(NotImplementedError, match="DVMark embedder.*64"):
        model._chunk_keys(True, 100)
    assert model._chunk_keys(False, 64) == 64
    with pytest.raises(NotImplementedError, match="64"):
        model._chunk_keys(False, 65)
