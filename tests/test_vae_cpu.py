"""The VAE embedder without a GPU: the float64 oracle against the reference's imgs_w (tests/golden/vae.pt) and the spread of its
delta, loading of cards and training checkpoints paired with each extractor family, the load-time rules at their edges through
spec_from_card and the C ABI, and the out-of-scope card keys that must raise at load."""
import copy
import ctypes as C
import os

import pytest
import torch

from tests import hidden_oracle as ho
from tests import vae_oracle as vo
from tests.util import tmpdir
from videoseal_b200 import _lib, cfg
from videoseal_b200.model import Videoseal, _create, delta_channels, native_desc, native_hidden_desc, native_vae_desc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vae.pt")
UNSUP, INVALID, STATE = -2, -1, -4


def test_oracle_matches_golden():
    from tests.make_golden_vae import CHUNK, NBITS, PRESETS, STEP, S, cases
    g = torch.load(GOLDEN, weights_only=False)
    assert g["seed"] == vo.SEED
    for preset in PRESETS:
        for K in NBITS:
            res = g["presets"][(preset, K)]
            spec = vo.spec_from_card(vo.card(preset, img_size=S, nbits=K))
            assert spec == res["spec"]
            orc = vo.VaeOracle(spec, vo.synth_state_dict(spec, vo.SEED))
            orc.chunk_size, orc.step_size = CHUNK, STEP
            for name, (x, m, is_video) in cases(K).items():
                assert torch.equal(m, res["cases"][name]["msgs"])
                o = orc.embed(x, m, is_video=is_video)["imgs_w"]
                # the reference ran in fp32: its rounding, not the oracle's, sets the bound
                assert (ho.sample(o) - res["cases"][name]["imgs_w"]).abs().max().item() <= 1e-5, (preset, K, name)


@pytest.mark.parametrize("preset", vo.PRESETS)
def test_delta_spread(preset):
    """the synthetic checkpoint's delta is neither saturated nor vanishing, and the message moves it, so parity cannot pass
    vacuously"""
    spec = vo.spec_from_card(vo.card(preset, img_size=128, nbits=32))
    sd = {k: v.double() for k, v in vo.synth_state_dict(spec, vo.SEED).items() if k.startswith("embedder.")}
    v = spec["vae_encoder"]
    x = torch.rand(2, v["in_channels"], 128, 128, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    m = torch.randint(0, 2, (2, 32), generator=torch.Generator().manual_seed(2))
    d = vo.vae_forward(sd, v, x, m)
    assert d.shape == (2, v["out_ch"], 128, 128)
    assert 0.05 <= d.std().item() <= 0.9 and d.abs().max().item() < 0.999
    assert (vo.vae_forward(sd, v, x, 1 - m) - d).abs().max().item() > 1e-2


@pytest.mark.parametrize("preset", vo.PRESETS)
def test_spec_of_each_preset(preset):
    spec = cfg.spec_from_card(vo.card(preset))
    want = vo.spec_from_card(vo.card(preset))["vae_encoder"]
    assert spec["vae_encoder"] == want and "unet" not in spec
    assert spec["yuv"] == ("yuv" in preset)
    assert delta_channels(spec) == want["out_ch"]


@pytest.mark.parametrize("ext", vo.EXTRACTORS)
def test_card_and_training_checkpoint_load(ext):
    """a card with each extractor family loads; a training checkpoint (embedder_model: vae_small) loads with each extractor preset of
    the package's configs/extractor.yaml.  That file has no SAM-ViT preset (no `sam_small`), so the SAM-ViT pairing is checked
    through the card only"""
    card = vo.card("vae_small", extractor=ext)
    spec = cfg.spec_from_card(card)
    model = Videoseal(spec)
    assert not model.temporal
    ext_model = {"convnext": "convnext_tiny", "sam": None}.get(ext, ext)
    if ext_model is None:
        return   # the package has no SAM-ViT extractor preset; the card above loads
    args = dict(card["args"], embedder_model="vae_small", extractor_model=ext_model)
    sd = vo.synth_state_dict(vo.spec_from_card(card), vo.SEED)
    path = tmpdir() / f"train_vae_small_{ext_model}.pth"
    torch.save({"model": sd, "args": args}, path)
    m = cfg.setup_model_from_checkpoint(str(path))
    assert m.spec["vae_encoder"]["ch"] == 32 and m.spec["hidden"] == spec["hidden"]
    assert m.state_dict()["embedder.decoder.conv_in.weight"].shape == (128, 4 + m.spec["hidden"], 3, 3)


@pytest.mark.parametrize("S,ok", [(128, True), (256, True), (384, True), (512, True), (640, True), (768, True), (896, False),
                                  (320, False)])
def test_size_rule(S, ok):
    """a multiple of 128 and at most 768 (with four levels the deepest map, S / 8, is then a multiple of 16)"""
    card = vo.card("vae_small", img_size=S)
    if ok:
        cfg.spec_from_card(card)
    else:
        with pytest.raises((NotImplementedError, RuntimeError), match="processing size"):
            cfg.spec_from_card(card)


def _params(preset="vae_small"):
    return copy.deepcopy(ho._presets("embedder")[preset])


def _with(part, key, value):
    def f(p):
        p[part][key] = value
    return f


OUT_OF_SCOPE = {
    "attn_resolutions": _with("encoder", "attn_resolutions", [32]),
    "dec_attn_resolutions": _with("decoder", "attn_resolutions", [32]),
    "use_linear_attn": _with("decoder", "use_linear_attn", True),
    "attn_type": _with("encoder", "attn_type", "linear"),
    "resamp_with_conv": _with("encoder", "resamp_with_conv", False),
    "double_z": _with("encoder", "double_z", True),
    "double_z_default": lambda p: p["encoder"].pop("double_z"),
    "give_pre_end": _with("decoder", "give_pre_end", True),
    "bw": _with("decoder", "bw", True),
    "msg_processor_type": _with("msg_processor", "msg_processor_type", "gaussian+concat"),
    "msg_mult": _with("msg_processor", "msg_mult", 2.0),
}


@pytest.mark.parametrize("what", sorted(OUT_OF_SCOPE))
def test_out_of_scope_keys_raise(what):
    card = vo.card("vae_small")
    p = _params()
    OUT_OF_SCOPE[what](p)
    card["embedder"]["params"] = p
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)


def test_ignored_keys():
    """the encoder's out_ch, resolution and dropout change nothing in eval"""
    card = vo.card("vae_small")
    base = cfg.spec_from_card(card)
    p = _params()
    p["encoder"].update(out_ch=7, resolution=64, dropout=0.3)
    card["embedder"]["params"] = p
    assert cfg.spec_from_card(card)["vae_encoder"] == base["vae_encoder"]


def test_unknown_embedder_names_vae():
    card = vo.card("vae_small")
    card["embedder"]["model"] = "patchmixer_tiny"
    with pytest.raises(NotImplementedError, match="vae\\*"):
        cfg.spec_from_card(card)


def _rc(spec, tweak_desc=None, tweak_vae=None):
    """status of vsb_model_create + vsb_model_set_vae_embedder with the descriptors changed by the tweaks"""
    L = _lib.lib()
    d = native_desc(spec)
    if tweak_desc:
        tweak_desc(d)
    v = native_vae_desc(spec["vae_encoder"])
    if tweak_vae:
        tweak_vae(v)
    h = C.c_void_p()
    rc = L.vsb_model_create(C.byref(d), C.byref(h))
    if rc != 0:
        return rc
    rc = L.vsb_model_set_vae_embedder(h, C.byref(v))
    L.vsb_model_destroy(h)
    return rc


def _set(field, value):
    return lambda d: setattr(d, field, value)


def _mult(*m):
    def f(v):
        v.levels = len(m)
        for i, x in enumerate(m):
            v.ch_mult[i] = x
    return f


def test_c_abi_rules():
    spec = cfg.spec_from_card(vo.card("vae_small"))
    yspec = cfg.spec_from_card(vo.card("vae_small_yuv"))
    assert _rc(spec) == 0 and _rc(yspec) == 0
    # widths 16, 32, 64, 128 on both sides of each edge; the head dim (last width) 64 or 128
    assert _rc(spec, tweak_vae=_set("ch", 16)) == 0                           # vae_tiny's 16, 32, 32, 64
    assert _rc(spec, tweak_vae=_set("ch", 48)) == UNSUP
    assert _rc(spec, tweak_vae=_mult(1, 2, 2, 8)) == UNSUP                    # 256 wide
    assert _rc(spec, tweak_vae=_mult(1, 2, 2, 2)) == 0                        # head dim 64
    assert _rc(spec, tweak_vae=_mult(1, 1, 1, 1)) == UNSUP                    # head dim 32
    assert _rc(spec, tweak_vae=lambda v: (_set("ch", 8)(v), _mult(2, 4, 8, 16)(v))) == UNSUP   # ch 8
    # the deepest map (the attention grid) at most 96 wide: fewer levels leave a wider one
    assert _rc(spec, tweak_vae=_mult(1, 2, 4)) == 0                           # 3 levels at 256: 64
    assert _rc(spec, tweak_vae=_mult(2, 4)) == UNSUP                          # 2 levels at 256: 128
    assert _rc(spec, tweak_desc=_set("img_size", 128), tweak_vae=_mult(2, 4)) == 0     # 2 levels at 128: 64
    assert _rc(spec, tweak_desc=_set("img_size", 768), tweak_vae=_mult(1, 2, 4)) == UNSUP   # 3 levels at 768: 192
    # z_channels <= 16, out_ch 1 or 3
    assert _rc(spec, tweak_vae=_set("z_channels", 16)) == 0
    assert _rc(spec, tweak_vae=_set("z_channels", 17)) == UNSUP
    for oc, want in ((1, 0), (2, UNSUP), (3, 0), (4, UNSUP)):
        assert _rc(spec, tweak_vae=_set("out_ch", oc)) == want, oc
    # processing sizes
    for S, want in ((128, 0), (256, 0), (768, 0), (896, UNSUP), (200, UNSUP), (0, UNSUP)):
        assert _rc(spec, tweak_desc=_set("img_size", S)) == want, S
    # yuv must match in_ch == 1
    assert _rc(spec, tweak_desc=_set("yuv", 1)) == INVALID
    assert _rc(yspec, tweak_desc=_set("yuv", 0)) == INVALID
    assert _rc(spec, tweak_vae=_set("in_ch", 2)) == INVALID
    assert _rc(spec, tweak_vae=_set("levels", 0)) == INVALID
    assert _rc(spec, tweak_vae=_set("levels", 7)) == INVALID
    assert _rc(spec, tweak_vae=_set("tanh_out", 2)) == INVALID
    assert _rc(spec, tweak_vae=_set("num_res_blocks", 0)) == INVALID
    L = _lib.lib()
    v = native_vae_desc(spec["vae_encoder"])
    h = _create(cfg.spec_from_card(ho.card("unet", "hidden")))       # the descriptor describes a U-Net
    assert L.vsb_model_set_vae_embedder(h, C.byref(v)) == INVALID
    L.vsb_model_destroy(h)
    # beside another embedder: HiDDeN, DVMark, temporal U-Net, in both orders
    hspec = cfg.spec_from_card(ho.card("hidden", "hidden"))
    h = _create(hspec)
    assert L.vsb_model_set_vae_embedder(h, C.byref(v)) == STATE
    L.vsb_model_destroy(h)
    h = _create(spec)
    assert L.vsb_model_set_hidden_embedder(h, C.byref(native_hidden_desc(hspec["hidden_encoder"], True))) == STATE
    assert L.vsb_model_set_dvmark_embedder(h, spec["nbits"]) == STATE
    L.vsb_model_destroy(h)
    from tests import dvmark_enc_oracle as de
    h = _create(cfg.spec_from_card(de.card("hidden")))
    assert L.vsb_model_set_vae_embedder(h, C.byref(v)) == STATE
    L.vsb_model_destroy(h)
    from tests import temporal_oracle as to
    h = _create(cfg.spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d")))
    assert L.vsb_model_set_vae_embedder(h, C.byref(v)) == STATE
    L.vsb_model_destroy(h)
