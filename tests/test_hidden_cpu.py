"""HiDDeN embedders and extractors without a GPU: the CPU oracle against the reference's outputs (tests/golden/hidden.pt), loading of
cards and training checkpoints for both presets and the mixed pairings, the load-time rules at their edges through spec_from_card
and the C ABI, and the configurations that are out of scope."""
import ctypes as C
import os

import pytest
import torch

from tests import hidden_oracle as ho
from tests.util import tmpdir
from videoseal_b200 import _lib, cfg
from videoseal_b200.model import _create, native_desc, native_hidden_desc

GOLDEN = os.path.join(ho.ROOT, "tests", "golden", "hidden.pt")


@pytest.mark.parametrize("preset", ho.PRESETS)
def test_oracle_matches_golden(preset):
    g = torch.load(GOLDEN, weights_only=False)
    assert g["seed"] == ho.SEED
    res = g["presets"][preset]
    spec = ho.spec_from_card(ho.card(preset, preset))
    assert spec == res["spec"]
    orc = ho.HiddenOracle(spec, ho.synth_state_dict(spec, ho.SEED))
    orc.chunk_size = 2
    from tests.make_golden_hidden import cases
    for name, (x, m, is_video) in cases(spec["nbits"]).items():
        c = res["cases"][name]
        assert torch.equal(m, c["msgs"])
        o = orc.embed(x, m, is_video=is_video)
        assert (ho.sample(o["imgs_w"]) - c["imgs_w_s"]).abs().max().item() <= 1e-6, name
        if c["preds_w_s"] is not None:
            assert (ho.sample(o["preds_w"]) - c["preds_w_s"]).abs().max().item() <= 1e-6, name
        lg = orc.detect(o["imgs_w"], is_video=is_video)["preds"]
        assert (lg - c["logits"]).abs().max().item() <= 1e-4 * (1 + c["logits"].abs().max().item()), name


@pytest.mark.parametrize("emb,ext", ho.PAIRINGS)
def test_card_and_training_checkpoint_load(emb, ext):
    card = ho.card(emb, ext)
    spec = cfg.spec_from_card(card)
    assert ("hidden_encoder" in spec) == emb.startswith("hidden") and ("hidden_decoder" in spec) == ext.startswith("hidden")
    assert ("unet" in spec) != ("hidden_encoder" in spec)
    osp = ho.spec_from_card(card)
    sd = ho.synth_state_dict(osp, ho.SEED)
    if emb.startswith("hidden") and ext.startswith("hidden"):
        # a training checkpoint (args naming the presets) loads through the package's configs
        args = dict(card["args"], embedder_model=emb, extractor_model=ext)
        path = tmpdir() / f"train_{emb}_{ext}.pth"
        torch.save({"model": sd, "args": args}, path)
        model = cfg.setup_model_from_checkpoint(str(path))
        assert model.spec["hidden_encoder"]["normalization"] == osp["hidden_encoder"]["normalization"][:5]
        assert model.spec["hidden_decoder"]["num_blocks"] == osp["hidden_decoder"]["num_blocks"]


def test_baseline_hidden_still_raises():
    with pytest.raises(NotImplementedError):
        cfg.setup_model_from_checkpoint("baseline/hidden")


@pytest.mark.parametrize("side,key,value", [
    ("embedder", "normalization", "layer"), ("embedder", "normalization", "rms"), ("embedder", "activation", "silu"),
    ("embedder", "activation", "leakyrelu"), ("embedder", "in_channels", 1), ("embedder", "out_channels", 1),
    ("extractor", "normalization", "layer"), ("extractor", "activation", "silu"), ("extractor", "pixelwise", True),
    ("extractor", "in_channels", 1)])
def test_out_of_scope_raises(side, key, value):
    card = ho.card("hidden", "hidden")
    card[side]["params"][key] = value
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)


@pytest.mark.parametrize("norm,act", [("batch", "relu"), ("batch", "gelu"), ("group", "relu"), ("group", "gelu")])
def test_norm_and_activation_are_independent(norm, act):
    card = ho.card("hidden", "hidden")
    for side in ("embedder", "extractor"):
        card[side]["params"].update(normalization=norm, activation=act)
    spec = cfg.spec_from_card(card)
    assert spec["hidden_encoder"]["normalization"] == norm and spec["hidden_decoder"]["activation"] == act


@pytest.mark.parametrize("z,ok", [(56, False), (64, True), (72, False), (128, False)])
def test_width_rule(z, ok):
    card = ho.card("hidden", "hidden")
    card["embedder"]["params"]["z_channels"] = z
    if ok:
        cfg.spec_from_card(card)
    else:
        with pytest.raises(NotImplementedError):
            cfg.spec_from_card(card)


@pytest.mark.parametrize("S,ok", [(128, True), (192, False), (256, True), (384, True)])
def test_size_rule(S, ok):
    card = ho.card("hidden", "hidden", img_size=S)
    if ok:
        cfg.spec_from_card(card)
    else:
        with pytest.raises(RuntimeError, match="multiple of 128"):
            cfg.spec_from_card(card)


def _rc(spec, emb=None, ext=None, tweak=None):
    """status of vsb_model_create + the HiDDeN setters on `spec` with the descriptors changed by `tweak`"""
    L = _lib.lib()
    d = native_desc(spec)
    he = native_hidden_desc(spec["hidden_encoder"], True) if "hidden_encoder" in spec else None
    hd = native_hidden_desc(spec["hidden_decoder"], False) if "hidden_decoder" in spec else None
    if tweak:
        tweak(d, he, hd)
    h = C.c_void_p()
    rc = L.vsb_model_create(C.byref(d), C.byref(h))
    if rc != 0:
        return rc
    if he is not None:
        rc = L.vsb_model_set_hidden_embedder(h, C.byref(he))
    if rc == 0 and hd is not None:
        rc = L.vsb_model_set_hidden_extractor(h, C.byref(hd))
    L.vsb_model_destroy(h)
    return rc


def test_c_abi_rules():
    spec = cfg.spec_from_card(ho.card("hidden", "hidden"))
    assert _rc(spec) == 0

    def t(field, value, which="he"):
        def f(d, he, hd):
            setattr({"he": he, "hd": hd, "d": d}[which], field, value)
        return f
    UNSUP, INVALID, STATE = -2, -1, -4
    assert _rc(spec, tweak=t("z_channels", 32)) == UNSUP
    assert _rc(spec, tweak=t("z_channels", 64)) == 0
    assert _rc(spec, tweak=t("norm", 2)) == UNSUP
    assert _rc(spec, tweak=t("act", 2, "hd")) == UNSUP
    assert _rc(spec, tweak=t("num_layers", 0)) == INVALID
    assert _rc(spec, tweak=t("num_layers", 1)) == 0
    assert _rc(spec, tweak=t("num_layers", 64, "hd")) == 0
    assert _rc(spec, tweak=t("num_layers", 65, "hd")) == INVALID
    assert _rc(spec, tweak=t("last_tanh", 1, "hd")) == INVALID
    assert _rc(spec, tweak=t("last_tanh", 2)) == INVALID
    assert _rc(spec, tweak=t("img_size", 192, "d")) == INVALID
    assert _rc(spec, tweak=t("img_size", 128, "d")) == 0
    assert _rc(spec, tweak=t("nbits", 0, "d")) == INVALID
    assert _rc(spec, tweak=t("nbits", 1, "d")) == 0
    # a descriptor that also describes the network a HiDDeN setter replaces
    assert _rc(spec, tweak=t("unet_levels", 4, "d")) in (INVALID, UNSUP)
    mixed = cfg.spec_from_card(ho.card("hidden", "convnext"))
    assert _rc(mixed) == 0

    def with_cnx(d, he, hd):
        d.ext_dims[0] = 96
    assert _rc(spec, tweak=with_cnx) == INVALID
    # call order: the HiDDeN extractor after a SAM-ViT trunk; set after finalize is VSB_ERR_STATE (finalize needs a GPU: not here)
    L = _lib.lib()
    sam = cfg.spec_from_card(ho.card("hidden", "sam"))
    h = _create(sam)
    hd = native_hidden_desc(spec["hidden_decoder"], False)
    assert L.vsb_model_set_hidden_extractor(h, C.byref(hd)) == STATE
    L.vsb_model_destroy(h)


def test_no_embedder_still_fails():
    """a descriptor with neither U-Net levels nor a HiDDeN embedder is no model: create fails (the U-Net's rule), or, with the RGB
    channels a HiDDeN embedder leaves, finalize does"""
    L = _lib.lib()
    spec = cfg.spec_from_card(ho.card("hidden", "convnext"))
    d = native_desc(spec)
    assert (d.unet_levels, d.unet_in_ch, d.unet_out_ch) == (0, 3, 3)
    h = C.c_void_p()
    assert L.vsb_model_create(C.byref(d), C.byref(h)) == 0
    assert L.vsb_model_finalize(h, 0) != 0
    L.vsb_model_destroy(h)
    d.unet_in_ch = 0
    assert L.vsb_model_create(C.byref(d), C.byref(h)) == -1


def step_frames(B, S, seed):
    """frames whose statistics differ from frame to frame (so that a frame given another's GroupNorm statistics is visible)"""
    x = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed))
    scale = torch.linspace(0.3, 1.0, B)[:, None, None, None]
    return (x * scale + (1 - scale) * torch.linspace(0.0, 0.6, B)[:, None, None, None]).clamp(0, 1)


@pytest.mark.parametrize("preset", ho.PRESETS)
def test_step_bounds_cover_fp16_emulation_and_catch_mutations(preset):
    """every step's float64 bound holds for an fp16 emulation of its kernel, and every mutation of tests/hidden_kernels.py leaves it"""
    from tests import hidden_kernels as hk
    spec = ho.spec_from_card(ho.card(preset, preset))
    sd = ho.synth_state_dict(spec, ho.SEED)
    x = step_frames(3, 64, 21)
    m = torch.randint(0, 2, (3, spec["nbits"]), generator=torch.Generator().manual_seed(22))
    J = hk.Judge()
    hk.check_encoder(sd, spec, x, m, hk.emulate(sd, spec, x, m, decoder=False), J)
    taps = hk.emulate(sd, spec, x, None, decoder=True)
    hk.check_decoder(sd, spec, x, taps, taps["logits"], J)
    grp = preset == "hidden"
    want = {"x01@conv3-64", "msg01@msg_table", "order@msg_table", "border@msg_table", "x01@concat_x+msg", "msg01@concat_x+msg",
            "border@concat_x+msg", "order@concat_conv", "tanh@norm_act+outc", "nobias@linear"}
    if grp:
        want |= {"interleaved@gn_stats", "interleaved@gn_apply", "frame0@gn_apply", "interleaved@norm_act+outc", "frame0@norm_act+outc",
                 "interleaved@norm_act+pool", "frame0@norm_act+pool"}
    assert want <= set(J.mutations), want - set(J.mutations)
    print(preset, {k: round(v, 3) for k, v in J.worst.items()}, {k: round(v, 1) for k, v in J.mutations.items()})


def test_unet_without_levels_fails_at_load():
    card = ho.card("unet", "convnext")
    card["embedder"]["params"]["unet"]["z_channels_mults"] = []
    with pytest.raises(RuntimeError, match="unet levels"):
        cfg.spec_from_card(card)
