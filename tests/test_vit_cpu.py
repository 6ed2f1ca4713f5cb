"""SAM-ViT extractor without a GPU: the load rules on both sides of each edge (through spec_from_card and through the C ABI), the
call order of vsb_model_set_vit_extractor, the img_size setter, and the test oracle against restate's."""
import ctypes as C

import pytest
import torch

from tests import vit_oracle as vo
from videoseal_b200 import _lib, cfg
from videoseal_b200.model import _create, native_desc, native_vit_desc

# (encoder overrides, img_size): accepted / rejected on the other side of the same edge
EDGES = [
    ("head dim", ({"num_heads": 6}, None), ({"num_heads": 12}, None)),                     # 64 vs 32
    ("window tokens", ({"window_size": 16}, None), ({"window_size": 4}, None)),            # 256 / 64 vs 16
    ("window divides grid", ({"window_size": 8}, None), ({"window_size": 14}, None)),
    ("global tokens", ({}, 512), ({}, 640)),                                               # 1024 vs 1600
    ("mlp_dim", ({"mlp_ratio": 4}, None), ({"mlp_ratio": 4.0625}, None)),                  # 1536 vs 1560
    ("out_chans", ({"out_chans": 384}, None), ({"out_chans": 392}, None)),
    ("depth", ({"depth": 32, "global_attn_indexes": [2, 31]}, None), ({"depth": 33, "global_attn_indexes": [2, 32]}, None)),
    ("use_abs_pos", ({"use_abs_pos": True}, None), ({"use_abs_pos": False}, None)),
    ("temporal_attention", ({"temporal_attention": False}, None), ({"temporal_attention": True}, None)),
    # relative positions: a table's 2n - 1 rows are staged in 64, so windows up to 32 tokens wide
    ("rel-pos window width", ({"window_size": 32, "global_attn_indexes": []}, 1024), ({"window_size": 64, "global_attn_indexes": []}, 1024)),
    ("rel-pos window 40", ({"window_size": 40, "global_attn_indexes": [], "use_rel_pos": False}, 640),
     ({"window_size": 40, "global_attn_indexes": [], "use_rel_pos": True}, 640)),
]


@pytest.mark.parametrize("edge", EDGES, ids=[e[0] for e in EDGES])
def test_load_rule_edges_through_spec_from_card(edge):
    _, (ok_enc, ok_size), (bad_enc, bad_size) = edge
    spec = cfg.spec_from_card(vo.vit_card(False, ok_size, ok_enc))
    assert "vit" in spec and "convnext" not in spec
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(vo.vit_card(False, bad_size, bad_enc))


def _abi(spec, **vit):
    """status of create + set_vit_extractor for spec with spec['vit'] fields overridden"""
    L = _lib.lib()
    h = C.c_void_p()
    _lib.check(L.vsb_model_create(C.byref(native_desc(spec)), C.byref(h)))
    try:
        return L.vsb_model_set_vit_extractor(h, C.byref(native_vit_desc({**spec["vit"], **vit})))
    finally:
        L.vsb_model_destroy(h)


def test_load_rule_edges_through_the_c_abi():
    spec = cfg.spec_from_card(vo.vit_card(False))
    assert _abi(spec) == 0
    for ok, bad in [({"num_heads": 6}, {"num_heads": 12}), ({"window_size": 16}, {"window_size": 4}),
                    ({"mlp_dim": 1536}, {"mlp_dim": 1560}), ({"out_chans": 384}, {"out_chans": 392}),
                    ({"depth": 32, "global_attn_indexes": [31]}, {"depth": 33, "global_attn_indexes": [2]}),
                    ({"patch_size": 16}, {"patch_size": 8})]:
        assert _abi(spec, **ok) == 0, ok
        assert _abi(spec, **bad) == -2, bad                # VSB_ERR_UNSUPPORTED
    big = {**spec, "img_size": 640}
    assert _abi({**spec, "img_size": 512}) == 0
    assert _abi(big) == -2 and b"1600" in _lib.lib().vsb_last_error()
    assert _abi(big, global_attn_indexes=[]) == 0          # windows of 64 tokens only: no global block
    # rel-pos tables of 2 * 40 - 1 = 79 rows do not fit the kernel's 64; without rel-pos the 1600-token windows run
    assert _abi(big, global_attn_indexes=[], window_size=40) == -2 and b"40-token-wide" in _lib.lib().vsb_last_error()
    assert _abi(big, global_attn_indexes=[], window_size=40, use_rel_pos=False) == 0
    assert _abi({**spec, "img_size": 1024}, global_attn_indexes=[], window_size=32) == 0
    assert _abi(spec, depth=0) == -1                        # invalid, not unsupported


def test_pixelwise_stages_on_the_vit_trunk():
    spec = cfg.spec_from_card(vo.vit_card(True))            # sam_small_pw: 384 -> 96 -> 48 -> 24 channels on a 16-token grid
    assert spec["pixel_decoder"] == {"pixelwise": True, "upscale_stages": [4, 2, 2]}
    card = vo.vit_card(True)
    card["extractor"]["params"]["pixel_decoder"]["upscale_stages"] = [2, 2, 2, 2, 2]   # a 12-channel last stage
    with pytest.raises(NotImplementedError):
        cfg.spec_from_card(card)


def test_call_order():
    spec = cfg.spec_from_card(vo.vit_card(True))
    L = _lib.lib()
    h = _create(spec)   # create, set_vit_extractor, set_pixel_decoder
    try:
        assert L.vsb_model_set_vit_extractor(h, C.byref(native_vit_desc(spec["vit"]))) == -4   # after set_pixel_decoder
    finally:
        L.vsb_model_destroy(h)


def test_img_size_setter():
    from videoseal_b200.model import Videoseal
    spec = cfg.spec_from_card(vo.vit_card(False))
    m = Videoseal(spec)
    m.img_size = 512                     # no weights yet: only the native rules apply
    assert m.img_size == 512
    with pytest.raises(NotImplementedError, match="2304"):
        m.img_size = 768                 # 2304 global tokens: outside the kernels, like any unsupported size
    m = Videoseal(spec)
    m.load_state_dict({"detector.image_encoder.pos_embed": torch.zeros(1, 16, 16, 384)})
    with pytest.raises(ValueError, match="pos_embed"):
        m.img_size = 384
    m.img_size = 256
    assert m.img_size == 256


def test_rejects_convnext_keys_under_a_sam_name():
    card = vo.vit_card(False)
    card["extractor"]["params"]["encoder"]["dims"] = [96, 192, 384, 768]
    with pytest.raises(NotImplementedError, match="ConvNeXt keys"):
        cfg.spec_from_card(card)


@pytest.mark.parametrize("variant", ["sam_small", "sam_small_pw"])
def test_oracle_matches_the_reference_fixture(variant):
    """tests/golden/vit.pt holds what the unmodified reference computed on these inputs (tests/make_golden_vit.py)"""
    import os
    from tests import pixelwise_oracle as pw
    golden = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vit.pt"), weights_only=False)["variants"][variant]
    pixelwise = variant.endswith("_pw")
    spec = vo.spec_from_card(vo.vit_card(pixelwise))
    orc = vo.OracleModel(spec, vo.synth_state_dict(spec, vo.SEED))
    orc.chunk_size = 2
    for name in ("img256", "img_resized", "vid"):
        c = golden["cases"][name]
        x = torch.rand(*c["shape"], generator=torch.Generator().manual_seed(c["gen_seed"]))
        with torch.no_grad():
            o = orc.detect(x, is_video=c["is_video"])["preds"]
        if pixelwise:
            assert torch.equal(pw.sample(o), c["maps_s"]), name
        else:
            assert torch.equal(o, c["logits"]), name
    x = torch.rand(*golden["cases"]["vid"]["shape"], generator=torch.Generator().manual_seed(2))
    for agg, a in golden["cases"]["extract"].items():
        with torch.no_grad():
            bits = orc.extract_message(x, aggregation=agg)
        assert torch.equal(bits[:, ::8, ::16, ::16] if pixelwise else bits, a["bits_s"]) and int(bits.sum()) == a["ones"], agg


def test_oracle_matches_restate():
    """tests/vit_oracle.py's pooled forward is restate.sam_extractor_forward (pinned to the reference by videoseal_0.0.pt), and its
    trunk is the same computation"""
    from oracle import restate
    spec = vo.spec_from_card(vo.vit_card(False, 128))
    sd = vo.synth_state_dict(spec)
    x = torch.rand(2, 3, 128, 128, generator=torch.Generator().manual_seed(0))
    t1, t2 = {}, {}
    a = vo.extractor_forward(sd, spec, x, t1)
    vo.trunk_forward(sd, spec, x, t2)
    assert torch.equal(a, restate.sam_extractor_forward(sd, spec, x))
    assert torch.equal(t1["blk11"], t2["blk11"])
