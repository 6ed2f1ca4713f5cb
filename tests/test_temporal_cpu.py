"""Temporal (conv3d) U-Net embedders without a GPU: the torch restatement of tests/temporal_oracle.py against the reference's outputs in
tests/golden/temporal.pt, and the load-time rules (a dry run of the native library's descriptor checks)."""
import copy
import os

import pytest
import torch

from oracle import restate
from tests import temporal_oracle as to

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "temporal.pt")


@pytest.mark.parametrize("preset", ["unet_small2_yuv_quant_conv3d", "unet_small2_quant_conv3d"])
def test_oracle_equals_reference_golden(preset):
    from tests.make_golden_temporal import cases
    gold = torch.load(GOLDEN, weights_only=False)["presets"][preset]
    spec = to.spec_from_card(to.preset_card(preset))
    orc = to.TemporalOracle(spec, to.synth_state_dict(spec, to.SEED))
    for name, (x, m, is_video, chunk, step) in cases(spec["nbits"]).items():
        g = gold["cases"][name]
        orc.chunk_size, orc.step_size = chunk, step
        with torch.no_grad():
            o = orc.embed(x, m, is_video=is_video)
        assert (to.sample(o["imgs_w"]) - g["imgs_w_s"]).abs().max().item() <= 1e-5, name
        if g["preds_w_s"] is not None:
            assert (to.sample(o["preds_w"]) - g["preds_w_s"]).abs().max().item() <= 1e-5, name


def test_frames_of_different_calls_never_interact():
    """one embedder call per group: the output of a group depends on its own frames only, and on their order"""
    spec = to.spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d", img_size=128))
    orc = to.TemporalOracle(spec, to.synth_state_dict(spec, to.SEED))
    x = torch.rand(4, 3, 128, 128, generator=torch.Generator().manual_seed(0))
    m = torch.randint(0, 2, (4, spec["nbits"]), generator=torch.Generator().manual_seed(1))
    with torch.no_grad():
        whole = orc.embedder(x, m)
        a, b = orc.embedder(x[:2], m[:2]), orc.embedder(x[2:], m[2:])
        swapped = orc.embedder(x[[1, 0]], m[[1, 0]])
    assert (whole[:2] - a).abs().max().item() > 1e-4             # frame 1 saw frame 2 in the single call
    assert (swapped[[1, 0]] - a).abs().max().item() > 1e-4       # order within a call matters


@pytest.mark.parametrize("preset", to.PRESETS)
def test_presets_load_from_training_checkpoints(built_lib, preset):
    import videoseal_b200.utils.cfg as vcfg
    card = to.preset_card(preset)
    spec = to.spec_from_card(card)
    model = vcfg.setup_model_from_checkpoint(to.training_checkpoint(card, to.synth_state_dict(spec, to.SEED), preset))
    assert model.temporal and model.spec["unet"]["temporal"]
    assert model.state_dict()[to.TEMPORAL_KEY_3D].dim() == 5                  # 5-D tensors are kept


INFLATE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "temporal_inflate.pt")


def _script_output(ext: str):
    """(card naming the 2-D presets, the reference's inflate script output restated on its seeded synthetic checkpoint)"""
    card = to.preset_card("unet_small2_yuv_quant") if ext == "convnext_tiny" else to.sam_card("unet_small2_yuv_quant")
    sd = restate.synth_state_dict(restate.spec_from_card(card), to.SEED)
    return card, to.inflate_script(sd, ext, torch.load(INFLATE, weights_only=False)[ext])


def _load(card, sd, tag):
    from videoseal_b200 import cfg
    path = to.tmpdir() / f"{tag}.pth"
    torch.save({"model": sd}, path)
    return cfg.setup_model(card, str(path))


@pytest.mark.parametrize("ext", ["convnext_tiny", "sam_small"])
def test_inflate_script_output_loads(built_lib, ext):
    """inflate_model_to_temporal.py keeps `args` (naming the 2-D presets), makes the U-Net temporal and adds the extractor's temporal
    parts at their identity: the U-Net loads temporal, the extractor as the 2-D extractor it still computes"""
    card, sd = _script_output(ext)
    assert sd[to.TEMPORAL_KEY_3D].shape[2:] == (3, 3, 3) and sd[to.TEMPORAL_KEY_3D][:, :, 0].abs().max() == 0
    model = _load(card, sd, f"inflated_{ext}")
    assert model.temporal
    kept = model.state_dict()
    assert not [k for k in kept if "temp_" in k or "temporal" in k]
    if ext == "convnext_tiny":
        assert "detector.convnext.downsample_layers.1.1.conv.weight" in sd
        for i in (1, 2, 3):
            assert torch.equal(kept[f"detector.convnext.downsample_layers.{i}.1.weight"],
                               sd[f"detector.convnext.downsample_layers.{i}.1.conv.weight"])


def test_inflated_unet_loads_through_a_training_checkpoint(built_lib):
    import videoseal_b200.utils.cfg as vcfg
    card, sd = _script_output("convnext_tiny")
    model = vcfg.setup_model_from_checkpoint(to.training_checkpoint(card, sd, "inflated_cpu", embedder_model="unet_small2_yuv_quant"))
    assert model.temporal


@pytest.mark.parametrize("ext,key,how", [
    ("convnext_tiny", "detector.convnext.stages.2.4.temp_block.mlp.lin2.bias", "nonzero"),
    ("convnext_tiny", "detector.convnext.stages.0.0.temp_block.mlp.lin2.weight", "missing"),
    ("convnext_tiny", "detector.convnext.downsample_layers.2.1.temp_conv.weight", "nonzero"),
    ("convnext_tiny", "detector.convnext.downsample_layers.3.1.temp_conv.weight", "missing"),
    ("sam_small", "detector.image_encoder.temp_blocks.11.mlp.lin2.weight", "nonzero"),
    ("sam_small", "detector.image_encoder.pos_embed_temporal", "nonzero"),
])
def test_trained_temporal_extractor_raises_at_load(built_lib, ext, key, how):
    """temporal extractor parts that are no longer the inflated identity change what the extractor computes: not implemented"""
    card, sd = _script_output(ext)
    assert key in sd
    if how == "missing":
        del sd[key]
    else:
        sd[key] = sd[key] + 1e-3
    with pytest.raises(NotImplementedError, match="temporal extractor"):
        _load(card, sd, f"trained_{ext}")


def _card_with(unet_over: dict) -> dict:
    card = to.preset_card("unet_small2_quant_conv3d")
    card = copy.deepcopy(card)
    card["embedder"]["params"]["unet"].update(unet_over)
    return card


@pytest.mark.parametrize("over", [{"conv_layer": "conv2p1d"}, {"activation": "silu", "normalization": "rms"},
                                  {"activation": "silu"}, {"normalization": "rms"}])
def test_unimplemented_temporal_variants_raise_at_load(built_lib, over):
    from videoseal_b200.cfg import spec_from_card
    with pytest.raises(NotImplementedError):
        spec_from_card(_card_with(over))


def test_2d_spec_is_not_temporal(built_lib):
    from videoseal_b200.cfg import spec_from_card
    spec = spec_from_card(to.preset_card("unet_small2_yuv_quant"))
    assert spec["unet"]["temporal"] is False
    assert spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d"))["unet"]["temporal"] is True


def test_group_length_rules_need_no_gpu(built_lib):
    """image mode with more than 64 images, or chunk_size > 64, is refused before any device work"""
    from videoseal_b200.model import Videoseal
    from videoseal_b200.cfg import spec_from_card
    m = Videoseal(spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d")))
    assert m._chunk_keys(False, 64) == 64 and m._chunk_keys(True, 1000) == m.chunk_size
    with pytest.raises(NotImplementedError, match="64"):
        m._chunk_keys(False, 65)
    m.chunk_size = 65
    with pytest.raises(NotImplementedError, match="64"):
        m._chunk_keys(True, 10)
    m2 = Videoseal(spec_from_card(to.preset_card("unet_small2_yuv_quant")))
    m2.chunk_size = 100
    assert m2._chunk_keys(True, 10) == 100 and m2._chunk_keys(False, 100) == 100   # 2-D: chunk_size as before


def test_shards_cut_on_chunk_boundaries(built_lib):
    from videoseal_b200.cfg import spec_from_card
    from videoseal_b200.dist import shard_bounds, shard_unit
    from videoseal_b200.model import Videoseal
    m = Videoseal(spec_from_card(to.preset_card("unet_small2_yuv_quant_conv3d")))
    m.chunk_size, m.step_size = 8, 4
    assert shard_unit(m) == 32
    assert all(s % 32 == 0 for s, _ in shard_bounds(200, 3, shard_unit(m)))
    m2 = Videoseal(spec_from_card(to.preset_card("unet_small2_yuv_quant")))
    m2.chunk_size, m2.step_size = 8, 4
    assert shard_unit(m2) == 4
