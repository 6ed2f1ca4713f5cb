"""unet_tiny_yuv_quant without a GPU: preset resolution from a training checkpoint, the CPU oracle against the reference's
fixture, and the load-time rules for U-Net widths and processing sizes."""
import copy
import os

import pytest
import torch

from oracle import restate
from tests import unet_tiny as ut
from videoseal_b200 import cfg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "unet_tiny.pt"), weights_only=False)


def test_training_checkpoint_naming_the_preset_resolves(built_lib):
    card = ut.tiny_card()
    spec = restate.spec_from_card(card)
    path = ut.training_checkpoint(card, restate.synth_state_dict(spec, ut.SEED), "cpu_resolve")
    c = cfg.get_config_from_checkpoint(path)
    assert c["embedder"]["model"] == "unet_tiny_yuv_quant" and c["extractor"]["model"] == "convnext_tiny"
    s = cfg.spec_from_card(c)
    assert s["unet"]["z"] == [8, 8, 16, 32, 64] and s["unet"]["num_blocks"] == 4
    assert s["unet"]["in_channels"] == 1 and s["unet"]["out_channels"] == 1 and s["yuv"] is True
    assert s["hidden"] == 256 and s["nbits"] == 256 and s["img_size"] == 256


@pytest.mark.parametrize("case", sorted(GOLDEN["cases"]))
def test_oracle_matches_reference_fixture(case):
    from tests.make_golden_unet_tiny import cases
    spec = restate.spec_from_card(ut.tiny_card())
    orc = restate.OracleModel(spec, restate.synth_state_dict(spec, GOLDEN["seed"]))
    x, m, is_video, mode, chunk = cases(spec["nbits"])[case]
    orc.chunk_size, orc.video_mode = chunk, mode
    with torch.no_grad():
        o = orc.embed(x, m, is_video=is_video)
    g = GOLDEN["cases"][case]
    assert (ut.sample(o["imgs_w"]) - g["imgs_w_s"]).abs().max().item() <= 1e-6
    if g["preds_w_s"] is not None:
        assert (ut.sample(o["preds_w"]) - g["preds_w_s"]).abs().max().item() <= 1e-6


@pytest.mark.parametrize("mults,what", [([1, 1, 3, 4, 8], "width 24"), ([1, 2, 4, 8, 1], "width 8"), ([2, 1, 2, 4, 8], "width 8"),
                                        ([1, 1, 1, 1, 1], "width 8")])
def test_unimplemented_widths_are_rejected_at_load(built_lib, mults, what):
    card = ut.tiny_card()
    card["embedder"]["params"]["unet"]["z_channels_mults"] = mults
    with pytest.raises(NotImplementedError, match=what):
        cfg.spec_from_card(card)


@pytest.mark.parametrize("size", [128, 896, 1024])
def test_unimplemented_processing_sizes_are_rejected_at_load(built_lib, size):
    with pytest.raises(NotImplementedError, match=f"img_size={size}"):
        cfg.spec_from_card(ut.tiny_card(img_size=size))


def test_img_size_setter_applies_the_same_rules(built_lib):
    from videoseal_b200.model import Videoseal
    m = Videoseal(cfg.spec_from_card(ut.tiny_card()))
    for bad in (128, 1024):
        with pytest.raises(NotImplementedError):
            m.img_size = bad
    assert m.img_size == 256
    m.img_size = 512
    assert m.img_size == 512


def test_four_level_cards_keep_their_sizes(built_lib):
    """the bottleneck rule leaves the 4-level cards at S >= 128 as they were"""
    from tests.util import load_card
    for name in ("videoseal_1.0", "pixelseal", "chunkyseal"):
        card = copy.deepcopy(load_card(name))
        for S in (128, 256, 1024):
            card["args"]["img_size_proc"] = S
            assert cfg.spec_from_card(card)["img_size"] == S
