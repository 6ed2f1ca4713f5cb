"""The unet_tiny_yuv_quant embedder (8-channel outer levels, five levels) on the videoseal_1.0 card: card, spec and a
(product model, CPU oracle) pair loaded from a training checkpoint that names the preset (utils/cfg.py:50-85)."""
import argparse
import copy
import os
from typing import Optional

import torch
import yaml

from oracle import restate
from tests.util import load_card, tmpdir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESET = "unet_tiny_yuv_quant"
SEED = 1234


def tiny_card(img_size: Optional[int] = None) -> dict:
    """videoseal_1.0 with its embedder replaced by the package's unet_tiny_yuv_quant preset"""
    card = copy.deepcopy(load_card("videoseal_1.0"))
    presets = yaml.safe_load(open(os.path.join(ROOT, "videoseal_b200", "configs", "embedder.yaml")))
    card["embedder"] = {"model": PRESET, "params": copy.deepcopy(presets[PRESET])}
    if img_size is not None:
        card["args"]["img_size_proc"] = img_size
    return card


def training_checkpoint(card: dict, sd: dict, tag: str) -> str:
    """a raw training checkpoint whose args name the embedder / extractor presets instead of carrying their parameters"""
    args = argparse.Namespace(**card["args"], embedder_model=card["embedder"]["model"], extractor_model=card["extractor"]["model"])
    args.attenuation_config = os.path.join(ROOT, "videoseal_b200", "configs", "attenuation.yaml")
    path = tmpdir() / f"train_{tag}.pth"
    torch.save({"model": sd, "args": args}, path)
    return str(path)


def model_pair(device: str = "cuda:0", seed: int = SEED, img_size: Optional[int] = None):
    """(product Videoseal, OracleModel on CPU, oracle spec) sharing one synthetic checkpoint"""
    import videoseal_b200.utils.cfg
    card = tiny_card(img_size)
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, seed)
    path = training_checkpoint(card, sd, f"{PRESET}_{seed}_{spec['img_size']}")
    model = videoseal_b200.utils.cfg.setup_model_from_checkpoint(path).eval()
    if device is not None:
        model = model.to(device)
    return model, restate.OracleModel(spec, sd), spec


def sample(t: torch.Tensor) -> torch.Tensor:
    """strided sample of a [F, C, H, W] tensor stored in the fixture"""
    return t[:, :, ::7, ::5].clone()
