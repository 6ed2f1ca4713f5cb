"""CPU oracle of the pixel-wise ConvNeXt extractors (test infrastructure only).

Extends oracle/restate.py with the staged pixel decoder of modules/pixel_decoder.py:44-83 (pixelwise=True): every stage is
modules/common.py:45-52 (bilinear x f, align_corners=False -> ReflectionPad2d(1) -> 3x3 valid conv without bias ->
channels-first LayerNorm eps 1e-6 -> GELU) with widths C, C // f, ..., then a 1x1 Conv2d to 1 + nbits maps.  The trunk is
restate's.  tests/make_golden_pixelwise.py pins this restatement against the unmodified reference (max |diff| = 0) and writes
tests/golden/pixelwise.pt.
"""
from __future__ import annotations

import copy
import os
import sys
from typing import Dict, Optional

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate  # noqa: E402

PRESETS = ("convnext_tiny_pw", "convnext_base_pw")
D = "detector.pixel_decoder."


def preset_card(preset: str, base_card: dict) -> dict:
    """`base_card` (the videoseal_1.0 card) with its extractor replaced by a preset of the package's configs/extractor.yaml."""
    import yaml
    ext = yaml.safe_load(open(os.path.join(ROOT, "videoseal_b200", "configs", "extractor.yaml")))
    card = copy.deepcopy(base_card)
    card["extractor"] = {"model": preset, "params": copy.deepcopy(ext[preset])}
    return card


def spec_from_card(card: dict) -> dict:
    spec = restate.spec_from_card(card)
    pd = card["extractor"]["params"].get("pixel_decoder", {})
    spec["pixel_decoder"] = {"pixelwise": bool(pd.get("pixelwise", False)),
                             "upscale_stages": [int(f) for f in pd.get("upscale_stages", [1])]}
    return spec


def synth_state_dict(spec: dict, seed: int = 0) -> Dict[str, torch.Tensor]:
    """restate.synth_state_dict with the pooled decoder replaced by the staged one (its own generator, seed + 1)."""
    sd = restate.synth_state_dict(spec, seed)
    for k in [k for k in sd if k.startswith(D)]:
        del sd[k]
    g = torch.Generator().manual_seed(seed + 1)
    c = spec["convnext"]["dims"][-1]
    for i, f in enumerate(spec["pixel_decoder"]["upscale_stages"]):
        sd[D + f"output_upscaling.{i}.upsample_block.2.weight"] = restate._kaiming_uniform((c // f, c, 3, 3), c * 9, g)
        sd[D + f"output_upscaling.{i}.upsample_block.3.weight"] = 1 + 0.1 * torch.randn(c // f, generator=g)
        sd[D + f"output_upscaling.{i}.upsample_block.3.bias"] = 0.1 * torch.randn(c // f, generator=g)
        c //= f
    no = 1 + spec["nbits"]
    sd[D + "linear.weight"] = restate._kaiming_uniform((no, c, 1, 1), c, g)
    sd[D + "linear.bias"] = restate._kaiming_uniform((no,), c, g)
    return sd


def extractor_forward(sd, spec, x: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    """models/extractor.py:154-167 + modules/pixel_decoder.py:61-83 with pixelwise=True: [B,3,S,S] -> [B,1+K,P,P].
    The trunk is restate.convnext_extractor_forward's, read from its `stage3` tap; its pooled head runs on zero weights that stand
    in for the pixel-wise decoder's keys (a 3x3 conv on the last map, discarded)."""
    c = spec["convnext"]["dims"][-1]
    z = dict(dtype=x.dtype)
    pooled = {D + "output_upscaling.0.upsample_block.2.weight": torch.zeros(c, c, 3, 3, **z),
              D + "output_upscaling.0.upsample_block.3.weight": torch.ones(c, **z),
              D + "output_upscaling.0.upsample_block.3.bias": torch.zeros(c, **z),
              D + "linear.weight": torch.zeros(1, c, **z), D + "linear.bias": torch.zeros(1, **z)}
    t = {} if taps is None else taps
    restate.convnext_extractor_forward({**sd, **pooled}, spec, x, t)
    x = t["stage3"]
    for i, f in enumerate(spec["pixel_decoder"]["upscale_stages"]):
        x = restate.upsample_block(sd, D + f"output_upscaling.{i}", x, "gelu", up_factor=f)
        t[f"pd{i}"] = x
    return F.conv2d(x, sd[D + "linear.weight"], sd[D + "linear.bias"])


class OracleModel(restate.OracleModel):
    def detector(self, imgs_res, taps=None):
        return extractor_forward(self.sd, self.spec, imgs_res, taps)


def sample(t: torch.Tensor, cstride: int = 8, stride: int = 16) -> torch.Tensor:
    """strided sample of [F, 1+K, P, P] maps (every cstride-th channel, every stride-th pixel)"""
    return t[:, ::cstride, ::stride, ::stride].contiguous().clone()


def stats(t: torch.Tensor) -> dict:
    t = t.double()
    return {"mean": t.mean().item(), "absmean": t.abs().mean().item(), "std": t.std().item(),
            "min": t.min().item(), "max": t.max().item()}


def model_pair(preset: str, device: str = "cuda:0", seed: int = 1234, nbits: Optional[int] = None, img_size: Optional[int] = None):
    """(product Videoseal loaded from a training checkpoint naming `preset`, oracle, spec): the checkpoint's args name the
    embedder / extractor presets (utils/cfg.py:50-85), so this also exercises the preset lookup."""
    import argparse
    import videoseal_b200.utils.cfg
    from tests.util import load_card, tmpdir
    card = preset_card(preset, load_card("videoseal_1.0"))
    if nbits is not None:
        card["args"]["nbits"] = nbits
    if img_size is not None:
        card["args"]["img_size_proc"] = img_size
    spec = spec_from_card(card)
    sd = synth_state_dict(spec, seed)
    args = argparse.Namespace(**card["args"], embedder_model=card["embedder"]["model"], extractor_model=preset)
    args.attenuation_config = os.path.join(ROOT, "videoseal_b200", "configs", "attenuation.yaml")
    path = tmpdir() / f"train_{preset}_{spec['nbits']}_{spec['img_size']}.pth"
    torch.save({"model": sd, "args": args}, path)
    model = videoseal_b200.utils.cfg.setup_model_from_checkpoint(str(path)).eval()
    if device is not None:
        model = model.to(device)
    return model, OracleModel(spec, sd), spec
