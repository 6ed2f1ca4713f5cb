"""SAM-ViT extractor cases for the tests (test infrastructure only).

The card is the videoseal_1.0 card (its BatchNorm/ReLU U-Net and args) with the videoseal_0.0 card's `sam_small` extractor block,
optionally made pixel-wise with upscale_stages [4, 2, 2] (the reference's `sam_small_pw`).  The trunk oracle is
oracle/restate.py's sam_extractor_forward, pinned to the reference through tests/golden/videoseal_0.0.pt; the pixel-wise decoder
stages are restate.upsample_block, as in tests/pixelwise_oracle.py.
"""
from __future__ import annotations

import argparse
import copy
import os
import sys
from typing import Dict, Optional

import torch
import torch.nn.functional as F
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate  # noqa: E402

D = "detector.pixel_decoder."
Q = "detector.image_encoder."
SEED = 1234


def vit_card(pixelwise: bool = False, img_size: Optional[int] = None, encoder: Optional[dict] = None, stages=(4, 2, 2)) -> dict:
    """videoseal_1.0 args and U-Net + the videoseal_0.0 extractor block (encoder keys overridden by `encoder`); a pixel-wise card
    has the upscale factors `stages`"""
    from tests.util import load_card
    card = load_card("videoseal_1.0")
    card["extractor"] = copy.deepcopy(load_card("videoseal_0.0")["extractor"])
    if encoder:
        card["extractor"]["params"]["encoder"].update(encoder)
    if pixelwise:
        card["extractor"]["model"] = "sam_small_pw"
        card["extractor"]["params"]["pixel_decoder"].update({"pixelwise": True, "upscale_stages": list(stages)})
    if img_size is not None:
        card["args"]["img_size_proc"] = img_size
    return card


def spec_from_card(card: dict) -> dict:
    spec = restate.spec_from_card(card)
    pd = card["extractor"]["params"].get("pixel_decoder", {})
    spec["pixel_decoder"] = {"pixelwise": bool(pd.get("pixelwise", False)),
                             "upscale_stages": [int(f) for f in pd.get("upscale_stages", [1])]}
    return spec


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, torch.Tensor]:
    """restate.synth_state_dict; a pixel-wise spec gets the staged decoder instead of the pooled one (generator seed + 1)"""
    sd = restate.synth_state_dict(spec, seed)
    if not spec["pixel_decoder"]["pixelwise"]:
        return sd
    for k in [k for k in sd if k.startswith(D)]:
        del sd[k]
    g = torch.Generator().manual_seed(seed + 1)
    c = int(spec["vit"]["out_chans"])
    for i, f in enumerate(spec["pixel_decoder"]["upscale_stages"]):
        sd[D + f"output_upscaling.{i}.upsample_block.2.weight"] = restate._kaiming_uniform((c // f, c, 3, 3), c * 9, g)
        sd[D + f"output_upscaling.{i}.upsample_block.3.weight"] = 1 + 0.1 * torch.randn(c // f, generator=g)
        sd[D + f"output_upscaling.{i}.upsample_block.3.bias"] = 0.1 * torch.randn(c // f, generator=g)
        c //= f
    no = 1 + spec["nbits"]
    sd[D + "linear.weight"] = restate._kaiming_uniform((no, c, 1, 1), c, g)
    sd[D + "linear.bias"] = restate._kaiming_uniform((no,), c, g)
    return sd


def trunk_forward(sd, spec, x: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    """restate's ViT trunk and neck: [B,3,S,S] -> [B, out_chans, S/16, S/16] (vit.py:111-143)"""
    v = spec["vit"]
    t = {} if taps is None else taps
    x = x * 2 - 1
    x = F.conv2d(x, sd[Q + "patch_embed.proj.weight"], sd[Q + "patch_embed.proj.bias"], stride=int(v["patch_size"])).permute(0, 2, 3, 1)
    x = x + sd[Q + "pos_embed"]
    glob = [int(i) for i in v["global_attn_indexes"]]
    for i in range(int(v["depth"])):
        x = restate._vit_block(sd, Q + f"blocks.{i}.", x, int(v["num_heads"]), 0 if i in glob else int(v["window_size"]),
                               bool(v.get("use_rel_pos", False)))
        t[f"blk{i}"] = x
    x = x.permute(0, 3, 1, 2).contiguous()
    x = F.conv2d(x, sd[Q + "neck.0.weight"], None)
    x = restate.layernorm_cf(x, sd[Q + "neck.1.weight"], sd[Q + "neck.1.bias"])
    x = F.conv2d(x, sd[Q + "neck.2.weight"], None, padding=1)
    x = restate.layernorm_cf(x, sd[Q + "neck.3.weight"], sd[Q + "neck.3.bias"])
    t["neck"] = x
    return x


def extractor_forward(sd, spec, x: torch.Tensor, taps: Optional[dict] = None) -> torch.Tensor:
    """pooled: restate.sam_extractor_forward; pixel-wise: the trunk, then pixel_decoder.py:61-83 stages -> [B,1+K,P,P]"""
    if not spec["pixel_decoder"]["pixelwise"]:
        return restate.sam_extractor_forward(sd, spec, x, taps)
    x = trunk_forward(sd, spec, x, taps)
    for i, f in enumerate(spec["pixel_decoder"]["upscale_stages"]):
        x = restate.upsample_block(sd, D + f"output_upscaling.{i}", x, "gelu", up_factor=f)
    return F.conv2d(x, sd[D + "linear.weight"], sd[D + "linear.bias"])


class OracleModel(restate.OracleModel):
    def detector(self, imgs_res, taps=None):
        return extractor_forward(self.sd, self.spec, imgs_res, taps)


def card_on_disk(card: dict, sd: dict, tag: str):
    """<tmp>/<tag>.yaml + .pth: a model card that spells the encoder out, as cards/videoseal_0.0.yaml does"""
    from tests.util import tmpdir
    d = tmpdir()
    card = copy.deepcopy(card)
    torch.save({"model": sd}, d / f"{tag}.pth")
    card["checkpoint_path"] = str(d / f"{tag}.pth")
    card["args"]["attenuation_config"] = os.path.join(ROOT, "videoseal_b200", "configs", "attenuation.yaml")
    path = d / f"{tag}.yaml"
    yaml.safe_dump(card, open(path, "w"))
    return path


def training_checkpoint(card: dict, sd: dict, tag: str):
    """<tmp>/<tag>.pth training checkpoint whose args.extractor_config names a YAML in the tmpdir defining the preset"""
    from tests.util import tmpdir
    d = tmpdir()
    preset = card["extractor"]["model"]
    ext_yaml = d / f"{tag}_extractor.yaml"
    yaml.safe_dump({"model": preset, preset: card["extractor"]["params"]}, open(ext_yaml, "w"))
    args = argparse.Namespace(**card["args"], embedder_model=card["embedder"]["model"], extractor_model=preset,
                              extractor_config=str(ext_yaml))
    args.attenuation_config = os.path.join(ROOT, "videoseal_b200", "configs", "attenuation.yaml")
    path = d / f"{tag}.pth"
    torch.save({"model": sd, "args": args}, path)
    return path


def model_pair(pixelwise: bool = False, img_size: Optional[int] = None, encoder: Optional[dict] = None, device: str = "cuda:0",
               seed: int = SEED, via_checkpoint: bool = False):
    """(product Videoseal on `device`, OracleModel, spec) sharing one synthetic checkpoint"""
    import videoseal_b200
    import videoseal_b200.utils.cfg
    card = vit_card(pixelwise, img_size, encoder)
    spec = spec_from_card(card)
    sd = synth_state_dict(spec, seed)
    tag = f"vit_{'pw' if pixelwise else 'pool'}_{spec['img_size']}_{seed}_{abs(hash(str(encoder))) % 10**8}"
    if via_checkpoint:
        model = videoseal_b200.utils.cfg.setup_model_from_checkpoint(str(training_checkpoint(card, sd, tag + "_train")))
    else:
        model = videoseal_b200.load(card_on_disk(card, sd, tag))
    model = model.eval()
    if device is not None:
        model = model.to(device)
    return model, OracleModel(spec, sd), spec
