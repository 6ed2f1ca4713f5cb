"""The HiDDeN embedder and extractor restated in torch (fp32, CPU): cards for the `hidden` / `hidden_orig` presets alone and paired
with the other families, the spec, a seeded synthetic checkpoint in the reference's key layout, and the forward passes with taps.

Reference: modules/hidden.py (ConvBNRelu = Conv2d 3x3 pad 1 + BatchNorm2d / GroupNorm(8, C) + ReLU / GELU; HiddenEncoder,
HiddenDecoder), models/embedder.py HiddenEmbedder (msgs = 2 m - 1, imgs = 2 x - 1), models/extractor.py HiddenExtractor
(imgs = 2 x - 1), modules/common.py get_normalization / get_activation.  The rest of the pipeline (resize, blend, video chunks) is
oracle/restate.OracleModel's: HiddenOracle only replaces its two leaves."""
import copy
import os
from typing import Dict, Optional

import torch
import torch.nn.functional as F
import yaml
from torch import Tensor

from oracle import restate
from tests.util import load_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 4321
PRESETS = ("hidden", "hidden_orig")
# (embedder, extractor) pairings: "unet" / "convnext" are videoseal_1.0's networks, "sam" is videoseal_0.0's SAM-ViT extractor
PAIRINGS = [("hidden", "hidden"), ("hidden_orig", "hidden_orig"), ("hidden", "convnext"), ("hidden_orig", "sam"),
            ("unet", "hidden"), ("unet", "hidden_orig")]


def _presets(kind: str) -> dict:
    return yaml.safe_load(open(os.path.join(ROOT, "videoseal_b200", "configs", f"{kind}.yaml")))


def card(emb: str, ext: str, img_size: Optional[int] = None, nbits: Optional[int] = None) -> dict:
    """videoseal_1.0 with its embedder and / or extractor replaced: a HiDDeN preset of the package's configs, "unet" / "convnext"
    (the card's own) or "sam" (videoseal_0.0's extractor)"""
    c = copy.deepcopy(load_card("videoseal_1.0"))
    if emb != "unet":
        c["embedder"] = {"model": emb, "params": copy.deepcopy(_presets("embedder")[emb])}
    if ext == "sam":
        c["extractor"] = copy.deepcopy(load_card("videoseal_0.0")["extractor"])
    elif ext != "convnext":
        c["extractor"] = {"model": ext, "params": copy.deepcopy(_presets("extractor")[ext])}
    if img_size is not None:
        c["args"]["img_size_proc"] = img_size
    if nbits is not None:
        c["args"]["nbits"] = nbits
    return c


def _hidden_params(p: dict, embedder: bool) -> dict:
    h = {"z_channels": int(p["z_channels"]), "num_blocks": int(p["num_blocks"]), "in_channels": int(p.get("in_channels", 3)),
         "normalization": str(p["normalization"]), "activation": str(p["activation"])}
    if embedder:
        h["out_channels"] = int(p.get("out_channels", 3))
        h["last_tanh"] = bool(p.get("last_tanh", True))
    return h


def spec_from_card(c: dict) -> dict:
    """restate.spec_from_card, with `hidden_encoder` / `hidden_decoder` for the HiDDeN sides (the U-Net / ConvNeXt entries of such
    a side are those of videoseal_1.0 and unused)"""
    base = copy.deepcopy(c)
    v1 = load_card("videoseal_1.0")
    emb_h = c["embedder"]["model"].startswith("hidden")
    ext_h = c["extractor"]["model"].startswith("hidden")
    if emb_h:
        base["embedder"] = copy.deepcopy(v1["embedder"])
    if ext_h:
        base["extractor"] = copy.deepcopy(v1["extractor"])
    spec = restate.spec_from_card(base)
    if emb_h:
        spec["hidden_encoder"] = _hidden_params(c["embedder"]["params"], True)
        spec["yuv"] = False
    if ext_h:
        spec["hidden_decoder"] = _hidden_params(c["extractor"]["params"], False)
    return spec


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, Tensor]:
    """restate.synth_state_dict with the HiDDeN sides in the reference's key layout: conv weights and biases U(-1/sqrt(fan_in), ..)
    as nn.Conv2d initialises them, BatchNorm running statistics and affines and GroupNorm affines randomised"""
    base = dict(spec)
    if base.get("ext_kind") == "hidden" or "hidden_decoder" in spec:
        base["ext_kind"] = "convnext"
    sd = restate.synth_state_dict(base, seed)
    if "hidden_encoder" in spec:
        sd = {k: v for k, v in sd.items() if not k.startswith("embedder.")}
    if "hidden_decoder" in spec:
        sd = {k: v for k, v in sd.items() if not k.startswith("detector.")}
    g = torch.Generator().manual_seed(seed + 7)

    def conv(key, cout, cin, k):
        b = 1.0 / (cin * k * k) ** 0.5
        sd[key + ".weight"] = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) * b
        sd[key + ".bias"] = (torch.rand(cout, generator=g) * 2 - 1) * b

    def block(key, cin, cout, norm):
        conv(key + ".layers.0", cout, cin, 3)
        sd[key + ".layers.1.weight"] = 1 + 0.1 * torch.randn(cout, generator=g)
        sd[key + ".layers.1.bias"] = 0.1 * torch.randn(cout, generator=g)
        if norm.startswith("batch"):
            sd[key + ".layers.1.running_mean"] = 0.1 * torch.randn(cout, generator=g)
            sd[key + ".layers.1.running_var"] = 0.5 + torch.rand(cout, generator=g)
            sd[key + ".layers.1.num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    K = spec["nbits"]
    if "hidden_encoder" in spec:
        h = spec["hidden_encoder"]
        z, P = h["z_channels"], "embedder.hidden_encoder."
        for i in range(h["num_blocks"]):
            block(P + f"conv_bns.{i}", h["in_channels"] if i == 0 else z, z, h["normalization"])
        block(P + "after_concat_layer", z + h["in_channels"] + K, z, h["normalization"])
        conv(P + "final_layer", h["out_channels"], z, 1)
    if "hidden_decoder" in spec:
        h = spec["hidden_decoder"]
        z, P = h["z_channels"], "detector.hidden_decoder."
        for i in range(h["num_blocks"] + 1):
            block(P + f"layers.{i}", h["in_channels"] if i == 0 else z, z, h["normalization"])
        b = 1.0 / z ** 0.5
        sd[P + "linear.weight"] = (torch.rand(1 + K, z, generator=g) * 2 - 1) * b
        sd[P + "linear.bias"] = (torch.rand(1 + K, generator=g) * 2 - 1) * b
    return sd


def norm(sd, key: str, kind: str, x: Tensor) -> Tensor:
    """BatchNorm2d (eval) or GroupNorm(8, C), eps 1e-5 (modules/common.py get_normalization)"""
    if kind.startswith("batch"):
        return F.batch_norm(x, sd[key + ".running_mean"], sd[key + ".running_var"], sd[key + ".weight"], sd[key + ".bias"],
                            False, 0.0, 1e-5)
    return F.group_norm(x, 8, sd[key + ".weight"], sd[key + ".bias"], 1e-5)


def act(kind: str, x: Tensor) -> Tensor:
    return F.relu(x) if kind == "relu" else F.gelu(x)


def conv_bn_relu(sd, key: str, h: dict, x: Tensor, taps: Optional[dict] = None, name: str = "") -> Tensor:
    y = F.conv2d(x, sd[key + ".layers.0.weight"], sd[key + ".layers.0.bias"], padding=1)
    if taps is not None:
        taps[name + ".pre"] = y
    return act(h["activation"], norm(sd, key + ".layers.1", h["normalization"], y))


def encoder_forward(sd, spec: dict, imgs: Tensor, msgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """HiddenEmbedder.forward: imgs [B,3,S,S] in [0,1], msgs [B,K] in {0,1} -> delta [B,3,S,S]"""
    h, P = spec["hidden_encoder"], "embedder.hidden_encoder."
    m = 2 * msgs.float() - 1
    x = 2 * imgs - 1
    enc = x
    for i in range(h["num_blocks"]):
        enc = conv_bn_relu(sd, P + f"conv_bns.{i}", h, enc, taps, f"henc.{i}")
        if taps is not None:
            taps[f"henc.{i}"] = enc
    planes = m[:, :, None, None].expand(-1, -1, x.shape[-2], x.shape[-1])
    cat = torch.cat([planes, enc, x], dim=1)
    y = conv_bn_relu(sd, P + "after_concat_layer", h, cat, taps, "henc.cat")
    y = F.conv2d(y, sd[P + "final_layer.weight"], sd[P + "final_layer.bias"])
    return torch.tanh(y) if h["last_tanh"] else y


def decoder_forward(sd, spec: dict, imgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """HiddenExtractor.forward: imgs [B,3,S,S] in [0,1] -> logits [B,1+K]"""
    h, P = spec["hidden_decoder"], "detector.hidden_decoder."
    x = 2 * imgs - 1
    for i in range(h["num_blocks"] + 1):
        x = conv_bn_relu(sd, P + f"layers.{i}", h, x, taps, f"hdec.{i}")
        if taps is not None:
            taps[f"hdec.{i}"] = x
    pooled = x.mean(dim=[-2, -1])
    if taps is not None:
        taps["head_pooled"] = pooled
    return F.linear(pooled, sd[P + "linear.weight"], sd[P + "linear.bias"])


class HiddenOracle(restate.OracleModel):
    """restate.OracleModel with HiDDeN leaves where the spec has them"""

    def embedder(self, imgs_res: Tensor, msgs: Tensor, taps=None) -> Tensor:
        if "hidden_encoder" in self.spec:
            return encoder_forward(self.sd, self.spec, imgs_res, msgs, taps)
        return super().embedder(imgs_res, msgs, taps)

    def detector(self, imgs_res: Tensor, taps=None) -> Tensor:
        if "hidden_decoder" in self.spec:
            return decoder_forward(self.sd, self.spec, imgs_res, taps)
        return super().detector(imgs_res, taps)


def sample(t: Tensor, n: int = 4096) -> Tensor:
    """a fixed strided sample of a tensor's elements (the fixture keeps samples, not whole outputs)"""
    flat = t.reshape(-1)
    step = max(1, flat.numel() // n)
    return flat[::step][:n].clone()
