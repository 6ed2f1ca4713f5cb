"""The DVMark embedder restated in torch (float64 or fp32, CPU or GPU): cards with the `dvmark` embedder preset paired with each
extractor family, the spec, a seeded synthetic checkpoint in the reference's key layout, and the forward pass with taps.

Reference: modules/dvmark.py DVMarkEncoder (lines 10-83) inside models/embedder.py DVMarkEmbedder (x = 2 imgs - 1; the messages
stay 0 / 1), built by build_embedder 'dvmark' with yuv False.  Its forward takes the B key frames of one call as ONE clip
[1, 3, T = B, H, W].  The rest of the pipeline (resize, video chunks, JND, blend) is oracle/restate.OracleModel's: EncOracle only
replaces the embedder (and takes the DVMark or HiDDeN detector where the card has one)."""
import copy
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from tests import dvmark_oracle as dv
from tests import hidden_oracle as ho

SEED = 6262
EXTRACTORS = ("dvmark", "convnext", "hidden", "sam")
P = "embedder.unet."


def card(ext: str = "dvmark", img_size: Optional[int] = None, nbits: Optional[int] = None) -> dict:
    """videoseal_1.0 with the `dvmark` embedder preset of the package's configs and the extractor `ext` ("dvmark" / "hidden": the
    package's presets, "convnext": the card's own, "sam": videoseal_0.0's)"""
    c = dv.card("hidden", img_size, nbits) if ext == "dvmark" else ho.card("hidden", ext, img_size, nbits)
    c["embedder"] = {"model": "dvmark", "params": copy.deepcopy(ho._presets("embedder")["dvmark"]["params"])}
    return c


def _base_card(c: dict) -> dict:
    """the card with a HiDDeN embedder in place of DVMark: the specs and checkpoints of the other oracles build the extractor side"""
    base = copy.deepcopy(c)
    base["embedder"] = {"model": "hidden", "params": copy.deepcopy(ho._presets("embedder")["hidden"])}
    return base


def _ext_spec(base: dict) -> dict:
    if base["extractor"]["model"] == "dvmark":
        return dv.spec_from_card(base)
    return ho.spec_from_card(base)


def spec_from_card(c: dict) -> dict:
    """the extractor side's oracle spec, with `dvmark_encoder` for the embedder and yuv False"""
    spec = _ext_spec(_base_card(c))
    del spec["hidden_encoder"]
    spec["dvmark_encoder"] = {"nbits": spec["nbits"]}
    spec["yuv"] = False
    return spec


# (key, cin, cout, time taps) of every Conv3d, K = nbits
def layers(K: int):
    return [("transform_layer.0", 3, 64, 1), ("transform_layer.2", 64, 64, 1), ("transform_layer.4", 64, 64, 1),
            ("transform_layer.6", 64, 64, 3),
            ("emb_layer1.0", 64 + K, 256, 3), ("emb_layer1.2", 256, 128, 3), ("emb_layer1.4", 128, 128, 3),
            ("emb_layer2.0", 128 + K, 512, 3), ("emb_layer2.2", 512, 256, 3), ("emb_layer2.4", 256, 256, 3),
            ("emb_layer3.0", 384, 256, 3), ("emb_layer3.2", 256, 128, 3), ("emb_layer3.4", 128, 3, 3)]


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, Tensor]:
    """the extractor side's synthetic checkpoint, with DVMarkEncoder's Conv3d layers under embedder.unet.*.  Weights are
    U(-a, a) with a = sqrt(6 / fan_in) (variance 2 / fan_in: ReLU layers keep the activations' scale, so the delta neither
    vanishes nor saturates the tanh), the output layer's halved; biases U(-0.05, 0.05)"""
    base = {k: v for k, v in spec.items() if k != "dvmark_encoder"}
    base["hidden_encoder"] = ho._hidden_params(ho._presets("embedder")["hidden"], True)
    gen = dv.synth_state_dict if "dvmark_decoder" in spec else ho.synth_state_dict
    sd = {k: v for k, v in gen(base, seed).items() if not k.startswith("embedder.")}
    g = torch.Generator().manual_seed(seed + 13)
    for key, cin, cout, kt in layers(spec["nbits"]):
        fan_in = cin * kt * 9
        a = (6.0 / fan_in) ** 0.5 * (0.5 if key == "emb_layer3.4" else 1.0)
        sd[P + key + ".weight"] = (torch.rand(cout, cin, kt, 3, 3, generator=g) * 2 - 1) * a
        sd[P + key + ".bias"] = (torch.rand(cout, generator=g) * 2 - 1) * 0.05
    return sd


def conv(sd, key: str, x: Tensor) -> Tensor:
    """Conv3d `key` (zero padding 1 in space, and in time for 3 taps) over the frames of one clip: x [T, C, H, W] -> [T, N, H, W]"""
    w = sd[P + key + ".weight"].to(x.dtype)
    pad = (w.shape[2] // 2, 1, 1)
    y = F.conv3d(x.permute(1, 0, 2, 3).unsqueeze(0), w, sd[P + key + ".bias"].to(x.dtype), padding=pad)
    return y.squeeze(0).permute(1, 0, 2, 3)


def planes(msgs: Tensor, h: int, dtype) -> Tensor:
    """frame t's bits as K constant 0 / 1 planes: [T, K, h, h]"""
    return msgs.to(dtype)[:, :, None, None].expand(-1, -1, h, h)


def up(x: Tensor, S: int) -> Tensor:
    """F.upsample_bilinear: bilinear with align_corners=True"""
    return F.interpolate(x, size=(S, S), mode="bilinear", align_corners=True)


def encoder_forward(sd, imgs: Tensor, msgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """DVMarkEmbedder.forward on ONE call: imgs [T, 3, S, S] in [0, 1], msgs [T, K] in {0, 1} -> delta [T, 3, S, S].  taps: the
    NCHW maps of the plan's taps (dve.*)"""
    S = imgs.shape[-1]
    t = taps if taps is not None else {}
    x = 2 * imgs - 1
    for i, name in ((0, "dve.t0"), (2, "dve.t2"), (4, "dve.t4")):
        x = t[name] = torch.relu(conv(sd, f"transform_layer.{i}", x))
    x = torch.relu(conv(sd, "transform_layer.6", x))
    x = t["dve.cat1"] = torch.cat([x, planes(msgs, S, x.dtype)], 1)
    x = t["dve.e1_0"] = torch.relu(conv(sd, "emb_layer1.0", x))
    x = t["dve.e1_2"] = torch.relu(conv(sd, "emb_layer1.2", x))
    skip = torch.relu(conv(sd, "emb_layer1.4", x))
    x = t["dve.cat2"] = torch.cat([F.avg_pool2d(skip, 2), planes(msgs, S // 2, x.dtype)], 1)
    x = t["dve.e2_0"] = torch.relu(conv(sd, "emb_layer2.0", x))
    x = t["dve.e2_2"] = torch.relu(conv(sd, "emb_layer2.2", x))
    x = t["dve.e2_4"] = torch.relu(conv(sd, "emb_layer2.4", x))
    x = t["dve.cat3"] = torch.cat([skip, up(x, S)], 1)
    x = t["dve.e3_0"] = torch.relu(conv(sd, "emb_layer3.0", x))
    x = t["dve.e3_2"] = torch.relu(conv(sd, "emb_layer3.2", x))
    d = t["delta"] = torch.tanh(conv(sd, "emb_layer3.4", x))
    return d


def grouped(sd, imgs: Tensor, msgs: Tensor, group: int) -> Tensor:
    """the calls of a batch cut into groups of `group` frames (the last may be shorter), concatenated"""
    return torch.cat([encoder_forward(sd, imgs[g:g + group], msgs[g:g + group]) for g in range(0, imgs.shape[0], group)])


class EncOracle(dv.DVMarkOracle):
    """restate.OracleModel with the DVMark embedder, and the DVMark / HiDDeN / ConvNeXt / SAM-ViT detector of the card.  The embedder
    runs in float64 on `device` (default: where the frames are); the rest of the pipeline in the frames' dtype where they are"""

    def __init__(self, spec: dict, sd: Dict[str, Tensor], device=None):
        super().__init__(spec, sd)
        self.emb_sd = {k: v.to(device, torch.float64) for k, v in sd.items() if k.startswith(P)}
        self.emb_device = device

    def embedder(self, imgs_res: Tensor, msgs: Tensor, taps=None) -> Tensor:
        dev = self.emb_device or imgs_res.device
        d = encoder_forward(self.emb_sd, imgs_res.to(dev, torch.float64), msgs.to(dev), taps)
        return d.to(imgs_res.device, imgs_res.dtype)

    def detector(self, imgs_res: Tensor, taps=None) -> Tensor:
        if "dvmark_decoder" in self.spec:
            return super().detector(imgs_res, taps)
        return ho.HiddenOracle.detector(self, imgs_res, taps)
