"""The temporal (conv_layer 'conv3d') BatchNorm + ReLU U-Net embedders restated in torch, on the videoseal_1.0 card: card, spec,
seeded synthetic checkpoint in the reference's Conv3dWrapper key layout, the forward pass and the embed grouping.

What is temporal (modules/unet.py:17-39, modules/common.py Conv3dWrapper): in every ResnetBlock `double_conv.0` / `double_conv.3`
(3x3x3, padding 1, no bias) and `res_conv` (1x1x1, with bias).  DBlock.down, the Upsample conv + LayerNorm, outc and the BatchNorms
stay 2-D.  The time axis is the batch of one embedder call: [B, C, H, W] -> [1, C, T = B, H, W], zero padding of one frame at both
ends.  A video call is one chunk of chunk_size key frames (models/videoseal.py:292-320), an image call the whole batch
(models/wam.py:134-204): OracleModel.embed already calls `embedder` exactly so, and TemporalOracle only replaces that leaf."""
import argparse
import copy
import os
import re
from typing import Dict, Optional

import torch
import torch.nn.functional as F
import yaml
from torch import Tensor

from oracle import restate
from tests.util import load_card, tmpdir

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = ("unet_small2_yuv_quant_conv3d", "unet_small2_quant_conv3d", "unet_small2_bw_quant_conv3d")
TWIN = {"unet_small2_yuv_quant_conv3d": "unet_small2_yuv_quant", "unet_small2_quant_conv3d": "unet_small2_quant"}
SEED = 1234
TEMPORAL_KEY_3D = "embedder.unet.inc.double_conv.0.conv.weight"
# the Conv3dWrapper convs of a U-Net state dict, by their 2-D key
_TEMPORAL = re.compile(r"^embedder\.unet\.(inc|downs\.\d+\.conv|bottleneck\.model\.\d+|ups\.\d+\.conv)\.(double_conv\.[03]|res_conv)\."
                       r"(weight|bias)$")


def preset_card(preset: str, img_size: Optional[int] = None) -> dict:
    """videoseal_1.0 with its embedder replaced by a preset of the package's configs/embedder.yaml"""
    card = copy.deepcopy(load_card("videoseal_1.0"))
    presets = yaml.safe_load(open(os.path.join(ROOT, "videoseal_b200", "configs", "embedder.yaml")))
    card["embedder"] = {"model": preset, "params": copy.deepcopy(presets[preset])}
    if img_size is not None:
        card["args"]["img_size_proc"] = img_size
    return card


def spec_from_card(card: dict) -> dict:
    spec = restate.spec_from_card(card)
    spec["unet"]["temporal"] = card["embedder"]["params"]["unet"].get("conv_layer", "conv2d") == "conv3d"
    return spec


def _conv3d_key(k: str) -> str:
    stem, leaf = k.rsplit(".", 1)
    return f"{stem}.conv.{leaf}"


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, Tensor]:
    """restate.synth_state_dict; for a temporal spec with the ResnetBlock convs as Conv3dWrapper tensors: random 3x3x3 weights (every time tap non-zero,
    nn.Conv3d's default U(-1/sqrt(fan_in), ..) with fan_in = 27 C) and the 1x1 res convs unsqueezed to 1x1x1"""
    sd = restate.synth_state_dict(spec, seed)
    if not spec["unet"].get("temporal", False):      # a 2-D preset (the twin of a temporal one) keeps its 2-D checkpoint
        return sd
    g = torch.Generator().manual_seed(seed + 1)
    for k in sorted(k for k in sd if _TEMPORAL.match(k)):
        v = sd.pop(k)
        if v.dim() == 4 and v.shape[-1] == 3:
            n, c = v.shape[:2]
            v = restate._kaiming_uniform((n, c, 3, 3, 3), c * 27, g)
        elif v.dim() == 4:
            v = v.unsqueeze(2)
        sd[_conv3d_key(k)] = v
    return sd


def inflate(sd: Dict[str, Tensor]) -> Dict[str, Tensor]:
    """scripts/inflate_model_to_temporal.py inflate_convs_unet_embedder_inplace, restated: a 2-D U-Net's 3x3 weights become 3x3x3 with
    zero t-1 / t+1 taps, 1x1 weights 1x1x1, and every ResnetBlock conv key gains `.conv.`"""
    out = dict(sd)
    for k in [k for k in sd if _TEMPORAL.match(k)]:
        v = out.pop(k)
        if v.dim() == 4 and v.shape[-1] == 3:
            z = torch.zeros_like(v).unsqueeze(2)
            v = torch.cat([z, v.unsqueeze(2), z], 2)
        elif v.dim() == 4:
            v = v.unsqueeze(2)
        out[_conv3d_key(k)] = v
    return out


def sam_card(preset: str) -> dict:
    """preset_card(preset) with videoseal_0.0's SAM-ViT (sam_small) extractor"""
    card = preset_card(preset)
    card["extractor"] = copy.deepcopy(load_card("videoseal_0.0")["extractor"])
    return card


def inflate_script(sd: Dict[str, Tensor], extractor_type: str, record: dict) -> Dict[str, Tensor]:
    """The whole of scripts/inflate_model_to_temporal.py restated: `inflate` on the U-Net, then the extractor part for
    --extractor_type `extractor_type`, whose removed / added keys are `record` (tests/golden/temporal_inflate.pt, written from the
    script itself).  ConvNeXt: downsample_layers.{1,2,3}.1.{weight,bias} move under `.1.conv.`, each gains an identity temp_conv
    (3 x 1 x 1, the centre tap the identity matrix); SAM: temp_blocks and pos_embed_temporal (zeros).  The temporal attention blocks'
    mlp.lin2 is zero, as the script sets it; their other tensors are default-initialised there and filled with 0.01 here (a block
    with a zero lin2 adds nothing, whatever they hold)."""
    out = inflate(sd)
    for k in record["removed"]:
        v = out.pop(k)
        out[_conv3d_key(k)] = v
    for k, shape in record["added"].items():
        if k in out:
            continue
        if k.endswith(".temp_conv.weight"):
            v = torch.zeros(shape)
            v[:, :, shape[2] // 2, 0, 0] = torch.eye(shape[0])
        elif k.endswith((".mlp.lin2.weight", ".mlp.lin2.bias", "pos_embed_temporal")):
            v = torch.zeros(shape)
        else:
            v = torch.full(shape, 0.01)
        out[k] = v
    return out


def conv3d_frames(x: Tensor, w: Tensor, b: Optional[Tensor] = None) -> Tensor:
    """Conv3dWrapper.forward: the frames of x [T, C, H, W] are the time axis of one [1, C, T, H, W] volume"""
    y = F.conv3d(x.permute(1, 0, 2, 3).unsqueeze(0), w, b, padding=w.shape[-1] // 2)
    return y.squeeze(0).permute(1, 0, 2, 3)


def resnet_block(sd, key: str, x: Tensor) -> Tensor:
    """modules/unet.py:17-39 with conv_layer=Conv3dWrapper, BatchNorm + ReLU"""
    h = conv3d_frames(x, sd[key + ".double_conv.0.conv.weight"])
    h = F.relu(restate._norm(sd, key + ".double_conv.1", "batch", h))
    h = conv3d_frames(h, sd[key + ".double_conv.3.conv.weight"])
    h = F.relu(restate._norm(sd, key + ".double_conv.4", "batch", h))
    return h + conv3d_frames(x, sd[key + ".res_conv.conv.weight"], sd[key + ".res_conv.conv.bias"])


def unet_forward(sd, spec, x: Tensor, msgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """models/embedder.py:151-165 + modules/unet.py:170-197 for one embedder call (the frames of x are one time axis)"""
    u = spec["unet"]
    P = "embedder.unet."
    x = x * 2 - 1
    hiddens = [resnet_block(sd, P + "inc", x)]
    nd = len(u["mults"]) - 1
    for i in range(nd):
        d = F.conv2d(hiddens[-1], sd[P + f"downs.{i}.down.weight"], sd[P + f"downs.{i}.down.bias"], stride=2, padding=1)
        hiddens.append(resnet_block(sd, P + f"downs.{i}.conv", d))
        if taps is not None:
            taps[f"down{i}"] = hiddens[-1]
    lat = hiddens.pop()
    m = restate.msg_embed(sd, spec, msgs)
    lat = torch.cat([lat, m[:, :, None, None].repeat(1, 1, lat.shape[-2], lat.shape[-1])], dim=1)
    hiddens.append(lat)
    x = lat
    for i in range(u["num_blocks"]):
        x = resnet_block(sd, P + f"bottleneck.model.{i}", x)
        if taps is not None:
            taps[f"bott{i}"] = x
    for j in range(nd):
        x = torch.cat((x, hiddens.pop() * (2 ** -0.5)), dim=1)
        x = restate.upsample_block(sd, P + f"ups.{j}.up", x, "relu")
        x = resnet_block(sd, P + f"ups.{j}.conv", x)
        if taps is not None:
            taps[f"up{j}"] = x
    x = F.conv2d(x, sd[P + "outc.weight"], sd[P + "outc.bias"])
    return torch.tanh(x) if u["last_tanh"] else x


class TemporalOracle(restate.OracleModel):
    """OracleModel whose embedder is the temporal U-Net: one `embedder` call = one time axis"""

    def embedder(self, imgs_res: Tensor, msgs: Tensor, taps=None) -> Tensor:
        x = restate.rgb_to_y(imgs_res) if self.spec["yuv"] else imgs_res
        return unet_forward(self.sd, self.spec, x, msgs, taps)


def training_checkpoint(card: dict, sd: dict, tag: str, embedder_model: Optional[str] = None) -> str:
    """a raw training checkpoint whose args name the embedder / extractor presets (utils/cfg.py:50-85)"""
    args = argparse.Namespace(**card["args"], embedder_model=embedder_model or card["embedder"]["model"],
                              extractor_model=card["extractor"]["model"])
    args.attenuation_config = os.path.join(ROOT, "videoseal_b200", "configs", "attenuation.yaml")
    path = tmpdir() / f"train_{tag}.pth"
    torch.save({"model": sd, "args": args}, path)
    return str(path)


def model_pair(preset: str, device: Optional[str] = "cuda:0", seed: int = SEED, img_size: Optional[int] = None):
    """(product Videoseal loaded from a training checkpoint naming `preset`, TemporalOracle on CPU, oracle spec)"""
    import videoseal_b200.utils.cfg
    card = preset_card(preset, img_size)
    spec = spec_from_card(card)
    sd = synth_state_dict(spec, seed)
    path = training_checkpoint(card, sd, f"{preset}_{seed}_{spec['img_size']}")
    model = videoseal_b200.utils.cfg.setup_model_from_checkpoint(path).eval()
    if device is not None:
        model = model.to(device)
    return model, TemporalOracle(spec, sd), spec


def sample(t: Tensor) -> Tensor:
    """strided sample of a [F, C, H, W] tensor stored in the fixture"""
    return t[:, :, ::7, ::5].clone()
