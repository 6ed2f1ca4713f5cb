"""The DVMark extractor restated in torch (float64 or fp32, CPU): cards with the `dvmark` extractor preset paired with each embedder
family, the spec, a seeded synthetic checkpoint in the reference's key layout, and the forward pass with taps.

Reference: modules/dvmark.py DVMarkDecoder (Conv3d 3x3x3 pad 1 with bias: 3 -> 128, ReLU, 128 -> 128, ReLU, AvgPool3d (1,2,2),
128 -> 256, ReLU, AvgPool3d (1,2,2), 256 -> 1 + K, mean over H and W), built by models/extractor.py build_extractor 'dvmark'.  Its
forward takes the B frames of one call as ONE clip [1, 3, T = B, H, W], in [0, 1] (no preprocess).  The rest of the pipeline (resize,
blend, video chunks) is oracle/restate.OracleModel's, via tests/hidden_oracle.HiddenOracle: DVMarkOracle only replaces the detector."""
import copy
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from tests import hidden_oracle as ho

SEED = 5151
WIDTHS = (128, 128, 256)   # out channels of layer1..layer3; layer4 has 1 + nbits
# embedders paired with the dvmark extractor: videoseal_1.0's own U-Net ("unet"), the package preset unet_small2_yuv_quant, and the
# HiDDeN encoder
EMBEDDERS = ("unet", "unet_small2_yuv_quant", "hidden")


def card(emb: str = "unet", img_size: Optional[int] = None, nbits: Optional[int] = None) -> dict:
    """videoseal_1.0 with the `dvmark` extractor preset of the package's configs and the embedder `emb` ("unet": the card's own, or
    a preset of configs/embedder.yaml)"""
    c = ho.card("unet" if emb == "unet" else emb, "convnext", img_size, nbits)
    c["extractor"] = {"model": "dvmark", "params": copy.deepcopy(ho._presets("extractor")["dvmark"]["params"])}
    return c


def spec_from_card(c: dict) -> dict:
    """hidden_oracle.spec_from_card with `dvmark_decoder` for the extractor (the ConvNeXt entries are videoseal_1.0's, unused)"""
    base = copy.deepcopy(c)
    base["extractor"] = copy.deepcopy(ho.load_card("videoseal_1.0")["extractor"])
    spec = ho.spec_from_card(base)
    spec["dvmark_decoder"] = {"nbits": spec["nbits"]}
    return spec


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, Tensor]:
    """hidden_oracle.synth_state_dict for the embedder, the detector replaced by DVMarkDecoder's layers: weights and biases
    U(-1/sqrt(fan_in), ..) as nn.Conv3d initialises them"""
    base = {k: v for k, v in spec.items() if k != "dvmark_decoder"}
    sd = {k: v for k, v in ho.synth_state_dict(base, seed).items() if not k.startswith("detector.")}
    g = torch.Generator().manual_seed(seed + 11)
    cin = 3
    for i, cout in enumerate(WIDTHS + (1 + spec["nbits"],)):
        b = 1.0 / (cin * 27) ** 0.5
        sd[f"detector.layers.layer{i + 1}.weight"] = (torch.rand(cout, cin, 3, 3, 3, generator=g) * 2 - 1) * b
        sd[f"detector.layers.layer{i + 1}.bias"] = (torch.rand(cout, generator=g) * 2 - 1) * b
        cin = cout
    return sd


def conv3d(x: Tensor, w: Tensor, b: Tensor) -> Tensor:
    """3x3x3 conv, zero padding 1 in time and space, over the frames of one clip: x [T, C, H, W] -> [T, N, H, W]"""
    y = F.conv3d(x.permute(1, 0, 2, 3).unsqueeze(0), w.to(x.dtype), b.to(x.dtype), padding=1)
    return y.squeeze(0).permute(1, 0, 2, 3)


def pool(x: Tensor) -> Tensor:
    return F.avg_pool2d(x, 2)


def decoder_forward(sd, imgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """DVMarkDecoder.forward on ONE call: imgs [T, 3, S, S] in [0, 1] -> logits [T, 1 + K] (taps: NCHW maps l1..l3 after ReLU)"""
    P = "detector.layers.layer"
    x = torch.relu(conv3d(imgs, sd[P + "1.weight"], sd[P + "1.bias"]))
    if taps is not None:
        taps["dvm.l1"] = x
    x = torch.relu(conv3d(x, sd[P + "2.weight"], sd[P + "2.bias"]))
    if taps is not None:
        taps["dvm.l2"] = x
    x = torch.relu(conv3d(pool(x), sd[P + "3.weight"], sd[P + "3.bias"]))
    if taps is not None:
        taps["dvm.l3"] = x
    x = conv3d(pool(x), sd[P + "4.weight"], sd[P + "4.bias"])
    return x.mean(dim=[2, 3])


def grouped(sd, imgs: Tensor, group: int, taps: Optional[dict] = None) -> Tensor:
    """the calls of a batch cut into groups of `group` frames (the last may be shorter), concatenated"""
    outs, parts = [], []
    for g0 in range(0, imgs.shape[0], group):
        t = {} if taps is not None else None
        outs.append(decoder_forward(sd, imgs[g0:g0 + group], t))
        parts.append(t)
    if taps is not None:
        for k in parts[0]:
            taps[k] = torch.cat([p[k] for p in parts])
    return torch.cat(outs)


# ---------------------------------------------------------------------------------------------------------------------------------
# the plans' frame slices (csrc/dvmark.cuh add_conv3d_sliced), restated: a 3x3x3 conv over C channels at h x h runs in launches of
# slice_frames(h * h * stack_width(C), B) frames, each stacking its frames' time taps into a [frames][h * h][stack_width(C)] operand

STACK_BUDGET = 512 << 20   # bytes of stacked operand per launch (kDvStackBudget)


def stack_width(C: int) -> int:
    return (3 * C + 63) // 64 * 64


def slice_frames(frame_elems: int, B: int) -> int:
    """dv_slice_frames: frames per launch whose fp16 stacked operand stays within the budget, at least one"""
    return max(1, min(B, STACK_BUDGET // (frame_elems * 2)))


def conv_slices(C: int, h: int, B: int):
    """(start, end) of each launch of the 3x3x3 conv over C channels at h x h on B frames"""
    fps = slice_frames(h * h * stack_width(C), B)
    return [(b0, min(b0 + fps, B)) for b0 in range(0, B, fps)]


def crossing_groups(slices, B: int, G: int):
    """the groups of G frames that some slice boundary cuts (the frames on either side are time neighbours)"""
    return [g for g in range(0, B, G) if any(g < b0 < min(g + G, B) for b0, _ in slices)]


def segments(B: int, G: int, slices=()):
    """(start, end) of the runs of frames that share a group and, given slices, a slice: the runs a 3x3x3 conv would see if its
    time neighbours were cut at slice boundaries too"""
    cuts = sorted({0, B} | set(range(0, B, G)) | {b0 for b0, _ in slices})
    return list(zip(cuts, cuts[1:]))


def slice_offset_ignored(ref: Tensor, slices) -> Tensor:
    """a conv output whose every slice was stacked from the first slice's frames: slice (b0, e) holds ref[0 : e - b0]"""
    return torch.cat([ref[:e - b0] for b0, e in slices])


class DVMarkOracle(ho.HiddenOracle):
    """HiddenOracle (and so restate.OracleModel) with the DVMark detector: one detector call is one clip"""

    def detector(self, imgs_res: Tensor, taps=None) -> Tensor:
        return decoder_forward(self.sd, imgs_res, taps)
