"""Synthetic checkpoints in the reference's format (`{'model': Videoseal.state_dict()}`), for benchmarking and smoke
runs when the real weights are not on disk (no network).  Key names / shapes follow the reference modules:
embedder.unet.* (modules/unet.py), detector.convnext.* (modules/convnext.py), detector.pixel_decoder.*
(modules/pixel_decoder.py).  Values: PyTorch-default-style uniform init, with randomised BatchNorm statistics, LayerNorm
affines and GRN gamma/beta so that weight-folding mistakes change the outputs."""
from __future__ import annotations

import math

import torch


def synth_state_dict(spec: dict, seed: int = 0) -> dict:
    """`spec` is videoseal_b200.cfg.spec_from_card(card)."""
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def uni(shape, fan_in):
        return (torch.rand(shape, generator=g) * 2 - 1) * (1.0 / math.sqrt(fan_in))

    def conv(key, cout, cin, k, bias, groups=1):
        fan_in = (cin // groups) * k * k
        sd[key + ".weight"] = uni((cout, cin // groups, k, k), fan_in)
        if bias:
            sd[key + ".bias"] = uni((cout,), fan_in)

    def linear(key, cout, cin):
        sd[key + ".weight"] = uni((cout, cin), cin)
        sd[key + ".bias"] = uni((cout,), cin)

    def affine(key, c):
        sd[key + ".weight"] = 1 + 0.1 * torch.randn(c, generator=g)
        sd[key + ".bias"] = 0.1 * torch.randn(c, generator=g)

    def bn(key, c):
        affine(key, c)
        sd[key + ".running_mean"] = 0.1 * torch.randn(c, generator=g)
        sd[key + ".running_var"] = 0.5 + torch.rand(c, generator=g)
        sd[key + ".num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)

    def resblock(key, cin, cout):
        conv(key + ".double_conv.0", cout, cin, 3, False)
        bn(key + ".double_conv.1", cout)
        conv(key + ".double_conv.3", cout, cout, 3, False)
        bn(key + ".double_conv.4", cout)
        conv(key + ".res_conv", cout, cin, 1, True)

    u = spec["unet"]
    z = list(u["z"])
    P = "embedder.unet."
    table = torch.randn(2 * spec["nbits"], spec["hidden"], generator=g)
    sd[P + "msg_processor.msg_embeddings.weight"] = table
    resblock(P + "inc", u["in_channels"], z[0])
    for i in range(len(z) - 1):
        conv(P + f"downs.{i}.down", z[i + 1], z[i], 3, True)
        resblock(P + f"downs.{i}.conv", z[i + 1], z[i + 1])
    zb = z[-1] + spec["hidden"]
    for i in range(u["num_blocks"]):
        resblock(P + f"bottleneck.model.{i}", zb, zb)
    zz = z[:-1] + [zb]
    for j, ii in enumerate(reversed(range(len(zz) - 1))):
        conv(P + f"ups.{j}.up.upsample_block.2", zz[ii], 2 * zz[ii + 1], 3, False)
        affine(P + f"ups.{j}.up.upsample_block.3", zz[ii])
        resblock(P + f"ups.{j}.conv", zz[ii], zz[ii])
    conv(P + "outc", u["out_channels"], zz[0], 1, True)
    sd["embedder.msg_processor.msg_embeddings.weight"] = table

    cn = spec["convnext"]
    dims, depths = cn["dims"], cn["depths"]
    Q = "detector.convnext."
    conv(Q + "downsample_layers.0.0", dims[0], 3, 4, True)
    affine(Q + "downsample_layers.0.1", dims[0])
    for i in range(3):
        affine(Q + f"downsample_layers.{i + 1}.0", dims[i])
        conv(Q + f"downsample_layers.{i + 1}.1", dims[i + 1], dims[i], 2, True)
    for s in range(4):
        for j in range(depths[s]):
            B = Q + f"stages.{s}.{j}."
            conv(B + "dwconv", dims[s], dims[s], 7, True, groups=dims[s])
            affine(B + "norm", dims[s])
            linear(B + "pwconv1", 4 * dims[s], dims[s])
            sd[B + "grn.gamma"] = 0.1 * torch.randn(1, 1, 1, 4 * dims[s], generator=g)
            sd[B + "grn.beta"] = 0.1 * torch.randn(1, 1, 1, 4 * dims[s], generator=g)
            linear(B + "pwconv2", dims[s], 4 * dims[s])
    D = "detector.pixel_decoder."
    pd = spec.get("pixel_decoder", {"pixelwise": False, "upscale_stages": [1]})
    c = dims[-1]
    for i, f in enumerate(pd["upscale_stages"]):      # pixel_decoder.py:44-50: widths c, c // f, ...
        conv(D + f"output_upscaling.{i}.upsample_block.2", c // f, c, 3, False)
        affine(D + f"output_upscaling.{i}.upsample_block.3", c // f)
        c //= f
    if pd["pixelwise"]:
        conv(D + "linear", 1 + spec["nbits"], c, 1, True)
    else:
        linear(D + "linear", 1 + spec["nbits"], c)
    return sd


def write_synthetic_checkpoint(card: dict, path: str, seed: int = 0) -> dict:
    from .cfg import spec_from_card
    spec = spec_from_card(card)
    torch.save({"model": synth_state_dict(spec, seed)}, path)
    return spec
