"""The VAE embedder restated in torch (float64 or fp32, CPU or GPU): cards with a `vae*` embedder preset paired with each extractor
family, the spec, a seeded synthetic checkpoint in the reference's key layout, and the forward pass with taps.

Reference: modules/vae.py (ResnetBlock, AttnBlock, Downsample, Upsample, VAEEncoder, VAEDecoder; GroupNorm(16, eps 1e-6), SiLU),
modules/msg_processor.py ('binary+concat': sum_k E[2k + m_k] as constant planes after the latent), models/embedder.py VAEEmbedder
(imgs = 2 x - 1) built by build_embedder 'vae*' (decoder z_channels = z + hidden, yuv = 'yuv' in the name).  The rest of the
pipeline (resize, video chunks, JND, blend, Y extraction) is oracle/restate.OracleModel's: VaeOracle only replaces the embedder."""
import copy
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import restate
from tests import dvmark_enc_oracle as de
from tests import hidden_oracle as ho

SEED = 9191
PRESETS = ("vae_tiny", "vae_tiny_yuv", "vae_small", "vae_small_yuv", "vae_small_bw", "vae_big")
EXTRACTORS = ("convnext", "sam", "hidden", "dvmark")
E, D, M = "embedder.encoder.", "embedder.decoder.", "embedder.msg_processor.msg_embeddings.weight"


def card(preset: str = "vae_small", img_size: Optional[int] = None, nbits: Optional[int] = None, extractor: str = "convnext") -> dict:
    """videoseal_1.0 with the `preset` embedder of the package's configs and the extractor `extractor` ("convnext": the card's own,
    "sam": videoseal_0.0's, "hidden" / "dvmark": the package's presets)"""
    c = de.card(extractor, img_size, nbits)
    c["embedder"] = {"model": preset, "params": copy.deepcopy(ho._presets("embedder")[preset])}
    return c


def spec_from_card(c: dict) -> dict:
    """the extractor side's oracle spec, with `vae_encoder` for the embedder (cfg._vae's fields) and yuv = 'yuv' in the name"""
    base = copy.deepcopy(c)
    base["embedder"] = {"model": "dvmark", "params": []}
    spec = de.spec_from_card(base)
    del spec["dvmark_encoder"]
    enc, dec = c["embedder"]["params"]["encoder"], c["embedder"]["params"]["decoder"]
    spec["vae_encoder"] = {"in_channels": int(enc["in_channels"]), "out_ch": int(dec["out_ch"]), "ch": int(enc["ch"]),
                           "ch_mult": [int(m) for m in enc["ch_mult"]], "num_res_blocks": int(enc["num_res_blocks"]),
                           "z_channels": int(enc["z_channels"]), "tanh_out": bool(dec.get("tanh_out", False))}
    spec["yuv"] = "yuv" in c["embedder"]["model"]
    return spec


def widths(v: dict):
    return [v["ch"] * m for m in v["ch_mult"]]


def synth_state_dict(spec: dict, seed: int = SEED) -> Dict[str, Tensor]:
    """the extractor side's synthetic checkpoint with the VAE embedder's keys.  Convs U(-a, a), a = sqrt(3 / fan_in) (unit-variance
    outputs), conv2 / proj_out weights halved so the residual stream grows slowly; biases U(-0.1, 0.1); GroupNorm affines
    1 + 0.2 N(0, 1) and 0.2 N(0, 1) (a wrong group layout or a dropped affine shows); embeddings N(0, 0.3)"""
    v = spec["vae_encoder"]
    base = {k: val for k, val in spec.items() if k != "vae_encoder"}
    base["dvmark_encoder"] = {"nbits": spec["nbits"]}
    sd = {k: t for k, t in de.synth_state_dict(base, seed).items() if not k.startswith("embedder.")}
    g = torch.Generator().manual_seed(seed + 29)

    def conv(key, cout, cin, k, gain=1.0):
        a = gain * (3.0 / (cin * k * k)) ** 0.5
        sd[key + ".weight"] = (torch.rand(cout, cin, k, k, generator=g) * 2 - 1) * a
        sd[key + ".bias"] = (torch.rand(cout, generator=g) * 2 - 1) * 0.1

    def gn(key, c):
        sd[key + ".weight"] = 1 + 0.2 * torch.randn(c, generator=g)
        sd[key + ".bias"] = 0.2 * torch.randn(c, generator=g)

    def res(key, cin, cout):
        gn(key + ".norm1", cin)
        conv(key + ".conv1", cout, cin, 3)
        gn(key + ".norm2", cout)
        conv(key + ".conv2", cout, cout, 3, 0.5)
        if cin != cout:
            conv(key + ".nin_shortcut", cout, cin, 1)

    def attn(key, c):
        gn(key + ".norm", c)
        for m in ("q", "k", "v"):
            conv(key + "." + m, c, c, 1)
        conv(key + ".proj_out", c, c, 1, 0.5)

    w, L, nr, z, hid = widths(v), len(v["ch_mult"]), v["num_res_blocks"], v["z_channels"], spec["hidden"]
    conv(E + "conv_in", v["ch"], v["in_channels"], 3)
    cin = v["ch"]
    for l in range(L):
        for i in range(nr):
            res(E + f"down.{l}.block.{i}", cin, w[l])
            cin = w[l]
        if l != L - 1:
            conv(E + f"down.{l}.downsample.conv", cin, cin, 3)
    res(E + "mid.block_1", cin, cin)
    attn(E + "mid.attn_1", cin)
    res(E + "mid.block_2", cin, cin)
    gn(E + "norm_out", cin)
    conv(E + "conv_out", z, cin, 3)
    sd[M] = 0.3 * torch.randn(2 * spec["nbits"], hid, generator=g)
    conv(D + "conv_in", w[-1], z + hid, 3)
    cin = w[-1]
    res(D + "mid.block_1", cin, cin)
    attn(D + "mid.attn_1", cin)
    res(D + "mid.block_2", cin, cin)
    for l in reversed(range(L)):
        for i in range(nr + 1):
            res(D + f"up.{l}.block.{i}", cin, w[l])
            cin = w[l]
        if l != 0:
            conv(D + f"up.{l}.upsample.conv", cin, cin, 3)
    gn(D + "norm_out", cin)
    conv(D + "conv_out", v["out_ch"], cin, 3, 0.5)
    return sd


# ---- the forward pass (NCHW, any float dtype); `t` collects the plan's taps in NCHW
def gn(sd, key, x, silu, eps=1e-6):
    y = F.group_norm(x, 16, sd[key + ".weight"].to(x.dtype), sd[key + ".bias"].to(x.dtype), eps)
    return F.silu(y) if silu else y


def conv(sd, key, x, stride=1, pad=1):
    w = sd[key + ".weight"].to(x.dtype)
    return F.conv2d(x, w, sd[key + ".bias"].to(x.dtype), stride=stride, padding=pad if w.shape[-1] == 3 else 0)


def resnet(sd, key, x, t, tp):
    a1 = t[tp + ".gn1"] = gn(sd, key + ".norm1", x, True)
    h = t[tp + ".conv1"] = conv(sd, key + ".conv1", a1)
    a2 = t[tp + ".gn2"] = gn(sd, key + ".norm2", h, True)
    sc = x
    if key + ".nin_shortcut.weight" in sd:
        sc = t[tp + ".nin"] = conv(sd, key + ".nin_shortcut", x)
    out = t[tp + ".out"] = sc + conv(sd, key + ".conv2", a2)
    return out


def attention(sd, key, x, t, tp):
    B, C, h, w = x.shape
    n = t[tp + ".gn"] = gn(sd, key + ".norm", x, False)
    q, k, v = (conv(sd, key + "." + m, n).reshape(B, C, h * w) for m in ("q", "k", "v"))
    t[tp + ".qkv"] = torch.cat([q, k, v], 1).reshape(B, 3 * C, h, w)
    p = torch.softmax(torch.bmm(q.permute(0, 2, 1), k) * C ** -0.5, dim=2)        # [B, queries, keys]
    o = t[tp + ".o"] = torch.bmm(v, p.permute(0, 2, 1)).reshape(B, C, h, w)
    out = t[tp + ".out"] = x + conv(sd, key + ".proj_out", o)
    return out


def aux(sd, msgs: Tensor, dtype) -> Tensor:
    """msg_processor 'binary+concat': [B, hidden] = sum_k E[2k + m_k]"""
    Em = sd[M].to(dtype)
    idx = 2 * torch.arange(msgs.shape[-1], device=msgs.device) + msgs.long()
    return Em[idx].sum(dim=-2)


def vae_forward(sd, v: dict, x: Tensor, msgs: Tensor, taps: Optional[dict] = None) -> Tensor:
    """VAEEmbedder.forward: x [B, in_ch, S, S] in [0, 1] (Y for yuv cards), msgs [B, K] -> delta [B, out_ch, S, S]"""
    t = taps if taps is not None else {}
    L, nr = len(v["ch_mult"]), v["num_res_blocks"]
    h = t["vae.enc.conv_in"] = conv(sd, E + "conv_in", 2 * x - 1)
    for l in range(L):
        for i in range(nr):
            h = resnet(sd, E + f"down.{l}.block.{i}", h, t, f"vae.enc.d{l}.{i}")
        if l != L - 1:
            h = t[f"vae.enc.down{l}"] = conv(sd, E + f"down.{l}.downsample.conv", F.pad(h, (0, 1, 0, 1)), stride=2, pad=0)
    h = resnet(sd, E + "mid.block_1", h, t, "vae.enc.mid1")
    h = attention(sd, E + "mid.attn_1", h, t, "vae.enc.attn")
    h = resnet(sd, E + "mid.block_2", h, t, "vae.enc.mid2")
    a = t["vae.enc.gn_out"] = gn(sd, E + "norm_out", h, True)
    lat = t["vae.latent"] = conv(sd, E + "conv_out", a)
    ax = aux(sd, msgs, x.dtype)
    z = torch.cat([lat, ax[:, :, None, None].expand(-1, -1, *lat.shape[-2:])], 1)
    h = t["vae.dec.conv_in"] = conv(sd, D + "conv_in", z)
    h = resnet(sd, D + "mid.block_1", h, t, "vae.dec.mid1")
    h = attention(sd, D + "mid.attn_1", h, t, "vae.dec.attn")
    h = resnet(sd, D + "mid.block_2", h, t, "vae.dec.mid2")
    for l in reversed(range(L)):
        for i in range(nr + 1):
            h = resnet(sd, D + f"up.{l}.block.{i}", h, t, f"vae.dec.u{l}.{i}")
        if l != 0:
            h = t[f"vae.dec.up{l}"] = conv(sd, D + f"up.{l}.upsample.conv", F.interpolate(h, scale_factor=2.0, mode="nearest"))
    a = t["vae.dec.gn_out"] = gn(sd, D + "norm_out", h, True)
    d = conv(sd, D + "conv_out", a)
    d = t["delta"] = torch.tanh(d) if v["tanh_out"] else d
    return d


class VaeOracle(de.EncOracle):
    """restate.OracleModel with the VAE embedder (float64 on `device`, default where the frames are) and the card's detector"""

    def __init__(self, spec: dict, sd: Dict[str, Tensor], device=None):
        super().__init__(spec, sd, device)
        self.emb_sd = {k: val.to(device, torch.float64) for k, val in sd.items() if k.startswith("embedder.")}

    def embedder(self, imgs_res: Tensor, msgs: Tensor, taps=None) -> Tensor:
        dev = self.emb_device or imgs_res.device
        x = imgs_res.to(dev, torch.float64)
        if self.spec["yuv"]:
            x = restate.rgb_to_y(x.float().cpu()).to(dev, torch.float64)
        d = vae_forward(self.emb_sd, self.spec["vae_encoder"], x, msgs.to(dev), taps)
        return d.to(imgs_res.device, imgs_res.dtype)
