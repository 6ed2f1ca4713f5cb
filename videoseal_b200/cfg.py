"""Model-card / checkpoint resolution and model assembly.

Mirrors videoseal/utils/cfg.py of the reference (setup_model_from_model_card :181-259, setup_model :88-154,
maybe_download_checkpoint :262-287) without OmegaConf: cards are read with PyYAML into plain dicts.  The card YAML
schema and the checkpoint format (`torch.load(..., weights_only=True)['model']` = Videoseal.state_dict()) are the
reference's, consumed as-is.
"""
from __future__ import annotations

import math
import os
import re
from pathlib import Path
from urllib.parse import urlparse

import torch
import yaml

DEFAULT_CARD = "videoseal_1.0"
PKG_DIR = Path(__file__).resolve().parent
CARDS_DIR = PKG_DIR / "cards"


def resolve_config_path(cfg_path) -> Path:
    """working directory first, then the package directory (cfg.py:40-48 of the reference)"""
    p = Path(cfg_path)
    if p.is_file():
        return p
    q = PKG_DIR / cfg_path
    if q.is_file():
        return q
    raise FileNotFoundError(f"config file {cfg_path} not found (cwd or {PKG_DIR})")


def is_url(s) -> bool:
    try:
        r = urlparse(str(s))
        return all([r.scheme, r.netloc])
    except ValueError:
        return False


def maybe_download_checkpoint(url: str) -> str:
    """same cache naming as the reference: ckpts/<parent>_<file> (cfg.py:262-287)"""
    parts = urlparse(url).path.split("/")
    basename = f"{parts[-2]}_{parts[-1]}" if len(parts) >= 2 else parts[-1]
    os.makedirs("ckpts", exist_ok=True)
    filename = os.path.abspath(os.path.join("ckpts", basename))
    if os.path.exists(filename):
        return filename
    try:
        import requests
        resp = requests.get(url, timeout=30)
        resp.raise_for_status()
        with open(filename, "wb") as f:
            f.write(resp.content)
    except Exception as e:  # no network in most deployments of this package
        raise FileNotFoundError(
            f"checkpoint {url} is not cached at {filename} and could not be downloaded ({e}); "
            "put the file there or point the card's checkpoint_path at a local .pth") from e
    return filename


def spec_from_card(card: dict) -> dict:
    """Architecture hyper-parameters from a card (build_embedder embedder.py:243-282, build_extractor
    extractor.py:170-213, back-compat renames cfg.py:101-118)."""
    a = card["args"]
    nbits = int(a["nbits"])
    hsm = a.get("hidden_size_multiplier", 2)
    img_size = a["img_size_proc"] if "img_size_proc" in a else a["img_size_extractor"]
    emb_name = str(card["embedder"]["model"])
    ext_name = str(card["extractor"]["model"])
    if not emb_name.startswith(("unet", "hidden", "dvmark", "vae")):
        raise NotImplementedError(f"embedder '{emb_name}': only the unet*, hidden*, dvmark* and vae* families are on the CUDA hot path")
    is_vit = ext_name.startswith("sam")
    if not (ext_name.startswith(("convnext", "hidden", "dvmark")) or is_vit):
        raise NotImplementedError(f"extractor '{ext_name}': only the convnext*, sam*, hidden* and dvmark* families are on the CUDA hot "
                                  "path")
    if str(a.get("blending_method", "additive")) != "additive":
        raise NotImplementedError("only additive blending is implemented (all shipped cards use it)")
    if emb_name.startswith("hidden"):
        embedder = {"hidden_encoder": _hidden(card["embedder"]["params"], embedder=True)}
    elif emb_name.startswith("dvmark"):
        # build_embedder: DVMarkEmbedder(DVMarkEncoder(nbits)); the preset has no parameters (params: [])
        embedder = {"dvmark_encoder": {"nbits": nbits}}
    elif emb_name.startswith("vae"):
        embedder = {"vae_encoder": _vae(card["embedder"]["params"], emb_name)}
    else:
        embedder = _unet(card["embedder"]["params"])
    if ext_name.startswith("hidden"):
        extractor = {"hidden_decoder": _hidden(card["extractor"]["params"], embedder=False),
                     "pixel_decoder": {"pixelwise": False, "upscale_stages": [1]}}
    elif ext_name.startswith("dvmark"):
        # build_extractor: DVMarkDecoder(nbits); the preset has no parameters (params: [])
        extractor = {"dvmark_decoder": {"nbits": nbits}, "pixel_decoder": {"pixelwise": False, "upscale_stages": [1]}}
    else:
        extractor = _trunk(card["extractor"]["params"], nbits, is_vit)
    att = str(a.get("attenuation", "None"))
    jnd = (0, 0)
    if att.lower().startswith("jnd"):
        att_cfg = yaml.safe_load(open(resolve_config_path(a.get("attenuation_config", "configs/attenuation.yaml"))))
        jnd = (int(att_cfg[att]["in_channels"]), int(att_cfg[att]["out_channels"]))
    spec = {
        "nbits": nbits, "hidden": int(nbits * hsm), "img_size": int(img_size), "yuv": "yuv" in emb_name,
        "scaling_w": float(a["scaling_w"]), "scaling_i": float(a["scaling_i"]),
        "chunk_size": int(a.get("videoseal_chunk_size", a.get("videowam_chunk_size", 8))),
        "step_size": int(a.get("videoseal_step_size", a.get("videowam_step_size", 4))),
        **embedder,
        **extractor,
        "jnd": jnd, "attenuation": att,
    }
    # the geometry rules of the kernels (widths, sizes, pixel-decoder stages) live in the native library: a dry run, no GPU needed
    from .model import check_native
    check_native(spec)
    return spec


_HIDDEN_NORMS = {"batch": 0, "group": 1}
_HIDDEN_ACTS = {"relu": 0, "gelu": 1}


def _hidden(p: dict, embedder: bool) -> dict:
    """spec['hidden_encoder'] / spec['hidden_decoder'] of a hidden* preset (modules/hidden.py HiddenEncoder / HiddenDecoder; the
    preset's num_bits is replaced by args.nbits, embedder.py:263-268, extractor.py:183-188)"""
    what = "HiDDeN embedder" if embedder else "HiDDeN extractor"
    norm, act = str(p["normalization"]), str(p["activation"])
    if not any(norm.startswith(k) for k in _HIDDEN_NORMS):   # common.py get_normalization matches on the prefix
        raise NotImplementedError(f"{what}: normalization '{norm}' is not implemented (batch, group)")
    if act not in _HIDDEN_ACTS:
        raise NotImplementedError(f"{what}: activation '{act}' is not implemented (relu, gelu)")
    if int(p.get("in_channels", 3)) != 3 or (embedder and int(p.get("out_channels", 3)) != 3):
        raise NotImplementedError(f"{what}: in_channels / out_channels other than 3 are not implemented")
    if not embedder and p.get("pixelwise", False):
        raise NotImplementedError(f"{what}: pixelwise=True (per-pixel maps) is not implemented")
    h = {"z_channels": int(p["z_channels"]), "num_blocks": int(p["num_blocks"]),
         "normalization": next(k for k in _HIDDEN_NORMS if norm.startswith(k)), "activation": act}
    if embedder:
        h["last_tanh"] = bool(p.get("last_tanh", True))
    return h


def _vae(p: dict, name: str) -> dict:
    """spec['vae_encoder'] of a vae* embedder (embedder.py:245-254, modules/vae.py VAEEncoder / VAEDecoder).  The decoder's
    z_channels is set by build_embedder (z + hidden); the encoder's out_ch, resolution and dropout do nothing in eval."""
    enc, dec, mp = p["encoder"], p["decoder"], p.get("msg_processor", {})
    if mp.get("msg_processor_type", "binary+concat") != "binary+concat":
        raise NotImplementedError("VAE embedder: only the 'binary+concat' message processor is implemented")
    if float(mp.get("msg_mult", 1.0)) != 1.0:
        raise NotImplementedError("VAE embedder: msg_mult other than 1 is not implemented")
    for part, c in (("encoder", enc), ("decoder", dec)):
        if list(c.get("attn_resolutions", [])):
            raise NotImplementedError(f"VAE {part}: attention blocks inside levels (attn_resolutions) are not implemented")
        if c.get("use_linear_attn", False) or str(c.get("attn_type", "vanilla")) != "vanilla":
            raise NotImplementedError(f"VAE {part}: only the vanilla AttnBlock is implemented (no linear attention)")
        if not c.get("resamp_with_conv", True):
            raise NotImplementedError(f"VAE {part}: resamp_with_conv=False (conv-less resampling) is not implemented")
    if enc.get("double_z", True):
        # the VAEEncoder default; build_embedder sizes the decoder for z_channels latent channels, so 2 z cannot be built
        raise NotImplementedError("VAE encoder: double_z=True is not implemented (build_embedder's channel arithmetic needs False)")
    if dec.get("give_pre_end", False):
        raise NotImplementedError("VAE decoder: give_pre_end=True is not implemented")
    if dec.get("bw", False):
        raise NotImplementedError("VAE decoder: bw=True is not implemented")
    mult = [int(m) for m in enc["ch_mult"]]
    if [int(m) for m in dec["ch_mult"]] != mult or int(dec["ch"]) != int(enc["ch"]) or \
            int(dec["num_res_blocks"]) != int(enc["num_res_blocks"]):
        raise NotImplementedError("VAE embedder: an encoder and decoder of different ch / ch_mult / num_res_blocks are not implemented")
    return {"in_channels": int(enc["in_channels"]), "out_ch": int(dec["out_ch"]), "ch": int(enc["ch"]), "ch_mult": mult,
            "num_res_blocks": int(enc["num_res_blocks"]), "z_channels": int(enc["z_channels"]),
            "tanh_out": bool(dec.get("tanh_out", False))}


def _unet(ep: dict) -> dict:
    """spec['unet'] of a unet* embedder (embedder.py:270-282)"""
    u = ep["unet"]
    mp = ep.get("msg_processor", {})
    if mp.get("msg_processor_type", "binary+concat") != "binary+concat":
        raise NotImplementedError("only 'binary+concat' message processors are implemented")
    conv_layer = str(u.get("conv_layer", "conv2d"))
    if conv_layer not in ("conv2d", "conv3d"):
        raise NotImplementedError(f"U-Net conv_layer '{conv_layer}' is not implemented (conv2d, or conv3d with BatchNorm + ReLU)")
    if conv_layer == "conv3d" and (str(u["activation"]) != "relu" or not str(u["normalization"]).startswith("batch")):
        raise NotImplementedError(f"temporal (conv3d) U-Net with {u['activation']}/{u['normalization']}: only BatchNorm + ReLU is "
                                  "implemented")
    return {"unet": {
        "in_channels": int(u["in_channels"]), "out_channels": int(u["out_channels"]),
        "z": [int(u["z_channels"]) * int(m) for m in u["z_channels_mults"]], "num_blocks": int(u["num_blocks"]),
        "activation": str(u["activation"]), "normalization": str(u["normalization"]),
        "last_tanh": bool(u.get("last_tanh", True)), "temporal": conv_layer == "conv3d",
    }}


def _trunk(ep: dict, nbits: int, is_vit: bool) -> dict:
    """spec['convnext'] or spec['vit'] and spec['pixel_decoder'] of a convnext* / sam* extractor"""
    pd = ep.get("pixel_decoder", {})
    pixelwise = bool(pd.get("pixelwise", False))
    stages = [int(f) for f in pd.get("upscale_stages", [1])]
    if pd.get("sigmoid_output", False):
        raise NotImplementedError("pixel decoder: sigmoid_output=True is not implemented")
    if not pixelwise and stages != [1]:
        raise NotImplementedError("pixel decoder: a pooled (pixelwise=False) decoder needs upscale_stages=[1]")
    if pixelwise and (not stages or any(f not in (2, 4) for f in stages)):
        raise NotImplementedError(f"pixel decoder: pixel-wise upscale_stages must be factors of 2 or 4, got {stages}")
    # modules/common.py:36-66: 'nearest', 'conv' and 'pixelshuffle' have other arithmetic (the first even the same weights)
    if pixelwise and str(pd.get("upscale_type", "bilinear")) != "bilinear":
        raise NotImplementedError(f"pixel decoder: upscale_type '{pd.get('upscale_type')}' is not implemented (only 'bilinear')")
    enc = ep["encoder"]
    trunk = _vit_trunk(enc) if is_vit else _convnext_trunk(ep, enc, nbits, pixelwise)
    return {**trunk, "pixel_decoder": {"pixelwise": pixelwise, "upscale_stages": stages}}


def _convnext_trunk(ep: dict, enc: dict, nbits: int, pixelwise: bool) -> dict:
    """spec['convnext'] of a convnext* extractor (extractor.py:188-213)"""
    if pixelwise and (ep.get("proportional_dim", False) or int(enc.get("stem_stride", 4)) != 4):
        raise NotImplementedError("pixel decoder: pixel-wise maps need a non-proportional ConvNeXt trunk with stem_stride 4")
    dims = [int(x) for x in enc["dims"]]
    if ep.get("proportional_dim", False):
        mult = math.sqrt(nbits / 128)
        dims = [int(x * mult) for x in dims]
    if enc.get("temporal_convs", False) or enc.get("temporal_attention", False):
        raise NotImplementedError("temporal ConvNeXt variants are out of scope")
    return {"convnext": {"depths": [int(x) for x in enc["depths"]], "dims": dims, "stem_stride": int(enc.get("stem_stride", 4))}}


_VIT_KEYS = ("embed_dim", "depth", "num_heads", "patch_size", "window_size", "global_attn_indexes", "mlp_ratio", "out_chans")
_CONVNEXT_KEYS = ("depths", "dims", "stem_stride", "drop_path_rate", "layer_scale_init_value", "head_init_scale")


def _vit_trunk(enc: dict) -> dict:
    """spec['vit'] of a sam* extractor (extractor.py:170-176, ImageEncoderViT vit.py:14-110); the processing size is the ViT's
    img_size (build_extractor overrides the card's)"""
    missing = [k for k in _VIT_KEYS if k not in enc]
    foreign = [k for k in _CONVNEXT_KEYS if k in enc]
    if missing or foreign:
        raise NotImplementedError(f"SAM-ViT extractor: the encoder block lacks {missing} / carries ConvNeXt keys {foreign}")
    if not enc.get("use_abs_pos", True):
        raise NotImplementedError("SAM-ViT extractor: use_abs_pos=False is not implemented")
    if enc.get("temporal_attention", False):
        raise NotImplementedError("SAM-ViT extractor: temporal_attention is out of scope")
    E, depth, ws = int(enc["embed_dim"]), int(enc["depth"]), int(enc["window_size"])
    glob = sorted({int(i) for i in enc["global_attn_indexes"]})
    if ws == 0:          # vit.py:79: window_size 0 makes every block global
        glob = list(range(depth))
    return {"vit": {
        "embed_dim": E, "depth": depth, "num_heads": int(enc["num_heads"]), "patch_size": int(enc["patch_size"]),
        "window_size": ws, "global_attn_indexes": [i for i in glob if 0 <= i < depth],
        "mlp_dim": int(E * float(enc["mlp_ratio"])), "out_chans": int(enc["out_chans"]),
        "qkv_bias": bool(enc.get("qkv_bias", True)), "use_rel_pos": bool(enc.get("use_rel_pos", False)),
    }}


# a Conv3dWrapper checkpoint key of every temporal U-Net (the first ResnetBlock's first conv)
TEMPORAL_KEY = "embedder.unet.inc.double_conv.0.conv.weight"


def is_temporal_state_dict(sd: dict) -> bool:
    """the U-Net of `sd` was built with conv_layer='conv3d' (5-D Conv3dWrapper weights)"""
    w = sd.get(TEMPORAL_KEY)
    return isinstance(w, torch.Tensor) and w.dim() == 5


# scripts/inflate_model_to_temporal.py also inflates the extractor (its --extractor_type): a ConvNeXt's downsample convs move under
# `.1.conv.` next to a temporal conv initialised as the identity, and temporal attention blocks (ConvNeXt stages, or a SAM-ViT's
# temp_blocks with pos_embed_temporal) are added with a zero output layer.  Temporal extractors do not run here.
_CNX_DS_CONV = re.compile(r"^(detector\.convnext\.downsample_layers\.\d+\.1)\.conv\.(weight|bias)$")
_TEMP_BLOCK = re.compile(r"^(detector\.convnext\.stages\.\d+\.\d+\.temp_block\.|detector\.image_encoder\.temp_blocks\.\d+\.)")


def strip_identity_temporal_extractor(sd: dict) -> dict:
    """`sd` without the temporal parts of its extractor, which must be exactly as scripts/inflate_model_to_temporal.py creates them:
    every temp_conv the identity over time, every temporal attention block's mlp.lin2 zero (weight and bias), pos_embed_temporal
    zero.  The extractor then computes what the 2-D extractor computes, so its renamed downsample convs are read under their 2-D
    keys.  Anything else (a trained temporal extractor) raises NotImplementedError: temporal_convs / temporal_attention
    extractors are not implemented."""
    renamed = {k: m for k in sd for m in [_CNX_DS_CONV.match(k)] if m}
    temporal = [k for k in sd if ".temp_conv." in k or _TEMP_BLOCK.match(k) or k == "detector.image_encoder.pos_embed_temporal"]
    if not renamed and not temporal:
        return sd

    def refuse(why: str):
        raise NotImplementedError(f"temporal extractor (temporal_convs / temporal_attention): {why}; only the 2-D extractor runs "
                                  "here, so a checkpoint whose temporal extractor parts differ from their inflated identity is not "
                                  "implemented")

    out = {k: v for k, v in sd.items() if k not in renamed and k not in temporal}
    for k, m in renamed.items():
        tc = sd.get(m.group(1) + ".temp_conv.weight")
        if not isinstance(tc, torch.Tensor) or tc.dim() != 5 or tc.shape[0] != tc.shape[1] or tc.shape[2] % 2 != 1 \
                or tc.shape[3:] != (1, 1):
            refuse(f"{m.group(1)} has no [C, C, t, 1, 1] temp_conv")
        ident = torch.zeros_like(tc)
        ident[:, :, tc.shape[2] // 2, 0, 0] = torch.eye(tc.shape[0], dtype=tc.dtype)
        if not torch.equal(tc, ident):
            refuse(f"{m.group(1)}.temp_conv is not the identity")
        out[f"{m.group(1)}.{m.group(2)}"] = sd[k]
    blocks = {_TEMP_BLOCK.match(k).group(1) for k in temporal if _TEMP_BLOCK.match(k)}
    for b in sorted(blocks):
        for leaf in ("mlp.lin2.weight", "mlp.lin2.bias"):
            v = sd.get(b + leaf)
            if not isinstance(v, torch.Tensor) or v.any():
                refuse(f"{b}{leaf} is not zero")
    pos = sd.get("detector.image_encoder.pos_embed_temporal")
    if pos is not None and pos.any():
        refuse("pos_embed_temporal is not zero")
    stray = [k for k in temporal if ".temp_conv." in k and k.replace(".temp_conv.", ".conv.") not in renamed]
    if stray:
        refuse(f"{stray[0]} belongs to no downsample conv")
    return out


def setup_model(card: dict, ckpt_path):
    from .model import Videoseal
    if not os.path.exists(ckpt_path):
        raise FileNotFoundError(f"Checkpoint path does not exist: {ckpt_path}")
    checkpoint = _safe_load(ckpt_path)
    checkpoint["model"] = strip_identity_temporal_extractor(checkpoint["model"])
    # scripts/inflate_model_to_temporal.py turns a 2-D checkpoint into a temporal one in place: it keeps the `args` (which still name
    # the 2-D preset) and only rewrites the U-Net's weights, so the weights say which conv_layer the U-Net has
    if is_temporal_state_dict(checkpoint["model"]):
        emb = card["embedder"]
        card = {**card, "embedder": {**emb, "params": {**emb["params"], "unet": {**emb["params"]["unet"], "conv_layer": "conv3d"}}}}
    spec = spec_from_card(card)
    model = Videoseal(spec)
    msg = model.load_state_dict(checkpoint["model"], strict=False)
    print(f"Model loaded successfully from {ckpt_path} with message: {msg}")
    return model


def _safe_load(ckpt_path):
    """torch.load with the safe unpickler only (weights_only=True, like utils/cfg.py:62,148 of the reference).  argparse.Namespace
    -- how training scripts save `args` next to `model` -- is allow-listed for the duration of the load: a plain attribute bag."""
    import argparse
    with torch.serialization.safe_globals([argparse.Namespace]):
        return torch.load(ckpt_path, map_location="cpu", weights_only=True)


def _plain(o):
    """checkpoint['args'] may be a dict, an argparse.Namespace or an OmegaConf container saved by the training script"""
    if hasattr(o, "items"):
        return {str(k): _plain(v) for k, v in o.items()}
    if hasattr(o, "__dict__") and not isinstance(o, (str, bytes)):
        return {str(k): _plain(v) for k, v in vars(o).items()}
    if isinstance(o, (list, tuple)):
        return [_plain(v) for v in o]
    return o


def get_config_from_checkpoint(ckpt_path) -> dict:
    """utils/cfg.py:50-85 of the reference: a raw training checkpoint carries its `args`; the embedder / extractor
    hyper-parameters are the presets named by args.embedder_model / args.extractor_model in the YAML files named by
    args.embedder_config / args.extractor_config (cwd first, then this package).  Returns a card-shaped dict."""
    # the safe unpickler only, like the reference (utils/cfg.py:62,148): a checkpoint is untrusted input.  Training scripts save
    # `args` as an argparse.Namespace, which is allow-listed for the duration of the load (a plain attribute bag, no code);
    # anything else the safe unpickler rejects (e.g. an OmegaConf container) is an error, never a silent full-pickle retry.
    checkpoint = _safe_load(ckpt_path)
    if "args" not in checkpoint:
        raise KeyError(f"{ckpt_path} holds no 'args': not a training checkpoint (use a model card for released weights)")
    args = _plain(checkpoint["args"])
    if not isinstance(args, dict):
        raise Exception("Expected logfile to contain params dictionary.")
    emb_cfg = yaml.safe_load(open(resolve_config_path(args.get("embedder_config", "configs/embedder.yaml"))))
    ext_cfg = yaml.safe_load(open(resolve_config_path(args.get("extractor_config", "configs/extractor.yaml"))))
    emb_model = args.get("embedder_model") or emb_cfg["model"]
    ext_model = args.get("extractor_model") or ext_cfg["model"]
    for name, cfg_, kind in ((emb_model, emb_cfg, "embedder"), (ext_model, ext_cfg, "extractor")):
        if name not in cfg_:
            raise NotImplementedError(f"{kind} preset '{name}' is not on the CUDA hot path (known: "
                                      f"{', '.join(k for k in cfg_ if k != 'model')})")
    return {"checkpoint_path": str(ckpt_path), "args": args,
            "embedder": {"model": emb_model, "params": emb_cfg[emb_model]},
            "extractor": {"model": ext_model, "params": ext_cfg[ext_model]}}


def setup_model_from_checkpoint(ckpt_path) -> "Videoseal":
    """utils/cfg.py:156-178 of the reference: a model-card name, or the path of a raw training checkpoint (.pth)."""
    ckpt_path = str(ckpt_path)
    if "baseline" in ckpt_path:
        raise NotImplementedError("baseline watermarkers (videoseal/models/baselines.py) are outside the CUDA hot path")
    if not ckpt_path.endswith(".pth") and "/" not in ckpt_path:
        return setup_model_from_model_card(ckpt_path)
    return setup_model(get_config_from_checkpoint(ckpt_path), ckpt_path)


def setup_model_from_model_card(model_card) -> "Videoseal":
    """`videoseal.load()`: card name (looked up in ./videoseal/cards, then in this package's cards/) or a Path to a YAML."""
    if model_card == "videoseal":
        model_card = DEFAULT_CARD
    if isinstance(model_card, str):
        candidates = [Path("videoseal/cards") / f"{model_card}.yaml", CARDS_DIR / f"{model_card}.yaml"]
        path = next((c for c in candidates if c.is_file()), None)
        if path is None:
            avail = sorted({c.stem for d in (Path("videoseal/cards"), CARDS_DIR) for c in d.glob("*.yaml")})
            print(f"Available model cards: {', '.join(avail)}")
            raise FileNotFoundError(f"Model card '{model_card}' not found")
    elif isinstance(model_card, Path):
        if not model_card.exists():
            raise FileNotFoundError(f"Model card file '{model_card}' not found")
        path = model_card
    else:
        raise TypeError("Model card must be a string or a Path object")
    with open(path, "r") as f:
        card = yaml.safe_load(f)
    cp = str(card["checkpoint_path"])
    if Path(cp).is_file():
        ckpt = Path(cp)
    elif (path.parent / cp).is_file():
        ckpt = path.parent / cp
    elif is_url(cp):
        ckpt = maybe_download_checkpoint(cp)
    else:
        raise RuntimeError(f"Path or uri {cp} is unknown or does not exist")
    return setup_model(card, ckpt)
