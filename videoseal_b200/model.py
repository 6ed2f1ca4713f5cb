"""`Videoseal`: host-side mirror of the reference's inference API (models/videoseal.py:258-428, models/wam.py:134-234)
whose compute is entirely in libvsb200.so (sm_100a kernels).  PyTorch is used for tensor plumbing only: allocating
outputs, holding the checkpoint, device placement and streams.

Drop-in surface kept (SURVEY.md §8b): `embed`, `detect`, `extract_message`, `get_random_msg`, mutable attributes
`blender.scaling_w/scaling_i`, `step_size`, `chunk_size`, `video_mode`, `img_size`, `clamp`, `attenuation` (may be set to
None), `embedder.yuv`, and the nn.Module verbs `.eval() .to(device) .compile()`.
"""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch
from torch import nn

from . import _lib

_DEF_INTERP = {"mode": "bilinear", "align_corners": False, "antialias": True}


def resize_flags(interpolation: dict, resizes: bool) -> int:
    """The resize bits of vsb_flags for the reference's `interpolation` dict, which it passes as F.interpolate(x, size=...,
    **interpolation) at both resize sites (wam.py:161-164, :183-185; videoseal.py:305, :329).  The reference calls F.interpolate only
    when the frames are not img_size x img_size (`resizes`); then this raises what F.interpolate raises for the dict: TypeError for
    a key it does not take, ValueError for align_corners with nearest / area, antialias with them, or a scale_factor next to the
    size.  Modes other than bilinear, bicubic, nearest and area raise NotImplementedError (as F.interpolate does for 4-D 'linear' /
    'trilinear'; 'nearest-exact' is not implemented here).  No device work: testable on the CPU."""
    if not resizes:
        return 0
    unknown = sorted(set(interpolation) - {"mode", "align_corners", "antialias", "scale_factor", "recompute_scale_factor"})
    if unknown:
        raise TypeError(f"interpolate() got an unexpected keyword argument '{unknown[0]}'")
    mode = interpolation.get("mode", "nearest")                      # F.interpolate's defaults
    align_corners = interpolation.get("align_corners")
    antialias = bool(interpolation.get("antialias", False))
    if mode in ("nearest", "area", "nearest-exact") and align_corners is not None:
        raise ValueError("align_corners option can only be set with the interpolating modes: linear | bilinear | bicubic | trilinear")
    if interpolation.get("scale_factor") is not None:
        raise ValueError("only one of size or scale_factor should be defined")
    if interpolation.get("recompute_scale_factor"):
        raise ValueError("recompute_scale_factor is not meaningful with an explicit size.")
    if antialias and mode not in ("bilinear", "bicubic"):
        raise ValueError("Anti-alias option is restricted to bilinear and bicubic modes and requires a 4-D tensor as input")
    if mode not in _lib.RESIZE_MODES:
        raise NotImplementedError(f"interpolation mode {mode!r} is not implemented (bilinear, bicubic, nearest, area)")
    f = _lib.RESIZE_MODES[mode] << _lib.FLAG_RESIZE_MODE_SHIFT
    if align_corners:
        f |= _lib.FLAG_RESIZE_ALIGN_CORNERS
    if not antialias:
        f |= _lib.FLAG_RESIZE_NO_AA
    return f


def native_desc(spec: dict) -> _lib.ModelDesc:
    """vsb_model_desc of `spec` (cfg.spec_from_card)"""
    d = _lib.ModelDesc()
    d.nbits, d.hidden, d.img_size, d.yuv = spec["nbits"], spec["hidden"], spec["img_size"], int(spec["yuv"])
    u = spec.get("unet")          # a HiDDeN, DVMark or VAE embedder spec leaves the U-Net fields zero but its RGB channels
    if u is None:
        d.unet_in_ch, d.unet_out_ch = 3, 3
    else:
        d.unet_in_ch, d.unet_out_ch, d.unet_levels = u["in_channels"], u["out_channels"], len(u["z"])
        for i, z in enumerate(u["z"]):
            d.unet_z[i] = z
        d.unet_num_blocks = u["num_blocks"]
        acts, norms = {"relu": 0, "silu": 1}, {"batch": 0, "rms": 1}
        if u["activation"] not in acts or not any(u["normalization"].startswith(k) for k in norms):
            raise NotImplementedError(f"U-Net activation/normalization {u['activation']}/{u['normalization']} not implemented")
        d.unet_act = acts[u["activation"]]
        d.unet_norm = 0 if u["normalization"].startswith("batch") else 1
        d.unet_last_tanh = int(u["last_tanh"])
    cn = spec.get("convnext")     # a SAM-ViT spec leaves the ConvNeXt fields zero
    if cn is not None:
        for i in range(4):
            d.ext_depths[i], d.ext_dims[i] = cn["depths"][i], cn["dims"][i]
        d.ext_stem_stride = cn["stem_stride"]
    d.jnd_in_ch, d.jnd_out_ch = spec["jnd"]
    return d


def native_vit_desc(vit: dict) -> _lib.VitDesc:
    """vsb_vit_desc of spec['vit'] (cfg.spec_from_card)"""
    v = _lib.VitDesc()
    v.embed_dim, v.depth, v.num_heads = vit["embed_dim"], vit["depth"], vit["num_heads"]
    v.patch_size, v.window_size = vit["patch_size"], vit["window_size"]
    v.global_mask = sum(1 << i for i in set(vit["global_attn_indexes"]) if 0 <= i < 32)
    v.mlp_dim, v.out_chans = vit["mlp_dim"], vit["out_chans"]
    v.qkv_bias, v.use_rel_pos = int(vit["qkv_bias"]), int(vit["use_rel_pos"])
    return v


def native_hidden_desc(h: dict, embedder: bool) -> _lib.HiddenDesc:
    """vsb_hidden_desc of spec['hidden_encoder'] / spec['hidden_decoder'] (cfg.spec_from_card): the encoder's conv_bns hold
    num_blocks ConvBNRelu, the decoder's layers num_blocks + 1"""
    v = _lib.HiddenDesc()
    v.z_channels, v.num_layers = h["z_channels"], h["num_blocks"] + (0 if embedder else 1)
    v.norm = {"batch": 0, "group": 1}[h["normalization"]]
    v.act = {"relu": 0, "gelu": 1}[h["activation"]]
    v.last_tanh = int(h.get("last_tanh", False))
    return v


def native_vae_desc(v: dict) -> _lib.VaeDesc:
    """vsb_vae_desc of spec['vae_encoder'] (cfg.spec_from_card)"""
    d = _lib.VaeDesc()
    d.in_ch, d.out_ch, d.ch, d.levels = v["in_channels"], v["out_ch"], v["ch"], len(v["ch_mult"])
    for i, m in enumerate(v["ch_mult"][:6]):
        d.ch_mult[i] = m
    d.num_res_blocks, d.z_channels, d.tanh_out = v["num_res_blocks"], v["z_channels"], int(v["tanh_out"])
    return d


def delta_channels(spec: dict) -> int:
    """channels of the embedder's output (the U-Net's or the VAE decoder's out channels; 3 for a HiDDeN or DVMark encoder)"""
    if "vae_encoder" in spec:
        return spec["vae_encoder"]["out_ch"]
    return spec["unet"]["out_channels"] if "unet" in spec else 3


def embedder_in_channels(spec: dict) -> int:
    if "vae_encoder" in spec:
        return spec["vae_encoder"]["in_channels"]
    return spec["unet"]["in_channels"] if "unet" in spec else 3


def trunk_map(spec: dict) -> int:
    """side of the extractor trunk's output map: img_size / 16 tokens for a SAM-ViT, img_size / 32 for the ConvNeXt trunks"""
    return spec["img_size"] // (16 if "vit" in spec else 32)


def _create(spec: dict):
    """Native handle of `spec` without weights or a device.  vsb_model_create, vsb_model_set_unet_temporal,
    vsb_model_set_hidden_embedder / _extractor, vsb_model_set_dvmark_embedder / _extractor, vsb_model_set_vae_embedder, vsb_model_set_vit_extractor and vsb_model_set_pixel_decoder check every rule the kernels place on the model's geometry; a
    model they do not implement raises NotImplementedError."""
    L = _lib.lib()
    if "hidden_encoder" not in spec and "dvmark_encoder" not in spec and "vae_encoder" not in spec and not spec["unet"]["z"]:
        # the descriptor of a U-Net without levels looks like one a HiDDeN embedder completes: reject it here, at load
        raise RuntimeError("libvsb200 error -1: unet levels: a U-Net needs 2 to 6 levels (z_channels_mults is empty)")
    h = C.c_void_p()
    _lib.check(L.vsb_model_create(C.byref(native_desc(spec)), C.byref(h)))
    pd = spec.get("pixel_decoder", {"pixelwise": False})
    f = pd["upscale_stages"] if pd["pixelwise"] else None
    rc = L.vsb_model_set_unet_temporal(h, 1) if spec.get("unet", {}).get("temporal", False) else 0
    if rc == 0 and "hidden_encoder" in spec:
        rc = L.vsb_model_set_hidden_embedder(h, C.byref(native_hidden_desc(spec["hidden_encoder"], True)))
    if rc == 0 and "dvmark_encoder" in spec:
        rc = L.vsb_model_set_dvmark_embedder(h, int(spec["dvmark_encoder"]["nbits"]))
    if rc == 0 and "vae_encoder" in spec:
        rc = L.vsb_model_set_vae_embedder(h, C.byref(native_vae_desc(spec["vae_encoder"])))
    if rc == 0 and "hidden_decoder" in spec:
        rc = L.vsb_model_set_hidden_extractor(h, C.byref(native_hidden_desc(spec["hidden_decoder"], False)))
    if rc == 0 and "dvmark_decoder" in spec:
        rc = L.vsb_model_set_dvmark_extractor(h, int(spec["dvmark_decoder"]["nbits"]))
    if rc == 0 and "vit" in spec:
        rc = L.vsb_model_set_vit_extractor(h, C.byref(native_vit_desc(spec["vit"])))
    if rc == 0 and f:
        rc = L.vsb_model_set_pixel_decoder(h, len(f), (C.c_int32 * len(f))(*f), 1)
    if rc != 0:
        L.vsb_model_destroy(h)
    _lib.check(rc)
    return h


def check_native(spec: dict) -> None:
    """Load-time dry run: the native library implements `spec` (no GPU needed)."""
    _lib.lib().vsb_model_destroy(_create(spec))


class Blender:
    """models/blender.py: only the additive method is on the hot path (all shipped cards)."""
    AVAILABLE_BLENDING_METHODS = ["additive"]

    def __init__(self, scaling_i: float, scaling_w: float, method: str = "additive"):
        if method != "additive":
            raise NotImplementedError(f"blending method '{method}' is not implemented")
        self.scaling_i, self.scaling_w, self.method = scaling_i, scaling_w, method


class JND:
    """modules/jnd.py stand-in: `heatmaps()` runs the fused CUDA kernel."""

    def __init__(self, owner: "Videoseal", in_channels: int, out_channels: int):
        self._owner, self.in_channels, self.out_channels = owner, in_channels, out_channels

    def to(self, *a, **k):
        return self

    def heatmaps(self, imgs: torch.Tensor) -> torch.Tensor:
        m = self._owner
        x = m._to_dev(imgs)
        out = torch.empty((x.shape[0], self.out_channels, x.shape[2], x.shape[3]), device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().vsb_jnd_heatmaps(m._handle(), x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[2], x.shape[3],
                                               m._stream()))
        return out.to(imgs.device)


class _Embedder:
    """models/embedder.py:130-165 UnetEmbedder seam: forward(imgs_res RGB [B,3,S,S] in [0,1], msgs [B,K]) -> delta"""

    def __init__(self, owner: "Videoseal"):
        self._owner = owner

    # the colour handling is baked into the native first layer (RGB -> Y fused): changing it rebuilds the native handle
    @property
    def yuv(self) -> bool:
        return bool(self._owner.spec["yuv"])

    @yuv.setter
    def yuv(self, v: bool):
        m = self._owner
        if bool(v) != bool(m.spec["yuv"]):
            want = 1 if v else 3
            if embedder_in_channels(m.spec) != want:
                raise ValueError(f"embedder.yuv={bool(v)} needs an embedder with {want} input channel(s); this checkpoint has "
                                 f"{embedder_in_channels(m.spec)}")
            m._respec(yuv=bool(v))

    def get_random_msg(self, bsz: int = 1, nb_repetitions: int = 1) -> torch.Tensor:
        nbits = self._owner.spec["nbits"]
        if nb_repetitions != 1:   # modules/msg_processor.py:43-57
            assert nbits % nb_repetitions == 0
            aux = torch.randint(0, 2, (bsz, nbits // nb_repetitions))
            return aux.unsqueeze(1).repeat(1, nb_repetitions, 1).view(bsz, nbits)
        return torch.randint(0, 2, (bsz, nbits))

    def __call__(self, imgs_res: torch.Tensor, msgs: torch.Tensor) -> torch.Tensor:
        m = self._owner
        x = m._to_dev(imgs_res)
        S = m.spec["img_size"]
        assert x.shape[1:] == (3, S, S), "embedder seam takes RGB frames at processing size (Y extraction is fused)"
        mm = m._msgs_u8(msgs)
        out = torch.empty((x.shape[0], delta_channels(m.spec), S, S), device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().vsb_embedder_forward(m._handle(), x.data_ptr(), mm.data_ptr(), mm.shape[0], out.data_ptr(),
                                                   x.shape[0], m._stream()))
        return out


class _Detector:
    """models/extractor.py:140-167 ConvnextExtractor seam: forward(imgs [B,3,S,S] in [0,1]) -> logits [B,1+K] (pixel-wise
    extractors: maps [B,1+K,S,S])"""

    def __init__(self, owner: "Videoseal"):
        self._owner = owner

    def __call__(self, imgs_res: torch.Tensor) -> torch.Tensor:
        return self._owner._detect_dev(self._owner._to_dev(imgs_res), 0)


class Videoseal(nn.Module):
    def __init__(self, spec: dict):
        super().__init__()
        self.spec = spec
        # checkpoint tensors live in a plain dict (not nn.Parameters): the network is executed by the native library
        self._sd: dict = {}
        self._native = None          # (device_index, ctypes handle)
        self._dev = torch.device("cpu")
        self._anchor = nn.Parameter(torch.zeros(1), requires_grad=False)  # lets `.to()` / `.device` behave like a module
        self.blender = Blender(spec["scaling_i"], spec["scaling_w"])
        self._attenuation: Optional[JND] = JND(self, *spec["jnd"]) if spec["jnd"][0] else None
        self.clamp = True
        self.chunk_size, self.step_size = spec["chunk_size"], spec["step_size"]
        self.video_mode = "repeat"
        self.lowres_attenuation = False
        self.embedder = _Embedder(self)
        self.detector = _Detector(self)

    # ------------------------------------------------------------------ attributes the native handle bakes in
    # (ModelDesc of vsb_model_create): assigning them rebuilds the handle on the next call instead of being a silent no-op
    def _respec(self, **changes):
        self.spec = {**self.spec, **changes}
        self._release()

    @property
    def img_size(self) -> int:
        return self.spec["img_size"]

    @img_size.setter
    def img_size(self, v: int):
        v = int(v)
        if v != self.spec["img_size"]:
            if v <= 0 or v % 128 != 0:
                raise ValueError(f"img_size={v}: the native path needs a processing size that is a positive multiple of 128")
            pos = self._sd.get("detector.image_encoder.pos_embed")
            if "vit" in self.spec and pos is not None and pos.dim() == 4 and pos.shape[1] != v // 16:
                # the reference fails here too (a shape error adding pos_embed in ImageEncoderViT.forward, vit.py:113-115)
                raise ValueError(f"img_size={v}: this ViT extractor's pos_embed is a {pos.shape[1]} x {pos.shape[2]} grid, "
                                 f"img_size / 16 = {v // 16} does not match")
            check_native({**self.spec, "img_size": v})
            self._respec(img_size=v)

    @property
    def attenuation(self) -> Optional[JND]:
        return self._attenuation

    @attenuation.setter
    def attenuation(self, jnd):
        """None switches the attenuation off (wam.py:196); a JND (ours or the reference's modules/jnd.py object: anything with
        in_channels / out_channels in {1, 3}) switches it on with that channel configuration"""
        if jnd is None:
            self._attenuation = None
            return
        cin, cout = int(getattr(jnd, "in_channels", 0)), int(getattr(jnd, "out_channels", 0))
        if cin not in (1, 3) or cout not in (1, 3):
            raise ValueError("attenuation must be None or a JND with in_channels / out_channels in {1, 3}")
        if (cin, cout) != tuple(self.spec["jnd"]):
            self._respec(jnd=(cin, cout))
        self._attenuation = jnd if isinstance(jnd, JND) and jnd._owner is self else JND(self, cin, cout)

    # ------------------------------------------------------------------ nn.Module plumbing
    @property
    def device(self) -> torch.device:
        return self._anchor.device

    def load_state_dict(self, state_dict, strict: bool = False):
        self._sd = {k: v.detach().to(torch.float32).cpu().contiguous() for k, v in state_dict.items()
                    if isinstance(v, torch.Tensor) and not k.endswith("num_batches_tracked")}
        self._release()
        return "<All keys matched successfully>" if self._sd else "<empty state dict>"

    def state_dict(self, *a, **k):
        return dict(self._sd)

    def compile(self, *a, **k):   # reference: nn.Module.compile only wraps forward(); embed/detect are unaffected
        return self

    def forward(self, *a, **k):
        raise NotImplementedError("training-time forward() is outside the inference hot path; use embed()/detect()")

    def _release(self):
        if self._native is not None:
            _lib.lib().vsb_model_destroy(self._native[1])
            self._native = None

    def __del__(self):
        try:
            self._release()
        except Exception:
            pass

    def _handle(self):
        dev = self.device
        if dev.type != "cuda":
            raise RuntimeError("videoseal_b200 runs on an NVIDIA H100 (sm_90a) only: call model.to('cuda') first; "
                               "there is no CPU fallback")
        idx = dev.index if dev.index is not None else torch.cuda.current_device()
        if self._native is not None and self._native[0] == idx:
            return self._native[1]
        self._release()
        L = _lib.lib()
        h = _create(self.spec)
        try:
            temporal, dvmark = self.temporal, self.dvmark
            for k, v in self._sd.items():
                # 5-D tensors: only the Conv3d weights of a temporal U-Net or a DVMark embedder and of a DVMark extractor are read
                if k.startswith(("attenuation.", "rgb2yuv.")) or (v.dim() > 4 and not (temporal and k.startswith("embedder.unet."))
                                                                   and not (dvmark and k.startswith("detector.layers."))):
                    continue
                shape = (C.c_int64 * max(1, v.dim()))(*v.shape)
                _lib.check(L.vsb_model_set_tensor(h, k.encode(), v.data_ptr(), shape, v.dim()))
            _lib.check(L.vsb_model_finalize(h, idx))
        except Exception:
            L.vsb_model_destroy(h)
            raise
        self._native = (idx, h)
        return h

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _to_dev(self, x: torch.Tensor) -> torch.Tensor:
        return x.to(device=self.device, dtype=torch.float32).contiguous()

    def _msgs_u8(self, msgs: torch.Tensor) -> torch.Tensor:
        if msgs.dim() != 2 or msgs.shape[1] != self.spec["nbits"]:
            raise ValueError(f"msgs must be [B, {self.spec['nbits']}], got {tuple(msgs.shape)}")
        # thresholded on the side the tensor lives on: a host tensor (the usual case) costs one small H2D copy and no device kernel
        return (msgs > 0.5).to(torch.uint8).contiguous().to(self.device)

    def _flags(self, interpolation: dict, lowres: bool = False, hw: Optional[tuple] = None) -> int:
        """vsb_flags of an embed / detect call on H x W frames (hw; None: as if they were resized)"""
        S = self.spec["img_size"]
        f = resize_flags(interpolation, hw is None or tuple(hw) != (S, S))
        if self.clamp:
            f |= _lib.FLAG_CLAMP
        if lowres:
            f |= _lib.FLAG_LOWRES_ATTN
        if self.attenuation is None:
            f |= _lib.FLAG_NO_ATTENUATION
        return f

    # ------------------------------------------------------------------ public API
    def get_random_msg(self, bsz: int = 1, nb_repetitions: int = 1) -> torch.Tensor:
        return self.embedder.get_random_msg(bsz, nb_repetitions)

    @torch.no_grad()
    def embed(self, imgs: torch.Tensor, msgs: torch.Tensor = None, is_video: bool = True, interpolation: dict = _DEF_INTERP,
              lowres_attenuation: bool = False) -> dict:
        """models/videoseal.py:258-350 (video) / models/wam.py:134-204 (images)."""
        if imgs.dim() != 4 or imgs.shape[1] != 3:
            raise ValueError("imgs must be [F, 3, H, W]")
        F_, H, W = imgs.shape[0], imgs.shape[2], imgs.shape[3]
        flags = self._flags(interpolation, lowres_attenuation, (H, W))
        if msgs is None:
            msgs = self.get_random_msg(F_ if not is_video else 1)
        elif is_video:
            assert msgs.shape[0] == 1, "Message should be unique"
        x = self._to_dev(imgs)
        mm = self._msgs_u8(msgs)
        if not is_video and mm.shape[0] != F_:
            raise ValueError("image mode needs one message per image")
        step = self.step_size if is_video else 1
        imgs_w = torch.empty_like(x)
        preds_w = None
        if not is_video:
            pc = delta_channels(self.spec)
            if self.attenuation is not None:       # hmaps * preds_w broadcasts to max(out_channels) channels (wam.py:189-193)
                pc = max(pc, self.attenuation.out_channels)
            preds_w = torch.empty((F_, pc, H, W), device=x.device, dtype=torch.float32)
        _lib.check(_lib.lib().vsb_embed(
            self._handle(), x.data_ptr(), mm.data_ptr(), mm.shape[0], imgs_w.data_ptr(),
            preds_w.data_ptr() if preds_w is not None else None, F_, H, W, step, _lib.VIDEO_MODES[self.video_mode],
            self._chunk_keys(is_video, F_), float(self.blender.scaling_i), float(self.blender.scaling_w), flags,
            self._stream()))
        if is_video:
            return {"imgs_w": imgs_w.to(imgs.device), "msgs": msgs[0:1].repeat(F_, 1)}
        return {"msgs": msgs, "preds_w": preds_w.to(imgs.device), "imgs_w": imgs_w.to(imgs.device)}

    @property
    def temporal(self) -> bool:
        """True when the embedder's 3x3x3 convs mix the key frames of one embedder call: a temporal U-Net (unet.conv_layer
        'conv3d') or a DVMark embedder"""
        return bool(self.spec.get("unet", {}).get("temporal", False)) or "dvmark_encoder" in self.spec

    def _chunk_keys(self, is_video: bool, num_frames: int) -> int:
        """vsb_embed's chunk_keys: key frames per reference embedder call.  A video call is one chunk of chunk_size key frames
        (videoseal.py:292-320); in image mode the whole batch is one call (wam.py:134-204), which matters only to a temporal
        U-Net or a DVMark embedder.  A temporal group must fit one 64-frame sub-batch."""
        keys = int(self.chunk_size) if is_video or not self.temporal else int(num_frames)
        if self.temporal and keys > 64:
            what = f"chunk_size={keys}" if is_video else f"image mode with {keys} images"
            net = "DVMark embedder" if "dvmark_encoder" in self.spec else "temporal U-Net"
            raise NotImplementedError(f"{net}: {what} puts more than 64 frames in one 3x3x3 conv group; at most 64 are "
                                      "implemented")
        return keys

    @property
    def dvmark(self) -> bool:
        """True for a DVMark extractor: its 3x3x3 convs mix the frames of one detector call"""
        return "dvmark_decoder" in self.spec

    def _detect_group(self, is_video: bool, num_frames: int) -> int:
        """vsb_detect_grouped's group: frames per reference detector call.  A video is detected in chunks of chunk_size frames
        (videoseal.py:373-379), so a clip shorter than chunk_size is one call of all its frames; in image mode the whole batch is
        one call (wam.py:206-234).  This matters only to a DVMark extractor, whose group must fit one 64-frame sub-batch."""
        g = min(int(self.chunk_size), int(num_frames)) if is_video else int(num_frames)
        if self.dvmark and g > 64:
            what = f"chunk_size={g}" if is_video else f"image mode with {g} images"
            raise NotImplementedError(f"DVMark extractor: {what} puts more than 64 frames in one 3x3x3 conv group; at most 64 are "
                                      "implemented")
        return g

    @property
    def pixelwise(self) -> bool:
        """True when detect() returns per-pixel maps [F, 1+K, P, P] (pixel_decoder.pixelwise of the card)."""
        return bool(self.spec.get("pixel_decoder", {}).get("pixelwise", False))

    def _detect_dev(self, x: torch.Tensor, flags: int, group: Optional[int] = None) -> torch.Tensor:
        """vsb_detect_grouped in groups of `group` frames (None: the whole batch is one detector call)"""
        shape = (x.shape[0], 1 + self.spec["nbits"])
        if self.pixelwise:   # trunk map (img_size / 32, a ViT's img_size / 16) x the product of the stage factors
            P = trunk_map(self.spec)
            for f in self.spec["pixel_decoder"]["upscale_stages"]:
                P *= f
            shape += (P, P)
        out = torch.empty(shape, device=x.device, dtype=torch.float32)
        g = self._detect_group(False, x.shape[0]) if group is None else group
        _lib.check(_lib.lib().vsb_detect_grouped(self._handle(), x.data_ptr(), out.data_ptr(), x.shape[0], x.shape[2], x.shape[3], g,
                                                 flags, self._stream()))
        return out

    @torch.no_grad()
    def detect(self, imgs: torch.Tensor, is_video: bool = True, interpolation: dict = _DEF_INTERP) -> dict:
        """models/videoseal.py:352-388; the chunk loop is internal to the library (only a DVMark extractor mixes the frames of a
        chunk)."""
        if not is_video:
            interpolation = _DEF_INTERP       # the reference drops `interpolation` on this branch (videoseal.py:374)
        flags = resize_flags(interpolation, tuple(imgs.shape[-2:]) != (self.img_size, self.img_size))
        preds = self._detect_dev(self._to_dev(imgs), flags, self._detect_group(is_video, imgs.shape[0]))
        return {"preds": preds.to(imgs.device)}

    def extract_message(self, imgs: torch.Tensor, aggregation: str = "avg",
                        interpolation: dict = {"mode": "bilinear", "align_corners": False, "antialias": False}) -> torch.Tensor:
        """models/videoseal.py:390-428"""
        preds = self.detect(imgs, is_video=True, interpolation=interpolation)["preds"]
        bit_preds = preds[:, 1:]
        if aggregation is None:
            decoded = bit_preds
        elif aggregation == "avg":
            decoded = bit_preds.mean(dim=0)
        elif aggregation == "squared_avg":
            decoded = (bit_preds * bit_preds.abs()).mean(dim=0)
        elif aggregation == "l1norm_avg":
            decoded = (bit_preds * torch.norm(bit_preds, p=1, dim=1).unsqueeze(1)).mean(dim=0)
        elif aggregation == "l2norm_avg":
            decoded = (bit_preds * torch.norm(bit_preds, p=2, dim=1).unsqueeze(1)).mean(dim=0)
        else:
            raise ValueError(f"unknown aggregation {aggregation}")
        return (decoded > 0).squeeze().unsqueeze(0)

    # ------------------------------------------------------------------ test seam
    def debug_tensor(self, name: str) -> torch.Tensor:
        """Intermediate activation of the most recent sub-batch as an fp32 NHWC tensor (tests only)."""
        L = _lib.lib()
        shape = (C.c_int64 * 4)()
        n = L.vsb_debug_get_tensor(self._handle(), name.encode(), None, 0, shape)
        if n < 0:
            raise KeyError(L.vsb_last_error().decode())
        out = torch.empty(list(shape), dtype=torch.float32)
        n = L.vsb_debug_get_tensor(self._handle(), name.encode(), out.data_ptr(), out.numel(), shape)
        if n < 0:
            raise RuntimeError(L.vsb_last_error().decode())
        return out
