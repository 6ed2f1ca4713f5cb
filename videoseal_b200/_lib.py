"""ctypes binding of libvsb200.so (include/vsb200.h).  Fails loudly when the library is missing: there is no
CPU or PyTorch fallback in this package."""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# VSB200_LIB selects another build of the library (e.g. one compiled from an earlier revision, to compare outputs)
LIB_PATH = os.environ.get("VSB200_LIB") or os.path.join(_HERE, "libvsb200.so")

EXPORTS = [
    "vsb_last_error", "vsb_version", "vsb_model_create", "vsb_model_set_tensor", "vsb_model_set_pixel_decoder", "vsb_model_finalize",
    "vsb_model_destroy", "vsb_embed", "vsb_embedder_forward", "vsb_detect", "vsb_jnd_heatmaps", "vsb_embed_host",
    "vsb_detect_host", "vsb_embed_detect_host", "vsb_frames_host_u8", "vsb_launch_count", "vsb_profile_enable", "vsb_profile_read", "vsb_debug_get_tensor", "vsb_debug_keep_inputs", "vsb_debug_plan_gemms",
    "vsb_debug_conv",
    "vsb_debug_resample_table", "vsb_debug_resample_table2", "vsb_debug_last_dispatch", "vsb_quality_workspace_bytes", "vsb_ssim", "vsb_model_set_vit_extractor",
    "vsb_augment_workspace_bytes", "vsb_augment", "vsb_model_set_unet_temporal", "vsb_model_set_hidden_embedder",
    "vsb_model_set_hidden_extractor", "vsb_model_set_dvmark_extractor", "vsb_detect_grouped",
    "vsb_model_set_dvmark_embedder", "vsb_model_set_vae_embedder",
]

FLAG_CLAMP, FLAG_LOWRES_ATTN, FLAG_NO_ATTENUATION, FLAG_RESIZE_NO_AA = 1, 2, 4, 8
FLAG_RESIZE_ALIGN_CORNERS, FLAG_RESIZE_MODE_SHIFT = 16, 5
# F.interpolate modes the resizes implement (vsb_resize_mode), in bits 5-6 of the flags
RESIZE_MODES = {"bilinear": 0, "bicubic": 1, "nearest": 2, "area": 3}
VIDEO_MODES = {"repeat": 0, "alternate": 1, "interpolate": 2}


class ModelDesc(C.Structure):
    _fields_ = [
        ("nbits", C.c_int32), ("hidden", C.c_int32), ("img_size", C.c_int32), ("yuv", C.c_int32),
        ("unet_in_ch", C.c_int32), ("unet_out_ch", C.c_int32), ("unet_levels", C.c_int32), ("unet_z", C.c_int32 * 6),
        ("unet_num_blocks", C.c_int32), ("unet_act", C.c_int32), ("unet_norm", C.c_int32), ("unet_last_tanh", C.c_int32),
        ("ext_depths", C.c_int32 * 4), ("ext_dims", C.c_int32 * 4), ("ext_stem_stride", C.c_int32),
        ("jnd_in_ch", C.c_int32), ("jnd_out_ch", C.c_int32),
    ]


class VitDesc(C.Structure):
    _fields_ = [
        ("embed_dim", C.c_int32), ("depth", C.c_int32), ("num_heads", C.c_int32), ("patch_size", C.c_int32),
        ("window_size", C.c_int32), ("global_mask", C.c_uint32), ("mlp_dim", C.c_int32), ("out_chans", C.c_int32),
        ("qkv_bias", C.c_int32), ("use_rel_pos", C.c_int32),
    ]


class HiddenDesc(C.Structure):
    _fields_ = [("z_channels", C.c_int32), ("num_layers", C.c_int32), ("norm", C.c_int32), ("act", C.c_int32), ("last_tanh", C.c_int32)]


class VaeDesc(C.Structure):
    _fields_ = [("in_ch", C.c_int32), ("out_ch", C.c_int32), ("ch", C.c_int32), ("levels", C.c_int32), ("ch_mult", C.c_int32 * 6),
                ("num_res_blocks", C.c_int32), ("z_channels", C.c_int32), ("tanh_out", C.c_int32)]


class ConvTest(C.Structure):
    _fields_ = [
        ("loader", C.c_int32), ("B", C.c_int32), ("IH", C.c_int32), ("IW", C.c_int32), ("C0", C.c_int32), ("C1", C.c_int32),
        ("R", C.c_int32), ("S", C.c_int32), ("stride", C.c_int32), ("pad", C.c_int32), ("pad_mode", C.c_int32),
        ("N", C.c_int32), ("epi", C.c_int32), ("act", C.c_int32), ("rows_per_sample", C.c_int32), ("block_n", C.c_int32),
        ("src0", C.c_void_p), ("src1", C.c_void_p), ("weights", C.c_void_p),
        ("bias", C.c_void_p), ("resid16", C.c_void_p), ("resid32", C.c_void_p),
        ("ln_w", C.c_void_p), ("ln_b", C.c_void_p),
        ("outc_w", C.c_void_p), ("outc_b", C.c_void_p), ("n_out", C.c_int32),
        ("out16", C.c_void_p), ("out32", C.c_void_p), ("delta", C.c_void_p), ("grn_stats", C.c_void_p),
        ("ld0", C.c_int32), ("ldw", C.c_int32), ("ld_out", C.c_int32),
        ("kernel", C.c_int32), ("kernel_ran", C.POINTER(C.c_int32)),
        ("grn_part", C.c_int32), ("w_samples", C.c_int32), ("longk_block_n", C.c_int32),
    ]


_lib = None


def lib():
    """Load the shared library (once).  Raises RuntimeError with build instructions if it is absent."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            f"{LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  videoseal_b200 has no CPU / PyTorch fallback.")
    L = C.CDLL(LIB_PATH)
    L.vsb_last_error.restype = C.c_char_p
    L.vsb_version.restype = C.c_int
    L.vsb_model_create.argtypes = [C.POINTER(ModelDesc), C.POINTER(C.c_void_p)]
    L.vsb_model_set_tensor.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.POINTER(C.c_int64), C.c_int32]
    L.vsb_model_set_pixel_decoder.argtypes = [C.c_void_p, C.c_int32, C.POINTER(C.c_int32), C.c_int32]
    L.vsb_model_set_vit_extractor.argtypes = [C.c_void_p, C.POINTER(VitDesc)]
    L.vsb_model_set_unet_temporal.argtypes = [C.c_void_p, C.c_int32]
    L.vsb_model_set_hidden_embedder.argtypes = [C.c_void_p, C.POINTER(HiddenDesc)]
    L.vsb_model_set_hidden_extractor.argtypes = [C.c_void_p, C.POINTER(HiddenDesc)]
    L.vsb_model_set_dvmark_extractor.argtypes = [C.c_void_p, C.c_int32]
    L.vsb_model_set_dvmark_embedder.argtypes = [C.c_void_p, C.c_int32]
    L.vsb_model_set_vae_embedder.argtypes = [C.c_void_p, C.POINTER(VaeDesc)]
    L.vsb_model_finalize.argtypes = [C.c_void_p, C.c_int32]
    L.vsb_model_destroy.argtypes = [C.c_void_p]
    L.vsb_model_destroy.restype = None
    L.vsb_embed.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                            C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32, C.c_void_p]
    L.vsb_embedder_forward.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_int32, C.c_void_p]
    L.vsb_detect.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.vsb_detect_grouped.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                                     C.c_void_p]
    L.vsb_jnd_heatmaps.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_void_p]
    L.vsb_embed_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                 C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32]
    L.vsb_detect_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.vsb_embed_detect_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                        C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32]
    L.vsb_frames_host_u8.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32,
                                     C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_float, C.c_int32]
    L.vsb_launch_count.argtypes = [C.c_int32]
    L.vsb_launch_count.restype = C.c_int64
    L.vsb_profile_enable.argtypes = [C.c_int32]
    L.vsb_profile_read.argtypes = [C.c_char_p, C.c_int64]
    L.vsb_profile_read.restype = C.c_int64
    L.vsb_debug_get_tensor.argtypes = [C.c_void_p, C.c_char_p, C.c_void_p, C.c_int64, C.POINTER(C.c_int64)]
    L.vsb_debug_get_tensor.restype = C.c_int64
    L.vsb_debug_keep_inputs.argtypes = [C.c_void_p, C.c_int32]
    L.vsb_debug_plan_gemms.argtypes = [C.c_void_p, C.c_char_p, C.c_int64]
    L.vsb_debug_plan_gemms.restype = C.c_int64
    L.vsb_debug_conv.argtypes = [C.POINTER(ConvTest), C.c_void_p]
    L.vsb_debug_resample_table.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int64]
    L.vsb_debug_resample_table2.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p,
                                            C.c_int64]
    L.vsb_debug_last_dispatch.argtypes = [C.c_void_p, C.POINTER(C.c_int32), C.c_int32]
    L.vsb_debug_last_dispatch.restype = C.c_int32
    L.vsb_quality_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.vsb_quality_workspace_bytes.restype = C.c_int64
    L.vsb_ssim.argtypes = [C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_float, C.c_void_p, C.c_void_p,
                           C.c_void_p, C.c_int64, C.c_void_p]
    L.vsb_augment_workspace_bytes.argtypes = [C.c_int32, C.c_int32, C.c_int32, C.c_int32]
    L.vsb_augment_workspace_bytes.restype = C.c_int64
    L.vsb_augment.argtypes = [C.c_int32, C.c_void_p, C.c_void_p, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32, C.c_int32,
                              C.POINTER(C.c_float), C.c_int32, C.c_void_p, C.c_void_p, C.c_int64, C.c_void_p]
    _lib = L
    return L


def check(rc: int):
    if rc != 0:
        msg = lib().vsb_last_error().decode("utf-8", "replace")
        if rc == -2:
            raise NotImplementedError(msg)
        raise RuntimeError(f"libvsb200 error {rc}: {msg}")
