"""The temporal (conv3d) BatchNorm + ReLU U-Net embedders on the GPU, against the torch restatement of tests/temporal_oracle.py (equal to
the reference on tests/golden/temporal.pt, test_temporal_cpu.py).

- embed parity (pixels <= 1e-3 abs, the README tolerance): video chunks with a short last chunk, image mode at 1, 3 and 64 frames,
  a clip whose chunks straddle a 64-frame sub-batch, the RGB preset, and the u8 host streaming entry;
- grouping: permuting frames across groups leaves each group's output unchanged, permuting within a group changes it;
- each new kernel on the exact inputs it read (debug taps) against float64 with per-element bounds: the CUDA-core first layer
  (27 taps) and the 3x3x3 tensor-core convs at every width the U-Net runs them (16 / 32 / 64 / 128 / 384 channels, the last block's
  fused outc + tanh), with mutations that must leave the bounds: no zero padding in time between groups, and the t-1 / t+1
  taps swapped;
- the step names of the temporal plan;
- the reference's inflate script output for both extractor types (embeds like its 2-D source, detects exactly as it), and the float
  host pipeline with slices that are whole chunks.
"""
import ctypes as C
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import restate
from tests import temporal_oracle as to

pytestmark = pytest.mark.gpu

YUV, RGB = "unet_small2_yuv_quant_conv3d", "unet_small2_quant_conv3d"
_models = {}


def pair(preset, img_size=None):
    key = (preset, img_size)
    if key not in _models:
        _models[key] = to.model_pair(preset, device="cuda", img_size=img_size)
    return _models[key]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for m, _, _ in _models.values():
        m._release()
    _models.clear()


def _frames(n, seed, size=256):
    return torch.rand(n, 3, size, size, generator=torch.Generator().manual_seed(seed))


def _msgs(n, nbits, seed):
    return torch.randint(0, 2, (n, nbits), generator=torch.Generator().manual_seed(seed))


def _embed_both(model, orc, x, m, is_video, chunk=None, step=None):
    if chunk is not None:
        model.chunk_size = orc.chunk_size = chunk
    if step is not None:
        model.step_size = orc.step_size = step
    out = model.embed(x.cuda(), m, is_video=is_video)
    ref = orc.embed(x, m, is_video=is_video)
    return out, ref


@pytest.mark.parametrize("preset,n,chunk,step", [(YUV, 7, 3, 2), (YUV, 12, 4, 1), (RGB, 7, 3, 2)])
def test_video_chunks(preset, n, chunk, step):
    """full chunks and a short last chunk (7 frames, step 2: keys 0 2 4 | 6; 12 frames, step 1: 4 | 4 | 4)"""
    model, orc, spec = pair(preset)
    out, ref = _embed_both(model, orc, _frames(n, 1), _msgs(1, spec["nbits"], 2), True, chunk, step)
    err = (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()
    assert err <= 1e-3, err


@pytest.mark.parametrize("preset,n,size", [(YUV, 1, None), (YUV, 3, None), (RGB, 3, None), (YUV, 64, 128)])
def test_image_mode(preset, n, size):
    """image mode: the whole batch is one time axis (64 images at a 128 processing size keeps the CPU oracle short)"""
    model, orc, spec = pair(preset, size)
    s = size or 256
    out, ref = _embed_both(model, orc, _frames(n, 3, s), _msgs(n, spec["nbits"], 4), False)
    for k in ("imgs_w", "preds_w"):
        err = (out[k].cpu() - ref[k]).abs().max().item()
        assert err <= 1e-3, (k, err)


def test_chunks_straddle_sub_batch():
    """chunk_size 40, 72 key frames: groups of 40 and 32; the embed loop cuts sub-batches of 40 and 32 frames, never at frame 64"""
    model, orc, spec = pair(YUV, 128)
    out, ref = _embed_both(model, orc, _frames(72, 5, 128), _msgs(1, spec["nbits"], 6), True, 40, 1)
    err = (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()
    assert err <= 1e-3, err


def test_group_over_64_frames_raises():
    model, _, spec = pair(YUV, 128)
    with pytest.raises(NotImplementedError, match="64"):
        model.embed(_frames(65, 0, 128).cuda(), _msgs(65, spec["nbits"], 0), is_video=False)
    model.chunk_size = 65
    with pytest.raises(NotImplementedError, match="64"):
        model.embed(_frames(65, 0, 128).cuda(), _msgs(1, spec["nbits"], 0), is_video=True)


def test_u8_streaming_entry():
    """vsb_frames_host_u8 (streaming.embed_video_clip: lowres attenuation, x = u8 / 255, out = trunc(imgs_w * 255)) on 14 frames
    with step 2 and chunk_size 3 (groups 3 | 3 | 1) against the oracle on the same float frames"""
    from videoseal_b200 import streaming
    model, orc, spec = pair(YUV)
    model.chunk_size = orc.chunk_size = 3
    model.step_size = orc.step_size = 2
    g = torch.Generator().manual_seed(7)
    clip = torch.randint(0, 256, (14, 256, 256, 3), generator=g, dtype=torch.uint8)
    m = _msgs(1, spec["nbits"], 8)
    out = torch.from_numpy(streaming.embed_video_clip(model, clip.numpy(), m)).float()
    x = clip.permute(0, 3, 1, 2).float() / 255
    ref = orc.embed(x, m, is_video=True, lowres_attenuation=True)["imgs_w"]
    ref8 = (ref * 255).to(torch.uint8).permute(0, 2, 3, 1).float()   # trunc, as the u8 conversion
    d = (out - ref8).abs()
    assert d.max().item() <= 1, d.max().item()
    assert (d > 0).float().mean().item() < 0.05


def test_permutation_across_and_within_groups():
    """chunk_size 4, step 1, 8 frames: two groups.  Swapping the groups swaps their outputs (unchanged per group); swapping two frames
    of one group changes that group's output"""
    model, _, spec = pair(YUV)
    model.chunk_size, model.step_size = 4, 1
    x, m = _frames(8, 9), _msgs(1, spec["nbits"], 10)
    base = model.embed(x.cuda(), m, is_video=True)["imgs_w"].cpu()
    perm = torch.tensor([4, 5, 6, 7, 0, 1, 2, 3])
    across = model.embed(x[perm].cuda(), m, is_video=True)["imgs_w"].cpu()
    assert (across - base[perm]).abs().max().item() <= 1e-6
    within = torch.tensor([1, 0, 2, 3, 4, 5, 6, 7])
    w = model.embed(x[within].cuda(), m, is_video=True)["imgs_w"].cpu()
    assert (w[4:] - base[4:]).abs().max().item() <= 1e-6                 # the other group is untouched
    assert (w[within][:4] - base[:4]).abs().max().item() > 1e-3        # the reordered group's frames see other neighbours


# ---------------------------------------------------------------------------------------------------------------------------------
# per-kernel float64 checks on the plan's debug taps


def _groups(B, G):
    return [(g0, min(g0 + G, B)) for g0 in range(0, B, G)]


def conv3d_f64(x, w, G, mutation=None):
    """x [B, C, H, W] float64, w [N, C, 3, 3, 3]: the 3x3x3 conv of every group of G frames.  mutation 'nopad': one group over the
    whole batch (no zero frame between groups); 'swap': the t-1 and t+1 taps exchanged"""
    if mutation == "swap":
        w = w.flip(2)
    groups = [(0, x.shape[0])] if mutation == "nopad" else _groups(x.shape[0], G)
    return torch.cat([to.conv3d_frames(x[a:b], w) for a, b in groups], 0)


def _bn(sd, key):
    s = sd[key + ".weight"].double() / torch.sqrt(sd[key + ".running_var"].double() + 1e-5)
    return s, sd[key + ".bias"].double() - sd[key + ".running_mean"].double() * s


def _tap(model, name):
    return model.debug_tensor(name).double().permute(0, 3, 1, 2)        # NHWC -> NCHW


def _judge(got, ref, bound, what):
    r = ((got - ref).abs() / bound).max().item()
    assert r <= 1.0, f"{what}: max err / bound = {r:.3f}"
    return r


def _conv_checks(sd, G, key, x):
    """h = relu(bn(conv3d(x))) of block `key` against float64 with the bound 2^-10 * (|w| * |x| + |ref|) + 1e-5 (fp16 weights and
    output, fp32 accumulation); returns the float64 output, its bound, and each mutation's reference"""
    w = sd[key + ".double_conv.0.conv.weight"].double()
    s, b = _bn(sd, key + ".double_conv.1")
    ref = F.relu(conv3d_f64(x, w, G) * s[:, None, None] + b[:, None, None])
    mag = conv3d_f64(x.abs(), w.abs(), G) * s.abs()[:, None, None]
    bound = 2 ** -10 * (mag + ref.abs()) + 1e-5
    muts = {m: F.relu(conv3d_f64(x, w, G, m) * s[:, None, None] + b[:, None, None]) for m in ("nopad", "swap")}
    return ref, bound, muts


# (name of the block's input tap, block) for every width: C=16 @ 256 (inc's second conv reads first_h), 32 @ 128, 64 @ 64, 128 @ 32,
# 384 @ 32 (bottleneck: 128 + 256 message channels at nbits 256), 16 @ 256 (the last up block, fused outc + tanh)
BLOCKS = [("down0_conv", "down0", "downs.0.conv"), ("down1_conv", "down1", "downs.1.conv"), ("down2_conv", "down2", "downs.2.conv"),
          ("cat", "bott0", "bottleneck.model.0"), ("up1_conv", "up1", "ups.1.conv"), ("up2_conv", "up2", "ups.2.conv")]


def test_kernels_against_float64():
    model, orc, spec = pair(YUV)
    sd = orc.sd
    model.chunk_size, model.step_size = 4, 1
    B, G = 10, 4                                                        # groups 4 | 4 | 2 in one sub-batch
    x = _frames(B, 11)
    model.embed(x.cuda(), _msgs(1, spec["nbits"], 12), is_video=True)
    P = "embedder.unet."
    # ---- first layer: 27 taps on CUDA cores (fp32 weights; fp16 outputs)
    y = (restate.rgb_to_y(x).double() * 2 - 1)
    w = sd[P + "inc.double_conv.0.conv.weight"].double()
    s, b = _bn(sd, P + "inc.double_conv.1")
    ref = F.relu(conv3d_f64(y, w, G) * s[:, None, None] + b[:, None, None])
    bound = 2 ** -10 * ref.abs() + 1e-4
    h1 = _tap(model, "first_h")
    _judge(h1, ref, bound, "first_h")
    for mut in ("nopad", "swap"):
        mref = F.relu(conv3d_f64(y, w, G, mut) * s[:, None, None] + b[:, None, None])
        assert ((h1 - mref).abs() / bound).max().item() > 1.0, f"first_h: mutation {mut} not detected"
    wr = sd[P + "inc.res_conv.conv.weight"].double()
    rref = to.conv3d_frames(y, wr, sd[P + "inc.res_conv.conv.bias"].double())
    _judge(_tap(model, "first_r"), rref, 2 ** -10 * rref.abs() + 1e-4, "first_r")
    # ---- inc's second conv (16 channels @ 256): x = relu(bn(conv3d(first_h))) + first_r
    w2 = sd[P + "inc.double_conv.3.conv.weight"].double()
    s2, b2 = _bn(sd, P + "inc.double_conv.4")
    r0 = _tap(model, "first_r")
    ref = F.relu(conv3d_f64(h1, w2, G) * s2[:, None, None] + b2[:, None, None]) + r0
    bound = 2 ** -10 * (conv3d_f64(h1.abs(), w2.abs(), G) * s2.abs()[:, None, None] + ref.abs()) + 1e-5
    _judge(_tap(model, "inc"), ref, bound, "inc")
    # ---- every block's first 3x3x3 conv; the mutations on each
    for src, name, key in BLOCKS:
        xin = _tap(model, src)
        ref, bound, muts = _conv_checks(sd, G, P + key, xin)
        got = _tap(model, name + ".h")
        _judge(got, ref, bound, name + ".h")
        for mut, mref in muts.items():
            assert ((got - mref).abs() / bound).max().item() > 1.0, f"{name}.h: mutation {mut} not detected"
    # ---- the last block's second conv with the fused outc + tanh
    key = P + "ups.2.conv"
    h = _tap(model, "up2.h")
    r = _tap(model, "up2.r")
    w2 = sd[key + ".double_conv.3.conv.weight"].double()
    s2, b2 = _bn(sd, key + ".double_conv.4")
    blk = F.relu(conv3d_f64(h, w2, G) * s2[:, None, None] + b2[:, None, None]) + r
    d_ref = torch.tanh(F.conv2d(blk, sd[P + "outc.weight"].double(), sd[P + "outc.bias"].double()))
    blk_bound = 2 ** -10 * (conv3d_f64(h.abs(), w2.abs(), G) * s2.abs()[:, None, None] + blk.abs()) + 1e-5
    d_bound = F.conv2d(blk_bound, sd[P + "outc.weight"].double().abs()) + 1e-5
    _judge(model.debug_tensor("delta").double(), d_ref, d_bound, "delta")


def _step_names(model, x, m, is_video):
    from videoseal_b200 import _lib
    L = _lib.lib()
    L.vsb_profile_enable(1)
    try:
        model.embed(x, m, is_video=is_video)
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    return sorted({ln.split("\t")[0] for ln in buf.value.decode().splitlines() if ln.startswith("unet.")})


# the temporal steps of unet_small2_yuv_quant_conv3d at 256 and 128 ("unet." prefix omitted); the up-convs, down convs and 1x1 res
# convs keep their 2-D kernels
TEMPORAL_STEPS = {
    256: ["conv3x3x3+outc.16-16@256", "conv3x3x3.128-128@32", "conv3x3x3.16-16@256", "conv3x3x3.32-32@128", "conv3x3x3.384-384@32",
          "conv3x3x3.64-64@64", "first3x3x3", "tstack.128-384@32", "tstack.16-64@256", "tstack.32-128@128", "tstack.384-1152@32",
          "tstack.64-192@64"],
    128: ["conv3x3x3+outc.16-16@128", "conv3x3x3.128-128@16", "conv3x3x3.16-16@128", "conv3x3x3.32-32@64", "conv3x3x3.384-384@16",
          "conv3x3x3.64-64@32", "first3x3x3", "tstack.128-384@16", "tstack.16-64@128", "tstack.32-128@64", "tstack.384-1152@16",
          "tstack.64-192@32"],
}


@pytest.mark.parametrize("size", [256, 128])
def test_step_names(size):
    model, _, spec = pair(YUV, None if size == 256 else size)
    names = _step_names(model, _frames(3, 0, size).cuda(), _msgs(3, spec["nbits"], 0), False)
    temporal = [n[len("unet."):] for n in names if "3x3x3" in n or "tstack" in n]
    assert temporal == TEMPORAL_STEPS[size], temporal
    assert "unet.first" not in names and not [n for n in names if n.startswith("unet.conv3x3d")]


@pytest.mark.parametrize("ext", ["convnext_tiny", "sam_small"])
def test_inflate_script_output_equals_2d_model(ext):
    """the reference's inflate_model_to_temporal.py output for --extractor_type `ext` (restated from the record of the script's own
    output, tests/golden/temporal_inflate.pt: zero t-1 / t+1 U-Net taps, identity temporal extractor parts, args naming the 2-D presets)
    embeds like the 2-D model it came from and detects exactly as it does"""
    from videoseal_b200 import cfg
    card = to.preset_card(to.TWIN[YUV]) if ext == "convnext_tiny" else to.sam_card(to.TWIN[YUV])
    spec2 = restate.spec_from_card(card)
    sd2 = restate.synth_state_dict(spec2, to.SEED)
    rec = torch.load(os.path.join(to.ROOT, "tests", "golden", "temporal_inflate.pt"), weights_only=False)[ext]
    paths = []
    for tag, sd in (("twin2d", sd2), ("inflated", to.inflate_script(sd2, ext, rec))):
        paths.append(to.tmpdir() / f"{tag}_{ext}.pth")
        torch.save({"model": sd}, paths[-1])
    m2 = cfg.setup_model(card, str(paths[0])).eval().to("cuda")
    m3 = cfg.setup_model(card, str(paths[1])).eval().to("cuda")
    assert m3.temporal and not m2.temporal
    x, m = _frames(5, 13), _msgs(5, spec2["nbits"], 14)
    a = m2.embed(x.cuda(), m, is_video=False)["imgs_w"]
    b = m3.embed(x.cuda(), m, is_video=False)["imgs_w"]
    err = (a - b).abs().max().item()
    d2 = m2.detect(x.cuda(), is_video=False)["preds"]
    d3 = m3.detect(x.cuda(), is_video=False)["preds"]
    m2._release(), m3._release()
    assert err <= 1e-3, err
    assert torch.equal(d2, d3)


def test_float_host_pipeline():
    """vsb_embed_detect_host (host frames in slices of 16, then 48 frames, rounded up to whole chunks) with chunk_size 5 and step 2:
    slices of 20 and 50 frames, neither a multiple of the defaults; 26 frames = 13 key frames in groups 5 | 5 | 3 against the oracle,
    and its logits against detect() of its own output"""
    from videoseal_b200 import _lib
    model, orc, spec = pair(YUV)
    model.chunk_size = orc.chunk_size = 5
    model.step_size = orc.step_size = 2
    F_ = 26
    x = _frames(F_, 15).pin_memory()
    m = _msgs(1, spec["nbits"], 16)
    out = torch.empty_like(x).pin_memory()
    logits = torch.empty(F_, 1 + spec["nbits"]).pin_memory()
    m8 = m.to(torch.uint8).contiguous()
    _lib.check(_lib.lib().vsb_embed_detect_host(model._handle(), x.data_ptr(), m8.data_ptr(), 1, out.data_ptr(), logits.data_ptr(), F_,
                                                256, 256, 2, 0, 5, float(model.blender.scaling_i), float(model.blender.scaling_w),
                                                model._flags(restate._DEF_INTERP, False, (256, 256))))
    ref = orc.embed(x, m, is_video=True)["imgs_w"]
    err = (out - ref).abs().max().item()
    assert err <= 1e-3, err
    det = model.detect(out.cuda(), is_video=False)["preds"].cpu()
    assert (logits - det).abs().max().item() <= 1e-3 * det.abs().max().item()
