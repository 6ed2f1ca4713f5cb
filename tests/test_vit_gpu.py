"""SAM-ViT extractors on the GPU (synthetic checkpoints: the videoseal_1.0 U-Net with the videoseal_0.0 card's `sam_small` block):
detect() against the CPU oracle, the attention kernel on its own inputs against float64, determinism, the C entry points, and
embed() unchanged by the extractor."""
import ctypes as C

import numpy as np
import pytest
import torch

from tests import vit_oracle as vo
from tests.vit_kernels import attention_bound, attention_f64

pytestmark = pytest.mark.gpu
AGGS = ("avg", "squared_avg", "l1norm_avg", "l2norm_avg")


@pytest.fixture(scope="module")
def pooled():
    model, orc, spec = vo.model_pair(False)
    yield model, orc, spec
    model._release()


def logits_contract(got, ref, what, v=3e-3, e=2.5e-2):
    """DESIGN.md §4, the ViT logits bound: the ConvNeXt contract's form (|d| <= e max(|ref|, 0.1 |ref|inf), |d|inf <= v |ref|inf,
    decisions exact above the 1e-2 |ref|inf margin) with e = 2.5e-2 and v = 3e-3: twelve blocks of five fp16-operand stages each
    land just above the ConvNeXt contract's 1e-2 / 1.5e-3 (measured on an H100 at 64 x 256^2: 1.23e-2 / 1.55e-3).  Frames
    down-scaled to 128 are held to the map bound (v = 5e-3, e = 5e-2; measured 4.8e-3 / 3.8e-2)."""
    got, ref = got.float().cpu(), ref.float()
    scale = ref.abs().max()
    d = (got - ref).abs()
    rel = (d / torch.maximum(ref.abs(), 0.1 * scale)).max().item()
    sure = ref.abs() > 1e-2 * scale
    flips = int(((got > 0) != (ref > 0))[sure].sum())
    print(f"[{what}] |d|inf / |ref|inf = {(d.max() / scale).item():.2e}, max elementwise rel = {rel:.2e}, flips = {flips}")
    assert (d.max() / scale).item() <= v, what
    assert rel <= e, what
    assert flips == 0, what


def map_bound(got, ref, what):
    """DESIGN.md §4 map bound of the pixel-wise maps, per frame"""
    got, ref = got.float().cpu(), ref.float()
    for f in range(ref.shape[0]):
        g, r = got[f], ref[f]
        ninf = r.abs().max().item()
        d = (g - r).abs()
        rel = (d / torch.maximum(r.abs(), torch.full_like(r, 0.1 * ninf))).max().item()
        flips = int(((g > 0) != (r > 0))[r.abs() > 1e-2 * ninf].sum())
        print(f"[{what}] frame {f}: |d|inf / |ref|inf = {d.max().item() / ninf:.2e}, max elementwise rel = {rel:.2e}, flips = {flips}")
        assert rel <= 5e-2 and d.max().item() <= 5e-3 * ninf and flips == 0, (what, f)


def test_detect_parity_pooled_full_batch(pooled):
    model, orc, spec = pooled
    x = torch.rand(64, 3, 256, 256, generator=torch.Generator().manual_seed(0))
    got = model.detect(x.cuda(), is_video=False)["preds"]
    assert got.shape == (64, 1 + spec["nbits"]) and got.dtype == torch.float32
    logits_contract(got, orc.detect(x, is_video=False)["preds"], "sam_small 64x256^2")
    # the neck output against the oracle's
    taps = {}
    vo.trunk_forward(orc.sd, spec, x[-1:] * 1.0, taps)
    neck = model.debug_tensor("vit.neck")[-1].permute(2, 0, 1)
    r = taps["neck"][0]
    assert (neck - r).abs().max().item() <= 2e-2 * r.abs().max().item()


def test_detect_against_the_reference_fixture(pooled):
    """tests/golden/vit.pt: what the unmodified reference computed (tests/make_golden_vit.py), pooled logits under the ViT bound and
    pixel-wise samples under the map bound's 5e-3 |ref|inf; the resized 384 x 480 frame's maps measured 5.3e-3 on an H100 and are held
    to 1e-2 (DESIGN.md §4)"""
    import os
    golden = torch.load(os.path.join(os.path.dirname(__file__), "golden", "vit.pt"), weights_only=False)["variants"]
    model, _, _ = pooled
    pw_model, _, _ = vo.model_pair(True)
    try:
        for name in ("img256", "img_resized", "vid"):
            for variant, m in (("sam_small", model), ("sam_small_pw", pw_model)):
                c = golden[variant]["cases"][name]
                x = torch.rand(*c["shape"], generator=torch.Generator().manual_seed(c["gen_seed"]))
                m.chunk_size = 2
                got = m.detect(x.cuda(), is_video=c["is_video"])["preds"].cpu()
                if variant == "sam_small":
                    logits_contract(got, c["logits"], f"fixture {name}")
                else:
                    s = got[:, ::8, ::16, ::16]
                    e = (s - c["maps_s"]).abs().max().item() / c["maps_s"].abs().max().item()
                    flips = int(((s > 0) != (c["maps_s"] > 0))[c["maps_s"].abs() > 1e-2 * c["maps_s"].abs().max()].sum())
                    print(f"[fixture pw {name}] sampled |d|inf / |ref|inf = {e:.2e}, flips = {flips}")
                    assert flips == 0 and e <= (1e-2 if name == "img_resized" else 5e-3), name
    finally:
        model.chunk_size = vo.spec_from_card(vo.vit_card())["chunk_size"]
        pw_model._release()


def test_each_block_against_the_oracle(pooled):
    """The residual stream after every block of the 12-block model against the oracle's blk{i} taps.  The plan reuses one stream
    buffer, so only the last block's tap exists; block k - 1 is read from the model of depth k, whose checkpoint is the same prefix
    (synth_state_dict draws the patch embedding, pos_embed and the blocks in order).  Measured on an H100: 5.4e-4 |ref|inf after the
    patch embedding (fp16 pixels and weights, K = 768), 7.5e-4 after block 0, at most 1.2e-3 over the 12 blocks: the error is that of
    the fp16 operands from the first GEMM on and grows slowly with depth.  Bounds: 1e-3 and 2e-3."""
    import torch.nn.functional as F
    model, orc, spec = pooled
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(9))
    taps = {}
    vo.trunk_forward(orc.sd, spec, x, taps)
    model.detect(x.cuda(), is_video=False)
    Q = vo.Q
    emb = F.conv2d(x * 2 - 1, orc.sd[Q + "patch_embed.proj.weight"], orc.sd[Q + "patch_embed.proj.bias"], stride=16).permute(0, 2, 3, 1)
    emb = emb + orc.sd[Q + "pos_embed"]
    e = (model.debug_tensor("vit.embed") - emb).abs().max().item() / emb.abs().max().item()
    print(f"[blocks] embed: |d|inf / |ref|inf = {e:.2e}")
    assert e <= 1e-3
    for k in range(1, 13):
        mk, ok_, _ = vo.model_pair(False, encoder={"depth": k})
        try:
            for key, v in ok_.sd.items():
                if key.startswith(Q + "blocks.") or key in (Q + "pos_embed", Q + "patch_embed.proj.weight"):
                    assert torch.equal(v, orc.sd[key]), key
            mk.detect(x.cuda(), is_video=False)
            got, ref = mk.debug_tensor(f"vit.blk{k - 1}"), taps[f"blk{k - 1}"]
            e = (got - ref).abs().max().item() / ref.abs().max().item()
            print(f"[blocks] blk{k - 1}: |d|inf / |ref|inf = {e:.2e}")
            assert e <= BLOCK_BOUND, k
        finally:
            mk._release()


BLOCK_BOUND = 2e-3


def test_window_of_1600_tokens_without_rel_pos():
    """without relative positions a window may exceed 32 tokens per side: 40 x 40 windows (25 key tiles) at img_size 640"""
    model, orc, spec = vo.model_pair(False, img_size=640, encoder={"window_size": 40, "global_attn_indexes": [], "use_rel_pos": False})
    try:
        x = torch.rand(2, 3, 640, 640, generator=torch.Generator().manual_seed(640))
        logits_contract(model.detect(x.cuda(), is_video=False)["preds"], orc.detect(x, is_video=False)["preds"], "window 40@640")
    finally:
        model._release()


@pytest.mark.parametrize("size", [128, 384, 512])
def test_detect_other_processing_sizes(size):
    model, orc, spec = vo.model_pair(False, img_size=size)
    try:
        x = torch.rand(3, 3, size, size, generator=torch.Generator().manual_seed(size))
        got = model.detect(x.cuda(), is_video=False)["preds"]
        logits_contract(got, orc.detect(x, is_video=False)["preds"], f"sam_small@{size}")
        # a resized frame: the resize runs first
        y = torch.rand(2, 3, 300, 340, generator=torch.Generator().manual_seed(size + 1))
        logits_contract(model.detect(y.cuda(), is_video=False)["preds"], orc.detect(y, is_video=False)["preds"], f"resized@{size}",
                        *((5e-3, 5e-2) if size == 128 else ()))
    finally:
        model._release()


def test_detect_parity_pixelwise():
    model, orc, spec = vo.model_pair(True, via_checkpoint=True)
    try:
        x = torch.rand(3, 3, 256, 256, generator=torch.Generator().manual_seed(5))
        got = model.detect(x.cuda(), is_video=False)["preds"]
        assert got.shape == (3, 1 + spec["nbits"], 256, 256)
        map_bound(got, orc.detect(x, is_video=False)["preds"], "sam_small_pw")
    finally:
        model._release()


# ---------------------------------------------------------------- the attention kernel on its own inputs

ATTN_CASES = {   # the model's only block (depth 1) is windowed or global, with or without the relative-position tables
    "win_rel": {"depth": 1, "global_attn_indexes": [], "use_rel_pos": True},
    "win_norel": {"depth": 1, "global_attn_indexes": [], "use_rel_pos": False},
    "global_rel": {"depth": 1, "global_attn_indexes": [0], "use_rel_pos": True},
    "global_norel": {"depth": 1, "global_attn_indexes": [0], "use_rel_pos": False},
    "win16_rel": {"depth": 1, "global_attn_indexes": [], "use_rel_pos": True, "window_size": 16},
}


@pytest.mark.parametrize("case", list(ATTN_CASES))
@pytest.mark.parametrize("size", [256, 512])
def test_attention_on_its_own_inputs(case, size):
    enc = ATTN_CASES[case]
    model, orc, spec = vo.model_pair(False, img_size=size, encoder=enc)
    try:
        B = 3 if size == 256 else 2
        x = torch.rand(B, 3, size, size, generator=torch.Generator().manual_seed(7))
        model.detect(x.cuda(), is_video=False)
        qkv = model.debug_tensor("vit.blk0.qkv")
        got = model.debug_tensor("vit.blk0.attn").double()
        G = size // 16
        n = G if enc["global_attn_indexes"] else int(enc.get("window_size", 8))
        sd = orc.sd
        rel = [sd[f"detector.image_encoder.blocks.0.attn.rel_pos_{a}"].half().float() for a in "hw"] if enc["use_rel_pos"] else [None, None]
        ref, a, se = attention_f64(qkv, 6, n, G, *rel)
        bound = attention_bound(ref, a, se)
        err = (got - ref).abs()
        print(f"[attn {case}@{size}] max |d| = {err.max().item():.3e}, max |d| / bound = {(err / bound).max().item():.3f}")
        assert bool((err <= bound).all()), (case, size)
        # the bound is tight enough to see the classic mistakes
        # (shifting the only window of a global block is a relabelling, invisible without rel-pos; with it, a real change)
        muts = (["shift"] if n < G or enc["use_rel_pos"] else []) + (["scaled", "transpose"] if enc["use_rel_pos"] else [])
        for m in muts:
            mref, _, _ = attention_f64(qkv, 6, n, G, *rel, mutate=m)
            assert bool((( got - mref).abs() > bound).any()), (case, size, m)
    finally:
        model._release()


# ---------------------------------------------------------------- determinism, video, host entry points, embed

def test_batch_split_and_repeat_are_bit_identical(pooled):
    model, _, _ = pooled
    x = torch.rand(70, 3, 256, 256, generator=torch.Generator().manual_seed(3)).cuda()
    full = model.detect(x, is_video=False)["preds"]
    assert torch.equal(full, model.detect(x, is_video=False)["preds"])
    for i in range(70):
        assert torch.equal(model.detect(x[i:i + 1], is_video=False)["preds"], full[i:i + 1]), i


def test_video_and_extract_message(pooled):
    model, orc, spec = pooled
    clip = torch.rand(7, 3, 240, 320, generator=torch.Generator().manual_seed(11))
    logits_contract(model.detect(clip.cuda(), is_video=True)["preds"], orc.detect(clip, is_video=True)["preds"], "video")
    p = orc.detect(clip, is_video=True, interpolation={"mode": "bilinear", "align_corners": False, "antialias": False})["preds"][:, 1:]
    aggregate = {"avg": p.mean(0), "squared_avg": (p * p.abs()).mean(0), "l1norm_avg": (p * p.abs().sum(1, keepdim=True)).mean(0),
                 "l2norm_avg": (p * p.norm(dim=1, keepdim=True)).mean(0)}
    for agg in AGGS:
        got = model.extract_message(clip.cuda(), agg).cpu().squeeze()
        ref = orc.extract_message(clip, agg).squeeze()
        # decisions exact wherever the aggregate is clear of zero (the 1e-2 margin of the logits contract)
        sure = aggregate[agg].abs() > 1e-2 * aggregate[agg].abs().max()
        print(f"[extract_message {agg}] {int((got != ref).sum())} of {got.numel()} bits differ, {int((~sure).sum())} within the margin")
        assert torch.equal(got[sure], ref[sure]), agg


def test_host_entry_points_match_device_path(pooled):
    from videoseal_b200 import _lib
    model, _, spec = pooled
    L = _lib.lib()
    g = torch.Generator().manual_seed(21)
    x = torch.rand(5, 3, 256, 256, generator=g)
    dev = model.detect(x.cuda(), is_video=False)["preds"].cpu()
    xh = np.ascontiguousarray(x.numpy())
    oh = np.empty((5, 1 + spec["nbits"]), dtype=np.float32)
    _lib.check(L.vsb_detect_host(model._handle(), xh.ctypes.data_as(C.c_void_p), oh.ctypes.data_as(C.c_void_p), 5, 256, 256, 0))
    assert torch.equal(torch.from_numpy(oh), dev)
    # embed + detect of the watermarked frames: logits equal to detect() of the imgs_w the same call returned
    m8 = np.ascontiguousarray(torch.randint(0, 2, (1, spec["nbits"]), generator=g).to(torch.uint8).numpy())
    iw = np.empty_like(xh)
    lg = np.empty_like(oh)
    _lib.check(L.vsb_embed_detect_host(model._handle(), xh.ctypes.data_as(C.c_void_p), m8.ctypes.data_as(C.c_void_p), 1,
                                       iw.ctypes.data_as(C.c_void_p), lg.ctypes.data_as(C.c_void_p), 5, 256, 256, 1, 0, 1, 1.0, 0.2, 0))
    assert torch.equal(torch.from_numpy(lg), model.detect(torch.from_numpy(iw).cuda(), is_video=False)["preds"].cpu())
    # uint8 frames: detect of u8 / 255
    clip = (torch.rand(4, 256, 256, 3, generator=g) * 255).to(torch.uint8)
    lu = np.empty((4, 1 + spec["nbits"]), dtype=np.float32)
    _lib.check(L.vsb_frames_host_u8(model._handle(), np.ascontiguousarray(clip.numpy()).ctypes.data_as(C.c_void_p), None, 0, None,
                                    lu.ctypes.data_as(C.c_void_p), 4, 256, 256, 1, 0, 1, 1.0, 0.2, 0))
    xu = (clip.permute(0, 3, 1, 2).float() / 255.0).contiguous()
    assert torch.equal(torch.from_numpy(lu), model.detect(xu.cuda(), is_video=False)["preds"].cpu())


def test_embed_is_unchanged_by_the_extractor(pooled):
    from tests.util import make_model_pair
    model, _, spec = pooled
    cnx, _, _ = make_model_pair("videoseal_1.0")
    try:
        g = torch.Generator().manual_seed(4)
        x = torch.rand(3, 3, 256, 256, generator=g).cuda()
        msgs = torch.randint(0, 2, (3, spec["nbits"]), generator=g)
        a = model.embed(x, msgs, is_video=False)
        b = cnx.embed(x, msgs, is_video=False)
        assert torch.equal(a["imgs_w"], b["imgs_w"]) and torch.equal(a["preds_w"], b["preds_w"])
    finally:
        cnx._release()
