"""The DVMark embedder on the GPU against the float64 oracle (tests/dvmark_enc_oracle.py; the embedder runs in float64 on the same
device, the resize / JND / blend of oracle/restate.OracleModel on the CPU): imgs_w within the 1e-3 contract in image mode at 256 and
384 with 96 bits across stacked-operand frame slices, in video mode with unequal chunks in every video_mode, on resized non-square input,
on 64 frames in two chunks and at K = 1 and 30; the DVMark extractor's bits on its output; the group rules; group isolation;
determinism; the streaming entry point; and every step of the plan on the exact fp16 inputs it read at 128, 256, 384 and 512
(STEP_CONFIGS), with a bound derived from the step's roundings and a mutated reference per step that must leave it."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests import dvmark_enc_oracle as de
from tests import dvmark_oracle as dv
from videoseal_b200 import _lib, cfg
from videoseal_b200.model import _DEF_INTERP, Videoseal

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 1e-3
U16 = 2.0 ** -11      # fp16 unit roundoff
U32 = 2.0 ** -24
SUB = 2.0 ** -25      # half the spacing of fp16 subnormals: the rounding of a value near zero


def _model(S, K, ext="dvmark"):
    card = de.card(ext, img_size=S, nbits=K)
    spec = cfg.spec_from_card(card)
    ospec = de.spec_from_card(card)
    sd = de.synth_state_dict(ospec, de.SEED)
    model = Videoseal(spec)
    model.load_state_dict(sd)
    orc = de.EncOracle(ospec, sd, device=DEV)
    return model.to(DEV), orc


def _frames(B, S, seed, W=None):
    return torch.rand(B, 3, S, W or S, generator=torch.Generator().manual_seed(seed))


def _msgs(n, K, seed):
    return torch.randint(0, 2, (n, K), generator=torch.Generator().manual_seed(seed))


def _embed_both(model, orc, x, m, is_video):
    out = model.embed(x.to(DEV), m, is_video=is_video)
    ref = orc.embed(x, m, is_video=is_video)
    err = (out["imgs_w"].cpu() - ref["imgs_w"]).abs().max().item()
    assert err <= TOL, err
    return out, ref, err


def test_image_mode_256_k96_12_frames():
    """12 frames in one call: every 3x3x3 conv at 256 x 256 runs in several frame slices"""
    _image_mode_k96_12_frames(256)


def test_image_mode_384_k96_12_frames():
    """the half-resolution convs (192 wide) run on the gather loader"""
    _image_mode_k96_12_frames(384)


def _image_mode_k96_12_frames(S):
    model, orc = _model(S, 96)
    x, m = _frames(12, S, 1), _msgs(12, 96, 2)
    out, ref, err = _embed_both(model, orc, x, m, False)
    assert (out["preds_w"].cpu() - ref["preds_w"]).abs().max().item() <= TOL
    print("image", S, "K=96 x12: max |imgs_w - oracle|", f"{err:.2e}")
    # the DVMark extractor reads the same bits from the GPU's imgs_w as from the oracle's wherever the oracle's logit clears the margin
    got = model.detect(out["imgs_w"], is_video=False)["preds"].double()
    sd = {k: v.to(DEV, torch.float64) for k, v in orc.sd.items() if k.startswith("detector.")}
    lref = dv.grouped(sd, ref["imgs_w"].to(DEV, torch.float64), 12)
    assert ((got - lref).abs().max() / lref.abs().max()).item() <= 1e-2
    sure = lref.abs() > 2e-2 * lref.abs().max()
    assert torch.equal((got > 0)[sure], (lref > 0)[sure])


@pytest.mark.parametrize("mode", ["repeat", "alternate", "interpolate"])
def test_video_unequal_chunks_every_mode(mode):
    """9 frames, step 2: key frames 0 2 4 6 8 in chunks of 3 and 2"""
    model, orc = _model(256, 32)
    model.chunk_size = orc.chunk_size = 3
    model.step_size = orc.step_size = 2
    model.video_mode = orc.video_mode = mode
    _, _, err = _embed_both(model, orc, _frames(9, 256, 3), _msgs(1, 32, 4), True)
    print(mode, f"{err:.2e}")


def test_resized_non_square():
    model, orc = _model(256, 32)
    model.chunk_size = orc.chunk_size = 2
    model.step_size = orc.step_size = 1
    _embed_both(model, orc, _frames(3, 300, 5, W=280), _msgs(1, 32, 6), True)
    _embed_both(model, orc, _frames(2, 200, 7, W=360), _msgs(2, 32, 8), False)


def test_64_frames_two_chunks_128():
    model, orc = _model(128, 96)
    model.chunk_size = orc.chunk_size = 32
    model.step_size = orc.step_size = 1
    _embed_both(model, orc, _frames(64, 128, 9), _msgs(1, 96, 10), True)


@pytest.mark.parametrize("K", [1, 30])
def test_small_and_unaligned_nbits(K):
    model, orc = _model(128, K)
    _embed_both(model, orc, _frames(3, 128, 11), _msgs(3, K, 12), False)


def test_group_rules_isolation_and_determinism():
    model, _ = _model(128, 8)
    with pytest.raises(NotImplementedError, match="64"):
        model.embed(_frames(65, 128, 0).to(DEV), _msgs(65, 8, 0), is_video=False)
    model.chunk_size, model.step_size = 65, 1
    with pytest.raises(NotImplementedError, match="64"):
        model.embed(_frames(70, 128, 0).to(DEV), _msgs(1, 8, 0), is_video=True)
    # chunks of 4 key frames: changing frame 5 leaves the first and third chunk bit-identical
    model.chunk_size = 4
    x, m = _frames(12, 128, 13), _msgs(1, 8, 14)
    a = model.embed(x.to(DEV), m, is_video=True)["imgs_w"]
    y = x.clone()
    y[5] = 1 - y[5]
    b = model.embed(y.to(DEV), m, is_video=True)["imgs_w"]
    assert torch.equal(a[:4], b[:4]) and torch.equal(a[8:], b[8:])
    assert (a[4:8] - b[4:8]).abs().max().item() > 1e-3
    assert torch.equal(a, model.embed(x.to(DEV), m, is_video=True)["imgs_w"]), "two runs differ"


def test_streaming_entry_matches_embed():
    """vsb_embed_detect_host (slices of whole chunks) with a DVMark embedder and a ConvNeXt extractor gives embed()'s imgs_w"""
    model, _ = _model(256, 32, "convnext")
    model.chunk_size, model.step_size = 8, 1
    F_ = 40
    x = _frames(F_, 256, 15).contiguous()
    m = _msgs(1, 32, 16).to(torch.uint8).contiguous()
    ref = model.embed(x.to(DEV), m, is_video=True)["imgs_w"].cpu()
    imgs_w = torch.empty_like(x)
    logits = torch.empty(F_, 33)
    flags = model._flags(_DEF_INTERP, False, (256, 256))
    _lib.check(_lib.lib().vsb_embed_detect_host(model._handle(), x.data_ptr(), m.data_ptr(), 1, imgs_w.data_ptr(), logits.data_ptr(),
                                                F_, 256, 256, 1, 0, 8, C.c_float(model.blender.scaling_i),
                                                C.c_float(model.blender.scaling_w), flags))
    err = (imgs_w - ref).abs().max().item()
    print("streaming vs embed(): max |imgs_w difference|", err)
    assert err <= TOL, err
    lg = model.detect(imgs_w.to(DEV), is_video=False)["preds"].cpu()
    assert ((lg - logits).abs().max() / lg.abs().max()).item() <= 1e-4


# ---------------------------------------------------------------------------------------------------------------------------------
# every step on the fp16 inputs it read (plan taps with vsb_debug_keep_inputs: each map in a buffer of its own)


def _nchw(t):
    return t.to(DEV, torch.float64).permute(0, 3, 1, 2)


def _judge(name, got, ref, bound, mutants):
    """|got - ref| <= bound everywhere; every mutant leaves the bound somewhere"""
    r = ((got - ref).abs() / bound).max().item()
    assert r <= 1.0, (name, r)
    for mname, mut in mutants.items():
        mr = ((got - mut).abs() / bound).max().item()
        assert mr > 1.0, (name, mname, mr)
    print(f"  {name:10s} err/bound {r:.3f}", {k: "rejected" for k in mutants})
    return r


# (S, B, G): 5 frames at 128 and 256 (K = 30; emb_layer3.0's 1152-wide operand in slices of 3 at 256), 3 at 384 (one-frame slices,
# the half-resolution convs on the gather loader) and at 512 (one-frame and two-frame slices, a short last slice)
STEP_CONFIGS = [(128, 5, 2), (256, 5, 2), (384, 3, 3), (512, 3, 3)]


def test_each_step_against_float64_on_its_inputs():
    """the STEP_CONFIGS row 128 x 5 G2: every conv in one launch"""
    _each_step(*STEP_CONFIGS[0])


@pytest.mark.parametrize("S,B,G", STEP_CONFIGS[1:], ids=[f"{s}x{b}-G{g}" for s, b, g in STEP_CONFIGS[1:]])
def test_each_step_across_frame_slices(S, B, G):
    """the STEP_CONFIGS rows in which some 3x3x3 conv runs in several frame slices"""
    _each_step(S, B, G)


def _each_step(S, B, G):
    """B frames in chunks of G key frames, K = 30, one message per frame.  Conv bound: fp16 weights (2^-11 each) and fp32 sums
    (K 2^-24) times sum |x| |w|, plus the fp16 output rounding (2^-11 |y|, and 2^-25 near zero).  Each 3x3x3 conv runs in the frame
    slices dv_slice_frames gives (pinned by the tstack launch counts).  Mutations: messages of the neighbouring frame,
    align_corners=False, the skip concat order swapped, the time taps reversed, and in every conv cut into slices, time neighbours
    zeroed at slice boundaries (slice_is_group) and every slice stacked from the first slice's frames (slice_offset_ignored)."""
    K = 30
    model, orc = _model(S, K)
    sd = orc.emb_sd
    x, m = _frames(B, S, 17).to(DEV), _msgs(B, K, 18).to(torch.uint8).to(DEV)
    out = torch.empty_like(x)
    L = _lib.lib()
    h = model._handle()
    P1, P2 = (64 + K + 7) // 8 * 8, (128 + K + 7) // 8 * 8
    # every 3x3x3 conv of the plan as (stacked channels, map side): its launches are the slices of conv_slices
    c3 = [(64, S), (P1, S), (256, S), (128, S), (P2, S // 2), (512, S // 2), (256, S // 2), (384, S), (256, S), (128, S)]
    want = {}
    for c, hh in c3:
        k = f"dvmark_enc.tstack.{c}-{dv.stack_width(c)}@{hh}"
        want[k] = want.get(k, 0) + len(dv.conv_slices(c, hh, B))
    _lib.check(L.vsb_debug_keep_inputs(h, 1))
    try:
        torch.cuda.synchronize()
        L.vsb_profile_enable(1)
        try:
            _lib.check(L.vsb_embed(h, x.data_ptr(), m.data_ptr(), B, out.data_ptr(), None, B, S, S, 1, 0, G,
                                   C.c_float(1.0), C.c_float(0.2), _lib.FLAG_NO_ATTENUATION, model._stream()))
            torch.cuda.synchronize()
            buf = C.create_string_buffer(1 << 16)
            L.vsb_profile_read(buf, len(buf))
        finally:
            L.vsb_profile_enable(0)
        launches = {ln.split("\t")[0]: int(ln.split("\t")[2]) for ln in buf.value.decode().splitlines()}
        assert {k: launches.get(k) for k in want} == want, launches
        t = {n: _nchw(model.debug_tensor(n)) for n in ("dve.t0", "dve.t2", "dve.t4", "dve.cat1", "dve.e1_0", "dve.e1_2", "dve.cat2",
                                                        "dve.e2_0", "dve.e2_2", "dve.e2_4", "dve.cat3", "dve.e3_0", "dve.e3_2")}
        delta = model.debug_tensor("delta").to(DEV, torch.float64)
    finally:
        _lib.check(L.vsb_debug_keep_inputs(h, 0))
    md = m.double()
    groups = dv.segments(B, G)

    def conv(key, inp, w=None, segs=groups):
        ww = sd[de.P + key + ".weight"] if w is None else w
        bb = sd[de.P + key + ".bias"] if w is None else torch.zeros_like(sd[de.P + key + ".bias"])
        pad = (ww.shape[2] // 2, 1, 1)
        return torch.cat([F.conv3d(inp[a:e].permute(1, 0, 2, 3).unsqueeze(0), ww, bb, padding=pad).squeeze(0).permute(1, 0, 2, 3)
                          for a, e in segs])

    def slice_mutants(key, inp, ref, C):
        """the two slicing mutations of a 3x3x3 conv over C stacked channels (none when it runs in one launch)"""
        slices = dv.conv_slices(C, inp.shape[-1], B)
        if len(slices) == 1:
            return {}
        assert dv.crossing_groups(slices, B, G), (key, "no group crosses a slice boundary", slices)
        return {"slice_is_group": conv(key, inp, segs=dv.segments(B, G, slices)),
                "slice_offset_ignored": dv.slice_offset_ignored(ref, slices)}

    def conv_step(name, key, inp, got, relu=True, fp16_w=True, mutants=None, C=None):
        w = sd[de.P + key + ".weight"]
        ref = conv(key, inp)
        kk = w[0].numel()
        mag = conv(key, inp.abs(), w.abs())
        bound = ((U16 if fp16_w else 0.0) + kk * U32) * mag
        mutants = dict(mutants or {})
        if w.shape[2] == 3:
            mutants.update(slice_mutants(key, inp, ref, C or inp.shape[1]))
        if relu:
            ref = torch.relu(ref)
            bound = bound + U16 * ref + SUB
        return _judge(name, got, ref, bound, {k: (torch.relu(v) if relu else v) for k, v in mutants.items()})

    xin = 2 * x.double() - 1
    conv_step("t0", "transform_layer.0", xin, t["dve.t0"], fp16_w=False)
    conv_step("t2", "transform_layer.2", t["dve.t0"], t["dve.t2"])
    conv_step("t4", "transform_layer.4", t["dve.t2"], t["dve.t4"])
    w6 = sd[de.P + "transform_layer.6.weight"]
    conv_step("t6", "transform_layer.6", t["dve.t4"], t["dve.cat1"][:, :64],
              mutants={"taps_reversed": conv("transform_layer.6", t["dve.t4"], w6.flip(2)) + sd[de.P + "transform_layer.6.bias"].view(1, -1, 1, 1)})
    # message planes: exact 0 / 1, zero pad channels
    planes = torch.zeros(B, P1 - 64, S, S, dtype=torch.float64, device=DEV)
    planes[:, :K] = md[:, :, None, None]
    _judge("planes", t["dve.cat1"][:, 64:], planes, torch.full_like(planes, 1e-30),
           {"neighbour_msgs": torch.roll(planes, 1, 0)})
    w10 = sd[de.P + "emb_layer1.0.weight"]
    cat1 = t["dve.cat1"][:, :64 + K]
    conv_step("e1_0", "emb_layer1.0", cat1, t["dve.e1_0"], C=P1,
              mutants={"taps_reversed": conv("emb_layer1.0", cat1, w10.flip(2)) + sd[de.P + "emb_layer1.0.bias"].view(1, -1, 1, 1)})
    conv_step("e1_2", "emb_layer1.2", t["dve.e1_0"], t["dve.e1_2"])
    skip = t["dve.cat3"][:, :128]
    conv_step("e1_4", "emb_layer1.4", t["dve.e1_2"], skip)
    # pool (one fp16 rounding of an fp32 mean) and the half-resolution planes
    pref = F.avg_pool2d(skip, 2)
    _judge("pool", t["dve.cat2"][:, :128], pref, U16 * pref + SUB, {"no_pool": skip[:, :, ::2, ::2]})
    planes2 = torch.zeros(B, P2 - 128, S // 2, S // 2, dtype=torch.float64, device=DEV)
    planes2[:, :K] = md[:, :, None, None]
    _judge("planes/2", t["dve.cat2"][:, 128:], planes2, torch.full_like(planes2, 1e-30), {"neighbour_msgs": torch.roll(planes2, 1, 0)})
    conv_step("e2_0", "emb_layer2.0", t["dve.cat2"][:, :128 + K], t["dve.e2_0"], C=P2)
    conv_step("e2_2", "emb_layer2.2", t["dve.e2_0"], t["dve.e2_2"])
    conv_step("e2_4", "emb_layer2.4", t["dve.e2_2"], t["dve.e2_4"])
    # up-sample: one fp16 rounding of an fp32 blend, plus the fp32 source coordinate (|error| <= 2^-24 * index in lambda)
    e24 = t["dve.e2_4"]
    uref = F.interpolate(e24, size=(S, S), mode="bilinear", align_corners=True)
    ubound = U16 * uref + 8 * U32 * S * e24.abs().amax(dim=(2, 3), keepdim=True) + SUB
    _judge("upsample", t["dve.cat3"][:, 128:], uref, ubound,
           {"align_corners_false": F.interpolate(e24, size=(S, S), mode="bilinear", align_corners=False)})
    cat3 = t["dve.cat3"]
    conv_step("e3_0", "emb_layer3.0", cat3, t["dve.e3_0"],
              mutants={"concat_swapped": conv("emb_layer3.0", torch.cat([cat3[:, 128:], cat3[:, :128]], 1))})
    conv_step("e3_2", "emb_layer3.2", t["dve.e3_0"], t["dve.e3_2"])
    # output layer: fp32 pre-tanh value (no fp16 rounding), tanh' <= 1, tanhf within a few ulp
    w34 = sd[de.P + "emb_layer3.4.weight"]
    pre = conv("emb_layer3.4", t["dve.e3_2"])
    dbound = (U16 + w34[0].numel() * U32) * conv("emb_layer3.4", t["dve.e3_2"], w34.abs()) + 4 * U32
    _judge("out+tanh", delta, torch.tanh(pre), dbound,
           {"taps_reversed": torch.tanh(conv("emb_layer3.4", t["dve.e3_2"], w34.flip(2)) + sd[de.P + "emb_layer3.4.bias"].view(1, -1, 1, 1)),
            **{k: torch.tanh(v) for k, v in slice_mutants("emb_layer3.4", t["dve.e3_2"], pre, 128).items()}})
    # the groups: the last group's output does not depend on the frames before it
    g0 = (B - 1) // G * G
    iso = conv("emb_layer3.4", t["dve.e3_2"][g0:], segs=[(0, B - g0)])
    assert (torch.tanh(iso) - delta[g0:]).abs().max().item() <= dbound[g0:].max().item()
    print(f"{S}x{B} G{G}: launches per stacked conv {want}")
