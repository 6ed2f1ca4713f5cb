"""The DVMark extractor on the GPU against the float64 oracle (tests/dvmark_oracle.py, run in float64 on the same device): end to end
in image and video mode, at 256, 384 and 640 with 96 bits and across the stacked-operand frame slices, extract_message, the group
rules through the C ABI, determinism, and every step of the plan on the exact fp16 inputs it read at every processing size from 128
to 768 (STEP_CONFIGS: one-frame, short and group-crossing slices), with a mutated reference per step that must leave the step's
bound."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

from tests import dvmark_oracle as dv
from videoseal_b200 import _lib, cfg
from videoseal_b200.model import Videoseal

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
LOGIT_REL = 1e-2


def _model(S, K, emb="hidden"):
    card = dv.card(emb, img_size=S, nbits=K)
    spec = cfg.spec_from_card(card)
    sd = dv.synth_state_dict(dv.spec_from_card(card), dv.SEED)
    model = Videoseal(spec)
    model.load_state_dict(sd)
    return model.to(DEV), {k: v.to(DEV, torch.float64) for k, v in sd.items()}


def _frames(B, S, seed):
    return torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(seed)).to(DEV)


def _check_logits(got, ref, what):
    err = ((got.double() - ref).abs().max() / ref.abs().max()).item()
    assert err <= LOGIT_REL, (what, err)
    # recovered bits: exact wherever the logit lies outside the error bound
    sure = ref.abs() > 2 * LOGIT_REL * ref.abs().max()
    assert torch.equal((got.double() > 0)[sure], (ref > 0)[sure]), what
    return err


def _image_mode_k96(S, B):
    model, sd = _model(S, 96)
    x = _frames(B, S, 1)
    got = model.detect(x, is_video=False)["preds"]
    ref = dv.grouped(sd, x.double(), B)
    print("image", S, "K=96 rel err", _check_logits(got, ref, "image"))


def test_image_mode_256_k96_across_frame_slices():
    """12 frames in one call: layer2's stacked operand is cut into slices of 10 frames at 256 x 256"""
    _image_mode_k96(256, 12)


@pytest.mark.parametrize("S,B", [(384, 6), (640, 3)])
def test_image_mode_k96_unaligned_half_size(S, B):
    """layer3's map (192, 320) does not tile by 128 pixels and runs on the gather loader; layer2 in slices of 4 (384) and 1 frame
    (640)"""
    _image_mode_k96(S, B)


def test_video_mode_two_unequal_chunks_and_extract_message():
    model, sd = _model(256, 96)
    model.chunk_size = 4
    x = _frames(7, 256, 2)                       # chunks of 4 and 3 frames
    got = model.detect(x, is_video=True)["preds"]
    ref = dv.grouped(sd, x.double(), 4)
    print("video 256 K=96 rel err", _check_logits(got, ref, "video"))
    bits = model.extract_message(x)
    assert torch.equal(bits.cpu(), (ref[:, 1:].mean(dim=0) > 0).unsqueeze(0).cpu())
    # a resized input takes the same groups
    big = torch.rand(7, 3, 300, 280, generator=torch.Generator().manual_seed(3)).to(DEV)
    got = model.detect(big, is_video=True)["preds"]
    res = F.interpolate(big, size=(256, 256), mode="bilinear", align_corners=False, antialias=True)
    _check_logits(got, dv.grouped(sd, res.double(), 4), "video resized")


def test_64_frames_in_two_chunks_256():
    """the profiled workload: layer2 runs in slices of 10 frames, layer3 in slices of 42 and 22"""
    model, sd = _model(256, 96)
    model.chunk_size = 32
    x = _frames(64, 256, 6)
    got = model.detect(x, is_video=True)["preds"]
    print("64 x 256^2, chunks of 32, rel err", _check_logits(got, dv.grouped(sd, x.double(), 32), "64 frames"))


def test_group_rules_through_the_c_abi_and_determinism():
    model, sd = _model(128, 8)
    x = _frames(65, 128, 4)
    out = torch.empty(65, 9, device=DEV)
    L = _lib.lib()
    h, st = model._handle(), model._stream()
    assert L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr(), 65, 128, 128, 65, 0, st) == -2
    assert "at most 64" in L.vsb_last_error().decode()
    assert L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr(), 65, 128, 128, 0, 0, st) == -1
    assert L.vsb_detect(h, x.data_ptr(), out.data_ptr(), 65, 128, 128, 0, st) == -2
    # a group longer than the call is the whole call: 20 frames with group 65 are one group of 20, in the plan of group 20
    _lib.check(L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr(), 20, 128, 128, 65, 0, st))
    _lib.check(L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr() + 4 * 20 * 9, 20, 128, 128, 20, 0, st))
    torch.cuda.synchronize()
    assert torch.equal(out[:20], out[20:40]), "group 65 over 20 frames differs from group 20"
    _check_logits(out[:20], dv.grouped(sd, x[:20].double(), 20), "20 frames, group 65")
    _lib.check(L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr(), 64, 128, 128, 64, 0, st))
    _check_logits(out[:64], dv.grouped(sd, x[:64].double(), 64), "64-frame group")
    # groups of 13 over 65 frames: sub-batches of 52 + 13 hold whole groups
    _lib.check(L.vsb_detect_grouped(h, x.data_ptr(), out.data_ptr(), 65, 128, 128, 13, 0, st))
    _check_logits(out, dv.grouped(sd, x.double(), 13), "groups of 13")
    again = torch.empty_like(out)
    _lib.check(L.vsb_detect_grouped(h, x.data_ptr(), again.data_ptr(), 65, 128, 128, 13, 0, st))
    torch.cuda.synchronize()
    assert torch.equal(out, again), "logits differ between two runs"
    # vsb_detect: the whole call is one group
    one = torch.empty(5, 9, device=DEV)
    _lib.check(L.vsb_detect(h, x.data_ptr(), one.data_ptr(), 5, 128, 128, 0, st))
    _check_logits(one, dv.grouped(sd, x[:5].double(), 5), "vsb_detect")


def _nchw(t):
    return t.to(DEV, torch.float64).permute(0, 3, 1, 2)


def _step(name, got, ref, mutants, bound_rel):
    """got within bound_rel * max|ref| of ref; every mutant reference outside it"""
    scale = ref.abs().max().item()
    err = (got - ref).abs().max().item() / scale
    assert err <= bound_rel, (name, err)
    for mname, m in mutants.items():
        merr = (got - m).abs().max().item() / scale
        assert merr > bound_rel, (name, mname, merr)
    print(f"  {name:12s} err {err:.2e} / {bound_rel:.0e}", {k: "rejected" for k in mutants})
    return err


def _head_mutant_no_borders(sd, l3, G):
    """layer4 + mean with every tap reading the whole map (border windows ignored: the wrong border class)"""
    P = "detector.layers.layer4"
    outs = []
    for g0 in range(0, l3.shape[0], G):
        s = F.avg_pool2d(l3[g0:g0 + G], 2).sum(dim=[2, 3])                 # [T, C]
        hw = (l3.shape[2] // 2) ** 2
        w = sd[P + ".weight"].sum(dim=[3, 4])                              # [N, C, 3 (t)]
        sp = F.pad(s.t(), (1, 1))                                          # [C, T + 2], zero frames at the group ends
        o = sum(sp[:, dt:dt + s.shape[0]].t() @ w[:, :, dt].t() for dt in range(3))
        outs.append(sd[P + ".bias"] + o / hw)
    return torch.cat(outs)


# (S, B, G): 5 frames at 128 fit one launch per conv; above, layer2's stacked operand is cut into slices of 10 (256), 4 (384), 2 (512)
# and 1 frame (640, 768), with a group across a slice boundary, a short last slice at 256, 384 and 512, and layer3 (on the gather
# loader at 384 and 640) in one launch
STEP_CONFIGS = [(128, 5, 2), (256, 12, 4), (384, 6, 3), (512, 5, 5), (640, 3, 3), (768, 3, 3)]


def _profiled(L, fn):
    """run fn with the per-launch profiler on: {step name: launches}"""
    torch.cuda.synchronize()
    L.vsb_profile_enable(1)
    try:
        fn()
        torch.cuda.synchronize()
        buf = C.create_string_buffer(1 << 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    return {ln.split("\t")[0]: int(ln.split("\t")[2]) for ln in buf.value.decode().splitlines()}


def _each_step(S, B, G):
    """each kernel against float64 on the fp16 taps it read: layer1 (CUDA cores) from the frames, layer2 from layer1, layer3 from
    layer2 (the pool fused into the stack), the head (rows, window sums, layer4 + mean) from layer3.  Each stacked conv runs in the
    frame slices dv_slice_frames gives (pinned by its tstack launch count).  Mutations: the time padding leaking across groups (one
    clip over the whole batch), the pool left out, the border windows ignored, and in a conv cut into slices, time neighbours zeroed
    at slice boundaries (slice_is_group) and every slice stacked from the first slice's frames (slice_offset_ignored)."""
    model, sd = _model(S, 32)
    x = _frames(B, S, 5)
    out = torch.empty(B, 33, device=DEV)
    L = _lib.lib()
    h2 = S // 2
    sl2, sl3 = dv.conv_slices(128, S, B), dv.conv_slices(128, h2, B)
    launches = _profiled(L, lambda: _lib.check(L.vsb_detect_grouped(model._handle(), x.data_ptr(), out.data_ptr(), B, S, S, G, 0,
                                                                     model._stream())))
    assert launches.get(f"dvmark.tstack.128-384@{S}") == len(sl2), launches
    assert launches.get(f"dvmark.tstack+pool.128-384@{h2}") == len(sl3), launches
    P = "detector.layers.layer"
    l1, l2, l3 = (_nchw(model.debug_tensor(f"dvm.l{i}")) for i in (1, 2, 3))
    xd = x.double()

    def conv(i, inp, segs):
        return torch.cat([torch.relu(dv.conv3d(inp[a:e], sd[P + f"{i}.weight"], sd[P + f"{i}.bias"])) for a, e in segs])

    def slice_mutants(i, inp, ref, slices):
        if len(slices) == 1:
            return {}
        assert dv.crossing_groups(slices, B, G), ("no group crosses a slice boundary", slices)
        return {"slice_is_group": conv(i, inp, dv.segments(B, G, slices)), "slice_offset_ignored": dv.slice_offset_ignored(ref, slices)}
    groups = dv.segments(B, G)

    def leak(f):   # one clip over the whole batch: a mutation only where the batch holds more than one group
        return {"leak": f()} if len(groups) > 1 else {}
    errs = {}
    # fp16 outputs (2^-11 relative) of fp32 sums; layers 2-3 also read fp16 weights (2^-12 relative each)
    errs["l1"] = _step("layer1", l1, conv(1, xd, groups), leak(lambda: conv(1, xd, [(0, B)])), 2e-3)
    ref2 = conv(2, l1, groups)
    errs["l2"] = _step("layer2", l2, ref2, {**leak(lambda: conv(2, l1, [(0, B)])), **slice_mutants(2, l1, ref2, sl2)}, 8e-3)
    del ref2, l1
    p2 = F.avg_pool2d(l2, 2).half().double()      # the stack kernel rounds the pooled operand to fp16
    ref3 = conv(3, p2, groups)
    errs["l3"] = _step("layer3", l3, ref3, {**leak(lambda: conv(3, p2, [(0, B)])), "no_pool": conv(3, l2[:, :, ::2, ::2], groups),
                                            **slice_mutants(3, p2, ref3, sl3)}, 8e-3)
    del ref3, l2, p2
    head = torch.cat([dv.conv3d(F.avg_pool2d(l3[a:e], 2), sd[P + "4.weight"], sd[P + "4.bias"]).mean(dim=[2, 3]) for a, e in groups])
    errs["head"] = _step("head", out.double(), head,
                         {**leak(lambda: dv.conv3d(F.avg_pool2d(l3, 2), sd[P + "4.weight"], sd[P + "4.bias"]).mean(dim=[2, 3])),
                          "borders": _head_mutant_no_borders(sd, l3, G)}, 1e-5)
    # the window sums the head read: per frame, tap (1, 1, 1) is the whole pooled map's sum; taps dt = 0 / 2 are zero exactly at the
    # first / last frame of each group
    win = model.debug_tensor("dvm.win").to(DEV, torch.float64).reshape(B, 27, 256)
    tot = F.avg_pool2d(l3, 2).sum(dim=[2, 3])
    _step("window sums", win[:, 13], tot, {}, 1e-5)
    zero = lambda t: torch.equal(t, torch.zeros_like(t))   # noqa: E731
    for b in range(B):
        assert zero(win[b, :9]) == (b % G == 0), ("previous-frame taps", b)
        assert zero(win[b, 18:]) == (b % G == G - 1 or b == B - 1), ("next-frame taps", b)
    print(f"{S}x{B} G{G}: layer2 slices {sl2}, layer3 slices {sl3}; step errors (relative to max|ref|):",
          {k: f"{v:.2e}" for k, v in errs.items()})


def test_each_step_against_float64_on_its_inputs():
    """the STEP_CONFIGS row 128 x 5 G2: every conv in one launch"""
    _each_step(*STEP_CONFIGS[0])


@pytest.mark.parametrize("S,B,G", STEP_CONFIGS[1:], ids=[f"{s}x{b}-G{g}" for s, b, g in STEP_CONFIGS[1:]])
def test_each_step_across_frame_slices(S, B, G):
    """the STEP_CONFIGS rows whose layer2 runs in several frame slices"""
    _each_step(S, B, G)
