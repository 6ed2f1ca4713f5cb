"""Pixel-wise ConvNeXt extractors on the GPU (synthetic checkpoints, nbits 256): per-pixel maps [F, 1+K, P, P] from detect()
against the CPU oracle and the reference's fixture, full batches, video, the harness, and the C entry points."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from tests import pixelwise_oracle as pw

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = torch.load(os.path.join(ROOT, "tests", "golden", "pixelwise.pt"), weights_only=False)
AGGS = ("avg", "squared_avg", "l1norm_avg", "l2norm_avg")


@pytest.fixture(scope="module", params=pw.PRESETS)
def pair(request):
    model, orc, spec = pw.model_pair(request.param)
    yield request.param, model, orc, spec
    model._release()


def contract(got: torch.Tensor, ref: torch.Tensor, what: str):
    """Per frame over every (channel, pixel) value.  DESIGN.md §4 states the logits contract (|d| <= 1e-2 max(|ref|, 0.1 |ref|inf),
    |d|inf <= 1.5e-3 |ref|inf); the pixel-wise maps pass three more fp16 stages and do not meet it (measured on an H100: |d|inf up
    to 2.9e-3 |ref|inf, elementwise up to 2.9e-2), so they are held to the separate map bound of §4: |d| <= 5e-2 max(|ref|,
    0.1 |ref|inf), |d|inf <= 5e-3 |ref|inf, and decisions exact wherever |ref| > 1e-2 |ref|inf.  Prints the measured errors."""
    got, ref = got.float().cpu(), ref.float()
    for f in range(ref.shape[0]):
        g, r = got[f], ref[f]
        ninf = r.abs().max().item()
        d = (g - r).abs()
        rel = (d / torch.maximum(r.abs(), torch.full_like(r, 0.1 * ninf))).max().item()
        big = r.abs() > 1e-2 * ninf
        flips = int(((g > 0) != (r > 0))[big].sum())
        print(f"[{what}] frame {f}: |d|inf / |ref|inf = {d.max().item() / ninf:.2e}, max elementwise rel = {rel:.2e}, "
              f"decision flips above the margin = {flips}")
        assert rel <= 5e-2, (what, f, rel)
        assert d.max().item() <= 5e-3 * ninf, (what, f, d.max().item() / ninf)
        assert flips == 0, (what, f)


def test_detect_parity_and_fixture(pair):
    preset, model, orc, spec = pair
    res = GOLDEN["presets"][preset]["cases"]
    for name in ("img256", "img_resized"):
        case = res[name]
        x = torch.rand(*case["shape"], generator=torch.Generator().manual_seed(case["gen_seed"]))
        got = model.detect(x.cuda(), is_video=False)["preds"]
        assert got.shape == (x.shape[0], 1 + spec["nbits"], 256, 256) and got.dtype == torch.float32
        ref = orc.detect(x, is_video=False)["preds"]
        contract(got, ref, f"{preset}/{name}")
        # the reference itself, through the fixture's strided samples
        s = pw.sample(got.cpu())
        assert (s - case["maps_s"]).abs().max().item() <= 5e-3 * case["maps_s"].abs().max().item()
        # the debug taps of the intermediate stages against the oracle's
        if name == "img256":
            taps = {}
            orc.detector(x, taps)
            for i in range(len(spec["pixel_decoder"]["upscale_stages"]) - 1):
                t = model.debug_tensor(f"pd{i}").permute(0, 3, 1, 2)
                assert t.shape == taps[f"pd{i}"].shape
                assert (t - taps[f"pd{i}"]).abs().max().item() <= 0.03 * taps[f"pd{i}"].abs().max().item()


@pytest.mark.parametrize("stages", [[4, 4, 2], [2, 4, 4]])
def test_detect_img_size_384(stages):
    """img_size 384: a 12 x 12 trunk map; [2, 4, 4] also runs the untiled gather (12 is not a multiple of 8) and a x4 head"""
    import copy
    model, orc, spec = pw.model_pair("convnext_tiny_pw", img_size=384, device=None)
    if stages != [4, 4, 2]:
        card_spec = copy.deepcopy(spec)
        card_spec["pixel_decoder"]["upscale_stages"] = stages
        sd = pw.synth_state_dict(card_spec, 7)
        from videoseal_b200.model import Videoseal
        model = Videoseal(model.spec | {"pixel_decoder": card_spec["pixel_decoder"]})
        model.load_state_dict(sd)
        orc = pw.OracleModel(card_spec, sd)
    model = model.eval().to("cuda")
    x = torch.rand(2, 3, 384, 384, generator=torch.Generator().manual_seed(11))
    got = model.detect(x.cuda(), is_video=False)["preds"]
    assert got.shape == (2, 257, 384, 384)
    contract(got, orc.detect(x, is_video=False)["preds"], f"img384/{stages}")
    model._release()


def test_full_batch(pair):
    preset, model, orc, spec = pair
    x = torch.rand(64, 3, 256, 256, generator=torch.Generator().manual_seed(21)).cuda()
    full = model.detect(x, is_video=False)["preds"]
    again = model.detect(x, is_video=False)["preds"]
    assert torch.equal(full, again), "repeated calls must be bit-identical"
    halves = torch.cat([model.detect(x[:32], is_video=False)["preds"], model.detect(x[32:], is_video=False)["preds"]])
    assert torch.equal(full, halves), "B=64 must equal 2 x 32"
    idx = [0, 17, 42, 63]
    contract(full[idx], orc.detect(x[idx].cpu(), is_video=False)["preds"], f"{preset}/b64")
    # sub-batches of more than 64 frames write at their offsets
    y = torch.cat([x, x[:6]])
    big = model.detect(y, is_video=False)["preds"]
    assert torch.equal(big[:64], full) and torch.equal(big[64:], full[:6])


def test_video_and_extract_message(pair):
    preset, model, orc, spec = pair
    case = GOLDEN["presets"][preset]["cases"]["vid"]
    x = torch.rand(*case["shape"], generator=torch.Generator().manual_seed(case["gen_seed"]))
    model.chunk_size, orc.chunk_size = 2, 2
    got = model.detect(x.cuda(), is_video=True)["preds"]
    ref = orc.detect(x, is_video=True)["preds"]
    contract(got, ref, f"{preset}/video")
    noaa = {"mode": "bilinear", "align_corners": False, "antialias": False}     # extract_message's default interpolation
    bits_ref = orc.detect(x, True, noaa)["preds"][:, 1:]
    bits_gpu = model.detect(x.cuda(), True, noaa)["preds"][:, 1:].cpu()

    def decode(bp, agg):
        if agg == "avg":
            return bp.mean(0)
        if agg == "squared_avg":
            return (bp * bp.abs()).mean(0)
        return (bp * torch.norm(bp, p=1 if agg == "l1norm_avg" else 2, dim=1, keepdim=True)).mean(0)
    for agg in AGGS:
        a = model.extract_message(x.cuda(), aggregation=agg).cpu()
        o = orc.extract_message(x, aggregation=agg)
        assert a.shape == o.shape == (1, spec["nbits"], 256, 256) and a.dtype == torch.bool
        dec_ref, dec_gpu = decode(bits_ref, agg), decode(bits_gpu, agg)
        assert torch.equal(a[0], dec_gpu > 0), agg          # the product's bits are its own maps, aggregated
        # bits may differ from the oracle's only where the decoded value is within the maps' error of zero
        err = (dec_gpu - dec_ref).abs().max().item()
        diff = (a != o)[0]
        n = int(diff.sum())
        top = dec_ref.abs().max().item()
        print(f"[{preset}] extract_message {agg}: {n} of {diff.numel()} bits differ; max |decoded error| = {err / top:.2e} max|decoded|")
        assert err <= 5e-3 * top, agg
        if n:
            assert dec_ref[diff].abs().max().item() <= err, agg
        g = GOLDEN["presets"][preset]["cases"]["extract"][agg]
        assert abs(int(a.sum()) - g["ones"]) <= max(8, n)
    model.chunk_size = spec["chunk_size"]


def test_harness_and_entry_points(pair, tmp_path):
    preset, model, orc, spec = pair
    from videoseal_b200 import _lib, jit, streaming
    from videoseal_b200.evals import full, metrics
    g = torch.Generator().manual_seed(31)
    img = torch.rand(3, 256, 256, generator=g)
    torch.manual_seed(5)
    rows = full.evaluate(model, [(img.cuda(),)], is_video=False, output_dir=str(tmp_path))
    # the same message again (evaluate draws it from the global generator) -> the oracle's maps of the product's watermarked image
    torch.manual_seed(5)
    out = model.embed(img[None].cuda(), is_video=False)
    ref_maps = orc.detect(out["imgs_w"].cpu(), is_video=False)["preds"]
    acc = metrics.bit_accuracy(ref_maps[:, 1:], out["msgs"].cpu()).mean().item()
    assert abs(rows[0]["bit_acc_Identity_0"] - acc) <= 1.0 / spec["nbits"]
    # TorchScript-style tensor API: the same maps as detect()
    x = torch.rand(2, 3, 256, 256, generator=g).cuda()
    ref = model.detect(x, is_video=False)["preds"]
    assert torch.equal(jit.TensorAPI(model).detect(x), ref)
    assert torch.equal(model.detector(x), ref)
    # host entry point
    L = _lib.lib()
    xh = np.ascontiguousarray(x.cpu().numpy())
    oh = np.empty(tuple(ref.shape), dtype=np.float32)
    _lib.check(L.vsb_detect_host(model._handle(), xh.ctypes.data_as(C.c_void_p), oh.ctypes.data_as(C.c_void_p), 2, 256, 256, 0))
    assert torch.equal(torch.from_numpy(oh), ref.cpu())
    # streaming forms are pooled-logit only
    clip = (torch.rand(4, 256, 256, 3, generator=g) * 255).to(torch.uint8).numpy()
    lg = np.empty((4, 1 + spec["nbits"]), dtype=np.float32)
    rc = L.vsb_frames_host_u8(model._handle(), clip.ctypes.data_as(C.c_void_p), None, 0, None, lg.ctypes.data_as(C.c_void_p), 4, 256, 256,
                              1, 0, 1, 1.0, 0.2, 0)
    assert rc == -2 and b"not implemented" in L.vsb_last_error()
    f32 = np.ascontiguousarray(x.cpu().numpy())
    m8 = np.zeros((1, spec["nbits"]), dtype=np.uint8)
    iw = np.empty_like(f32)
    rc = L.vsb_embed_detect_host(model._handle(), f32.ctypes.data_as(C.c_void_p), m8.ctypes.data_as(C.c_void_p), 1,
                                 iw.ctypes.data_as(C.c_void_p), lg.ctypes.data_as(C.c_void_p), 2, 256, 256, 1, 0, 1, 1.0, 0.2, 0)
    assert rc == -2
    with pytest.raises(NotImplementedError):
        streaming.detect_video_clip(model, clip)
    with pytest.raises(NotImplementedError):
        streaming.embed_detect_video_clip(model, clip)
    # the setter belongs before finalize
    f = (C.c_int32 * 3)(4, 4, 2)
    assert L.vsb_model_set_pixel_decoder(model._handle(), 3, f, 1) == -4
