"""Every kernel of the U-Net embed plan on its own inputs (the plan's debug taps) against float64 references with derived
error bounds (tests/unet_kernels.py), at each card and processing size whose dispatch differs; mutated references prove the
bounds see the defects that matter; the profile names pin which kernel variant each configuration runs."""
import ctypes as C

import pytest
import torch

from tests import unet_kernels as uk
from tests import unet_tiny as ut
from tests.util import make_model_pair

pytestmark = pytest.mark.gpu

# name: (card, overrides, processing size, frames, per-frame messages)
CONFIGS = {
    "v1_256_b64": ("videoseal_1.0", None, 256, 64, True),     # ring convs wrap over a full 64-frame sub-batch
    "v1_256_b3": ("videoseal_1.0", None, 256, 3, False),      # ragged last tile, one broadcast message
    "v1_128_b64": ("videoseal_1.0", None, 128, 64, True),     # phase-folded up-conv + border fix instead of tap GEMM + gather
    "v1_512_b16": ("videoseal_1.0", None, 512, 16, False),    # rings that no longer fit: GEMM down conv / 3x3
    "v1_1024_b2": ("videoseal_1.0", None, 1024, 2, True),     # 16-channel 3x3 ring too long: halo GEMM, with the fused outc
    "v1_256_b70": ("videoseal_1.0", None, 256, 70, True),     # taps of the 6-frame second sub-batch
    "pix_256_b32": ("pixelseal", None, 256, 32, True),        # 512-channel bottleneck, untiled gather (128 channels)
    "chunky_256_b8": ("chunkyseal", {"num_blocks": 1}, 256, 8, False),   # RGB, 2560-channel bottleneck, GEMM + fused 3-output outc
    "tiny_256_b64": ("unet_tiny_yuv_quant", None, 256, 64, True),       # 8-channel direct kernels
    "tiny_512_b2": ("unet_tiny_yuv_quant", None, 512, 2, False),
}

# every U-Net step name each configuration runs (vsb_profile_read; "unet." prefix omitted): a layer that moves to another
# kernel variant changes its name
V1_256 = """first msg conv3x3d.16-16@256 conv1x1d.16-16@256 conv3x3d+outc.16-16@256 down3x3s2d.16-32@128 conv3x3d.32-32@128
    conv1x1d.32-32@128 down3x3s2.32-64@64 conv3x3d.64-64@64 conv1x1d.64-64@64 down3x3s2.64-128@32 conv3x3.128-128@32
    conv1x1.128-128@32 conv3x3.384-384@32 conv1x1.384-384@32 uptap1x1.768-576@32 upgather.64@64 uptap1x1.128-288@64
    upgather.32@128 uptap1x1.64-144@128 upgather.16@256"""
EXPECT = {
    "v1_256_b64": V1_256, "v1_256_b3": V1_256, "v1_256_b70": V1_256,
    "v1_128_b64": """first msg conv3x3d.16-16@128 conv1x1d.16-16@128 conv3x3d+outc.16-16@128 down3x3s2d.16-32@64
        conv3x3d.32-32@64 conv1x1d.32-32@64 down3x3s2.32-64@32 conv3x3d.64-64@32 conv1x1d.64-64@32 down3x3s2.64-128@16
        conv3x3.128-128@16 conv1x1.128-128@16 conv3x3.384-384@16 conv1x1.384-384@16 uptap1x1.768-576@16 upgather.64@32
        uptap1x1.128-288@32 upgather.32@64 upphase.64-16@128 upborder.16@128""",
    "v1_512_b16": """first msg conv3x3d.16-16@512 conv1x1d.16-16@512 conv3x3d+outc.16-16@512 down3x3s2.16-32@256
        conv3x3d.32-32@256 conv1x1d.32-32@256 down3x3s2.32-64@128 conv3x3.64-64@128 conv1x1d.64-64@128 down3x3s2.64-128@64
        conv3x3.128-128@64 conv1x1.128-128@64 conv3x3.384-384@64 conv1x1.384-384@64 uptap1x1.768-576@64 upgather.64@128
        uptap1x1.128-288@128 upgather.32@256 uptap1x1.64-144@256 upgather.16@512""",
    "v1_1024_b2": """first msg conv3x3.16-16@1024 conv1x1d.16-16@1024 conv3x3+outc.16-16@1024 down3x3s2.16-32@512
        conv3x3.32-32@512 conv1x1d.32-32@512 down3x3s2.32-64@256 conv3x3.64-64@256 conv1x1.64-64@256 down3x3s2.64-128@128
        conv3x3.128-128@128 conv1x1.128-128@128 conv3x3.384-384@128 conv1x1.384-384@128 uptap1x1.768-576@128 upgather.64@256
        uptap1x1.128-288@256 upgather.32@512 uptap1x1.64-144@512 upgather.16@1024""",
    "pix_256_b32": """first msg conv3x3d.32-32@256 conv1x1d.32-32@256 conv3x3d+outc.32-32@256 down3x3s2.32-64@128
        conv3x3.64-64@128 conv1x1d.64-64@128 down3x3s2.64-128@64 conv3x3.128-128@64 conv1x1.128-128@64 down3x3s2.128-256@32
        conv3x3.256-256@32 conv1x1.256-256@32 conv3x3.512-512@32 conv1x1.512-512@32 uptap1x1.1024-1152@32 upgather.128@64
        uptap1x1.256-576@64 upgather.64@128 uptap1x1.128-288@128 upgather.32@256""",
    "chunky_256_b8": """first msg conv3x3.64-64@256 conv1x1.64-64@256 conv3x3+outc.64-64@256 down3x3s2.64-128@128
        conv3x3.128-128@128 conv1x1.128-128@128 down3x3s2.128-256@64 conv3x3.256-256@64 conv1x1.256-256@64 down3x3s2.256-512@32
        conv3x3.512-512@32 conv1x1.512-512@32 conv3x3.2560-2560@32 conv1x1.2560-2560@32 uptap1x1.5120-2304@32 upgather.256@64
        uptap1x1.512-1152@64 upgather.128@128 uptap1x1.256-576@128 upgather.64@256""",
    "tiny_256_b64": """first msg conv3x3d.8-8@256 conv1x1d.8-8@256 conv3x3d+outc.8-8@256 down3x3s2d.8-8@128 conv3x3d.8-8@128
        conv1x1d.8-8@128 down3x3s2.8-16@64 conv3x3d.16-16@64 conv1x1d.16-16@64 down3x3s2d.16-32@32 conv3x3d.32-32@32
        conv1x1d.32-32@32 down3x3s2.32-64@16 conv3x3d.64-64@16 conv1x1d.64-64@16 conv3x3.64-64@16 conv3x3.320-320@16
        conv1x1.320-320@16 uptap1x1.640-288@16 upgather.32@32 upphase.64-16@64 upborder.16@64 uptap1x1.32-72@64
        upgather.8@128 uptap1x1.16-72@128 upgather.8@256""",
    "tiny_512_b2": """first msg conv3x3d.8-8@512 conv1x1d.8-8@512 conv3x3d+outc.8-8@512 down3x3s2d.8-8@256 conv3x3d.8-8@256
        conv1x1d.8-8@256 down3x3s2.8-16@128 conv3x3d.16-16@128 conv1x1d.16-16@128 down3x3s2d.16-32@64 conv3x3d.32-32@64
        conv1x1d.32-32@64 down3x3s2.32-64@32 conv3x3d.64-64@32 conv1x1d.64-64@32 conv3x3.64-64@32 conv3x3.320-320@32
        conv1x1.320-320@32 uptap1x1.640-288@32 upgather.32@64 upphase.64-16@128 upborder.16@128 uptap1x1.32-72@128
        upgather.8@256 uptap1x1.16-72@256 upgather.8@512""",
}
EXPECT = {k: {"unet." + n for n in v.split()} for k, v in EXPECT.items()}

_models, _results = {}, {}


def _model(card, ov):
    key = (card, str(ov))
    if key not in _models:
        _models[key] = ut.model_pair() if card == "unet_tiny_yuv_quant" else make_model_pair(card, tiny=ov)
    return _models[key]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for m, _, _ in _models.values():
        m._release()
    _models.clear()


def _profiled_embedder(model, x, m):
    L = uk_lib()
    L.vsb_profile_enable(1)
    try:
        model.embedder(x, m)
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    return {line.split("\t")[0] for line in buf.value.decode().splitlines() if line.startswith("unet.")}


def uk_lib():
    from videoseal_b200 import _lib
    return _lib.lib()


def results(cfg: str) -> dict:
    """runs one embedder call of the configuration and judges every step from its taps (memoised: the taps belong to the most
    recent call, so each configuration is judged right after its own call)"""
    if cfg in _results:
        return _results[cfg]
    card, ov, S, B, per_frame = CONFIGS[cfg]
    model, orc, spec = _model(card, ov)
    model.img_size = S
    g = torch.Generator().manual_seed(S + B)
    imgs = torch.rand(B, 3, S, S, generator=g)
    msgs = torch.randint(0, 2, (B if per_frame else 1, spec["nbits"]), generator=g)
    names = _profiled_embedder(model, imgs.cuda(), msgs)
    b0 = (B - 1) // 64 * 64                 # the taps are those of the last 64-frame sub-batch
    sub = imgs[b0:].cuda()
    sub_msgs = msgs[b0:] if per_frame else msgs.expand(B - b0, -1)
    net = uk.Net(orc.sd, spec, "cuda")
    cache = {}

    def tap(n):
        if n not in cache:
            t = model.debug_tensor(n)
            t = t if n == "delta" else t.permute(0, 3, 1, 2)     # delta is stored NCHW, every other tap NHWC
            cache[n] = t.to("cuda", torch.float64)
        return cache[n]

    def has_tap(n):
        try:
            tap(n)
            return True
        except KeyError:
            return False
    steps = []
    with torch.no_grad():
        for ck in uk.plan_checks(net, tap, sub, sub_msgs, has_tap):
            assert ck.got.shape == ck.ref.shape and ck.got.shape[0] == B - b0, (ck.step, ck.got.shape, ck.ref.shape)
            steps.append(uk.judge(ck))
            del ck
    cache.clear()
    torch.cuda.empty_cache()
    _results[cfg] = {"names": names, "steps": steps}
    return _results[cfg]


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_step_within_its_bound(cfg):
    r = results(cfg)
    bad = []
    for s in r["steps"]:
        print(f"[{cfg}] max err/tol {s['ratio']:.3f}  {s['step']}" + (f"  (LayerNorm range fallback on {s['fallback']:.2e} of pixels)"
                                                                    if s["fallback"] else ""))
        # a pixel on the LayerNorm fallback bound cannot fail: none may use it
        if s["nan"] or not s["ratio"] <= 1.0 or s["fallback"] > 0:
            bad.append((s["step"], s["ratio"], s["nan"], s["fallback"]))
    assert not bad, bad


def _step_family(step: str) -> str:
    for k in ("unet.first", "msg", "outc", "gather", "phase", "tap GEMM", "3x3 s2", "1x1", "3x3"):
        if k in step:
            return k
    raise ValueError(step)


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_mutation_is_detected(cfg):
    """each mutation is violated in every step family that has it (at up0 of the 256-bit cards the bottleneck's message channels
    are constant in space, so a border or sampling defect there can stay under the bound: the family's other levels see it),
    and the violations of border-only / last-frame-only defects lie on the border / in the last frame, at every step"""
    r = results(cfg)
    hits, bad = {}, []
    for s in r["steps"]:
        for m in s["mutations"]:
            print(f"[{cfg}] {s['step']}: {m['name']}: {m['violations']} violations"
                  + (f" ({m['outside']} off the {m['where'].replace('_', ' ')})" if m["where"] else ""))
            key = (_step_family(s["step"]), m["name"])
            hits[key] = hits.get(key, 0) + m["violations"]
            if m["outside"] != 0:
                bad.append((s["step"], m))
    missed = sorted(k for k, n in hits.items() if n == 0)
    assert not bad and not missed, (bad, missed)


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_dispatch_is_pinned(cfg):
    names = results(cfg)["names"]
    print(f"[{cfg}] {sorted(names)}")
    assert names == EXPECT[cfg], (sorted(EXPECT[cfg] - names), sorted(names - EXPECT[cfg]))


def _family(name: str) -> str:
    """profile name -> kernel family; the up gather splits by variant (pointwise_host.cuh launch_unet_upgather and the tile rule
    of UNet::build: tiled when the low-resolution side is a multiple of 8 and ups_tile_smem(2, C) <= 160 KB)"""
    fam = name.split(".")[1]
    if fam == "upgather":
        c, ho = (int(v) for v in name.split(".")[2].split("@"))
        if (ho // 2) % 8 == 0 and 10 * 10 * 9 * c * 2 <= 160 * 1024:
            return "upgather tiled"
        return f"upgather untiled VPT{1 if c <= 256 else 2}"
    if fam in ("conv3x3", "conv3x3+outc"):
        c = int(name.split(".")[-1].split("-")[0])
        return fam + (" halo GEMM" if c <= 16 else " TMA GEMM")
    return fam


def test_dispatch_union_covers_every_family():
    fams = set()
    for cfg in CONFIGS:
        fams |= {_family(n) for n in results(cfg)["names"]}
    print("[dispatch union]", sorted(fams))
    need = {"first", "conv3x3d", "conv1x1d", "conv3x3d+outc", "conv3x3 TMA GEMM", "conv3x3 halo GEMM", "conv1x1",
            "conv3x3+outc TMA GEMM", "conv3x3+outc halo GEMM", "down3x3s2d", "down3x3s2", "msg", "uptap1x1", "upgather tiled",
            "upgather untiled VPT1", "upphase", "upborder"}
    assert need <= fams, sorted(need - fams)
