"""Every kernel of the pixel-wise decoder on its own inputs (the plan's debug taps: the trunk's fp16 output, pd{i}_y, pd{i}) and the
caller's maps, against float64 references with derived error bounds (tests/pd_kernels.py), at configurations that together reach
every gather and fused-head instantiation a model can dispatch; mutated references prove the bounds see the defects that matter;
the profile names pin which kernel each configuration runs."""
import ctypes as C

import pytest
import torch

from tests import cnx_kernels as ck
from tests import pd_kernels as pk
from tests import pixelwise_oracle as pw
from tests import vit_oracle as vo

pytestmark = pytest.mark.gpu

# every pixel-decoder step name each configuration runs (vsb_profile_read; "pd." prefix omitted)
B256_44 = "uptap1x1.1024-2304@8 upgather.256x4@32 uptap1x1.256-576@32 upgather.64x4@128 "
EXPECT = {
    "tiny256_b70": "uptap1x1.768-1728@8 upgather.192x4@32 uptap1x1.192-432@32 upgather.48x4@128 uptap1x1.48-216@128 gather_head.24x2@256",
    "tiny256_424": "uptap1x1.768-1728@8 upgather.192x4@32 uptap1x1.192-864@32 upgather.96x2@64 uptap1x1.96-216@64 gather_head.24x4@256",
    "tiny384_b5": "uptap1x1.768-3456@12 upgather_untiled.384x2@24 uptap1x1.384-864@24 upgather.96x4@96 uptap1x1.96-216@96 "
                  "gather_head.24x4@384",
    "wide256": "uptap1x1.1536-3456@8 upgather_untiled.384x4@32 uptap1x1.384-864@32 upgather.96x4@128 uptap1x1.96-216@128 "
               "gather_head.24x4@512",
    "base256_442": B256_44 + "uptap1x1.64-288@128 gather_head.32x2@256",
    "base256_424": "uptap1x1.1024-2304@8 upgather.256x4@32 uptap1x1.256-1152@32 upgather.128x2@64 uptap1x1.128-288@64 gather_head.32x4@256",
    "base256_444": B256_44 + "uptap1x1.64-144@128 gather_head.16x4@512",
    "base256_4424": B256_44 + "uptap1x1.64-288@128 upgather.32x2@256 uptap1x1.32-72@256 gather_head.8x4@1024",
    "base256_4442": B256_44 + "uptap1x1.64-144@128 upgather.16x4@512 uptap1x1.16-72@512 gather_head.8x2@1024",
    "narrow384_244": "uptap1x1.256-1152@12 upgather_untiled.128x2@24 uptap1x1.128-288@24 upgather.32x4@96 uptap1x1.32-72@96 "
                     "gather_head.8x4@384",
    "vit256_422": "uptap1x1.256-576@16 upgather.64x4@64 uptap1x1.64-288@64 upgather.32x2@128 uptap1x1.32-144@128 gather_head.16x2@256",
}
EXPECT = {k: {"pd." + n for n in v.split()} for k, v in EXPECT.items()}
assert set(EXPECT) == set(pk.CONFIGS)

_models, _results = {}, {}


def _lib():
    from videoseal_b200 import _lib as lib
    return lib


def _model(cfg):
    if cfg not in _models:
        import videoseal_b200
        card = pk.config_card(cfg)
        orc = vo if pk.CONFIGS[cfg][0] == "vit" else pw
        spec = orc.spec_from_card(card)
        sd = orc.synth_state_dict(spec, 77)
        model = videoseal_b200.load(vo.card_on_disk(card, sd, f"pd_{cfg}")).eval().to("cuda")
        _models[cfg] = (model, sd, spec)
    return _models[cfg]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for m, _, _ in _models.values():
        m._release()
    _models.clear()


def _profiled_detect(model, x):
    """(maps, {profile step name: launches}) of one detect call"""
    L = _lib().lib()
    L.vsb_profile_enable(1)         # clears what earlier calls accumulated
    try:
        out = model.detect(x, is_video=False)["preds"]
        torch.cuda.synchronize()
        n = L.vsb_profile_read(None, 0)
        buf = C.create_string_buffer(int(n) + 16)
        L.vsb_profile_read(buf, len(buf))
    finally:
        L.vsb_profile_enable(0)
    rows = [line.split("\t") for line in buf.value.decode().splitlines()]
    return out, {r[0]: int(r[2]) for r in rows if len(r) >= 3}


def results(cfg: str) -> dict:
    """runs one detect call of the configuration and judges every pixel-decoder step from its taps (memoised: the taps belong to
    the most recent call, so each configuration is judged right after its own call)"""
    if cfg in _results:
        return _results[cfg]
    ext, stages, S, B, _, _ = pk.CONFIGS[cfg]
    model, sd, spec = _model(cfg)
    g = torch.Generator().manual_seed(S + B)
    imgs = torch.rand(B, 3, S, S, generator=g)      # already at the processing size: no resize
    maps, prof = _profiled_detect(model, imgs.cuda())
    b0 = (B - 1) // 64 * 64                          # the taps are those of the last 64-frame sub-batch
    names = {n for n in prof if n.startswith("pd.")}
    cache = {}

    def tap(n):
        if n not in cache:
            cache[n] = model.debug_tensor(n).permute(0, 3, 1, 2).to("cuda", torch.float64)
        return cache[n]
    # stage i ran the untiled gather when its profile name says so (the head is always tiled)
    tiled = [not any(n.startswith("pd.upgather_untiled.") and n.endswith(f"@{tap(f'pd{i}').shape[-1]}") for n in names)
             if i + 1 < len(stages) else True for i in range(len(stages))]
    sd64 = {k: v.to("cuda", torch.float64) for k, v in sd.items() if k.startswith(pk.D)}
    x0 = tap("vit.neck" if ext == "vit" else "stage3_16")
    steps = []
    with torch.no_grad():
        for c in pk.plan_checks(sd64, stages, x0, tap, maps[b0:].to(torch.float64), tiled):
            assert c.got.shape == c.ref.shape and c.got.shape[0] == B - b0, (c.step, c.got.shape, c.ref.shape)
            steps.append(ck.judge(c))
            del c
    cache.clear()
    del maps
    torch.cuda.empty_cache()
    _results[cfg] = {"names": names, "steps": steps}
    return _results[cfg]


@pytest.mark.parametrize("cfg", list(pk.CONFIGS))
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


def test_every_mutation_is_detected():
    """each mutation is violated in every step family that has it, over all configurations, and the violations of border-,
    tile-edge- and last-frame-only defects lie inside their footprints, at every step"""
    hits, bad = {}, []
    for cfg in pk.CONFIGS:
        for s in results(cfg)["steps"]:
            for m in s["mutations"]:
                print(f"[{cfg}] {s['step']}: {m['name']}: {m['violations']} violations"
                      + (f" ({m['outside']} off the footprint {m['where']})" if m["where"] is not None else ""))
                key = (pk.family(s["step"]), m["name"])
                hits[key] = hits.get(key, 0) + m["violations"]
                if m["outside"] != 0:
                    bad.append((cfg, s["step"], m))
    for (fam, name), n in sorted(hits.items()):
        print(f"[mutations] {fam}: {name}: {n} violations")
    missed = sorted(k for k, n in hits.items() if n == 0)
    assert not bad and not missed, (bad, missed)


@pytest.mark.parametrize("cfg", list(pk.CONFIGS))
def test_dispatch_is_pinned(cfg):
    names = results(cfg)["names"]
    print(f"[{cfg}] {sorted(names)}")
    assert names == EXPECT[cfg], (sorted(EXPECT[cfg] - names), sorted(names - EXPECT[cfg]))


def _vpt(c: int) -> int:
    """Decoder::vpt: 16-byte vectors per thread of a C-channel intermediate stage"""
    return next(v for v in (1, 3) if c % (8 * v) == 0 and (c // (8 * v)) & (c // (8 * v) - 1) == 0 and c // (8 * v) <= 32)


def test_dispatch_union_covers_every_instantiation():
    """the configurations reach every fused head (F 2 / 4 x VPT 1..4) and every (F, VPT) gather, tiled and untiled, that a model can
    dispatch (untiled F4/VPT1 cannot be: see tests/pd_kernels.py)"""
    got = set()
    for cfg in pk.CONFIGS:
        for n in results(cfg)["names"]:
            _, kind, geo = n.split(".")
            if kind == "uptap1x1":
                continue
            c, f = (int(v) for v in geo.split("@")[0].split("x"))
            got.add((kind, f, c // 8 if kind == "gather_head" else _vpt(c)))
    print("[dispatch union]", sorted(got))
    need = {("gather_head", f, v) for f in (2, 4) for v in (1, 2, 3, 4)} | {("upgather", f, v) for f in (2, 4) for v in (1, 3)}
    need |= {("upgather_untiled", 2, 1), ("upgather_untiled", 2, 3), ("upgather_untiled", 4, 3)}
    assert need <= got, sorted(need - got)


def test_taps_leave_the_maps_unchanged():
    """the pd{i}_y taps are pointers into the plan's own buffers: the plan runs no extra step and repeated calls give bit-identical
    maps"""
    model, _, _ = _model("tiny256_424")
    x = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(7)).cuda()
    a, pa = _profiled_detect(model, x)
    b, pb = _profiled_detect(model, x)
    assert not any(n.startswith("dbg.") for n in pa) and pa == pb
    assert torch.equal(a, b)
    for i in range(3):
        assert model.debug_tensor(f"pd{i}_y").shape[-1] == 9 * (192, 96, 24)[i]
