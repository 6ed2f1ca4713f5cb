"""Every kernel of the ConvNeXt detect plan on its own inputs (the plan's debug taps, with vsb_debug_keep_inputs on) against float64
references with derived error bounds (tests/cnx_kernels.py), at each trunk geometry and GRN mode detect dispatches; mutated
references prove the bounds see the defects that matter; the profile names pin which kernel variant each configuration runs."""
import ctypes as C

import pytest
import torch

from tests import cnx_kernels as ck
from tests.util import make_model_pair

pytestmark = pytest.mark.gpu

D1 = {"depths": [1, 1, 1, 1]}
# name: (card, overrides, processing size, frames)
CONFIGS = {
    "v1_256_b64": ("videoseal_1.0", D1, 256, 64),        # stem GEMM; rings R 32; full-row strips; fold at s0-s1; partial rows
    "v1_256_b70": ("videoseal_1.0", D1, 256, 70),        # taps of the 6-frame second sub-batch
    "v1_128_b64": ("videoseal_1.0", D1, 128, 64),        # ring 192@16 (R 16); edge strips; float-atomic GRN statistics
    "v1_384_b5": ("videoseal_1.0", D1, 384, 5),          # ring 192@48 (R 16); ragged 768@12 strip; atomics; odd batch
    "v1_full_128_b16": ("videoseal_1.0", None, 128, 16),  # last block of each stage: statistics ping-pong across blocks
    "v1_full_256_b16": ("videoseal_1.0", None, 256, 16),  # last block, partial rows, head at full depth
    "chunky_256_b4": ("chunkyseal", D1, 256, 4),         # stem_ln_kernel; wide dwconv on padded rows; odd maps; atomics
    "base_256_b16": ("videoseal_1.0", {"extractor": "convnext_base", **D1}, 256, 16),   # wide dwconv on dense rows, fold at 128 / 256
}

# every ConvNeXt step name each geometry runs (vsb_profile_read; "cnx." prefix omitted)
V1_256 = """stem_im2col stem_gemm.96@64 dwconv7_ln.ring.96@64 pwconv1.96@64 grn_wscale.96@64 pwconv2.96@64 ln_rows
    down2x2s2.96-192@32 dwconv7_ln.ring.192@32 pwconv1.192@32 grn_wscale.192@32 pwconv2.192@32 down2x2s2.192-384@16
    dwconv7_ln.row.384@16 pwconv1.384@16 grn_apply.384@16 pwconv2.384@16 down2x2s2.384-768@8 dwconv7_ln.row.768@8 pwconv1.768@8
    grn_apply.768@8 pwconv2.768@8 head3x3.768@8 head_tail"""
V1_128 = """stem_im2col stem_gemm.96@32 grn_clear dwconv7_ln.ring.96@32 pwconv1.96@32 grn_wscale.96@32 pwconv2.96@32 ln_rows
    down2x2s2.96-192@16 dwconv7_ln.ring.192@16 pwconv1.192@16 grn_apply.192@16 pwconv2.192@16 down2x2s2.192-384@8
    dwconv7_ln.strip.384@8 pwconv1.384@8 grn_apply.384@8 pwconv2.384@8 down2x2s2.384-768@4 dwconv7_ln.strip.768@4 pwconv1.768@4
    grn_apply.768@4 pwconv2.768@4 head3x3.768@4 head_tail"""
EXPECT = {
    "v1_256_b64": V1_256, "v1_256_b70": V1_256, "v1_full_256_b16": V1_256, "v1_128_b64": V1_128, "v1_full_128_b16": V1_128,
    "v1_384_b5": """stem_im2col stem_gemm.96@96 grn_clear dwconv7_ln.ring.96@96 pwconv1.96@96 grn_wscale.96@96 pwconv2.96@96 ln_rows
        down2x2s2.96-192@48 dwconv7_ln.ring.192@48 pwconv1.192@48 grn_wscale.192@48 pwconv2.192@48 down2x2s2.192-384@24
        dwconv7_ln.strip.384@24 pwconv1.384@24 grn_apply.384@24 pwconv2.384@24 down2x2s2.384-768@12 dwconv7_ln.strip.768@12
        pwconv1.768@12 grn_apply.768@12 pwconv2.768@12 head3x3.768@12 head_tail""",
    "chunky_256_b4": """stem_ln.362@127 grn_clear dwconv7_ln.wide.362@127 pwconv1.362@127 grn_apply.362@127 pwconv2.362@127 ln_rows
        down2x2s2.362-724@63 dwconv7_ln.wide.724@63 pwconv1.724@63 grn_apply.724@63 pwconv2.724@63 down2x2s2.724-1448@31
        dwconv7_ln.wide.1448@31 pwconv1.1448@31 grn_apply.1448@31 pwconv2.1448@31 down2x2s2.1448-2896@15 dwconv7_ln.wide.2896@15
        pwconv1.2896@15 grn_apply.2896@15 pwconv2.2896@15 head3x3.2896@15 head_tail""",
    "base_256_b16": """stem_im2col stem_gemm.128@64 dwconv7_ln.wide.128@64 pwconv1.128@64 grn_wscale.128@64 pwconv2.128@64 ln_rows
        down2x2s2.128-256@32 dwconv7_ln.wide.256@32 pwconv1.256@32 grn_wscale.256@32 pwconv2.256@32 down2x2s2.256-512@16
        dwconv7_ln.wide.512@16 pwconv1.512@16 grn_apply.512@16 pwconv2.512@16 down2x2s2.512-1024@8 dwconv7_ln.wide.1024@8
        pwconv1.1024@8 grn_apply.1024@8 pwconv2.1024@8 head3x3.1024@8 head_tail""",
}
EXPECT = {k: {"cnx." + n for n in v.split()} for k, v in EXPECT.items()}

_models, _results = {}, {}


def _lib():
    from videoseal_b200 import _lib as lib
    return lib


def _model(card, ov):
    key = (card, str(ov))
    if key not in _models:
        _models[key] = make_model_pair(card, tiny=ov)
    return _models[key]


@pytest.fixture(scope="module", autouse=True)
def _release():
    yield
    for m, _, _ in _models.values():
        m._release()
    _models.clear()


def _profiled_detect(model, x, keep: bool):
    """(logits, {profile step name: launches}) of one detect call with the input-keeping seam set to `keep`"""
    L = _lib().lib()
    _lib().check(L.vsb_debug_keep_inputs(model._handle(), int(keep)))
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
    """runs one detect call of the configuration with the seam on and judges every step from its taps (memoised: the taps belong
    to the most recent call, so each configuration is judged right after its own call)"""
    if cfg in _results:
        return _results[cfg]
    card, ov, S, B = CONFIGS[cfg]
    model, orc, spec = _model(card, ov)
    model.img_size = S
    g = torch.Generator().manual_seed(S + B)
    imgs = torch.rand(B, 3, S, S, generator=g)      # already at the processing size: no resize, the stem reads these frames
    logits, prof = _profiled_detect(model, imgs.cuda(), True)
    b0 = (B - 1) // 64 * 64                          # the taps are those of the last 64-frame sub-batch
    tr = ck.Trunk(orc.sd, spec, "cuda")
    cache = {}

    def tap(n):
        if n not in cache:
            t = model.debug_tensor(n)
            if n.endswith("_w2s"):
                t = t[:, :, 0, :]                        # [B, C, 1, 4C] -> [B, C, 4C]
            elif n == "head_pooled":
                t = t[:, 0, 0, :]
            else:
                t = t.permute(0, 3, 1, 2)
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
        for c in ck.plan_checks(tr, tap, has_tap, imgs[b0:].cuda(), logits[b0:].cuda()):
            assert c.got.shape == c.ref.shape and c.got.shape[0] == B - b0, (c.step, c.got.shape, c.ref.shape)
            steps.append(ck.judge(c))
            del c
    # the dwconv variant of each stage, from its profile name cnx.dwconv7_ln.<variant>.<C>@<map>
    kind = {int(n.split(".")[3].split("@")[0]): n.split(".")[2] for n in prof if n.startswith("cnx.dwconv7_ln.")}
    for st in steps:
        if ck.family(st["step"]) == "dwconv7_ln":
            st["family"] = "dwconv7_ln." + kind[spec["convnext"]["dims"][int(st["step"][1])]]
    cache.clear()
    torch.cuda.empty_cache()
    _results[cfg] = {"names": {n for n in prof if n.startswith("cnx.")}, "steps": steps}
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


@pytest.mark.parametrize("cfg", list(CONFIGS))
def test_every_mutation_is_detected(cfg):
    """each mutation is violated in every step family that has it (each dwconv variant is a family of its own), and the violations
    of border-only / last-frame-only defects lie on the border / in the last frame, at every step"""
    r = results(cfg)
    hits, bad = {}, []
    for s in r["steps"]:
        for m in s["mutations"]:
            print(f"[{cfg}] {s['step']}: {m['name']}: {m['violations']} violations"
                  + (f" ({m['outside']} off the footprint {m['where']})" if m["where"] is not None else ""))
            key = (s.get("family", ck.family(s["step"])), m["name"])
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


def test_dispatch_union_covers_every_family():
    fams = set()
    for cfg in CONFIGS:
        for n in results(cfg)["names"]:
            p = n.split(".")
            fams.add(".".join(p[1:3]) if p[1] == "dwconv7_ln" else p[1])
    print("[dispatch union]", sorted(fams))
    need = {"stem_im2col", "stem_gemm", "stem_ln", "grn_clear", "ln_rows", "down2x2s2", "dwconv7_ln.ring", "dwconv7_ln.row",
            "dwconv7_ln.strip", "dwconv7_ln.wide", "pwconv1", "grn_wscale", "grn_apply", "pwconv2", "head3x3", "head_tail"}
    assert need <= fams, sorted(need - fams)


def test_kept_inputs_leave_the_plan_and_the_logits_unchanged():
    """with the seam on, the plan runs the same ConvNeXt steps plus the copies, and the logits are bit-identical (per-warp partial
    GRN rows: run to run reproducible)"""
    model, _, _ = _model("videoseal_1.0", D1)
    model.img_size = 256
    x = torch.rand(4, 3, 256, 256, generator=torch.Generator().manual_seed(7)).cuda()
    off, p_off = _profiled_detect(model, x, False)
    on, p_on = _profiled_detect(model, x, True)
    _, p_off2 = _profiled_detect(model, x, False)
    keep = {n for n in p_on if n.startswith("dbg.keep.")}
    assert keep == {f"dbg.keep.s{s}_ds" for s in range(4)}, keep
    assert not any(n.startswith("dbg.") for n in p_off) and p_off == p_off2
    assert {n: c for n, c in p_on.items() if n not in keep} == p_off
    assert torch.equal(off, on)
