"""Every kernel of the SAM-ViT detect plan on its own inputs (the plan's debug taps, with vsb_debug_keep_inputs on) against float64
references with derived error bounds (tests/vit_kernels.py), at each width, token grid and batch the configurations of
vit_kernels.CONFIGS reach; mutated references prove the bounds see the defects that matter; the step names and the GEMM dispatch
record (vsb_debug_plan_gemms) pin which kernel variant each configuration runs."""
import ctypes as C

import pytest
import torch

from tests import cnx_kernels as ck
from tests import vit_kernels as vk
from tests import vit_oracle as vo

pytestmark = pytest.mark.gpu

_results = {}


def _lib():
    from videoseal_b200 import _lib as lib
    return lib


def _text(read) -> str:
    n = read(None, 0)
    assert n > 0
    buf = C.create_string_buffer(int(n) + 16)
    read(buf, len(buf))
    return buf.value.decode()


def _profiled_detect(model, x, keep: bool):
    """(logits, {profile step name: launches}, the GEMM record of the last sub-batch's plan) of one detect call with the
    input-keeping seam set to `keep`"""
    L = _lib().lib()
    _lib().check(L.vsb_debug_keep_inputs(model._handle(), int(keep)))
    L.vsb_profile_enable(1)         # clears what earlier calls accumulated
    try:
        out = model.detect(x, is_video=False)["preds"]
        torch.cuda.synchronize()
        prof = _text(L.vsb_profile_read)
    finally:
        L.vsb_profile_enable(0)
    gemms = _text(lambda b, n: L.vsb_debug_plan_gemms(model._handle(), b, n))
    rows = [line.split("\t") for line in prof.splitlines()]
    return out, {r[0]: int(r[2]) for r in rows if len(r) >= 3}, [g for g in gemms.splitlines() if g]


def results(cfg: str) -> dict:
    """runs one detect call of the configuration with the seam on and judges every step from its taps (memoised)"""
    if cfg in _results:
        return _results[cfg]
    enc, S, B = vk.CONFIGS[cfg]
    model, orc, spec = vo.model_pair(False, img_size=S, encoder=enc)
    try:
        imgs = torch.rand(B, 3, S, S, generator=torch.Generator().manual_seed(S + B))   # at the processing size: no resize
        logits, prof, gemms = _profiled_detect(model, imgs.cuda(), True)
        b0 = (B - 1) // 64 * 64                          # the taps are those of the last 64-frame sub-batch
        vt = vk.Vit(orc.sd, spec, "cuda")
        cache = {}

        def tap(n):
            if n not in cache:
                cache[n] = model.debug_tensor(n).to("cuda", torch.float64)
            return cache[n]
        steps = []
        with torch.no_grad():
            for c in vk.plan_checks(vt, tap, imgs[b0:].to("cuda", torch.float64), logits[b0:]):
                assert c.got.shape == c.ref.shape and c.got.shape[0] == B - b0, (c.step, c.got.shape, c.ref.shape)
                steps.append(ck.judge(c))
                del c
        cache.clear()
    finally:
        model._release()
        torch.cuda.empty_cache()
    _results[cfg] = {"names": {n for n in prof if n.startswith("vit.")}, "gemms": [g for g in gemms if g.startswith("vit.")],
                     "steps": steps}
    return _results[cfg]


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_every_step_within_its_bound(cfg):
    r = results(cfg)
    bad = []
    for s in r["steps"]:
        print(f"[{cfg}] max err/tol {s['ratio']:.3f}  {s['step']}" + (f"  (LayerNorm range fallback on {s['fallback']:.2e} of rows)"
                                                                    if s["fallback"] else ""))
        if s["nan"] or not s["ratio"] <= 1.0 or s["fallback"] > 0:
            bad.append((s["step"], s["ratio"], s["nan"], s["fallback"]))
    assert not bad, bad


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_every_mutation_is_detected(cfg):
    """each mutation is violated in every step that has it, and the violations of border-only / last-frame-only defects lie on
    the border / in the last frame"""
    r = results(cfg)
    hits, bad = {}, []
    for s in r["steps"]:
        for m in s["mutations"]:
            print(f"[{cfg}] {s['step']}: {m['name']}: {m['violations']} violations"
                  + (f" ({m['outside']} off the footprint {m['where']})" if m["where"] is not None else ""))
            hits[(s["step"], m["name"])] = m["violations"]
            if m["outside"] != 0:
                bad.append((s["step"], m))
    missed = sorted(k for k, n in hits.items() if n == 0)
    assert not bad and not missed, (bad, missed)


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_dispatch_is_pinned(cfg):
    r = results(cfg)
    print(f"[{cfg}] {sorted(r['names'])}")
    for g in r["gemms"]:
        print(f"[{cfg}] {g}")
    assert r["names"] == EXPECT_NAMES[cfg], (sorted(EXPECT_NAMES[cfg] - r["names"]), sorted(r["names"] - EXPECT_NAMES[cfg]))
    got = {" ".join([g.split("\t")[0]] + [kv.split("=")[1] for kv in g.split("\t")[1:]]) for g in r["gemms"]}
    want = {" ".join(line.split()) for line in EXPECT_GEMMS[cfg].strip().splitlines()}
    assert got == want, (sorted(want - got), sorted(got - want))


def test_kept_inputs_leave_the_plan_and_the_logits_unchanged():
    """with the seam on, the plan runs the same ViT steps plus the copies, with the same GEMM variants, and the logits and every
    tap both runs have are bit-identical"""
    enc, S, _ = vk.CONFIGS["small_256_b3"]
    model, _, _ = vo.model_pair(False, img_size=S, encoder=enc)
    try:
        x = torch.rand(4, 3, S, S, generator=torch.Generator().manual_seed(7)).cuda()
        taps = ["vit.patches", "vit.embed", "vit.blk1.qkv", "vit.blk1.attn", "vit.blk1.ln2", "vit.blk1.hid", "vit.blk1", "vit.x16",
                "vit.neck_ln1", "vit.neck3x3", "vit.neck", "head_conv", "head_pooled"]
        off, p_off, g_off = _profiled_detect(model, x, False)
        t_off = {n: model.debug_tensor(n) for n in taps}
        on, p_on, g_on = _profiled_detect(model, x, True)
        t_on = {n: model.debug_tensor(n) for n in taps}
        _, p_off2, _ = _profiled_detect(model, x, False)
    finally:
        model._release()
    keep = {n for n in p_on if n.startswith("dbg.keep.")}
    assert keep == {"dbg.keep.vit.blk1.in", "dbg.keep.vit.blk1.ln1", "dbg.keep.vit.blk1.mid", "dbg.keep.vit.neck1x1"}, keep
    assert not any(n.startswith("dbg.") for n in p_off) and p_off == p_off2
    assert {n: c for n, c in p_on.items() if n not in keep} == p_off
    assert g_on == g_off
    assert torch.equal(off, on)
    for n in taps:
        assert torch.equal(t_off[n], t_on[n]), n


# every ViT step name each configuration runs (vsb_profile_read): the common ones, the attention regions and the head
_COMMON = {'vit.head_tail', 'vit.lin1', 'vit.lin2', 'vit.ln', 'vit.neck1x1', 'vit.neck3x3', 'vit.neck_ln', 'vit.patch', 'vit.proj', 'vit.qkv'}
EXPECT_NAMES = {
    'small_256_b3': _COMMON | {'vit.attn_global.256', 'vit.attn_win.64', 'vit.head3x3.384@16'},
    'small_256_b64': _COMMON | {'vit.attn_global.256', 'vit.attn_win.64', 'vit.head3x3.384@16'},
    'small_256_b70': _COMMON | {'vit.attn_win.64', 'vit.head3x3.384@16'},
    'tiny_256_b4': _COMMON | {'vit.attn_global.256', 'vit.attn_win.64', 'vit.head3x3.192@16'},
    'base_256_b3': _COMMON | {'vit.attn_global.256', 'vit.attn_win.64', 'vit.head3x3.768@16'},
    'small_128_b3': _COMMON | {'vit.attn_win.64', 'vit.head3x3.384@8'},
    'small_384_b3': _COMMON | {'vit.attn_global.576', 'vit.attn_win.64', 'vit.head3x3.384@24'},
    'small_512_b2': _COMMON | {'vit.attn_global.1024', 'vit.attn_win.64', 'vit.head3x3.384@32'},
    'win40_640_b2': _COMMON | {'vit.attn_win.1600', 'vit.head3x3.384@40'},
    'nobias_norel_256_b3': _COMMON | {'vit.attn_win.64', 'vit.head3x3.384@16'},
    'e448_256_b3': _COMMON | {'vit.attn_win.64', 'vit.head3x3.320@16'},
}
# the distinct GEMM records of each configuration's last plan (vsb_debug_plan_gemms), ViT steps only:
#   name  M  N  K  block_n  tma_store  b_resident  b_fixed_ntile  kernel  bias_global  m_tiles
EXPECT_GEMMS = {
    'small_256_b3': """
        vit.head3x3.384@16 768 384 3456 128 0 0 0 128 0 whole
        vit.lin1 768 1536 384 128 1 0 0 128 1 whole
        vit.lin2 768 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 768 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 768 384 3456 128 0 0 0 128 0 whole
        vit.patch 768 384 768 128 0 0 0 128 0 whole
        vit.proj 768 384 384 64 2 0 0 128 1 whole
        vit.qkv 768 1152 384 128 1 0 0 128 1 whole
        """,
    'small_256_b64': """
        vit.head3x3.384@16 16384 384 3456 128 0 0 0 128 0 whole
        vit.lin1 16384 1536 384 128 1 0 0 128 1 whole
        vit.lin2 16384 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 16384 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 16384 384 3456 128 0 0 0 128 0 whole
        vit.patch 16384 384 768 128 0 0 0 128 0 whole
        vit.proj 16384 384 384 64 2 0 0 128 1 whole
        vit.qkv 16384 1152 384 128 1 0 0 128 1 whole
        """,
    'small_256_b70': """
        vit.head3x3.384@16 1536 384 3456 128 0 0 0 128 0 whole
        vit.lin1 1536 1536 384 128 1 0 0 128 1 whole
        vit.lin2 1536 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 1536 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 1536 384 3456 128 0 0 0 128 0 whole
        vit.patch 1536 384 768 128 0 0 0 128 0 whole
        vit.proj 1536 384 384 64 2 0 0 128 1 whole
        vit.qkv 1536 1152 384 128 1 0 0 128 1 whole
        """,
    'tiny_256_b4': """
        vit.head3x3.192@16 1024 192 1728 96 0 0 0 128 0 whole
        vit.lin1 1024 768 192 128 1 0 0 128 1 whole
        vit.lin2 1024 192 768 64 0 0 0 128 1 whole
        vit.lin2 1024 192 768 64 2 0 0 128 1 whole
        vit.neck1x1 1024 192 192 96 0 0 0 128 0 whole
        vit.neck3x3 1024 192 1728 96 0 0 0 128 0 whole
        vit.patch 1024 192 768 96 0 0 0 128 0 whole
        vit.proj 1024 192 192 64 2 0 0 128 1 whole
        vit.qkv 1024 576 192 96 1 0 0 128 1 whole
        """,
    'base_256_b3': """
        vit.head3x3.768@16 768 768 6912 128 0 0 0 128 0 whole
        vit.lin1 768 3072 768 128 1 0 0 128 1 whole
        vit.lin2 768 768 3072 64 0 0 0 128 1 whole
        vit.neck1x1 768 768 768 128 0 0 0 128 0 whole
        vit.neck3x3 768 768 6912 128 0 0 0 128 0 whole
        vit.patch 768 768 768 128 0 0 0 128 0 whole
        vit.proj 768 768 768 64 2 0 0 128 1 whole
        vit.qkv 768 2304 768 128 1 0 0 128 1 whole
        """,
    'small_128_b3': """
        vit.head3x3.384@8 192 384 3456 128 0 0 0 128 0 ragged
        vit.lin1 192 1536 384 128 0 0 0 128 1 ragged
        vit.lin2 192 384 1536 64 0 0 0 128 1 ragged
        vit.neck1x1 192 384 384 128 0 0 0 128 0 ragged
        vit.neck3x3 192 384 3456 128 0 0 0 128 0 ragged
        vit.patch 192 384 768 128 0 0 0 128 0 ragged
        vit.proj 192 384 384 64 0 0 0 128 1 ragged
        vit.qkv 192 1152 384 128 0 0 0 128 1 ragged
        """,
    'small_384_b3': """
        vit.head3x3.384@24 1728 384 3456 128 0 0 0 128 0 ragged
        vit.lin1 1728 1536 384 128 0 0 0 128 1 ragged
        vit.lin2 1728 384 1536 64 0 0 0 128 1 ragged
        vit.neck1x1 1728 384 384 128 0 0 0 128 0 ragged
        vit.neck3x3 1728 384 3456 128 0 0 0 128 0 ragged
        vit.patch 1728 384 768 128 0 0 0 128 0 ragged
        vit.proj 1728 384 384 64 0 0 0 128 1 ragged
        vit.qkv 1728 1152 384 128 0 0 0 128 1 ragged
        """,
    'small_512_b2': """
        vit.head3x3.384@32 2048 384 3456 128 0 0 0 128 0 whole
        vit.lin1 2048 1536 384 128 1 0 0 128 1 whole
        vit.lin2 2048 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 2048 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 2048 384 3456 128 0 0 0 128 0 whole
        vit.patch 2048 384 768 128 0 0 0 128 0 whole
        vit.proj 2048 384 384 64 2 0 0 128 1 whole
        vit.qkv 2048 1152 384 128 1 0 0 128 1 whole
        """,
    'win40_640_b2': """
        vit.head3x3.384@40 3200 384 3456 128 0 0 0 128 0 whole
        vit.lin1 3200 1536 384 128 1 0 0 128 1 whole
        vit.lin2 3200 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 3200 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 3200 384 3456 128 0 0 0 128 0 whole
        vit.patch 3200 384 768 128 0 0 0 128 0 whole
        vit.proj 3200 384 384 64 2 0 0 128 1 whole
        vit.qkv 3200 1152 384 128 1 0 0 128 1 whole
        """,
    'nobias_norel_256_b3': """
        vit.head3x3.384@16 768 384 3456 128 0 0 0 128 0 whole
        vit.lin1 768 1536 384 128 1 0 0 128 1 whole
        vit.lin2 768 384 1536 64 0 0 0 128 1 whole
        vit.neck1x1 768 384 384 128 0 0 0 128 0 whole
        vit.neck3x3 768 384 3456 128 0 0 0 128 0 whole
        vit.patch 768 384 768 128 0 0 0 128 0 whole
        vit.proj 768 384 384 64 2 0 0 128 1 whole
        vit.qkv 768 1152 384 128 1 0 0 128 0 whole
        """,
    'e448_256_b3': """
        vit.head3x3.320@16 768 320 2880 80 0 0 0 128 0 whole
        vit.lin1 768 1792 448 128 1 0 0 128 1 whole
        vit.lin2 768 448 1792 64 0 0 0 128 1 whole
        vit.neck1x1 768 320 448 80 0 0 0 128 0 whole
        vit.neck3x3 768 320 2880 80 0 0 0 128 0 whole
        vit.patch 768 448 768 112 0 0 0 128 0 whole
        vit.proj 768 448 448 64 2 0 0 128 1 whole
        vit.qkv 768 1344 448 112 1 0 0 128 1 whole
        """,
}
