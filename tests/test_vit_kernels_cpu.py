"""The per-kernel float64 references and error bounds of tests/vit_kernels.py, checked without a GPU, at two frames of every
configuration tests/test_vit_kernels_gpu.py runs: chained, they reproduce vit_oracle.trunk_forward and
restate.sam_extractor_forward; each bound covers an emulation of its step in the kernels' precision (fp16 operands, fp32
accumulation in 64-wide K blocks); each mutation moves the reference by more than the bound; and every configuration passes the
load-time rules through the library's dry run."""
import functools

import pytest
import torch

from oracle import restate
from tests import vit_kernels as vk
from tests import vit_oracle as vo

# the steps whose reference rounds what the float64 chain keeps exact (the pixels, the stream, the relative-position tables the
# attention kernel stages in fp16): the emulation checks them
ROUNDING_STEPS = {"vit_patch_im2col", "x16 copy", "attention"}


def _case(cfg: str, zero_unused_bias: bool = False):
    enc, S, _ = vk.CONFIGS[cfg]
    spec = vo.spec_from_card(vo.vit_card(False, S, enc))
    sd = vo.synth_state_dict(spec)
    if zero_unused_bias and not spec["vit"]["qkv_bias"]:   # restate adds the qkv bias unconditionally: a zero one stands for none
        for k in [k for k in sd if k.endswith("attn.qkv.bias")]:
            sd[k] = torch.zeros_like(sd[k])
    imgs = torch.rand(2, 3, S, S, generator=torch.Generator().manual_seed(S)).to(torch.float64)
    return vk.Vit(sd, spec), spec, sd, imgs


@functools.lru_cache(maxsize=None)
def _chain(cfg: str, zero_unused_bias: bool = False):
    """the float64 chain of a configuration, shared by the tests that read it"""
    vt, spec, sd, imgs = _case(cfg, zero_unused_bias)
    taps = vk.chain(vt, imgs)
    taps["imgs"] = imgs
    return vt, spec, sd, imgs, taps


def _checks(vt, taps):
    return vk.plan_checks(vt, lambda n: taps[n], taps["imgs"], taps["logits"])


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_chained_references_reproduce_the_extractor(cfg):
    vt, spec, sd, imgs, taps = _chain(cfg, zero_unused_bias=True)
    sd64 = {k: v.to(torch.float64) for k, v in sd.items() if v.is_floating_point()}
    rt = {}
    vo.trunk_forward(sd64, spec, imgs, rt)
    last = rt[f"blk{vt.L}"]
    assert (taps[f"vit.blk{vt.L}"] - last).abs().max() <= 1e-12 * last.abs().max()
    neck = vk.nhwc(rt["neck"])
    assert (taps["vit.neck"] - neck).abs().max() <= 1e-12 * neck.abs().max()
    ref = restate.sam_extractor_forward(sd64, spec, imgs)
    assert (taps["logits"] - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    worst = 0.0
    for c in _checks(vt, taps):
        if c.step in ROUNDING_STEPS:
            continue
        rel = ((c.got - c.ref).abs().max() / c.ref.abs().max().clamp_min(1e-30)).item()
        worst = max(worst, rel)
        assert rel <= 1e-12, (c.step, rel)
    print(f"[{cfg}] chained references: max relative difference {worst:.2e}")


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_bounds_cover_emulation(cfg):
    vt, spec, sd, imgs = _case(cfg)
    taps = vk.chain(vt, imgs, emulate=True)
    taps["imgs"] = imgs
    for c in _checks(vt, taps):
        r = vk.ck.judge(c)
        print(f"[{cfg}] emulated err / bound {r['ratio']:.3f}  {c.step}")
        assert not r["nan"] and r["ratio"] <= 1.0 and r["fallback"] == 0, (c.step, r["ratio"], r["fallback"])


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_mutations_move_the_reference_beyond_the_bound(cfg):
    """each deliberate defect changes the float64 reference by more than the step's bound somewhere, and only on the border / in
    the last frame where that is its footprint"""
    # the bias-less configuration keeps the checkpoint's unused qkv bias (its mutation adds it); elsewhere zeroing changes nothing
    # and the chain is the one the test above made
    vt, spec, sd, imgs, taps = _chain(cfg, zero_unused_bias=vk.CONFIGS[cfg][0].get("qkv_bias", True))
    seen = set()
    for c in _checks(vt, taps):
        for mname, mref, where in c.mutations:
            v = (mref - c.ref).abs() > c.tol
            assert v.any(), (c.step, mname)
            assert vk.ck.outside(v, where) == 0, (c.step, mname)
            seen.add((c.step, mname))
    print(f"[{cfg}] mutations detected: {sorted(seen)}")


@pytest.mark.parametrize("cfg", list(vk.CONFIGS))
def test_every_configuration_passes_the_load_rules(cfg):
    from videoseal_b200 import cfg as vcfg
    enc, S, _ = vk.CONFIGS[cfg]
    spec = vcfg.spec_from_card(vo.vit_card(False, S, enc))   # the native library's dry run: raises on a rule the kernels break
    v = spec["vit"]
    assert spec["img_size"] == S and v["depth"] == enc["depth"]
    assert v["embed_dim"] == enc.get("embed_dim", 384) and v["out_chans"] == enc.get("out_chans", 384)
