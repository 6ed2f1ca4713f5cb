"""The per-kernel float64 references and error bounds of tests/cnx_kernels.py, checked without a GPU: chained, they reproduce
restate.convnext_extractor_forward; each bound covers an emulation of its step in the kernels' precision (fp32 arithmetic, the
stem's one-pass LayerNorm, fp16 roundings; ATen's summation order, not the kernels'); each mutation moves the reference by more
than the bound.  The tiny trunk runs at depth 1 and at its card's depth; the chunkyseal trunk (362..2896 channels, stem
stride 2, odd maps) at depth 1 and at two blocks on stages 0 and 2 (its card's 3, 3, 27, 3 is several GB of float64 weights)."""
import pytest
import torch

from oracle import restate
from tests import cnx_kernels as ck
from tests.util import apply_overrides, load_card

TRUNKS = {   # name: (card, depths, processing size)
    "tiny_d1": ("videoseal_1.0", [1, 1, 1, 1], 128),
    "tiny_card": ("videoseal_1.0", None, 128),
    "chunky_d1": ("chunkyseal", [1, 1, 1, 1], 64),
    "chunky_d2": ("chunkyseal", [2, 1, 2, 1], 64),
}


@pytest.fixture(scope="module", params=list(TRUNKS))
def case(request):
    card_name, depths, S = TRUNKS[request.param]
    card = load_card(card_name)
    if depths:
        card = apply_overrides(card, {"depths": depths})
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, seed=1234)
    g = torch.Generator().manual_seed(0)
    imgs = torch.rand(2, 3, S, S, generator=g).to(torch.float64)
    return request.param, ck.Trunk(sd, spec), spec, sd, imgs


def _checks(tr, taps, fold):
    return ck.plan_checks(tr, lambda n: taps[n], lambda n: fold[int(n[1])] and n in taps, taps["imgs"], taps["logits"])


FOLDS = {"fold": [True] * 4, "apply": [False] * 4}


@pytest.mark.parametrize("mode", list(FOLDS))
def test_chained_references_reproduce_the_extractor(case, mode):
    """each step's reference, fed the float64 taps of the steps before, reproduces that step's tap; the chain ends at
    restate.convnext_extractor_forward in float64 (the GRN fold into W2 / its beta into the bias included)"""
    name, tr, spec, sd, imgs = case
    taps = ck.chain(tr, imgs, FOLDS[mode])
    taps["imgs"] = imgs
    rt = {}
    ref = restate.convnext_extractor_forward(tr.sd, spec, imgs, rt)
    for s in range(4):
        assert (taps[f"stage{s}"] - rt[f"stage{s}"]).abs().max() <= 1e-12 * rt[f"stage{s}"].abs().max(), s
    assert (taps["logits"] - ref).abs().max().item() <= 1e-12 * ref.abs().max().item()
    worst = 0.0
    for c in _checks(tr, taps, FOLDS[mode]):
        rel = ((c.got - c.ref).abs().max() / c.ref.abs().max().clamp_min(1e-30)).item()
        worst = max(worst, rel)
        assert rel <= 1e-12, (c.step, rel)
    print(f"[{name} {mode}] chained references: max relative difference {worst:.2e}")


@pytest.mark.parametrize("mode", list(FOLDS))
def test_bounds_cover_emulation(case, mode):
    """every step's bound holds for an emulation of its kernel in fp32 arithmetic with its fp16 roundings"""
    name, tr, spec, sd, imgs = case
    taps = ck.chain(tr, imgs, FOLDS[mode], emulate=True)
    taps["imgs"] = imgs
    worst = {}
    for c in _checks(tr, taps, FOLDS[mode]):
        r = ck.judge(c)
        assert not r["nan"] and r["ratio"] <= 1.0 and r["fallback"] == 0, (c.step, r["ratio"], r["fallback"])
        f = ck.family(c.step)
        worst[f] = max(worst.get(f, 0.0), r["ratio"])
    for f, r in sorted(worst.items()):
        print(f"[{name} {mode}] emulated err / bound {r:.3f}  {f}")


@pytest.mark.parametrize("mode", list(FOLDS))
def test_mutations_move_the_reference_beyond_the_bound(case, mode):
    """each deliberate defect changes the float64 reference by more than the step's bound somewhere, and only on the border /
    in the last frame where that is its footprint"""
    name, tr, spec, sd, imgs = case
    taps = ck.chain(tr, imgs, FOLDS[mode])
    taps["imgs"] = imgs
    seen = set()
    for c in _checks(tr, taps, FOLDS[mode]):
        for mname, mref, where in c.mutations:
            v = (mref - c.ref).abs() > c.tol
            assert v.any(), (c.step, mname)
            assert ck.outside(v, where) == 0, (c.step, mname)
            seen.add((ck.family(c.step), mname))
    print(f"[{name} {mode}] mutations detected: {sorted(seen)}")
