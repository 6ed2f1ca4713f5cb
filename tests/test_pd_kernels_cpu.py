"""The per-kernel float64 references and error bounds of tests/pd_kernels.py, checked without a GPU: chained from the trunk's
output they reproduce the pixel-wise oracles (tests/pixelwise_oracle.py, tests/vit_oracle.py); each bound covers an emulation of
its kernel in the kernels' precision (the packed fp16 corner mix in the kernel's order and index arithmetic, fp32 sums, fp16
roundings); each mutation moves the reference by more than the bound, and only inside its footprint.  Both factors and both
head factors run, on trunk maps of two tiles or more so that the tile-edge mutation has tiles to tell apart; every configuration
the GPU tests run is accepted at load."""
import pytest
import torch

from tests import cnx_kernels as ck
from tests import pd_kernels as pk
from tests import pixelwise_oracle as pw
from tests import vit_oracle as vo
from tests.util import apply_overrides, load_card

CASES = {   # name: (extractor, upscale stages); processing size 256, nbits 8
    "tiny_442": ("convnext_tiny_pw", [4, 4, 2]),    # trunk map 8: F4, F4, head F2 (24 channels)
    "base_424": ("convnext_base_pw", [4, 2, 4]),    # F4, F2, head F4 (32 channels)
    "vit_422": ("vit", [4, 2, 2]),                  # trunk map 16 (vit.neck, out_chans 256): F4, F2, head F2 (16 channels)
}


def build_case(name):
    """(name, float64 state dict, stages, the trunk's float64 output, the oracle's maps, tiled flags) of one case"""
    ext, stages = CASES[name]
    if ext == "vit":
        card = vo.vit_card(True, 256, {"out_chans": 256, "depth": 1}, stages)
        card["args"]["nbits"] = 8
        spec = vo.spec_from_card(card)
        sd = vo.synth_state_dict(spec, 5)
        fwd = vo.extractor_forward
        trunk = "neck"
    else:
        card = apply_overrides(pw.preset_card(ext, load_card("videoseal_1.0")), {"depths": [1, 1, 1, 1], "nbits": 8})
        card["extractor"]["params"]["pixel_decoder"]["upscale_stages"] = stages
        spec = pw.spec_from_card(card)
        sd = pw.synth_state_dict(spec, 5)
        fwd = pw.extractor_forward
        trunk = "stage3"
    imgs = torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    sd64 = {k: v.double() for k, v in sd.items()}
    taps = {}
    with torch.no_grad():
        maps = fwd(sd64, spec, imgs, taps)
    x0 = taps[trunk]
    tiled = [True] * len(stages)   # every stage's map here is a whole number of tiles, two or more a side
    return name, sd64, stages, x0, maps, tiled


@pytest.fixture(scope="module", params=list(CASES))
def case(request):
    return build_case(request.param)


def _checks(sd, stages, taps, x0, tiled):
    return pk.plan_checks(sd, stages, x0, lambda n: taps[n], taps["maps"], tiled)


def test_chained_references_reproduce_the_oracle(case):
    """the float64 chain from the trunk's output ends at the oracle's maps, and each step's reference reproduces the chain's tap"""
    name, sd, stages, x0, maps, tiled = case
    taps = pk.chain(sd, stages, x0)
    assert (taps["maps"] - maps).abs().max().item() <= 1e-12 * maps.abs().max().item()
    for c in _checks(sd, stages, taps, x0, tiled):
        rel = ((c.got - c.ref).abs().max() / c.ref.abs().max()).item()
        assert rel <= 1e-12, (c.step, rel)


def test_bounds_cover_emulation(case):
    """every step's bound holds for the emulation of its kernel from the fp16-rounded trunk output"""
    name, sd, stages, x0, maps, tiled = case
    x16 = ck.r16(x0)
    taps = pk.emulate(sd, stages, x16)
    for c in _checks(sd, stages, taps, x16, tiled):
        r = ck.judge(c)
        print(f"[{name}] emulated err / bound {r['ratio']:.3f}  {c.step}")
        assert not r["nan"] and r["ratio"] <= 1.0 and r["fallback"] == 0, (c.step, r["ratio"], r["fallback"])


def test_kernel_gather_is_the_bilinear_gather(case):
    """the kernel's index and weight arithmetic (src_table) is bilinear x F with reflect padding: in float64 without the fp16
    roundings it equals unet_kernels.gather"""
    name, sd, stages, x0, maps, tiled = case
    y = torch.randn(1, 9 * 8, 8, 8, generator=torch.Generator().manual_seed(1), dtype=torch.float64)
    for f in (2, 4):
        exact = torch.zeros(1, 8, 8 * f, 8 * f, dtype=torch.float64)
        for r in range(3):
            ya, yb, wy = pk.src_table(8 * f, 8, f, r)
            for s in range(3):
                xa, xb, wx = pk.src_table(8 * f, 8, f, s)
                Y = y[:, (3 * r + s) * 8:(3 * r + s + 1) * 8]
                at = lambda ii, jj: Y[:, :, ii][:, :, :, jj]   # noqa: E731
                Wy, Wx = wy[:, None], wx[None, :]
                exact += Wy * Wx * at(ya, xa) + Wy * (1 - Wx) * at(ya, xb) + (1 - Wy) * Wx * at(yb, xa) + (1 - Wy) * (1 - Wx) * at(yb, xb)
        assert (exact - pk.gather(y, 8, f=f)).abs().max().item() <= 1e-12


def test_mutations_move_the_reference_beyond_the_bound(case):
    name, sd, stages, x0, maps, tiled = case
    taps = pk.chain(sd, stages, x0)
    seen = set()
    for c in _checks(sd, stages, taps, x0, tiled):
        for mname, mref, where in c.mutations:
            v = (mref - c.ref).abs() > c.tol
            assert v.any(), (c.step, mname)
            assert ck.outside(v, where) == 0, (c.step, mname)
            seen.add((pk.family(c.step), mname))
    print(f"[{name}] mutations detected: {sorted(seen)}")


@pytest.mark.parametrize("cfg", list(pk.CONFIGS))
def test_gpu_configurations_load(built_lib, cfg):
    """each configuration of tests/test_pd_kernels_gpu.py passes the load-time rules with the stages it names"""
    from videoseal_b200 import cfg as vcfg
    spec = vcfg.spec_from_card(pk.config_card(cfg))
    assert spec["pixel_decoder"] == {"pixelwise": True, "upscale_stages": pk.CONFIGS[cfg][1]}
    assert spec["img_size"] == pk.CONFIGS[cfg][2]
