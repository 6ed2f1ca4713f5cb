"""The VAE embedder's per-step bounds and mutations (tests/vae_kernels.py) without a GPU: every step of the fp16 emulation of the plan
stays within its bound and every mutation leaves it, at each GroupNorm group width (C / 16 = 1, 2, 4, 8) and both attention head dims
(64: vae_tiny, 128: vae_small); eps 1e-5 is caught on small-variance groups."""
import pytest
import torch

from tests import vae_kernels as vk
from tests import vae_oracle as vo


def _emulated(preset, S=128, B=2, K=16):
    spec = vo.spec_from_card(vo.card(preset, img_size=S, nbits=K))
    sd = {k: v.double() for k, v in vo.synth_state_dict(spec, vo.SEED).items() if k.startswith("embedder.")}
    v = spec["vae_encoder"]
    x = torch.rand(B, v["in_channels"], S, S, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    m = torch.randint(0, 2, (B, K), generator=torch.Generator().manual_seed(4))
    t = {}
    d = vk.vae_forward_emulated(sd, v, x, m, vk.Plan16(), t)
    return sd, v, x, m, t, d


@pytest.mark.parametrize("preset", ["vae_tiny", "vae_small", "vae_big"])
def test_every_step_of_the_emulation_within_its_bound(preset):
    sd, v, x, m, t, d = _emulated(preset)
    res = vk.run_steps(sd, v, x, m, t, d)
    widths = {c for c in vo.widths(v)} | {v["ch"]}
    assert any(n.endswith(".attn") for n in res) and len(res) > 40
    print(preset, "group widths", sorted(c // 16 for c in widths), "max err/bound", max(res.values()))


@pytest.mark.parametrize("C", [16, 32, 64, 128])
@pytest.mark.parametrize("silu", [True, False])
def test_groupnorm_eps_and_layouts_on_small_variance_groups(C, silu):
    """groups of C / 16 = 1, 2, 4, 8 channels: the emulated step (one fp16 rounding of the exact result) is within the bound, and
    eps 1e-5, interleaved groups, GELU and another frame's statistics all leave it"""
    x = vk.small_variance_map(2, C, 16, seed=C)
    g = torch.Generator().manual_seed(C + 1)
    gamma, beta = 1 + 0.2 * torch.randn(C, generator=g, dtype=torch.float64), 0.2 * torch.randn(C, generator=g, dtype=torch.float64)
    pre = torch.nn.functional.group_norm(x, 16, gamma, beta, 1e-6)
    got = vk.r16(torch.nn.functional.silu(pre) if silu else pre)
    r = vk.judge(f"gn{C}", *vk.gn_step(x, gamma, beta, silu, got, eps_mutant=True))
    assert r <= 1.0


def test_emulated_error_of_each_preset_end_to_end():
    """the fp16 emulation's delta error (no kernel in the loop): the size of the fp16 error the plan's roundings alone produce,
    which the GPU parity tests are compared with"""
    for preset in ("vae_tiny", "vae_small"):
        spec = vo.spec_from_card(vo.card(preset, img_size=128, nbits=16))
        sd = {k: v.double() for k, v in vo.synth_state_dict(spec, vo.SEED).items() if k.startswith("embedder.")}
        v = spec["vae_encoder"]
        x = torch.rand(2, v["in_channels"], 128, 128, generator=torch.Generator().manual_seed(5), dtype=torch.float64)
        m = torch.randint(0, 2, (2, 16), generator=torch.Generator().manual_seed(6))
        e = (vk.vae_forward_emulated(sd, v, x, m, vk.Plan16()) - vo.vae_forward(sd, v, x, m)).abs().max().item()
        assert 1e-4 < e < 5e-2, (preset, e)
