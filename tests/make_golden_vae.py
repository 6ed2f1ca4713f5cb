"""Writes tests/golden/vae.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_vae

For vae_tiny, vae_small, vae_tiny_yuv and vae_small_bw with nbits 8 and 32 at 128 x 128 (convnext extractor), builds the UNMODIFIED
reference Videoseal of the card (tests/vae_oracle.card), loads the seeded synthetic checkpoint (tests/vae_oracle.synth_state_dict;
the reference's load_state_dict must find every embedder and detector key and no other), checks the float64 oracle against it on
every pixel and stores a fixed strided sample (hidden_oracle.sample) of the reference's imgs_w of: image mode on 1 and on 3 frames,
and a 5-frame video with chunk_size 2 and step_size 1.
"""
import os
import sys

import torch

from oracle import ref_import
from tests import vae_oracle as vo
from tests.hidden_oracle import sample
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRESETS = ("vae_tiny", "vae_small", "vae_tiny_yuv", "vae_small_bw")
NBITS = (8, 32)
S = 128
CHUNK, STEP = 2, 1


def cases(K: int) -> dict:
    """name -> (frames, msgs, is_video); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(11)
    return {"img1": (torch.rand(1, 3, S, S, generator=g), torch.randint(0, 2, (1, K), generator=g), False),
            "img3": (torch.rand(3, 3, S, S, generator=g), torch.randint(0, 2, (3, K), generator=g), False),
            "vid5_chunk2": (torch.rand(5, 3, S, S, generator=g), torch.randint(0, 2, (1, K), generator=g), True)}


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": vo.SEED, "torch": str(torch.__version__), "presets": {}}
    for preset in PRESETS:
        for K in NBITS:
            card = vo.card(preset, img_size=S, nbits=K)
            spec = vo.spec_from_card(card)
            sd = vo.synth_state_dict(spec, vo.SEED)
            ref = build_reference_from_card(card)
            msg = ref.load_state_dict(sd, strict=False)
            assert not msg.unexpected_keys, msg.unexpected_keys
            assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
            assert type(ref.embedder).__name__ == "VAEEmbedder"
            assert ref.embedder.yuv == spec["yuv"]
            ref.eval()
            ref.chunk_size, ref.step_size = CHUNK, STEP
            orc = vo.VaeOracle(spec, sd)
            orc.chunk_size, orc.step_size = CHUNK, STEP
            res = {"spec": spec, "cases": {}}
            for name, (x, m, is_video) in cases(K).items():
                with torch.no_grad():
                    r = ref.embed(x, msgs=m, is_video=is_video)["imgs_w"]
                    o = orc.embed(x, m, is_video=is_video)["imgs_w"]
                e = (o - r.double()).abs().max().item()
                print(f"{preset} K={K} {name}: max|oracle (fp64 embedder) - reference (fp32)| of imgs_w = {e:.2e}", flush=True)
                assert e < 1e-5, (preset, K, name, e)
                res["cases"][name] = {"is_video": is_video, "msgs": m.clone(), "imgs_w": sample(r)}
            out["presets"][(preset, K)] = res
    path = os.path.join(ROOT, "tests", "golden", "vae.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
