"""Writes tests/golden/dvmark_embed.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_dvmark_embed

For the `dvmark` embedder preset with nbits 8 and 32 at 128 x 128, builds the UNMODIFIED reference Videoseal of a dvmark / dvmark card
(tests/dvmark_enc_oracle.card), loads the seeded synthetic checkpoint (tests/dvmark_enc_oracle.synth_state_dict, which also checks
the checkpoint key names: the reference's load_state_dict must find every embedder and detector key and no other), checks the
float64 oracle against it on every pixel and stores a fixed strided sample (hidden_oracle.sample) of the reference's imgs_w of: image mode on 1 and on 3 frames (one embedder call each), and a
5-frame video with chunk_size 2 and step_size 1 (calls of 2, 2 and 1 key frames).
"""
import os
import sys

import torch

from oracle import ref_import
from tests import dvmark_enc_oracle as de
from tests.hidden_oracle import sample
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NBITS = (8, 32)
S = 128
CHUNK, STEP = 2, 1


def cases(K: int) -> dict:
    """name -> (frames, msgs, is_video); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(7)
    return {"img1": (torch.rand(1, 3, S, S, generator=g), torch.randint(0, 2, (1, K), generator=g), False),
            "img3": (torch.rand(3, 3, S, S, generator=g), torch.randint(0, 2, (3, K), generator=g), False),
            "vid5_chunk2": (torch.rand(5, 3, S, S, generator=g), torch.randint(0, 2, (1, K), generator=g), True)}


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": de.SEED, "torch": str(torch.__version__), "nbits": {}}
    for K in NBITS:
        card = de.card("dvmark", img_size=S, nbits=K)
        spec = de.spec_from_card(card)
        sd = de.synth_state_dict(spec, de.SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        assert type(ref.embedder).__name__ == "DVMarkEmbedder" and type(ref.detector).__name__ == "DVMarkDecoder"
        assert not ref.embedder.yuv
        ref.eval()
        ref.chunk_size, ref.step_size = CHUNK, STEP
        orc = de.EncOracle(spec, sd)
        orc.chunk_size, orc.step_size = CHUNK, STEP
        res = {"spec": spec, "cases": {}}
        for name, (x, m, is_video) in cases(K).items():
            with torch.no_grad():
                r = ref.embed(x, msgs=m, is_video=is_video)["imgs_w"]
                o = orc.embed(x, m, is_video=is_video)["imgs_w"]
            e = (o - r.double()).abs().max().item()
            print(f"K={K} {name}: max|oracle (fp64 embedder) - reference (fp32)| of imgs_w = {e:.2e}", flush=True)
            assert e < 1e-5, (K, name, e)
            res["cases"][name] = {"is_video": is_video, "msgs": m.clone(), "imgs_w": sample(r)}
        out["nbits"][K] = res
    path = os.path.join(ROOT, "tests", "golden", "dvmark_embed.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
