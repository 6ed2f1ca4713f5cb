"""Writes tests/golden/dvmark.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_dvmark

For the `dvmark` extractor preset with nbits 8 and 32 at 128 x 128, builds the UNMODIFIED reference Videoseal of the card
(tests/dvmark_oracle.card: videoseal_1.0's U-Net embedder), loads the seeded synthetic checkpoint (tests/dvmark_oracle.synth_state_dict,
which also checks the checkpoint key names: the reference's load_state_dict must find every detector key and no other), checks the
float64 oracle against it and stores the reference's logits of: image mode on 1 and on 3 frames (one detector call each), and a
5-frame video with chunk_size 2 (calls of 2, 2 and 1 frames).
"""
import os
import sys

import torch

from oracle import ref_import
from tests import dvmark_oracle as dv
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NBITS = (8, 32)
S = 128


def cases() -> dict:
    """name -> (frames, is_video); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(3)
    return {"img1": (torch.rand(1, 3, S, S, generator=g), False), "img3": (torch.rand(3, 3, S, S, generator=g), False),
            "vid5_chunk2": (torch.rand(5, 3, S, S, generator=g), True)}


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": dv.SEED, "torch": str(torch.__version__), "nbits": {}}
    for K in NBITS:
        card = dv.card("unet", img_size=S, nbits=K)
        spec = dv.spec_from_card(card)
        sd = dv.synth_state_dict(spec, dv.SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        assert type(ref.detector).__name__ == "DVMarkDecoder"
        ref.eval()
        ref.chunk_size = 2
        sd64 = {k: v.double() for k, v in sd.items()}
        res = {"spec": spec, "cases": {}}
        for name, (x, is_video) in cases().items():
            with torch.no_grad():
                r = ref.detect(x, is_video=is_video)["preds"]
                groups = 2 if is_video else x.shape[0]
                o = dv.grouped(sd64, x.double(), groups)
            e = ((o - r.double()).abs().max() / r.abs().max()).item()
            print(f"K={K} {name}: max|oracle(fp64) - reference(fp32)| / max|logit| = {e:.2e}", flush=True)
            assert e < 1e-5, (K, name, e)
            res["cases"][name] = {"is_video": is_video, "logits": r.clone()}
        out["nbits"][K] = res
    path = os.path.join(ROOT, "tests", "golden", "dvmark.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
