"""Writes tests/golden/vit.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_vit

For the SAM-ViT cards of tests/vit_oracle.py (the videoseal_1.0 card with the videoseal_0.0 card's `sam_small` extractor, pooled and
pixel-wise [4, 2, 2]) this builds the UNMODIFIED reference Videoseal, loads the seeded synthetic checkpoint, checks the restatement
against it (max |diff| must be 0) and stores the logits (pooled) or strided samples + statistics of the maps (pixel-wise).
"""
import os
import sys
import time

import torch

from oracle import ref_import
from tests import pixelwise_oracle as pw
from tests import vit_oracle as vo
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
AGGS = ("avg", "squared_avg", "l1norm_avg", "l2norm_avg")


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": vo.SEED, "torch": str(torch.__version__), "variants": {}}
    for variant, pixelwise in (("sam_small", False), ("sam_small_pw", True)):
        t0 = time.time()
        card = vo.vit_card(pixelwise)
        spec = vo.spec_from_card(card)
        sd = vo.synth_state_dict(spec, vo.SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        orc = vo.OracleModel(spec, sd)
        res = {"cases": {}}
        # A: 2 frames at processing size; B: a 384 x 480 frame that is resized; C: a ragged video with chunk_size < F
        cases = {"img256": (torch.rand(2, 3, 256, 256, generator=torch.Generator().manual_seed(0)), False),
                 "img_resized": (torch.rand(1, 3, 384, 480, generator=torch.Generator().manual_seed(1)), False),
                 "vid": (torch.rand(5, 3, 288, 272, generator=torch.Generator().manual_seed(2)), True)}
        ref.chunk_size, orc.chunk_size = 2, 2
        for name, (x, is_video) in cases.items():
            with torch.no_grad():
                r = ref.detect(x, is_video=is_video)["preds"]
                o = orc.detect(x, is_video=is_video)["preds"]
            err = (r - o).abs().max().item()
            print(variant, name, tuple(r.shape), "max|oracle - reference| =", err)
            assert err == 0.0, err
            c = {"gen_seed": {"img256": 0, "img_resized": 1, "vid": 2}[name], "shape": tuple(x.shape), "is_video": is_video,
                 "oracle_vs_ref": err}
            if pixelwise:
                c.update(maps_s=pw.sample(r), stats=pw.stats(r))
            else:
                c["logits"] = r.clone()
            res["cases"][name] = c
        x = cases["vid"][0]
        aggs = {}
        for agg in AGGS:
            with torch.no_grad():
                a_ref = ref.extract_message(x, aggregation=agg)
                a_orc = orc.extract_message(x, aggregation=agg)
            n_diff = int((a_ref != a_orc).sum())
            print(variant, "extract", agg, tuple(a_ref.shape), "differing bits:", n_diff)
            assert n_diff == 0, agg
            aggs[agg] = {"bits_s": (a_ref[:, ::8, ::16, ::16] if pixelwise else a_ref).clone(), "ones": int(a_ref.sum()),
                         "oracle_vs_ref": n_diff}
        res["cases"]["extract"] = aggs
        out["variants"][variant] = res
        print(variant, f"{time.time() - t0:.1f}s")
    path = os.path.join(ROOT, "tests", "golden", "vit.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
