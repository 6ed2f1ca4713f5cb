"""Writes tests/golden/pixelwise.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_pixelwise

For each pixel-wise preset (the videoseal_1.0 card with its extractor replaced by convnext_tiny_pw / convnext_base_pw) this
builds the UNMODIFIED reference Videoseal, loads the seeded synthetic checkpoint of tests/pixelwise_oracle.py, checks the
restatement against it (max |diff| must be 0) and stores strided samples + full-map statistics of the maps.
"""
import os
import sys
import time

import torch

from oracle import ref_import
from tests import pixelwise_oracle as pw
from tests.util import load_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEED = 1234
AGGS = ("avg", "squared_avg", "l1norm_avg", "l2norm_avg")


def build_reference_from_card(card: dict):
    """oracle/ref_import.build_reference_model of a card dict: the card is written to a temporary YAML whose absolute path (without
    the suffix) is passed as the card name, so that the reference is built by the same code as for the shipped cards"""
    import tempfile
    import yaml
    d = tempfile.mkdtemp(prefix="vsb200_pw_")
    yaml.safe_dump(card, open(os.path.join(d, "card.yaml"), "w"))
    return ref_import.build_reference_model(os.path.join(d, "card"))[0]


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": SEED, "torch": str(torch.__version__), "presets": {}}
    for preset in pw.PRESETS:
        t0 = time.time()
        card = pw.preset_card(preset, load_card("videoseal_1.0"))
        spec = pw.spec_from_card(card)
        sd = pw.synth_state_dict(spec, SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        orc = pw.OracleModel(spec, sd)
        res = {"spec": spec, "cases": {}}
        # A: image mode at processing size; B: a 384 x 480 input that is resized; C: a ragged video with chunk_size < F
        g = torch.Generator().manual_seed(0)
        cases = {"img256": (torch.rand(2, 3, 256, 256, generator=g), False),
                 "img_resized": (torch.rand(1, 3, 384, 480, generator=torch.Generator().manual_seed(1)), False),
                 "vid": (torch.rand(5, 3, 288, 272, generator=torch.Generator().manual_seed(2)), True)}
        ref.chunk_size, orc.chunk_size = 2, 2
        for name, (x, is_video) in cases.items():
            with torch.no_grad():
                r = ref.detect(x, is_video=is_video)["preds"]
                o = orc.detect(x, is_video=is_video)["preds"]
            err = (r - o).abs().max().item()
            print(preset, name, tuple(r.shape), "max|oracle - reference| =", err)
            assert err == 0.0, err
            res["cases"][name] = {"gen_seed": {"img256": 0, "img_resized": 1, "vid": 2}[name], "shape": tuple(x.shape),
                                  "is_video": is_video, "maps_s": pw.sample(r), "stats": stats_all(r), "oracle_vs_ref": err}
        # D: extract_message with every aggregation on the video of case C ([1, K, S, S] bool)
        x = cases["vid"][0]
        aggs = {}
        for agg in AGGS:
            with torch.no_grad():
                a_ref = ref.extract_message(x, aggregation=agg)
                a_orc = orc.extract_message(x, aggregation=agg)
            n_diff = int((a_ref != a_orc).sum())
            print(preset, "extract", agg, tuple(a_ref.shape), "differing bits:", n_diff)
            assert n_diff == 0, agg
            aggs[agg] = {"bits_s": a_ref[:, ::8, ::16, ::16].clone(), "ones": int(a_ref.sum()), "oracle_vs_ref": n_diff}
        res["cases"]["extract"] = aggs
        out["presets"][preset] = res
        print(preset, f"{time.time() - t0:.1f}s")
    path = os.path.join(ROOT, "tests", "golden", "pixelwise.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


def stats_all(maps: torch.Tensor) -> dict:
    """full-map statistics: of every value, and of the detection channel alone"""
    return {"all": pw.stats(maps), "det": pw.stats(maps[:, :1])}


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
