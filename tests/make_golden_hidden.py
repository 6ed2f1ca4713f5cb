"""Writes tests/golden/hidden.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_hidden

For the `hidden` (GroupNorm + GELU, tanh) and `hidden_orig` (BatchNorm + ReLU, no tanh) presets, each as embedder and extractor of
the videoseal_1.0 card, builds the UNMODIFIED reference Videoseal, loads the seeded synthetic checkpoint
(tests/hidden_oracle.synth_state_dict), checks the CPU oracle against it (max |diff| must be 0) and stores strided samples of
imgs_w / preds_w and the whole logits of: image mode on two 256 x 256 images, one 384 x 480 image that is resized, and a ragged
5-frame 288 x 272 video with chunk_size 2.
"""
import os
import sys
import time

import torch

from oracle import ref_import
from tests import hidden_oracle as ho
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cases(nbits: int) -> dict:
    """name -> (frames, msgs, is_video); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(0)
    img = torch.rand(2, 3, 256, 256, generator=g)
    img_m = torch.randint(0, 2, (2, nbits), generator=g)
    g = torch.Generator().manual_seed(1)
    big = torch.rand(1, 3, 384, 480, generator=g)
    big_m = torch.randint(0, 2, (1, nbits), generator=g)
    g = torch.Generator().manual_seed(2)
    vid = torch.rand(5, 3, 288, 272, generator=g)
    vid_m = torch.randint(0, 2, (1, nbits), generator=g)
    return {"img256": (img, img_m, False), "img_resized": (big, big_m, False), "vid5_chunk2": (vid, vid_m, True)}


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": ho.SEED, "torch": str(torch.__version__), "presets": {}}
    for preset in ho.PRESETS:
        t0 = time.time()
        card = ho.card(preset, preset)
        spec = ho.spec_from_card(card)
        sd = ho.synth_state_dict(spec, ho.SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        ref.eval()
        orc = ho.HiddenOracle(spec, sd)
        ref.chunk_size = orc.chunk_size = 2
        res = {"spec": spec, "cases": {}}
        for name, (x, m, is_video) in cases(spec["nbits"]).items():
            with torch.no_grad():
                r = ref.embed(x, m, is_video=is_video)
                o = orc.embed(x, m, is_video=is_video)
                rl = ref.detect(r["imgs_w"], is_video=is_video)["preds"]
                ol = orc.detect(r["imgs_w"], is_video=is_video)["preds"]
            e_img = (r["imgs_w"] - o["imgs_w"]).abs().max().item()
            e_pw = (r["preds_w"] - o["preds_w"]).abs().max().item() if "preds_w" in r else 0.0
            e_lg = (rl - ol).abs().max().item()
            print(preset, name, "max|oracle - reference| imgs_w", e_img, "preds_w", e_pw, "logits", e_lg, flush=True)
            assert e_img == 0.0 and e_pw == 0.0 and e_lg == 0.0, (preset, name, e_img, e_pw, e_lg)
            res["cases"][name] = {"shape": tuple(x.shape), "is_video": is_video, "msgs": m.clone(),
                                  "imgs_w_s": ho.sample(r["imgs_w"]),
                                  "preds_w_s": ho.sample(r["preds_w"]) if "preds_w" in r else None,
                                  "logits": rl.clone()}
        out["presets"][preset] = res
        print(preset, f"{time.time() - t0:.1f}s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "hidden.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
