"""Writes tests/golden/interp.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_interp

Builds the UNMODIFIED reference Videoseal for the videoseal_1.0 card (one block per U-Net level and ConvNeXt stage, as the GPU
tests' model), loads the seeded synthetic checkpoint, and runs embed (image batch and video clip), detect and extract_message
with each interpolation dict of DICTS, on inputs regenerated from seeds by inputs().  It checks that oracle/restate.py gives the
same outputs (max |diff| must be 0) and stores every sixth row and column of each image output (the full tensors would be ~10 MB).
"""
import os
import sys
import time

import torch

from oracle import ref_import, restate
from tests.make_golden_pixelwise import build_reference_from_card
from tests.util import SEED, apply_overrides, load_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TINY = {"num_blocks": 1, "depths": [1, 1, 1, 1]}
STEP, CHUNK = 2, 2
# every mode the reference CLIs offer, each in a dict F.interpolate accepts (nearest / area take no align_corners)
DICTS = {
    "bicubic_aa": {"mode": "bicubic", "align_corners": False, "antialias": True},
    "bicubic_noaa": {"mode": "bicubic", "align_corners": False, "antialias": False},
    "bilinear_ac": {"mode": "bilinear", "align_corners": True, "antialias": False},
    "nearest": {"mode": "nearest", "antialias": False},
    "area": {"mode": "area"},
}


def sub(t: torch.Tensor) -> torch.Tensor:
    """every sixth row and column"""
    return t[..., ::6, ::6].clone()


def inputs():
    """a 2-image batch that is down-scaled to 256, and a 5-frame clip that is up-scaled to it"""
    g = torch.Generator().manual_seed(11)
    return torch.rand(2, 3, 288, 352, generator=g), torch.rand(5, 3, 144, 176, generator=g)


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    card = apply_overrides(load_card("videoseal_1.0"), TINY)
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, seed=SEED)
    ref = build_reference_from_card(card)
    msg = ref.load_state_dict(sd, strict=False)
    assert not msg.unexpected_keys, msg.unexpected_keys
    ref.eval()
    orc = restate.OracleModel(spec, sd)
    for m in (ref, orc):
        m.step_size, m.chunk_size = STEP, CHUNK
    imgs, clip = inputs()
    g = torch.Generator().manual_seed(12)
    msgs_img = torch.randint(0, 2, (imgs.shape[0], spec["nbits"]), generator=g)
    msgs_vid = torch.randint(0, 2, (1, spec["nbits"]), generator=g)
    out = {"seed": SEED, "torch": str(torch.__version__), "step": STEP, "chunk": CHUNK, "msgs_img": msgs_img, "msgs_vid": msgs_vid,
           "dicts": {}}
    for key, interp in DICTS.items():
        t0 = time.time()
        res = {}
        with torch.no_grad():
            for name, m in (("ref", ref), ("orc", orc)):
                e = m.embed(imgs, msgs_img, is_video=False, interpolation=interp)
                v = m.embed(clip, msgs_vid, is_video=True, interpolation=interp)
                p = m.detect(v["imgs_w"], is_video=True, interpolation=interp)["preds"]
                b = m.extract_message(v["imgs_w"], interpolation=interp)
                res[name] = {"img_imgs_w": e["imgs_w"], "img_preds_w": e["preds_w"], "vid_imgs_w": v["imgs_w"], "vid_preds": p,
                             "extract_bits": b}
        r, o = res["ref"], res["orc"]
        err = max((r[k].float() - o[k].float()).abs().max().item() for k in r)
        print(key, "max|oracle - reference| =", err, f"{time.time() - t0:.1f}s")
        assert err == 0.0, (key, err)
        out["dicts"][key] = {"interpolation": interp, "oracle_vs_ref": err, "img_imgs_w": sub(r["img_imgs_w"]),
                             "img_preds_w": sub(r["img_preds_w"]), "vid_imgs_w": sub(r["vid_imgs_w"]), "vid_preds": r["vid_preds"].clone(),
                             "extract_bits": r["extract_bits"].clone()}
    path = os.path.join(ROOT, "tests", "golden", "interp.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
