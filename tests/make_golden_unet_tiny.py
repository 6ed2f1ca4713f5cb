"""Writes tests/golden/unet_tiny.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_unet_tiny

Builds the UNMODIFIED reference Videoseal for the videoseal_1.0 card with its embedder replaced by unet_tiny_yuv_quant, loads
the seeded synthetic checkpoint (oracle/restate.synth_state_dict, seed 1234), checks the CPU oracle against it (max |diff|
must be 0) and stores strided samples of imgs_w / preds_w.
"""
import os
import sys
import time

import torch

from oracle import ref_import, restate
from tests import unet_tiny as ut
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def cases(nbits: int) -> dict:
    """name -> (input, msgs, is_video, video_mode, chunk_size); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(0)
    img = torch.rand(2, 3, 256, 256, generator=g)
    img_m = torch.randint(0, 2, (2, nbits), generator=g)
    g = torch.Generator().manual_seed(1)
    res = torch.rand(1, 3, 384, 480, generator=g)
    res_m = torch.randint(0, 2, (1, nbits), generator=g)
    g = torch.Generator().manual_seed(2)
    vid = torch.rand(5, 3, 288, 272, generator=g)
    vid_m = torch.randint(0, 2, (1, nbits), generator=g)
    out = {"img256": (img, img_m, False, "repeat", 2), "img_resized": (res, res_m, False, "repeat", 2)}
    for mode in ("repeat", "alternate", "interpolate"):
        out[f"vid_{mode}"] = (vid, vid_m, True, mode, 2)
    return out


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    t0 = time.time()
    card = ut.tiny_card()
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, ut.SEED)
    ref = build_reference_from_card(card)
    msg = ref.load_state_dict(sd, strict=False)
    assert not msg.unexpected_keys, msg.unexpected_keys
    assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
    ref.eval()
    orc = restate.OracleModel(spec, sd)
    out = {"seed": ut.SEED, "torch": str(torch.__version__), "spec": spec, "cases": {}}
    for name, (x, m, is_video, mode, chunk) in cases(spec["nbits"]).items():
        ref.chunk_size = orc.chunk_size = chunk
        ref.video_mode = orc.video_mode = mode
        with torch.no_grad():
            r = ref.embed(x, m, is_video=is_video)
            o = orc.embed(x, m, is_video=is_video)
        e_img = (r["imgs_w"] - o["imgs_w"]).abs().max().item()
        e_pw = (r["preds_w"] - o["preds_w"]).abs().max().item() if "preds_w" in r else 0.0   # image mode only
        print(name, tuple(x.shape), "max|oracle - reference| imgs_w", e_img, "preds_w", e_pw)
        assert e_img == 0.0 and e_pw == 0.0, (name, e_img, e_pw)
        out["cases"][name] = {"shape": tuple(x.shape), "is_video": is_video, "video_mode": mode, "chunk_size": chunk,
                              "imgs_w_s": ut.sample(r["imgs_w"]), "preds_w_s": ut.sample(r["preds_w"]) if "preds_w" in r else None,
                              "oracle_vs_ref": max(e_img, e_pw)}
    path = os.path.join(ROOT, "tests", "golden", "unet_tiny.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB", f"{time.time() - t0:.1f}s")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
