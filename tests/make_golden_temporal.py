"""Writes tests/golden/temporal.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_temporal

For the two temporal presets the GPU tests run (unet_small2_yuv_quant_conv3d and the RGB unet_small2_quant_conv3d), builds the
UNMODIFIED reference Videoseal for the videoseal_1.0 card with that embedder (UNetMsg(conv_layer="conv3d")), loads the seeded
synthetic Conv3dWrapper checkpoint (tests/temporal_oracle.synth_state_dict), checks the CPU oracle against it (max |diff| must be
0) and stores strided samples of imgs_w / preds_w: image mode on 3 images (one time axis), and a 7-frame video with step 2 and
chunk_size 3 (key frames 0, 2, 4 in one call, key frame 6 alone in the short last one).

Also writes tests/golden/temporal_inflate.pt: what the reference's scripts/inflate_model_to_temporal.py does to the extractor part
of a checkpoint, for both of its --extractor_type values (convnext_tiny on the videoseal_1.0 card, sam_small on that card with
videoseal_0.0's extractor): the keys it removes and the keys it adds with their shapes.  tests/temporal_oracle.inflate_script
restates the whole script from that record, and this program checks that restatement against the script's own functions.
"""
import os
import sys
import time

import torch

from oracle import ref_import, restate
from tests import temporal_oracle as to
from tests.make_golden_pixelwise import build_reference_from_card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_PRESETS = ("unet_small2_yuv_quant_conv3d", "unet_small2_quant_conv3d")


def cases(nbits: int) -> dict:
    """name -> (input, msgs, is_video, chunk_size, step_size); generator seeds are part of the fixture"""
    g = torch.Generator().manual_seed(0)
    img = torch.rand(3, 3, 256, 256, generator=g)
    img_m = torch.randint(0, 2, (3, nbits), generator=g)
    g = torch.Generator().manual_seed(1)
    vid = torch.rand(7, 3, 256, 256, generator=g)
    vid_m = torch.randint(0, 2, (1, nbits), generator=g)
    return {"img3": (img, img_m, False, 8, 1), "vid7_chunk3_step2": (vid, vid_m, True, 3, 2)}


def inflate_record():
    import importlib.util
    ref_import.install_stubs()
    path = os.path.join(ref_import.REF_ROOT, "scripts", "inflate_model_to_temporal.py")
    spec_ = importlib.util.spec_from_file_location("inflate_ref", path)
    script = importlib.util.module_from_spec(spec_)
    spec_.loader.exec_module(script)
    out = {}
    for ext, card in (("convnext_tiny", to.preset_card("unet_small2_yuv_quant")), ("sam_small", to.sam_card("unet_small2_yuv_quant"))):
        sd = restate.synth_state_dict(restate.spec_from_card(card), to.SEED)
        ref = dict(sd)
        script.inflate_convs_unet_embedder_inplace(ref)
        if ext == "convnext_tiny":
            script.add_temporal_attention_into_convnext_inplace(ref)
        else:
            script.add_temporal_attention_into_sam_inplace(ref)
        ext_removed = sorted(k for k in sd if k not in ref and k.startswith("detector."))
        ext_added = {k: tuple(v.shape) for k, v in ref.items() if k not in sd and k.startswith("detector.")}
        out[ext] = {"removed": ext_removed, "added": ext_added}
        mine = to.inflate_script(sd, ext, out[ext])
        assert sorted(mine) == sorted(ref), (ext, set(mine) ^ set(ref))
        for k, v in ref.items():
            if k.startswith("embedder.") or k.endswith((".temp_conv.weight", ".mlp.lin2.weight", ".mlp.lin2.bias", "pos_embed_temporal")) \
                    or not (".temp_" in k or "temporal" in k):
                assert torch.equal(mine[k], v), (ext, k)       # every value the loader reads or checks is the script's
        print(ext, "removed", len(ext_removed), "added", len(ext_added), flush=True)
    return out


def main():
    torch.set_num_threads(os.cpu_count() or 8)
    out = {"seed": to.SEED, "torch": str(torch.__version__), "presets": {}}
    for preset in GOLDEN_PRESETS:
        t0 = time.time()
        card = to.preset_card(preset)
        spec = to.spec_from_card(card)
        sd = to.synth_state_dict(spec, to.SEED)
        ref = build_reference_from_card(card)
        msg = ref.load_state_dict(sd, strict=False)
        assert not msg.unexpected_keys, msg.unexpected_keys
        assert not [k for k in msg.missing_keys if not k.startswith("attenuation.")], msg.missing_keys
        ref.eval()
        orc = to.TemporalOracle(spec, sd)
        res = {"spec": spec, "cases": {}}
        for name, (x, m, is_video, chunk, step) in cases(spec["nbits"]).items():
            ref.chunk_size = orc.chunk_size = chunk
            ref.step_size = orc.step_size = step
            with torch.no_grad():
                r = ref.embed(x, m, is_video=is_video)
                o = orc.embed(x, m, is_video=is_video)
            e_img = (r["imgs_w"] - o["imgs_w"]).abs().max().item()
            e_pw = (r["preds_w"] - o["preds_w"]).abs().max().item() if "preds_w" in r else 0.0
            print(preset, name, "max|oracle - reference| imgs_w", e_img, "preds_w", e_pw, flush=True)
            assert e_img == 0.0 and e_pw == 0.0, (preset, name, e_img, e_pw)
            res["cases"][name] = {"shape": tuple(x.shape), "is_video": is_video, "chunk_size": chunk, "step_size": step,
                                  "imgs_w_s": to.sample(r["imgs_w"]),
                                  "preds_w_s": to.sample(r["preds_w"]) if "preds_w" in r else None}
        out["presets"][preset] = res
        print(preset, f"{time.time() - t0:.1f}s", flush=True)
    path = os.path.join(ROOT, "tests", "golden", "temporal.pt")
    torch.save(out, path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")
    path = os.path.join(ROOT, "tests", "golden", "temporal_inflate.pt")
    torch.save(inflate_record(), path)
    print("->", path, os.path.getsize(path) // 1024, "KiB")


if __name__ == "__main__":
    if not ref_import.available():
        sys.exit("needs the reference tree at " + ref_import.REF_ROOT)
    main()
