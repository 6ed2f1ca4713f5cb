"""Identity-augmentation slice of the reference's full evaluation (videoseal/evals/full.py:57-248 with only_identity=True):
per item embed -> image metrics -> extract -> bit accuracy / p-value / capacity, one CSV row per item with the reference's
column names (`psnr`, `ssim`, `msssim`, `bit_acc_Identity_0`, `pvalue_Identity_0`, `log_pvalue_Identity_0`,
`capacity_Identity_0`, `embed_time`, `extract_time`, ...), so that its reports line up with the reference's own runs.
`image_metrics` picks the quality columns: PSNR by default; "ssim" and "msssim" run on the GPU (evals/metrics.py), and
image_metrics=("psnr", "ssim", "msssim") gives the reference's columns (full.py:132-142) without LPIPS / VMAF.
With only_identity=False each item's imgs_w also goes through the reference's validation bank (augmentation.get_validation_augs,
run by the GPU kernels of videoseal_b200.augmentation) at frame resolution before detection, and every (augmentation, strength)
adds its `bit_acc_<key>` / `pvalue_<key>` / `log_pvalue_<key>` / `capacity_<key>` group in the reference's order and key rule
(full.py:188-239).  Every non-identity video list of the reference holds a codec, so a video run takes an explicit list; the CLI's
--codec_free_video True passes augmentation.get_codec_free_video_augs(): the reference's video list without its codecs, plus the
temporal attacks (SpeedChange, WindowAveraging, DropFrame, TemporalReorder) that may change the clip's frame count before
extract_message.  Deviation: only_identity defaults to True here (the reference's default is False), so that a default run keeps
its Identity-only columns; `extract_time` times the Identity detection.  The video codecs (H264 / H265 / VP9), LPIPS / VMAF, the
detection (mask IoU) columns and the image dumps need packages outside this path."""
from __future__ import annotations

import math
import os
import time
from typing import Iterable

import torch

from .metrics import _quality, bit_accuracy, capacity, psnr, pvalue

IMAGE_METRICS = ("psnr", "ssim", "msssim")   # the reference's column order

_DEF_INTERP = {"mode": "bilinear", "align_corners": False, "antialias": True}


def _sync(x: torch.Tensor):
    if x.is_cuda:
        torch.cuda.synchronize(x.device)


@torch.no_grad()
def evaluate(model, dataset: Iterable, is_video: bool, output_dir: str, num_frames: int = 24 * 3, video_aggregation: str = "avg",
             decoding: bool = True, interpolation: dict = _DEF_INTERP, lowres_attenuation: bool = False,
             skip_image_metrics: bool = False, image_metrics: Iterable[str] = ("psnr",), only_identity: bool = True,
             only_combined: bool = False, validation_augs: list | None = None):
    image_metrics = set(image_metrics)
    augs = None
    if decoding and (validation_augs is not None or not only_identity):
        from ..augmentation import get_validation_augs
        augs = validation_augs if validation_augs is not None else get_validation_augs(is_video, only_identity, only_combined)
    unknown = image_metrics - set(IMAGE_METRICS)
    if unknown:
        raise ValueError(f"unknown image metrics {sorted(unknown)}; choose from {IMAGE_METRICS}")
    os.makedirs(output_dir, exist_ok=True)
    all_metrics = []
    path = os.path.join(output_dir, "metrics.csv")
    with open(path, "w") as f:
        for it, item in enumerate(dataset):
            if item is None:
                continue
            imgs = item[0]
            if not is_video:
                imgs = imgs.unsqueeze(0)
            m = {"iteration": it, "t": imgs.shape[-4], "h": imgs.shape[-2], "w": imgs.shape[-1]}
            _sync(imgs)
            t0 = time.time()
            out = model.embed(imgs, is_video=is_video, interpolation=interpolation, lowres_attenuation=lowres_attenuation)
            _sync(out["imgs_w"])
            m["embed_time"] = time.time() - t0
            msgs, imgs_w = out["msgs"][:num_frames], out["imgs_w"][:num_frames]
            imgs = imgs[:num_frames]
            if not skip_image_metrics:
                ref = imgs.to(imgs_w.device)
                if "psnr" in image_metrics:
                    m["psnr"] = psnr(imgs_w, ref, is_video).mean().item()
                if "ssim" in image_metrics or "msssim" in image_metrics:
                    s, ms = _quality(imgs_w, ref, 1.0, "ssim" in image_metrics, "msssim" in image_metrics)
                    if s is not None:
                        m["ssim"] = s.mean().item()
                    if ms is not None:
                        m["msssim"] = ms.mean().item()
            if decoding:
                t0 = time.time()
                if is_video:
                    bit_preds = model.extract_message(imgs_w, video_aggregation, interpolation).float() * 2 - 1   # bool [1,K] -> +-1
                    msgs = msgs[:1]
                else:
                    bit_preds = model.detect(imgs_w, is_video=False)["preds"][:, 1:]
                _sync(bit_preds)
                m["extract_time"] = time.time() - t0
                bit_preds, tgt = bit_preds.cpu(), msgs.cpu()
                pv = pvalue(bit_preds, tgt).nanmean().item()
                m["bit_acc_Identity_0"] = bit_accuracy(bit_preds, tgt).nanmean().item()
                m["pvalue_Identity_0"] = pv
                m["log_pvalue_Identity_0"] = -math.log10(pv) if pv > 0 else -100
                m["capacity_Identity_0"] = capacity(bit_preds, tgt).nanmean().item()
                if augs is not None:
                    m.update(_augmented_rows(model, imgs_w, tgt, augs, is_video, video_aggregation, interpolation))
            all_metrics.append(m)
            if len(all_metrics) == 1:
                f.write(",".join(m.keys()) + "\n")
            f.write(",".join(map(str, m.values())) + "\n")
            f.flush()
    return all_metrics


def _decode_stats(bit_preds: torch.Tensor, tgt: torch.Tensor, key: str) -> dict:
    pv = pvalue(bit_preds, tgt).nanmean().item()
    return {f"bit_acc_{key}": bit_accuracy(bit_preds, tgt).nanmean().item(), f"pvalue_{key}": pv,
            f"log_pvalue_{key}": -math.log10(pv) if pv > 0 else -100, f"capacity_{key}": capacity(bit_preds, tgt).nanmean().item()}


def _augmented_rows(model, imgs_w, tgt, augs, is_video, video_aggregation, interpolation) -> dict:
    """The column groups of every (augmentation, strength) after Identity_0, which the caller has already written."""
    from ..augmentation import column_key
    out = {}
    for aug, strengths in augs:
        for strength in strengths:
            key = column_key(aug, strength)
            if key == "Identity_0":
                continue
            imgs_aug, _ = aug(imgs_w, None, strength)
            if is_video:
                bit_preds = model.extract_message(imgs_aug, video_aggregation, interpolation).float() * 2 - 1
            else:
                bit_preds = model.detect(imgs_aug, is_video=False)["preds"][:, 1:]
            out.update(_decode_stats(bit_preds.cpu(), tgt, key))
    return out


def main(argv=None):
    import argparse
    from ..cfg import setup_model_from_checkpoint
    from .speed import _bool, add_interpolation_args, interpolation_of, synthetic_items
    ap = argparse.ArgumentParser(description="identity-augmentation evaluation of a card / checkpoint on this backend")
    ap.add_argument("--checkpoint", required=True)
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--is_video", type=_bool, default=False)
    ap.add_argument("--num_frames", type=int, default=24 * 3)
    ap.add_argument("--num_samples", type=int, default=10)
    ap.add_argument("--size", type=int, nargs="+", default=[768])
    ap.add_argument("--video_aggregation", default="avg")
    ap.add_argument("--lowres_attenuation", type=_bool, default=False)
    ap.add_argument("--scaling_w", default=None)
    ap.add_argument("--output_dir", default="output/full")
    ap.add_argument("--image_metrics", nargs="+", default=["psnr"], choices=IMAGE_METRICS,
                    help="quality columns (psnr ssim msssim gives the reference's; ssim / msssim need the GPU)")
    ap.add_argument("--only_identity", type=_bool, default=True,
                    help="only the Identity rows (the reference defaults to False: the whole validation bank)")
    ap.add_argument("--only_combined", type=_bool, default=False, help="with --only_identity False: only the combined augmentations")
    ap.add_argument("--codec_free_video", type=_bool, default=False,
                    help="with --is_video True --only_identity False: the video bank without its codecs, plus the temporal attacks")
    add_interpolation_args(ap)
    a = ap.parse_args(argv)
    augs = None
    if a.codec_free_video:
        if not a.is_video or a.only_identity or a.only_combined:
            ap.error("--codec_free_video True needs --is_video True --only_identity False (and not --only_combined)")
        from ..augmentation import get_codec_free_video_augs
        augs = get_codec_free_video_augs()
    model = setup_model_from_checkpoint(a.checkpoint).eval().to(a.device)
    if a.scaling_w is not None:
        model.blender.scaling_w = float(a.scaling_w)
    rows = evaluate(model, synthetic_items(a.num_samples, a.is_video, a.num_frames, a.size[0], a.size[-1], a.device), a.is_video,
                    a.output_dir, a.num_frames, a.video_aggregation, interpolation=interpolation_of(a), lowres_attenuation=a.lowres_attenuation,
                    image_metrics=a.image_metrics, only_identity=a.only_identity, only_combined=a.only_combined, validation_augs=augs)
    keys = [k for k in rows[0] if k not in ("iteration", "t", "h", "w")]
    print({k: sum(r[k] for r in rows) / len(rows) for k in keys})


if __name__ == "__main__":
    main()
