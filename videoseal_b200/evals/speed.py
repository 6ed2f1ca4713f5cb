"""Speed test with the semantics of the reference's videoseal/evals/speed.py:36-148 (warm-up runs, then `num_runs` timed runs of
embed and of extraction, each bracketed by device synchronisation, averaged per item) for any object with the
embed / detect / extract_message API - this package's Videoseal or the reference's.

    python -m videoseal_b200.evals.speed --checkpoint videoseal_1.0 --is_video true --num_frames 72 --size 768

`--checkpoint` takes a card name or a training checkpoint (setup_model_from_checkpoint).  Datasets of the reference need
decoders that are not part of this path, so the CLI times seeded synthetic clips / images of the requested size; the
SpeedTester class itself accepts any iterable of (imgs, masks) items like the reference's."""
from __future__ import annotations

import argparse
import csv
import os
import time
from typing import Any, Dict, Iterable

import torch

_DEF_INTERP = {"mode": "bilinear", "align_corners": False, "antialias": True}


class SpeedTester:
    def __init__(self, device: str = "cuda"):
        self.device = device

    def _sync(self):
        if str(self.device).startswith("cuda"):
            torch.cuda.synchronize()

    @torch.no_grad()
    def test_speed(self, model, dataset: Iterable, is_video: bool, num_frames: int = 24 * 3, video_aggregation: str = "avg",
                   lowres_attenuation: bool = False, interpolation: dict = _DEF_INTERP, num_runs: int = 3,
                   warmup_runs: int = 1) -> Dict[str, Any]:
        m: Dict[str, Any] = {"device": self.device, "model_name": getattr(model, "name", "unknown"),
                             "checkpoint": getattr(model, "checkpoint_path", "unknown"), "is_video": is_video,
                             "embedding_time": [], "extraction_time": [], "image_shape": []}

        def extract(x):
            if is_video:
                return model.extract_message(x, video_aggregation, interpolation)
            return model.detect(x, is_video=False)

        for item in dataset:
            if item is None:
                continue
            imgs = item[0]
            if not is_video:
                imgs = imgs.unsqueeze(0)
            m["image_shape"].append(f"{imgs.shape[-4]}x{imgs.shape[-2]}x{imgs.shape[-1]}")
            imgs = imgs[:num_frames]
            for _ in range(warmup_runs):
                out = model.embed(imgs, is_video=is_video, interpolation=interpolation, lowres_attenuation=lowres_attenuation)
                extract(out["imgs_w"])
            t_embed = []
            for _ in range(num_runs):
                self._sync()
                t0 = time.time()
                out = model.embed(imgs, is_video=is_video, interpolation=interpolation, lowres_attenuation=lowres_attenuation)
                self._sync()
                t_embed.append(time.time() - t0)
            m["embedding_time"].append(sum(t_embed) / num_runs)
            imgs_w = out["imgs_w"]
            t_ext = []
            for _ in range(num_runs):
                self._sync()
                t0 = time.time()
                extract(imgs_w)
                self._sync()
                t_ext.append(time.time() - t0)
            m["extraction_time"].append(sum(t_ext) / num_runs)
        m["avg_embedding_time"] = sum(m["embedding_time"]) / len(m["embedding_time"])
        m["avg_extraction_time"] = sum(m["extraction_time"]) / len(m["extraction_time"])
        if is_video:
            frames = sum(int(s.split("x")[0]) for s in m["image_shape"]) / len(m["image_shape"])
            frames = min(frames, num_frames)
            m["avg_embedding_ms_per_frame"] = m["avg_embedding_time"] / frames * 1000
            m["avg_extraction_ms_per_frame"] = m["avg_extraction_time"] / frames * 1000
        return m


def synthetic_items(n: int, is_video: bool, num_frames: int, h: int, w: int, device: str, seed: int = 0):
    g = torch.Generator().manual_seed(seed)
    for _ in range(n):
        x = torch.rand((num_frames, 3, h, w) if is_video else (3, h, w), generator=g)
        yield (x.to(device), None)


def _bool(s: str) -> bool:
    return str(s).lower() in ("1", "true", "yes", "y")


def add_interpolation_args(ap: argparse.ArgumentParser):
    """the reference CLIs' resize options (evals/full.py:296-302, evals/speed.py:186-192), same names, choices and defaults"""
    ap.add_argument("--interpolation_mode", default="bilinear", choices=["nearest", "bilinear", "bicubic", "area"],
                    help="interpolation mode for resizing")
    ap.add_argument("--interpolation_align_corners", type=_bool, default=False, help="align corners for interpolation")
    ap.add_argument("--interpolation_antialias", type=_bool, default=True, help="use antialiasing for interpolation")


def interpolation_of(a: argparse.Namespace) -> dict:
    """the dict the reference builds from those options, all three keys set (evals/full.py:345-349, evals/speed.py:215-219).  As
    there, nearest and area raise ValueError on frames that are resized: the dict always carries align_corners."""
    return {"mode": a.interpolation_mode, "align_corners": a.interpolation_align_corners, "antialias": a.interpolation_antialias}


def main(argv=None):
    ap = argparse.ArgumentParser(description="embed / extraction speed of a card or checkpoint on this backend")
    ap.add_argument("--checkpoint", nargs="+", required=True)
    ap.add_argument("--device", default="cuda")
    ap.add_argument("--num_runs", type=int, default=3)
    ap.add_argument("--warmup_runs", type=int, default=1)
    ap.add_argument("--is_video", type=_bool, default=False)
    ap.add_argument("--num_frames", type=int, default=24 * 3)
    ap.add_argument("--num_samples", type=int, default=5)
    ap.add_argument("--size", type=int, nargs="+", default=[768], help="H [W] of the synthetic inputs")
    ap.add_argument("--video_aggregation", default="avg")
    ap.add_argument("--lowres_attenuation", type=_bool, default=False)
    ap.add_argument("--scaling_w", default=None)
    ap.add_argument("--videoseal_chunk_size", type=int, default=32)
    ap.add_argument("--videoseal_step_size", type=int, default=4)
    ap.add_argument("--videoseal_mode", default="repeat")
    add_interpolation_args(ap)
    ap.add_argument("--output_dir", default="output/speed")
    ap.add_argument("--output_file", default="speed_results.csv")
    a = ap.parse_args(argv)
    from ..cfg import setup_model_from_checkpoint
    h, w = a.size[0], a.size[-1]
    rows = []
    for ck in a.checkpoint:
        model = setup_model_from_checkpoint(ck).eval().to(a.device)
        model.name, model.checkpoint_path = os.path.basename(str(ck)), str(ck)
        if a.scaling_w is not None:
            model.blender.scaling_w = float(a.scaling_w)
        model.chunk_size, model.step_size, model.video_mode = a.videoseal_chunk_size, a.videoseal_step_size, a.videoseal_mode
        interp = interpolation_of(a)
        res = SpeedTester(a.device).test_speed(model, synthetic_items(a.num_samples, a.is_video, a.num_frames, h, w, a.device),
                                               a.is_video, a.num_frames, a.video_aggregation, a.lowres_attenuation, interp,
                                               a.num_runs, a.warmup_runs)
        rows.append({k: v for k, v in res.items() if not isinstance(v, list)})
        print(rows[-1])
    os.makedirs(a.output_dir, exist_ok=True)
    path = os.path.join(a.output_dir, a.output_file)
    with open(path, "w", newline="") as f:
        wr = csv.DictWriter(f, fieldnames=sorted({k for r in rows for k in r}))
        wr.writeheader()
        wr.writerows(rows)
    print("wrote", path)


if __name__ == "__main__":
    main()
