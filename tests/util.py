"""Shared helpers for tests / smoke / bench: synthetic checkpoints in the reference's format, cards on disk, and the
(product model, CPU oracle) pair built from the same card + checkpoint."""
import os
import sys
import tempfile
from pathlib import Path

import torch
import yaml

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import restate  # noqa: E402  (test infrastructure)

CARDS_DIR = Path(ROOT) / "videoseal_b200" / "cards"
SEED = 1234   # same seed as oracle/make_golden.py -> same synthetic checkpoint as the golden fixtures

_tmpdir = None


def tmpdir() -> Path:
    global _tmpdir
    if _tmpdir is None:
        _tmpdir = Path(tempfile.mkdtemp(prefix="vsb200_"))
    return _tmpdir


def load_card(card_name: str) -> dict:
    return yaml.safe_load(open(CARDS_DIR / f"{card_name}.yaml"))


def synthetic_card_on_disk(card_name: str, seed: int = SEED, tiny: dict | None = None):
    """Write <tmp>/<card>.yaml + <card>.pth (checkpoint['model'] = synthetic state_dict). Returns (card_path, spec, sd)."""
    card = load_card(card_name)
    if tiny:
        card = apply_overrides(card, tiny)
    spec = restate.spec_from_card(card)
    sd = restate.synth_state_dict(spec, seed=seed)
    d = tmpdir()
    tag = card_name + ("_" + "_".join(f"{k}{v}" for k, v in sorted(tiny.items())) if tiny else "")
    tag = tag.replace("[", "").replace("]", "").replace(",", "-").replace(" ", "")
    ckpt = d / f"{tag}.pth"
    torch.save({"model": sd}, ckpt)
    card["checkpoint_path"] = str(ckpt)
    card["args"]["attenuation_config"] = str(Path(ROOT) / "videoseal_b200" / "configs" / "attenuation.yaml")
    cpath = d / f"{tag}.yaml"
    yaml.safe_dump(card, open(cpath, "w"))
    return cpath, spec, sd


def apply_overrides(card: dict, o: dict) -> dict:
    import copy
    card = copy.deepcopy(card)
    if "nbits" in o:
        card["args"]["nbits"] = o["nbits"]
    if "num_blocks" in o:
        card["embedder"]["params"]["unet"]["num_blocks"] = o["num_blocks"]
    if "attenuation" in o:
        card["args"]["attenuation"] = o["attenuation"]
    if "extractor" in o:   # a preset of configs/extractor.yaml in place of the card's extractor
        ext = yaml.safe_load(open(Path(ROOT) / "videoseal_b200" / "configs" / "extractor.yaml"))
        card["extractor"] = {"model": o["extractor"], "params": copy.deepcopy(ext[o["extractor"]])}
    if "depths" in o:
        card["extractor"]["params"]["encoder"]["depths"] = o["depths"]
    return card


def make_model_pair(card_name: str, device: str = "cuda:0", seed: int = SEED, tiny: dict | None = None):
    """(product Videoseal on `device`, OracleModel on CPU, oracle spec) sharing one synthetic checkpoint."""
    import videoseal_b200
    cpath, spec, sd = synthetic_card_on_disk(card_name, seed, tiny)
    model = videoseal_b200.load(cpath)
    model = model.eval().to(device)
    return model, restate.OracleModel(spec, sd), spec
