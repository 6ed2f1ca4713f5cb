"""Writes tests/golden/augment_video.pt (test infrastructure only; needs the reference source tree, see oracle/ref_import.py):

    python -m tests.make_golden_augment_video

Runs the UNMODIFIED reference temporal attacks (videoseal/augmentation/video.py: SpeedChange, TemporalReorder, WindowAveraging,
DropFrame) on seeded clips of T in {1, 2, 3, 8, 13, 72} frames at 3 x 24 x 40, reseeding Python's `random` before each call, at
each strength of the reference's commented-out video rows and at fixed / random parameters.  The clips are u8 / 255, stored as
uint8.  A re-indexing attack's output is stored as its index table: the generator runs the same call on a clip whose frame t holds
the value t, reads the table off it, and checks that the real output equals the clip indexed by it.  WindowAveraging outputs are
stored at every sixth row and eighth column (the GPU test also checks the kernel on every pixel against float64).  Also stores the
random draws for fixed seeds, the reprs and column keys of the temporal rows, and the column keys of the reference's video list."""
import os
import random

import torch

from oracle import ref_import

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "augment_video.pt")
TS = (1, 2, 3, 8, 13, 72)
H, W = 24, 40
SEEDS = (0, 1, 2)
# (class, constructor kwargs, call) per case; a call is ("strength", s) through the evaluation's aug(x, mask, s), ("kw", {...}),
# or ("random", None) for the reference's own draws
ROWS = {"SpeedChange": [0.5, 2.0], "WindowAveraging": [(3, 1.0)], "DropFrame": [0.2, 0.5], "TemporalReorder": [(4, 0.7)]}
WINDOW_KW = [dict(window_size=w, alpha=a) for w, a in ((1, 0.3), (2, 0.7), (3, 1.0), (4, 0.5), (5, 0.3), (8, 0.0), (17, 0.7))]
SPEED_KW = [dict(speed_factor=s) for s in (0.5, 0.7, 1.0, 1.3, 2.0)]
REORDER_KW = [dict(chunk_size=c, swap_probability=p) for c, p in ((2, 0.5), (3, 1.0), (4, 0.7), (5, 0.0))]
DROP_KW = [dict(drop_prob=p) for p in (0.0, 0.2, 0.5, 1.0)]


def clips():
    g = torch.Generator().manual_seed(11)
    return {T: torch.randint(0, 256, (T, 3, H, W), generator=g, dtype=torch.uint8) for T in TS}


def main():
    ref_import.install_stubs()
    import videoseal.augmentation as A
    import videoseal.augmentation.video as V
    u8 = clips()
    cases = []
    for T in TS:
        x = u8[T].float() / 255
        ramp = torch.arange(T, dtype=torch.float32).view(T, 1, 1, 1)
        xi, mi = ramp.expand(T, 3, 2, 2).contiguous(), ramp.expand(T, 1, 2, 2).contiguous()
        calls = [("SpeedChange", {}, ("strength", s)) for s in ROWS["SpeedChange"]]
        calls += [("SpeedChange", {}, ("kw", kw)) for kw in SPEED_KW] + [("SpeedChange", {}, ("random", None))]
        calls += [("TemporalReorder", {}, ("strength", s)) for s in ROWS["TemporalReorder"]]
        calls += [("TemporalReorder", {}, ("kw", kw)) for kw in REORDER_KW] + [("TemporalReorder", {}, ("random", None))]
        calls += [("DropFrame", {}, ("strength", s)) for s in ROWS["DropFrame"]]
        calls += [("DropFrame", {}, ("kw", kw)) for kw in DROP_KW] + [("DropFrame", {}, ("random", None))]
        calls += [("WindowAveraging", {}, ("strength", s)) for s in ROWS["WindowAveraging"]]
        calls += [("WindowAveraging", {}, ("kw", kw)) for kw in WINDOW_KW] + [("WindowAveraging", {}, ("random", None))]
        calls += [("WindowAveraging", dict(min_window_size=0), ("kw", dict(window_size=3, alpha=0.7)))]
        for seed in SEEDS:
            for name, ctor, (kind, arg) in calls:
                if kind != "random" and seed != SEEDS[0] and name != "DropFrame" and name != "TemporalReorder":
                    continue        # only the random draws depend on the seed
                aug = getattr(V, name)(**ctor)

                def run(frames, mask):
                    random.seed(seed)
                    if kind == "kw":
                        return aug(frames.clone(), mask.clone(), **arg)
                    if kind == "strength":
                        # a tuple strength fills the forward's parameters in order (the reference would fail on the tuple)
                        return aug(frames.clone(), mask.clone(), *(arg if isinstance(arg, tuple) else (arg,)))
                    return aug(frames.clone(), mask.clone())

                case = {"T": T, "seed": seed, "cls": name, "ctor": ctor, "kind": kind, "arg": arg}
                if name == "WindowAveraging":
                    y, _ = run(x, mi)
                    case["out"] = y[..., ::6, ::8].clone()
                else:
                    yi, mo = run(xi, mi)
                    idx = yi[:, 0, 0, 0].round().long()
                    y, ym = run(x, mi)
                    assert torch.equal(y, x[idx]), (name, T, seed, kind, arg)
                    case["index"] = idx.tolist()
                    case["mask_index"] = mo[:, 0, 0, 0].round().long().tolist()
                    assert torch.equal(ym, mo)
                cases.append(case)
    draws = {}
    for seed in SEEDS:
        random.seed(seed)
        d = {"speed": V.SpeedChange().get_random_speed(), "chunk": V.TemporalReorder().get_random_chunk_size(),
             "window": V.WindowAveraging().get_random_window_size(), "alpha": V.WindowAveraging().get_random_alpha(),
             "state_after": random.random()}
        draws[seed] = d
    reprs = {name: str(getattr(V, name)()) for name in ROWS}
    keys = {name: [(str(getattr(V, name)()) + f"_{s}").replace(", ", "_") for s in ss] for name, ss in ROWS.items()}
    video_names = [(str(a) + f"_{s}").replace(", ", "_") for a, ss in A.get_validation_augs(is_video=True) for s in ss]
    torch.save({"shape": (H, W), "clips": u8, "cases": cases, "draws": draws, "reprs": reprs, "keys": keys,
                "video_names": video_names}, OUT)
    print(f"wrote {OUT}: {os.path.getsize(OUT) / 1024:.0f} KB, {len(cases)} cases")


if __name__ == "__main__":
    main()
