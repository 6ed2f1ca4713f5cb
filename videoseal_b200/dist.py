"""Frame sharding across the GPUs of one box (SURVEY.md §8e): frames are independent units at inference, so a clip is cut
into contiguous frame ranges aligned to `step_size` (the key-frame groups of models/videoseal.py:292-340 stay whole), every
rank runs embed+detect on its own range with its own replica of the weights, and ONE all-gather (NCCL over NVLink on GPUs,
gloo in the CPU tests) reassembles the outputs.  There is no other exchange on the data path.

The reference has no inference-time parallelism (single process, single device: models/wam.py:20-23); its NCCL use is
training-only (utils/dist.py).  One process per GPU, launched with torchrun.
"""
from __future__ import annotations

import math
from typing import Callable, List, Tuple

import torch
import torch.distributed as dist


def shard_bounds(num_frames: int, world_size: int, step_size: int = 1) -> List[Tuple[int, int]]:
    """Contiguous [start, end) frame ranges, one per rank, boundaries on multiples of `step_size` (so that each key-frame
    group lives on one rank and `repeat` / `alternate` video modes give results identical to the unsharded call).
    Ranks may get empty ranges when there are fewer key-frame groups than ranks."""
    if num_frames < 0 or world_size < 1 or step_size < 1:
        raise ValueError("bad sharding arguments")
    groups = (num_frames + step_size - 1) // step_size
    base, rem = divmod(groups, world_size)
    bounds, g0 = [], 0
    for r in range(world_size):
        g1 = g0 + base + (1 if r < rem else 0)
        bounds.append((min(g0 * step_size, num_frames), min(g1 * step_size, num_frames)))
        g0 = g1
    return bounds


def shard_unit(model) -> int:
    """The `step_size` to shard a clip for `model` with: frames that one embed call must see together.  That is a key frame and
    its step_size - 1 followers, or, for a temporal U-Net or a DVMark embedder, whose 3x3x3 convs mix the key frames of one reference chunk
    (models/videoseal.py:292-320), whole chunks of chunk_size * step_size frames.  A DVMark extractor mixes the frames of one
    detect chunk (videoseal.py:373-379), so its shards also hold whole chunks of chunk_size frames."""
    step = int(model.step_size)
    unit = step * int(model.chunk_size) if getattr(model, "temporal", False) else step
    return math.lcm(unit, int(model.chunk_size)) if getattr(model, "dvmark", False) else unit


def subshard_bounds(num_frames: int, world_size: int, step_size: int = 1, subshards: int = 2) -> List[List[Tuple[int, int]]]:
    """Interleaved sharding for OVERLAPPED reassembly: the clip is cut into `subshards` contiguous segments and every segment into
    `world_size` contiguous ranges (boundaries on multiples of `step_size`); rank r owns range r of every segment.  The all-gather of
    segment s then reassembles frames [seg_start_s, seg_end_s) in frame order without any copy, and it can run (on NCCL's stream)
    while the ranks are still computing segment s+1.  Returns bounds[rank][segment] = (start, end).
    Requires equal ranges (num_frames a multiple of world_size * subshards * step_size)."""
    unit = world_size * subshards * step_size
    if num_frames % unit != 0:
        raise ValueError(f"interleaved sub-shards need num_frames % (world_size * subshards * step_size) == 0, got {num_frames} % {unit}")
    n = num_frames // (world_size * subshards)
    return [[((s * world_size + r) * n, (s * world_size + r + 1) * n) for s in range(subshards)] for r in range(world_size)]


def all_gather_ragged(local: torch.Tensor, sizes: List[int], group=None) -> torch.Tensor:
    """All-gather along dim 0 of per-rank tensors with different leading sizes (`sizes[r]` rows on rank r): each rank pads to
    the maximum, one `all_gather`, padding dropped.  Returns the concatenation in rank order on every rank."""
    world = dist.get_world_size(group)
    assert len(sizes) == world and local.shape[0] == sizes[dist.get_rank(group)]
    mx = max(sizes)
    if mx == 0:
        return local
    pad = torch.zeros((mx,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    pad[: local.shape[0]] = local
    out = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(out, pad, group=group)
    return torch.cat([o[:n] for o, n in zip(out, sizes)], dim=0)


def embed_detect_sharded(embed_fn: Callable, detect_fn: Callable, frames: torch.Tensor, msgs: torch.Tensor, step_size: int,
                         gather_frames: bool = True, group=None, model=None):
    """Shard `frames` [F,3,H,W] (present on every rank, or at least this rank's range) over the process group, cut on multiples
    of `step_size`, and with `model` given (the Videoseal behind embed_fn) also on multiples of shard_unit(model), so that a temporal
    U-Net's chunks stay whole; run
    `embed_fn(frames_shard, msgs) -> imgs_w_shard` and `detect_fn(imgs_w_shard) -> logits_shard` locally, and all-gather.
    Returns (imgs_w [F,3,H,W] or the local shard if not gather_frames, logits [F, 1+K], (start, end) of this rank)."""
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    if model is not None:
        step_size = math.lcm(step_size, shard_unit(model))
    bounds = shard_bounds(frames.shape[0], world, step_size)
    s, e = bounds[rank]
    local = frames[s:e]
    if e > s:
        imgs_w = embed_fn(local, msgs)
        logits = detect_fn(imgs_w)
    else:
        imgs_w = local.new_zeros((0,) + tuple(frames.shape[1:]))
        logits = None
    sizes = [b[1] - b[0] for b in bounds]
    # logits width is only known to ranks that ran detect: agree on it first
    width = torch.tensor([0 if logits is None else logits.shape[1]], device=frames.device)
    dist.all_reduce(width, op=dist.ReduceOp.MAX, group=group)
    if logits is None:
        logits = frames.new_zeros((0, int(width.item())))
    all_logits = all_gather_ragged(logits.contiguous(), sizes, group)
    all_imgs = all_gather_ragged(imgs_w.contiguous(), sizes, group) if gather_frames else imgs_w
    return all_imgs, all_logits, (s, e)


def extract_message_sharded(logits_local: torch.Tensor, group=None) -> torch.Tensor:
    """`extract_message(aggregation='avg')` over a sharded clip (models/videoseal.py:411-428): local sum of bit logits +
    frame count, one all-reduce of K+1 floats, threshold at 0."""
    if logits_local.dim() != 2:
        raise NotImplementedError("extract_message_sharded takes pooled logits [F, 1+K]; per-pixel maps of a pixel-wise model "
                                  "are not sharded")
    k = logits_local.shape[1] - 1
    buf = torch.zeros(k + 1, device=logits_local.device, dtype=torch.float32)
    if logits_local.shape[0]:
        buf[:k] = logits_local[:, 1:].sum(dim=0)
        buf[k] = logits_local.shape[0]
    dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    return ((buf[:k] / buf[k].clamp_min(1)) > 0).unsqueeze(0)
