"""Multi-GPU plumbing: one process per GPU (torchrun), independent utterances sharded across ranks.

The path has no per-step collective — utterances never interact (cfm.py:340-365; attention is per
(b, h), LayerNorm per row, GRN per utterance).  The ONLY collective is one broadcast of the packed
weight buffer at load (PackedDiT.broadcast).  Outputs are gathered on the host side.

Caveat kept from the reference: a ragged batch is padded to the batch maximum N, which leaks into
GRN and into the ODE on padded frames.  To reproduce an unsharded ragged batch
bit-for-bit every shard must pad to the GLOBAL N — `global_frames()` computes it with one
all-reduce(MAX) of an integer; equal-length batches (all BASELINE configs) never need it.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Tuple

import torch
import torch.distributed as dist


def world() -> Tuple[int, int]:
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def shard_range(n_items: int, world_size: int, rank: int) -> range:
    """Contiguous, balanced shards: the first (n_items % world_size) ranks get one extra item."""
    base, extra = divmod(n_items, world_size)
    start = rank * base + min(rank, extra)
    return range(start, start + base + (1 if rank < extra else 0))


def load_weights_distributed(model, weights_fn: Callable[[], dict], src: int = 0):
    """Rank `src` builds + packs the weights, all other ranks allocate the same layout and receive
    the packed buffer in ONE broadcast (NCCL over NVLink for CUDA buffers, gloo in CPU tests)."""
    rank, _ = world()
    if rank == src:
        model.load_weights(weights_fn())
    else:
        model.allocate_weights()
    model.packed.broadcast(src=src)
    return model


def global_frames(local_max_frames: int, device=None) -> int:
    rank, ws = world()
    if ws == 1:
        return int(local_max_frames)
    t = torch.tensor([int(local_max_frames)], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return int(t.item())


def gather_objects(local: list) -> Optional[list]:
    """Host-side gather of per-rank result lists to rank 0 (flattened in rank order)."""
    rank, ws = world()
    if ws == 1:
        return list(local)
    out: List[Optional[list]] = [None] * ws if rank == 0 else None
    dist.gather_object(local, out, dst=0)
    if rank != 0:
        return None
    return [x for part in out for x in part]


def sample_sharded(f5, cond: torch.Tensor, text, duration: torch.Tensor, **kw):
    """Data-parallel F5TTS.sample over the ranks of the default process group: utterance i of the global batch goes
    to the rank whose shard_range holds it, every shard pads to the GLOBAL frame count (one int all-reduce — the only
    communication before the host-side gather), and rank 0 receives the mel outputs in global order (others: None).
    `cond` (b, n, mel), `text` (b, nt) int tensor or list of str, `duration` (b,) are the GLOBAL batch on every rank;
    `y0`, if given, is the global noise (b, N, mel)."""
    rank, ws = world()
    b = cond.shape[0]
    mine = shard_range(b, ws, rank)
    duration = torch.as_tensor(duration).reshape(-1)
    dev = f5.transformer.device
    if len(mine) == 0:
        global_frames(0, device=dev)
        return gather_objects([])
    sl = slice(mine.start, mine.stop)
    text_l = text[sl] if not isinstance(text, list) else text[mine.start:mine.stop]
    # the frame count sample() will derive for this shard (cfm.py:301-319), then the global maximum
    if isinstance(text_l, list):
        text_len = torch.tensor([len(t) for t in text_l])
    else:
        text_len = (text_l != -1).sum(dim=-1)
    lens = torch.maximum(text_len.float(), torch.full((len(mine),), float(cond.shape[1])))
    n_local = int(torch.clip(torch.maximum(lens + 1, duration[sl].float()), 0, kw.get("max_duration", 4096)).max().item())
    n_glob = global_frames(n_local, device=dev)
    y0 = kw.pop("y0", None)
    if y0 is not None:
        y0 = y0[sl]
    out, _ = f5.sample(cond[sl], text_l, duration[sl], y0=y0, pad_frames=n_glob, return_trajectory=False, **kw)
    return gather_objects([o.cpu() for o in out])
