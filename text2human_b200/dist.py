"""Multi-GPU plumbing for the replica-sharded hot path.

The encode/quantize/decode and sampling paths shard over independent images (SURVEY.md §8e):
every rank runs the same network on its own slice of the batch, there is no data-path collective.
torch.distributed is used only for rendezvous, the bracketing barriers and the max-over-ranks
timing reduction (NCCL on GPUs, gloo in the CPU tests).
"""
import os

import torch
import torch.distributed as dist


def env_rank():
    """(rank, local_rank, world_size) from the torchrun environment (1-process defaults)."""
    return (int(os.environ.get("RANK", "0")), int(os.environ.get("LOCAL_RANK", "0")),
            int(os.environ.get("WORLD_SIZE", "1")))


def init(backend=None, device=None):
    rank, local_rank, world = env_rank()
    if world > 1 and not dist.is_initialized():
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        os.environ.setdefault("MASTER_PORT", "29500")
        kw = {}
        if device is not None and backend == "nccl":
            kw["device_id"] = device
        dist.init_process_group(backend or ("nccl" if torch.cuda.is_available() else "gloo"), **kw)
    return rank, local_rank, world


def world_size():
    """ranks in the default process group (1 without one)"""
    return dist.get_world_size() if dist.is_initialized() else 1


def shard_range(n_items, rank, world):
    """Contiguous, balanced [start, stop) slice of n_items for `rank` (first n_items % world ranks get
    one extra item); empty for ranks beyond n_items."""
    base, extra = divmod(n_items, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


def shard_batch(tensors, rank, world):
    """Slice every tensor of a batch dict / tuple along dim 0 for this rank."""
    def cut(t):
        a, b = shard_range(t.shape[0], rank, world)
        return t[a:b]
    if isinstance(tensors, dict):
        return {k: cut(v) for k, v in tensors.items()}
    return tuple(cut(t) for t in tensors)


def barrier():
    if dist.is_initialized():
        dist.barrier()


def max_over_ranks(value, device=None):
    """max of a python float over all ranks (a step's time is the slowest rank's)."""
    if not dist.is_initialized():
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return t.item()


def sum_over_ranks(value, device=None):
    if not dist.is_initialized():
        return float(value)
    t = torch.tensor([float(value)], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return t.item()


def gather_concat(t):
    """all-gather variable-length dim-0 slices back into the full batch (used by tests / eval only)."""
    if not dist.is_initialized():
        return t
    world = dist.get_world_size()
    sizes = [torch.zeros(1, dtype=torch.long, device=t.device) for _ in range(world)]
    dist.all_gather(sizes, torch.tensor([t.shape[0]], dtype=torch.long, device=t.device))
    mx = int(max(s.item() for s in sizes))
    pad = torch.zeros((mx,) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
    pad[:t.shape[0]] = t
    outs = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(outs, pad)
    return torch.cat([o[:int(s.item())] for o, s in zip(outs, sizes)], 0)
