"""
Read-sharded multi-GPU execution (SURVEY.md section 8e): one process per GPU, chunks are independent from
`chunk()` to `stitch()` (`bonito/crf/basecall.py:63-77`), so the only collective on the path is one
broadcast of the parameters at start-up.  The reference itself has no multi-device support (single `--device`,
`bonito/cli/basecaller.py:177`).
"""

import torch
import torch.distributed as dist


def broadcast_parameters(model, src=0):
    """
    Rank `src`'s parameters and buffers to every rank as ONE collective per dtype: the tensors are packed into a flat blob
    (hac: 12.9 MB, sup: 157 MB of fp16), broadcast once (NCCL over NVLink on GPUs, gloo on CPU) and unpacked in place --
    the single start-up broadcast of SURVEY.md section 8e, instead of one small collective per tensor.
    """
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return model
    with torch.no_grad():
        groups = {}
        for t in list(model.parameters()) + list(model.buffers()):
            groups.setdefault((t.dtype, t.device), []).append(t.data)
        for (dtype, device), tensors in sorted(groups.items(), key=lambda kv: str(kv[0])):
            flat = torch.cat([t.reshape(-1) for t in tensors]) if len(tensors) > 1 else tensors[0].reshape(-1).clone()
            dist.broadcast(flat, src=src)
            offset = 0
            for t in tensors:
                t.copy_(flat[offset:offset + t.numel()].view_as(t))
                offset += t.numel()
    if hasattr(model, "invalidate_plan"):
        model.invalidate_plan()
    return model


def pin_to_local_cores(local_rank, local_world):
    """Restrict this process to its share of the host cores (rank r of R gets the r-th contiguous slice), so that the R
    Python processes of one node do not migrate across sockets / share cores while they enqueue kernels."""
    import os
    try:
        cores = sorted(os.sched_getaffinity(0))
        per = len(cores) // max(local_world, 1)
        if per >= 1:
            os.sched_setaffinity(0, cores[local_rank * per:(local_rank + 1) * per])
            return per
    except (AttributeError, OSError):
        pass
    return 0


def shard_reads(reads, rank=None, world=None):
    """Deal whole reads round-robin to ranks, so stitching stays rank-local and no result exchange is needed."""
    if rank is None:
        rank = dist.get_rank() if dist.is_initialized() else 0
    if world is None:
        world = dist.get_world_size() if dist.is_initialized() else 1
    for i, read in enumerate(reads):
        if i % world == rank:
            yield read


def gather_counts(n_samples, device="cpu"):
    """Sum of per-rank sample counts (the `samples per second` line of the CLI, bonito/cli/basecaller.py:160-164)."""
    if not (dist.is_available() and dist.is_initialized()):
        return n_samples
    t = torch.tensor([n_samples], dtype=torch.int64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.SUM)
    return int(t.item())
