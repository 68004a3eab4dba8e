"""Multi-GPU: hyper-samples shard across ranks; ONE all-reduce of the per-candidate EI sum.

The only data-parallel axis of the path is the independent loop over hyper-samples
(chooser/GPEIOptChooser.py:333-340) and the only exchange is the mean over samples
(OPT:270, OPT:294).  One process per GPU (torch.distributed, NCCL over NVLink/NVSwitch):
rank r owns samples r, r+W, r+2W, ...; every rank holds the (small) observed set and the
candidate grid; the message is M floats (400 KB at M=100k) -- latency-sized, so it is issued on the
compute stream right behind the last EI sweep.  The sample->rank map and the summation order inside
a rank are fixed, so results are reproducible for a given world size.
"""
import torch.distributed as dist


def shard(S, rank, world):
    """Indices of the hyper-samples owned by ``rank`` (round-robin, SURVEY.md 8e)."""
    return list(range(rank, S, world))


def world():
    if dist.is_available() and dist.is_initialized():
        return dist.get_rank(), dist.get_world_size()
    return 0, 1


def allreduce_sum_(t, group=None):
    if dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)
    return t


def agree_on_error(exc, device="cpu", group=None):
    """Raise on EVERY rank if any rank failed (e.g. a factorisation that is not positive definite in one rank's shard of
    hyper-samples): a rank that raised alone would leave the others waiting in the EI all-reduce until the NCCL
    timeout.  ``exc``: this rank's exception or None.  One 4-byte MAX all-reduce; a no-op for a single process."""
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1):
        if exc is not None:
            raise exc
        return
    import numpy as np
    import torch
    flag = torch.tensor([1 if exc is not None else 0], dtype=torch.int32, device=device)
    dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
    if int(flag[0]) != 0:
        if exc is not None:
            raise exc
        raise np.linalg.LinAlgError("a hyper-sample owned by another rank is not positive definite")


def allgather_object(obj, device="cpu", group=None):
    """[object of rank 0, object of rank 1, ...] on every rank: ``obj`` pickled into a byte tensor on ``device`` (the
    rank's own GPU with NCCL, "cpu" with gloo), one all-gather of the lengths and one of the padded bytes."""
    if not (dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1):
        return [obj]
    import pickle
    import torch
    W = dist.get_world_size(group)
    data = torch.frombuffer(bytearray(pickle.dumps(obj, protocol=2)), dtype=torch.uint8).to(device)
    n = torch.tensor([data.numel()], dtype=torch.int64, device=device)
    ns = [torch.zeros_like(n) for _ in range(W)]
    dist.all_gather(ns, n, group=group)
    size = max(int(x[0]) for x in ns)
    buf = torch.zeros((size,), dtype=torch.uint8, device=device)
    buf[:data.numel()] = data
    bufs = [torch.zeros_like(buf) for _ in range(W)]
    dist.all_gather(bufs, buf, group=group)
    return [pickle.loads(b[:int(k[0])].cpu().numpy().tobytes()) for b, k in zip(bufs, ns)]


def sharded_mean_ei(local_ei_sum_fn, S, group=None):
    """mean_s EI[s, :] from per-rank partial sums.

    ``local_ei_sum_fn(sample_indices)`` returns this rank's sum over its samples as a 1-D tensor
    (device tensor with NCCL, CPU tensor with gloo).  Ranks with no samples contribute zeros of the
    same shape (obtained by calling with an empty list)."""
    rank, W = world()
    mine = shard(S, rank, W)
    part = local_ei_sum_fn(mine)
    allreduce_sum_(part, group)
    return part / float(S)
