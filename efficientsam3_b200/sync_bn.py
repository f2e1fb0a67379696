"""Synchronised BatchNorm for the native training graphs: `nn.SyncBatchNorm` in train mode, as
`torch.nn.SyncBatchNorm.convert_sync_batchnorm(model)` leaves the students' BatchNorms (the reference trainers' `--use-sync-bn`).

A BatchNorm is synchronised only when it is an `nn.SyncBatchNorm`, in train mode, `torch.distributed` is initialised and the world
size of its `process_group` (default: WORLD) is > 1 -- the conditions of torch's `SyncBatchNorm.forward`.  Everything else (plain
`BatchNorm2d`, frozen BN, one rank) runs the per-rank kernels unchanged.

When it is synchronised:
  forward   es3_bn_stats_partial (count, mean, M2 of this rank, fp64) -> all-gather -> es3_bn_stats_combine (Chan's formula in
            rank order: mean / invstd / scale / shift, running buffers over the total count, num_batches_tracked)
  backward  es3_bn_act_bwd_partial (sum g, sum g (z - mean) of this rank; this rank's dgamma / dbeta, as torch: the gradient
            exchange averages them) -> all-gather -> es3_bn_bwd_coef -> the unchanged es3_bn_act_bwd_apply
Partials, not running sums, are exchanged, and every rank combines them in the same order: the statistics and the running
buffers are bit-identical on every rank.  On NCCL nothing waits on the host.

On NCCL the partials travel on a private communicator over the group's ranks: one NCCL communicator runs its collectives in
order, so an exchange queued behind the asynchronous head all-reduce (stage1.optim.FlatAdamW.head_grads_ready) would hold the
body backward until that all-reduce finished.
"""
from __future__ import annotations

import torch
import torch.distributed as dist
import torch.nn as nn

from . import ops

__all__ = ["sync_group", "repmixer_sync_group", "exchange_group", "all_gather_partials", "batch_stats", "bn_act_bwd", "exchanges"]

exchanges = 0           # all-gathers issued by this process (scripts/bench_syncbn.py counts them per step)
_PRIVATE: dict = {}     # process group -> its private NCCL communicator for the BN exchanges
_PRIVATE_WORLD = None   # the default group _PRIVATE was filled under (a new init_process_group starts a fresh cache)


def sync_group(norm) -> object | None:
    """The process group `norm` synchronises over, or None when it normalises with this rank's statistics alone."""
    if not isinstance(norm, nn.SyncBatchNorm) or not norm.training:
        return None
    if not (dist.is_available() and dist.is_initialized()):
        return None
    group = norm.process_group if norm.process_group is not None else dist.group.WORLD
    return group if dist.get_world_size(group) > 1 else None


def repmixer_sync_group(bns) -> object | None:
    """The process group the four BatchNorms of a RepMixerBlock synchronise over, or None; they must agree."""
    groups = [sync_group(bn) for bn in bns]
    if all(g is None for g in groups):
        return None
    if any(g is not groups[0] for g in groups):
        raise NotImplementedError("the BatchNorms of one RepMixerBlock must all synchronise over the same process group, or none of "
                                  "them (convert_sync_batchnorm converts all of them with one group)")
    return groups[0]


def _uses_nccl(group, on_cuda: bool) -> bool:
    # "nccl", or a multi-device backend such as "cpu:gloo,cuda:nccl" (init_process_group() without a backend): CUDA tensors go to NCCL
    return on_cuda and "nccl" in dist.get_backend(group)


def exchange_group(group, on_cuda: bool):
    """The group the partials of a BN synchronised over `group` travel on: on NCCL a private communicator over the same ranks."""
    global _PRIVATE_WORLD
    if not _uses_nccl(group, on_cuda):
        return group
    if _PRIVATE_WORLD is not dist.group.WORLD:      # destroy_process_group + a new init: the cached communicators are gone
        _PRIVATE.clear()
        _PRIVATE_WORLD = dist.group.WORLD
    g = _PRIVATE.get(group)
    if g is None:   # created once, by every member at the same (first) synchronised forward
        g = dist.new_group(ranks=dist.get_process_group_ranks(group), backend="nccl", use_local_synchronization=True)
        _PRIVATE[group] = g
    return g


def all_gather_partials(part: torch.Tensor, group) -> torch.Tensor:
    """[W, *part.shape]: every rank's `part`, in rank order.  NCCL: all_gather_into_tensor (no host sync); other backends: the
    list form, as torch's SyncBatchNorm uses on gloo."""
    global exchanges
    part = part.contiguous()
    W = dist.get_world_size(group)
    out = torch.empty((W, *part.shape), dtype=part.dtype, device=part.device)
    if _uses_nccl(group, part.is_cuda):
        dist.all_gather_into_tensor(out, part, group=group)
    else:
        dist.all_gather(list(out.unbind(0)), part, group=group)
    exchanges += 1
    return out


def batch_stats(norm, z, gamma=None, beta=None, running_mean=None, running_var=None):
    """Train-mode statistics of `norm` over z [..., C] bf16 -> (mean, invstd, scale, shift, sync).  gamma / beta / running
    buffers default to the module's own (a caller that pads channels passes padded copies).  `sync` is None for per-rank
    statistics, else what bn_act_bwd needs to synchronise the backward."""
    gamma = norm.weight.detach() if gamma is None else gamma
    beta = norm.bias.detach() if beta is None else beta
    running_mean = norm.running_mean if running_mean is None else running_mean
    running_var = norm.running_var if running_var is None else running_var
    group = sync_group(norm)
    if group is None:
        return (*ops.bn_stats(z, gamma, beta, norm.eps, norm.momentum, running_mean, running_var, norm.num_batches_tracked), None)
    group = exchange_group(group, z.is_cuda)
    parts = all_gather_partials(ops.bn_stats_partial(z), group)
    mean, invstd, scale, shift, total = ops.bn_stats_combine(parts, gamma, beta, norm.eps, norm.momentum, running_mean, running_var,
                                                             norm.num_batches_tracked)
    return mean, invstd, scale, shift, (group, total)


def bn_act_bwd(da, z, scale, shift, act, mode, mean, invstd, dgamma, dbeta, sync=None):
    """ops.bn_act_bwd, with the batch-statistics sums taken over every rank of the group when `sync` (from batch_stats) is set."""
    if sync is None:
        return ops.bn_act_bwd(da, z, scale, shift, act, mode, mean, invstd, dgamma, dbeta)
    group, total = sync
    part = ops.bn_act_bwd_partial(da, z, scale, shift, act, mean, invstd, dgamma, dbeta)
    coef = ops.bn_bwd_coef(all_gather_partials(part, group), total, scale, mean, invstd)
    return ops.bn_act_bwd_apply(da, z, scale, shift, act, coef)
