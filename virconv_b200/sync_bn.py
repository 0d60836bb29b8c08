"""SyncBatchNorm on the fast path (tools/train.py --sync_bn: `torch.nn.SyncBatchNorm.convert_sync_batchnorm` before DDP).

torch's SyncBatchNorm (torch/nn/modules/_functions.py) takes a training forward's mean and biased variance over the union of
all ranks' rows, updates the running statistics with the global count, and all-reduces `sum_dy` / `sum_dy_xmu` in the
backward while `dgamma` / `dbeta` stay local.  In eval mode, at world size 1 or without an initialised process group it is
plain BatchNorm.  The plan executor (csrc/executor.cu, vc_exec_forward_sync) and the fused voxel pooling (voxel_pool.py) do
the same by handing small float64 slots of per-channel sums to a REDUCER, `reducer(slot, key)`, which sums `slot` in place
over the ranks on the current stream; `key` = (stream or module tag, layer, 'forward' | 'backward') names the exchange point.

The default reducer is `torch.distributed.all_reduce` on the layers' process group (NCCL is capturable, so a captured step
replays it).  A model's `bn_reducer` attribute, when set, replaces it — and then the exchange runs even at world size 1
(tests substitute a fake through it; a no-op reducer measures the split conv / BN path a multi-rank step runs)."""
from __future__ import annotations

import torch
import torch.distributed as dist

NOT_SET = object()


def _sync_layers(bns):
    return [bn for bn in bns if isinstance(bn, torch.nn.SyncBatchNorm)]


def group_of(bns):
    """The one process group of the SyncBatchNorm layers among `bns` (None: the default group), or NOT_SET when there is none.
    Raises ValueError when they name different groups, or when only some of the layers are SyncBatchNorm: the layers of one
    executor plan exchange over one group."""
    sync = _sync_layers(bns)
    if not sync:
        return NOT_SET
    if len(sync) != len(bns):
        raise ValueError('SyncBatchNorm: %d of %d BatchNorm layers of one plan are SyncBatchNorm' % (len(sync), len(bns)))
    groups = {id(bn.process_group) for bn in sync}
    if len(groups) != 1:
        raise ValueError('SyncBatchNorm: the layers of one plan are on %d different process groups' % len(groups))
    return sync[0].process_group


def world_size(bns):
    """The number of ranks the statistics of the SyncBatchNorm layers among `bns` are taken over: 1 without SyncBatchNorm or
    without an initialised torch.distributed."""
    sync = _sync_layers(bns)
    if not sync or not (dist.is_available() and dist.is_initialized()):
        return 1
    return dist.get_world_size(sync[0].process_group)


def default_reducer(group):
    """The sum of a slot over the ranks of `group`: torch.distributed.all_reduce on the current stream."""
    def reduce(slot, key):
        dist.all_reduce(slot, group=group)
    return reduce


def active(owner, bns):
    """The layers exchange their sums: training-mode SyncBatchNorm with `owner.bn_reducer` set or more than one rank."""
    sync = _sync_layers(bns)
    return bool(sync) and sync[0].training and (getattr(owner, 'bn_reducer', None) is not None or world_size(bns) > 1)


def reducer_for(owner, bns):
    """The reducer of a training forward over the BatchNorm layers `bns` of `owner` (a backbone or a voxel-pooling module),
    None for plain BatchNorm: `owner.bn_reducer` when set, else all_reduce on the layers' group at world size > 1."""
    if not active(owner, bns):
        return None
    hook = getattr(owner, 'bn_reducer', None)
    return hook if hook is not None else default_reducer(group_of(bns))
