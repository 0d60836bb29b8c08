"""Fused voxel-RoI grid pooling of TEDMHead (SURVEY §8f row 3): a drop-in `NeighborVoxelSAModuleMSG`
(pcdet/ops/pointnet2/pointnet2_stack/voxel_pool_modules.py:8-130) on the sm_90a kernels of csrc/voxel_pool.cu.

Per grouper, the query, the grouping, the position MLP (Conv2d(3->C) + BatchNorm2d), the add, the ReLU and the max over the
samples run as one query pass and one pooling pass, forward and backward, without any [M, C, nsample] tensor.  The
BatchNorm2d statistics come from the nine moments of the relative positions (the conv has no bias); its fold and
running-stat update, and its parameter gradients, are one small float64 kernel each: nothing reads the device on the host,
so a forward + backward can be captured in a CUDA graph.  `mlps_in` / `mlps_out` stay the module's own torch layers.

CUDA fp32 tensors only; C in {16, 32, 64} and nsample <= 64 (the compiled-in limits), `max_pool` only — other
configurations are rejected at construction: use the reference class for them."""
from __future__ import annotations

from typing import List

import torch
import torch.nn as nn

from . import _lib, ops, sync_bn
from ._lib import check
from .roi_pool import VoxelQueryAndGrouping, _i32

CHANNELS = (16, 32, 64)
MAX_NSAMPLE = 64


def voxel_pool_query(max_range, radius, nsample, xyz, new_xyz, new_coords, point_indices, with_moments,
                     deterministic=False):
    """The fused path's query pass: vc_voxel_query's rule (new_coords as (b, z, y, x) int32) -> (idx [M, nsample] int32 of
    global rows, empty [M] uint8, moments [9] float64 of r = xyz[idx] - new_xyz (see vc_voxel_pool_query) or None).
    deterministic: the moments from per-chunk partials added in chunk order (vc_voxel_pool_query_det), the same bits on
    every run; the query itself is the same either way."""
    lib = _lib.load()
    dev = xyz.device
    M = new_coords.shape[0]
    B, Z, Y, X = point_indices.shape
    idx = torch.empty((M, nsample), dtype=torch.int32, device=dev)
    empty = torch.empty((M,), dtype=torch.uint8, device=dev)
    z_range, y_range, x_range = max_range
    args = (M, Z, Y, X, int(nsample), float(radius), int(z_range), int(y_range), int(x_range), new_xyz.data_ptr(),
            xyz.data_ptr(), new_coords.data_ptr(), point_indices.data_ptr(), idx.data_ptr(), empty.data_ptr())
    if deterministic and with_moments:
        moments = torch.empty((9,), dtype=torch.float64, device=dev)
        ws = _workspace(lib.vc_voxel_pool_query_det_ws_bytes(M), dev)
        check(lib.vc_voxel_pool_query_det(*args, moments.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()),
              'vc_voxel_pool_query_det')
        return idx, empty, moments
    moments = torch.zeros((9,), dtype=torch.float64, device=dev) if with_moments else None
    check(lib.vc_voxel_pool_query(*args, ops._p(moments), ops._stream()), 'vc_voxel_pool_query')
    return idx, empty, moments


def _workspace(nbytes, dev):
    """a caller-owned workspace from torch's caching allocator on the current stream (so a CUDA-graph capture takes it
    from the graph's private pool)"""
    return torch.empty((max(int(nbytes), 256),), dtype=torch.uint8, device=dev)


class _VoxelPool(torch.autograd.Function):
    """features_in [N, C], w_pos [C, 3, 1, 1], gamma / beta [C] -> pooled [M, C] (+ argmax, idx, empty, moments: not
    differentiable).  `bn` is the position branch's BatchNorm2d (running statistics, eps, momentum, train / eval).

    Under torch.use_deterministic_algorithms(True) (read once, by the forward) the moments and the backward run the
    deterministic kernels (rules D1-D3 of csrc/voxel_pool.cu): the same bits on every run.  The backward follows the mode
    of its forward, whatever the flag says when it runs."""

    @staticmethod
    def forward(ctx, features_in, w_pos, gamma, beta, xyz, new_xyz, new_coords, point_indices, bn, max_range, radius,
                nsample, reducer, tag):
        lib = _lib.load()
        dev = features_in.device
        N, C = features_in.shape
        M = new_coords.shape[0]
        training = bn.training
        det = torch.are_deterministic_algorithms_enabled()
        idx, empty, moments = voxel_pool_query(max_range, radius, nsample, xyz, new_xyz, new_coords, point_indices, training,
                                               deterministic=det)
        n = M * nsample
        # the position branch's BatchNorm2d: statistics from the moments, running-stat update, fold (one launch)
        w32 = w_pos.detach().reshape(C, 3).contiguous()
        scale = torch.empty((C,), dtype=torch.float32, device=dev)
        shift = torch.empty((C,), dtype=torch.float32, device=dev)
        stat = torch.empty((C, 2), dtype=torch.float64, device=dev)
        momentum = -1.0 if bn.momentum is None else float(bn.momentum)
        sync = reducer is not None and training
        if sync:
            # SyncBatchNorm: [moments, slot count] summed over the ranks, the statistics over the union of their slots
            m10 = torch.empty((10,), dtype=torch.float64, device=dev)
            m10[:9].copy_(moments)
            m10[9:].fill_(float(n))
            reducer(m10, (tag, 0, 'forward'))
            check(lib.vc_voxel_pool_bn_fold_sync(C, 1, m10.data_ptr(), w32.data_ptr(), gamma.data_ptr(), beta.data_ptr(),
                                                 bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                                                 bn.num_batches_tracked.data_ptr(), float(bn.eps), momentum, scale.data_ptr(),
                                                 shift.data_ptr(), stat.data_ptr(), ops._stream()), 'vc_voxel_pool_bn_fold_sync')
            ctx.sync = (reducer, tag, m10)
        else:
            check(lib.vc_voxel_pool_bn_fold(C, n, int(training), ops._p(moments), w32.data_ptr(), gamma.data_ptr(),
                                            beta.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                                            bn.num_batches_tracked.data_ptr(), float(bn.eps), momentum, scale.data_ptr(),
                                            shift.data_ptr(), stat.data_ptr(), ops._stream()), 'vc_voxel_pool_bn_fold')
            ctx.sync = None
        pooled = torch.empty((M, C), dtype=torch.float32, device=dev)
        argmax = torch.empty((M, C), dtype=torch.uint8, device=dev)
        check(lib.vc_voxel_pool_fwd(M, C, int(nsample), features_in.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr(),
                                    idx.data_ptr(), empty.data_ptr(), w32.data_ptr(), scale.data_ptr(), shift.data_ptr(),
                                    pooled.data_ptr(), argmax.data_ptr(), ops._stream()), 'vc_voxel_pool_fwd')
        ctx.save_for_backward(pooled, argmax, idx, empty, xyz, new_xyz, w32, gamma.detach(), stat,
                              moments if training else stat)
        ctx.dims = (N, C, nsample, n, training)
        ctx.deterministic = det
        ctx.mark_non_differentiable(argmax, idx, empty, *(() if moments is None else (moments,)))
        return pooled, argmax, idx, empty, moments

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, grad_pooled, *_):
        lib = _lib.load()
        pooled, argmax, idx, empty, xyz, new_xyz, w32, gamma, stat, moments = ctx.saved_tensors
        N, C, nsample, n, training = ctx.dims
        M = pooled.shape[0]
        dev = pooled.device
        saved = (pooled.data_ptr(), argmax.data_ptr(), idx.data_ptr(), empty.data_ptr(), xyz.data_ptr(), new_xyz.data_ptr())
        if grad_pooled is not None and ctx.deterministic:
            # every element written, in a fixed order (rules D2, D3)
            grad_features_in = torch.empty((N, C), dtype=torch.float32, device=dev)
            sums = torch.empty((C, 4), dtype=torch.float64, device=dev)
            grad_pooled = grad_pooled.contiguous()
            ws = _workspace(lib.vc_voxel_pool_bwd_det_ws_bytes(M, C, N, nsample), dev)
            check(lib.vc_voxel_pool_bwd_det(M, C, N, nsample, grad_pooled.data_ptr(), *saved, grad_features_in.data_ptr(),
                                            sums.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()),
                  'vc_voxel_pool_bwd_det')
        else:
            grad_features_in = torch.zeros((N, C), dtype=torch.float32, device=dev)
            sums = torch.zeros((C, 4), dtype=torch.float64, device=dev)
            if grad_pooled is not None:
                grad_pooled = grad_pooled.contiguous()
                check(lib.vc_voxel_pool_bwd(M, C, N, nsample, grad_pooled.data_ptr(), *saved, grad_features_in.data_ptr(),
                                            sums.data_ptr(), ops._stream()), 'vc_voxel_pool_bwd')
        dw = torch.empty((C, 3, 1, 1), dtype=torch.float32, device=dev)
        dgamma = torch.empty((C,), dtype=torch.float32, device=dev)
        dbeta = torch.empty((C,), dtype=torch.float32, device=dev)
        if ctx.sync is not None:
            # the [C, 4] sums over all ranks for the coupling term of dw; dgamma / dbeta and the local sum dy * r stay local
            reducer, tag, m10 = ctx.sync
            gsums = sums.clone()
            reducer(gsums, (tag, 0, 'backward'))
            check(lib.vc_voxel_pool_bn_grad_sync(C, m10[9:].data_ptr(), sums.data_ptr(), gsums.data_ptr(), moments.data_ptr(),
                                                 w32.data_ptr(), gamma.data_ptr(), stat.data_ptr(), dw.data_ptr(),
                                                 dgamma.data_ptr(), dbeta.data_ptr(), ops._stream()),
                  'vc_voxel_pool_bn_grad_sync')
        else:
            check(lib.vc_voxel_pool_bn_grad(C, n, int(training), sums.data_ptr(), moments.data_ptr() if training else None,
                                            w32.data_ptr(), gamma.data_ptr(), stat.data_ptr(), dw.data_ptr(), dgamma.data_ptr(),
                                            dbeta.data_ptr(), ops._stream()), 'vc_voxel_pool_bn_grad')
        return grad_features_in, dw, dgamma, dbeta, None, None, None, None, None, None, None, None, None, None


def voxel_pool(features_in, xyz, new_xyz, new_coords, voxel2point_indices, mlp_pos, max_range, radius, nsample, owner=None,
               tag=0):
    """One grouper of NeighborVoxelSAModuleMSG between mlps_in[k] and mlps_out[k], fused.

    features_in [N, C] fp32 (the output of mlps_in[k], rows as in voxel2point_indices), xyz [N, 3], new_xyz [M, 3],
    new_coords [M, 4] int32 as (b, z, y, x), voxel2point_indices [B, Z, Y, X] int32 (global rows, -1 = no voxel),
    mlp_pos = Sequential(Conv2d(3, C, 1, bias=False), BatchNorm2d(C)); in train mode its statistics are computed over all
    M * nsample slots and its running statistics advance.
    -> pooled [M, C] fp32 (differentiable in features_in and mlp_pos's parameters), argmax [M, C] uint8 (first maximising
    slot), idx [M, nsample] int32 (global rows), empty [M] bool, moments [9] float64 of the relative positions (train mode;
    None in eval mode).
    A SyncBatchNorm mlp_pos[1] in train mode takes its statistics over the ranks of its process group (sync_bn; moments and
    gradient sums exchanged through `owner.bn_reducer` when set, else all_reduce; `tag` names the grouper in the reducer's
    key).  At world size 1 without a reducer it is the BatchNorm2d above."""
    ops._require_cuda(features_in, xyz, new_xyz, new_coords, voxel2point_indices)
    assert features_in.dtype == torch.float32 and xyz.dtype == torch.float32 and new_xyz.dtype == torch.float32
    conv, bn = mlp_pos[0], mlp_pos[1]
    pooled, argmax, idx, empty, moments = _VoxelPool.apply(
        features_in.contiguous(), conv.weight, bn.weight, bn.bias, xyz.contiguous(), new_xyz.contiguous(), _i32(new_coords),
        _i32(voxel2point_indices), bn, tuple(max_range), radius, int(nsample), sync_bn.reducer_for(owner, [bn]),
        ('voxel_pool', tag))
    return pooled, argmax, idx, empty.bool(), moments


class NeighborVoxelSAModuleMSG(nn.Module):
    """`NeighborVoxelSAModuleMSG` (voxel_pool_modules.py:8-130): same constructor, submodules (state_dict keys and
    shapes), initialisation, forward signature and output, with each grouper's query .. max-pool fused (voxel_pool).
    `bn_reducer` (sync_bn) replaces the all-reduce of a SyncBatchNorm position branch's exchanged sums."""

    bn_reducer = None

    def __init__(self, *, query_ranges: List[List[int]], radii: List[float], nsamples: List[int], mlps: List[List[int]],
                 use_xyz: bool = True, pool_method='max_pool'):
        super().__init__()
        assert len(query_ranges) == len(nsamples) == len(mlps)
        alt = 'use pcdet.ops.pointnet2.pointnet2_stack.voxel_pool_modules.NeighborVoxelSAModuleMSG (the reference class)'
        if pool_method != 'max_pool':
            raise ValueError(f'pool_method={pool_method!r}: the fused voxel pooling implements max_pool only; {alt}')
        for spec, ns in zip(mlps, nsamples):
            if spec[1] not in CHANNELS or not 0 < ns <= MAX_NSAMPLE:
                raise ValueError(f'mlp {list(spec)} with nsample {ns}: the fused voxel pooling is compiled for C in {CHANNELS} '
                                 f'and nsample <= {MAX_NSAMPLE}; {alt}')
        self.groupers = nn.ModuleList()
        self.mlps_in = nn.ModuleList()
        self.mlps_pos = nn.ModuleList()
        self.mlps_out = nn.ModuleList()
        for i in range(len(query_ranges)):
            self.groupers.append(VoxelQueryAndGrouping(query_ranges[i], radii[i], nsamples[i]))
            mlp_spec = mlps[i]
            self.mlps_in.append(nn.Sequential(nn.Conv1d(mlp_spec[0], mlp_spec[1], kernel_size=1, bias=False),
                                              nn.BatchNorm1d(mlp_spec[1])))
            self.mlps_pos.append(nn.Sequential(nn.Conv2d(3, mlp_spec[1], kernel_size=1, bias=False),
                                               nn.BatchNorm2d(mlp_spec[1])))
            self.mlps_out.append(nn.Sequential(nn.Conv1d(mlp_spec[1], mlp_spec[2], kernel_size=1, bias=False),
                                               nn.BatchNorm1d(mlp_spec[2]), nn.ReLU()))
        self.relu = nn.ReLU()
        self.pool_method = pool_method
        self.init_weights()

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, (nn.Conv2d, nn.Conv1d)):
                nn.init.kaiming_normal_(m.weight)
                if m.bias is not None:
                    nn.init.constant_(m.bias, 0)
            if isinstance(m, (nn.BatchNorm2d, nn.BatchNorm1d)):
                nn.init.constant_(m.weight, 1.0)
                nn.init.constant_(m.bias, 0)

    def forward(self, xyz, xyz_batch_cnt, new_xyz, new_xyz_batch_cnt, new_coords, features, voxel2point_indices):
        """xyz [N, 3], new_xyz [M, 3], new_coords [M, 4] (b, x, y, z), features [N, C_in], voxel2point_indices [B, Z, Y, X]
        -> [M, sum_k mlps[k][-1]].  The batch counts are not read: the query uses the global rows of voxel2point_indices and
        the batch index in new_coords (reading the counts would cost a device round trip)."""
        ops._require_cuda(xyz, new_xyz, new_coords, features, voxel2point_indices)
        if xyz.requires_grad or new_xyz.requires_grad:
            raise ValueError('NeighborVoxelSAModuleMSG (fused): no gradient flows to xyz / new_xyz; pass them detached')
        if xyz.dtype != torch.float32 or new_xyz.dtype != torch.float32 or features.dtype != torch.float32:
            raise ValueError('NeighborVoxelSAModuleMSG (fused): fp32 tensors only')
        xyz, new_xyz = xyz.contiguous(), new_xyz.contiguous()
        # change the order to [batch_idx, z, y, x] (no host-built index tensor, so capturable)
        new_coords = _i32(torch.cat([new_coords[:, :1], new_coords[:, 1:].flip(1)], 1))
        v2p = _i32(voxel2point_indices)
        new_features_list = []
        for k in range(len(self.groupers)):
            features_in = self.mlps_in[k](features.permute(1, 0).unsqueeze(0))
            features_in = features_in.permute(0, 2, 1).contiguous()
            features_in = features_in.view(-1, features_in.shape[-1])
            g = self.groupers[k]
            pooled = voxel_pool(features_in, xyz, new_xyz, new_coords, v2p, self.mlps_pos[k], g.max_range, g.radius,
                                g.nsample, owner=self, tag=k)[0]
            new_features = self.mlps_out[k](pooled.t().unsqueeze(0))       # (1, C, M)
            new_features_list.append(new_features.squeeze(dim=0).permute(1, 0))
        return torch.cat(new_features_list, dim=1)
