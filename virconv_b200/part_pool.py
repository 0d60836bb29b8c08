"""Part-score RoI pooling of TEDMHead's PART branch (VirConv-T / -S) on the sm_90a kernels of csrc/part_pool.cu, which
states the rules.

  * `part_pool`         = gen_sample_grid + bilinear_interpolate_torch_gridsample + the mean of
                          TEDMHead.obtain_conf_preds (ted_head.py:110-156, 425-442) for all scenes in one call, as a
                          torch.autograd.Function whose backward gives the part map's gradient;
  * `obtain_conf_preds` = the drop-in method (bound by reference_env.install(use_fused_part_pool=True)).

The reference loops over the scenes in Python, reads the device once per scene (`nonzero()` in gen_sample_grid) and
takes the part map's gradient through grid_sample's atomic backward, which torch refuses under
`torch.use_deterministic_algorithms(True)`.  Here forward and backward are one launch each, read nothing on the host
(capturable in a CUDA graph), and the backward is bit-identical run to run.  The RoIs get no gradient: VirConv builds
them without one (assign_targets runs under no_grad); RoIs that require one go to the reference method."""
from __future__ import annotations

import torch

from . import _lib, ops
from ._lib import check

MAX_ROIS = 1024     # VC_PART_POOL_MAX_ROIS: RoIs per scene
MAX_GRID = 16       # VC_PART_POOL_MAX_GRID: grid size S (S * S part channels)
GRID_SIZE = 7       # gen_sample_grid's default, which TEDMHead's partial does not override
_REF = 'pcdet.models.roi_heads.ted_head.TEDMHead.obtain_conf_preds (the reference method)'


def _check(parts, rois, grid_size):
    ops._require_cuda(parts, rois)
    if parts.dtype != torch.float32 or rois.dtype != torch.float32:
        raise ValueError(f'part_pool: parts and rois must be float32 (got {parts.dtype}, {rois.dtype}); use {_REF}')
    if not 2 <= grid_size <= MAX_GRID:
        raise ValueError(f'part_pool: grid size {grid_size} outside [2, {MAX_GRID}]; use {_REF}')
    if parts.dim() != 4 or parts.shape[1] != grid_size * grid_size:
        raise ValueError(f'part_pool: parts {tuple(parts.shape)} is not [B, {grid_size * grid_size}, H, W] for a '
                         f'{grid_size} x {grid_size} grid; use {_REF}')
    if rois.dim() != 3 or rois.shape[0] != parts.shape[0] or rois.shape[2] < 7:
        raise ValueError(f'part_pool: rois {tuple(rois.shape)} is not [{parts.shape[0]}, N, >= 7]; use {_REF}')
    if rois.shape[1] > MAX_ROIS:
        raise ValueError(f'part_pool: {rois.shape[1]} RoIs per scene, more than the {MAX_ROIS} the fused kernel '
                         f'supports; use {_REF}')


class _PartPool(torch.autograd.Function):
    @staticmethod
    def forward(ctx, parts, rois, grid_size, grid_offsets, spatial_scale):
        parts_c, rois_c = parts.contiguous(), rois.contiguous()
        B, S2, H, W = parts_c.shape
        N, ld = rois_c.shape[1], rois_c.shape[2]
        geo = (int(grid_size), float(grid_offsets[0]), float(grid_offsets[1]), float(spatial_scale))
        out = torch.empty((B * N, 1), dtype=torch.float32, device=parts.device)
        check(_lib.load().vc_part_pool_fwd(parts_c.data_ptr(), rois_c.data_ptr(), B, N, ld, geo[0], H, W, geo[1], geo[2],
                                           geo[3], out.data_ptr(), ops._stream()), 'vc_part_pool_fwd')
        ctx.save_for_backward(rois_c)
        ctx.geo = geo
        ctx.shape = (B, S2, H, W)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        if not ctx.needs_input_grad[0]:
            return None, None, None, None, None
        (rois,) = ctx.saved_tensors
        S, ox, oy, scale = ctx.geo
        B, S2, H, W = ctx.shape
        N, ld = rois.shape[1], rois.shape[2]
        g = grad_out.contiguous()
        dparts = torch.empty(ctx.shape, dtype=torch.float32, device=rois.device)
        lib = _lib.load()
        nbytes = lib.vc_part_pool_bwd_ws_bytes(B, N, S)
        ws = torch.empty((nbytes,), dtype=torch.uint8, device=rois.device) if nbytes else None
        check(lib.vc_part_pool_bwd(rois.data_ptr(), g.data_ptr(), B, N, ld, S, H, W, ox, oy, scale, dparts.data_ptr(),
                                   ops._p(ws), nbytes, ops._stream()), 'vc_part_pool_bwd')
        return dparts, None, None, None, None


def part_pool(parts, rois, grid_size, grid_offsets, spatial_scale):
    """parts [B, grid_size**2, H, W], rois [B, N, >= 7] (x, y, z, dx, dy, dz, heading), CUDA fp32 -> [B * N, 1]: the mean
    over the grid_size x grid_size parts of each RoI, part p sampling channel p bilinearly (torch.cat of the reference's
    per-scene confi).  Differentiable with respect to parts only.  No host read: capturable."""
    _check(parts, rois, int(grid_size))
    return _PartPool.apply(parts, rois, int(grid_size), grid_offsets, spatial_scale)


_reference_obtain_conf_preds = None     # TEDMHead.obtain_conf_preds as the reference defines it (set by reference_env)


def obtain_conf_preds(self, confi_im, anchors):
    """TEDMHead.obtain_conf_preds (bound by reference_env.install(use_fused_part_pool=True)): confi_im [B, 49, H, W] part
    map, anchors [B, N, >= 7] RoIs -> [B * N, 1] part scores ((0,) when N == 0, as the reference's torch.cat of empty
    tensors gives).  Reads self.grid_offsets and self.featmap_stride (ted_head.py:371-372); the grid is 7 x 7."""
    if anchors.requires_grad:
        if _reference_obtain_conf_preds is None:
            raise RuntimeError('obtain_conf_preds: RoIs that require a gradient need the reference method, which '
                               'reference_env.install(use_fused_part_pool=True) records before binding this one')
        return _reference_obtain_conf_preds(self, confi_im, anchors)
    ops._require_cuda(confi_im, anchors)
    if confi_im.dim() != 4 or confi_im.shape[1] != GRID_SIZE * GRID_SIZE:
        raise ValueError(f'obtain_conf_preds: a part map of shape {tuple(confi_im.shape)}; the 7 x 7 grid needs '
                         f'{GRID_SIZE * GRID_SIZE} channels ({_REF} fails in grid_sample there too)')
    if anchors.dim() == 3 and anchors.shape[1] == 0:
        return torch.empty(0, dtype=confi_im.dtype, device=confi_im.device)
    return part_pool(confi_im, anchors, GRID_SIZE, self.grid_offsets, 1 / self.featmap_stride)
