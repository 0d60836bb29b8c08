"""Rotated-box IoU and NMS for the detector heads, with the reference's names, arguments and results, on the sm_90a kernels
of csrc/iou3d_nms.cu (rules stated there).

Mirrors `pcdet/ops/iou3d_nms/iou3d_nms_utils.py` (`boxes_bev_iou_cpu`, `boxes_iou_bev`, `boxes_iou3d_gpu`, `nms_gpu`,
`nms_normal_gpu`), and adds what the per-scene reference cannot do without reading the device from the host:
`nms_batched` (one NMS over B segments, device results) and `proposal_layer` (`RoIHeadTemplate.proposal_layer`,
roi_head_template.py:80-118, for MULTI_CLASSES_NMS: False) — both free of host reads, so they can be captured in a CUDA
graph.  The GPU functions take CUDA tensors only; `boxes_bev_iou_cpu` takes CPU tensors (or numpy arrays), as in the
reference."""
from __future__ import annotations

import numpy as np
import torch

from . import _lib, ops
from ._lib import check


def _boxes7(t):
    assert t.dim() == 2 and t.shape[1] == 7, f'boxes must be (N, 7), got {tuple(t.shape)}'
    assert t.dtype == torch.float32, t.dtype
    return t.contiguous()


def _pairwise(fn, what, boxes_a, boxes_b):
    ops._require_cuda(boxes_a, boxes_b)
    lib = _lib.load()
    a, b = _boxes7(boxes_a), _boxes7(boxes_b)
    out = torch.empty((a.shape[0], b.shape[0]), dtype=torch.float32, device=a.device)
    check(getattr(lib, fn)(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], out.data_ptr(), ops._stream()), what)
    return out


def boxes_bev_iou_cpu(boxes_a, boxes_b):
    """(N, 7), (M, 7) CPU tensors or numpy arrays -> (N, M) BEV IoU of the same type (iou3d_nms_utils.py:12-28).  Computes
    bit for bit what `boxes_iou_bev` computes on the GPU."""
    is_numpy = isinstance(boxes_a, np.ndarray)
    a = torch.from_numpy(boxes_a) if isinstance(boxes_a, np.ndarray) else boxes_a
    b = torch.from_numpy(boxes_b) if isinstance(boxes_b, np.ndarray) else boxes_b
    assert not (a.is_cuda or b.is_cuda), 'Only support CPU tensors'
    assert a.shape[1] == 7 and b.shape[1] == 7
    a, b = a.float().contiguous(), b.float().contiguous()
    out = torch.zeros((a.shape[0], b.shape[0]), dtype=torch.float32)
    check(_lib.load().vc_boxes_iou_bev_host(a.data_ptr(), a.shape[0], b.data_ptr(), b.shape[0], out.data_ptr()),
          'vc_boxes_iou_bev_host')
    return out.numpy() if is_numpy else out


def boxes_overlap_bev(boxes_a, boxes_b):
    """(N, 7), (M, 7) -> (N, M) BEV intersection area (`iou3d_nms_cuda.boxes_overlap_bev_gpu`)."""
    return _pairwise('vc_boxes_overlap_bev', 'vc_boxes_overlap_bev', boxes_a, boxes_b)


def boxes_iou_bev(boxes_a, boxes_b):
    """(N, 7), (M, 7) -> (N, M) BEV IoU (iou3d_nms_utils.py:31-45)."""
    return _pairwise('vc_boxes_iou_bev', 'vc_boxes_iou_bev', boxes_a, boxes_b)


def boxes_iou3d_gpu(boxes_a, boxes_b):
    """(N, 7), (M, 7) -> (N, M) 3-D IoU (iou3d_nms_utils.py:67-100) in one launch."""
    return _pairwise('vc_boxes_iou3d', 'vc_boxes_iou3d', boxes_a, boxes_b)


def _nms_sorted(boxes, counts, thresh, post_max, normal):
    """boxes [B, n, ld] (each segment sorted by descending score), counts [B] int32 on the device -> keep [B, post_max]
    int32 (row indices, tail -1), num_keep [B] int32."""
    lib = _lib.load()
    B, n, ld = boxes.shape
    assert boxes.dtype == torch.float32 and boxes.stride(2) == 1 and boxes.stride(1) == ld and boxes.stride(0) == n * ld, \
        'boxes must be a contiguous [B, n, ld] float32 tensor'
    keep = torch.empty((B, post_max), dtype=torch.int32, device=boxes.device)
    num = torch.empty((B,), dtype=torch.int32, device=boxes.device)
    ws = torch.empty((max(1, lib.vc_nms_ws_bytes(B, n)),), dtype=torch.uint8, device=boxes.device)
    check(lib.vc_nms_boxes(boxes.data_ptr(), B, n, ld, counts.data_ptr(), float(thresh), 1 if normal else 0, int(post_max),
                           keep.data_ptr(), num.data_ptr(), ws.data_ptr(), ws.numel(), ops._stream()), 'vc_nms_boxes')
    return keep, num


def _nms_one(boxes, scores, thresh, pre_maxsize, normal):
    ops._require_cuda(boxes, scores)
    assert boxes.shape[1] == 7
    order = scores.sort(0, descending=True)[1]
    if pre_maxsize is not None:
        order = order[:pre_maxsize]
    n = order.shape[0]
    if n == 0:
        return order.contiguous(), None
    sboxes = boxes[order].float().contiguous()
    counts = torch.full((1,), n, dtype=torch.int32, device=boxes.device)
    keep, num = _nms_sorted(sboxes.view(1, n, 7), counts, thresh, n, normal)
    k = int(num.item())           # the result length is data dependent
    return order[keep[0, :k].long()].contiguous(), None


def nms_gpu(boxes, scores, thresh, pre_maxsize=None, **kwargs):
    """Rotated BEV NMS (iou3d_nms_utils.py:103-118): boxes (N, 7), scores (N) -> (indices of the kept boxes in descending
    score order, None).  Reads back the kept count."""
    return _nms_one(boxes, scores, thresh, pre_maxsize, False)


def nms_normal_gpu(boxes, scores, thresh, **kwargs):
    """Axis-aligned NMS, heading ignored (iou3d_nms_utils.py:121-135)."""
    return _nms_one(boxes, scores, thresh, None, True)


def nms_batched(boxes, scores, counts, thresh, pre_maxsize, post_maxsize, normal=False):
    """NMS of B segments at once, no host read.  boxes [B, n, ld] (ld >= 7, columns 0..6 used), scores [B, n], counts [B]
    (device) = valid leading rows per segment.  Per segment: the valid rows sorted by descending score, the first
    pre_maxsize of them, greedy NMS at `thresh`, at most post_maxsize kept — what nms_gpu(boxes[b, :counts[b]], ...,
    pre_maxsize)[0][:post_maxsize] returns.  -> keep [B, post_maxsize] int64 row indices into boxes[b] (tail -1),
    num_keep [B] int32."""
    ops._require_cuda(boxes, scores, counts)
    B, n, ld = boxes.shape
    assert ld >= 7 and scores.shape == (B, n)
    k = n if pre_maxsize is None else min(int(pre_maxsize), n)
    if k == 0 or post_maxsize == 0:
        return (torch.full((B, int(post_maxsize)), -1, dtype=torch.int64, device=boxes.device),
                torch.zeros((B,), dtype=torch.int32, device=boxes.device))
    rows = torch.arange(n, device=boxes.device)
    valid = rows.view(1, n) < counts.view(B, 1)
    masked = torch.where(valid, scores, torch.full_like(scores, -float('inf')))
    # stable: padding rows (-inf) stay behind valid rows of equal score
    order = torch.sort(masked, dim=1, descending=True, stable=True)[1][:, :k]
    sboxes = torch.gather(boxes[..., :7].float(), 1, order.unsqueeze(-1).expand(B, k, 7)).contiguous()
    cnt = torch.clamp(counts.to(torch.int32), max=k).contiguous()
    keep, num = _nms_sorted(sboxes, cnt, thresh, int(post_maxsize), normal)
    kl = keep.long()
    sel = torch.gather(order, 1, kl.clamp(min=0))
    return torch.where(kl >= 0, sel, torch.full_like(sel, -1)), num


def _cfg(cfg, name):
    return cfg[name] if isinstance(cfg, dict) else getattr(cfg, name)


def proposal_layer(batch_box_preds, batch_cls_preds, nms_config):
    """`RoIHeadTemplate.proposal_layer` (roi_head_template.py:80-118) for MULTI_CLASSES_NMS: False, as one batched call with
    no host read: batch_box_preds [B, N, 7+C], batch_cls_preds [B, N, num_class] -> rois [B, post, 7+C], roi_scores
    [B, post], roi_labels [B, post] int64 — per scene the top NMS_PRE_MAXSIZE scores (max over classes), NMS_TYPE
    (nms_gpu / nms_normal_gpu) at NMS_THRESH, the first NMS_POST_MAXSIZE kept; rows past the kept count are zero, labels
    are +1 (so 1 in those rows), as in the reference."""
    if _cfg(nms_config, 'MULTI_CLASSES_NMS'):
        raise NotImplementedError('MULTI_CLASSES_NMS (the reference raises as well)')
    ops._require_cuda(batch_box_preds, batch_cls_preds)
    assert batch_box_preds.dim() == 3 and batch_cls_preds.dim() == 3
    nms_type = _cfg(nms_config, 'NMS_TYPE')
    assert nms_type in ('nms_gpu', 'nms_normal_gpu'), nms_type
    B, N, C = batch_box_preds.shape
    post = int(_cfg(nms_config, 'NMS_POST_MAXSIZE'))
    k = min(int(_cfg(nms_config, 'NMS_PRE_MAXSIZE')), N)
    if k == 0 or post == 0:
        return (batch_box_preds.new_zeros((B, post, C)), batch_box_preds.new_zeros((B, post)),
                torch.ones((B, post), dtype=torch.int64, device=batch_box_preds.device))
    scores, labels = torch.max(batch_cls_preds, dim=2)
    _, indices = torch.topk(scores, k=k, dim=1)
    boxes_for_nms = torch.gather(batch_box_preds[..., :7].float(), 1, indices.unsqueeze(-1).expand(B, k, 7)).contiguous()
    counts = torch.full((B,), k, dtype=torch.int32, device=batch_box_preds.device)
    keep, _ = _nms_sorted(boxes_for_nms, counts, float(_cfg(nms_config, 'NMS_THRESH')), post, nms_type == 'nms_normal_gpu')
    kl = keep.long()
    valid = kl >= 0
    selected = torch.gather(indices, 1, kl.clamp(min=0))
    rois = torch.gather(batch_box_preds, 1, selected.unsqueeze(-1).expand(B, post, C))
    rois = torch.where(valid.unsqueeze(-1), rois, 0.0)
    roi_scores = torch.where(valid, torch.gather(scores, 1, selected), 0.0)
    roi_labels = torch.where(valid, torch.gather(labels, 1, selected), 0)
    return rois, roi_scores, roi_labels + 1
