"""Operator API of the hot path - same names / argument meaning as the reference's `mmdet.ops`
and `mmdet.core` entry points, backed by the C ABI (PyTorch tensors in, PyTorch tensors out).

  CropSplit / crop_split   <- MM/mmdet/ops/crop/crop_split.py:12-49
  nms                      <- MM/mmdet/ops/nms/nms_wrapper.py:7-60
  multiclass_nms_idx       <- MM/mmdet/core/post_processing/bbox_nms.py:79-146
  fast_nms                 <- MM/mmdet/models/anchor_heads/sipmask_head.py:868-910
  mask_assemble            <- MM/mmdet/models/anchor_heads/sipmask_head.py:609-627 (fused)
  DeformConv(Pack) / deform_conv        <- MM/mmdet/ops/dcn/deform_conv.py:14-94,192-300 (with the backward)
  SigmoidFocalLoss / sigmoid_focal_loss <- MM/mmdet/ops/sigmoid_focal_loss/sigmoid_focal_loss.py:8-52
  sipmask_mask_targets / sipmask_mask_loss / sipmask_head_mask_loss
                           <- MM/mmdet/models/anchor_heads/sipmask_head.py:403-484 (the mask loss, fused)
All tensors must be CUDA tensors on an sm_90 device; there is no CPU path.
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import _lib as L


def _need_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.SmbError('sipmask_b200 ops need CUDA tensors (no CPU fallback); got %s' % t.device)


def _dt(t):
    if t.dtype == torch.float32:
        return L.F32
    if t.dtype == torch.float16:
        return L.F16
    raise L.SmbError('unsupported dtype %s' % t.dtype)


# ------------------------------------------------------------------------------------------ CropSplit
@L.device_guard
def crop_split(data, rois, c=2):
    """data [c*c,H,W,N] contiguous, rois [N,4] -> [H,W,N] (ops/crop/crop_split.py:12-25)."""
    _need_cuda(data, rois)
    if not data.is_contiguous():
        raise L.SmbError('input must be contiguous')       # AT_CHECK in crop_split_cuda.cpp:17
    cc, H, W, N = data.shape
    rois = rois.to(data.dtype).contiguous()
    out = torch.empty((H, W, N), dtype=data.dtype, device=data.device)
    L.check(L.lib().smb_crop_split_forward(L.ptr(data), L.ptr(rois), L.ptr(out), _dt(data), H, W, int(c), N,
                                           L.stream_ptr()), 'smb_crop_split_forward')
    return out


@L.device_guard
def crop_split_backward(grad_output, rois, c=2):
    """grad_output [H,W,N], rois [N,4] -> grad_input [c*c,H,W,N] (ops/crop/crop_split.py:27-38)."""
    _need_cuda(grad_output, rois)
    g = grad_output.contiguous()
    H, W, N = g.shape
    rois = rois.to(g.dtype).contiguous()
    out = torch.empty((c * c, H, W, N), dtype=g.dtype, device=g.device)
    L.check(L.lib().smb_crop_split_backward(L.ptr(g), L.ptr(rois), L.ptr(out), _dt(g), H, W, int(c), N, L.stream_ptr()),
            'smb_crop_split_backward')
    return out


@L.device_guard
def crop_split_gt(data, rois, c=2):
    """data [H,W,N], rois [N,4] -> data inside roi n, 0 outside (ops/crop/crop_split_gt.py:9-25); also its own backward."""
    _need_cuda(data, rois)
    if not data.is_contiguous():
        raise L.SmbError('input must be contiguous')
    H, W, N = data.shape
    rois = rois.to(data.dtype).contiguous()
    out = torch.empty_like(data)
    L.check(L.lib().smb_crop_split_gt(L.ptr(data), L.ptr(rois), L.ptr(out), _dt(data), H, W, N, L.stream_ptr()),
            'smb_crop_split_gt')
    return out


class _CropSplitFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, rois, c):
        ctx.c = c
        ctx.save_for_backward(rois)
        return crop_split(data, rois, c)

    @staticmethod
    def backward(ctx, grad_output):
        (rois,) = ctx.saved_tensors
        return crop_split_backward(grad_output, rois, ctx.c), None, None


class _CropSplitGtFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, rois, c):
        ctx.c = c
        ctx.save_for_backward(rois)
        return crop_split_gt(data, rois, c)

    @staticmethod
    def backward(ctx, grad_output):
        (rois,) = ctx.saved_tensors
        return crop_split_gt(grad_output.contiguous(), rois, ctx.c), None, None


class CropSplit(nn.Module):
    """mmdet.ops.CropSplit (ops/crop/crop_split.py:42-49), differentiable w.r.t. `data` like the reference."""

    def __init__(self, c=2):
        super().__init__()
        self.c = c

    def forward(self, data, rois):
        if data.requires_grad and torch.is_grad_enabled():
            return _CropSplitFn.apply(data, rois, self.c)
        return crop_split(data, rois, self.c)


class CropSplitGt(nn.Module):
    """mmdet.ops.CropSplitGt (ops/crop/crop_split_gt.py:29-36)."""

    def __init__(self, c=2):
        super().__init__()
        self.c = c

    def forward(self, data, rois):
        if data.requires_grad and torch.is_grad_enabled():
            return _CropSplitGtFn.apply(data, rois, self.c)
        return crop_split_gt(data, rois, self.c)


# ------------------------------------------------------------------------------------------------ nms
@L.device_guard
def nms(dets, iou_thr, device_id=None, cmp_ge=False):
    """Same contract as mmdet.ops.nms: returns (dets[inds], inds); numpy in -> numpy out."""
    is_numpy = isinstance(dets, np.ndarray)
    if is_numpy:
        dev = 'cuda:%d' % (device_id if device_id is not None else torch.cuda.current_device())
        dets_th = torch.from_numpy(dets).to(dev)
    elif isinstance(dets, torch.Tensor):
        dets_th = dets
    else:
        raise TypeError('dets must be either a Tensor or numpy array, but got {}'.format(type(dets)))
    _need_cuda(dets_th)
    n = dets_th.shape[0]
    if n == 0:
        inds = dets_th.new_zeros(0, dtype=torch.long)
    else:
        d = dets_th.float().contiguous()
        keep = torch.empty(n, dtype=torch.long, device=d.device)
        cnt = torch.zeros(1, dtype=torch.int32, device=d.device)
        L.check(L.lib().smb_nms(L.ptr(d), n, ctypes.c_float(iou_thr), int(cmp_ge), 1, L.ptr(keep), L.ptr(cnt),
                                L.stream_ptr()), 'smb_nms')
        inds = keep[:int(cnt.item())]
    if is_numpy:
        inds = inds.cpu().numpy()
        return dets[inds, :], inds
    return dets[inds, :], inds


SOFT_NMS_METHODS = {'linear': 1, 'gaussian': 2}         # SMB_SOFT_NMS_LINEAR / SMB_SOFT_NMS_GAUSSIAN (nms_wrapper.py:107)
SOFT_NMS_MAX = 5120                                     # candidates per list (MAXN in nms.cu)


def _soft_method(method):
    if method not in SOFT_NMS_METHODS:
        raise ValueError('Invalid method for SoftNMS: {}'.format(method))
    return SOFT_NMS_METHODS[method]


@L.device_guard
def soft_nms(dets, iou_thr, method='linear', sigma=0.5, min_score=1e-3, device_id=None):
    """Same contract as mmdet.ops.soft_nms (nms_wrapper.py:63-118): returns (new_dets, inds) of the input's type and dtype,
    the kept rows in selection order with their decayed scores, and their positions in `dets`.  Numpy input runs on the
    current device (or device_id) and returns numpy.  The arithmetic is float32 whatever the dtype: float64 input is
    rounded to float32 and the result converted back (the reference would compute in float64).  Empty input returns empty
    arrays (the reference raises IndexError).  At most 5120 rows."""
    code = _soft_method(method)
    is_numpy = isinstance(dets, np.ndarray)
    if is_numpy:
        dev = 'cuda:%d' % (device_id if device_id is not None else torch.cuda.current_device())
        dets_th = torch.from_numpy(dets).to(dev)
    elif isinstance(dets, torch.Tensor):
        dets_th = dets
    else:
        raise TypeError('dets must be either a Tensor or numpy array, but got {}'.format(type(dets)))
    _need_cuda(dets_th)
    n = dets_th.shape[0]
    if n > SOFT_NMS_MAX:
        raise L.SmbError('soft_nms: %d boxes, at most %d per list' % (n, SOFT_NMS_MAX))
    d = dets_th.float().contiguous().reshape(n, 5)
    out = torch.empty((n, 5), dtype=torch.float32, device=d.device)
    inds = torch.empty((n,), dtype=torch.long, device=d.device)
    cnt = torch.zeros(1, dtype=torch.int32, device=d.device)
    L.check(L.lib().smb_soft_nms(L.ptr(d), n, ctypes.c_float(iou_thr), code, ctypes.c_float(sigma), ctypes.c_float(min_score),
                                 L.ptr(out), L.ptr(inds), L.ptr(cnt), L.stream_ptr()), 'smb_soft_nms')
    k = int(cnt.item())
    new_dets, inds = out[:k].to(dets_th.dtype), inds[:k]
    if is_numpy:
        return new_dets.cpu().numpy().astype(dets.dtype), inds.cpu().numpy().astype(np.int64)
    return new_dets, inds


def nms_type(nms_cfg):
    """The `type` of an nms config (bbox_nms.py:108: 'nms' when absent)."""
    if isinstance(nms_cfg, dict):
        return nms_cfg.get('type', 'nms')
    return getattr(nms_cfg, 'type', None) or 'nms'


def soft_nms_args(nms_cfg):
    """(iou_thr, method code, sigma, min_score) of a soft_nms config, with soft_nms's defaults."""
    get = nms_cfg.get if isinstance(nms_cfg, dict) else (lambda k, d: getattr(nms_cfg, k, d))
    if get('iou_thr', None) is None:
        raise ValueError('soft_nms config needs iou_thr (soft_nms(dets, iou_thr, ...) has no default)')
    return (float(get('iou_thr', None)), _soft_method(get('method', 'linear')), float(get('sigma', 0.5)),
            float(get('min_score', 1e-3)))


# ------------------------------------------------------------------------------------- decode + top-k
def level_descs(cls_list, box_list, ctr_list, strides, box_scales):
    """smb_level_t array for one image's per-level channel-last fp32 views (cls [h,w,C], box [h,w,4], ctr [h,w,1|]):
    pointers and row pitches from the views, (box_scales[l], strides[l]) as the box scale when box_scales is given.
    Returns (levels, views to keep alive while the array is in use)."""
    nl = len(cls_list)
    lv = (L.Level * nl)()
    keep_alive = []
    for i in range(nl):
        c, b, t = cls_list[i], box_list[i], ctr_list[i]
        _need_cuda(c, b, t)
        assert c.dtype == torch.float32 and b.dtype == torch.float32 and t.dtype == torch.float32
        assert c.stride(-1) == 1 and b.stride(-1) == 1
        h, w = c.shape[0], c.shape[1]
        assert c.stride(0) == w * c.stride(1) and b.stride(0) == w * b.stride(1)
        t2 = t if t.dim() == 3 else t.reshape(h, w, -1)      # a reshape would renumber the strides of a 1-wide level
        assert t2.stride(0) == w * t2.stride(1)
        keep_alive.append(t2)
        bs, bm = (1.0, 1.0) if box_scales is None else (float(box_scales[i]), float(strides[i]))
        lv[i] = L.Level(c.data_ptr(), t2.data_ptr(), b.data_ptr(), c.stride(1), t2.stride(1), b.stride(1), h, w,
                        int(strides[i]), bs, bm)
    return lv, keep_alive


def decode_workspace_bytes(levels, nms_pre):
    return int(L.lib().smb_decode_workspace_bytes(len(levels), levels, int(nms_pre)))


@L.device_guard
def decode_topk(cls_list, box_list, ctr_list, strides, img_shape, nms_pre, scale_factor=None, box_scales=None, geom=None,
                out=None, workspace=None):
    """Per-level tensors channel-last fp32: cls [h,w,C], box [h,w,4] (distances x stride), ctr [h,w,1|].
    geom: a device geometry row (geom_row), read when the kernels run in place of img_shape and scale_factor.
    out / workspace: the (boxes, scores, ctr, loc) buffers and a uint8 tensor of decode_workspace_bytes to use; with both
    the call only launches (graph-capturable).

    Returns cand_boxes [n,4], cand_scores [n,C], cand_ctr [n], cand_loc [n] int32."""
    nl = len(cls_list)
    C = cls_list[0].shape[-1]
    lv, keep_alive = level_descs(cls_list, box_list, ctr_list, strides, box_scales)
    lib = L.lib()
    dev = cls_list[0].device
    if workspace is None:
        workspace = torch.empty(decode_workspace_bytes(lv, nms_pre), dtype=torch.uint8, device=dev)
    if out is None:
        n = sum(min(c.shape[0] * c.shape[1], nms_pre) if nms_pre > 0 else c.shape[0] * c.shape[1] for c in cls_list)
        out = (torch.empty((n, 4), dtype=torch.float32, device=dev), torch.empty((n, C), dtype=torch.float32, device=dev),
               torch.empty((n,), dtype=torch.float32, device=dev), torch.empty((n,), dtype=torch.int32, device=dev))
    args = [L.ptr(t) for t in out] + [L.ptr(workspace), ctypes.c_size_t(workspace.numel()), L.stream_ptr()]
    if geom is not None:
        L.check(lib.smb_decode_topk_dev(nl, lv, C, int(nms_pre), L.ptr(geom), *args), 'smb_decode_topk_dev')
        return out
    sf = None
    if scale_factor is not None:
        a = np.atleast_1d(np.asarray(scale_factor, dtype=np.float32))
        sf = L.f4(a if a.size == 4 else [a[0]] * 4)
    L.check(lib.smb_decode_topk(nl, lv, C, int(nms_pre), int(img_shape[0]), int(img_shape[1]), sf, *args), 'smb_decode_topk')
    return out


def pair_decode_workspace_bytes(levels, num_classes, nms_pre):
    return int(L.lib().smb_pair_decode_workspace_bytes(len(levels), levels, int(num_classes), int(nms_pre)))


@L.device_guard
def pair_decode_topk(cls_list, box_list, ctr_list, strides, img_shape, nms_pre=1000, score_thr=0.05, box_scales=None,
                     geom=None, out=None, workspace=None):
    """SipMask-benchmark candidate selection (smb_pair_decode_topk).  Per-level channel-last fp32 tensors as decode_topk:
    cls [h,w,C] logits, ctr [h,w,1|], box [h,w,4]; distances are relu(box * box_scales[l]) * strides[l] when box_scales is
    given (raw bbox_pred), else relu(box).  Returns (boxes [n,4], scores [n] = sqrt(cls * ctr), labels [n] int32 0-based,
    loc [n] int32, n_cand device int32 [1]); n is the slot capacity, rows past n_cand are zero / -1.
    geom / out / workspace as decode_topk (geom in place of img_shape; the workspace of pair_decode_workspace_bytes)."""
    nl = len(cls_list)
    C = cls_list[0].shape[-1]
    lv, keep_alive = level_descs(cls_list, box_list, ctr_list, strides, box_scales)
    lib = L.lib()
    dev = cls_list[0].device
    if out is None:
        n = lib.smb_pair_decode_slots(nl, lv, C, int(nms_pre))
        if n < 0:
            raise L.SmbError('pair_decode_topk: unsupported levels / nms_pre=%d' % nms_pre)
        out = (torch.empty((n, 4), dtype=torch.float32, device=dev), torch.empty((n,), dtype=torch.float32, device=dev),
               torch.empty((n,), dtype=torch.int32, device=dev), torch.empty((n,), dtype=torch.int32, device=dev),
               torch.empty((1,), dtype=torch.int32, device=dev))
    if workspace is None:
        workspace = torch.empty(pair_decode_workspace_bytes(lv, C, nms_pre), dtype=torch.uint8, device=dev)
    args = [L.ptr(t) for t in out] + [out[0].shape[0], L.ptr(workspace), ctypes.c_size_t(workspace.numel()), L.stream_ptr()]
    if geom is not None:
        L.check(lib.smb_pair_decode_topk_dev(nl, lv, C, ctypes.c_float(score_thr), int(nms_pre), L.ptr(geom), *args),
                'smb_pair_decode_topk_dev')
    else:
        L.check(lib.smb_pair_decode_topk(nl, lv, C, ctypes.c_float(score_thr), int(nms_pre), int(img_shape[0]),
                                         int(img_shape[1]), *args), 'smb_pair_decode_topk')
    return out


def ml_nms_workspace_bytes(cap):
    return int(L.lib().smb_ml_nms_workspace_bytes(int(cap)))


@L.device_guard
def ml_nms_topk(boxes, scores, labels, n_cand, iou_thr=0.6, max_per_img=100, out_cap=None, out=None, workspace=None):
    """SipMask-benchmark label-aware NMS + k-th-value cut (smb_ml_nms_topk) over the first *n_cand rows of boxes [cap,4],
    scores [cap], labels [cap] int32.  Returns (det [out_cap,5], labels int64, idx int64, count int32 [1], kept_total
    int32 [1]); out_cap defaults to cap.  out / workspace: those five buffers and a uint8 tensor of ml_nms_workspace_bytes
    to use; with both the call only launches."""
    _need_cuda(boxes, scores, labels, n_cand)
    boxes, scores = boxes.float().contiguous(), scores.float().contiguous()
    labels, n_cand = labels.to(torch.int32).contiguous(), n_cand.to(torch.int32).contiguous()
    cap = boxes.shape[0]
    out_cap = cap if out_cap is None else int(out_cap)
    dev = boxes.device
    if workspace is None:
        workspace = torch.empty(max(ml_nms_workspace_bytes(cap), 1), dtype=torch.uint8, device=dev)
    if out is None:
        out = (torch.empty((out_cap, 5), dtype=torch.float32, device=dev), torch.empty((out_cap,), dtype=torch.long, device=dev),
               torch.empty((out_cap,), dtype=torch.long, device=dev), torch.empty((1,), dtype=torch.int32, device=dev),
               torch.empty((1,), dtype=torch.int32, device=dev))
    L.check(L.lib().smb_ml_nms_topk(L.ptr(boxes), L.ptr(scores), L.ptr(labels), L.ptr(n_cand), cap, ctypes.c_float(iou_thr),
                                    int(max_per_img), out_cap, *[L.ptr(t) for t in out], L.ptr(workspace),
                                    ctypes.c_size_t(workspace.numel()), L.stream_ptr()), 'smb_ml_nms_topk')
    return out


# ------------------------------------------------------------------------------------ multi-class NMS
def _nms_record(out, max_num, dev):
    """The (det [max_num,5], labels int64, idx int64, count int32 [1]) buffers an NMS writes: `out`, or new ones."""
    if out is not None:
        return out
    return (torch.empty((max_num, 5), dtype=torch.float32, device=dev), torch.empty((max_num,), dtype=torch.long, device=dev),
            torch.empty((max_num,), dtype=torch.long, device=dev), torch.zeros(1, dtype=torch.int32, device=dev))


def _nms_result(rec, whole):
    """The record itself (whole), or its first count rows of (det, labels, idx) after reading the count on the host."""
    if whole:
        return rec
    k = int(rec[3].item())
    return rec[0][:k], rec[1][:k], rec[2][:k]


def multiclass_nms_workspace_bytes(n, num_classes, soft=False):
    lib = L.lib()
    f = lib.smb_multiclass_soft_nms_workspace_bytes if soft else lib.smb_multiclass_nms_workspace_bytes
    return int(f(int(n), int(num_classes)))


@L.device_guard
def multiclass_nms_idx(multi_bboxes, multi_scores, score_thr, nms_cfg, max_num=-1, score_factors=None,
                       has_bg_column=True, cmp_ge=False, return_count_tensor=False, out=None, workspace=None):
    """Same contract as mmdet.core.multiclass_nms_idx (bbox_nms.py:79-146): returns
    (dets [k,5], labels [k] int64 0-based, idxs [k] int64).  `multi_scores` carries the background
    column 0 like the reference unless has_bg_column=False.  nms_cfg['type'] selects 'nms' (the default) or 'soft_nms'
    (smb_multiclass_soft_nms: decayed scores in dets, each class in selection order); any other type raises.
    out / workspace: the (det, labels, idx, count) buffers and a uint8 tensor of multiclass_nms_workspace_bytes to use; with
    both and score_factors the call only launches and returns the whole record, as return_count_tensor does."""
    _need_cuda(multi_bboxes, multi_scores)
    kind = nms_type(nms_cfg) if isinstance(nms_cfg, dict) else 'nms'
    if kind not in ('nms', 'soft_nms'):
        raise ValueError("multiclass_nms_idx: nms type %r (supported: 'nms', 'soft_nms')" % (kind,))
    soft = kind == 'soft_nms'
    if soft:
        iou_thr, method, sigma, min_score = soft_nms_args(nms_cfg)
    else:
        iou_thr = nms_cfg.get('iou_thr', 0.5) if isinstance(nms_cfg, dict) else float(nms_cfg)
    scores = (multi_scores[:, 1:] if has_bg_column else multi_scores).float().contiguous()
    boxes = multi_bboxes.float().contiguous()
    n, C = scores.shape
    if soft and n > SOFT_NMS_MAX:
        raise L.SmbError('multiclass soft_nms: %d candidates, at most %d' % (n, SOFT_NMS_MAX))
    dev = boxes.device
    ctr = torch.ones(n, dtype=torch.float32, device=dev) if score_factors is None else score_factors.float().contiguous()
    if max_num is None or max_num <= 0:
        max_num = 1024
    if workspace is None:
        workspace = torch.empty(multiclass_nms_workspace_bytes(n, C, soft), dtype=torch.uint8, device=dev)
    rec = _nms_record(out, max_num, dev)
    head = (L.ptr(boxes), L.ptr(scores), L.ptr(ctr), n, C, ctypes.c_float(score_thr), ctypes.c_float(iou_thr), int(max_num))
    tail = [L.ptr(t) for t in rec] + [L.ptr(workspace), ctypes.c_size_t(workspace.numel()), L.stream_ptr()]
    if soft:
        L.check(L.lib().smb_multiclass_soft_nms(*head, method, ctypes.c_float(sigma), ctypes.c_float(min_score), *tail),
                'smb_multiclass_soft_nms')
    else:
        L.check(L.lib().smb_multiclass_nms(*head, int(cmp_ge), *tail), 'smb_multiclass_nms')
    return _nms_result(rec, return_count_tensor or out is not None)


def fast_nms_workspace_bytes(n, num_classes, top_k):
    return int(L.lib().smb_fast_nms_workspace_bytes(int(n), int(num_classes), int(top_k)))


@L.device_guard
def fast_nms(boxes, scores, ctr, iou_threshold=0.5, top_k=200, score_thr=0.1, max_num=100,
             return_count_tensor=False, out=None, workspace=None):
    """boxes [n,4], scores [n,C] sigmoid (NOT yet multiplied by ctr), ctr [n].
    Returns (dets [k,5], classes [k], idx [k]) like SipMaskHead.fast_nms (sipmask_head.py:868-910)
    with the coefficient gather left to the caller (`cofs[idx]`).  out / workspace as multiclass_nms_idx (the workspace of
    fast_nms_workspace_bytes)."""
    _need_cuda(boxes, scores, ctr)
    boxes = boxes.float().contiguous()
    scores = scores.float().contiguous()
    ctr = ctr.float().contiguous()
    n, C = scores.shape
    if workspace is None:
        workspace = torch.empty(fast_nms_workspace_bytes(n, C, top_k), dtype=torch.uint8, device=boxes.device)
    rec = _nms_record(out, max_num, boxes.device)
    L.check(L.lib().smb_fast_nms(L.ptr(boxes), L.ptr(scores), L.ptr(ctr), n, C, ctypes.c_float(score_thr),
                                 ctypes.c_float(iou_threshold), int(top_k), int(max_num), *[L.ptr(t) for t in rec],
                                 L.ptr(workspace), ctypes.c_size_t(workspace.numel()), L.stream_ptr()), 'smb_fast_nms')
    return _nms_result(rec, return_count_tensor or out is not None)


@L.device_guard
def gather_rows(src, idx, count, max_rows):
    """dst[i] = src[idx[i]] for i < count (device int32), zeros after; src [n,E] fp32 (row pitch = stride(0))."""
    _need_cuda(src, idx, count)
    assert src.dtype == torch.float32 and src.stride(1) == 1
    E = src.shape[1]
    dst = torch.empty((max_rows, E), dtype=torch.float32, device=src.device)
    L.check(L.lib().smb_gather_rows_f32(L.ptr(src), src.stride(0), L.ptr(idx), L.ptr(count), int(max_rows), E,
                                        L.ptr(dst), L.stream_ptr()), 'smb_gather_rows_f32')
    return dst


@L.device_guard
def gather_det_inputs(cof_src, cand_loc, idx, det, count, det_cofs, det_boxes, loc_out=None, level_hw=None, n_img=1, img=0):
    """smb_gather_det_inputs, the gather between NMS and mask assembly (mlvl_cofs[idxs_keep], det_bboxes[:, :4];
    sipmask_head.py:612,623) in one launch: det_cofs[i] = cof_src[cand_loc[idx[i]]] and det_boxes[i] = det[i, :4] for
    i < count (device int32 [1]), zeros after; loc_out (int64, optional) receives the kept locations, -1 after count.
    cof_src [rows, E] fp32 with row pitch stride(0) is one image's level-concatenated table (level_hw None), or a batched
    level-major buffer [level][n_img][h_l * w_l] of which image `img` is gathered (level_hw: h_l * w_l per level)."""
    _need_cuda(cof_src, cand_loc, idx, det, count, det_cofs, det_boxes, loc_out)
    max_rows, E = det_cofs.shape
    hw = None if level_hw is None else (ctypes.c_int * len(level_hw))(*level_hw)
    L.check(L.lib().smb_gather_det_inputs(L.ptr(cof_src), cof_src.stride(0), L.ptr(cand_loc), L.ptr(idx), L.ptr(det),
                                          L.ptr(count), max_rows, E, L.ptr(det_cofs), L.ptr(det_boxes), L.ptr(loc_out),
                                          0 if hw is None else len(hw), hw, int(n_img), int(img), L.stream_ptr()),
            'smb_gather_det_inputs')


@L.device_guard
def gather_track_feats(track_feats, det, count, scale_factor=1.0, feat_stride=8.0, geom=None, out=None):
    """SipMask-VIS `extract_box_feature_center_single`: track_feats [512,h,w] (reference layout) or [h,w,512] channel-last
    fp32, det [max,5], count device int -> [max,512] features at floor((x1+x2) * sf / 2 / 8) (zeros after count).
    geom: a device geometry row whose track scale is read when the kernel runs, in place of scale_factor.  out: the
    [max,512] buffer to write."""
    _need_cuda(track_feats, det, count)
    t = track_feats.float()
    if t.shape[0] == 512 and t.shape[-1] != 512:
        t = t.permute(1, 2, 0)
    t = t.contiguous()
    h, w, C = t.shape
    det = det.float().contiguous()
    count = count.to(torch.int32)
    if out is None:
        out = torch.empty((det.shape[0], C), dtype=torch.float32, device=det.device)
    if geom is not None:
        L.check(L.lib().smb_gather_track_feats_dev(L.ptr(t), h, w, C, L.ptr(det), L.ptr(count), det.shape[0], L.ptr(geom),
                                                   ctypes.c_float(feat_stride), L.ptr(out), L.stream_ptr()),
                'smb_gather_track_feats_dev')
        return out
    a = np.atleast_1d(np.asarray(scale_factor, dtype=np.float32))
    sx, sy = float(a[0]), float(a[1] if a.size >= 2 else a[0])
    L.check(L.lib().smb_gather_track_feats(L.ptr(t), h, w, C, L.ptr(det), L.ptr(count), det.shape[0], ctypes.c_float(sx),
                                           ctypes.c_float(sy), ctypes.c_float(feat_stride), L.ptr(out), L.stream_ptr()),
            'smb_gather_track_feats')
    return out


# -------------------------------------------------------------------------------------- mask assembly
@L.device_guard
def set_mask_tensor_dot(on):
    """fp16 prototypes: tensor-core (True) or scalar-fmaf (False) mask kernels for later calls (smb_mask_set_tensor_dot);
    on=None only queries.  Returns the previous setting."""
    return bool(L.lib().smb_mask_set_tensor_dot(-1 if on is None else int(bool(on))))


def mask_assemble(protos, cofs, boxes, box_scale, layout='chw', out_dtype=torch.float32, out=None, geom=None):
    """protos [32,H,W] ('chw') or [H,W,32] ('hwc'), fp32/fp16; cofs [N,128] fp32; boxes [N,4] fp32
    (image space); rois = boxes * box_scale (scalar or 4-vector), or * the roi scale of the device geometry row `geom`
    read when the kernel runs (box_scale is then unused).  Returns pos_masks [N,H,W]."""
    _need_cuda(protos, cofs, boxes)
    protos = protos.contiguous()
    if layout == 'chw':
        _, H, W = protos.shape
    else:
        H, W, _ = protos.shape
    N = cofs.shape[0]
    cofs = cofs.float().contiguous()
    boxes = boxes.float().contiguous()
    if out is None:
        out = torch.empty((N, H, W), dtype=out_dtype, device=protos.device)
    hwc = 1 if layout == 'hwc' else 0
    if geom is not None:
        L.check(L.lib().smb_mask_assemble_dev(L.ptr(protos), _dt(protos), hwc, L.ptr(cofs), L.ptr(boxes), L.ptr(geom),
                                              L.ptr(out), _dt(out), H, W, N, L.stream_ptr()), 'smb_mask_assemble_dev')
        return out
    a = np.atleast_1d(np.asarray(box_scale, dtype=np.float32))
    bs = L.f4(a if a.size == 4 else [a[0]] * 4)
    L.check(L.lib().smb_mask_assemble(L.ptr(protos), _dt(protos), hwc, L.ptr(cofs), L.ptr(boxes), bs, L.ptr(out), _dt(out),
                                      H, W, N, L.stream_ptr()), 'smb_mask_assemble')
    return out


def resize_spec(H, W, up, legacy_interp=False):
    """F.interpolate(scale_factor=up, mode='bilinear', align_corners=False) on an [H, W] map -> (full_h, full_w, ry, rx):
    interpolated size floor(H * up_h), floor(W * up_w) (computed in double like torch) and the source step per output pixel,
    float32(1 / up) as PyTorch >= 1.6 uses it, or 0 (= in / out, recompute_scale_factor=True, PyTorch <= 1.5) when
    legacy_interp.  `up` is a float or an (h, w) pair: 2 / scale_factor (sipmask_head.py:629-633)."""
    import math
    uh, uw = (float(up[0]), float(up[1])) if isinstance(up, (tuple, list)) else (float(up), float(up))
    full_h, full_w = int(math.floor(float(H) * uh)), int(math.floor(float(W) * uw))
    if legacy_interp:
        return full_h, full_w, 0.0, 0.0
    return full_h, full_w, float(np.float32(1.0 / uh)), float(np.float32(1.0 / uw))


@L.device_guard
def mask_resize_threshold(pos, up, out_hw, thr=0.4, out=None, legacy_interp=False):
    """pos [N,H,W] -> uint8 [N,out_h,out_w]: bilinear resize by `up` (align_corners=False), > thr, top-left paste
    (sipmask_head.py:629-633,648-654)."""
    _need_cuda(pos)
    pos = pos.contiguous()
    N, H, W = pos.shape
    fh, fw, ry, rx = resize_spec(H, W, up, legacy_interp)
    if out is None:
        out = torch.empty((N, int(out_hw[0]), int(out_hw[1])), dtype=torch.uint8, device=pos.device)
    L.check(L.lib().smb_mask_resize_threshold(L.ptr(pos), _dt(pos), L.ptr(out), N, H, W, fh, fw, ctypes.c_float(ry),
                                              ctypes.c_float(rx), int(out_hw[0]), int(out_hw[1]), ctypes.c_float(thr),
                                              L.stream_ptr()), 'smb_mask_resize_threshold')
    return out


@L.device_guard
def mask_resize_threshold_pack(pos, up, out_hw, thr=0.4, out=None, legacy_interp=False):
    """Bit-packed masks: int32 [N,out_h,ceil(out_w/32)], pixel x = bit (x & 31) of word (x >> 5)."""
    _need_cuda(pos)
    pos = pos.contiguous()
    N, H, W = pos.shape
    fh, fw, ry, rx = resize_spec(H, W, up, legacy_interp)
    words = (int(out_hw[1]) + 31) // 32
    if out is None:
        out = torch.empty((N, int(out_hw[0]), words), dtype=torch.int32, device=pos.device)
    L.check(L.lib().smb_mask_resize_threshold_pack(L.ptr(pos), _dt(pos), L.ptr(out), N, H, W, fh, fw, ctypes.c_float(ry),
                                                   ctypes.c_float(rx), int(out_hw[0]), int(out_hw[1]), ctypes.c_float(thr),
                                                   L.stream_ptr()), 'smb_mask_resize_threshold_pack')
    return out


def mask_upsample2_threshold(pos, out_hw, thr=0.4, out=None):
    """scale_factor == 1 shorthand: x2 bilinear (align_corners=False), > thr, top-left paste."""
    return mask_resize_threshold(pos, 2.0, out_hw, thr, out)


def mask_upsample2_threshold_pack(pos, out_hw, thr=0.4, out=None):
    return mask_resize_threshold_pack(pos, 2.0, out_hw, thr, out)


@L.device_guard
def mask_assemble_pack(protos, cofs, boxes, box_scale, out_hw, thr=0.4, layout='chw', out=None, up=2.0, legacy_interp=False):
    """Fused mask path: prototypes -> bit-packed thresholded masks int32 [N,out_h,ceil(out_w/32)] (no pos_masks tensor);
    `up` = 2 / scale_factor (float or (h, w)) is the bilinear resize factor of sipmask_head.py:629-633."""
    _need_cuda(protos, cofs, boxes)
    protos = protos.contiguous()
    if layout == 'chw':
        _, H, W = protos.shape
    else:
        H, W, _ = protos.shape
    N = cofs.shape[0]
    cofs = cofs.float().contiguous()
    boxes = boxes.float().contiguous()
    a = np.atleast_1d(np.asarray(box_scale, dtype=np.float32))
    bs = L.f4(a if a.size == 4 else [a[0]] * 4)
    fh, fw, ry, rx = resize_spec(H, W, up, legacy_interp)
    words = (int(out_hw[1]) + 31) // 32
    if out is None:
        out = torch.empty((N, int(out_hw[0]), words), dtype=torch.int32, device=protos.device)
    L.check(L.lib().smb_mask_assemble_pack(L.ptr(protos), _dt(protos), 1 if layout == 'hwc' else 0, L.ptr(cofs), L.ptr(boxes),
                                           bs, L.ptr(out), H, W, N, fh, fw, ctypes.c_float(ry), ctypes.c_float(rx),
                                           int(out_hw[0]), int(out_hw[1]), ctypes.c_float(thr), L.stream_ptr()),
            'smb_mask_assemble_pack')
    return out


@L.device_guard
def mask_assemble_pack_dev(protos, cofs, boxes, geom, tile_r, cap_hw, thr=0.4, layout='hwc', out=None):
    """The engine's fused mask call (smb_mask_assemble_pack_dev): roi scale, resize and canvas read from the device row
    `geom` (int32 words of an smb_img_geom_t, see geom_row) when the kernel runs; the tile is sized for the source steps
    tile_r = (max_ry, max_rx), which must be at least the row's.  Bit planes int32 [N, cap_h, ceil(cap_w / 32)]."""
    _need_cuda(protos, cofs, boxes, geom)
    protos = protos.contiguous()
    if layout == 'chw':
        _, H, W = protos.shape
    else:
        H, W, _ = protos.shape
    N = cofs.shape[0]
    cofs = cofs.float().contiguous()
    boxes = boxes.float().contiguous()
    cap_h, cap_w = int(cap_hw[0]), int(cap_hw[1])
    if out is None:
        out = torch.empty((N, cap_h, (cap_w + 31) // 32), dtype=torch.int32, device=protos.device)
    L.check(L.lib().smb_mask_assemble_pack_dev(L.ptr(protos), _dt(protos), 1 if layout == 'hwc' else 0, L.ptr(cofs),
                                               L.ptr(boxes), L.ptr(geom), ctypes.c_float(tile_r[0]), ctypes.c_float(tile_r[1]),
                                               L.ptr(out), H, W, N, cap_h, cap_w, ctypes.c_float(thr), L.stream_ptr()),
            'smb_mask_assemble_pack_dev')
    return out


def geom_row(g, device):
    """An smb_img_geom_t (postproc.image_geometry) as the device row of int32 words the *_dev entry points read."""
    return torch.from_numpy(np.frombuffer(bytes(g), dtype=np.int32).copy()).to(device)


def unpack_mask_bits(bits, out_w):
    """int32 [N,h,words] -> uint8 [N,h,out_w] (host or device tensor); used by tests and result conversion."""
    b = bits.view(torch.uint8) if bits.dtype == torch.int32 else bits
    b = b.reshape(bits.shape[0], bits.shape[1], -1)                     # little-endian bytes
    sh = torch.arange(8, device=b.device, dtype=torch.uint8)
    px = ((b.unsqueeze(-1) >> sh) & 1).reshape(b.shape[0], b.shape[1], -1)
    return px[:, :, :out_w].contiguous()


@L.device_guard
def mask_rle_counts(mask_bits, H, W, n_valid=None, cap=8192):
    """Device-side COCO RLE (smb_mask_rle_counts): bit-packed masks int32 [N,mask_h,words] cropped to H x W ->
    (counts uint32-as-int32 [N,cap] column-major run lengths, n_counts int32 [N]).  n_valid: optional device int tensor."""
    _need_cuda(mask_bits)
    assert mask_bits.dtype == torch.int32 and mask_bits.is_contiguous() and mask_bits.dim() == 3
    N, mask_h, words = mask_bits.shape
    counts = torch.empty((N, cap), dtype=torch.int32, device=mask_bits.device)
    n_counts = torch.empty((N,), dtype=torch.int32, device=mask_bits.device)
    if n_valid is not None:
        n_valid = n_valid.to(torch.int32).contiguous()
    L.check(L.lib().smb_mask_rle_counts(L.ptr(mask_bits), N, mask_h, words, int(H), int(W), L.ptr(n_valid), L.ptr(counts),
                                        int(cap), L.ptr(n_counts), L.stream_ptr()), 'smb_mask_rle_counts')
    return counts, n_counts


def rle_to_string(counts):
    """Host helper of the ABI (smb_rle_to_string): run lengths (numpy / CPU tensor, any int type) -> pycocotools bytes."""
    c = np.ascontiguousarray(np.asarray(counts).astype(np.uint32))
    cap = 8 * c.size + 8
    buf = ctypes.create_string_buffer(cap)
    n = L.lib().smb_rle_to_string(c.ctypes.data_as(ctypes.c_void_p), int(c.size), buf, cap)
    if n < 0:
        raise L.SmbError('smb_rle_to_string: buffer too small')
    return buf.raw[:n]


@L.device_guard
def masks_to_rle(mask_bits, H, W, k, cap=8192):
    """k valid bit-packed masks -> list of k COCO RLE dicts {'size': [H, W], 'counts': bytes}: one kernel, one small D2H
    (k * runs * 4 bytes instead of k * H * W mask bytes), string packing in C on the host."""
    if k == 0:
        return []
    counts, n = mask_rle_counts(mask_bits[:k].contiguous(), H, W, cap=cap)
    n_host = n.cpu().numpy()
    if (n_host < 0).any():                                    # pathological (noise-like) mask: retry with the exact capacity
        need = int((-n_host).max()) + 1
        counts, n = mask_rle_counts(mask_bits[:k].contiguous(), H, W, cap=need)
        n_host = n.cpu().numpy()
    width = int(n_host.max())
    c_host = counts[:, :width].cpu().numpy()
    return [{'size': [int(H), int(W)], 'counts': rle_to_string(c_host[j, :n_host[j]])} for j in range(k)]


def rle_encode_workspace_bytes(N, max_num, run_cap):
    return int(L.lib().smb_rle_encode_workspace_bytes(int(N), int(max_num), int(run_cap)))


@L.device_guard
def rle_encode_dev(mask_bits, count, geom, dst_word, img_bytes, run_cap, workspace):
    """smb_rle_encode_dev: the pycocotools strings of every detection of a batch of records, packed per image into the
    arena whose device address the int64 device word dst_word holds (see rle.read_region for the layout).
    mask_bits int32 [N, max_num, cap_h, words], count int32 [N], geom the engine's geometry rows [N, words of a row]."""
    _need_cuda(mask_bits, count, geom, dst_word, workspace)
    assert mask_bits.dtype == torch.int32 and mask_bits.is_contiguous() and mask_bits.dim() == 4
    assert count.dtype == torch.int32 and dst_word.dtype == torch.int64 and workspace.dtype == torch.uint8
    N, mx, cap_h, words = mask_bits.shape
    L.check(L.lib().smb_rle_encode_dev(L.ptr(mask_bits), N, mx, cap_h, words, L.ptr(count), L.ptr(geom), int(run_cap),
                                       L.ptr(dst_word), int(img_bytes), L.ptr(workspace), ctypes.c_size_t(workspace.numel()),
                                       L.stream_ptr()), 'smb_rle_encode_dev')


def track_assoc_workspace_bytes(lanes, max_num, capacity):
    return int(L.lib().smb_track_assoc_workspace_bytes(int(lanes), int(max_num), int(capacity)))


@L.device_guard
def track_assoc(frames, det, labels, count, track_feats, state, match_coeff=(1.0, 2.0, 10.0), ids=None, workspace=None):
    """smb_track_assoc_dev: the tracker association of a batch of frame records on the device, in one launch.
    frames int32 [N, 2] device rows (lane, is_first); det [N, max, 5] f32, labels [N, max] int64, count int32 [N],
    track_feats [N, max, 512] f32; state = dict(boxes [lanes, cap, 5] f32, labels [lanes, cap] int64,
    feats [lanes, cap, 512] f32, n_obj int32 [lanes], status int32 [lanes]), updated in place.  Returns ids int32 [N, max]."""
    _need_cuda(frames, det, labels, count, track_feats)
    N, mx = det.shape[0], det.shape[1]
    lanes, cap = state['boxes'].shape[0], state['boxes'].shape[1]
    assert frames.dtype == torch.int32 and tuple(frames.shape) == (N, 2) and frames.is_contiguous()
    assert det.dtype == torch.float32 and tuple(det.shape) == (N, mx, 5) and det.is_contiguous()
    assert labels.dtype == torch.int64 and tuple(labels.shape) == (N, mx) and labels.is_contiguous()
    assert count.dtype == torch.int32 and count.numel() == N and count.is_contiguous()
    assert track_feats.dtype == torch.float32 and tuple(track_feats.shape) == (N, mx, 512) and track_feats.is_contiguous()
    want = dict(boxes=((lanes, cap, 5), torch.float32), labels=((lanes, cap), torch.int64),
                feats=((lanes, cap, 512), torch.float32), n_obj=((lanes,), torch.int32), status=((lanes,), torch.int32))
    for name, (shape, dtype) in want.items():
        t = state[name]
        if t.device != det.device or t.dtype != dtype or tuple(t.shape) != shape or not t.is_contiguous():
            raise ValueError('track_assoc: state[%r] must be a contiguous %s %s tensor on %s, got %s %s on %s'
                             % (name, dtype, list(shape), det.device, t.dtype, list(t.shape), t.device))
    for name, t in (('frames', frames), ('labels', labels), ('count', count), ('track_feats', track_feats)):
        if t.device != det.device:
            raise ValueError('track_assoc: %s is on %s, det on %s' % (name, t.device, det.device))
    if ids is None:
        ids = torch.empty((N, mx), dtype=torch.int32, device=det.device)
    if ids.device != det.device or ids.dtype != torch.int32 or tuple(ids.shape) != (N, mx) or not ids.is_contiguous():
        raise ValueError('track_assoc: ids must be a contiguous int32 [%d, %d] tensor on %s' % (N, mx, det.device))
    need = track_assoc_workspace_bytes(lanes, mx, cap)
    if workspace is None:
        workspace = torch.empty(need, dtype=torch.uint8, device=det.device)
    if (workspace.device != det.device or workspace.dtype != torch.uint8 or not workspace.is_contiguous()
            or workspace.numel() < need):
        raise ValueError('track_assoc: workspace must be a contiguous uint8 tensor of >= %d bytes on %s' % (need, det.device))
    coef = (ctypes.c_float * 3)(*[float(np.float32(c)) for c in match_coeff])
    L.check(L.lib().smb_track_assoc_dev(L.ptr(frames), N, L.ptr(det), L.ptr(labels), L.ptr(count), L.ptr(track_feats), mx,
                                        L.ptr(state['boxes']), L.ptr(state['labels']), L.ptr(state['feats']),
                                        L.ptr(state['n_obj']), L.ptr(state['status']), lanes, cap, coef, L.ptr(ids),
                                        L.ptr(workspace), ctypes.c_size_t(workspace.numel()), L.stream_ptr()),
            'smb_track_assoc_dev')
    return ids


def segm_raster_workspace_bytes(n_items, max_hw, max_w):
    return int(L.lib().smb_segm_raster_workspace_bytes(int(n_items), ctypes.c_int64(int(max_hw)), int(max_w)))


@L.device_guard
def render(rows, n, max_hw, mask_bits, det, count, palette, rule, score_thr, boxes=True, labels=None, obj_ids=None):
    """smb_render_dev on the current stream: n images (rows: device smb_render_img_t rows, uint8) drawn from a record
    mask_bits [n, max, cap_h, words] int32, det [n, max, 5] fp32, count [n] int32 and labels [n, max] int64
    (rule RENDER_IMAGES) or obj_ids [n, max] int32 (RENDER_VIDEO); palette [rows, 3] uint8 on the device.  score_thr is
    compared in fp32.  The caller validates the rows against max_hw and the record (render.render_images does)."""
    _need_cuda(rows, mask_bits, det, count, palette, labels, obj_ids)
    mx = det.shape[1]
    assert mask_bits.dtype == torch.int32 and mask_bits.dim() == 4 and mask_bits.is_contiguous()
    assert tuple(mask_bits.shape[:2]) == (n, mx) and tuple(det.shape) == (n, mx, 5) and det.dtype == torch.float32
    assert det.is_contiguous() and count.dtype == torch.int32 and count.numel() >= n and count.is_contiguous()
    assert palette.dtype == torch.uint8 and palette.dim() == 2 and palette.shape[1] == 3 and palette.is_contiguous()
    assert rows.dtype == torch.uint8 and rows.numel() >= n * ctypes.sizeof(L.RenderImg)
    for t, dt in ((labels, torch.int64), (obj_ids, torch.int32)):
        if t is not None:
            assert t.dtype == dt and tuple(t.shape) == (n, mx) and t.is_contiguous()
    cap_h, words = mask_bits.shape[2:]
    L.check(L.lib().smb_render_dev(L.ptr(rows), int(n), int(max_hw[0]), int(max_hw[1]), L.ptr(mask_bits), int(mx),
                                   int(cap_h), int(words), L.ptr(det), L.ptr(labels), L.ptr(count), L.ptr(obj_ids),
                                   L.ptr(palette), int(palette.shape[0]), int(rule),
                                   ctypes.c_float(float(np.float32(score_thr))), int(bool(boxes)), L.stream_ptr()),
            'smb_render_dev')


@L.device_guard
def segm_raster(items, n_items, xy, n_xy, counts, n_counts, max_hw, max_w, planes, n_planes, plane_stride, pitch, status,
                area=None, area_stride=1, ext=None, ext_stride=4, workspace=None):
    """smb_segm_raster_dev: zero planes [n_planes, plane_stride words] (int32, rows of `pitch` words) and rasterize
    n_items segmentations into them on the current stream.  items: smb_segm_item_t rows, xy: the float64 vertex pool
    (n_xy vertices), counts: the uint32 run-length pool, all device tensors (segm_raster.SegmPack builds them); max_hw /
    max_w: the largest canvas of any item.  area / ext: device int32 tensors whose element p * stride (.. + 3) receives
    plane p's pixel count / extents.  status: int32 [1], SMB_SEGM_RANGE is OR-ed into it."""
    _need_cuda(items, planes, status)
    assert planes.dtype == torch.int32 and planes.is_contiguous() and status.dtype == torch.int32
    if planes.numel() < int(n_planes) * int(plane_stride):
        raise ValueError('segm_raster: %d planes of %d words in a tensor of %d' % (n_planes, plane_stride, planes.numel()))
    for t in (area, ext):                          # views into the caller's rows: only the caller knows their extent
        if t is not None and (t.dtype != torch.int32 or t.device != planes.device):
            raise ValueError('segm_raster: area / ext must be int32 tensors on %s' % planes.device)
    need = segm_raster_workspace_bytes(n_items, max_hw, max_w)
    if workspace is None:
        workspace = torch.empty(max(need, 16), dtype=torch.uint8, device=planes.device)
    if workspace.device != planes.device or workspace.dtype != torch.uint8 or workspace.numel() < need:
        raise ValueError('segm_raster: workspace must be a uint8 tensor of >= %d bytes on %s' % (need, planes.device))
    L.check(L.lib().smb_segm_raster_dev(L.ptr(items), int(n_items), L.ptr(xy), ctypes.c_int64(int(n_xy)), L.ptr(counts),
                                        ctypes.c_int64(int(n_counts)), ctypes.c_int64(int(max_hw)), int(max_w),
                                        L.ptr(planes), int(n_planes), ctypes.c_int64(int(plane_stride)), int(pitch),
                                        L.ptr(area), ctypes.c_int64(int(area_stride)), L.ptr(ext),
                                        ctypes.c_int64(int(ext_stride)), L.ptr(status), L.ptr(workspace),
                                        ctypes.c_size_t(workspace.numel()), L.stream_ptr()), 'smb_segm_raster_dev')


def host_device_pointer(pinned):
    """The device address of a page-locked host tensor (cudaHostGetDevicePointer), for the current device."""
    if not pinned.is_pinned():
        raise ValueError('host_device_pointer: the tensor is not in page-locked memory')
    out = ctypes.c_void_p(0)
    L.check(L.lib().smb_host_device_pointer(ctypes.c_void_p(pinned.data_ptr()), ctypes.byref(out)), 'smb_host_device_pointer')
    return int(out.value)


@L.device_guard
def conv3x3s2_relu(x, weight, bias):
    """One `convs_scoring` ConvModule (sipmask_head.py:200-214): NCHW fp32 conv3x3 stride 2 pad 0 + bias + ReLU."""
    _need_cuda(x, weight, bias)
    x, weight, bias = x.float().contiguous(), weight.float().contiguous(), bias.float().contiguous()
    N, Cin, H, W = x.shape
    Cout = weight.shape[0]
    assert weight.shape == (Cout, Cin, 3, 3)
    out = torch.empty((N, Cout, (H - 3) // 2 + 1, (W - 3) // 2 + 1), dtype=torch.float32, device=x.device)
    L.check(L.lib().smb_conv3x3s2_relu_f32(L.ptr(x), L.ptr(weight), L.ptr(bias), L.ptr(out), N, Cin, H, W, Cout, L.stream_ptr()),
            'smb_conv3x3s2_relu_f32')
    return out


@L.device_guard
def mask_rescore(pos_masks, conv_weights, conv_biases, w1x1, b1x1, labels, det, n_valid=None):
    """SipMask++ rescoring (sipmask_head.py:635-643): pos_masks [N,Hm,Wm] fp32 (cropped stride-2 masks) -> mask_scores [N]."""
    x = pos_masks.float().unsqueeze(1)
    for w, b in zip(conv_weights, conv_biases):
        x = conv3x3s2_relu(x, w, b)
    N, C, h, w_ = x.shape
    w1 = w1x1.float().reshape(w1x1.shape[0], -1).contiguous()
    scores = torch.empty((N,), dtype=torch.float32, device=x.device)
    if n_valid is not None:
        n_valid = n_valid.to(torch.int32).contiguous()
    L.check(L.lib().smb_mask_rescore(L.ptr(x), N, C, h, w_, L.ptr(w1), L.ptr(b1x1.float().contiguous()), int(w1.shape[0]),
                                     L.ptr(labels.long().contiguous()), L.ptr(det.float().contiguous()), L.ptr(n_valid),
                                     L.ptr(scores), L.stream_ptr()), 'smb_mask_rescore')
    return scores


RESCORE_CHANNELS = (1, 16, 16, 16, 32, 64, 128)       # convs_scoring (sipmask_head.py:200-215)


def rescore_flops_per_row(H, W):
    """Algorithmic FLOPs of one detection through the six stride-2 convolutions and its own mask_scoring row (36.5 M at
    272 x 272)."""
    fl, h, w = 0, H, W
    for cin, cout in zip(RESCORE_CHANNELS[:-1], RESCORE_CHANNELS[1:]):
        h, w = (h - 3) // 2 + 1, (w - 3) // 2 + 1
        fl += 2 * h * w * cout * 9 * cin
    return fl + 2 * h * w * RESCORE_CHANNELS[-1]


class RescoreWeights(object):
    """convs_scoring (6 x [Cout, Cin, 3, 3] + bias) and mask_scoring ([C, 128(, 1, 1)] + bias) packed for
    smb_mask_rescore_f16: fp16 [Cout, 9 * Cin] via conv.pack_weight, fp32 biases; `struct` points at the device tensors."""

    def __init__(self, conv_weights, conv_biases, w1x1, b1x1, device):
        from . import conv as C
        if len(conv_weights) != 6 or len(conv_biases) != 6:
            raise ValueError('rescoring needs six convs_scoring layers, got %d' % len(conv_weights))
        for i, w in enumerate(conv_weights):
            want = (RESCORE_CHANNELS[i + 1], RESCORE_CHANNELS[i], 3, 3)
            if tuple(w.shape) != want:
                raise ValueError('convs_scoring.%d: weight shape %s, expected %s' % (i, tuple(w.shape), want))
        if w1x1.shape[1] != RESCORE_CHANNELS[-1]:
            raise ValueError('mask_scoring: %d input channels, expected 128' % w1x1.shape[1])
        self.conv_w = [C.pack_weight(w, device=device)[0] for w in conv_weights]
        self.conv_b = [b.detach().float().contiguous().to(device) for b in conv_biases]
        self.num_classes = int(w1x1.shape[0])
        self.score_w = C.pack_weight(w1x1.reshape(self.num_classes, -1, 1, 1), device=device)[0]
        self.score_b = b1x1.detach().float().contiguous().to(device)
        self.struct = L.RescoreWeights()
        for i in range(6):
            self.struct.conv_w[i] = self.conv_w[i].data_ptr()
            self.struct.conv_b[i] = self.conv_b[i].data_ptr()
        self.struct.score_w, self.struct.score_b = self.score_w.data_ptr(), self.score_b.data_ptr()
        self.struct.num_classes = self.num_classes


def mask_rescore_f16_workspace_bytes(rows, H, W):
    return int(L.lib().smb_mask_rescore_f16_workspace_bytes(int(rows), int(H), int(W)))


def mask_rescore_f16_layers(workspace, rows, H, W):
    """The activations of layers 2-5 that smb_mask_rescore_f16 leaves in its uint8 `workspace` for `rows` masks of H x W:
    fp16 views [rows, h, w, C] with C = 16, 16, 32, 64 (h = (h_prev - 3) // 2 + 1 from the mask size), each starting on a
    256-byte boundary.  They span exactly mask_rescore_f16_workspace_bytes(rows, H, W) bytes."""
    hs, ws = [int(H)], [int(W)]
    for _ in range(5):
        hs.append((hs[-1] - 3) // 2 + 1)
        ws.append((ws[-1] - 3) // 2 + 1)
    views, o = [], 0
    for l in range(2, 6):
        n = int(rows) * hs[l] * ws[l] * RESCORE_CHANNELS[l]
        views.append(workspace[o:o + 2 * n].view(torch.float16).view(int(rows), hs[l], ws[l], RESCORE_CHANNELS[l]))
        o = (o + 2 * n + 255) // 256 * 256
    if o != mask_rescore_f16_workspace_bytes(rows, H, W) or workspace.numel() < o:
        raise L.SmbError('mask_rescore_f16_layers: layout of %d bytes does not match the %d-byte workspace of %d x %d x %d '
                         '(buffer %d bytes)' % (o, mask_rescore_f16_workspace_bytes(rows, H, W), rows, H, W, workspace.numel()))
    return views


@L.device_guard
def mask_rescore_f16(pos_masks, count, weights, labels, det, workspace=None, out=None):
    """SipMask++ rescoring on tensor cores (smb_mask_rescore_f16): pos_masks [n_img, max_rows, H, W] fp16 cropped stride-2
    masks, count device int32 [n_img], weights a RescoreWeights, labels int64 [n_img, max_rows], det [n_img, max_rows, 5]
    -> mask_scores fp32 [n_img, max_rows] (exactly 0 after count)."""
    _need_cuda(pos_masks, count, labels, det)
    if pos_masks.dtype != torch.float16 or pos_masks.dim() != 4 or not pos_masks.is_contiguous():
        raise L.SmbError('mask_rescore_f16: pos_masks must be a contiguous fp16 [n_img, max_rows, H, W] tensor')
    n_img, max_rows, H, W = pos_masks.shape
    if tuple(labels.shape) != (n_img, max_rows) or tuple(det.shape) != (n_img, max_rows, 5) or count.numel() != n_img:
        raise L.SmbError('mask_rescore_f16: labels / det / count do not match pos_masks %s' % (tuple(pos_masks.shape),))
    count = count.to(torch.int32).contiguous()
    labels, det = labels.long().contiguous(), det.float().contiguous()
    if workspace is None:
        workspace = torch.empty(max(mask_rescore_f16_workspace_bytes(n_img * max_rows, H, W), 1), dtype=torch.uint8,
                                device=pos_masks.device)
    if out is None:
        out = torch.empty((n_img, max_rows), dtype=torch.float32, device=pos_masks.device)
    L.check(L.lib().smb_mask_rescore_f16(L.ptr(pos_masks), n_img, max_rows, H, W, L.ptr(count), ctypes.byref(weights.struct),
                                         L.ptr(labels), L.ptr(det), L.ptr(out), L.ptr(workspace),
                                         ctypes.c_size_t(workspace.numel()), L.stream_ptr()), 'smb_mask_rescore_f16')
    return out


# ----------------------------------------------------------------------------------- DeformConv (operator API)
class DeformConv(nn.Module):
    """Drop-in for `mmdet.ops.DeformConv` (MM/mmdet/ops/dcn/deform_conv.py:192-255): same constructor keywords, same
    `weight` parameter ([out, in, kh, kw], uniform(-1/sqrt(fan_in), +)), `forward(x[N,C,H,W], offset[N,dg*2*k*k,H,W])`.

    Replaces deform_conv_cuda.deform_conv_forward_cuda (ops/dcn/src/deform_conv_cuda.cpp:152-260: im2col kernel + addmm)
    by `smb_deform_im2col` (channel-last bilinear gather, fp16 columns) + the wgmma GEMM (fp32 accumulate).  The hot
    path only uses 3x3 / stride 1 / padding 1 / dilation 1 / groups 1 (FeatureAlign `conv_adaption`, sipmask_head.py:35-41,
    and DeformConvPack in the ++ backbone, resnet.py:146-168); other geometries raise.  NCHW in, NCHW out, x.dtype kept."""

    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1,
                 deformable_groups=1, bias=False):
        super().__init__()
        assert not bias
        assert in_channels % groups == 0, 'in_channels {} cannot be divisible by groups {}'.format(in_channels, groups)
        assert out_channels % groups == 0, 'out_channels {} cannot be divisible by groups {}'.format(out_channels, groups)
        pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)       # noqa: E731
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding, self.dilation = pair(kernel_size), pair(stride), pair(padding), pair(dilation)
        self.groups, self.deformable_groups = groups, deformable_groups
        self.transposed, self.output_padding = False, (0,)
        self.weight = nn.Parameter(torch.Tensor(out_channels, in_channels // groups, *self.kernel_size))
        self.reset_parameters()
        self._packed = None

    def reset_parameters(self):
        n = self.in_channels
        for k in self.kernel_size:
            n *= k
        stdv = 1. / np.sqrt(n)
        self.weight.data.uniform_(-stdv, stdv)

    def _check_geometry(self):
        if not (self.kernel_size == (3, 3) and self.stride == (1, 1) and self.padding == (1, 1) and self.dilation == (1, 1)
                and self.groups == 1):
            raise NotImplementedError('sipmask_b200.ops.DeformConv: only 3x3 / stride 1 / padding 1 / dilation 1 / groups 1 '
                                      '(the geometries on the SipMask inference path)')
        c, dg = self.in_channels, self.deformable_groups
        if c % 64 or self.out_channels % 16 or c % dg or (c // dg) % 8:
            raise NotImplementedError('sipmask_b200.ops.DeformConv: in_channels %% 64, out_channels %% 16 and '
                                      '(in_channels / deformable_groups) %% 8 must be 0 (got %d, %d, dg=%d)'
                                      % (c, self.out_channels, dg))

    @torch.no_grad()
    def forward(self, x, offset):
        from . import conv as C
        _need_cuda(x, offset, self.weight)
        self._check_geometry()
        kh, kw = self.kernel_size
        input_pad = x.size(2) < kh or x.size(3) < kw                      # deform_conv.py:242-254
        if input_pad:
            pad_h, pad_w = max(kh - x.size(2), 0), max(kw - x.size(3), 0)
            x = torch.nn.functional.pad(x, (0, pad_w, 0, pad_h), 'constant', 0).contiguous()
            offset = torch.nn.functional.pad(offset, (0, pad_w, 0, pad_h), 'constant', 0).contiguous()
        N, Cin, H, W = x.shape
        if offset.shape != (N, self.deformable_groups * 2 * kh * kw, H, W):
            raise L.SmbError('DeformConv: offset shape %s does not match input %s (deform_conv_cuda.cpp:62-150)'
                             % (tuple(offset.shape), tuple(x.shape)))
        key = (self.weight._version, self.weight.data_ptr(), x.device)
        if self._packed is None or self._packed[0] != key:
            self._packed = (key, C.pack_weight(self.weight, device=x.device)[0])
        y = _deform_conv_forward(x, offset, self._packed[1], self.deformable_groups)
        if input_pad:
            y = y[:, :, :y.size(2) - pad_h, :y.size(3) - pad_w]
        return y.contiguous()


def _channels_last(x, offset):
    """x [N,C,H,W] -> fp16 [N,H,W,C]; offset [N,dg*18,H,W] -> fp32 [N,H,W,dg*18] (the layouts smb_deform_im2col reads)."""
    return (x.permute(0, 2, 3, 1).contiguous().to(torch.float16), offset.permute(0, 2, 3, 1).contiguous().float())


def _deform_conv_forward(x, offset, wk, dg):
    """The DeformConv forward on an input at least as large as the kernel: `smb_deform_im2col` + the wgmma GEMM with the
    packed weight wk [Cout, 9*C] fp16 -> y [N, Cout, H, W] in x.dtype (a permuted view)."""
    from . import conv as C
    N, _, H, W = x.shape
    with torch.cuda.device(x.device):
        xh, off = _channels_last(x, offset)
        col = C.deform_im2col(xh, off, dg)
        out = torch.empty((N, H, W, wk.shape[0]), dtype=torch.float16, device=x.device)
        C.ConvPlan(col, wk, out, 1, 1).run()
        return out.permute(0, 3, 1, 2).to(x.dtype)


# ------------------------------------------------------------------------------ DeformConv with autograd (fine-tuning)
def _check_deform_args(x, offset, weight, stride, padding, dilation, groups, dg):
    """What the sm_90a forward and backward support; raises before anything is launched."""
    if x.dtype not in (torch.float32, torch.float16) or offset.dtype not in (torch.float32, torch.float16) \
            or weight.dtype != torch.float32:
        raise L.SmbError('deform_conv: input / offset must be fp32 or fp16 and weight fp32 (got %s, %s, %s)'
                         % (x.dtype, offset.dtype, weight.dtype))
    pair = lambda v: tuple(v) if isinstance(v, (tuple, list)) else (v, v)       # noqa: E731
    cout, cin = weight.shape[0], weight.shape[1]
    if not (tuple(weight.shape[2:]) == (3, 3) and pair(stride) == (1, 1) and pair(padding) == (1, 1)
            and pair(dilation) == (1, 1) and groups == 1):
        raise NotImplementedError('sipmask_b200.ops.deform_conv: only 3x3 / stride 1 / padding 1 / dilation 1 / groups 1')
    if x.size(1) != cin or cin % 64 or cout % 64 or cin % dg or (cin // dg) % 8 or cin > 1024:
        raise NotImplementedError('sipmask_b200.ops.deform_conv: in_channels %% 64 (<= 1024), out_channels %% 64 and '
                                  '(in_channels / deformable_groups) %% 8 must be 0 (got %d, %d, dg=%d)' % (cin, cout, dg))
    N, _, H, W = x.shape
    if tuple(offset.shape) != (N, dg * 18, H, W):
        raise L.SmbError('deform_conv: offset shape %s does not match input %s (deform_conv_cuda.cpp:62-150)'
                         % (tuple(offset.shape), tuple(x.shape)))
    _need_cuda(x, offset, weight)


class DeformConvFunction(torch.autograd.Function):
    """mmdet.ops.dcn.DeformConvFunction (MM/mmdet/ops/dcn/deform_conv.py:14-94) on sm_90a, same arguments.

    forward: the path of ops.DeformConv (smb_deform_im2col + the wgmma GEMM), bit for bit.
    backward (deform_conv_cuda.cpp:262-470), for the inputs that need a gradient:
      s * grad_out -> fp16 NHWC (smb_deform_grad_scale, s a power of two chosen on the device);
      x or offset: grad_col = (s * grad_out) . W on the convolution GEMM (fp32 out), then smb_deform_col2im -> grad_offset
        (deterministic) and grad_input (atomics), divided by s;
      weight: the columns recomputed by smb_deform_im2col (as the reference does), dW by smb_deform_weight_grad (wgmma,
        fixed-order split reduction: the same bits on every run), divided by s.
    Only the SipMask geometry: 3x3 / stride 1 / padding 1 / dilation 1 / groups 1, in_channels and out_channels
    multiples of 64."""

    @staticmethod
    def forward(ctx, input, offset, weight, stride=1, padding=0, dilation=1, groups=1, deformable_groups=1,
                im2col_step=64):
        from . import conv as C
        if input is not None and input.dim() != 4:
            raise ValueError('Expected 4D tensor as input, got {}D tensor instead.'.format(input.dim()))
        cur_im2col_step = min(im2col_step, input.shape[0])
        assert (input.shape[0] % cur_im2col_step) == 0, 'im2col step must divide batchsize'
        _check_deform_args(input, offset, weight, stride, padding, dilation, groups, deformable_groups)
        ctx.deformable_groups = deformable_groups
        ctx.save_for_backward(input, offset, weight)
        wk = C.pack_weight(weight, device=input.device)[0]
        return _deform_conv_forward(input, offset, wk, deformable_groups).contiguous()

    @staticmethod
    @once_differentiable
    def backward(ctx, grad_output):
        from . import conv as C
        x, offset, weight = ctx.saved_tensors
        need_x, need_off, need_w = ctx.needs_input_grad[:3]
        grad_input = grad_offset = grad_weight = None
        _need_cuda(grad_output)
        if need_x or need_off or need_w:
            dg = ctx.deformable_groups
            N, cin, H, W = x.shape
            cout = weight.shape[0]
            with torch.cuda.device(x.device):
                g16, scale = C.deform_grad_scale(grad_output.float().contiguous())
                xh, off = _channels_last(x, offset)
                if need_x or need_off:
                    wt = C.pack_weight(weight)[0].t().contiguous().to(x.device)     # W^T [9*C, Cout], K-major
                    gcol = torch.empty((N, H, W, 9 * cin), dtype=torch.float32, device=x.device)
                    C.ConvPlan(g16, wt, gcol, 1, 1).run()
                    gin, goff = C.deform_col2im(gcol, xh, off, dg, scale, grad_input=need_x, grad_offset=need_off)
                    if need_x:
                        grad_input = gin.permute(0, 3, 1, 2).to(x.dtype).contiguous()
                    if need_off:
                        grad_offset = goff.permute(0, 3, 1, 2).to(offset.dtype).contiguous()
                if need_w:
                    col = C.deform_im2col(xh, off, dg)
                    dw = C.deform_weight_grad(g16, col, scale)
                    grad_weight = dw.view(cout, 3, 3, cin).permute(0, 3, 1, 2).contiguous()
        return grad_input, grad_offset, grad_weight, None, None, None, None, None, None


deform_conv = DeformConvFunction.apply


class TrainableDeformConv(DeformConv):
    """ops.DeformConv whose forward runs through `deform_conv`, so x, the offsets and `weight` get gradients (ops.DeformConv
    itself runs under no_grad).  Inputs smaller than the kernel are zero-padded outside the Function and the output
    cropped back, as MM/mmdet/ops/dcn/deform_conv.py:242-254 does."""

    def forward(self, x, offset):
        kh, kw = self.kernel_size
        input_pad = x.size(2) < kh or x.size(3) < kw
        if input_pad:
            pad_h, pad_w = max(kh - x.size(2), 0), max(kw - x.size(3), 0)
            x = torch.nn.functional.pad(x, (0, pad_w, 0, pad_h), 'constant', 0).contiguous()
            offset = torch.nn.functional.pad(offset, (0, pad_w, 0, pad_h), 'constant', 0).contiguous()
        out = deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                          self.deformable_groups)
        if input_pad:
            out = out[:, :, :out.size(2) - pad_h, :out.size(3) - pad_w].contiguous()
        return out


class DeformConvPack(TrainableDeformConv):
    """mmdet.ops.DeformConvPack (MM/mmdet/ops/dcn/deform_conv.py:258-300): the offsets come from `conv_offset`, an
    nn.Conv2d with bias initialised to zero, so the state-dict keys (weight, conv_offset.weight, conv_offset.bias) are the
    reference's and SipMask++ checkpoints load strictly.  Version-1 checkpoints' `<name>_offset.*` keys are renamed on load
    as the reference does."""

    _version = 2

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
        self.conv_offset = nn.Conv2d(self.in_channels, self.deformable_groups * 2 * self.kernel_size[0] * self.kernel_size[1],
                                     kernel_size=self.kernel_size, stride=self.stride, padding=self.padding, bias=True)
        self.init_offset()

    def init_offset(self):
        self.conv_offset.weight.data.zero_()
        self.conv_offset.bias.data.zero_()

    def forward(self, x):
        offset = self.conv_offset(x)
        return deform_conv(x, offset, self.weight, self.stride, self.padding, self.dilation, self.groups,
                           self.deformable_groups)

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        version = local_metadata.get('version', None)
        if version is None or version < 2:
            for k in ('weight', 'bias'):
                if prefix + 'conv_offset.' + k not in state_dict and prefix[:-1] + '_offset.' + k in state_dict:
                    state_dict[prefix + 'conv_offset.' + k] = state_dict.pop(prefix[:-1] + '_offset.' + k)
        super()._load_from_state_dict(state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys,
                                      error_msgs)


# ----------------------------------------------------------------------------------------------- sigmoid focal loss
def _check_focal(pred, target):
    if pred.dtype != torch.float32 or pred.dim() != 2:
        raise L.SmbError('sigmoid_focal_loss: logits must be a 2-D fp32 tensor [N, C] (got %s %s)'
                         % (pred.dtype, tuple(pred.shape)))
    if target.dtype != torch.int64 or target.dim() != 1 or target.shape[0] != pred.shape[0]:
        raise L.SmbError('sigmoid_focal_loss: targets must be int64 [N] (got %s %s)' % (target.dtype, tuple(target.shape)))
    if pred.shape[1] < 1:
        raise L.SmbError('sigmoid_focal_loss: no classes')
    _need_cuda(pred, target)


class SigmoidFocalLossFunction(torch.autograd.Function):
    """mmdet.ops.sigmoid_focal_loss (MM/mmdet/ops/sigmoid_focal_loss/sigmoid_focal_loss.py:8-33): per-element loss
    [N, C] and its gradient by smb_sigmoid_focal_loss_forward / _backward, the reference kernel's bits."""

    @staticmethod
    def forward(ctx, input, target, gamma=2.0, alpha=0.25):
        _check_focal(input, target)
        input, target = input.contiguous(), target.contiguous()
        ctx.save_for_backward(input, target)
        ctx.gamma, ctx.alpha = float(gamma), float(alpha)
        loss = torch.empty_like(input)
        if input.numel():
            with torch.cuda.device(input.device):
                L.check(L.lib().smb_sigmoid_focal_loss_forward(L.ptr(input), L.ptr(target), input.shape[0], input.shape[1],
                                                               ctypes.c_float(ctx.gamma), ctypes.c_float(ctx.alpha),
                                                               L.ptr(loss), L.stream_ptr()),
                        'smb_sigmoid_focal_loss_forward')
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, d_loss):
        input, target = ctx.saved_tensors
        _need_cuda(d_loss)
        d_loss = d_loss.float().contiguous()
        d_input = torch.empty_like(input)
        if input.numel():
            with torch.cuda.device(input.device):
                L.check(L.lib().smb_sigmoid_focal_loss_backward(L.ptr(input), L.ptr(target), L.ptr(d_loss), input.shape[0],
                                                                input.shape[1], ctypes.c_float(ctx.gamma),
                                                                ctypes.c_float(ctx.alpha), L.ptr(d_input), L.stream_ptr()),
                        'smb_sigmoid_focal_loss_backward')
        return d_input, None, None, None


def sigmoid_focal_loss(pred, target, gamma=2.0, alpha=0.25):
    """Per-element sigmoid focal loss [N, C] of fp32 CUDA logits and int64 targets (1-based, 0 background, < 0 ignored),
    differentiable w.r.t. `pred`."""
    return SigmoidFocalLossFunction.apply(pred, target, gamma, alpha)


class SigmoidFocalLoss(nn.Module):
    """mmdet.ops.SigmoidFocalLoss (sigmoid_focal_loss.py:36-52): the summed loss."""

    def __init__(self, gamma, alpha):
        super().__init__()
        self.gamma = gamma
        self.alpha = alpha

    def forward(self, logits, targets):
        return sigmoid_focal_loss(logits, targets, self.gamma, self.alpha).sum()

    def __repr__(self):
        return self.__class__.__name__ + '(gamma={}, alpha={})'.format(self.gamma, self.alpha)


# ----------------------------------------------------------------------------------------------- SipMask mask loss
def _mask_planes_u8(m, device):
    """one image's gt masks -> uint8 {0, 1} [G, Hf, Wf] on `device` (bool / uint8 / float, tensor or numpy)"""
    if isinstance(m, np.ndarray):
        m = torch.from_numpy(m)
    if m.dim() != 3:
        raise L.SmbError('sipmask_mask_targets: masks must be [G, Hf, Wf] (got %s)' % (tuple(m.shape),))
    if m.dtype not in (torch.uint8, torch.bool, torch.float32, torch.float64, torch.float16):
        raise L.SmbError('sipmask_mask_targets: masks must be uint8, bool or float (got %s)' % m.dtype)
    m = m.to(device)
    return (m != 0).to(torch.uint8) if m.dtype != torch.uint8 else m


@L.device_guard
def sipmask_mask_targets(gt_masks, mask_hw, device=None):
    """SipMaskHead.loss's targets (sipmask_head.py:437-442) for a batch, in one launch: per-image gt masks [G_i, Hf, Wf]
    (uint8, bool or float; {0, 1}) -> (bits [sum G_i, H, ceil(W / 32)] int32 holding uint32 words, bit x % 32 of word
    x / 32 is pixel x; gt_offsets [B + 1] int64, image i's planes are rows gt_offsets[i] .. gt_offsets[i + 1] - 1).
    Bit for bit F.interpolate(scale_factor=0.5, bilinear, align_corners=False) -> zero pad / crop to (H, W) -> gt(0.5)."""
    H, W = int(mask_hw[0]), int(mask_hw[1])
    if H <= 0 or W <= 0:
        raise L.SmbError('sipmask_mask_targets: bad mask size %s' % (tuple(mask_hw),))
    if device is None:
        device = next((m.device for m in gt_masks if isinstance(m, torch.Tensor) and m.is_cuda), None)
    if device is None or torch.device(device).type != 'cuda':
        raise L.SmbError('sipmask_mask_targets: needs a CUDA device (no CPU fallback)')
    planes = [_mask_planes_u8(m, device) for m in gt_masks]
    counts = [int(m.shape[0]) for m in planes]
    gt_offsets = torch.tensor(np.concatenate([[0], np.cumsum(counts)]).astype(np.int64), device=device)
    G = sum(counts)
    bits = torch.empty((G, H, (W + 31) // 32), dtype=torch.int32, device=device)
    if G == 0:
        return bits, gt_offsets
    table, off = [], 0
    for m in planes:
        for _ in range(m.shape[0]):
            table.append((off, m.shape[1], m.shape[2]))
            off += m.shape[1] * m.shape[2]
    src = torch.cat([m.reshape(-1) for m in planes])
    table = torch.tensor(table, dtype=torch.int64).to(device)
    with torch.cuda.device(device):
        L.check(L.lib().smb_mask_targets(L.ptr(src), L.ptr(table), G, H, W, L.ptr(bits), L.stream_ptr()),
                'smb_mask_targets')
    return bits, gt_offsets


def _check_mask_loss(feat, cofs, boxes, img_offsets, targets, gt_rows, weights):
    """What smb_mask_loss accepts; raises before anything is launched."""
    def need(cond, msg):
        if not cond:
            raise L.SmbError('sipmask_mask_loss: ' + msg)
    ts = dict(feat_masks=feat, cofs=cofs, boxes=boxes, img_offsets=img_offsets, targets=targets, gt_rows=gt_rows,
              weights=weights)
    for k, t in ts.items():
        need(isinstance(t, torch.Tensor), '%s must be a tensor' % k)
    need(feat.dtype == torch.float32 and feat.dim() == 4 and feat.shape[1] == 32,
         'feat_masks must be fp32 [B, 32, H, W] (got %s %s)' % (feat.dtype, tuple(feat.shape)))
    B, _, H, W = feat.shape
    need(B > 0 and H > 0 and W > 0, 'empty feat_masks %s' % (tuple(feat.shape),))
    need(cofs.dtype == torch.float32 and cofs.dim() == 2 and cofs.shape[1] == 128,
         'cofs must be fp32 [M, 128] (got %s %s)' % (cofs.dtype, tuple(cofs.shape)))
    M = cofs.shape[0]
    need(boxes.dtype == torch.float32 and tuple(boxes.shape) == (M, 4),
         'boxes must be fp32 [M, 4] (got %s %s)' % (boxes.dtype, tuple(boxes.shape)))
    need(weights.dtype == torch.float32 and tuple(weights.shape) == (M,),
         'weights must be fp32 [M] (got %s %s)' % (weights.dtype, tuple(weights.shape)))
    need(gt_rows.dtype in (torch.int32, torch.int64) and tuple(gt_rows.shape) == (M,),
         'gt_rows must be int32 / int64 [M] (got %s %s)' % (gt_rows.dtype, tuple(gt_rows.shape)))
    need(img_offsets.dtype in (torch.int32, torch.int64) and tuple(img_offsets.shape) == (B + 1,),
         'img_offsets must be int32 / int64 [B + 1] (got %s %s)' % (img_offsets.dtype, tuple(img_offsets.shape)))
    need(targets.dtype == torch.int32 and targets.dim() == 3 and tuple(targets.shape[1:]) == (H, (W + 31) // 32),
         'targets must be sipmask_mask_targets bits [G, %d, %d] (got %s %s)'
         % (H, (W + 31) // 32, targets.dtype, tuple(targets.shape)))
    _need_cuda(*ts.values())
    for k, t in ts.items():
        need(t.is_contiguous(), '%s must be contiguous' % k)
        need(t.device == feat.device, '%s is on %s, feat_masks on %s' % (k, t.device, feat.device))


def _mask_loss_launch(feat, cofs, boxes, offs, targets, rows, weights, g, loss, d_feat, d_cofs):
    B, _, H, W = feat.shape
    M = cofs.shape[0]
    ws = torch.empty(max(int(L.lib().smb_mask_loss_workspace_bytes(B, M, H, W)), 1), dtype=torch.uint8, device=feat.device)
    with torch.cuda.device(feat.device):
        L.check(L.lib().smb_mask_loss(L.ptr(feat), L.ptr(cofs), L.ptr(boxes), L.ptr(offs), L.ptr(targets),
                                      int(targets.shape[0]), L.ptr(rows), L.ptr(weights), L.ptr(g), B, M, H, W,
                                      L.ptr(loss), L.ptr(d_feat), L.ptr(d_cofs), L.ptr(ws), ctypes.c_size_t(ws.numel()),
                                      L.stream_ptr()), 'smb_mask_loss')


class SipMaskMaskLossFunction(torch.autograd.Function):
    """The mask loss of SipMaskHead.loss (sipmask_head.py:446-463) per image, fused: loss[b] and, in backward, d feat_masks
    and d cofs, recomputing the logits (K = 32) instead of keeping any [H, W, M] tensor.  boxes, weights and the targets
    get no gradient, as in the reference (bbox_dt and weighting are detached)."""

    @staticmethod
    def forward(ctx, feat_masks, cofs, boxes, img_offsets, targets, gt_rows, weights):
        _check_mask_loss(feat_masks, cofs, boxes, img_offsets, targets, gt_rows, weights)
        offs, rows = img_offsets.to(torch.int32), gt_rows.to(torch.int32)
        ctx.save_for_backward(feat_masks, cofs, boxes, offs, targets, rows, weights)
        loss = torch.empty(feat_masks.shape[0], dtype=torch.float32, device=feat_masks.device)
        _mask_loss_launch(feat_masks, cofs, boxes, offs, targets, rows, weights, None, loss, None, None)
        return loss

    @staticmethod
    @once_differentiable
    def backward(ctx, g):
        feat, cofs, boxes, offs, targets, rows, weights = ctx.saved_tensors
        need_x, need_c = ctx.needs_input_grad[:2]
        d_feat = d_cofs = None
        if need_x or need_c:
            _need_cuda(g)
            g = g.float().contiguous()
            d_feat = torch.empty_like(feat) if need_x else None
            d_cofs = torch.empty_like(cofs) if need_c else None
            if need_x or cofs.shape[0]:
                _mask_loss_launch(feat, cofs, boxes, offs, targets, rows, weights, g, None, d_feat, d_cofs)
        return d_feat, d_cofs, None, None, None, None, None


def sipmask_mask_loss(feat_masks, cofs, boxes, img_offsets, targets, gt_rows, weights):
    """Per-image SipMask mask loss [B] (sipmask_head.py:446-463 before the sum over images):
      feat_masks [B, 32, H, W] fp32, cofs [M, 128] fp32 (instances of image b are rows img_offsets[b] ..
      img_offsets[b + 1] - 1), boxes [M, 4] fp32 in mask coordinates (bbox_dt), targets / gt_rows: the planes of
      sipmask_mask_targets and each instance's row in them, weights [M] fp32 (the detached weighting).
    loss[b] = sum_n w_n / (M_b bw_n bh_n) sum over n's box of BCE(CropSplit(sigmoid(feat . cof)), gt); differentiable
    w.r.t. feat_masks and cofs."""
    return SipMaskMaskLossFunction.apply(feat_masks, cofs, boxes, img_offsets, targets, gt_rows, weights)


def _bbox_overlaps_aligned(b1, b2):
    """mmdet v1 bbox_overlaps(b1, b2, is_aligned=True) (core/bbox/geometry.py:57-69), the +1 box convention"""
    lt = torch.max(b1[:, :2], b2[:, :2])
    rb = torch.min(b1[:, 2:], b2[:, 2:])
    wh = (rb - lt + 1).clamp(min=0)
    overlap = wh[:, 0] * wh[:, 1]
    area1 = (b1[:, 2] - b1[:, 0] + 1) * (b1[:, 3] - b1[:, 1] + 1)
    area2 = (b2[:, 2] - b2[:, 0] + 1) * (b2[:, 3] - b2[:, 1] + 1)
    return overlap / (area1 + area2 - overlap)


def sipmask_head_mask_loss(feat_masks, flatten_cof_preds, flatten_cls_scores1, det_bboxes, label_list, gt_inds, gt_bboxes,
                           gt_masks):
    """`loss_mask` of SipMaskHead.loss (SipMask-mmdetection sipmask_head.py:403-484, SipMask-VIS :467-548) without
    rescoring, with the per-image block batched into one sipmask_mask_targets and one sipmask_mask_loss call.  The
    arguments are the reference's local variables of the same names (gt_masks: the per-image mask arrays).  Per image:
    the positives (labels > 0) of det_bboxes / 2 with area > 1; weighting = sigmoid(cls score of the label) x aligned IoU
    with the gt box / 2 (+1 convention), normalised to mean ~1 (/ (sum + 1e-4) * count).  Returns the batch mean; the
    gradient flows to feat_masks and flatten_cof_preds only."""
    num_imgs = feat_masks.shape[0]
    H, W = int(feat_masks.shape[2]), int(feat_masks.shape[3])
    device = feat_masks.device
    bits, _ = sipmask_mask_targets(gt_masks, (H, W), device=device)
    gt_off = np.concatenate([[0], np.cumsum([int(m.shape[0]) for m in gt_masks])]).tolist()   # on the host: no sync
    cofs, boxes, rows, weights, offsets = [], [], [], [], [0]
    for i in range(num_imgs):
        labels = torch.cat([lv.flatten() for lv in label_list[i]])
        bbox_dt = (det_bboxes[i] / 2).detach()
        pos_inds = (labels > 0).nonzero().view(-1)
        keep_box = bbox_dt[pos_inds, :4]
        area = (keep_box[:, 2] - keep_box[:, 0]) * (keep_box[:, 3] - keep_box[:, 1])
        keep = area > 1.0
        bbox = keep_box[keep]
        idx_gt = gt_inds[i][keep]
        if bbox.shape[0] > 0:
            cls_score = flatten_cls_scores1[i, pos_inds, labels[pos_inds] - 1].sigmoid().detach()[keep]
            ious = _bbox_overlaps_aligned(gt_bboxes[i][idx_gt] / 2, bbox)
            with torch.no_grad():
                weighting = cls_score * ious
                weighting = weighting / (torch.sum(weighting) + 0.0001) * len(weighting)
            cofs.append(flatten_cof_preds[i][pos_inds][keep])
            boxes.append(bbox)
            rows.append(idx_gt.to(torch.int64) + gt_off[i])
            weights.append(weighting.detach())
        offsets.append(offsets[-1] + int(bbox.shape[0]))
    if offsets[-1] == 0:
        cofs = flatten_cof_preds.new_zeros((0, 128)) + flatten_cof_preds.sum() * 0
        boxes = torch.zeros((0, 4), dtype=torch.float32, device=device)
        rows = torch.zeros((0,), dtype=torch.int64, device=device)
        weights = torch.zeros((0,), dtype=torch.float32, device=device)
    else:
        cofs, boxes = torch.cat(cofs).float().contiguous(), torch.cat(boxes).float().contiguous()
        rows, weights = torch.cat(rows), torch.cat(weights).float().contiguous()
    offs = torch.tensor(offsets, dtype=torch.int32).to(device)
    loss = sipmask_mask_loss(feat_masks.float().contiguous(), cofs, boxes, offs, bits, rows, weights)
    return loss.sum() / num_imgs
