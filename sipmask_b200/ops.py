"""Operator API of the hot path - same names / argument meaning as the reference's `mmdet.ops`
and `mmdet.core` entry points, backed by the C ABI (PyTorch tensors in, PyTorch tensors out).

  CropSplit / crop_split   <- MM/mmdet/ops/crop/crop_split.py:12-49
  nms                      <- MM/mmdet/ops/nms/nms_wrapper.py:7-60
  multiclass_nms_idx       <- MM/mmdet/core/post_processing/bbox_nms.py:79-146
  fast_nms                 <- MM/mmdet/models/anchor_heads/sipmask_head.py:868-910
  mask_assemble            <- MM/mmdet/models/anchor_heads/sipmask_head.py:609-627 (fused)
All tensors must be CUDA tensors on an sm_90 device; there is no CPU path.
"""
import ctypes

import numpy as np
import torch
import torch.nn as nn

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


@L.device_guard
def decode_topk(cls_list, box_list, ctr_list, strides, img_shape, nms_pre, scale_factor=None, box_scales=None):
    """Per-level tensors channel-last fp32: cls [h,w,C], box [h,w,4] (distances x stride), ctr [h,w,1|].

    Returns cand_boxes [n,4], cand_scores [n,C], cand_ctr [n], cand_loc [n] int32."""
    nl = len(cls_list)
    C = cls_list[0].shape[-1]
    lv, keep_alive = level_descs(cls_list, box_list, ctr_list, strides, box_scales)
    lib = L.lib()
    dev = cls_list[0].device
    ws_bytes = lib.smb_decode_workspace_bytes(nl, lv, int(nms_pre))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    n = sum(min(c.shape[0] * c.shape[1], nms_pre) if nms_pre > 0 else c.shape[0] * c.shape[1] for c in cls_list)
    boxes = torch.empty((n, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n, C), dtype=torch.float32, device=dev)
    ctr = torch.empty((n,), dtype=torch.float32, device=dev)
    loc = torch.empty((n,), dtype=torch.int32, device=dev)
    sf = None
    if scale_factor is not None:
        a = np.atleast_1d(np.asarray(scale_factor, dtype=np.float32))
        sf = L.f4(a if a.size == 4 else [a[0]] * 4)
    L.check(lib.smb_decode_topk(nl, lv, C, int(nms_pre), int(img_shape[0]), int(img_shape[1]), sf, L.ptr(boxes),
                                L.ptr(scores), L.ptr(ctr), L.ptr(loc), L.ptr(ws), ctypes.c_size_t(ws_bytes),
                                L.stream_ptr()), 'smb_decode_topk')
    return boxes, scores, ctr, loc


@L.device_guard
def pair_decode_topk(cls_list, box_list, ctr_list, strides, img_shape, nms_pre=1000, score_thr=0.05, box_scales=None):
    """SipMask-benchmark candidate selection (smb_pair_decode_topk).  Per-level channel-last fp32 tensors as decode_topk:
    cls [h,w,C] logits, ctr [h,w,1|], box [h,w,4]; distances are relu(box * box_scales[l]) * strides[l] when box_scales is
    given (raw bbox_pred), else relu(box).  Returns (boxes [n,4], scores [n] = sqrt(cls * ctr), labels [n] int32 0-based,
    loc [n] int32, n_cand device int32 [1]); n is the slot capacity, rows past n_cand are zero / -1."""
    nl = len(cls_list)
    C = cls_list[0].shape[-1]
    lv, keep_alive = level_descs(cls_list, box_list, ctr_list, strides, box_scales)
    lib = L.lib()
    dev = cls_list[0].device
    n = lib.smb_pair_decode_slots(nl, lv, C, int(nms_pre))
    if n < 0:
        raise L.SmbError('pair_decode_topk: unsupported levels / nms_pre=%d' % nms_pre)
    ws_bytes = lib.smb_pair_decode_workspace_bytes(nl, lv, C, int(nms_pre))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    boxes = torch.empty((n, 4), dtype=torch.float32, device=dev)
    scores = torch.empty((n,), dtype=torch.float32, device=dev)
    labels = torch.empty((n,), dtype=torch.int32, device=dev)
    loc = torch.empty((n,), dtype=torch.int32, device=dev)
    n_cand = torch.empty((1,), dtype=torch.int32, device=dev)
    L.check(lib.smb_pair_decode_topk(nl, lv, C, ctypes.c_float(score_thr), int(nms_pre), int(img_shape[0]), int(img_shape[1]),
                                     L.ptr(boxes), L.ptr(scores), L.ptr(labels), L.ptr(loc), L.ptr(n_cand), n, L.ptr(ws),
                                     ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_pair_decode_topk')
    return boxes, scores, labels, loc, n_cand


@L.device_guard
def ml_nms_topk(boxes, scores, labels, n_cand, iou_thr=0.6, max_per_img=100, out_cap=None):
    """SipMask-benchmark label-aware NMS + k-th-value cut (smb_ml_nms_topk) over the first *n_cand rows of boxes [cap,4],
    scores [cap], labels [cap] int32.  Returns (det [out_cap,5], labels int64, idx int64, count int32 [1], kept_total
    int32 [1]); out_cap defaults to cap."""
    _need_cuda(boxes, scores, labels, n_cand)
    boxes, scores = boxes.float().contiguous(), scores.float().contiguous()
    labels, n_cand = labels.to(torch.int32).contiguous(), n_cand.to(torch.int32).contiguous()
    cap = boxes.shape[0]
    out_cap = cap if out_cap is None else int(out_cap)
    dev = boxes.device
    lib = L.lib()
    ws_bytes = lib.smb_ml_nms_workspace_bytes(cap)
    ws = torch.empty(max(ws_bytes, 1), dtype=torch.uint8, device=dev)
    det = torch.empty((out_cap, 5), dtype=torch.float32, device=dev)
    lab = torch.empty((out_cap,), dtype=torch.long, device=dev)
    idx = torch.empty((out_cap,), dtype=torch.long, device=dev)
    cnt = torch.empty((1,), dtype=torch.int32, device=dev)
    total = torch.empty((1,), dtype=torch.int32, device=dev)
    L.check(lib.smb_ml_nms_topk(L.ptr(boxes), L.ptr(scores), L.ptr(labels), L.ptr(n_cand), cap, ctypes.c_float(iou_thr),
                                int(max_per_img), out_cap, L.ptr(det), L.ptr(lab), L.ptr(idx), L.ptr(cnt), L.ptr(total),
                                L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_ml_nms_topk')
    return det, lab, idx, cnt, total


# ------------------------------------------------------------------------------------ multi-class NMS
@L.device_guard
def multiclass_nms_idx(multi_bboxes, multi_scores, score_thr, nms_cfg, max_num=-1, score_factors=None,
                       has_bg_column=True, cmp_ge=False, return_count_tensor=False):
    """Same contract as mmdet.core.multiclass_nms_idx (bbox_nms.py:79-146): returns
    (dets [k,5], labels [k] int64 0-based, idxs [k] int64).  `multi_scores` carries the background
    column 0 like the reference unless has_bg_column=False."""
    _need_cuda(multi_bboxes, multi_scores)
    iou_thr = nms_cfg.get('iou_thr', 0.5) if isinstance(nms_cfg, dict) else float(nms_cfg)
    scores = multi_scores[:, 1:] if has_bg_column else multi_scores
    scores = scores.float().contiguous()
    boxes = multi_bboxes.float().contiguous()
    n, C = scores.shape
    dev = boxes.device
    if score_factors is None:
        score_factors = torch.ones(n, dtype=torch.float32, device=dev)
    ctr = score_factors.float().contiguous()
    if max_num is None or max_num <= 0:
        max_num = 1024
    lib = L.lib()
    ws_bytes = lib.smb_multiclass_nms_workspace_bytes(n, C)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    det = torch.empty((max_num, 5), dtype=torch.float32, device=dev)
    lab = torch.empty((max_num,), dtype=torch.long, device=dev)
    idx = torch.empty((max_num,), dtype=torch.long, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    L.check(lib.smb_multiclass_nms(L.ptr(boxes), L.ptr(scores), L.ptr(ctr), n, C, ctypes.c_float(score_thr),
                                   ctypes.c_float(iou_thr), int(max_num), int(cmp_ge), L.ptr(det), L.ptr(lab),
                                   L.ptr(idx), L.ptr(cnt), L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
            'smb_multiclass_nms')
    if return_count_tensor:
        return det, lab, idx, cnt
    k = int(cnt.item())
    return det[:k], lab[:k], idx[:k]


@L.device_guard
def fast_nms(boxes, scores, ctr, iou_threshold=0.5, top_k=200, score_thr=0.1, max_num=100,
             return_count_tensor=False):
    """boxes [n,4], scores [n,C] sigmoid (NOT yet multiplied by ctr), ctr [n].
    Returns (dets [k,5], classes [k], idx [k]) like SipMaskHead.fast_nms (sipmask_head.py:868-910)
    with the coefficient gather left to the caller (`cofs[idx]`)."""
    _need_cuda(boxes, scores, ctr)
    boxes = boxes.float().contiguous()
    scores = scores.float().contiguous()
    ctr = ctr.float().contiguous()
    n, C = scores.shape
    dev = boxes.device
    lib = L.lib()
    ws_bytes = lib.smb_fast_nms_workspace_bytes(n, C, int(top_k))
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    det = torch.empty((max_num, 5), dtype=torch.float32, device=dev)
    lab = torch.empty((max_num,), dtype=torch.long, device=dev)
    idx = torch.empty((max_num,), dtype=torch.long, device=dev)
    cnt = torch.zeros(1, dtype=torch.int32, device=dev)
    L.check(lib.smb_fast_nms(L.ptr(boxes), L.ptr(scores), L.ptr(ctr), n, C, ctypes.c_float(score_thr),
                             ctypes.c_float(iou_threshold), int(top_k), int(max_num), L.ptr(det), L.ptr(lab),
                             L.ptr(idx), L.ptr(cnt), L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
            'smb_fast_nms')
    if return_count_tensor:
        return det, lab, idx, cnt
    k = int(cnt.item())
    return det[:k], lab[:k], idx[:k]


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
def gather_track_feats(track_feats, det, count, scale_factor=1.0, feat_stride=8.0):
    """SipMask-VIS `extract_box_feature_center_single`: track_feats [512,h,w] (reference layout) or [h,w,512] channel-last
    fp32, det [max,5], count device int -> [max,512] features at floor((x1+x2) * sf / 2 / 8) (zeros after count)."""
    _need_cuda(track_feats, det, count)
    t = track_feats.float()
    if t.shape[0] == 512 and t.shape[-1] != 512:
        t = t.permute(1, 2, 0)
    t = t.contiguous()
    h, w, C = t.shape
    a = np.atleast_1d(np.asarray(scale_factor, dtype=np.float32))
    sx, sy = float(a[0]), float(a[1] if a.size >= 2 else a[0])
    det = det.float().contiguous()
    out = torch.empty((det.shape[0], C), dtype=torch.float32, device=det.device)
    L.check(L.lib().smb_gather_track_feats(L.ptr(t), h, w, C, L.ptr(det), L.ptr(count.to(torch.int32)), det.shape[0],
                                           ctypes.c_float(sx), ctypes.c_float(sy), ctypes.c_float(feat_stride), L.ptr(out),
                                           L.stream_ptr()), 'smb_gather_track_feats')
    return out


# -------------------------------------------------------------------------------------- mask assembly
@L.device_guard
def set_mask_tensor_dot(on):
    """fp16 prototypes: tensor-core (True) or scalar-fmaf (False) mask kernels for later calls (smb_mask_set_tensor_dot);
    on=None only queries.  Returns the previous setting."""
    return bool(L.lib().smb_mask_set_tensor_dot(-1 if on is None else int(bool(on))))


def mask_assemble(protos, cofs, boxes, box_scale, layout='chw', out_dtype=torch.float32, out=None):
    """protos [32,H,W] ('chw') or [H,W,32] ('hwc'), fp32/fp16; cofs [N,128] fp32; boxes [N,4] fp32
    (image space); rois = boxes * box_scale (scalar or 4-vector).  Returns pos_masks [N,H,W]."""
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
    if out is None:
        out = torch.empty((N, H, W), dtype=out_dtype, device=protos.device)
    L.check(L.lib().smb_mask_assemble(L.ptr(protos), _dt(protos), 1 if layout == 'hwc' else 0, L.ptr(cofs),
                                      L.ptr(boxes), bs, L.ptr(out), _dt(out), H, W, N, L.stream_ptr()),
            'smb_mask_assemble')
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
        wk = self._packed[1]
        with torch.cuda.device(x.device):
            xh = x.permute(0, 2, 3, 1).contiguous().to(torch.float16)
            off = offset.permute(0, 2, 3, 1).contiguous().float()
            col = C.deform_im2col(xh, off, self.deformable_groups)
            out = torch.empty((N, H, W, self.out_channels), dtype=torch.float16, device=x.device)
            C.ConvPlan(col, wk, out, 1, 1).run()
            y = out.permute(0, 3, 1, 2).to(x.dtype)
        if input_pad:
            y = y[:, :, :y.size(2) - pad_h, :y.size(3) - pad_w]
        return y.contiguous()
