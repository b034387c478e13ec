"""Oracle restatements of the reference operators on the hot path (CPU, fp32).

TEST INFRASTRUCTURE ONLY - see oracle/__init__.py.

All citations are relative to /root/reference/SipMask-mmdetection/ (MM/).
"""
import numpy as np
import torch
import torch.nn.functional as F


# ----------------------------------------------------------------------------
# Deformable convolution v1 forward
#   MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:85-115 (bilinear)
#   MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:191-243 (im2col)
#   MM/mmdet/ops/dcn/src/deform_conv_cuda.cpp:152-260 (im2col -> addmm)
# ----------------------------------------------------------------------------
def deform_im2col(x, offset, kh, kw, stride, pad, dil, deformable_groups):
    """x [B,C,H,W], offset [B,dg*2*kh*kw,Ho,Wo] -> columns [B, C*kh*kw, Ho*Wo].

    Column row index = c*kh*kw + i*kw + j (kernel.cu:203, 239)."""
    B, C, H, W = x.shape
    Ho = (H + 2 * pad - (dil * (kh - 1) + 1)) // stride + 1
    Wo = (W + 2 * pad - (dil * (kw - 1) + 1)) // stride + 1
    cpg = C // deformable_groups
    dt = x.dtype
    hs = torch.arange(Ho, dtype=dt).view(1, Ho, 1) * stride - pad
    ws = torch.arange(Wo, dtype=dt).view(1, 1, Wo) * stride - pad
    cols = x.new_zeros(B, C, kh * kw, Ho, Wo)
    xf = x.reshape(B, C, H * W)
    for g in range(deformable_groups):
        xg = xf[:, g * cpg:(g + 1) * cpg]                       # [B,cpg,HW]
        for i in range(kh):
            for j in range(kw):
                t = i * kw + j
                off_h = offset[:, g * 2 * kh * kw + 2 * t]          # [B,Ho,Wo]
                off_w = offset[:, g * 2 * kh * kw + 2 * t + 1]
                h_im = hs + i * dil + off_h
                w_im = ws + j * dil + off_w
                inside = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)   # kernel.cu:229
                h_low = torch.floor(h_im)
                w_low = torch.floor(w_im)
                lh = h_im - h_low
                lw = w_im - w_low
                hh, hw = 1 - lh, 1 - lw
                h_low = h_low.long()
                w_low = w_low.long()
                h_high = h_low + 1
                w_high = w_low + 1

                def corner(hi, wi, ok):
                    ok = ok & inside
                    idx = (hi.clamp(0, H - 1) * W + wi.clamp(0, W - 1)).view(B, 1, Ho * Wo)
                    v = torch.gather(xg, 2, idx.expand(B, cpg, Ho * Wo))
                    return v * ok.view(B, 1, Ho * Wo).to(dt)

                v1 = corner(h_low, w_low, (h_low >= 0) & (w_low >= 0))
                v2 = corner(h_low, w_high, (h_low >= 0) & (w_high <= W - 1))
                v3 = corner(h_high, w_low, (h_high <= H - 1) & (w_low >= 0))
                v4 = corner(h_high, w_high, (h_high <= H - 1) & (w_high <= W - 1))
                w1 = (hh * hw).view(B, 1, -1)
                w2 = (hh * lw).view(B, 1, -1)
                w3 = (lh * hw).view(B, 1, -1)
                w4 = (lh * lw).view(B, 1, -1)
                val = w1 * v1 + w2 * v2 + w3 * v3 + w4 * v4          # kernel.cu:111-113
                cols[:, g * cpg:(g + 1) * cpg, t] = val.view(B, cpg, Ho, Wo)
    return cols.view(B, C * kh * kw, Ho * Wo), Ho, Wo


USE_C_CROP_SPLIT = False      # bench.py's CPU baseline: C restatement (oracle/csrc/oracle_c.c) instead of numpy
USE_TORCHVISION_DCN = False   # bench.py's CPU baseline flips this: same arithmetic (tests/test_oracle_golden.py
                              # ::test_deform_conv_matches_torchvision), C++ speed instead of python gathers


def deform_conv(x, offset, weight, stride=1, padding=1, dilation=1, deformable_groups=1):
    """DeformConv forward, groups=1, no bias (MM/mmdet/ops/dcn/deform_conv.py:192-255)."""
    Cout, Cin, kh, kw = weight.shape
    if USE_TORCHVISION_DCN and x.size(2) >= kh and x.size(3) >= kw:
        from torchvision.ops import deform_conv2d
        return deform_conv2d(x, offset, weight, stride=stride, padding=padding, dilation=dilation)
    # inputs smaller than the kernel are zero-padded first (deform_conv.py:242-254)
    pad_h = max(kh - x.size(2), 0)
    pad_w = max(kw - x.size(3), 0)
    if pad_h or pad_w:
        x = F.pad(x, (0, pad_w, 0, pad_h))
        offset = F.pad(offset, (0, pad_w, 0, pad_h))
    cols, Ho, Wo = deform_im2col(x, offset, kh, kw, stride, padding, dilation, deformable_groups)
    out = torch.matmul(weight.view(Cout, -1), cols).view(x.size(0), Cout, Ho, Wo)
    if pad_h or pad_w:
        out = out[:, :, :out.size(2) - pad_h, :out.size(3) - pad_w].contiguous()
    return out


# ----------------------------------------------------------------------------
# CropSplit forward  (MM/mmdet/ops/crop/src/crop_split_cuda_kernel.cu:19-59,
#                     MM/mmdet/ops/crop/crop_split.py:12-25)
# ----------------------------------------------------------------------------
def crop_split(data, rois, c=2):
    """data [c*c,H,W,N] fp32, rois [N,4] fp32 -> [H,W,N].

    out[h,w,n] = data[cell,h,w,n] if x1 <= w < x2 and y1 <= h < y2 else 0,
    cell = int((h-y1)/roi_h)*c + int((w-x1)/roi_w),
    roi_w = float32((x2-x1+0.1)/c) with the `+0.1` and `/c` evaluated in double
    (0.1 is a double literal, kernel.cu:46-47)."""
    cc, H, W, N = data.shape
    assert cc == c * c
    if USE_C_CROP_SPLIT and c == 2:
        from . import cbind
        return torch.from_numpy(cbind.crop_split(data.detach().cpu().numpy(), rois.detach().cpu().numpy()))
    d = data.detach().cpu().numpy().astype(np.float32)
    r = rois.detach().cpu().numpy().astype(np.float32)
    x1, y1, x2, y2 = r[:, 0], r[:, 1], r[:, 2], r[:, 3]
    roi_w = (((x2 - x1).astype(np.float32)).astype(np.float64) + 0.1) / c
    roi_h = (((y2 - y1).astype(np.float32)).astype(np.float64) + 0.1) / c
    roi_w = roi_w.astype(np.float32)
    roi_h = roi_h.astype(np.float32)
    pw = np.arange(W, dtype=np.float32).reshape(1, W, 1)
    ph = np.arange(H, dtype=np.float32).reshape(H, 1, 1)
    inside = (pw >= x1) & (ph >= y1) & (pw < x2) & (ph < y2)          # [H,W,N]
    with np.errstate(divide='ignore', invalid='ignore'):
        idx_w = ((pw - x1).astype(np.float32) / roi_w).astype(np.float32)
        idx_h = ((ph - y1).astype(np.float32) / roi_h).astype(np.float32)
    idx_w = np.where(inside, idx_w, 0).astype(np.int64)                # (int) truncation
    idx_h = np.where(inside, idx_h, 0).astype(np.int64)
    cell = np.clip(idx_h * c + idx_w, 0, cc - 1)
    sel = np.take_along_axis(d, cell[None], axis=0)[0]
    out = np.where(inside, sel, np.float32(0))
    return torch.from_numpy(out.astype(np.float32))


# ----------------------------------------------------------------------------
# NMS  (GPU semantics MM/mmdet/ops/nms/src/nms_kernel.cu:14-22,24-68,71-138;
#       CPU semantics MM/mmdet/ops/nms/src/nms_cpu.cpp:6-60)
# ----------------------------------------------------------------------------
def nms(dets, iou_thr, cmp_ge=False, plus_one=True):
    """Greedy NMS on dets [n,5] (x1,y1,x2,y2,score) float32.

    Returns kept ORIGINAL indices in ascending order (nms_kernel.cu:135-138;
    nms_cpu.cpp:59 `nonzero(suppressed == 0)`), int64.
    cmp_ge=False: suppress when IoU >  thr (CUDA path, nms_kernel.cu:61)
    cmp_ge=True : suppress when IoU >= thr (CPU path,  nms_cpu.cpp:56)
    Ties in score are broken by ascending original index (stable sort)."""
    d = np.ascontiguousarray(np.asarray(dets, dtype=np.float32))
    n = d.shape[0]
    if n == 0:
        return np.zeros((0,), dtype=np.int64)
    one = np.float32(1.0 if plus_one else 0.0)
    x1, y1, x2, y2, sc = d[:, 0], d[:, 1], d[:, 2], d[:, 3], d[:, 4]
    areas = ((x2 - x1 + one) * (y2 - y1 + one)).astype(np.float32)
    order = np.argsort(-sc, kind='stable')
    suppressed = np.zeros(n, dtype=bool)
    thr = np.float32(iou_thr)
    for _i in range(n):
        i = order[_i]
        if suppressed[i]:
            continue
        rest = order[_i + 1:]
        xx1 = np.maximum(x1[i], x1[rest])
        yy1 = np.maximum(y1[i], y1[rest])
        xx2 = np.minimum(x2[i], x2[rest])
        yy2 = np.minimum(y2[i], y2[rest])
        w = np.maximum(np.float32(0), (xx2 - xx1 + one).astype(np.float32))
        h = np.maximum(np.float32(0), (yy2 - yy1 + one).astype(np.float32))
        inter = (w * h).astype(np.float32)
        ovr = (inter / ((areas[i] + areas[rest]).astype(np.float32) - inter).astype(np.float32)).astype(np.float32)
        sup = (ovr >= thr) if cmp_ge else (ovr > thr)
        suppressed[rest[sup]] = True
    return np.nonzero(~suppressed)[0].astype(np.int64)


def multiclass_nms_idx(multi_bboxes, multi_scores, score_thr, iou_thr, max_num=-1,
                       score_factors=None, cmp_ge=False, nms_fn=None):
    """MM/mmdet/core/post_processing/bbox_nms.py:79-146.

    multi_bboxes [n,4], multi_scores [n,C+1] (col 0 = background).  nms_fn(dets, thr, cmp_ge) may replace the numpy
    `nms` with a restatement of the same contract (oracle.cbind.nms, for speed).
    Returns dets [k,5] f32, labels [k] i64 (0-based), idxs [k] i64."""
    nms_fn = nms_fn or (lambda d, thr, cmp_ge: nms(d, thr, cmp_ge=cmp_ge))
    num_classes = multi_scores.shape[1]
    bboxes, labels, idxs = [], [], []
    multi_idxs = torch.arange(0, multi_scores.shape[0], dtype=torch.long)
    for i in range(1, num_classes):
        cls_inds = multi_scores[:, i] > score_thr                  # raw score (bbox_nms.py:111)
        if not cls_inds.any():
            continue
        _bboxes = multi_bboxes[cls_inds, :]
        _scores = multi_scores[cls_inds, i]
        _idxs = multi_idxs[cls_inds]
        if score_factors is not None:
            _scores = _scores * score_factors[cls_inds]           # bbox_nms.py:122
        cls_dets = torch.cat([_bboxes, _scores[:, None]], dim=1)
        ki = torch.from_numpy(nms_fn(cls_dets.numpy(), iou_thr, cmp_ge))
        cls_dets = cls_dets[ki]
        bboxes.append(cls_dets)
        labels.append(torch.full((cls_dets.shape[0],), i - 1, dtype=torch.long))
        idxs.append(_idxs[ki])
    if bboxes:
        bboxes = torch.cat(bboxes)
        labels = torch.cat(labels)
        idxs = torch.cat(idxs)
        if bboxes.shape[0] > max_num:
            # reference: bboxes[:, -1].sort(descending=True) (bbox_nms.py:136);
            # the oracle fixes the tie order to "first in class-major order"
            _, inds = bboxes[:, -1].sort(descending=True, stable=True)
            inds = inds[:max_num]
            bboxes, labels, idxs = bboxes[inds], labels[inds], idxs[inds]
    else:
        bboxes = multi_bboxes.new_zeros((0, 5))
        labels = torch.zeros((0,), dtype=torch.long)
        idxs = torch.zeros((0,), dtype=torch.long)
    return bboxes, labels, idxs


# ----------------------------------------------------------------------------
# fast_nms (SSD / VIS path)  MM/mmdet/models/anchor_heads/sipmask_head.py:868-959
# ----------------------------------------------------------------------------
def jaccard(box_a, box_b):
    """[C,A,4] x [C,B,4] -> IoU [C,A,B], no +1 (sipmask_head.py:912-959)."""
    max_xy = torch.min(box_a[:, :, None, 2:], box_b[:, None, :, 2:])
    min_xy = torch.max(box_a[:, :, None, :2], box_b[:, None, :, :2])
    inter = torch.clamp(max_xy - min_xy, min=0)
    inter = inter[..., 0] * inter[..., 1]
    area_a = ((box_a[:, :, 2] - box_a[:, :, 0]) * (box_a[:, :, 3] - box_a[:, :, 1]))[:, :, None]
    area_b = ((box_b[:, :, 2] - box_b[:, :, 0]) * (box_b[:, :, 3] - box_b[:, :, 1]))[:, None, :]
    union = area_a + area_b - inter
    return inter / union


def fast_nms(boxes, scores, cofs, iou_threshold=0.5, top_k=200, score_thr=0.1, max_num=100):
    """boxes [n,4], scores [C,n] (already x centerness), cofs [n,128].

    Returns dets [k,5], classes [k] i64, cofs [k,128], idx [k] i64 (row of `boxes`).
    Sorts are stable (ties -> lower index first); the reference's are unspecified."""
    scores, idx = scores.sort(dim=1, descending=True, stable=True)
    idx = idx[:, :top_k].contiguous()
    scores = scores[:, :top_k]
    num_classes, num_dets = idx.size()
    bx = boxes[idx.view(-1), :].view(num_classes, num_dets, 4)
    iou = jaccard(bx, bx)
    iou.triu_(diagonal=1)
    iou_max, _ = iou.max(dim=1)
    keep = (iou_max <= iou_threshold)
    keep = keep & (scores > score_thr)
    classes = torch.arange(num_classes)[:, None].expand_as(keep)[keep]
    kept_idx = idx[keep]
    kept_scores = scores[keep]
    kept_scores, order = kept_scores.sort(dim=0, descending=True, stable=True)
    order = order[:max_num]
    kept_scores = kept_scores[:max_num]
    classes = classes[order]
    kept_idx = kept_idx[order]
    dets = torch.cat([boxes[kept_idx], kept_scores[:, None]], dim=1)
    return dets, classes, cofs[kept_idx], kept_idx


# ----------------------------------------------------------------------------
# Box decode  (MM/mmdet/core/bbox/transforms.py:202-223; sipmask_head.py:685-695)
# ----------------------------------------------------------------------------
def get_points_single(h, w, stride, dtype=torch.float32):
    x_range = torch.arange(0, w * stride, stride, dtype=dtype)
    y_range = torch.arange(0, h * stride, stride, dtype=dtype)
    y, x = torch.meshgrid(y_range, x_range, indexing='ij')
    return torch.stack((x.reshape(-1), y.reshape(-1)), dim=-1) + stride // 2


def distance2bbox(points, distance, max_shape=None):
    x1 = points[:, 0] - distance[:, 0]
    y1 = points[:, 1] - distance[:, 1]
    x2 = points[:, 0] + distance[:, 2]
    y2 = points[:, 1] + distance[:, 3]
    if max_shape is not None:
        x1 = x1.clamp(min=0, max=max_shape[1] - 1)
        y1 = y1.clamp(min=0, max=max_shape[0] - 1)
        x2 = x2.clamp(min=0, max=max_shape[1] - 1)
        y2 = y2.clamp(min=0, max=max_shape[0] - 1)
    return torch.stack([x1, y1, x2, y2], -1)


# ----------------------------------------------------------------------------
# COCO RLE (column-major run lengths; un-vendored pycocotools maskApi.c rleEncode /
# rleToString, pycocotools 2.0 - "parity unpinned": no reference vector exists)
# ----------------------------------------------------------------------------
def rle_counts(mask):
    """mask [H,W] uint8 -> list of run lengths, column-major, starting with zeros."""
    flat = np.asarray(mask, dtype=np.uint8).T.reshape(-1)      # column-major
    if flat.size == 0:
        return []
    change = np.nonzero(flat[1:] != flat[:-1])[0] + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    runs = np.diff(bounds).tolist()
    if flat[0] != 0:
        runs = [0] + runs
    return runs


def rle_to_string(counts):
    """pycocotools rleToString: LEB128-like, 5 bits/char, delta vs counts[i-2] for i>2."""
    out = []
    for i, c in enumerate(counts):
        x = int(c)
        if i > 2:
            x -= int(counts[i - 2])
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(chr(ch + 48))
    return ''.join(out).encode('ascii')
