"""COCO result json of one image's record, exactly as the reference writes it (host only).

MM (SipMask-mmdetection/mmdet/datasets/coco.py:120-127,159-194, `_segm2json` over bbox2result's per-class lists):
detections grouped by label in ascending order, detection order inside a label; bbox = xyxy2xywh (+1 on width and height,
python floats of the float32 boxes); the segm score is the mask score when the record carries one (SipMask++ rescoring,
sipmask_head.py:641-643,659-660), the box score otherwise; counts decoded to str.

SipMask-benchmark (fcos_core/data/datasets/evaluation/coco/coco_eval.py:70-160, prepare_for_coco_detection /
prepare_for_coco_segmentation): detections in record order; boxes resized from the img_shape to the ori_shape canvas with
BoxList.resize arithmetic (float32 tensors times python-float ratios, one ratio when both axes agree), then to xywh with
TO_REMOVE = 1; labels are 0-based in the record (the reference's are 1-based: cat_ids[label] maps the same class).
"""
import numpy as np
import torch


def _np(t):
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t)


def _segm(rle):
    counts = rle['counts']
    return {'size': list(rle['size']), 'counts': counts.decode() if isinstance(counts, bytes) else counts}


def coco_json(rec, image_id, cat_ids, benchmark=False, meta=None):
    """rec: one image's record with det_bboxes [>= count, 5], det_labels (0-based), count, segms (the image's RLE dicts in
    detection order) and, for SipMask++, mask_scores.  cat_ids: COCO category id per 0-based label.  meta: dict with
    img_shape / ori_shape (default rec['meta']; benchmark=True only).  Returns (bbox_json, segm_json), two lists of dicts."""
    k = int(_np(rec['count']).reshape(-1)[0])
    det = _np(rec['det_bboxes'])[:k].astype(np.float32)
    labels = _np(rec['det_labels'])[:k].astype(np.int64)
    segms = rec['segms']
    if len(segms) != k:
        raise ValueError('coco_json: %d segms for %d detections' % (len(segms), k))
    if benchmark:
        return _bm_json(det, labels, segms, image_id, cat_ids, meta if meta is not None else rec['meta'])
    mask_scores = _np(rec['mask_scores'])[:k].astype(np.float32) if 'mask_scores' in rec else None
    bbox_json, segm_json = [], []
    for label in sorted(set(labels.tolist())):
        rows = np.flatnonzero(labels == label)
        for i in rows:
            b = det[i].tolist()
            bbox_json.append(dict(image_id=image_id, bbox=[b[0], b[1], b[2] - b[0] + 1, b[3] - b[1] + 1], score=float(det[i][4]),
                                  category_id=cat_ids[label]))
        for i in rows:
            b = det[i].tolist()
            score = float(mask_scores[i]) if mask_scores is not None else float(det[i][4])
            segm_json.append(dict(image_id=image_id, bbox=[b[0], b[1], b[2] - b[0] + 1, b[3] - b[1] + 1], score=score,
                                  category_id=cat_ids[label], segmentation=_segm(segms[i])))
    return bbox_json, segm_json


def _bm_json(det, labels, segms, image_id, cat_ids, meta):
    if len(det) == 0:                               # `if len(prediction) == 0: continue`
        return [], []
    ih, iw = int(meta['img_shape'][0]), int(meta['img_shape'][1])
    oh, ow = int(meta['ori_shape'][0]), int(meta['ori_shape'][1])
    box = torch.from_numpy(det[:, :4].copy())
    rw, rh = float(ow) / float(iw), float(oh) / float(ih)
    if rw == rh:
        box = box * rw
    else:
        x1, y1, x2, y2 = box.split(1, dim=-1)
        box = torch.cat((x1 * rw, y1 * rh, x2 * rw, y2 * rh), dim=-1)
    x1, y1, x2, y2 = box.split(1, dim=-1)
    boxes = torch.cat((x1, y1, x2 - x1 + 1, y2 - y1 + 1), dim=-1).tolist()
    scores = torch.from_numpy(det[:, 4].copy()).tolist()
    cats = [cat_ids[int(l)] for l in labels]
    bbox_json = [dict(image_id=image_id, category_id=cats[i], bbox=boxes[i], score=scores[i]) for i in range(len(boxes))]
    segm_json = [dict(image_id=image_id, category_id=cats[i], segmentation=_segm(segms[i]), score=scores[i])
                 for i in range(len(boxes))]
    return bbox_json, segm_json
