"""Generate tests/golden/ref_coco_json.json: the COCO result json the UNMODIFIED reference writes for a few synthetic
records, with the records themselves.

    python tests/golden/gen_golden_coco_json.py        (needs the reference trees; run from the repository root)

MM: CocoDataset._segm2json (SipMask-mmdetection/mmdet/datasets/coco.py:159-194) over bbox2result's per-class boxes and
the per-class RLE lists get_bboxes builds (sipmask_head.py:641-662), imported through tests/golden/_ref_import.py; the
rescoring case passes the (cls_segms, mask_scores) tuple.
SipMask-benchmark: prepare_for_coco_detection / prepare_for_coco_segmentation (fcos_core/data/datasets/evaluation/coco/
coco_eval.py:70-160) on a BoxList in img_shape coordinates, imported through tests/golden/_ref_import_bm.py.  pycocotools
is absent: its `encode` is bound to sipmask_b200.rle.encode (pinned against the oracle by tests/test_head_api.py), so both
sides see the same strings and only the json layout, order, scores and box arithmetic are compared.
"""
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'ref_coco_json.json')


def _record(seed, k, ncls, ori, rescoring):
    from sipmask_b200 import rle
    rs = np.random.RandomState(seed)
    oh, ow = ori
    x1 = rs.uniform(0, ow * 0.6, k)
    y1 = rs.uniform(0, oh * 0.6, k)
    det = np.stack([x1, y1, x1 + rs.uniform(1, ow * 0.4, k), y1 + rs.uniform(1, oh * 0.4, k), rs.uniform(0.05, 1, k)], 1)
    det = det.astype(np.float32)
    labels = rs.randint(0, ncls, k).astype(np.int64)
    masks = (rs.rand(k, oh, ow) < 0.02).astype(np.uint8)
    segms = [rle.encode(m) for m in masks]
    rec = dict(det=det.tolist(), labels=labels.tolist(), segms=[s['counts'].decode() for s in segms], size=[oh, ow])
    if rescoring:
        rec['mask_scores'] = rs.uniform(0, 1, k).astype(np.float32).tolist()
    return rec, masks


def _mm_cases():
    sys.path.insert(0, HERE)
    import _ref_import
    _ref_import.install()
    from mmdet.core import bbox2result
    from mmdet.datasets.coco import CocoDataset
    ncls, cat_ids = 8, [1, 2, 3, 5, 7, 11, 13, 17]
    out = []
    for seed, k, rescoring in ((0, 9, False), (1, 7, True), (2, 0, False)):
        rec, _ = _record(seed, k, ncls, (37, 53), rescoring)
        det = torch.tensor(rec['det'], dtype=torch.float32).reshape(-1, 5)
        labels = torch.tensor(rec['labels'], dtype=torch.int64)
        bbox_result = bbox2result(det, labels, ncls + 1)
        cls_segms = [[] for _ in range(ncls)]
        for i in range(k):                                # sipmask_head.py:645-657: per detection, into its label's list
            cls_segms[rec['labels'][i]].append({'size': rec['size'], 'counts': rec['segms'][i].encode()})
        if rescoring:
            ms = np.asarray(rec['mask_scores'], np.float32)
            lab = np.asarray(rec['labels'])
            seg = (cls_segms, [ms[lab == i] for i in range(ncls)])
        else:
            seg = cls_segms
        ds = object.__new__(CocoDataset)
        ds.img_infos, ds.img_ids, ds.cat_ids = [None], [1000 + seed], cat_ids
        bbox_json, segm_json = ds._segm2json([(bbox_result, seg)])
        out.append(dict(kind='mm', image_id=1000 + seed, cat_ids=cat_ids, rec=rec, bbox_json=bbox_json, segm_json=segm_json))
    return out


def _bm_cases():
    sys.path.insert(0, HERE)
    from _ref_import_bm import load
    load()
    from sipmask_b200 import rle
    sys.modules['pycocotools.mask'].encode = lambda a: [rle.encode(np.asarray(a)[:, :, 0])]
    import importlib.util
    from _ref_import_bm import REF_BM
    from fcos_core.structures.bounding_box import BoxList
    # the file itself: the fcos_core.data package's __init__ needs torch._six, which current torch no longer has
    spec = importlib.util.spec_from_file_location(
        'coco_eval', os.path.join(REF_BM, 'fcos_core/data/datasets/evaluation/coco/coco_eval.py'))
    coco_eval = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(coco_eval)
    coco_eval.tqdm = lambda x: x
    ncls, cat_ids = 8, [1, 2, 3, 5, 7, 11, 13, 17]
    out = []
    # (img_shape, ori_shape): unequal ratios, equal ratios, no detections
    for seed, k, img, ori in ((10, 8, (40, 61), (37, 53)), (11, 5, (74, 106), (37, 53)), (12, 0, (40, 61), (37, 53))):
        rec, masks = _record(seed, k, ncls, ori, False)
        det = np.asarray(rec['det'], np.float32).reshape(-1, 5)
        # boxes in img_shape coordinates
        det[:, :4] *= np.asarray([img[1] / ori[1], img[0] / ori[0]] * 2, np.float32)
        rec['det'] = det.tolist()
        rec['img_shape'], rec['ori_shape'] = list(img), list(ori)
        pred = BoxList(torch.from_numpy(det[:, :4].copy()), (img[1], img[0]), mode='xyxy')
        pred.add_field('scores', torch.from_numpy(det[:, 4].copy()))
        pred.add_field('labels', torch.tensor(rec['labels'], dtype=torch.int64) + 1)
        pred.add_field('mask', torch.from_numpy(masks[:, None]))

        class DS(object):
            id_to_img_map = {0: 2000 + seed}
            contiguous_category_id_to_json_id = {i + 1: c for i, c in enumerate(cat_ids)}

            @staticmethod
            def get_img_info(i):
                return {'width': ori[1], 'height': ori[0]}
        bbox_json = coco_eval.prepare_for_coco_detection([pred], DS)
        segm_json = coco_eval.prepare_for_coco_segmentation([pred], DS)
        out.append(dict(kind='bm', image_id=2000 + seed, cat_ids=cat_ids, rec=rec, bbox_json=bbox_json, segm_json=segm_json))
    return out


if __name__ == '__main__':
    sys.path.insert(0, ROOT)
    if len(sys.argv) > 1:
        cases = _mm_cases() if sys.argv[1] == 'mm' else _bm_cases()
        json.dump(cases, sys.stdout)
    else:
        # one reference tree per process (both import shims own sys.modules)
        cases = []
        for kind in ('mm', 'bm'):
            cases += json.loads(subprocess.check_output([sys.executable, os.path.abspath(__file__), kind], cwd=ROOT))
        with open(OUT, 'w') as f:
            json.dump(cases, f, indent=1)
        print('wrote %s (%d cases)' % (OUT, len(cases)))
