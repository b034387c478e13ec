"""Generate tests/golden/ref_render.npz by calling the UNMODIFIED reference show_result functions on small cases.

Run in the build container only (needs /root/reference):   python tests/golden/gen_golden_render.py
Each reference tree has its own `mmdet` package, so the MM tree (mmdet/apis/inference.py:119-184, show_result) and the
VIS tree (mmdet/models/detectors/base.py:90-192, BaseDetector.show_result(is_video=True)) run in two child processes.
Bindings around the reference code (nothing in it is changed):
  maskUtils.decode        -> identity (the cases hand dense masks)
  mmcv.imread             -> identity
  mmcv.concat_list        -> itertools.chain
  mmcv.imshow_det_bboxes  -> a recorder of the image, boxes, labels and score_thr it is handed (the box drawing itself is
                             OpenCV's, which is not installed here: the fixture pins which boxes are handed over)
  tensor2imgs (VIS)       -> returns the case image, so the reference draws into it
  np.random.randint (MM)  -> the numpy function, with its draws recorded (the colours the reference used)
  np.bool                 -> bool (numpy 2 removed the alias the 2019 trees use), in these processes only
Stored per case c: the input (c<c>_img, _det, _labels, _ids, _masks), MM's returned image and recorded arguments
(c<c>_mm_*), VIS's drawn image and recorded arguments (c<c>_vis_*, absent when the reference returned early), and the
colour tables (mm_colors: the longest list of draws, vis_palette: the detector's color_mask).
"""
import itertools
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
NUM_CLASSES = 81
SCORE_THR = 0.3


def cases():
    """Small images (widths not multiples of 32, a 1 x 1) with engine-like records: det [k, 5] fp32, labels, obj_ids and
    dense masks [k, h, w].  Labels come unsorted, masks overlap across labels and touch every border, scores sit on both
    sides of 0.3 and exactly at float32(0.3), ids include -1, duplicates and 252, corners fall outside the image."""
    rs = np.random.RandomState(5)
    t = np.float32(SCORE_THR)
    up = np.nextafter(t, np.float32(1))
    out = []

    def record(h, w, labels, scores, ids):
        k = len(labels)
        img = rs.randint(0, 256, (h, w, 3)).astype(np.uint8)
        masks = np.zeros((k, h, w), np.uint8)
        det = np.zeros((k, 5), np.float32)
        for i in range(k):
            y0, x0 = rs.randint(0, h), rs.randint(0, w)
            masks[i, y0:y0 + rs.randint(1, h + 1), x0:x0 + rs.randint(1, w + 1)] = 1
            masks[i] ^= (rs.rand(h, w) < 0.1).astype(np.uint8)
            det[i, :4] = np.sort(rs.uniform(-6, w + 6, 2)).tolist()[:1] + np.sort(rs.uniform(-6, h + 6, 2)).tolist()[:1] + \
                [rs.uniform(-6, w + 6), rs.uniform(-6, h + 6)]
        det[:, 4] = scores
        return dict(img=img, det=det, labels=np.array(labels, np.int64), ids=np.array(ids, np.int64), masks=masks)

    c = record(7, 45, [3, 1, 3, 0, 1, 2, 79], [0.9, t, 0.31, 0.29, 0.5, 0.8, up], [-1, 4, 4, 252, 0, 7, 4])
    c['masks'][0] = 0
    c['masks'][0, 0, :] = c['masks'][0, -1, :] = c['masks'][0, :, 0] = c['masks'][0, :, -1] = 1      # every border
    c['det'][0, :4] = (-0.7, -3.2, 44.9, 6.99)
    c['det'][2, :4] = (30.5, 5.0, 2.2, 1.9)                                                           # corners swapped
    out.append(c)
    k = 14
    c = record(33, 70, list(rs.randint(0, 10, k)), list(rs.uniform(0.05, 1, k).astype(np.float32)),
               [3, -1, 252, 3, 5, 0, 0, -1, 9, 252, 1, 3, 2, 6])
    c['det'][3, 4] = t
    c['det'][5, 4] = 0.1                                    # id 0's first detection is below the threshold, its last above
    c['det'][6, 4] = 0.7
    c['det'][9, 4] = 0.2                                    # id 252's last detection is below the threshold
    c['det'][4, :4] = (-20.0, -15.0, 100.0, 50.0)           # every side outside the image
    out.append(c)
    out.append(record(1, 1, [79, 0, 5], [0.95, 0.4, 0.2], [252, -1, 252]))
    out.append(record(5, 33, [2, 1], [0.1, t], [-1, -1]))
    return out


def _bbox_segm_result(c):
    """bbox2result / the head's per-class segms of a case: per label a [n, 5] array and a list of masks."""
    bbox = [c['det'][c['labels'] == l] for l in range(NUM_CLASSES - 1)]
    segm = [[c['masks'][i] for i in np.nonzero(c['labels'] == l)[0]] for l in range(NUM_CLASSES - 1)]
    return bbox, segm


def _recorder(log):
    def imshow_det_bboxes(img, bboxes, labels, class_names=None, score_thr=0, **kw):
        log.append(dict(img=np.array(img, copy=True), bboxes=np.array(bboxes, copy=True), labels=np.array(labels, copy=True),
                        score_thr=np.array(score_thr, np.float64)))
    return imshow_det_bboxes


def run_mm(dst):
    sys.path.insert(0, HERE)
    import _ref_import
    _ref_import.install()
    np.bool = bool
    from mmdet.apis import inference as inf
    log, draws = [], []
    inf.maskUtils = type('maskUtils', (), {'decode': staticmethod(lambda m: m)})
    inf.mmcv.imread = lambda img: img
    inf.mmcv.concat_list = lambda lists: list(itertools.chain(*lists))
    inf.mmcv.imshow_det_bboxes = _recorder(log)
    randint = np.random.randint

    def recorded(*a, **k):
        r = randint(*a, **k)
        draws[-1].append(np.array(r, copy=True))
        return r
    np.random.randint = recorded
    out = {}
    names = ['class%d' % i for i in range(NUM_CLASSES - 1)]
    for n, c in enumerate(cases()):
        draws.append([])
        log.clear()
        img = inf.show_result(c['img'].copy(), _bbox_segm_result(c), names, score_thr=SCORE_THR, show=False)
        assert len(log) == 1
        out['c%d_mm_img' % n] = img
        for k in ('bboxes', 'labels', 'score_thr'):
            out['c%d_mm_%s' % (n, k)] = log[0][k]
        assert np.array_equal(log[0]['img'], img)
    longest = max(draws, key=len)
    out['mm_colors'] = np.concatenate(longest).reshape(-1, 3)
    for d in draws:                                        # every call drew a prefix of the same stream
        assert np.array_equal(np.concatenate(d).reshape(-1, 3), out['mm_colors'][:len(d)])
    np.savez(dst, **out)


def run_vis(dst):
    sys.path.insert(0, HERE)
    import collections
    import collections.abc
    for n in ('Sequence', 'Mapping', 'Iterable'):
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    import _ref_import
    _ref_import.install('/root/reference/SipMask-VIS')
    np.bool = bool
    import torch
    from mmdet.core.bbox.transforms import bbox2result_with_id
    from mmdet.models.detectors import base
    log = []
    base.maskUtils = type('maskUtils', (), {'decode': staticmethod(lambda m: m)})
    base.mmcv.imshow_det_bboxes = _recorder(log)
    det = base.BaseDetector()
    out = {}
    names = ['class%d' % i for i in range(NUM_CLASSES - 1)]
    for n, c in enumerate(cases()):
        img = c['img'].copy()
        base.tensor2imgs = lambda tensor, **kw: [img]
        ids = [int(v) for v in c['ids']]
        bbox_result = bbox2result_with_id(torch.from_numpy(c['det']), torch.from_numpy(c['labels']), ids)
        segm_result = {}
        for i, oid in enumerate(ids):                      # the head's obj_segms: the last detection of an id wins
            if oid >= 0:
                segm_result[oid] = c['masks'][i]
        meta = dict(img_shape=img.shape, video_id=0, frame_id=n)
        data = dict(img=[None], img_meta=[type('DC', (), {'data': [[meta]]})()])
        log.clear()
        det.show_result(data, (bbox_result, segm_result), dict(mean=0, std=1), dataset=names, is_video=True,
                        score_thr=SCORE_THR)
        if log:
            out['c%d_vis_img' % n] = img
            for k in ('bboxes', 'labels'):
                out['c%d_vis_%s' % (n, k)] = log[0][k]
            assert np.array_equal(log[0]['img'], img)
    out['vis_palette'] = det.color_mask
    np.savez(dst, **out)


def main():
    with tempfile.TemporaryDirectory() as tmp:
        parts = {}
        for tree in ('mm', 'vis'):
            parts[tree] = os.path.join(tmp, tree + '.npz')
            subprocess.check_call([sys.executable, os.path.abspath(__file__), tree, parts[tree]], cwd=ROOT)
        out = {}
        for n, c in enumerate(cases()):
            for k, v in c.items():
                out['c%d_%s' % (n, k)] = v
        out['n_cases'] = np.array(len(cases()))
        out['num_classes'] = np.array(NUM_CLASSES)
        out['score_thr'] = np.array(SCORE_THR)
        for p in parts.values():
            with np.load(p) as z:
                out.update({k: z[k] for k in z.files})
    np.savez_compressed(os.path.join(HERE, 'ref_render.npz'), **out)
    print('wrote', sorted(out))


if __name__ == '__main__':
    if len(sys.argv) == 3:
        {'mm': run_mm, 'vis': run_vis}[sys.argv[1]](sys.argv[2])
    else:
        main()
