"""Test restatement of the youtubevos pycocotools fork's YTVOSeval for iouType 'segm' with default Params, function by
function, in plain Python and numpy: loadRes's per-frame areas, _toMask's avg_area, _prepare, computeIoU's iou_seq over
decoded masks, evaluateVid, accumulate and summarize.  Independent of the library's kernels and of the decomposition of
the union they use; COCOeval's mask decoding and accumulate are taken from tests/cocoeval_ref.py.  The library itself is
not available, so this is a reading of its published ytvoseval.py / ytvos.py, not a run of it.
"""
import numpy as np

import cocoeval_ref as C

AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 128 ** 2], [128 ** 2, 256 ** 2], [256 ** 2, 1e5 ** 2]]


def avg_area(areas):
    vals = [a for a in areas if a]
    return 0 if len(vals) == 0 else np.array(vals).mean()


def iou_seq(d_seq, g_seq):
    """iou_seq over decoded masks (None: absent)."""
    i, u = .0, .0
    for d, g in zip(d_seq, g_seq):
        if d is not None and g is not None:
            i += int(np.logical_and(d, g).sum())
            u += int(np.logical_or(d, g).sum())
        elif d is None and g is not None:
            u += int(g.sum())
        elif d is not None and g is None:
            u += int(d.sum())
    return i / u if u > .0 else .0


class YTVOSevalRef(C.COCOevalRef):
    """YTVOSeval(ytvosGt, ytvosDt, 'segm') with params.vidIds = vid_ids; results = the loadRes list.  Reuses
    COCOevalRef's accumulate / summarize with the video as the image and YTVIS's area ranges."""

    def __init__(self, gt, results, vid_ids=None):
        assert len(results) > 0
        self.iou_type = 'segm'
        vids = {v['id']: v for v in gt['videos']}
        self.img_ids = list(np.unique(vid_ids if vid_ids is not None else sorted(vids)))
        self.cat_ids = sorted(c['id'] for c in gt['categories'])
        cats = set(self.cat_ids)

        def masks(segs, v):
            return [None if s is None else C.ann_to_mask(s, vids[v]['height'], vids[v]['width']) for s in segs]
        gts, dts = {}, {}
        for a in gt['annotations']:
            if a['video_id'] in self.img_ids and a['category_id'] in cats:
                g = dict(a, ignore=int(bool(a.get('iscrowd', 0))), iscrowd=int(bool(a.get('iscrowd', 0))))
                g['masks'] = masks(a['segmentations'], a['video_id'])
                g['avg_area'] = avg_area(a['areas'])
                gts.setdefault((a['video_id'], a['category_id']), []).append(g)
        for n, r in enumerate(results):               # loadRes: id = n + 1, areas = maskUtils.area per frame
            d = dict(r, id=n + 1)
            d['masks'] = masks(r['segmentations'], r['video_id'])
            d['avg_area'] = avg_area([None if m is None else int(m.sum()) for m in d['masks']])
            if r['video_id'] in self.img_ids and r['category_id'] in cats:
                dts.setdefault((r['video_id'], r['category_id']), []).append(d)
        self._gts, self._dts = gts, dts

    def compute_iou(self, vid, cat):
        gt, dt = self._gts.get((vid, cat), []), self._dts.get((vid, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds][:C.MAX_DETS[-1]]
        out = np.zeros((len(dt), len(gt)))
        for a, d in enumerate(dt):
            for b, g in enumerate(gt):
                out[a, b] = iou_seq(d['masks'], g['masks'])
        return out

    def evaluate_img(self, vid, cat, a_rng, max_det):
        # evaluateVid is evaluateImg with avg_area in place of area
        for lst in (self._gts.get((vid, cat), []), self._dts.get((vid, cat), [])):
            for o in lst:
                o['area'] = o['avg_area']
        return C.COCOevalRef.evaluate_img(self, vid, cat, a_rng, max_det)

    def evaluate(self):
        self.ious = {(i, c): self.compute_iou(i, c) for i in self.img_ids for c in self.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a, C.MAX_DETS[-1])
                          for c in self.cat_ids for a in AREA_RNG for i in self.img_ids]


def run(gt, results, vid_ids=None):
    e = YTVOSevalRef(gt, results, vid_ids)
    e.evaluate()
    e.accumulate()
    e.summarize()
    return e
