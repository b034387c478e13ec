"""COCOeval with p.useCats, p.catIds and any maxDets: a numpy restatement of pycocotools 2.0 pinned to hand-computed
answers, and the checks of CocoParams2 / smb_coco_params2_t that need no device.  The device evaluation is checked
against the restatement in test_gpu_cocoeval_cats.py."""
import ctypes

import numpy as np
import pytest

from cocoeval_ref import IOU_THRS, REC_THRS, AREA_RNG, AREA_RNG_LBL, ann_to_mask, bb_iou, mask_iou


class COCOevalParamsRef:
    """COCOeval(cocoGt, cocoDt, iouType) with params.imgIds = img_ids, params.useCats = use_cats, params.catIds = cat_ids
    (None: sorted(getCatIds())) and params.maxDets = max_dets; results = the loadRes list.  Read from pycocotools 2.0's
    cocoeval.py: evaluate() de-duplicates catIds only when useCats; _prepare loads every annotation of the images when
    not useCats; computeIoU / evaluateImg concatenate the (image, category) lists over p.catIds when not useCats;
    accumulate runs on p.catIds = [-1].  mask_cache: segmentation object id -> decoded mask (results shared by runs)."""

    def __init__(self, gt, results, iou_type, img_ids=None, use_cats=1, cat_ids=None, max_dets=None, mask_cache=None):
        assert len(results) > 0
        self.iou_type, self.use_cats = iou_type, use_cats
        imgs = {im['id']: im for im in gt['images']}
        self.img_ids = [int(i) for i in np.unique(img_ids if img_ids is not None else sorted(imgs))]
        cats = sorted(c['id'] for c in gt['categories']) if cat_ids is None else list(cat_ids)
        self.cat_ids = [int(c) for c in np.unique(cats)] if use_cats else [int(c) for c in cats]
        self.max_dets = sorted(max_dets if max_dets is not None else [1, 10, 100])
        cache = {} if mask_cache is None else mask_cache

        def mask(segm, im):
            k = id(segm)
            if k not in cache:
                cache[k] = ann_to_mask(segm, im['height'], im['width'])
            return cache[k]

        gts, dts = {}, {}
        for a in gt['annotations']:                   # getAnnIds(imgIds[, catIds])
            if a['image_id'] in self.img_ids and (not use_cats or a['category_id'] in self.cat_ids):
                g = dict(a, ignore=int(bool(a['iscrowd'])))
                if iou_type == 'segm':
                    g['mask'] = mask(a['segmentation'], imgs[a['image_id']])
                gts.setdefault((a['image_id'], a['category_id']), []).append(g)
        for n, r in enumerate(results):               # loadRes: id = n + 1, area
            d = dict(r, id=n + 1)
            if iou_type == 'bbox':
                d['area'] = r['bbox'][2] * r['bbox'][3]
            else:
                d['mask'] = mask(r['segmentation'], imgs[r['image_id']])
                d['area'] = int(d['mask'].sum())
            if r['image_id'] in self.img_ids and (not use_cats or r['category_id'] in self.cat_ids):
                dts.setdefault((r['image_id'], r['category_id']), []).append(d)
        self._gts, self._dts = gts, dts

    def lists(self, img, cat):
        if self.use_cats:
            return self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        return ([g for c in self.cat_ids for g in self._gts.get((img, c), [])],
                [d for c in self.cat_ids for d in self._dts.get((img, c), [])])

    def compute_iou(self, img, cat):
        gt, dt = self.lists(img, cat)
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds][:self.max_dets[-1]]
        out = np.zeros((len(dt), len(gt)))
        for a, d in enumerate(dt):
            for b, g in enumerate(gt):
                if self.iou_type == 'bbox':
                    out[a, b] = bb_iou([float(v) for v in d['bbox']], [float(v) for v in g['bbox']], g['iscrowd'])
                else:
                    out[a, b] = mask_iou(d['mask'], g['mask'], g['iscrowd'])
        return out

    def evaluate_img(self, img, cat, a_rng, max_det):
        gt, dt = self.lists(img, cat)
        if len(gt) == 0 and len(dt) == 0:
            return None
        ig = [1 if (g['ignore'] or (g['area'] < a_rng[0] or g['area'] > a_rng[1])) else 0 for g in gt]
        gtind = np.argsort(ig, kind='mergesort')
        gt = [gt[i] for i in gtind]
        gt_ig = np.array([ig[i] for i in gtind])
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:max_det]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[img, cat]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        dt_ig = np.zeros((T, D))
        if len(ious) != 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gt_ig[m] == 0 and gt_ig[gind] == 1:
                            break
                        if ious[dind, gind] < iou:
                            continue
                        iou = ious[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dt_ig[tind, dind] = gt_ig[m]
                    dtm[tind, dind] = gt[m]['id']
                    gtm[tind, m] = d['id']
        a = np.array([d['area'] < a_rng[0] or d['area'] > a_rng[1] for d in dt]).reshape((1, len(dt)))
        dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return dict(dtIds=[d['id'] for d in dt], gtIds=[g['id'] for g in gt], dtMatches=dtm, gtIgnore=gt_ig,
                    dtIgnore=dt_ig, dtScores=[d['score'] for d in dt])

    def evaluate(self):
        cats = self.cat_ids if self.use_cats else [-1]
        self.ious = {(i, c): self.compute_iou(i, c) for i in self.img_ids for c in cats}
        self.eval_imgs = [self.evaluate_img(i, c, a, self.max_dets[-1]) for c in cats for a in AREA_RNG
                          for i in self.img_ids]

    def accumulate(self):
        K = len(self.cat_ids) if self.use_cats else 1
        T, R, A, M = len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(self.max_dets)
        precision, recall, scores = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M)), -np.ones((T, R, K, A, M))
        I0, A0 = len(self.img_ids), len(AREA_RNG)
        for k in range(K):
            for a in range(A):
                for m, max_det in enumerate(self.max_dets):
                    E = [self.eval_imgs[k * A0 * I0 + a * I0 + i] for i in range(I0)]
                    E = [e for e in E if e is not None]
                    if len(E) == 0:
                        continue
                    dt_scores = np.concatenate([e['dtScores'][0:max_det] for e in E])
                    inds = np.argsort(-dt_scores, kind='mergesort')
                    dt_scores_sorted = dt_scores[inds]
                    dtm = np.concatenate([e['dtMatches'][:, 0:max_det] for e in E], axis=1)[:, inds]
                    dt_ig = np.concatenate([e['dtIgnore'][:, 0:max_det] for e in E], axis=1)[:, inds]
                    gt_ig = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gt_ig == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dt_ig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        tp, fp = np.array(tp), np.array(fp)
                        nd = len(tp)
                        rc = tp / npig
                        pr = tp / (fp + tp + np.spacing(1))
                        q, ss = np.zeros((R,)), np.zeros((R,))
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        pr, q = pr.tolist(), q.tolist()
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        inds = np.searchsorted(rc, REC_THRS, side='left')
                        try:
                            for ri, pi in enumerate(inds):
                                q[ri] = pr[pi]
                                ss[ri] = dt_scores_sorted[pi]
                        except IndexError:
                            pass
                        precision[t, :, k, a, m] = np.array(q)
                        scores[t, :, k, a, m] = np.array(ss)
        self.precision, self.recall, self.scores = precision, recall, scores

    def summarize(self):
        md = self.max_dets

        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(AREA_RNG_LBL) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(md) if mDet == maxDets]
            s = self.precision if ap == 1 else self.recall
            if iouThr is not None:
                s = s[np.where(iouThr == IOU_THRS)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        st = np.zeros((12,))
        st[0] = _summarize(1)
        st[1] = _summarize(1, iouThr=.5, maxDets=md[2])
        st[2] = _summarize(1, iouThr=.75, maxDets=md[2])
        st[3] = _summarize(1, areaRng='small', maxDets=md[2])
        st[4] = _summarize(1, areaRng='medium', maxDets=md[2])
        st[5] = _summarize(1, areaRng='large', maxDets=md[2])
        st[6] = _summarize(0, maxDets=md[0])
        st[7] = _summarize(0, maxDets=md[1])
        st[8] = _summarize(0, maxDets=md[2])
        st[9] = _summarize(0, areaRng='small', maxDets=md[2])
        st[10] = _summarize(0, areaRng='medium', maxDets=md[2])
        st[11] = _summarize(0, areaRng='large', maxDets=md[2])
        self.stats = st
        return st


def run(gt, results, iou_type, img_ids=None, use_cats=1, cat_ids=None, max_dets=None, mask_cache=None):
    e = COCOevalParamsRef(gt, results, iou_type, img_ids, use_cats, cat_ids, max_dets, mask_cache)
    e.evaluate()
    e.accumulate()
    if len(e.max_dets) == 3:
        e.summarize()
    return e


# ---------------------------------------------------------------------------------------------------- known answers
def _gt(anns, cats=(1, 2)):
    return dict(images=[dict(id=1, height=40, width=40)], categories=[dict(id=c) for c in cats],
                annotations=[dict(id=i + 1, image_id=1, category_id=c, bbox=list(b), area=float(b[2] * b[3]), iscrowd=0,
                                  segmentation=[[b[0], b[1], b[0], b[1] + b[3], b[0] + b[2], b[1] + b[3], b[0] + b[2],
                                                 b[1]]])
                             for i, (c, b) in enumerate(anns)])


def _det(c, b, s):
    return dict(image_id=1, category_id=c, bbox=[float(v) for v in b], score=s)


def known_cases():
    """(name, gt, results, use_cats, cat_ids) of the hand-computed cases below."""
    g = [0, 0, 10, 10]
    return [
        ('wrong_category_1', _gt([(1, g)]), [_det(2, g, .9)], 1, None),
        ('wrong_category_0', _gt([(1, g)]), [_det(2, g, .9)], 0, None),
        ('tie_12', _gt([(1, g)]), [_det(1, [0, 0, 10, 6], .5), _det(2, [0, 0, 10, 9], .5)], 0, [1, 2]),
        ('tie_21', _gt([(1, g)]), [_det(1, [0, 0, 10, 6], .5), _det(2, [0, 0, 10, 9], .5)], 0, [2, 1]),
        ('gt_order_12', _gt([(1, g), (2, g)]), [_det(1, g, .7)], 0, [1, 2]),
        ('gt_order_21', _gt([(1, g), (2, g)]), [_det(1, g, .7)], 0, [2, 1]),
        ('absent_id', _gt([(1, g)]), [_det(1, g, .8), _det(5, g, .6)], 1, [5, 1]),
    ]


def test_restatement_known_answers():
    cases = {name: run(gt, dt, 'bbox', use_cats=u, cat_ids=c) for name, gt, dt, u, c in known_cases()}
    # a detection of another category: no match per category (cat 1 has a ground truth and no detection: recall 0,
    # precision 0; cat 2 has no ground truth: -1), a match of every threshold when pooled
    # (area ranges all and small hold the 10 x 10 ground truth; medium and large have none: -1)
    e = cases['wrong_category_1']
    assert e.precision.shape[2] == 2 and (e.recall[:, 0, :2] == 0).all() and (e.precision[:, :, 0, :2] == 0).all()
    assert (e.recall[:, 1] == -1).all() and (e.precision[:, :, 1] == -1).all() and (e.recall[:, :, 2:] == -1).all()
    e = cases['wrong_category_0']
    assert e.precision.shape[2] == 1 and (e.recall[:, :, :2] == 1).all() and np.allclose(e.precision[:, :, :, :2], 1, rtol=0, atol=1e-12)
    # equal scores across categories rank in catIds order: A (cat 1, IoU .6) before B (cat 2, IoU .9) for [1, 2]
    e = cases['tie_12'].eval_imgs[0]
    assert e['dtIds'] == [1, 2] and list(e['dtMatches'][0]) == [1, 0] and list(e['dtMatches'][5]) == [0, 1]
    e = cases['tie_21'].eval_imgs[0]
    assert e['dtIds'] == [2, 1] and list(e['dtMatches'][0]) == [1, 0] and list(e['dtMatches'][5]) == [1, 0]
    # ground truths concatenate in catIds order; of two equal IoUs the greedy loop keeps the later ground truth
    e = cases['gt_order_12'].eval_imgs[0]
    assert e['gtIds'] == [1, 2] and (e['dtMatches'] == 2).all()
    e = cases['gt_order_21'].eval_imgs[0]
    assert e['gtIds'] == [2, 1] and (e['dtMatches'] == 1).all()
    # an id no annotation has: its column is -1 even with results of it; K follows the sorted catIds
    e = cases['absent_id']
    assert e.cat_ids == [1, 5] and (e.precision[:, :, 1] == -1).all() and (e.recall[:, 1] == -1).all()
    assert np.allclose(e.precision[:, :, 0, :2], 1, rtol=0, atol=1e-12)


def test_restatement_default_params_equal_cocoeval_ref():
    import cocoeval_ref as R
    from test_cocoeval_host import known_cases as plain_cases
    for name, gt, dt in plain_cases():
        a, b = R.run(gt, dt, 'bbox'), run(gt, dt, 'bbox')
        for key in ('precision', 'recall', 'scores', 'stats'):
            assert np.array_equal(getattr(a, key), getattr(b, key)), (name, key)


def test_restatement_max_dets_cut():
    """maxDets [1, 2, 3]: the third detection of a (image, category) is cut by computeIoU, the second counts only at 2."""
    g = [0, 0, 10, 10]
    gt = _gt([(1, g), (1, [20, 20, 10, 10]), (1, [0, 20, 10, 10])])
    dt = [_det(1, g, .9), _det(1, [20, 20, 10, 10], .8), _det(1, [0, 20, 10, 10], .7)]
    e = run(gt, dt, 'bbox', max_dets=[1, 2, 2])
    assert np.allclose(e.recall[0, 0, 0], [1 / 3, 2 / 3, 2 / 3])
    e = run(gt, dt, 'bbox', max_dets=[1, 3, 1000])
    assert np.allclose(e.recall[0, 0, 0], [1 / 3, 1, 1])


# ---------------------------------------------------------------------------------------------------- Params
def test_params2_limits():
    from sipmask_b200 import cocoeval as C
    assert C.CocoParams2().shape == (10, 101, 4, 3) and C.CocoParams2().summarizable()
    assert C.CocoParams2(iou_thrs=[.5] * 16, area_rng=[[0, 1]] * 4, area_rng_lbl='abcd').shape == (16, 101, 4, 3)
    assert not C.CocoParams2(max_dets=[100]).summarizable()
    assert C.CocoParams2(max_dets=[1000, 100, 300]).max_dets == [100, 300, 1000]
    bad = [(dict(iou_thrs=[.5] * 17), 'T * A <= 64'), (dict(iou_thrs=[]), 'T * A'),
           (dict(area_rng=np.zeros((0, 2)), area_rng_lbl=[]), 'T * A'), (dict(max_dets=[1, 2, 3, 4]), '1 to 3'),
           (dict(max_dets=[]), '1 to 3'), (dict(max_dets=[1, 1001]), '[1, 1000]'), (dict(max_dets=[0]), '[1, 1000]'),
           (dict(max_dets=[1.5]), 'integers'), (dict(rec_thrs=np.zeros(102)), '1 to 101'),
           (dict(rec_thrs=[]), '1 to 101'), (dict(iou_thrs=[np.nan]), 'NaN'), (dict(area_rng=[[0, np.nan]]), 'NaN'),
           (dict(area_rng=[[0, 1], [1, 2]]), 'labels'), (dict(use_cats=2), 'useCats'), (dict(use_cats='0'), 'useCats'),
           (dict(cat_ids=[]), 'empty'), (dict(use_cats=0, cat_ids=[]), 'empty'),
           (dict(use_cats=0, cat_ids=[3, 1, 3]), 'repeats'), (dict(cat_ids=[1.5]), 'integers'),
           (dict(cat_ids=list(range(2049))), 'at most 2048')]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg.replace('*', r'\*').replace('[', r'\[')):
            C.CocoParams2(**kw)
    # CocoParams keeps its limits and points at CocoParams2
    for kw, msg in ((dict(max_dets=[1, 101]), r'\[1, 100\]'), (dict(use_cats=0), 'CocoParams2'),
                    (dict(cat_ids=[1]), 'CocoParams2')):
        with pytest.raises(ValueError, match=msg):
            C.CocoParams(**kw)


def test_params_categories():
    from sipmask_b200 import cocoeval as C
    gt_cats = [1, 2, 3, 7]
    for p in (C.CocoParams(), C.CocoParams2()):
        assert p.use_cats == 1 and p.cat_ids is None and not p.extended
        assert p.eval_cats(gt_cats) == gt_cats and p.cat_axis(gt_cats) == gt_cats
    assert isinstance(C.CocoParams2(), C.CocoParams)
    p = C.CocoParams2(cat_ids=[7, 3, 7, 99])                  # evaluate(): np.unique
    assert p.cat_ids == [3, 7, 99] and p.cat_axis(gt_cats) == [3, 7, 99] and not p.extended
    p = C.CocoParams2(use_cats=0, cat_ids=[7, 3, 99])          # the order given, K = 1
    assert p.eval_cats(gt_cats) == [7, 3, 99] and p.cat_axis(gt_cats) == [-1] and p.extended
    p = C.CocoParams2(use_cats=False)
    assert p.use_cats == 0 and p.eval_cats(gt_cats) == gt_cats and p.cat_axis(gt_cats) == [-1]
    assert C.CocoParams2(use_cats=True, max_dets=[100, 300, 1000]).extended
    assert not C.CocoParams2(max_dets=[100]).extended
    assert bytes(C.CocoParams2(max_dets=[5, 50]).c_struct()) == bytes(C.CocoParams(max_dets=[5, 50]).c_struct())


def test_ground_truth_subset():
    from sipmask_b200 import cocoeval as C
    gt = _gt([(1, [0, 0, 5, 5]), (2, [1, 1, 5, 5]), (1, [2, 2, 5, 5]), (4, [3, 3, 5, 5])])
    g = C.CocoGroundTruth(gt)
    assert [a['id'] for a in g.anns[1]] == [1, 2, 3]             # category 4 is not listed: not a default category
    v = g.subset([4, 2, 1])                                       # getAnnIds(catIds) keeps it
    rows, off, _ = v.image(1, masks=False)
    assert list(rows['id']) == [4, 2, 1, 3] and list(off) == [0, 1, 2, 4]
    assert v.cat_index == {4: 0, 2: 1, 1: 2} and g.cat_ids == [1, 2]
    rows, off, _ = g.subset([2]).image(1, masks=False)
    assert list(rows['id']) == [2] and list(off) == [0, 1]


def test_metric_names():
    from sipmask_b200 import cocoeval as C
    assert C.check_metrics(('bbox', 'segm', 'proposal')) == ['bbox', 'segm', 'proposal']
    with pytest.raises(ValueError, match='proposal_fast'):
        C.check_metrics(['bbox', 'proposal_fast'])
    with pytest.raises(ValueError, match='SipMask-benchmark'):
        C.check_metrics('proposal', benchmark=True)
    with pytest.raises(KeyError):
        C.check_metrics(['recall'])
    st = np.array([0] * 6 + [0.12345, 0.5, 0.75049, 0.1, 0.2, 0.3])
    assert C.proposal_results(st) == {'AR@100': 0.123, 'AR@300': 0.5, 'AR@1000': 0.75, 'AR_s@1000': 0.1,
                                      'AR_m@1000': 0.2, 'AR_l@1000': 0.3}


def test_params2_limits_at_the_abi():
    """smb_coco_params2_t is checked before any launch (no device needed); smb_coco_params_t keeps its limit of 100."""
    from sipmask_b200 import _lib as L, cocoeval as C
    lib = L.lib()
    p = C.CocoParams2(max_dets=[100, 300, 1000], use_cats=0).c_struct()
    assert ctypes.sizeof(p) == ctypes.sizeof(C._ParamsC) and p.use_cats == 0
    assert lib.smb_coco_params2_check(ctypes.byref(p)) == 0
    assert lib.smb_coco_match_params2_workspace_bytes(3, ctypes.byref(p)) > lib.smb_coco_match_workspace_bytes(3)
    for field, value in (('use_cats', 2), ('use_cats', -1), ('M', 4), ('T', 0)):
        q = C.CocoParams2(max_dets=[100, 300, 1000], use_cats=0).c_struct()
        setattr(q, field, value)
        assert lib.smb_coco_params2_check(ctypes.byref(q)) != 0, (field, value)
        assert lib.smb_coco_match_params2_workspace_bytes(3, ctypes.byref(q)) == 0
    q = C.CocoParams2(max_dets=[100, 300, 1000]).c_struct()
    q.max_dets[2] = 1001
    assert lib.smb_coco_params2_check(ctypes.byref(q)) != 0 and b'maxDet' in lib.smb_last_error()
    rc = lib.smb_coco_accumulate_params2_dev(None, ctypes.c_int64(0), None, 1, None, ctypes.byref(q), None, None, None,
                                             None)
    assert rc != 0
    q = C.CocoParams(max_dets=[100]).c_struct()                 # the old struct: maxDets in [1, 100]
    q.max_dets[0] = 101
    assert lib.smb_coco_params_check(ctypes.byref(q)) != 0
