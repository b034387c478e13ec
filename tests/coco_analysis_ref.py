"""Test restatement of pycocotools 2.0's COCOeval with its Params as instance attributes, and of SipMask-mmdetection's
tools/coco_error_analysis.py (analyze_results / analyze_individual_category), in plain Python and numpy.  Independent of
the library's kernels; the rasterizer and the IoU functions are cocoeval_ref's.  Like cocoeval_ref, a reading of the
sources, not a run of them (neither pycocotools nor matplotlib is available).
"""
import copy

import numpy as np

import cocoeval_ref as C


class COCOevalParams(C.COCOevalRef):
    """COCOeval(cocoGt, cocoDt, iouType) whose params.iouThrs / recThrs / maxDets / areaRng / areaRngLbl are set after
    construction, as a user of pycocotools sets them."""

    def __init__(self, gt, results, iou_type, img_ids=None, iou_thrs=None, rec_thrs=None, max_dets=None, area_rng=None,
                 area_rng_lbl=None):
        # cocoeval_ref's __init__ without loadRes' refusal of an empty list: the tool filters an already loaded result
        # set per category, which may leave it empty
        self.iou_type = iou_type
        self.imgs = {im['id']: im for im in gt['images']}
        self.img_ids = list(np.unique(img_ids if img_ids is not None else sorted(self.imgs)))
        self.cat_ids = sorted(c['id'] for c in gt['categories'])
        cats = set(self.cat_ids)
        gts, dts = {}, {}
        for a in gt['annotations']:
            if a['image_id'] in self.img_ids and a['category_id'] in cats:
                gts.setdefault((a['image_id'], a['category_id']), []).append(dict(a, ignore=int(bool(a['iscrowd']))))
        for n, r in enumerate(results):
            d = dict(r, id=n + 1)
            if iou_type == 'bbox':
                d['area'] = r['bbox'][2] * r['bbox'][3]
            else:
                im = self.imgs[r['image_id']]
                d['mask'] = C.ann_to_mask(r['segmentation'], im['height'], im['width'])
                d['area'] = int(d['mask'].sum())
            if r['image_id'] in self.img_ids and r['category_id'] in cats:
                dts.setdefault((r['image_id'], r['category_id']), []).append(d)
        if iou_type == 'segm':
            for (i, _), lst in gts.items():
                for g in lst:
                    g['mask'] = C.ann_to_mask(g['segmentation'], self.imgs[i]['height'], self.imgs[i]['width'])
        self._gts, self._dts = gts, dts
        self.iouThrs = C.IOU_THRS if iou_thrs is None else np.array(iou_thrs, dtype=np.float64)
        self.recThrs = C.REC_THRS if rec_thrs is None else np.array(rec_thrs, dtype=np.float64)
        self.maxDets = C.MAX_DETS if max_dets is None else list(max_dets)
        self.areaRng = C.AREA_RNG if area_rng is None else [list(r) for r in area_rng]
        self.areaRngLbl = C.AREA_RNG_LBL if area_rng_lbl is None else list(area_rng_lbl)

    def compute_iou(self, img, cat):
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds][:self.maxDets[-1]]
        out = np.zeros((len(dt), len(gt)))
        for a, d in enumerate(dt):
            for b, g in enumerate(gt):
                if self.iou_type == 'bbox':
                    out[a, b] = C.bb_iou([float(v) for v in d['bbox']], [float(v) for v in g['bbox']], g['iscrowd'])
                else:
                    out[a, b] = C.mask_iou(d['mask'], g['mask'], g['iscrowd'])
        return out

    def evaluate_img(self, img, cat, a_rng, max_det):
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return None
        for g in gt:
            g['_ignore'] = 1 if (g['ignore'] or (g['area'] < a_rng[0] or g['area'] > a_rng[1])) else 0
        gtind = np.argsort([g['_ignore'] for g in gt], kind='mergesort')
        gt = [gt[i] for i in gtind]
        dtind = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in dtind[0:max_det]]
        iscrowd = [int(o['iscrowd']) for o in gt]
        ious = self.ious[img, cat]
        ious = ious[:, gtind] if len(ious) > 0 else ious
        T, G, D = len(self.iouThrs), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        gt_ig = np.array([g['_ignore'] for g in gt])
        dt_ig = np.zeros((T, D))
        if len(ious) != 0:
            for tind, t in enumerate(self.iouThrs):
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
        return dict(dtMatches=dtm, gtIgnore=gt_ig, dtIgnore=dt_ig, dtScores=[d['score'] for d in dt])

    def evaluate(self):
        self.maxDets = sorted(self.maxDets)                   # COCOeval.evaluate: p.maxDets = sorted(p.maxDets)
        self.ious = {(i, c): self.compute_iou(i, c) for i in self.img_ids for c in self.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a, self.maxDets[-1])
                          for c in self.cat_ids for a in self.areaRng for i in self.img_ids]

    def accumulate(self):
        T, R, K, A, M = len(self.iouThrs), len(self.recThrs), len(self.cat_ids), len(self.areaRng), len(self.maxDets)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        I0, A0 = len(self.img_ids), len(self.areaRng)
        for k in range(K):
            Nk = k * A0 * I0
            for a in range(A):
                Na = a * I0
                for m, max_det in enumerate(self.maxDets):
                    E = [self.eval_imgs[Nk + Na + i] for i in range(I0)]
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
                        inds = np.searchsorted(rc, self.recThrs, side='left')
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
        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(self.areaRngLbl) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(self.maxDets) if mDet == maxDets]
            s = self.precision if ap == 1 else self.recall
            if iouThr is not None:
                s = s[np.where(iouThr == self.iouThrs)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        st = np.zeros((12,))
        md = self.maxDets
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


def run(gt, results, iou_type, img_ids=None, summarize=True, **params):
    e = COCOevalParams(gt, results, iou_type, img_ids, **params)
    e.evaluate()
    e.accumulate()
    if summarize:
        e.summarize()
    return e


# ---------------------------------------------------------------------------------------------------- coco_error_analysis
def _cats(gt):
    return {c['id']: c for c in gt['categories']}


def analyze_individual_category(k, results, gt, cat_id, iou_type):
    """analyze_individual_category: precision[0, :, k] of the Sim and the Oth evaluation of category cat_id."""
    cats = _cats(gt)
    nm = cats[cat_id]
    img_ids = [im['id'] for im in gt['images']]
    dt = [copy.deepcopy(r) for r in results if r['category_id'] == cat_id]
    out = {}
    # Sim: the other categories of cat_id's supercategory become crowd, ignored annotations of cat_id
    g = copy.deepcopy(gt)
    child = [c['id'] for c in g['categories'] if c['supercategory'] in [nm['supercategory']]]   # getCatIds(supNms)
    for ann in g['annotations']:
        if ann['category_id'] in child and ann['category_id'] != cat_id:
            ann['ignore'] = 1
            ann['iscrowd'] = 1
            ann['category_id'] = cat_id
    e = run(g, dt, iou_type, img_ids, summarize=False, max_dets=[100], iou_thrs=[.1])
    out['ps_supercategory'] = e.precision[0, :, k, :, :]
    # Oth: every other category
    g = copy.deepcopy(gt)
    for ann in g['annotations']:
        if ann['category_id'] != cat_id:
            ann['ignore'] = 1
            ann['iscrowd'] = 1
            ann['category_id'] = cat_id
    e = run(g, dt, iou_type, img_ids, summarize=False, max_dets=[100], iou_thrs=[.1])
    out['ps_allcategory'] = e.precision[0, :, k, :, :]
    return k, out


def analyze_results(gt, results, iou_type):
    """analyze_results' ps [7, R, K, 4, 1] of one result type (without the plots); K in the file's category order, which
    is p.catIds' order when the file lists its categories sorted by id."""
    img_ids = [im['id'] for im in gt['images']]
    e = run(copy.deepcopy(gt), copy.deepcopy(results), iou_type, img_ids, summarize=False, iou_thrs=[.75, .5, .1],
            max_dets=[100])
    ps = e.precision
    ps = np.vstack([ps, np.zeros((4, *ps.shape[1:]))])
    cat_ids = [c['id'] for c in gt['categories']]
    res = [analyze_individual_category(k, results, gt, c, iou_type) for k, c in enumerate(cat_ids)]
    for k, cat_id in enumerate(cat_ids):
        assert res[k][0] == k
        ps[3, :, k, :, :] = res[k][1]['ps_supercategory']
        ps[4, :, k, :, :] = res[k][1]['ps_allcategory']
        ps[ps == -1] = 0
        ps[5, :, k, :, :] = (ps[4, :, k, :, :] > 0)
        ps[6, :, k, :, :] = 1.0
    return ps
