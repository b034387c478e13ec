"""Test restatement of pycocotools 2.0's COCO / COCOeval for iouType 'bbox' and 'segm' with default Params, function by
function, in plain Python and numpy.  Independent of the library's C rasterizer and of its kernels: the device
evaluation (sipmask_b200.cocoeval) is checked against it.  pycocotools itself is not available, so this is a reading of
its source (coco.py, cocoeval.py, maskApi.c), not a run of it.
"""
import math

import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_RNG_LBL = ['all', 'small', 'medium', 'large']
INT_MIN = -2 ** 31


def _c_int(x):
    """C's (int) cast of a double on x86-64: truncation, NaN -> INT_MIN."""
    if math.isnan(x):
        return INT_MIN
    return int(x)


# ---------------------------------------------------------------------------------------------------- maskApi.c
def rle_fr_poly(xy, h, w):
    """rleFrPoly: upsample by 5, walk each edge, keep the x-boundary crossings, sort, difference, fold zero runs."""
    k = len(xy) // 2
    scale = 5.0
    x = [_c_int(scale * xy[2 * j] + .5) for j in range(k)]
    y = [_c_int(scale * xy[2 * j + 1] + .5) for j in range(k)]
    if k:
        x.append(x[0])
        y.append(y[0])
    u, v = [], []
    for j in range(k):
        xs, xe, ys, ye = x[j], x[j + 1], y[j], y[j + 1]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx >= dy:
            s = (ye - ys) / dx if dx else float('nan')        # 0/0 = NaN in C
            for d in range(dx + 1):
                t = dx - d if flip else d
                u.append(t + xs)
                v.append(_c_int(ys + s * t + .5))
        else:
            s = (xe - xs) / dy
            for d in range(dy + 1):
                t = dy - d if flip else d
                v.append(t + ys)
                u.append(_c_int(xs + s * t + .5))
    a = []
    for j in range(1, len(u)):
        if u[j] == u[j - 1]:
            continue
        xd = float(u[j] if u[j] < u[j - 1] else u[j] - 1)
        xd = (xd + .5) / scale - .5
        if math.floor(xd) != xd or xd < 0 or xd > w - 1:
            continue
        yd = float(v[j] if v[j] < v[j - 1] else v[j - 1])
        yd = (yd + .5) / scale - .5
        if yd < 0:
            yd = 0
        elif yd > h:
            yd = h
        yd = math.ceil(yd)
        a.append(int(xd) * h + int(yd))
    a.append(h * w)
    a.sort()
    p = 0
    for j in range(len(a)):
        t = a[j]
        a[j] -= p
        p = t
    b = [a[0]]
    j = 1
    while j < len(a):
        if a[j] > 0:
            b.append(a[j])
            j += 1
        else:
            j += 1
            if j < len(a):
                b[-1] += a[j]
                j += 1
    return b


def rle_fr_string(s):
    """rleFrString."""
    if isinstance(s, str):
        s = s.encode()
    cnts, p = [], 0
    while p < len(s):
        x, k, more = 0, 0, 1
        while more:
            c = s[p] - 48
            x |= (c & 0x1f) << 5 * k
            more = c & 0x20
            p += 1
            k += 1
            if not more and (c & 0x10):
                x |= -1 << 5 * k
        if len(cnts) > 2:
            x += cnts[-2]
        cnts.append(x)
    return cnts


def counts_to_mask(cnts, h, w):
    flat = np.zeros(h * w, bool)
    pos = 0
    for i, c in enumerate(cnts):
        if i & 1:
            flat[pos:pos + c] = True
        pos += c
    assert pos == h * w, (pos, h, w)
    return flat.reshape(w, h).T


def ann_to_mask(segm, h, w):
    """COCO.annToRLE then decode: polygons (frPyObjects + merge; a first element of 4 numbers = frBbox), uncompressed
    or compressed RLE."""
    if isinstance(segm, list):
        if len(segm[0]) == 4:
            polys = [[b[0], b[1], b[0], b[1] + b[3], b[0] + b[2], b[1] + b[3], b[0] + b[2], b[1]] for b in segm]
        else:
            polys = segm
        m = np.zeros((h, w), bool)
        for p in polys:
            m |= counts_to_mask(rle_fr_poly([float(v) for v in p], h, w), h, w)
        return m
    assert list(segm['size']) == [h, w]
    c = segm['counts']
    return counts_to_mask(c if isinstance(c, list) else rle_fr_string(c), h, w)


def bb_iou(d, g, crowd):
    da, ga = d[2] * d[3], g[2] * g[3]
    w = min(d[2] + d[0], g[2] + g[0]) - max(d[0], g[0])
    if w <= 0:
        return 0.0
    h = min(d[3] + d[1], g[3] + g[1]) - max(d[1], g[1])
    if h <= 0:
        return 0.0
    i = w * h
    u = da if crowd else da + ga - i
    return i / u


def mask_iou(dm, gm, crowd):
    i = int(np.logical_and(dm, gm).sum())
    if i == 0:
        return 0.0
    u = int(dm.sum()) if crowd else int(dm.sum()) + int(gm.sum()) - i
    return float(i) / float(u)


# ---------------------------------------------------------------------------------------------------- cocoeval.py
class COCOevalRef:
    """COCOeval(cocoGt, cocoDt, iouType) with params.imgIds = img_ids; results = the loadRes list."""

    def __init__(self, gt, results, iou_type, img_ids=None):
        assert len(results) > 0                       # loadRes indexes anns[0]
        self.iou_type = iou_type
        self.imgs = {im['id']: im for im in gt['images']}
        self.img_ids = list(np.unique(img_ids if img_ids is not None else sorted(self.imgs)))
        self.cat_ids = sorted(c['id'] for c in gt['categories'])
        cats = set(self.cat_ids)
        gts, dts = {}, {}
        for a in gt['annotations']:                   # getAnnIds(imgIds, catIds): imgToAnns order
            if a['image_id'] in self.img_ids and a['category_id'] in cats:
                gts.setdefault((a['image_id'], a['category_id']), []).append(dict(a, ignore=int(bool(a['iscrowd']))))
        for n, r in enumerate(results):               # loadRes: id = n + 1, area
            d = dict(r, id=n + 1)
            if iou_type == 'bbox':
                d['area'] = r['bbox'][2] * r['bbox'][3]
            else:
                im = self.imgs[r['image_id']]
                d['mask'] = ann_to_mask(r['segmentation'], im['height'], im['width'])
                d['area'] = int(d['mask'].sum())
            if r['image_id'] in self.img_ids and r['category_id'] in cats:
                dts.setdefault((r['image_id'], r['category_id']), []).append(d)
        if iou_type == 'segm':
            for (i, _), lst in gts.items():
                for g in lst:
                    g['mask'] = ann_to_mask(g['segmentation'], self.imgs[i]['height'], self.imgs[i]['width'])
        self._gts, self._dts = gts, dts

    def compute_iou(self, img, cat):
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if len(gt) == 0 and len(dt) == 0:
            return []
        inds = np.argsort([-d['score'] for d in dt], kind='mergesort')
        dt = [dt[i] for i in inds][:MAX_DETS[-1]]
        out = np.zeros((len(dt), len(gt)))
        for a, d in enumerate(dt):
            for b, g in enumerate(gt):
                if self.iou_type == 'bbox':
                    out[a, b] = bb_iou([float(v) for v in d['bbox']], [float(v) for v in g['bbox']], g['iscrowd'])
                else:
                    out[a, b] = mask_iou(d['mask'], g['mask'], g['iscrowd'])
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
        T, G, D = len(IOU_THRS), len(gt), len(dt)
        gtm, dtm = np.zeros((T, G)), np.zeros((T, D))
        gt_ig = np.array([g['_ignore'] for g in gt])
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
        return dict(dtMatches=dtm, gtIgnore=gt_ig, dtIgnore=dt_ig, dtScores=[d['score'] for d in dt])

    def evaluate(self):
        self.ious = {(i, c): self.compute_iou(i, c) for i in self.img_ids for c in self.cat_ids}
        self.eval_imgs = [self.evaluate_img(i, c, a, MAX_DETS[-1])
                          for c in self.cat_ids for a in AREA_RNG for i in self.img_ids]

    def accumulate(self):
        T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(self.cat_ids), len(AREA_RNG), len(MAX_DETS)
        precision = -np.ones((T, R, K, A, M))
        recall = -np.ones((T, K, A, M))
        scores = -np.ones((T, R, K, A, M))
        I0, A0 = len(self.img_ids), len(AREA_RNG)
        for k in range(K):
            Nk = k * A0 * I0
            for a in range(A):
                Na = a * I0
                for m, max_det in enumerate(MAX_DETS):
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
        def _summarize(ap=1, iouThr=None, areaRng='all', maxDets=100):
            aind = [i for i, aRng in enumerate(AREA_RNG_LBL) if aRng == areaRng]
            mind = [i for i, mDet in enumerate(MAX_DETS) if mDet == maxDets]
            s = self.precision if ap == 1 else self.recall
            if iouThr is not None:
                s = s[np.where(iouThr == IOU_THRS)[0]]
            s = s[:, :, :, aind, mind] if ap == 1 else s[:, :, aind, mind]
            return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        st = np.zeros((12,))
        st[0] = _summarize(1)
        st[1] = _summarize(1, iouThr=.5, maxDets=100)
        st[2] = _summarize(1, iouThr=.75, maxDets=100)
        st[3] = _summarize(1, areaRng='small', maxDets=100)
        st[4] = _summarize(1, areaRng='medium', maxDets=100)
        st[5] = _summarize(1, areaRng='large', maxDets=100)
        st[6] = _summarize(0, maxDets=1)
        st[7] = _summarize(0, maxDets=10)
        st[8] = _summarize(0, maxDets=100)
        st[9] = _summarize(0, areaRng='small', maxDets=100)
        st[10] = _summarize(0, areaRng='medium', maxDets=100)
        st[11] = _summarize(0, areaRng='large', maxDets=100)
        self.stats = st
        return st


def run(gt, results, iou_type, img_ids=None):
    e = COCOevalRef(gt, results, iou_type, img_ids)
    e.evaluate()
    e.accumulate()
    e.summarize()
    return e
