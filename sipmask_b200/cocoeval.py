"""COCO box and mask AP on the device: pycocotools 2.0 COCOeval (iouType 'bbox' / 'segm') as MM's CocoDataset.evaluate
(SipMask-mmdetection/mmdet/datasets/coco.py:290-392) and SipMask-benchmark's coco_eval.py run it, with the default Params
or user-given ones (CocoParams: IoU thresholds, recall thresholds, maxDets and area ranges as data; CocoParams2: also
useCats, catIds and maxDets up to 1000), and MM's class-agnostic 'proposal' metric.

Host: the ground truth (CocoGroundTruth: pycocotools COCO's indexing; annToRLE through the library's C restatement of
rleFrPoly / rleFrString as the public host rasterizer, segm_plane) and summarize (numpy, the code of COCOeval.summarize).
Device: the masks of ground truth and result files (csrc/segm_raster.cu, from packed vertices and run lengths), the result
json's values from the engine record, computeIoU + evaluateImg for every (image, category) after every batch, and
accumulate's precision / recall / scores arrays at evaluate() (csrc/cocoeval.cu).

Restated only: pycocotools is neither vendored in the reference nor installed where this was written, so the semantics
are pycocotools 2.0's as read from its source, not pinned by running it.
"""
import copy
import ctypes

import numpy as np
import torch

from . import _lib as L

DET_DTYPE = np.dtype([('box', '<f8', (4,)), ('score', '<f8', (2,)), ('area_box', '<f8'), ('plane', '<i8'),
                      ('area_mask', '<i4'), ('cat', '<i4'), ('ext', '<i4', (4,)), ('order', '<i4'), ('pad', '<i4')])
GT_DTYPE = np.dtype([('box', '<f8', (4,)), ('area', '<f8'), ('plane', '<i8'), ('id', '<i8'), ('crowd', '<i4'),
                     ('area_mask', '<i4'), ('ext', '<i4', (4,))])
IMG_DTYPE = np.dtype([('h', '<i4'), ('w', '<i4'), ('det_pitch', '<i4'), ('gt_pitch', '<i4'), ('n_det', '<i4'),
                      ('pad', '<i4'), ('image_id', '<i8'), ('out_off', '<i8')])
OUT_DTYPE = np.dtype([('score', '<f8'), ('image_id', '<i8'), ('matched', '<u8'), ('ignored', '<u8'), ('cat', '<i4'),
                      ('rank', '<i4')])
assert (DET_DTYPE.itemsize, GT_DTYPE.itemsize, IMG_DTYPE.itemsize, OUT_DTYPE.itemsize) == (96, 80, 40, 40)

# COCOeval Params (iouType 'segm' / 'bbox'), as float64 data
IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_RNG_LBL = ['all', 'small', 'medium', 'large']
METRIC_ITEMS = ['mAP', 'mAP_50', 'mAP_75', 'mAP_s', 'mAP_m', 'mAP_l']
DET_CAP = 4096                       # SMB_COCO_DET_CAP: detections of one image in one launch
MAX_CATS = 2048                      # SMB_COCO_MAX_CATS
LABEL_RANGE, CAPACITY, ANALYSIS_RANGE = 1, 2, 4   # status bits
MAX_TA, MAX_M, MAX_DET = 64, 3, 100  # SMB_COCO_MAX_TA, SMB_COCO_MAX_M, SMB_COCO_MAX_DET
MAX_DET2 = 1000                      # SMB_COCO_MAX_DET2: maxDets through the Params2 entry points
PROPOSAL_NUMS = (100, 300, 1000)     # CocoDataset.evaluate's default proposal_nums
PROPOSAL_ITEMS = ['AR@100', 'AR@300', 'AR@1000', 'AR_s@1000', 'AR_m@1000', 'AR_l@1000']


class _ParamsC(ctypes.Structure):
    """smb_coco_params_t (include/sipmask_b200.h)."""
    _fields_ = [('T', ctypes.c_int32), ('A', ctypes.c_int32), ('M', ctypes.c_int32), ('R', ctypes.c_int32),
                ('max_dets', ctypes.c_int32 * MAX_M), ('pad', ctypes.c_int32), ('iou_thr', ctypes.c_double * MAX_TA),
                ('area_rng', ctypes.c_double * (2 * MAX_TA)), ('rec_thr', ctypes.c_double * 101)]


class _Params2C(ctypes.Structure):
    """smb_coco_params2_t (include/sipmask_b200.h): smb_coco_params_t with use_cats in place of its padding."""
    _fields_ = [('T', ctypes.c_int32), ('A', ctypes.c_int32), ('M', ctypes.c_int32), ('R', ctypes.c_int32),
                ('max_dets', ctypes.c_int32 * MAX_M), ('use_cats', ctypes.c_int32),
                ('iou_thr', ctypes.c_double * MAX_TA), ('area_rng', ctypes.c_double * (2 * MAX_TA)),
                ('rec_thr', ctypes.c_double * 101)]


class CocoParams:
    """COCOeval's Params as data: iouThrs, recThrs, maxDets, areaRng and areaRngLbl (default: COCOeval's, iouType 'bbox'
    / 'segm').  Thresholds and area ranges keep the order given, as pycocotools keeps them; maxDets are sorted, as
    COCOeval.evaluate() sorts them (p.maxDets = sorted(p.maxDets)) before anything reads them.  Limits, each a ValueError
    here:
      1 <= T (IoU thresholds), 1 <= A (area ranges), T * A <= 64: a detection's matched / ignored bits are one uint64;
      1 <= M <= 3 maxDets, each an integer in [1, 100]; 1 <= R <= 101 recall thresholds; no NaN;
      one label per area range.
    Not supported here: useCats = 0, catIds subsets and maxDets above 100 (every category of the ground truth is
    evaluated); CocoParams2 takes them."""
    _MAX_DET = MAX_DET

    def __init__(self, iou_thrs=None, rec_thrs=None, max_dets=None, area_rng=None, area_rng_lbl=None, use_cats=1,
                 cat_ids=None):
        if use_cats != 1:
            raise ValueError('CocoParams: useCats = 0 is not supported (categories are always used; CocoParams2 '
                             'takes it)')
        if cat_ids is not None:
            raise ValueError('CocoParams: catIds subsets are not supported (every ground-truth category is evaluated; '
                             'CocoParams2 takes them)')
        self.use_cats, self.cat_ids = 1, None
        self._set(iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl)

    def _set(self, iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl):
        name = type(self).__name__
        self.iou_thrs = self._floats(IOU_THRS if iou_thrs is None else iou_thrs, 'iou_thrs')
        self.rec_thrs = self._floats(REC_THRS if rec_thrs is None else rec_thrs, 'rec_thrs')
        self.area_rng = self._floats(AREA_RNG if area_rng is None else area_rng, 'area_rng', (-1, 2))
        self.area_rng_lbl = list(AREA_RNG_LBL if area_rng_lbl is None else area_rng_lbl)
        md = list(MAX_DETS if max_dets is None else max_dets)
        if not all(isinstance(m, (int, np.integer)) and not isinstance(m, bool) for m in md):
            raise ValueError('%s: maxDets must be integers, got %r' % (name, md))
        self.max_dets = sorted(int(m) for m in md)
        T, A, M, R = len(self.iou_thrs), len(self.area_rng), len(self.max_dets), len(self.rec_thrs)
        if T < 1 or A < 1 or T * A > MAX_TA:
            raise ValueError('%s: %d IoU thresholds x %d area ranges; need 1 <= T, 1 <= A and T * A <= %d '
                             '(the matched / ignored bits of a detection are one uint64)' % (name, T, A, MAX_TA))
        if not 1 <= M <= MAX_M:
            raise ValueError('%s: %d maxDets; 1 to %d are supported' % (name, M, MAX_M))
        if any(not 1 <= m <= self._MAX_DET for m in self.max_dets):
            raise ValueError('%s: maxDets %r; each must be in [1, %d]' % (name, self.max_dets, self._MAX_DET))
        if not 1 <= R <= 101:
            raise ValueError('%s: %d recall thresholds; 1 to 101 are supported' % (name, R))
        if len(self.area_rng_lbl) != A:
            raise ValueError('%s: %d area range labels for %d area ranges' % (name, len(self.area_rng_lbl), A))

    @staticmethod
    def _floats(v, name, shape=(-1,)):
        try:
            a = np.array(v, dtype=np.float64).reshape(shape)
        except (TypeError, ValueError) as e:
            raise ValueError('CocoParams: %s: %s' % (name, e))
        if np.isnan(a).any():
            raise ValueError('CocoParams: %s has a NaN' % name)
        return np.ascontiguousarray(a)

    @property
    def shape(self):
        """(T, R, A, M): precision / scores are [T, R, K, A, M], recall [T, K, A, M]."""
        return len(self.iou_thrs), len(self.rec_thrs), len(self.area_rng), len(self.max_dets)

    @property
    def extended(self):
        """Whether these Params need the Params2 entry points (useCats = 0 or a maxDet above 100)."""
        return self.use_cats == 0 or self.max_dets[-1] > MAX_DET

    def eval_cats(self, gt_cat_ids):
        """The category ids evaluated against a ground truth whose categories are gt_cat_ids (sorted), in the order of
        their category index on the device: cat_ids as normalized here, or the ground truth's."""
        return list(gt_cat_ids) if self.cat_ids is None else list(self.cat_ids)

    def cat_axis(self, gt_cat_ids):
        """The category ids along K of precision / recall / scores: eval_cats with useCats 1, [-1] with useCats 0 (as
        accumulate sets p.catIds)."""
        return self.eval_cats(gt_cat_ids) if self.use_cats else [-1]

    def summarizable(self):
        """Whether COCOeval.summarize runs on these Params: three maxDets and the labels all / small / medium / large."""
        return len(self.max_dets) == 3 and all(l in self.area_rng_lbl for l in AREA_RNG_LBL)

    def c_struct(self):
        T, R, A, M = self.shape
        p = _Params2C(T=T, A=A, M=M, R=R, use_cats=self.use_cats) if self.extended else _ParamsC(T=T, A=A, M=M, R=R)
        p.max_dets[:M] = self.max_dets
        p.iou_thr[:T] = self.iou_thrs.tolist()
        p.area_rng[:2 * A] = self.area_rng.reshape(-1).tolist()
        p.rec_thr[:R] = self.rec_thrs.tolist()
        return p


class CocoParams2(CocoParams):
    """CocoParams plus p.useCats, p.catIds and maxDets up to 1000 (smb_coco_params2_t where needed).
      use_cats 1: one evaluation per category of cat_ids (None: every ground-truth category), sorted and de-duplicated
                  as evaluate() does (p.catIds = list(np.unique(p.catIds))); the K axis of the arrays is that list.
                  An id no ground-truth annotation has gets a column of -1.
      use_cats 0: one pooled evaluation per image over the ground truth and results of cat_ids (None: every
                  ground-truth category, sorted), concatenated in the order given (computeIoU / evaluateImg); K = 1.
                  pycocotools would repeat a repeated id's annotations, so duplicates are refused.
    Results and annotations of other categories are not evaluated.  Limits: CocoParams', except each maxDet in
    [1, 1000]; use_cats 0 or 1; cat_ids non-empty, at most 2048 ids.  With use_cats 1, no cat_ids and maxDets up to 100
    these Params compute what the same CocoParams compute, through the same entry points."""
    _MAX_DET = MAX_DET2

    def __init__(self, iou_thrs=None, rec_thrs=None, max_dets=None, area_rng=None, area_rng_lbl=None, use_cats=1,
                 cat_ids=None):
        if isinstance(use_cats, (bool, np.bool_)) or (isinstance(use_cats, (int, np.integer)) and use_cats in (0, 1)):
            self.use_cats = int(use_cats)
        else:
            raise ValueError('CocoParams2: useCats must be 0 or 1, got %r' % (use_cats,))
        self.cat_ids = None
        if cat_ids is not None:
            ids = list(cat_ids)
            if not all(isinstance(c, (int, np.integer)) and not isinstance(c, bool) for c in ids):
                raise ValueError('CocoParams2: catIds must be integers, got %r' % (ids[:8],))
            ids = [int(c) for c in ids]
            if not ids:
                raise ValueError('CocoParams2: catIds is empty')
            if self.use_cats:
                ids = sorted(set(ids))                                # evaluate(): list(np.unique(p.catIds))
            elif len(set(ids)) != len(ids):
                raise ValueError('CocoParams2: catIds %r repeats an id; with useCats = 0 pycocotools would evaluate '
                                 'its annotations twice' % (ids[:8],))
            if len(ids) > MAX_CATS:
                raise ValueError('CocoParams2: %d catIds; at most %d' % (len(ids), MAX_CATS))
            self.cat_ids = ids
        self._set(iou_thrs, rec_thrs, max_dets, area_rng, area_rng_lbl)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


# ---------------------------------------------------------------------------------------------------- host RLE / masks
def string_to_counts(s):
    """pycocotools rleFrString: a compressed counts string (str or bytes) -> uint32 run lengths."""
    b = s.encode() if isinstance(s, str) else bytes(s)
    out = np.zeros(len(b) + 1, np.uint32)                   # every count takes at least one character
    n = ctypes.c_int(0)
    if L.lib().smb_coco_rle_from_string(b, len(b), _ptr(out), out.size, ctypes.byref(n)) != 0:
        raise ValueError('malformed RLE string: %s' % L.lib().smb_last_error().decode())
    return out[:n.value]


def poly_counts(xy, h, w):
    """rleFrPoly's run lengths of one polygon [x0, y0, x1, y1, ...] in an h x w canvas (the C restatement)."""
    xy = np.asarray(xy, dtype=np.float64).reshape(-1)
    xy = np.ascontiguousarray(xy[:xy.size // 2 * 2])
    k, n = xy.size // 2, ctypes.c_int(0)
    L.check(L.lib().smb_coco_poly_counts(_ptr(xy), k, int(h), int(w), None, 0, ctypes.byref(n)), 'smb_coco_poly_counts')
    out = np.zeros(max(n.value, 1), np.uint32)
    L.check(L.lib().smb_coco_poly_counts(_ptr(xy), k, int(h), int(w), _ptr(out), out.size, ctypes.byref(n)),
            'smb_coco_poly_counts')
    return out[:n.value]


def _check_size(rle, h, w, what):
    size = rle.get('size')
    if not isinstance(size, (list, tuple)) or len(size) != 2 or [int(size[0]), int(size[1])] != [h, w]:
        raise ValueError('%s: RLE size %r differs from the image canvas %dx%d' % (what, size, h, w))


def _or_counts(plane, cnts, h, w, what):
    cnts = np.ascontiguousarray(np.asarray(cnts, dtype=np.int64))
    if cnts.ndim != 1 or (cnts.size and (cnts.min() < 0 or cnts.max() > 0xffffffff)):
        raise ValueError('%s: run lengths must be a list of non-negative integers' % what)
    c = cnts.astype(np.uint32)
    if L.lib().smb_coco_rle_to_bits(_ptr(c), c.size, h, w, _ptr(plane), plane.shape[1]) != 0:
        raise ValueError('%s: %s' % (what, L.lib().smb_last_error().decode()))


def segm_plane(segm, h, w, what='segmentation'):
    """COCO.annToRLE of a ground-truth segmentation, as a bit plane [h, ceil(w / 32)] uint32: polygons (frPyObjects + merge,
    a first element of exactly 4 numbers makes every element a box, frBbox), an uncompressed RLE, or a compressed one."""
    pitch = (w + 31) // 32
    plane = np.zeros((h, pitch), np.uint32)
    lib = L.lib()
    if isinstance(segm, list):
        if len(segm) == 0 or not isinstance(segm[0], (list, tuple)):
            raise ValueError('%s: a polygon list needs lists of coordinates' % what)
        n0 = len(segm[0])
        if n0 == 4:                                           # frBbox: [x, y, x, y+h, x+w, y+h, x+w, y]
            polys = []
            for bb in segm:
                if len(bb) != 4:
                    raise ValueError('%s: boxes must have 4 numbers' % what)
                x, y, bw, bh = [float(v) for v in bb]
                xe, ye = x + bw, y + bh
                polys.append([x, y, x, ye, xe, ye, xe, y])
        elif n0 > 4:
            polys = [[float(v) for v in p] for p in segm]
        else:
            raise ValueError('%s: input type is not supported (a polygon of %d numbers)' % (what, n0))
        for p in polys:
            xy = np.ascontiguousarray(np.asarray(p, dtype=np.float64)[:len(p) // 2 * 2])
            L.check(lib.smb_coco_poly_to_bits(_ptr(xy), xy.size // 2, h, w, _ptr(plane), pitch), 'smb_coco_poly_to_bits')
        return plane
    if not isinstance(segm, dict) or 'counts' not in segm or 'size' not in segm:
        raise ValueError('%s: not a polygon list or an RLE dict' % what)
    _check_size(segm, h, w, what)
    counts = segm['counts']
    if isinstance(counts, list):
        _or_counts(plane, counts, h, w, what)
    elif isinstance(counts, (str, bytes)):
        _or_counts(plane, string_to_counts(counts), h, w, what)
    else:
        raise ValueError('%s: counts must be a list or a string' % what)
    return plane


def plane_stats(plane, w):
    s = np.zeros(5, np.int32)
    p = np.ascontiguousarray(plane, dtype=np.uint32)
    L.check(L.lib().smb_coco_plane_stats(_ptr(p), p.shape[0], int(w), p.shape[1], _ptr(s)), 'smb_coco_plane_stats')
    return int(s[0]), s[1:].copy()


# ---------------------------------------------------------------------------------------------------- ground truth
class CocoGroundTruth:
    """A loaded COCO annotation json, indexed as pycocotools' COCO and COCOeval._prepare see it.
      img_ids : sorted unique image ids (COCOeval.evaluate: np.unique(p.imgIds))
      cat_ids : sorted category ids (p.catIds = sorted(getCatIds()))
      names / supercategories: per sorted category, its 'name' and 'supercategory' (None where the file has none)
    Per image, its annotations of those categories in annotation-file order (imgToAnns)."""

    def __init__(self, ann_dict):
        try:
            images, cats, anns = ann_dict['images'], ann_dict['categories'], ann_dict['annotations']
            self.hw = {int(im['id']): (int(im['height']), int(im['width'])) for im in images}
            self.cat_ids = sorted(int(c['id']) for c in cats)
            info = {int(c['id']): c for c in cats}
        except (KeyError, TypeError, ValueError) as e:
            raise ValueError('CocoGroundTruth: malformed images / categories: %r' % (e,))
        if len(set(self.cat_ids)) != len(self.cat_ids) or not 0 < len(self.cat_ids) <= MAX_CATS:
            raise ValueError('CocoGroundTruth: need 1..%d distinct category ids' % MAX_CATS)
        self.img_ids = sorted(self.hw)
        self.cat_index = {c: i for i, c in enumerate(self.cat_ids)}
        self.names = [str(info[c].get('name', c)) for c in self.cat_ids]
        self.supercategories = [info[c].get('supercategory') for c in self.cat_ids]
        self.anns = {i: [] for i in self.img_ids}
        self._all_anns = {i: [] for i in self.img_ids}       # imgToAnns, whatever the category (subset() filters it)
        for a in anns:
            try:
                img, cat = int(a['image_id']), int(a['category_id'])
                bbox = [float(v) for v in a['bbox']]
                row = dict(id=int(a['id']), cat=cat, bbox=bbox, area=float(a['area']), iscrowd=int(a['iscrowd']),
                           segmentation=a.get('segmentation'))
            except (KeyError, TypeError, ValueError) as e:
                raise ValueError('CocoGroundTruth: malformed annotation %r: %r' % (a.get('id') if isinstance(a, dict) else a, e))
            if len(bbox) != 4:
                raise ValueError('CocoGroundTruth: annotation %d: bbox needs 4 numbers' % row['id'])
            if img in self.anns and cat in self.cat_index:        # getAnnIds(imgIds=p.imgIds, catIds=p.catIds)
                self.anns[img].append(row)
            if img in self._all_anns:
                self._all_anns[img].append(row)

    def subset(self, cat_ids):
        """The ground truth as COCOeval indexes it with p.catIds = cat_ids: the same images, category index = position in
        cat_ids (in the order given), and per image its annotations of those ids in file order (getAnnIds(imgIds,
        catIds), which also keeps an id the file's categories do not list).  Rows of image() are then category-major in
        that order, which is the order useCats = 0 concatenates them in."""
        v = copy.copy(self)
        v.cat_ids = [int(c) for c in cat_ids]
        v.cat_index = {c: i for i, c in enumerate(v.cat_ids)}
        info = dict(zip(self.cat_ids, zip(self.names, self.supercategories)))
        v.names = [info[c][0] if c in info else str(c) for c in v.cat_ids]
        v.supercategories = [info[c][1] if c in info else None for c in v.cat_ids]
        v.anns = {i: [a for a in self._all_anns[i] if a['cat'] in v.cat_index] for i in self.img_ids}
        return v

    def image(self, img_id, masks=True):
        """One image's ground truth for a match launch: (rows GT_DTYPE, per-category offsets [K+1], planes [G, h, pitch]
        or None).  Rows are grouped by category index, annotation order inside a category."""
        h, w = self.hw[img_id]
        anns = self.anns[img_id]
        K = len(self.cat_ids)
        order = sorted(range(len(anns)), key=lambda i: self.cat_index[anns[i]['cat']])      # stable
        rows = np.zeros(len(anns), GT_DTYPE)
        pitch = (w + 31) // 32
        planes = np.zeros((len(anns), h, pitch), np.uint32) if masks else None
        cnt = np.zeros(K + 1, np.int32)
        for r, i in enumerate(order):
            a = anns[i]
            rows[r]['box'] = a['bbox']
            rows[r]['area'] = a['area']
            rows[r]['id'] = a['id']
            rows[r]['crowd'] = a['iscrowd']
            cnt[self.cat_index[a['cat']] + 1] += 1
            if masks:
                if a['segmentation'] is None:
                    raise ValueError('CocoGroundTruth: annotation %d has no segmentation' % a['id'])
                planes[r] = segm_plane(a['segmentation'], h, w, 'annotation %d' % a['id'])
                area, ext = plane_stats(planes[r], w)
                rows[r]['area_mask'] = area
                rows[r]['ext'] = ext
        return rows, np.cumsum(cnt).astype(np.int32), planes

    def positions(self, img_id):
        """[G] int32: the position of image()'s row r in the image's annotation order."""
        anns = self.anns[img_id]
        return np.array(sorted(range(len(anns)), key=lambda i: self.cat_index[anns[i]['cat']]), np.int32)

    def supercategory_index(self):
        """[K] int32 index of each category's supercategory (numbered by first appearance) and the number of them.
        Raises ValueError when a category has none (the error analysis' Sim evaluation groups categories by it)."""
        missing = [c for c, s in zip(self.cat_ids, self.supercategories) if s is None]
        if missing:
            raise ValueError('CocoGroundTruth: categories %r have no supercategory' % missing[:8])
        index = {}
        for s in self.supercategories:
            index.setdefault(s, len(index))
        return np.array([index[s] for s in self.supercategories], np.int32), len(index)

    def packed(self, img_id):
        """image()'s rows and offsets with the segmentations packed for the device rasterizer instead of rasterized:
        (rows with area_mask / ext left zero, per-category offsets [K+1], segm_raster.SegmPack with row r's
        segmentation in plane r).  Raises what image() raises, from the numbers alone."""
        from .segm_raster import SegmPack
        rows, off, _ = self.image(img_id, masks=False)
        h, w = self.hw[img_id]
        anns = self.anns[img_id]
        pack = SegmPack()
        for r, i in enumerate(sorted(range(len(anns)), key=lambda i: self.cat_index[anns[i]['cat']])):
            a = anns[i]
            if a['segmentation'] is None:
                raise ValueError('CocoGroundTruth: annotation %d has no segmentation' % a['id'])
            pack.add(a['segmentation'], h, w, r, 'annotation %d' % a['id'])
        return rows, off, pack


# ---------------------------------------------------------------------------------------------------- summarize (host)
def summarize(precision, recall, area_rng_lbl=AREA_RNG_LBL, max_dets=MAX_DETS, iou_thrs=IOU_THRS):
    """COCOeval.summarize's 12 stats of the accumulated arrays (its _summarize / _summarizeDets code).  area_rng_lbl /
    max_dets / iou_thrs: the Params' areaRngLbl, maxDets and iouThrs (YTVOSeval keeps COCO's labels for its own ranges);
    a stat whose IoU threshold, range label or maxDet the Params lack is -1, as in pycocotools."""
    iouThrs, maxDets, areaRngLbl = np.asarray(iou_thrs, dtype=np.float64), list(max_dets), list(area_rng_lbl)

    def _summarize(ap=1, iouThr=None, areaRng='all', maxDets_=100):
        aind = [i for i, aRng in enumerate(areaRngLbl) if aRng == areaRng]
        mind = [i for i, mDet in enumerate(maxDets) if mDet == maxDets_]
        if ap == 1:
            s = precision
            if iouThr is not None:
                t = np.where(iouThr == iouThrs)[0]
                s = s[t]
            s = s[:, :, :, aind, mind]
        else:
            s = recall
            if iouThr is not None:
                t = np.where(iouThr == iouThrs)[0]
                s = s[t]
            s = s[:, :, aind, mind]
        if len(s[s > -1]) == 0:
            mean_s = -1
        else:
            mean_s = np.mean(s[s > -1])
        return mean_s

    stats = np.zeros((12,))
    stats[0] = _summarize(1)
    stats[1] = _summarize(1, iouThr=.5, maxDets_=maxDets[2])
    stats[2] = _summarize(1, iouThr=.75, maxDets_=maxDets[2])
    stats[3] = _summarize(1, areaRng='small', maxDets_=maxDets[2])
    stats[4] = _summarize(1, areaRng='medium', maxDets_=maxDets[2])
    stats[5] = _summarize(1, areaRng='large', maxDets_=maxDets[2])
    stats[6] = _summarize(0, maxDets_=maxDets[0])
    stats[7] = _summarize(0, maxDets_=maxDets[1])
    stats[8] = _summarize(0, maxDets_=maxDets[2])
    stats[9] = _summarize(0, areaRng='small', maxDets_=maxDets[2])
    stats[10] = _summarize(0, areaRng='medium', maxDets_=maxDets[2])
    stats[11] = _summarize(0, areaRng='large', maxDets_=maxDets[2])
    return stats


def classwise_table(precision, names):
    """Per-category AP of an accumulated precision array [T, R, K, A, M] (as CocoDataset.evaluate(classwise=True) of
    later mmdetection computes it): for category k, the mean of precision[:, :, k, 0, -1] (area range 'all', the last
    maxDet) over its values > -1, nan when there are none.  Returns [(name, ap)] in the order of K."""
    precision = np.asarray(precision)
    if precision.shape[2] != len(names):
        raise ValueError('classwise: %d names for %d categories' % (len(names), precision.shape[2]))
    out = []
    for k, name in enumerate(names):
        p = precision[:, :, k, 0, -1]
        p = p[p > -1]
        out.append((name, float(np.mean(p)) if p.size else float('nan')))
    return out


def mm_results(metric, stats):
    """CocoDataset.evaluate's entries of one metric: rounded stats[:6] and the copypaste string."""
    out = {}
    for i, item in enumerate(METRIC_ITEMS):
        out['{}_{}'.format(metric, item)] = float('{:.3f}'.format(stats[i]))
    out['{}_mAP_copypaste'.format(metric)] = ('{ap[0]:.3f} {ap[1]:.3f} {ap[2]:.3f} {ap[3]:.3f} '
                                             '{ap[4]:.3f} {ap[5]:.3f}').format(ap=stats[:6])
    return out


# ---------------------------------------------------------------------------------------------------- accumulate
def accumulate(row_parts, npig, K, dev, params=None):
    """COCOeval.accumulate on the device: the precision / recall / scores arrays (numpy) of the OUT_DTYPE rows (a list
    of uint8 device tensors) and npig [K, A], on the current stream.  params: CocoParams (None: the default Params)."""
    parts = [r.view(torch.int64).view(-1, 5) for r in row_parts]
    rows = torch.cat(parts) if parts else torch.zeros((0, 5), dtype=torch.int64, device=dev)
    score = rows[:, 0].contiguous().view(torch.float64)
    img = rows[:, 1].contiguous()
    cat = (rows[:, 4] & 0xffffffff).to(torch.int32)      # little-endian {cat, rank} in the last word
    rank = (rows[:, 4] >> 32).to(torch.int32)
    # global order: category, score descending, image id, rank (stable sorts from the last key to the first)
    o = torch.argsort(rank, stable=True)
    o = o[torch.argsort(img[o], stable=True)]
    o = o[torch.argsort(-score[o], stable=True)]
    o = o[torch.argsort(cat[o], stable=True)]
    srt = rows[o].contiguous()
    cat_off = torch.searchsorted(cat[o].contiguous(), torch.arange(K + 1, dtype=torch.int32, device=dev)).to(torch.int32)
    T, R, A, M = (len(IOU_THRS), len(REC_THRS), len(AREA_RNG), len(MAX_DETS)) if params is None else params.shape
    precision = torch.empty((T, R, K, A, M), dtype=torch.float64, device=dev)
    scores = torch.empty_like(precision)
    recall = torch.empty((T, K, A, M), dtype=torch.float64, device=dev)
    if params is not None and params.extended:
        pc = params.c_struct()
        L.check(L.lib().smb_coco_accumulate_params2_dev(L.ptr(srt), ctypes.c_int64(srt.shape[0]), L.ptr(cat_off), K,
                                                        L.ptr(npig), ctypes.byref(pc), L.ptr(precision), L.ptr(recall),
                                                        L.ptr(scores), L.stream_ptr()), 'smb_coco_accumulate_params2_dev')
    elif params is None:
        rec_thr = torch.from_numpy(np.ascontiguousarray(REC_THRS)).to(dev)
        md = (ctypes.c_int * 3)(*MAX_DETS)
        L.check(L.lib().smb_coco_accumulate_dev(L.ptr(srt), ctypes.c_int64(srt.shape[0]), L.ptr(cat_off), K, L.ptr(npig),
                                                L.ptr(rec_thr), md, L.ptr(precision), L.ptr(recall), L.ptr(scores),
                                                L.stream_ptr()), 'smb_coco_accumulate_dev')
    else:
        pc = params.c_struct()
        L.check(L.lib().smb_coco_accumulate_params_dev(L.ptr(srt), ctypes.c_int64(srt.shape[0]), L.ptr(cat_off), K,
                                                       L.ptr(npig), ctypes.byref(pc), L.ptr(precision), L.ptr(recall),
                                                       L.ptr(scores), L.stream_ptr()), 'smb_coco_accumulate_params_dev')
    return precision.cpu().numpy(), recall.cpu().numpy(), scores.cpu().numpy()


# ---------------------------------------------------------------------------------------------------- error analysis
# SipMask-mmdetection's tools/coco_error_analysis.py: one COCOeval of every result with these Params (ps[0:3]), and per
# category k two more of k's results against relabelled ground truth (Sim, Oth: iouThrs [.1], maxDets [100]).  On the
# device the two per-category evaluations are one more match per image (smb_coco_analysis_match_dev) whose rows carry
# Sim in bits 0..3 and Oth in bits 4..7, accumulated as two "thresholds".
ANALYSIS_PARAMS = CocoParams(iou_thrs=[.75, .5, .1], max_dets=[100])
_SIM_OTH_PARAMS = CocoParams(iou_thrs=[.1, .1], max_dets=[100])
ANALYSIS_TYPES = ['C75', 'C50', 'Loc', 'Sim', 'Oth', 'BG', 'FN']
ANALYSIS_AREAS = ['allarea', 'small', 'medium', 'large']


def analysis_arrays(p3, p2):
    """coco_error_analysis.py's ps [7, R, K, 4, 1] from the precision of the [.75, .5, .1] evaluation (p3) and of the
    Sim / Oth rows (p2 [2, R, K, 4, 1]): C75, C50, Loc, Sim, Oth with -1 -> 0, then BG = Oth > 0 and FN = 1."""
    ps = np.zeros((7,) + p3.shape[1:])
    ps[0:3] = p3
    ps[3:5] = p2
    ps[ps == -1] = 0
    ps[5] = ps[4] > 0
    ps[6] = 1.0
    return ps


def analysis_table(ps, gt):
    """The numbers the tool's plot legends show: per class k, type t and area a, ps[t, :, k, a, 0].mean(); for
    'allclass', the mean over recall thresholds and classes.  Returns dict(types, areas, cat_ids, names,
    classes [K, 7, 4], allclass [7, 4])."""
    ps = np.asarray(ps)
    return dict(types=list(ANALYSIS_TYPES), areas=list(ANALYSIS_AREAS), cat_ids=list(gt.cat_ids), names=list(gt.names),
                classes=ps[..., 0].mean(axis=1).transpose(1, 0, 2), allclass=ps[..., 0].mean(axis=(1, 2)))


def analyze_json(gt, bbox_json=None, segm_json=None, img_ids=None, chunk=64, device=None):
    """coco_error_analysis.py's arrays of result lists against `gt` on the device: {metric: ps [7, R, K, 4, 1]}, K in
    the order of gt.cat_ids (sorted ids; the tool uses the file's order of categories, the same when the file lists
    them sorted by id, as COCO's does).  Raises ValueError when a category has no supercategory."""
    metrics = [m for m, j in (('bbox', bbox_json), ('segm', segm_json)) if j is not None]
    return _run_json(gt, gt.cat_ids, bbox_json, segm_json, img_ids, chunk, device, None, True, metrics)['analysis']


# ---------------------------------------------------------------------------------------------------- evaluator
def _dev_bytes(arr, dev):
    return torch.from_numpy(np.ascontiguousarray(arr).view(np.uint8).reshape(-1)).to(dev)


def check_metrics(metrics, benchmark=False):
    """CocoDataset.evaluate's metric names this evaluator runs: 'bbox', 'segm' and 'proposal' (box recall of the bbox
    results, class-agnostic).  Raises KeyError for a name CocoDataset.evaluate does not know either, ValueError for
    'proposal_fast' and, on SipMask-benchmark records, for 'proposal'."""
    metrics = [metrics] if isinstance(metrics, str) else list(metrics)
    for m in metrics:
        if m == 'proposal_fast':
            raise ValueError("metric 'proposal_fast' is not supported: it evaluates proposal arrays (eval_recalls reads "
                             "proposals[i].ndim), which SipMask's (bboxes, masks) results are not; 'proposal' gives "
                             "AR@100 / 300 / 1000 of the bbox results")
        if m not in ('bbox', 'segm', 'proposal'):
            raise KeyError('metric {} is not supported'.format(m))
    if benchmark and 'proposal' in metrics:
        raise ValueError("metric 'proposal' is not supported on SipMask-benchmark records: its evaluation never "
                         "evaluates box proposals of SipMask (box_only=False)")
    return metrics


def proposal_results(stats):
    """CocoDataset.evaluate's entries of metric 'proposal': stats[6:12] rounded, under its names whatever proposal_nums
    are."""
    return {item: float('{:.3f}'.format(stats[i + 6])) for i, item in enumerate(PROPOSAL_ITEMS)}


class _View:
    """What one metric is matched and accumulated with: its Params (None: the default entry points), the ground truth as
    they index it (gv: index into the evaluator's distinct views), the category index of each record label, K of the
    match launches (categories the rows index) and of accumulate (1 with useCats 0)."""

    def __init__(self, params, gv, label_cat_host, dev, K):
        self.params, self.gv, self.K = params, gv, K
        self.K_acc = K if params is None or params.use_cats else 1
        self.A = len(AREA_RNG) if params is None else params.shape[2]
        self.pc = params.c_struct() if params is not None else None
        self.label_cat_host = label_cat_host
        self.label_cat = torch.from_numpy(label_cat_host).to(dev)


class CocoEvaluator:
    """Device state of one COCO evaluation: per evaluated image, its detections' matched / ignored flags (per metric),
    and npig per (category, area range).  Images are added as engine records (add_records) or result lists
    (add_results); evaluate() accumulates and summarizes.
      gt      : CocoGroundTruth
      cat_ids : COCO category id per 0-based record label (as coco.coco_json takes it)
      benchmark: SipMask-benchmark records (BoxList.resize boxes, box scores for segm)
      params  : CocoParams or CocoParams2 (None: COCOeval's default Params)
      analyze : also run, for every image added, the matches of coco_error_analysis.py (see analysis_arrays), so that
                evaluate() returns its precision arrays as well (every ground-truth category: not with a cat_ids
                subset)
      metrics : 'bbox', 'segm' and / or 'proposal': MM's proposal metric, COCOeval of the bbox results (boxes and box
                scores) with the default Params but useCats = 0 and maxDets = proposal_nums, whatever `params` are."""

    def __init__(self, gt, cat_ids, metrics=('bbox', 'segm'), benchmark=False, device=None, params=None, analyze=False,
                 proposal_nums=PROPOSAL_NUMS):
        metrics = check_metrics(metrics, benchmark)
        if params is not None and not isinstance(params, CocoParams):
            raise ValueError('params must be a CocoParams')
        self.gt, self.metrics, self.benchmark, self.params = gt, metrics, bool(benchmark), params
        self.dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.K = len(gt.cat_ids)
        self.label_cat_host = np.array([gt.cat_index.get(int(c), -1) for c in cat_ids], np.int32)
        self.proposal_params = (CocoParams2(max_dets=[int(n) for n in proposal_nums], use_cats=0)
                                if 'proposal' in metrics else None)
        self._gviews, self._gcats, self.views = [], [], {}
        for m in metrics:
            p = self.proposal_params if m == 'proposal' else params
            cats = list(gt.cat_ids) if p is None else p.eval_cats(gt.cat_ids)
            if cats not in self._gcats:
                self._gcats.append(cats)
                self._gviews.append(gt if cats == list(gt.cat_ids) else gt.subset(cats))
            gv = self._gcats.index(cats)
            lc = np.array([self._gviews[gv].cat_index.get(int(c), -1) for c in cat_ids], np.int32)
            self.views[m] = _View(p, gv, lc, self.dev, len(cats))
        self._segm_gv = self.views['segm'].gv if 'segm' in metrics else 0
        if analyze and any(self._gviews[self.views[m].gv] is not gt for m in metrics if m != 'proposal'):
            raise ValueError('analyze: the error analysis evaluates every ground-truth category (no cat_ids subset)')
        self.npig = {m: torch.zeros(v.K_acc * v.A, dtype=torch.int32, device=self.dev) for m, v in self.views.items()}
        self.rows = {m: [] for m in metrics}
        self.status = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.raster_status = torch.zeros(1, dtype=torch.int32, device=self.dev)
        self.n_results = {m: torch.zeros((), dtype=torch.int64, device=self.dev) for m in metrics}
        self.image_ids = []
        self._seen = set()
        self._iou_thr = np.ascontiguousarray(IOU_THRS, dtype=np.float64)
        self._area_rng = np.ascontiguousarray(np.array(AREA_RNG, dtype=np.float64).reshape(-1))
        self.analyze = bool(analyze)
        if self.analyze:
            sup, self.n_sup = gt.supercategory_index()
            self.sup = torch.from_numpy(sup).to(self.dev)
            self._ana_c = ANALYSIS_PARAMS.c_struct()
            ana = [m for m in metrics if m != 'proposal']
            self.npig_ana = {m: torch.zeros(self.K * len(AREA_RNG), dtype=torch.int32, device=self.dev) for m in ana}
            self.rows_c = {m: [] for m in ana}             # ps[0:3]: iouThrs [.75, .5, .1], maxDets [100]
            self.rows_so = {m: [] for m in ana}            # ps[3:5]: Sim / Oth rows

    # ---- bookkeeping
    def _claim(self, image_ids, ori_hws=None):
        ids = [int(i) for i in image_ids]
        for n, i in enumerate(ids):
            if i not in self.gt.hw:
                raise ValueError('image id %d is not in the ground truth' % i)
            if i in self._seen or ids.count(i) > 1:
                raise ValueError('image id %d is evaluated twice' % i)
            if ori_hws is not None and tuple(int(v) for v in ori_hws[n][:2]) != self.gt.hw[i]:
                raise ValueError('image %d: ori_shape %r differs from the annotation %dx%d'
                                 % (i, tuple(ori_hws[n][:2]), self.gt.hw[i][0], self.gt.hw[i][1]))
        return ids

    def stage_gt(self, image_id, stream=None, masks=None):
        """Pack one image's ground truth (rows, per-category offsets and, for 'segm', what describes its masks: polygon
        vertices and run lengths) and upload it from pinned memory on `stream` (default: the current stream); its planes
        are reserved on the device and rasterized there right before the image's first segm match.  Returns its device
        tensors, for add_records(..., gts=[...]) on a stream that is ordered after `stream`.  masks: whether the masks
        are needed (default: when 'segm' is evaluated).  When the metrics index the ground truth differently (a cat_ids
        subset beside 'proposal'), each such view is staged too, under 'views'."""
        want = 'segm' in self.metrics if masks is None else bool(masks)
        staged = [self._stage_view(g, int(image_id), stream, want and v == self._segm_gv)
                  for v, g in enumerate(self._gviews)]
        staged[0]['views'] = staged
        return staged[0]

    def _stage_view(self, gv, image_id, stream, segm):
        from . import segm_raster as SR
        rows, off, pack = gv.packed(image_id) if segm else gv.image(image_id, False)[:2] + (None,)
        h, w = self.gt.hw[image_id]
        pitch = (w + 31) // 32
        n_gt = len(rows)
        if segm:
            rows['plane'] = np.arange(n_gt, dtype=np.int64) * (h * pitch)
        stream = stream or torch.cuda.current_stream(self.dev)
        extra = (rows, off) + ((gv.positions(image_id),) if self.analyze else ())
        with torch.cuda.device(self.dev), torch.cuda.stream(stream):
            st, views = SR.staged(pack if segm else SR.SegmPack(), self.dev, extra)
            planes = torch.empty(max(n_gt * h * pitch, 1) if segm else 1, dtype=torch.int32, device=self.dev)
        rows_dev, off_dev = views[:2]
        pos = views[2].view(torch.int32) if self.analyze else None
        return dict(rows=rows_dev, off=off_dev.view(torch.int32), pos=pos, planes=planes, n_gt=n_gt,
                    plane_words=n_gt * h * pitch if segm else 0, stream=stream,
                    raster=dict(st, stride=h * pitch, pitch=pitch) if segm and n_gt else None)

    def _raster_gt(self, gt):
        """Rasterize a staged ground truth into its planes on the current stream, with each plane's pixel count and
        extents written into its row."""
        from . import segm_raster as SR
        r, gt['raster'] = gt['raster'], None
        rows = gt['rows'].view(torch.int32)              # smb_coco_gt_t: area_mask is int32 15, ext 16..19 of 20
        SR.raster(r, gt['planes'], gt['n_gt'], r['stride'], r['pitch'], self.raster_status, area=rows[15:],
                  area_stride=GT_DTYPE.itemsize // 4, ext=rows[16:], ext_stride=GT_DTYPE.itemsize // 4)

    def _outs(self, metric, n_rows):
        """Output rows of a batch: the plain match's and, when analyzing, those of the two analysis matches."""
        return [torch.empty(n_rows * OUT_DTYPE.itemsize, dtype=torch.uint8, device=self.dev)
                for _ in range(3 if self.analyze and metric != 'proposal' else 1)]

    def _keep(self, metric, outs):
        self.rows[metric].append(outs[0])
        if self.analyze and metric != 'proposal':
            self.rows_c[metric].append(outs[1])
            self.rows_so[metric].append(outs[2])

    def _match(self, metric, imgs, n, dets, det_cap, det_planes, det_plane_words, gt, outs):
        """The match launches of image n of a batch (imgs / dets: the batch's device rows) on the current stream."""
        lib = L.lib()
        view = self.views[metric]
        gt = gt['views'][view.gv] if 'views' in gt else gt
        cur = torch.cuda.current_stream(self.dev)
        if gt['stream'] != cur:                          # uploaded on another stream: keep it until this stream is done
            for key in ('rows', 'off', 'planes', 'pos'):
                if gt.get(key) is not None:
                    gt[key].record_stream(cur)
        if metric == 'segm' and gt['raster'] is not None:
            self._raster_gt(gt)
        out_rows = outs[0]
        n_out = out_rows.numel() // OUT_DTYPE.itemsize
        args = (ctypes.c_void_p(imgs.data_ptr() + n * IMG_DTYPE.itemsize), 1,
                ctypes.c_void_p(dets.data_ptr() + n * det_cap * DET_DTYPE.itemsize), det_cap, L.ptr(det_planes),
                ctypes.c_int64(det_plane_words), L.ptr(gt['rows']), gt['n_gt'], L.ptr(gt['planes']),
                ctypes.c_int64(gt['plane_words']), L.ptr(gt['off']), view.K, 1 if metric == 'segm' else 0)
        tail = (L.ptr(out_rows), ctypes.c_int64(n_out), L.ptr(self.npig[metric]), L.ptr(self.status))
        if view.pc is None:
            ws_bytes = lib.smb_coco_match_workspace_bytes(gt['n_gt'])
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
            L.check(lib.smb_coco_match_dev(*args, _ptr(self._iou_thr), _ptr(self._area_rng), *tail, L.ptr(ws),
                                           ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_coco_match_dev')
        elif view.params.extended:
            pc = ctypes.byref(view.pc)
            ws_bytes = lib.smb_coco_match_params2_workspace_bytes(gt['n_gt'], pc)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
            L.check(lib.smb_coco_match_params2_dev(*args, pc, *tail, L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
                    'smb_coco_match_params2_dev')
        else:
            pc = ctypes.byref(view.pc)
            ws_bytes = lib.smb_coco_match_params_workspace_bytes(gt['n_gt'], pc)
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
            L.check(lib.smb_coco_match_params_dev(*args, pc, *tail, L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
                    'smb_coco_match_params_dev')
        if not self.analyze or metric == 'proposal':
            return
        pc = ctypes.byref(self._ana_c)
        ws_bytes = lib.smb_coco_match_params_workspace_bytes(gt['n_gt'], pc)
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
        L.check(lib.smb_coco_match_params_dev(*args, pc, L.ptr(outs[1]), ctypes.c_int64(n_out), L.ptr(self.npig_ana[metric]),
                                              L.ptr(self.status), L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
                'smb_coco_match_params_dev')
        ws_bytes = lib.smb_coco_analysis_workspace_bytes(gt['n_gt'])
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
        L.check(lib.smb_coco_analysis_match_dev(*args[:11], L.ptr(gt['pos']), L.ptr(self.sup), self.n_sup, *args[11:],
                                                _ptr(self._area_rng), L.ptr(outs[2]), ctypes.c_int64(n_out),
                                                L.ptr(self.status), L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
                'smb_coco_analysis_match_dev')

    def _img_rows(self, ids, det_pitch, det_cap, n_det=None):
        imgs = np.zeros(len(ids), IMG_DTYPE)
        for n, i in enumerate(ids):
            h, w = self.gt.hw[i]
            imgs[n]['h'], imgs[n]['w'] = h, w
            imgs[n]['det_pitch'] = det_pitch[n] if hasattr(det_pitch, '__len__') else det_pitch
            imgs[n]['gt_pitch'] = (w + 31) // 32
            imgs[n]['n_det'] = 0 if n_det is None else n_det[n]
            imgs[n]['image_id'] = i
            imgs[n]['out_off'] = n * det_cap
        return imgs

    # ---- engine records
    def check_image(self, image_id, ori_shape):
        """Raises ValueError unless image_id can be evaluated next with this ori_shape (in the ground truth, not evaluated
        yet, ori_shape equal to the annotation's height x width)."""
        self._claim([image_id], [ori_shape])

    def add_records(self, rec, geom, image_ids, ori_shapes, gts=None):
        """Evaluate the first len(image_ids) images of a batch of engine records (det_bboxes, det_labels, count,
        mask_bits, mask_scores when present; device tensors of the engine's last forward) on the current stream.
        geom: the engine's device geometry rows of that forward; ori_shapes: each image's ori_shape (checked against the
        annotation's height x width); gts: each image's stage_gt (default: staged here on the current stream).  The record
        may be overwritten once the stream has passed these launches."""
        with torch.cuda.device(self.dev):
            ids = self._claim(image_ids, ori_shapes)
            B = len(ids)
            if B == 0:
                return
            det, labels, count, bits = rec['det_bboxes'], rec['det_labels'], rec['count'], rec['mask_bits']
            ms = rec.get('mask_scores') if not self.benchmark else None
            N, max_num, cap_h, words = bits.shape
            if B > N or det.shape[:2] != (N, max_num) or labels.shape[:2] != (N, max_num) or max_num > DET_CAP:
                raise ValueError('add_records: %d image ids for a record of %d images x %d detections' % (B, N, max_num))
            for t, dt in ((det, torch.float32), (labels, torch.int64), (count, torch.int32), (bits, torch.int32),
                          (geom, torch.int32)):
                if t.device != self.dev or t.dtype != dt or not t.is_contiguous():
                    raise ValueError('add_records: record tensors must be contiguous on %s' % self.dev)
            if ms is not None and (ms.dtype != torch.float32 or ms.shape[:2] != (N, max_num) or not ms.is_contiguous()):
                raise ValueError('add_records: mask_scores must be a contiguous float32 [N, max_num] tensor')
            if gts is None:
                gts = [self.stage_gt(i) for i in ids]
            lib = L.lib()
            imgs = _dev_bytes(self._img_rows(ids, words, max_num), self.dev)
            dets = {}                                     # per ground-truth view: its category index of every label
            for m in self.metrics:
                v = self.views[m]
                if v.gv in dets:
                    continue
                dets[v.gv] = torch.empty(B * max_num * DET_DTYPE.itemsize, dtype=torch.uint8, device=self.dev)
                L.check(lib.smb_coco_det_from_record_dev(L.ptr(det), L.ptr(labels), L.ptr(count), L.ptr(ms), L.ptr(bits),
                                                         B, max_num, cap_h, words, L.ptr(geom), L.ptr(v.label_cat),
                                                         len(v.label_cat_host), int(self.benchmark), L.ptr(dets[v.gv]),
                                                         L.ptr(imgs), L.ptr(self.status), L.stream_ptr()),
                        'smb_coco_det_from_record_dev')
            n_json = count[:B].clamp(0, max_num).sum()
            for m in self.metrics:
                outs = self._outs(m, B * max_num)
                for n in range(B):
                    self._match(m, imgs, n, dets[self.views[m].gv], max_num, bits, bits.numel(), gts[n], outs)
                self._keep(m, outs)
                self.n_results[m] += n_json
            self.image_ids += ids
            self._seen.update(ids)

    # ---- result lists
    def add_results(self, per_image, metric):
        """Evaluate `metric` of images from result-json entries (dicts with image_id, category_id, score, and bbox or
        segmentation).  per_image: [(image_id, its entries in list order)].  Used by evaluate_json, one metric at a time,
        for images it has claimed.  'proposal' reads the bbox results."""
        gv = self._gviews[self.views[metric].gv]
        box = metric != 'segm'
        with torch.cuda.device(self.dev):
            ids = [int(i) for i, _ in per_image]
            det_cap = max([1] + [len(v) for _, v in per_image])
            if det_cap > DET_CAP:
                raise ValueError('add_results: %d results for one image (at most %d)' % (det_cap, DET_CAP))
            B = len(ids)
            dets = np.zeros(B * det_cap, DET_DTYPE)
            dets['cat'] = -1
            from . import segm_raster as SR
            # segm: every result's counts go into one launch; the chunk's planes share the largest canvas' stride and pitch
            pack, rows_of_plane = SR.SegmPack(), []
            pitch = max([1] + [(self.gt.hw[i][1] + 31) // 32 for i in ids])
            stride = max([1] + [self.gt.hw[i][0] for i in ids]) * pitch
            n_det = []
            for n, (i, res) in enumerate(zip(ids, (v for _, v in per_image))):
                h, w = self.gt.hw[i]
                n_det.append(len(res))
                for j, r in enumerate(res):
                    d = dets[n * det_cap + j]
                    d['order'] = j
                    try:
                        score = float(r['score'])
                        cat = int(r['category_id'])
                        if box:
                            bb = [float(v) for v in r['bbox']]
                            if len(bb) != 4:
                                raise ValueError('bbox needs 4 numbers')
                            d['box'] = bb
                            d['area_box'] = bb[2] * bb[3]
                        else:
                            seg = r['segmentation']
                            if not isinstance(seg, dict):
                                raise ValueError('result of image %d: segmentation must be an RLE dict' % i)
                            pack.add(seg, h, w, len(rows_of_plane), 'result of image %d' % i)
                            d['plane'] = len(rows_of_plane) * stride
                            rows_of_plane.append(n * det_cap + j)
                    except (KeyError, TypeError) as e:
                        raise ValueError('add_results: malformed result %r: %r' % (r, e))
                    d['score'][0 if box else 1] = score
                    d['cat'] = gv.cat_index.get(cat, -1)
            imgs = _dev_bytes(self._img_rows(ids, pitch, det_cap, n_det), self.dev)
            P = len(rows_of_plane)
            st, (dd, at) = SR.staged(pack, self.dev, (dets, np.array(rows_of_plane, np.int64)))
            pd = torch.empty(max(P * stride, 1), dtype=torch.int32, device=self.dev)
            if P:
                # pixel counts and extents of the planes, scattered into their rows (smb_coco_det_t: area_mask is
                # int32 16, ext 18..21 of 24)
                stats = torch.zeros((P, 5), dtype=torch.int32, device=self.dev)
                SR.raster(st, pd, P, stride, pitch, self.raster_status, area=stats, area_stride=5, ext=stats[:, 1:],
                          ext_stride=5)
                at = at.view(torch.int64)[:P]
                rows32 = dd.view(torch.int32)[:B * det_cap * 24].view(B * det_cap, 24)
                rows32[at, 16] = stats[:, 0]
                rows32[at[:, None], torch.arange(18, 22, device=self.dev)[None]] = stats[:, 1:]
            outs = self._outs(metric, B * det_cap)
            for n, i in enumerate(ids):
                self._match(metric, imgs, n, dd, det_cap, pd, pd.numel(), self.stage_gt(i, masks=metric == 'segm'), outs)
            self._keep(metric, outs)

    # ---- accumulate + summarize
    def _accumulate(self, metric):
        v = self.views[metric]
        return accumulate(self.rows[metric], self.npig[metric], v.K_acc, self.dev, v.params)

    # ---- state across processes
    def state(self):
        """This evaluator's device state as a flat dict of 1-D tensors on its device, for merge() in another evaluator
        of the same settings (dist.gather_eval_state carries it between ranks): 'image_ids' (int64), 'status' and
        'raster_status', and per metric m 'rows/m' (the OUT_DTYPE rows, uint8), 'npig/m', 'n_results/m' and, when
        analyzing, 'rows_c/m', 'rows_so/m' and 'npig_ana/m'."""
        def cat(parts):
            return torch.cat(parts) if parts else torch.zeros(0, dtype=torch.uint8, device=self.dev)
        st = {'image_ids': torch.tensor(self.image_ids, dtype=torch.int64).to(self.dev),
              'status': self.status.clone(), 'raster_status': self.raster_status.clone()}
        for m in self.metrics:
            st['rows/' + m] = cat(self.rows[m])
            st['npig/' + m] = self.npig[m].clone()
            st['n_results/' + m] = self.n_results[m].reshape(1).clone()
            if self.analyze and m != 'proposal':
                st['rows_c/' + m] = cat(self.rows_c[m])
                st['rows_so/' + m] = cat(self.rows_so[m])
                st['npig_ana/' + m] = self.npig_ana[m].clone()
        return st

    def merge(self, states):
        """Add other evaluators' state() (same ground truth, cat_ids, metrics, Params and analyze) to this one: their
        rows are appended, npig and n_results summed, status bits OR-ed.  evaluate() then gives what one evaluator of
        all their images gives (accumulate orders the rows itself).  Raises ValueError for a state of other settings
        and for an image id evaluated here or in two states, before anything is merged."""
        states = list(states)
        want = set(self.state_keys())
        seen = set(self._seen)
        ids = []
        for st in states:
            if set(st) != want:
                raise ValueError('merge: a state of an evaluator with other metrics / analyze settings')
            for m in self.metrics:
                if st['npig/' + m].numel() != self.npig[m].numel():
                    raise ValueError('merge: a state of an evaluator with another ground truth or Params (%s)' % m)
            for i in st['image_ids'].cpu().tolist():
                if i in seen:
                    raise ValueError('merge: image id %d is evaluated twice (in two states, or here and in a state)' % i)
                if i not in self.gt.hw:
                    raise ValueError('merge: image id %d is not in the ground truth' % i)
                seen.add(i)
                ids.append(i)
        for st in states:
            self.status |= st['status'].to(self.dev)
            self.raster_status |= st['raster_status'].to(self.dev)
            for m in self.metrics:
                self.rows[m].append(st['rows/' + m].to(self.dev))
                self.npig[m] += st['npig/' + m].to(self.dev)
                self.n_results[m] += st['n_results/' + m].to(self.dev).reshape(())
                if self.analyze and m != 'proposal':
                    self.rows_c[m].append(st['rows_c/' + m].to(self.dev))
                    self.rows_so[m].append(st['rows_so/' + m].to(self.dev))
                    self.npig_ana[m] += st['npig_ana/' + m].to(self.dev)
        self.image_ids += ids
        self._seen.update(ids)

    def state_keys(self):
        """The keys of state(), in a fixed order."""
        keys = ['image_ids', 'status', 'raster_status']
        for m in self.metrics:
            keys += [s + m for s in ('rows/', 'npig/', 'n_results/')]
            if self.analyze and m != 'proposal':
                keys += [s + m for s in ('rows_c/', 'rows_so/', 'npig_ana/')]
        return keys

    def evaluate(self, classwise=False):
        """Accumulate and summarize every metric.  Returns 'arrays' ({metric: {'precision', 'recall', 'scores'}}) with
        COCOeval's eval arrays in the Params' shapes (K along CocoParams.cat_axis) and, where COCOeval.summarize runs on
        the Params (three maxDets and the labels all / small / medium / large), MM's dict (bbox_mAP, ...,
        segm_mAP_copypaste; AR@100, ..., AR_l@1000 for 'proposal') and 'stats'.  With analyze=True, also 'analysis'
        ({metric: ps}, see analysis_arrays).  classwise=True adds 'classwise' ({metric: classwise_table} for 'bbox' /
        'segm': per-category AP with the ground truth's category names); it needs per-category arrays (useCats = 1)."""
        if classwise:
            for m in self.metrics:
                p = self.views[m].params
                if m != 'proposal' and p is not None and not p.use_cats:
                    raise ValueError('classwise: %s is evaluated class-agnostically (useCats = 0)' % m)
        with torch.cuda.device(self.dev):
            status = int(self.status.item())
            if status & LABEL_RANGE:
                raise ValueError('a record label is outside the %d labels of cat_ids' % len(self.label_cat_host))
            if status & ANALYSIS_RANGE:
                raise L.SmbError('COCO error analysis: an annotation position or supercategory index is out of range')
            if status:
                raise L.SmbError('COCO evaluation status %d' % status)
            from .segm_raster import check_status
            check_status(self.raster_status)
            out, stats, arrays = {}, {}, {}
            for m in self.metrics:
                if int(self.n_results[m].item()) == 0:
                    raise ValueError('%s: the results of the evaluated images are empty' % m)
                p, r, s = self._accumulate(m)
                arrays[m] = dict(precision=p, recall=r, scores=s)
                prm = self.views[m].params
                if prm is None:
                    stats[m] = summarize(p, r)
                elif prm.summarizable():
                    stats[m] = summarize(p, r, prm.area_rng_lbl, prm.max_dets, prm.iou_thrs)
                else:
                    continue
                out.update(proposal_results(stats[m]) if m == 'proposal' else mm_results(m, stats[m]))
            if stats:
                out['stats'] = stats
            out['arrays'] = arrays
            if self.analyze:
                out['analysis'] = {m: self._analysis(m) for m in self.metrics if m != 'proposal'}
            if classwise:
                out['classwise'] = {m: classwise_table(arrays[m]['precision'], self._gviews[self.views[m].gv].names)
                                    for m in self.metrics if m != 'proposal'}
            return out

    def _analysis(self, m):
        p3 = accumulate(self.rows_c[m], self.npig_ana[m], self.K, self.dev, ANALYSIS_PARAMS)[0]
        p2 = accumulate(self.rows_so[m], self.npig_ana[m], self.K, self.dev, _SIM_OTH_PARAMS)[0]
        return analysis_arrays(p3, p2)


def evaluate_json(gt, cat_ids, bbox_json=None, segm_json=None, img_ids=None, chunk=64, device=None, params=None,
                  proposal=False, proposal_nums=PROPOSAL_NUMS, classwise=False):
    """COCOeval of result lists (coco.coco_json output or a loaded results file) against `gt` on the device: the same
    kernels as CocoEvaluator, with the detections' RLE strings parsed to run lengths on the host and rasterized on the
    device.  img_ids: the evaluated images
    (p.imgIds; default every ground-truth image).  As in pycocotools, a result whose image is not in the ground truth
    raises (loadRes), and results of ground-truth images outside img_ids are not evaluated (_prepare).  params:
    CocoParams (None: the default Params).  proposal: also MM's 'proposal' metric of bbox_json (useCats = 0, maxDets =
    proposal_nums).  classwise: also the per-category AP tables (CocoEvaluator.evaluate).  Returns
    CocoEvaluator.evaluate()'s dict for the metrics given."""
    metrics = [m for m, j in (('bbox', bbox_json), ('segm', segm_json)) if j is not None]
    if proposal:
        if bbox_json is None:
            raise ValueError("evaluate_json: 'proposal' evaluates the bbox results; bbox_json is None")
        metrics.append('proposal')
    return _run_json(gt, cat_ids, bbox_json, segm_json, img_ids, chunk, device, params, False, metrics, proposal_nums,
                     classwise)


def _run_json(gt, cat_ids, bbox_json, segm_json, img_ids, chunk, device, params, analyze, metrics,
              proposal_nums=PROPOSAL_NUMS, classwise=False):
    ev = CocoEvaluator(gt, cat_ids, metrics=metrics, device=device, params=params, analyze=analyze,
                       proposal_nums=proposal_nums)
    ids = ev._claim(gt.img_ids if img_ids is None else sorted(set(int(i) for i in img_ids)))
    for m, res in (('bbox', bbox_json), ('segm', segm_json), ('proposal', bbox_json)):
        if res is None or m not in metrics:
            continue
        per = {i: [] for i in ids}
        for r in res:
            if not isinstance(r, dict) or 'image_id' not in r:
                raise ValueError('%s results: malformed entry %r' % (m, r))
            i = int(r['image_id'])
            if i not in gt.hw:                       # loadRes: 'Results do not correspond to current coco set'
                raise ValueError('%s results: image %r is not in the ground truth' % (m, r['image_id']))
            if i in per:
                per[i].append(r)
        for c in range(0, len(ids), chunk):
            ev.add_results([(i, per[i]) for i in ids[c:c + chunk]], m)
        ev.n_results[m] += len(res)                   # loadRes fails on an empty list
    ev.image_ids = list(ids)
    ev._seen.update(ids)
    return ev.evaluate(classwise)
