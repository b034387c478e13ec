"""CPU checks of COCOeval with user-given Params and of the COCO error analysis: hand-derived answers of the restated
coco_error_analysis.py (coco_analysis_ref) on tiny datasets, CocoParams' limits (in Python and at the C ABI), the
ground truth's supercategories and positions, and summarize's iou_thrs."""
import ctypes

import numpy as np
import pytest

import coco_analysis_ref as AR

CATS = [dict(id=1, name='cat', supercategory='animal'), dict(id=2, name='dog', supercategory='animal'),
        dict(id=3, name='car', supercategory='vehicle')]
K_OF = {1: 0, 2: 1, 3: 2}
BA, BB, BC, BD = [10, 10, 30, 30], [50, 10, 30, 30], [10, 50, 30, 30], [50, 50, 30, 30]   # disjoint 30 x 30 boxes


def _gt(anns, n_img=1, cats=CATS):
    out = dict(images=[dict(id=i + 1, height=100, width=100) for i in range(n_img)], categories=cats, annotations=[])
    for n, (img, cat, box, crowd) in enumerate(anns):
        x, y, w, h = box
        out['annotations'].append(dict(id=n + 1, image_id=img, category_id=cat, bbox=list(map(float, box)),
                                       area=float(w * h), iscrowd=crowd,
                                       segmentation=[[x, y, x, y + h, x + w, y + h, x + w, y]]))
    return out


def _dt(dets):
    return [dict(image_id=img, category_id=cat, bbox=list(map(float, box)), score=s) for img, cat, box, s in dets]


def known_cases():
    """(name, gt, results, category id, {type index: precision at every recall threshold, 'all' areas})."""
    cases = []
    # a dog detection over a cat (same supercategory) and a true dog: FP in C75 / C50 / Loc, ignored in Sim and Oth
    cases.append(('sibling', _gt([(1, 1, BA, 0), (1, 2, BB, 0)]), _dt([(1, 2, BA, .9), (1, 2, BB, .8)]), 2,
                  {0: .5, 1: .5, 2: .5, 3: 1., 4: 1., 5: 1., 6: 1.}))
    # a car detection over a cat (another supercategory): FP in Sim as well, ignored in Oth
    cases.append(('other', _gt([(1, 1, BA, 0), (1, 3, BB, 0)]), _dt([(1, 3, BA, .9), (1, 3, BB, .8)]), 3,
                  {0: .5, 1: .5, 2: .5, 3: .5, 4: 1., 5: 1., 6: 1.}))
    # a cat detection on background: FP everywhere
    cases.append(('background', _gt([(1, 1, BA, 0), (1, 2, BB, 0)]), _dt([(1, 1, BD, .9), (1, 1, BA, .8)]), 1,
                  {0: .5, 1: .5, 2: .5, 3: .5, 4: .5, 5: 1., 6: 1.}))
    # a crowd cat annotation after a dog annotation on the same box: the cat detection there is ignored in every
    # evaluation (own crowd in the plain one, crowd either way in Sim / Oth)
    cases.append(('crowd', _gt([(1, 2, BC, 0), (1, 1, BC, 1), (1, 1, BA, 0)]), _dt([(1, 1, BC, .9), (1, 1, BA, .8)]), 1,
                  {0: 1., 1: 1., 2: 1., 3: 1., 4: 1., 5: 1., 6: 1.}))
    # image 2 has no cat, only a car the cat detection overlaps (IoU 0.36 >= .1): no FP in Oth, npig stays 1
    cases.append(('no_own_gt', _gt([(1, 1, BA, 0), (2, 3, [10, 10, 30, 30], 0)], n_img=2),
                  _dt([(2, 1, [16, 16, 30, 30], .9), (1, 1, BA, .8)]), 1,
                  {0: .5, 1: .5, 2: .5, 3: .5, 4: 1., 5: 1., 6: 1.}))
    return cases


@pytest.mark.parametrize('case', range(5))
def test_restated_tool_known_answers(case):
    name, gt, dt, cat, want = known_cases()[case]
    ps = AR.analyze_results(gt, dt, 'bbox')
    assert ps.shape == (7, 101, 3, 4, 1)
    k = K_OF[cat]
    for t, v in want.items():
        # pr = tp / (fp + tp + spacing(1)): within an ulp or two of the hand-derived fraction
        assert np.allclose(ps[t, :, k, 0, 0], v, rtol=0, atol=1e-12), (name, t, ps[t, :, k, 0, 0][:3], v)


def test_restated_params_keep_pycocotools_quirks():
    """Unsorted recall thresholds: everything after the first one that is not reached stays 0 (IndexError)."""
    gt = _gt([(1, 1, BA, 0), (1, 1, BB, 0)])
    dt = _dt([(1, 1, BA, .9)])
    e = AR.run(gt, dt, 'bbox', summarize=False, rec_thrs=[.9, .2, .5], iou_thrs=[.5])
    assert list(e.precision[0, :, 0, 0, 2]) == [0., 0., 0.]
    e = AR.run(gt, dt, 'bbox', summarize=False, rec_thrs=[.2, .5, .9], iou_thrs=[.5])
    assert np.allclose(e.precision[0, :, 0, 0, 2], [1., 1., 0.], rtol=0, atol=1e-12)


def test_params_limits():
    from sipmask_b200 import cocoeval as C
    assert C.CocoParams().shape == (10, 101, 4, 3) and C.CocoParams().summarizable()
    assert C.CocoParams(iou_thrs=[.5] * 16, area_rng=[[0, 1]] * 4, area_rng_lbl='abcd').shape == (16, 101, 4, 3)
    assert not C.CocoParams(max_dets=[100]).summarizable()
    assert C.CocoParams(max_dets=[100, 1, 10]).max_dets == [1, 10, 100]     # COCOeval.evaluate sorts maxDets
    assert not C.CocoParams(area_rng=[[0, 1], [1, 2]], area_rng_lbl=['all', 'small']).summarizable()
    bad = [(dict(iou_thrs=[.5] * 17), 'T * A <= 64'), (dict(iou_thrs=[]), 'T * A'),
           (dict(area_rng=np.zeros((0, 2)), area_rng_lbl=[]), 'T * A'), (dict(max_dets=[1, 2, 3, 4]), '1 to 3'),
           (dict(max_dets=[]), '1 to 3'), (dict(max_dets=[1, 101]), '[1, 100]'), (dict(max_dets=[0]), '[1, 100]'),
           (dict(max_dets=[1.5]), 'integers'), (dict(rec_thrs=np.zeros(102)), '1 to 101'),
           (dict(rec_thrs=[]), '1 to 101'), (dict(iou_thrs=[np.nan]), 'NaN'), (dict(area_rng=[[0, np.nan]]), 'NaN'),
           (dict(area_rng=[[0, 1], [1, 2]]), 'labels'), (dict(use_cats=0), 'useCats'), (dict(cat_ids=[1]), 'catIds')]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg.replace('*', r'\*').replace('[', r'\[')):
            C.CocoParams(**kw)


def test_params_limits_at_the_abi():
    """The library refuses the same Params with SMB_EINVAL before any launch (no device needed)."""
    from sipmask_b200 import _lib as L, cocoeval as C
    lib = L.lib()
    assert lib.smb_coco_params_check(ctypes.byref(C.CocoParams().c_struct())) == 0
    assert lib.smb_coco_params_check(ctypes.byref(C.ANALYSIS_PARAMS.c_struct())) == 0
    for field, value in (('T', 17), ('T', 0), ('A', 0), ('M', 4), ('M', 0), ('R', 102), ('R', 0)):
        p = C.CocoParams().c_struct()
        setattr(p, field, value)
        assert lib.smb_coco_params_check(ctypes.byref(p)) != 0, (field, value)
        assert lib.smb_coco_match_params_workspace_bytes(3, ctypes.byref(p)) == 0
        rc = lib.smb_coco_accumulate_params_dev(None, ctypes.c_int64(0), None, 1, None, ctypes.byref(p), None, None,
                                                None, None)
        assert rc != 0
    p = C.CocoParams().c_struct()
    p.max_dets[2] = 101
    assert lib.smb_coco_params_check(ctypes.byref(p)) != 0
    assert b'maxDet' in lib.smb_last_error()
    p = C.CocoParams().c_struct()
    p.max_dets[0], p.max_dets[2] = 100, 1                # unsorted maxDets: COCOeval.evaluate would have sorted them
    assert lib.smb_coco_params_check(ctypes.byref(p)) != 0
    assert b'ascending' in lib.smb_last_error()
    p = C.CocoParams().c_struct()
    p.rec_thr[7] = float('nan')
    assert lib.smb_coco_params_check(ctypes.byref(p)) != 0


def test_ground_truth_supercategories_and_positions():
    from sipmask_b200 import cocoeval as C
    cats = [dict(id=9, name='z', supercategory='b'), dict(id=2, name='y', supercategory='a'),
            dict(id=5, name='x', supercategory='b')]
    gt = _gt([(1, 9, BA, 0), (1, 2, BB, 0), (1, 5, BC, 0), (1, 2, BD, 1), (1, 7, BA, 0)], cats=cats)
    g = C.CocoGroundTruth(gt)
    assert g.cat_ids == [2, 5, 9] and g.names == ['y', 'x', 'z']
    sup, n = g.supercategory_index()
    assert n == 2 and list(sup) == [0, 1, 1]
    # rows grouped by category (2, 2, 5, 9); their positions in the image's annotation order (category 7 is not listed)
    assert list(g.positions(1)) == [1, 3, 2, 0]
    rows, off, _ = g.image(1, masks=False)
    assert list(rows['id']) == [2, 4, 3, 1] and list(off) == [0, 2, 3, 4]
    cats[1] = dict(id=2, name='y')
    with pytest.raises(ValueError, match='supercategory'):
        C.CocoGroundTruth(_gt([], cats=cats)).supercategory_index()


def test_summarize_iou_thrs():
    from sipmask_b200 import cocoeval as C
    rng = np.random.default_rng(0)
    p = rng.random((10, 101, 3, 4, 3))
    r = rng.random((10, 3, 4, 3))
    assert np.array_equal(C.summarize(p, r), C.summarize(p, r, iou_thrs=C.IOU_THRS))
    p2, r2 = p[[5, 0]], r[[5, 0]]                    # thresholds .75, .5
    s = C.summarize(p2, r2, iou_thrs=[.75, .5])
    assert s[1] == np.mean(p2[1, :, :, 0, 2]) and s[2] == np.mean(p2[0, :, :, 0, 2])
    assert s[0] == np.mean(p2[:, :, :, 0, 2])
    s = C.summarize(p2, r2, iou_thrs=[.75, .6])      # no .5: that stat is -1, as in pycocotools
    assert s[1] == -1 and s[2] == np.mean(p2[0, :, :, 0, 2])


def test_analysis_arrays_and_table():
    from sipmask_b200 import cocoeval as C
    p3 = np.full((3, 101, 2, 4, 1), -1.0)
    p3[:, :, 0] = 0.25
    p2 = np.full((2, 101, 2, 4, 1), -1.0)
    p2[0, :, 0] = 0.5
    p2[1, :, 0] = 0.75
    ps = C.analysis_arrays(p3, p2)
    assert ps.shape == (7, 101, 2, 4, 1)
    assert np.all(ps[0:3, :, 0] == .25) and np.all(ps[3, :, 0] == .5) and np.all(ps[4, :, 0] == .75)
    assert np.all(ps[0:5, :, 1] == 0) and np.all(ps[5, :, 0] == 1) and np.all(ps[5, :, 1] == 0) and np.all(ps[6] == 1)
    g = C.CocoGroundTruth(_gt([], cats=CATS[:2]))
    t = C.analysis_table(ps, g)
    assert t['classes'].shape == (2, 7, 4) and t['allclass'].shape == (7, 4) and t['names'] == ['cat', 'dog']
    assert t['classes'][0, 4, 0] == .75 and t['allclass'][4, 0] == .375
