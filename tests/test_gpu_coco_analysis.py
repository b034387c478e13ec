"""GPU checks of COCOeval with user-given Params and of the COCO error analysis on the device, against the test
restatements (coco_analysis_ref): float64 arrays equal element for element, stats equal where summarize runs."""
import numpy as np
import pytest
import torch

import coco_analysis_ref as AR
import cocoeval_ref as R
from test_gpu_cocoeval import _mask_rle, _rect, _record_json, fake_records

pytestmark = pytest.mark.gpu

SUPS = {1: 'animal', 2: 'animal', 4: 'vehicle', 5: 'vehicle', 7: 'animal', 8: 'food'}


def analysis_dataset(seed, n_img=10):
    """Three supercategories; polygon, uncompressed and compressed ground truth; crowds; detections labelled with their
    own category, a sibling or another supercategory's category; repeated scores; background detections; one image with
    more than 100 detections of one category."""
    from sipmask_b200 import rle
    rng = np.random.default_rng(seed)
    cats = sorted(SUPS)
    gt = dict(images=[], annotations=[],
              categories=[dict(id=c, name='c%d' % c, supercategory=SUPS[c]) for c in cats])
    sibling = {c: [d for d in cats if SUPS[d] == SUPS[c] and d != c] for c in cats}
    other = {c: [d for d in cats if SUPS[d] != SUPS[c]] for c in cats}
    bbox, segm = [], []
    scores = [0.9, 0.75, 0.5, 0.5, 0.3]
    aid = 0
    for i in range(n_img):
        img = 7 + 2 * i
        h, w = int(rng.integers(60, 110)), int(rng.integers(70, 130))
        gt['images'].append(dict(id=img, height=h, width=w))
        boxes = []
        for g in range(0 if i == 4 else int(rng.integers(1, 8))):
            aid += 1
            cat = int(rng.choice(cats))
            x0, y0 = int(rng.integers(0, w - 20)), int(rng.integers(0, h - 20))
            x1, y1 = int(rng.integers(x0 + 4, w + 1)), int(rng.integers(y0 + 4, h + 1))
            m = _rect(h, w, x0, y0, x1, y1)
            kind = g % 3
            if kind == 0:
                seg = [[x0, y0, x0, y1, x1, y1, x1, y0]]
                m = R.ann_to_mask(seg, h, w)
            elif kind == 1:
                seg = {'size': [h, w], 'counts': rle.counts(m).tolist()}
            else:
                seg = _mask_rle(m)
            gt['annotations'].append(dict(id=aid, image_id=img, category_id=cat, bbox=[x0, y0, x1 - x0, y1 - y0],
                                          area=float(m.sum()) if rng.random() < .7 else float(rng.integers(10, 9000)),
                                          iscrowd=int(rng.random() < .15), segmentation=seg))
            boxes.append((cat, x0, y0, x1, y1))
        dets = []
        for cat, x0, y0, x1, y1 in boxes:
            for _ in range(int(rng.integers(1, 4))):
                u = rng.random()
                lab = cat if u < .5 else int(rng.choice(sibling[cat] or other[cat])) if u < .75 else int(rng.choice(other[cat]))
                dx, dy = int(rng.integers(-4, 5)), int(rng.integers(-4, 5))
                dets.append((lab, x0 + dx, y0 + dy, x1 + dx + int(rng.integers(-3, 4)), y1 + dy))
        n_bg = 120 if i == 3 else int(rng.integers(0, 6))
        for _ in range(n_bg):
            x0, y0 = int(rng.integers(0, w - 5)), int(rng.integers(0, h - 5))
            dets.append((cats[0] if i == 3 else int(rng.choice(cats)), x0, y0, x0 + int(rng.integers(2, 40)),
                         y0 + int(rng.integers(2, 40))))
        for cat, x0, y0, x1, y1 in dets:
            s = float(rng.choice(scores)) if rng.random() < .5 else float(np.float32(rng.random()))
            bbox.append(dict(image_id=img, category_id=cat, bbox=[float(x0), float(y0), float(x1 - x0), float(y1 - y0)],
                             score=s))
            segm.append(dict(image_id=img, category_id=cat, score=s, segmentation=_mask_rle(_rect(h, w, x0, y0, x1, y1))))
    return gt, bbox, segm


PARAMS = {
    'analysis': dict(iou_thrs=[.75, .5, .1], max_dets=[100]),
    'one_threshold': dict(iou_thrs=[.6]),
    'max_dets_1_10': dict(max_dets=[1, 10]),
    'two_ranges': dict(area_rng=[[0, 40 ** 2], [20 ** 2, 1e5 ** 2]], area_rng_lbl=['lo', 'hi']),
    'rec_11': dict(rec_thrs=np.linspace(0, 1, 11)),
    'ta_64': dict(iou_thrs=np.linspace(.2, .95, 16)),
    'unsorted': dict(iou_thrs=[.9, .5, .7], rec_thrs=[.5, .1, .9, .3, 1.], max_dets=[100, 5, 20],
                     area_rng=[[32 ** 2, 96 ** 2], [0, 1e10], [96 ** 2, 1e10], [0, 32 ** 2]],
                     area_rng_lbl=['medium', 'all', 'large', 'small']),
}


def _assert_arrays(res, ref, name):
    for key in ('precision', 'recall', 'scores'):
        x, y = res[key], getattr(ref, key)
        assert x.shape == y.shape, (name, key, x.shape, y.shape)
        bad = np.argwhere(x != y)
        assert bad.size == 0, (name, key, len(bad), [(tuple(i), x[tuple(i)], y[tuple(i)]) for i in bad[:4]])


@pytest.mark.parametrize('name', sorted(PARAMS))
def test_params_equal_restatement(name):
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = analysis_dataset(1)
    kw = PARAMS[name]
    p = C.CocoParams(**kw)
    if name == 'unsorted':
        assert p.max_dets == [5, 20, 100]                # COCOeval.evaluate sorts maxDets; summarize reads 100
    g = C.CocoGroundTruth(gt)
    res = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, chunk=4, params=p)
    for m, dt in (('bbox', bbox), ('segm', segm)):
        ref = AR.run(gt, dt, m, summarize=p.summarizable(), **kw)
        _assert_arrays(res['arrays'][m], ref, (name, m))
        if p.summarizable():
            assert np.array_equal(res['stats'][m], ref.stats), (name, m)
            assert res[m + '_mAP'] == float('{:.3f}'.format(ref.stats[0]))
        else:
            assert 'stats' not in res and m + '_mAP' not in res


def test_default_params_equal_no_params():
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = analysis_dataset(2)
    g = C.CocoGroundTruth(gt)
    a = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm)
    b = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, params=C.CocoParams())
    assert sorted(a) == sorted(b)
    for m in ('bbox', 'segm'):
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(a['arrays'][m][key], b['arrays'][m][key])
        assert np.array_equal(a['stats'][m], b['stats'][m])
        assert a[m + '_mAP_copypaste'] == b[m + '_mAP_copypaste']


def test_known_answers_on_device():
    from test_coco_analysis_host import known_cases
    from sipmask_b200 import cocoeval as C
    for name, gt, dt, _, _ in known_cases():
        g = C.CocoGroundTruth(gt)
        ps = C.analyze_json(g, bbox_json=dt)['bbox']
        assert np.array_equal(ps, AR.analyze_results(gt, dt, 'bbox')), name


@pytest.mark.parametrize('seed', [3, 4])
def test_analyze_json_equals_restated_tool(seed):
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = analysis_dataset(seed)
    g = C.CocoGroundTruth(gt)
    out = C.analyze_json(g, bbox_json=bbox, segm_json=segm, chunk=3)
    for m, dt in (('bbox', bbox), ('segm', segm)):
        ref = AR.analyze_results(gt, dt, m)
        bad = np.argwhere(out[m] != ref)
        assert bad.size == 0, (m, len(bad), [(tuple(i), out[m][tuple(i)], ref[tuple(i)]) for i in bad[:4]])
        assert (ref[3] != ref[4]).any() and (ref[1] != ref[3]).any()      # the data separates Sim, Oth and C50


def _with_sups(gt):
    for n, c in enumerate(gt['categories']):
        c['supercategory'] = 'abc'[n % 3]
    return gt


def test_records_and_batching():
    """CocoEvaluator(analyze=True) over engine records equals analyze_json of their coco_json, at any batching and
    image order; its plain and Params arrays are unchanged by analyze."""
    from sipmask_b200 import cocoeval as C
    rec, metas, geom, gt, cat_ids = fake_records(6, rescoring=True)
    g = C.CocoGroundTruth(_with_sups(gt))
    ids = [10, 11, 12]
    bbox, segm = _record_json(rec, metas, cat_ids, False, ids)
    ref = C.analyze_json(g, bbox_json=bbox, segm_json=segm)
    plain = C.evaluate_json(g, cat_ids, bbox_json=bbox, segm_json=segm)
    outs = []
    ev = C.CocoEvaluator(g, cat_ids, analyze=True)
    ev.add_records(rec, geom, ids, [m[1] for m in metas])
    outs.append(ev.evaluate())
    ev = C.CocoEvaluator(g, cat_ids, analyze=True)
    for n in (2, 0, 1):
        one = {k: v[n:n + 1].contiguous() for k, v in rec.items()}
        ev.add_records(one, geom[n:n + 1].contiguous(), [ids[n]], [metas[n][1]])
    outs.append(ev.evaluate())
    for o in outs:
        for m in ('bbox', 'segm'):
            assert np.array_equal(o['analysis'][m], ref[m]), m
            for key in ('precision', 'recall', 'scores'):
                assert np.array_equal(o['arrays'][m][key], plain['arrays'][m][key])
    assert np.array_equal(ref['segm'], AR.analyze_results(gt, segm, 'segm'))


def test_runner_analyze_and_params():
    from test_gpu_cocoeval import _first_pass_gt, _runner_images, _runner_kw
    from sipmask_b200 import cocoeval as C, coco
    from sipmask_b200.serving import CocoEvalRunner
    imgs = _runner_images(5, seed=31)
    cat_ids = [1 + label % 12 for label in range(80)]
    gt = _with_sups(_first_pass_gt(imgs, cat_ids, seed=4))
    g = C.CocoGroundTruth(gt)
    p = C.CocoParams(iou_thrs=[.6, .3], max_dets=[3, 100])
    sd, kw = _runner_kw(4, 'rle')
    runner = CocoEvalRunner(sd, g, cat_ids, params=p, analyze=True, **kw)
    tickets = [runner.submit(imgs[n].pin_memory(), 1000 + n) for n in (3, 0, 4, 1, 2)]
    res = runner.evaluate()
    torch.cuda.synchronize()
    bbox, segm = [], []
    for t, n in zip(tickets, (3, 0, 4, 1, 2)):
        r = runner.result(t)
        b, s = coco.coco_json(r, 1000 + n, cat_ids)
        bbox += b
        segm += [dict(x, segmentation={'size': x['segmentation']['size'], 'counts': x['segmentation']['counts']})
                 for x in s]
    ref = C.analyze_json(g, bbox_json=bbox, segm_json=segm)
    own = C.evaluate_json(g, cat_ids, bbox_json=bbox, segm_json=segm, params=p)
    assert 'stats' not in res
    for m in ('bbox', 'segm'):
        assert np.array_equal(res['analysis'][m], ref[m]), m
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(res['arrays'][m][key], own['arrays'][m][key]), (m, key)


def test_rejected_before_launch():
    from sipmask_b200 import cocoeval as C
    gt, bbox, _ = analysis_dataset(5, n_img=2)
    gt['categories'][2] = dict(id=gt['categories'][2]['id'], name='x')
    g = C.CocoGroundTruth(gt)
    with pytest.raises(ValueError, match='supercategory'):
        C.analyze_json(g, bbox_json=bbox)
    with pytest.raises(ValueError, match='T \\* A'):
        C.evaluate_json(g, g.cat_ids, bbox_json=bbox, params=C.CocoParams(iou_thrs=np.linspace(.1, .9, 17)))
    with pytest.raises(ValueError, match='100'):
        C.evaluate_json(g, g.cat_ids, bbox_json=bbox, params=C.CocoParams(max_dets=[1, 10, 1000]))
    with pytest.raises(ValueError):
        C.CocoEvaluator(g, g.cat_ids, params=dict(iou_thrs=[.5]))


def test_tool_writes_arrays_and_tables(tmp_path):
    import json
    import subprocess
    import sys
    import os
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = analysis_dataset(6, n_img=4)
    res = [dict(b, segmentation=s['segmentation']) for b, s in zip(bbox, segm)]
    (tmp_path / 'ann.json').write_text(json.dumps(gt))
    (tmp_path / 'res.json').write_text(json.dumps(res))
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    p = subprocess.run([sys.executable, os.path.join(root, 'tools', 'coco_error_analysis.py'), str(tmp_path / 'res.json'),
                        str(tmp_path / 'out'), '--ann', str(tmp_path / 'ann.json'), '--types', 'bbox', 'segm'],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
    ref = C.analyze_json(C.CocoGroundTruth(gt), bbox_json=res, segm_json=res)
    for m in ('bbox', 'segm'):
        z = np.load(tmp_path / 'out' / m / 'analysis.npz')
        assert np.array_equal(z['ps'], ref[m]) and list(z['cat_ids']) == sorted(SUPS)
        text = (tmp_path / 'out' / m / 'analysis.txt').read_text()
        assert text.splitlines()[0].split()[2:] == C.ANALYSIS_TYPES and 'allclass' in text
