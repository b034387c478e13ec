"""GPU checks of COCOeval with useCats, catIds subsets and maxDets up to 1000 (CocoParams2, the Params2 entry points) and
of MM's 'proposal' metric, against the restatement in test_cocoeval_cats_host: precision / recall / scores equal
element for element, from result files, engine records and CocoEvalRunner."""
import numpy as np
import pytest
import torch

import test_cocoeval_cats_host as P
from test_gpu_cocoeval import _mask_rle, _rect, random_dataset, fake_records, _record_json

pytestmark = pytest.mark.gpu


def _same_arrays(a, ref, name):
    for key in ('precision', 'recall', 'scores'):
        x, y = a[key], getattr(ref, key)
        assert x.shape == y.shape, (name, key, x.shape, y.shape)
        bad = np.argwhere(x != y)
        assert bad.size == 0, (name, key, len(bad), [(tuple(i), x[tuple(i)], y[tuple(i)]) for i in bad[:4]])


def test_known_answers_on_device():
    from sipmask_b200 import cocoeval as C
    for name, gt, dt, u, cats in P.known_cases():
        g = C.CocoGroundTruth(gt)
        segm = [dict(image_id=r['image_id'], category_id=r['category_id'], score=r['score'],
                     segmentation=_mask_rle(_rect(40, 40, *[int(v) for v in (r['bbox'][0], r['bbox'][1],
                                                                             r['bbox'][0] + r['bbox'][2],
                                                                             r['bbox'][1] + r['bbox'][3])])))
                for r in dt]
        params = C.CocoParams2(use_cats=u, cat_ids=cats)
        res = C.evaluate_json(g, g.cat_ids, bbox_json=dt, segm_json=segm, params=params)
        _same_arrays(res['arrays']['bbox'], P.run(gt, dt, 'bbox', use_cats=u, cat_ids=cats), name)
        _same_arrays(res['arrays']['segm'], P.run(gt, segm, 'segm', use_cats=u, cat_ids=cats), name)


def crowded_dataset(seed):
    """random_dataset plus two images with more than 1000 results (near copies of their ground truths in every
    category, score ties across categories, false positives), so that maxDets 1000 truncates there."""
    gt, bbox, segm = random_dataset(seed, n_img=10)
    rng = np.random.default_rng(seed + 100)
    cats = [c['id'] for c in gt['categories']]
    for im in gt['images'][3:5]:
        h, w = im['height'], im['width']
        anns = [a for a in gt['annotations'] if a['image_id'] == im['id']]
        n = 0
        while n < 1100:
            if anns and n % 3 == 0:
                x, y, bw, bh = anns[n % len(anns)]['bbox']
                box = [x + int(rng.integers(-2, 3)), y + int(rng.integers(-2, 3)), bw, bh]
            else:
                x0, y0 = int(rng.integers(0, w - 5)), int(rng.integers(0, h - 5))
                box = [x0, y0, int(rng.integers(2, 40)), int(rng.integers(2, 40))]
            s = float([0.9, 0.5, 0.25][n % 3]) if n % 2 == 0 else float(np.float32(rng.random()))
            for c in (cats if n % 5 == 0 else [cats[n % len(cats)]]):   # the same box and score in every category
                bbox.append(dict(image_id=im['id'], category_id=c, bbox=[float(v) for v in box], score=s))
                segm.append(dict(image_id=im['id'], category_id=c, score=s,
                                 segmentation=_mask_rle(_rect(h, w, box[0], box[1], box[0] + box[2], box[1] + box[3]))))
                n += 1
    return gt, bbox, segm


CASES = [  # (use_cats, cat_ids, max_dets)
    (1, None, [100, 300, 1000]),
    (0, None, [100, 300, 1000]),
    (0, None, [1, 10, 100]),
    (1, [3], [1, 10, 100]),
    (0, [3], [100, 300, 1000]),
    (1, [7, 1], [100, 300, 1000]),
    (0, [7, 1], [1, 10, 100]),
    (0, [7, 1, 3], [100, 300, 1000]),
    (1, [3, 99], [100, 300, 1000]),
    (0, [99, 3, 1], [1, 10, 100]),
]


@pytest.mark.parametrize('metric', ['bbox', 'segm'])
def test_evaluate_json_equals_restatement(metric):
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = crowded_dataset(0)
    per_img = {}
    for r in bbox:
        per_img[r['image_id']] = per_img.get(r['image_id'], 0) + 1
    assert max(per_img.values()) > 1000
    res_json = bbox if metric == 'bbox' else segm
    g = C.CocoGroundTruth(gt)
    cache = {}
    for u, cats, md in CASES:
        params = C.CocoParams2(use_cats=u, cat_ids=cats, max_dets=md)
        kw = dict(bbox_json=bbox) if metric == 'bbox' else dict(segm_json=segm)
        res = C.evaluate_json(g, g.cat_ids, params=params, chunk=4, **kw)
        ref = P.run(gt, res_json, metric, use_cats=u, cat_ids=cats, max_dets=md, mask_cache=cache)
        _same_arrays(res['arrays'][metric], ref, (metric, u, cats, md))
        assert np.array_equal(res['stats'][metric], ref.stats), (metric, u, cats, md)
        assert res['arrays'][metric]['precision'].shape[2] == len(params.cat_axis(g.cat_ids))


def test_proposal_metric_equals_restatement():
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = crowded_dataset(1)
    g = C.CocoGroundTruth(gt)
    for nums in ((100, 300, 1000), (10, 50, 200)):
        res = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, proposal=True, proposal_nums=nums,
                              params=C.CocoParams2(cat_ids=[7, 1]))
        ref = P.run(gt, bbox, 'bbox', use_cats=0, max_dets=list(nums))
        _same_arrays(res['arrays']['proposal'], ref, nums)
        assert np.array_equal(res['stats']['proposal'], ref.stats)
        for i, item in enumerate(['AR@100', 'AR@300', 'AR@1000', 'AR_s@1000', 'AR_m@1000', 'AR_l@1000']):
            assert res[item] == float('{:.3f}'.format(ref.stats[i + 6])), (nums, item)
        _same_arrays(res['arrays']['bbox'], P.run(gt, bbox, 'bbox', cat_ids=[7, 1]), 'bbox subset')
    with pytest.raises(ValueError, match='bbox_json'):
        C.evaluate_json(g, g.cat_ids, segm_json=segm, proposal=True)


@pytest.mark.parametrize('flavour', ['mm', 'mm_rescoring'])
def test_records_equal_coco_json(flavour):
    from sipmask_b200 import cocoeval as C
    rec, metas, geom, gt, cat_ids = fake_records(7, rescoring=flavour == 'mm_rescoring')
    g = C.CocoGroundTruth(gt)
    ids = [10, 11, 12]
    bbox, segm = _record_json(rec, metas, cat_ids, False, ids)
    for params in (C.CocoParams2(cat_ids=[9, 2]), C.CocoParams2(use_cats=0, cat_ids=[9, 2, 4], max_dets=[10, 100, 300]),
                   C.CocoParams2(cat_ids=[4, 2, 11], max_dets=[100, 300, 1000])):
        ev = C.CocoEvaluator(g, cat_ids, metrics=('bbox', 'segm', 'proposal'), params=params)
        ev.add_records(rec, geom, ids, [m[1] for m in metas])
        res = ev.evaluate()
        ref = C.evaluate_json(g, cat_ids, bbox_json=bbox, segm_json=segm, params=params, proposal=True)
        for m in ('bbox', 'segm', 'proposal'):
            for key in ('precision', 'recall', 'scores'):
                assert np.array_equal(res['arrays'][m][key], ref['arrays'][m][key]), (flavour, m, key)
        u, cats, md = params.use_cats, params.cat_ids, params.max_dets
        _same_arrays(res['arrays']['bbox'], P.run(gt, bbox, 'bbox', use_cats=u, cat_ids=cats, max_dets=md), 'bbox')
        _same_arrays(res['arrays']['segm'], P.run(gt, segm, 'segm', use_cats=u, cat_ids=cats, max_dets=md), 'segm')
        _same_arrays(res['arrays']['proposal'], P.run(gt, bbox, 'bbox', use_cats=0, max_dets=[100, 300, 1000]), 'ar')


def test_runner_equals_coco_json():
    from sipmask_b200 import cocoeval as C, coco, rle
    from sipmask_b200.serving import CocoEvalRunner
    from test_gpu_cocoeval import _runner_images, _runner_kw, _first_pass_gt
    imgs = _runner_images(5, seed=23)
    cat_ids = [1 + label % 12 for label in range(80)]
    gt = _first_pass_gt(imgs, cat_ids, seed=4)
    params = C.CocoParams2(use_cats=1, cat_ids=[5, 2, 999, 1])
    sd, kw = _runner_kw(2, 'bits')
    runner = CocoEvalRunner(sd, C.CocoGroundTruth(gt), cat_ids, metrics=('bbox', 'segm', 'proposal'), params=params,
                            **kw)
    bbox, segm, seen, ids = [], [], set(), {}

    def collect():                                    # a record is valid until its slot is reused
        for k, images in enumerate(runner.slot_images):
            for m in images:
                if m['ticket'] in seen:
                    continue
                seen.add(m['ticket'])
                r = runner.result(m['ticket'])
                cnt = int(r['count'][0])
                r['segms'] = rle.encode_planes(r['mask_bits'][:cnt].numpy(), m['ori_shape'][:2])
                b, s = coco.coco_json(r, ids[m['ticket']], cat_ids)
                bbox.extend(b)
                segm.extend(dict(x, segmentation={'size': x['segmentation']['size'],
                                                  'counts': x['segmentation']['counts']}) for x in s)
    for n, img in enumerate(imgs):
        before = runner.dispatched
        ids[runner.i] = 1000 + n
        runner.submit(img.pin_memory(), 1000 + n)
        if runner.dispatched != before:
            collect()
    res = runner.evaluate()
    torch.cuda.synchronize()
    collect()
    ref = C.evaluate_json(C.CocoGroundTruth(gt), cat_ids, bbox_json=bbox, segm_json=segm, params=params, proposal=True)
    for m in ('bbox', 'segm', 'proposal'):
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(res['arrays'][m][key], ref['arrays'][m][key]), (m, key)
    assert res['AR@100'] == ref['AR@100'] and res['bbox_mAP'] == ref['bbox_mAP']
    _same_arrays(res['arrays']['proposal'], P.run(gt, bbox, 'bbox', use_cats=0, max_dets=[100, 300, 1000]), 'ar')


def test_params2_rejected_before_launch():
    from sipmask_b200 import cocoeval as C
    from test_gpu_coco_analysis import analysis_dataset
    gt, bbox, _ = analysis_dataset(5, n_img=2)
    gt['categories'][2] = dict(id=gt['categories'][2]['id'], name='x')
    g = C.CocoGroundTruth(gt)
    with pytest.raises(ValueError, match='supercategory'):
        C.analyze_json(g, bbox_json=bbox)
    with pytest.raises(ValueError, match='T \\* A'):
        C.evaluate_json(g, g.cat_ids, bbox_json=bbox, params=C.CocoParams2(iou_thrs=np.linspace(.1, .9, 17)))
    with pytest.raises(ValueError, match='1000'):
        C.evaluate_json(g, g.cat_ids, bbox_json=bbox, params=C.CocoParams2(max_dets=[1, 10, 1001]))
    with pytest.raises(ValueError, match='100'):                 # CocoParams keeps its limit; CocoParams2 takes more
        C.evaluate_json(g, g.cat_ids, bbox_json=bbox, params=C.CocoParams(max_dets=[1, 10, 1000]))
    with pytest.raises(ValueError):
        C.CocoEvaluator(g, g.cat_ids, params=dict(iou_thrs=[.5]))
    with pytest.raises(ValueError, match='proposal_fast'):
        C.CocoEvaluator(g, g.cat_ids, metrics=('bbox', 'proposal_fast'))
    with pytest.raises(ValueError, match='SipMask-benchmark'):
        C.CocoEvaluator(g, g.cat_ids, metrics=('proposal',), benchmark=True)
    with pytest.raises(ValueError, match='cat_ids subset'):
        C.CocoEvaluator(g, g.cat_ids, params=C.CocoParams2(cat_ids=g.cat_ids[:1]), analyze=True)
