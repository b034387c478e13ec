"""CPU checks of the YouTube-VIS evaluation: hand-derived known answers of the test restatement of YTVOSeval
(ytviseval_ref), the ground-truth parsing of polygons, uncompressed and compressed RLE with absent frames, and the checks
made before anything is enqueued."""
import numpy as np
import pytest

import ytviseval_ref as R


def _rect(h, w, y0, x0, y1, x1):
    m = np.zeros((h, w), bool)
    m[y0:y1, x0:x1] = True
    return m


def _rle(m, compressed=True):
    from sipmask_b200 import rle
    if compressed:
        r = rle.encode(m)
        return {'size': r['size'], 'counts': r['counts'].decode()}
    return {'size': [int(m.shape[0]), int(m.shape[1])], 'counts': [int(c) for c in rle.counts(m)]}


def _gt(objs, hw=(40, 60), length=2, cats=(1, 2), vid=1, videos=None):
    """objs: dicts(masks (None per absent frame), cat, crowd, id, areas)."""
    vids = videos or [(vid, hw, length)]
    out = dict(videos=[dict(id=v, height=s[0], width=s[1], length=n) for v, s, n in vids],
               categories=[dict(id=c) for c in cats], annotations=[])
    for n, o in enumerate(objs):
        ms = o['masks']
        out['annotations'].append(dict(
            id=o.get('id', n + 1), video_id=o.get('vid', vid), category_id=o.get('cat', 1), iscrowd=o.get('crowd', 0),
            segmentations=[None if m is None else _rle(m) for m in ms],
            areas=o.get('areas', [None if m is None else int(m.sum()) for m in ms])))
    return out


def _res(masks, score, cat=1, vid=1):
    return dict(video_id=vid, score=score, category_id=cat, segmentations=[None if m is None else _rle(m) for m in masks])


def known_cases():
    """(name, ground truth, results) of the hand-derived cases; the GPU tests run the kernels on them too."""
    H, W = 40, 60
    a, b = _rect(H, W, 0, 0, 2, 2), _rect(H, W, 1, 0, 3, 2)            # areas 4 and 4, overlap 2
    c = _rect(H, W, 10, 10, 12, 13)                                    # area 6
    z = np.zeros((H, W), bool)
    cases = []
    # IoU 2 / (6 + 6) = 1/6 with the detection absent in frame 1: below every threshold
    cases.append(('absent_frame', _gt([dict(masks=[b, c])]), [_res([a, None], 0.9)]))
    # an empty mask that is present adds nothing to the union: IoU 4 / 4 = 1 although the detection is absent in frame 1
    cases.append(('empty_present', _gt([dict(masks=[a, z])]), [_res([a, None], 0.9)]))
    # u == 0: an empty ground truth and an empty detection give IoU 0, and avg_area 0 (zeros dropped)
    cases.append(('u_zero', _gt([dict(masks=[z, None])]), [_res([z, None], 0.9)]))
    # a perfect detection and a wrong one
    cases.append(('ap1', _gt([dict(masks=[a, c])]), [_res([a, c], 0.9)]))
    cases.append(('ap0', _gt([dict(masks=[a, c])]), [_res([c, a], 0.9)]))
    # a crowd ground truth absorbs a detection (ignored); a true positive on the other object
    cases.append(('crowd', _gt([dict(masks=[c, c], crowd=1), dict(masks=[a, a])]),
                  [_res([c, c], 0.95), _res([a, a], 0.6)]))
    # objects exactly on the 128^2 and 256^2 boundaries: in both neighbouring ranges
    for side, name in ((128, 'edge128'), (256, 'edge256')):
        m = _rect(side + 2, side + 2, 1, 1, side + 1, side + 1)
        cases.append((name, _gt([dict(masks=[m])], hw=(side + 2, side + 2), length=1), [_res([m], 0.8)]))
    return cases


def _case(name):
    return [c for c in known_cases() if c[0] == name][0]


def test_iou_seq_hand_derived():
    H, W = 40, 60
    a, b, c = _rect(H, W, 0, 0, 2, 2), _rect(H, W, 1, 0, 3, 2), _rect(H, W, 10, 10, 12, 13)
    z = np.zeros((H, W), bool)
    assert R.iou_seq([a, None], [b, c]) == 2 / 12
    assert R.iou_seq([a, None], [a, z]) == 1.0
    assert R.iou_seq([z, None], [b, None]) == 0.0
    assert R.iou_seq([None, None], [None, z]) == 0.0            # u == 0
    assert R.iou_seq([a, z], [None, c]) == 0.0


def test_avg_area_drops_none_and_zeros():
    assert R.avg_area([None, 0, 4, 8]) == 6.0
    assert R.avg_area([None, 0]) == 0 and R.avg_area([]) == 0
    from sipmask_b200.ytviseval import avg_area
    assert avg_area([None, 0, 4, 8]) == 6.0 and avg_area([0, None]) == 0


def test_known_absent_frame_and_empty_present():
    _, gt, dt = _case('absent_frame')
    e = R.run(gt, dt)
    assert e.ious[1, 1][0, 0] == 2 / 12 and e.stats[0] == 0
    _, gt, dt = _case('empty_present')
    e = R.run(gt, dt)
    assert e.ious[1, 1][0, 0] == 1.0 and np.isclose(e.stats[0], 1.0)


def test_known_u_zero():
    _, gt, dt = _case('u_zero')
    e = R.run(gt, dt)
    assert e.ious[1, 1][0, 0] == 0.0
    assert e.stats[0] == 0 and e.stats[3] == 0                  # avg_area 0 for both: 'small'


def test_known_ap1_ap0_crowd():
    e = R.run(*_case('ap1')[1:])
    assert np.isclose(e.stats[0], 1.0) and np.isclose(e.stats[8], 1.0)
    e = R.run(*_case('ap0')[1:])
    assert e.stats[0] == 0 and e.stats[8] == 0
    e = R.run(*_case('crowd')[1:])
    assert np.isclose(e.stats[0], 1.0)                          # the crowd match is ignored, not a false positive
    ev = e.evaluate_img(1, 1, R.AREA_RNG[0], 100)
    assert ev['dtIgnore'][0].tolist() == [True, False]


def test_known_area_range_boundaries():
    for name, both in (('edge128', (1, 2)), ('edge256', (2, 3))):
        e = R.run(*_case(name)[1:])
        for a in range(1, 4):
            p = e.precision[0, 0, 0, a, 2]
            assert (np.isclose(p, 1.0) if a in both else p == -1), (name, a, p)


def test_ground_truth_parsing_polygon_rle_and_absent_frames():
    from sipmask_b200.ytviseval import YtvisGroundTruth
    import cocoeval_ref as C
    H, W = 37, 70
    m1 = _rect(H, W, 3, 40, 20, 69)
    poly = [[5.0, 4.0, 30.5, 4.0, 30.5, 25.25, 5.0, 25.25]]
    segs = [poly, None, _rle(m1, compressed=False), _rle(m1), None]
    ann = dict(videos=[dict(id=3, height=H, width=W, length=5)], categories=[dict(id=2)],
               annotations=[dict(id=11, video_id=3, category_id=2, iscrowd=0, segmentations=segs,
                                 areas=[500.0, None, 493, 0, None])])
    gt = YtvisGroundTruth(ann)
    assert gt.anns[3][0]['avg_area'] == np.array([500.0, 493]).mean()
    for f, s in enumerate(segs):
        rows, planes, areas = gt.frame(3, f)
        if s is None:
            assert len(rows) == 0
            continue
        want = C.ann_to_mask(s, H, W)
        got = np.unpackbits(planes[0].view(np.uint8), axis=1, bitorder='little')[:, :W].astype(bool)
        assert np.array_equal(got, want) and areas[0] == want.sum() and rows[0]['g'] == 0
    rows, off = gt.video(3)
    assert off.tolist() == [0, 1] and rows[0]['id'] == 11


def test_checks_before_anything_is_enqueued():
    from sipmask_b200.ytviseval import YtvisGroundTruth, evaluate_json
    _, ann, dt = _case('ap1')
    gt = YtvisGroundTruth(ann)
    with pytest.raises(ValueError, match='not in the ground truth'):
        gt.check_frame(5, 0, (40, 60))
    with pytest.raises(ValueError, match='frame of'):
        gt.check_frame(1, 0, (40, 61))
    with pytest.raises(ValueError, match='has 2 frames'):
        gt.check_frame(1, 2, (40, 60))
    with pytest.raises(ValueError, match='max_gts'):
        gt.check_frame(1, 0, (40, 60), max_gts=0)
    with pytest.raises(ValueError, match='not in the ground truth'):
        evaluate_json(gt, [dict(dt[0], video_id=9)])
    with pytest.raises(ValueError, match='segmentations'):
        evaluate_json(gt, [dict(dt[0], segmentations=dt[0]['segmentations'][:1])])
    with pytest.raises(ValueError, match='category'):
        evaluate_json(gt, [dict(dt[0], category_id=7)])
    with pytest.raises(ValueError, match='empty'):
        evaluate_json(gt, [])
    bad = dict(ann, annotations=[dict(ann['annotations'][0], segmentations=[None])])
    with pytest.raises(ValueError, match='segmentations'):
        YtvisGroundTruth(bad)
