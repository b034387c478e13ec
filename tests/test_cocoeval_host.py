"""CPU checks of the COCO evaluation: hand-derived known answers of the test restatement of COCOeval (cocoeval_ref), the
library's C rasterizer against the restatement's Python one, the compressed-string decoder, and malformed inputs."""
import numpy as np
import pytest

import cocoeval_ref as R


def _gt(anns, cats=(1,), images=((1, 400, 500),)):
    out = dict(images=[dict(id=i, height=h, width=w) for i, h, w in images], categories=[dict(id=c) for c in cats],
               annotations=[])
    for n, a in enumerate(anns):
        x, y, w, h = a['bbox']
        out['annotations'].append(dict(id=a.get('id', n + 1), image_id=a.get('image_id', 1), category_id=a.get('cat', 1),
                                       bbox=[x, y, w, h], area=a.get('area', w * h), iscrowd=a.get('crowd', 0),
                                       segmentation=[[x, y, x, y + h, x + w, y + h, x + w, y]]))
    return out


def _det(bbox, score, cat=1, image_id=1):
    return dict(image_id=image_id, category_id=cat, bbox=list(bbox), score=score)


def known_cases():
    """(name, ground truth, bbox results, expectation on the restatement)."""
    cases = []
    # one medium ground truth (area 2000), one detection at IoU 1640 / 2000 = 0.82: matched at .50 ... .80
    cases.append(('iou082', _gt([dict(bbox=[10, 10, 50, 40])]), [_det([10, 10, 41, 40], 0.9)]))
    # a false positive ranked above the true positive: precision 0.5 after the envelope
    cases.append(('fp_first', _gt([dict(bbox=[10, 10, 50, 40])]),
                  [_det([300, 300, 50, 40], 0.9), _det([10, 10, 50, 40], 0.8)]))
    # a crowd region absorbs three detections, which are ignored; one true positive elsewhere
    cases.append(('crowd', _gt([dict(bbox=[0, 0, 100, 100], crowd=1), dict(bbox=[200, 200, 50, 50])]),
                  [_det([10, 10, 20, 20], 0.9), _det([40, 40, 30, 30], 0.8), _det([5, 60, 20, 30], 0.7),
                   _det([200, 200, 50, 50], 0.6)]))
    # an unmatched small detection: counted in 'all', ignored in 'medium'
    cases.append(('area_ignore', _gt([dict(bbox=[10, 10, 50, 40])]),
                  [_det([300, 300, 10, 10], 0.9), _det([10, 10, 50, 40], 0.8)]))
    # maxDets truncation per (image, category)
    cases.append(('maxdets', _gt([dict(bbox=[10, 10, 50, 40]), dict(bbox=[10, 10, 50, 40], image_id=2)],
                                 images=((1, 400, 500), (2, 400, 500))),
                  [_det([300, 300, 50, 40], 0.9), _det([10, 10, 50, 40], 0.8), _det([10, 10, 50, 40], 0.95, image_id=2)]))
    # detections of a category without ground truth
    cases.append(('no_gt_cat', _gt([dict(bbox=[10, 10, 50, 40])], cats=(1, 2)),
                  [_det([10, 10, 50, 40], 0.9), _det([10, 10, 50, 40], 0.8, cat=2)]))
    # two identical ground truths: the tie goes to the later one
    cases.append(('tie', _gt([dict(bbox=[10, 10, 50, 40], id=7), dict(bbox=[10, 10, 50, 40], id=9)]),
                  [_det([10, 10, 50, 40], 0.9)]))
    return cases


def _case(name):
    return [c for c in known_cases() if c[0] == name][0]


def test_known_iou082():
    _, gt, dt = _case('iou082')
    e = R.run(gt, dt, 'bbox')
    assert np.isclose(e.stats[0], 0.7) and np.isclose(e.stats[1], 1) and np.isclose(e.stats[2], 1)   # 1 / (1 + eps)
    assert e.stats[3] == -1 and np.isclose(e.stats[4], 0.7) and e.stats[5] == -1
    assert np.allclose(e.precision[:7, :, 0, 0, 2], 1) and e.precision[7:, :, 0, 0, 2].max() == 0


def test_known_fp_first():
    _, gt, dt = _case('fp_first')
    e = R.run(gt, dt, 'bbox')
    assert np.all(e.precision[:, :, 0, 0, 2] == 0.5) and e.stats[0] == 0.5


def test_known_crowd_absorbs():
    _, gt, dt = _case('crowd')
    e = R.run(gt, dt, 'bbox')
    ev = e.eval_imgs[0]                                        # category 1, area 'all', image 1
    assert ev['dtIgnore'][:, :3].all() and not ev['dtIgnore'][:, 3].any()
    assert np.isclose(e.stats[0], 1)


def test_known_area_ignore():
    _, gt, dt = _case('area_ignore')
    e = R.run(gt, dt, 'bbox')
    assert e.stats[0] == 0.5 and np.isclose(e.stats[4], 1)


def test_known_maxdets_per_image():
    _, gt, dt = _case('maxdets')
    e = R.run(gt, dt, 'bbox')
    assert e.stats[6] == 0.5 and e.stats[7] == 1


def test_known_category_without_gt():
    _, gt, dt = _case('no_gt_cat')
    e = R.run(gt, dt, 'bbox')
    assert np.all(e.precision[:, :, 1] == -1) and np.all(e.recall[:, 1] == -1) and np.all(e.scores[:, :, 1] == -1)


def test_known_tie_goes_to_later_gt():
    _, gt, dt = _case('tie')
    e = R.run(gt, dt, 'bbox')
    assert np.all(e.eval_imgs[0]['dtMatches'][:, 0] == 9)


# ---------------------------------------------------------------------------------------------------- C rasterizer
def random_polys(seed, n=60, h=37, w=45):
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        k = int(rng.integers(3, 9))
        xy = np.stack([rng.uniform(-8, w + 8, k), rng.uniform(-8, h + 8, k)], 1)
        if i % 4 == 0:                                         # integer and half-integer vertices, duplicates
            xy = np.round(xy * 2) / 2
            xy = np.repeat(xy, rng.integers(1, 3, k), axis=0)
        if i % 5 == 0:
            xy = xy * rng.uniform(0.05, 0.3)                  # tiny rings near the origin
        out.append(xy.reshape(-1).tolist())
    return out


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_c_rasterizer_equals_restatement(seed):
    from sipmask_b200 import cocoeval as C
    h, w = 37, 45
    polys = random_polys(seed, h=h, w=w)
    polys.append([3, 3, 3, 3, 20, 3, 20, 3, 20, 15, 3, 15])    # duplicate consecutive vertices: the INT_MIN path
    polys.append([0, 0, 30, 30, 30, 0, 0, 30])                # self-intersecting
    polys.append([-5, -5, 60, -2, 50, 50])                    # beyond every edge
    for p in polys:
        assert C.poly_counts(p, h, w).tolist() == R.rle_fr_poly(p, h, w), p
        plane = C.segm_plane([p], h, w)
        bits = np.unpackbits(plane.view(np.uint8), axis=-1, bitorder='little')[:, :w].astype(bool)
        assert np.array_equal(bits, R.ann_to_mask([p], h, w))


def test_c_rasterizer_unions_and_boxes():
    from sipmask_b200 import cocoeval as C
    h, w = 40, 50
    segms = [random_polys(7, n=3, h=h, w=w), [[2.5, 3.2, 10, 12], [20, 5, 7.7, 30]], [[0, 0, 49.9, 39.9]]]
    for s in segms:
        plane = C.segm_plane(s, h, w)
        bits = np.unpackbits(plane.view(np.uint8), axis=-1, bitorder='little')[:, :w].astype(bool)
        assert np.array_equal(bits, R.ann_to_mask(s, h, w))
    area, ext = C.plane_stats(C.segm_plane(segms[1], h, w), w)
    assert area == int(R.ann_to_mask(segms[1], h, w).sum()) and ext[1] > ext[0]


def test_string_decoder_round_trips():
    from sipmask_b200 import cocoeval as C, rle
    rng = np.random.default_rng(3)
    for _ in range(50):
        m = rng.random((int(rng.integers(1, 40)), int(rng.integers(1, 40)))) < rng.uniform(0.05, 0.95)
        c = rle.counts(m)
        s = rle.to_string(c)
        assert C.string_to_counts(s).tolist() == c.tolist() == R.rle_fr_string(s)
        plane = C.segm_plane({'size': list(m.shape), 'counts': s}, *m.shape)
        bits = np.unpackbits(plane.view(np.uint8), axis=-1, bitorder='little')[:, :m.shape[1]].astype(bool)
        assert np.array_equal(bits, m)
    assert C.string_to_counts(b'').size == 0


def test_malformed_inputs_raise():
    from sipmask_b200 import cocoeval as C
    with pytest.raises(ValueError):
        C.string_to_counts('0#')                              # character below '0'
    with pytest.raises(ValueError):
        C.string_to_counts('o')                               # continuation bit without a next character
    with pytest.raises(ValueError):
        C.segm_plane({'size': [4, 4], 'counts': [3, 20]}, 4, 4)   # runs past the canvas
    with pytest.raises(ValueError):
        C.segm_plane({'size': [4, 5], 'counts': [20]}, 4, 4)      # size differs from the image
    with pytest.raises(ValueError):
        C.segm_plane([[1, 2]], 4, 4)                          # a first polygon of 2 numbers
    with pytest.raises(ValueError):
        C.segm_plane({'counts': 'abc'}, 4, 4)
    gt = _gt([dict(bbox=[1, 2, 3, 4])])
    bad = dict(gt, annotations=[dict(gt['annotations'][0])])
    del bad['annotations'][0]['iscrowd']
    with pytest.raises(ValueError):
        C.CocoGroundTruth(bad)
    bad = dict(gt, annotations=[dict(gt['annotations'][0], bbox=[1, 2, 3])])
    with pytest.raises(ValueError):
        C.CocoGroundTruth(bad)
    with pytest.raises(ValueError):
        C.CocoGroundTruth(dict(gt, categories=[]))
    g = C.CocoGroundTruth(gt)
    assert g.img_ids == [1] and g.cat_ids == [1]
    rows, off, planes = g.image(1)
    assert off.tolist() == [0, 1] and rows[0]['area_mask'] == int(R.ann_to_mask(gt['annotations'][0]['segmentation'],
                                                                                  400, 500).sum())


def test_summarize_matches_restatement():
    from sipmask_b200 import cocoeval as C
    for name, gt, dt in known_cases():
        e = R.run(gt, dt, 'bbox')
        assert np.array_equal(C.summarize(e.precision, e.recall), e.stats), name
