"""The device rasterizer (csrc/segm_raster.cu) against the host one, bit for bit: polygons, boxes and run lengths into
planes with their pixel counts and extents, bounds reported through the status word, and the evaluators on top of it."""
import json
import os

import numpy as np
import pytest
import torch

import cocoeval_ref as R
import ytviseval_ref as YR
from test_cocoeval_host import random_polys
from test_segm_raster_host import hard_cases, seeded_polys

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


def _host(segms, h, w):
    from sipmask_b200 import cocoeval as C
    planes = np.stack([C.segm_plane(s, h, w) for s in segms])
    stats = np.array([[a] + list(e) for a, e in (C.plane_stats(p, w) for p in planes)], np.int32)
    return planes, stats


def _check(segms, h, w, name=''):
    from sipmask_b200 import segm_raster as SR
    planes, stats = SR.rasterize(segms, h, w)
    ref_p, ref_s = _host(segms, h, w)
    got = planes.cpu().numpy().view(np.uint32)
    bad = np.argwhere(got != ref_p)
    assert bad.size == 0, (name, len(bad), bad[:5].tolist())
    assert np.array_equal(stats.cpu().numpy(), ref_s), (name, stats.cpu().numpy()[:4], ref_s[:4])


# ---------------------------------------------------------------------------------------------------- polygons
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_polygons_of_the_host_rasterizer_test(seed):
    h, w = 37, 45
    polys = random_polys(seed, h=h, w=w)
    polys += [[3, 3, 3, 3, 20, 3, 20, 3, 20, 15, 3, 15], [0, 0, 30, 30, 30, 0, 0, 30], [-5, -5, 60, -2, 50, 50]]
    _check([[p] for p in polys], h, w)
    _check([random_polys(7, n=3, h=40, w=50), [[2.5, 3.2, 10, 12], [20, 5, 7.7, 30]], [[0, 0, 49.9, 39.9]]], 40, 50)


@pytest.mark.parametrize('case', hard_cases(), ids=[c[0] for c in hard_cases()])
def test_hard_cases(case):
    name, segm, h, w = case
    _check([segm], h, w, name)


@pytest.mark.parametrize('h,w,n,seed', [(60, 83, 40, 1), (480, 640, 24, 2), (333, 500, 16, 3), (1080, 1920, 6, 4)])
def test_seeded_polygons(h, w, n, seed):
    polys = seeded_polys(seed, n, h, w)
    segms = [[p] for p in polys] + [polys[:3], polys[3:6]]        # and two merges of overlapping rings
    _check(segms, h, w)


# ---------------------------------------------------------------------------------------------------- run lengths
def _blobs(seed, n, h, w):
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        m = np.zeros((h, w), bool)
        for _ in range(int(rng.integers(1, 5))):
            y0, x0 = int(rng.integers(0, h)), int(rng.integers(0, w))
            m[y0:y0 + int(rng.integers(1, h)), x0:x0 + int(rng.integers(1, w))] ^= True
        out.append(m | (rng.random((h, w)) < 0.02))
    return out


def test_run_lengths():
    h, w = 7, 9
    segms = [{'size': [h, w], 'counts': c} for c in ([63], [0, 63], [5, 0, 0, 10, 48], [0, 3, 0, 0, 4, 56], [10, 5, 0, 5, 43],
                                                     [62, 1], [3, 4, 56, 0])]
    _check(segms, h, w)


@pytest.mark.parametrize('h,w', [(33, 70), (100, 31), (427, 640)])
def test_encoded_blobs_round_trip(h, w):
    from sipmask_b200 import rle, segm_raster as SR
    masks = _blobs(11, 12, h, w) + [np.zeros((h, w), bool), np.ones((h, w), bool)]
    segms = []
    for i, m in enumerate(masks):
        e = rle.encode(m)
        segms.append({'size': e['size'], 'counts': e['counts'] if i % 2 else rle.counts(m).tolist()})
    planes, stats = SR.rasterize(segms, h, w)
    bits = np.unpackbits(planes.cpu().numpy().view(np.uint8), axis=-1, bitorder='little')[:, :, :w].astype(bool)
    assert np.array_equal(bits, np.stack(masks))
    assert stats[:, 0].cpu().tolist() == [int(m.sum()) for m in masks]
    _check(segms, h, w)


def test_golden_strings():
    with open(os.path.join(HERE, 'golden', 'ref_coco_json.json')) as f:
        found = []

        def walk(o):
            if isinstance(o, dict):
                if 'counts' in o and 'size' in o:
                    found.append(o)
                for v in o.values():
                    walk(v)
            elif isinstance(o, list):
                for v in o:
                    walk(v)
        walk(json.load(f))
    assert found
    by_size = {}
    for s in found:
        by_size.setdefault(tuple(s['size']), []).append(s)
    for (h, w), segms in by_size.items():
        _check(segms, h, w)


# ---------------------------------------------------------------------------------------------------- status
def test_out_of_range_items_set_the_status_and_write_nothing():
    from sipmask_b200 import _lib as L, ops, segm_raster as SR
    h, w, pitch = 20, 40, 2
    pack = SR.SegmPack()
    pack.add([[2, 2, 30, 2, 30, 15, 2, 15]], h, w, 0)
    pack.add({'size': [h, w], 'counts': [100, 50, 650]}, h, w, 1)
    good, xy, counts = pack.arrays()
    ref, _ = _host([[[2, 2, 30, 2, 30, 15, 2, 15]], {'size': [h, w], 'counts': [100, 50, 650]}], h, w)
    bad = []
    for field, row, value in (('plane', 0, 2), ('plane', 1, -1), ('off', 0, 1), ('n', 1, 4), ('off', 1, -1), ('kind', 0, 7),
                              ('w', 0, 41), ('h', 1, 21), ('w', 1, 65)):
        items = good.copy()
        items[field][row] = value
        bad.append((field, row, items))
    for field, row, items in bad:
        dev = torch.device('cuda')
        views = SR.upload([items, xy, counts], dev)
        guard = 64
        buf = torch.full((2 * h * pitch + 2 * guard,), 0x5a5a5a5a, dtype=torch.int32, device=dev)
        planes = buf[guard:guard + 2 * h * pitch]
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        stats = torch.full((2, 5), -7, dtype=torch.int32, device=dev)
        ops.segm_raster(views[0], 2, views[1], pack.n_xy, views[2], pack.n_counts, h * w, w, planes, 2, h * pitch, pitch,
                        status, area=stats, area_stride=5, ext=stats[:, 1:], ext_stride=5)
        torch.cuda.synchronize()
        assert int(status.item()) == 1, (field, row)
        out = buf.cpu().numpy()
        assert (out[:guard] == 0x5a5a5a5a).all() and (out[-guard:] == 0x5a5a5a5a).all(), (field, row)
        got = out[guard:-guard].view(np.uint32).reshape(2, h, pitch)
        assert np.array_equal(got[1 - row], ref[1 - row]), (field, row)          # the other item is rasterized
        assert not got[row].any(), (field, row)                                  # the refused one wrote nothing
        with pytest.raises(L.SmbError, match='rasterizer'):
            SR.check_status(status)


# ---------------------------------------------------------------------------------------------------- evaluators
def _poly_dataset(seed):
    """test_gpu_cocoeval's seeded dataset, with every third polygon ground truth replaced by rings (several per
    annotation, reaching outside the canvas) and every fourth by frBbox boxes."""
    from test_gpu_cocoeval import random_dataset
    gt, bbox, segm = random_dataset(seed)
    hw = {im['id']: (im['height'], im['width']) for im in gt['images']}
    n = 0
    for a in gt['annotations']:
        if isinstance(a['segmentation'], list):
            h, w = hw[a['image_id']]
            n += 1
            if n % 3 == 0:
                a['segmentation'] = seeded_polys(seed * 100 + n, 1 + n % 3, h, w, kmax=30)
            elif n % 4 == 0:
                a['segmentation'] = [list(a['bbox']), [1.5, 2.5, 10, 10]]
    return gt, bbox, segm


@pytest.mark.parametrize('seed', [0, 1])
def test_staged_ground_truth_equals_host_image(seed):
    from sipmask_b200 import cocoeval as C
    gt, _, _ = _poly_dataset(seed)
    g = C.CocoGroundTruth(gt)
    ev = C.CocoEvaluator(g, g.cat_ids, metrics=('segm',))
    for i in g.img_ids:
        rows, off, planes = g.image(i)
        st = ev.stage_gt(i)
        assert st['n_gt'] == len(rows) and st['off'].cpu().tolist() == off.tolist()
        if not len(rows):
            continue
        ev._raster_gt(st)
        got = np.frombuffer(st['rows'].cpu().numpy().tobytes()[:len(rows) * C.GT_DTYPE.itemsize], C.GT_DTYPE)
        for key in ('box', 'area', 'id', 'crowd', 'area_mask', 'ext'):
            assert np.array_equal(got[key], rows[key]), (i, key)
        assert got['plane'].tolist() == [r * planes[0].size for r in range(len(rows))]
        assert np.array_equal(st['planes'].cpu().numpy().view(np.uint32).reshape(planes.shape), planes), i
    assert int(ev.raster_status.item()) == 0


@pytest.mark.parametrize('seed', [0, 1])
def test_coco_evaluate_json_with_polygon_ground_truth(seed):
    from sipmask_b200 import cocoeval as C
    from test_gpu_cocoeval import _assert_same
    gt, bbox, segm = _poly_dataset(seed)
    g = C.CocoGroundTruth(gt)
    res = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, chunk=5)
    _assert_same(res, {'bbox': R.run(gt, bbox, 'bbox'), 'segm': R.run(gt, segm, 'segm')})


def _ytvis_dataset(seed):
    """test_gpu_ytviseval's seeded dataset with some ground-truth frames as polygons and boxes."""
    from test_gpu_ytviseval import _synthetic
    ann, res = _synthetic(seed)
    hw = {v['id']: (v['height'], v['width']) for v in ann['videos']}
    n = 0
    for a in ann['annotations']:
        h, w = hw[a['video_id']]
        for f, s in enumerate(a['segmentations']):
            n += 1
            if s is None or n % 3:
                continue
            s = seeded_polys(seed * 1000 + n, 1 + n % 2, h, w, kmax=20) if n % 2 else [[3.5, 2.0, w / 3.0, h / 2.0]]
            a['segmentations'][f] = s
            a['areas'][f] = float(R.ann_to_mask(s, h, w).sum())
    return ann, res


@pytest.mark.parametrize('seed', [0, 1])
def test_ytvis_staged_frames_and_evaluate_json(seed):
    from sipmask_b200.ytviseval import GTF_DTYPE, YtvisEvaluator, YtvisGroundTruth, evaluate_json
    from test_gpu_ytviseval import _same
    ann, res = _ytvis_dataset(seed)
    gt = YtvisGroundTruth(ann)
    ev = YtvisEvaluator(gt, slots=1, objects=4, max_gts=8)
    for vid in gt.vid_ids:
        v = gt.videos[vid]
        ev.begin_video(vid, 0)
        total = np.zeros(8, np.int64)
        for f in range(v['length']):
            rows, planes, areas = gt.frame(vid, f)
            st = ev.stage_frame(vid, f)
            dets = torch.zeros(max(planes[0].size if len(planes) else 1, 1), dtype=torch.int32, device='cuda')
            ovl = ev.overlap([st], [dets.data_ptr()], dets.numel(), st['pitch'], 1, n_det=[0])
            ev.scatter(ovl, torch.full((1, 1), -1, dtype=torch.int32, device='cuda'))
            ev.commit_frame(st)
            np.add.at(total, rows['g'], areas)
            if not len(rows):
                continue
            got = np.frombuffer(ovl['gts'].cpu().numpy().tobytes()[:len(rows) * GTF_DTYPE.itemsize], GTF_DTYPE)
            assert np.array_equal(got['ext'], rows['ext']) and got['g'].tolist() == rows['g'].tolist(), (vid, f)
            assert ovl['gt_area'].cpu().tolist()[:len(rows)] == areas.tolist(), (vid, f)
            assert np.array_equal(st['planes'].cpu().numpy().view(np.uint32).reshape(planes.shape), planes), (vid, f)
        assert ev.gt_area[0].cpu().tolist() == total.tolist(), vid
        ev.abort_video(vid)
    assert int(ev.raster_status.item()) == 0 and int(ev.status.item()) == 0
    _same(evaluate_json(YtvisGroundTruth(ann), res, chunk=2), YR.run(ann, res))


# ---------------------------------------------------------------------------------------------------- errors
def test_malformed_segmentations_raise_from_submit_and_the_runner_goes_on():
    from sipmask_b200 import cocoeval as C
    from sipmask_b200.serving import CocoEvalRunner
    from test_gpu_cocoeval import _runner_images, _runner_kw
    imgs = _runner_images(2, seed=22)
    bad = [{'size': [4, 4], 'counts': [3, 20]}, [[1, 2]], {'counts': 'abc'}, None, {'size': [0, 0], 'counts': '0#'}]
    gt = dict(images=[], categories=[dict(id=1)], annotations=[])
    for n, seg in enumerate([[[1, 1, 1, 31, 31, 31, 31, 1]]] + bad):
        h, w = imgs[n % 2].shape[:2]
        if isinstance(seg, dict) and 'size' in seg:
            seg = dict(seg, size=[h, w])
        gt['images'].append(dict(id=n + 1, height=h, width=w))
        gt['annotations'].append(dict(id=n + 1, image_id=n + 1, category_id=1, bbox=[1.0, 1.0, 30.0, 30.0], area=900.0,
                                      iscrowd=0, segmentation=seg))
    sd, kw = _runner_kw(1, 'rle')
    g = C.CocoGroundTruth(gt)
    runner = CocoEvalRunner(sd, g, [1] * 80, **kw)
    for n in range(1, len(bad) + 1):
        with pytest.raises(ValueError) as dev:
            runner.submit(imgs[n % 2].pin_memory(), n + 1)
        with pytest.raises(ValueError) as host:
            g.image(n + 1)
        assert str(dev.value) == str(host.value)
        assert runner.i == 0 and not runner._eval_rows
    runner.submit(imgs[0].pin_memory(), 1)
    try:
        assert 'segm_mAP' in runner.evaluate()
    except ValueError as e:                                    # synthetic weights may detect nothing in one image
        assert 'empty' in str(e)
