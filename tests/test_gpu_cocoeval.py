"""GPU checks of the device COCO evaluation (sipmask_b200.cocoeval) against the test restatement of pycocotools' COCOeval
(cocoeval_ref): precision / recall / scores arrays equal element for element, and the 12 stats equal."""
import ctypes

import numpy as np
import pytest
import torch

import cocoeval_ref as R

pytestmark = pytest.mark.gpu


def _mask_rle(m):
    from sipmask_b200 import rle
    e = rle.encode(m)
    return {'size': e['size'], 'counts': e['counts'].decode()}


def _rect(h, w, x0, y0, x1, y1):
    m = np.zeros((h, w), bool)
    m[max(y0, 0):max(y1, 0), max(x0, 0):max(x1, 0)] = True
    return m


def _assert_same(res, ref_by_metric, name=''):
    for m, ref in ref_by_metric.items():
        a = res['arrays'][m]
        for key in ('precision', 'recall', 'scores'):
            x, y = a[key], getattr(ref, key)
            bad = np.argwhere(x != y)
            assert bad.size == 0, (name, m, key, len(bad), [(tuple(i), x[tuple(i)], y[tuple(i)]) for i in bad[:4]])
        assert np.array_equal(res['stats'][m], ref.stats), (name, m, res['stats'][m], ref.stats)


def _segm_results(gt, bbox_results):
    hw = {im['id']: (im['height'], im['width']) for im in gt['images']}
    out = []
    for r in bbox_results:
        h, w = hw[r['image_id']]
        x, y, bw, bh = [int(round(v)) for v in r['bbox']]
        out.append(dict(image_id=r['image_id'], category_id=r['category_id'], score=r['score'],
                        segmentation=_mask_rle(_rect(h, w, x, y, x + bw, y + bh))))
    return out


def test_known_answers_on_device():
    from test_cocoeval_host import known_cases
    from sipmask_b200 import cocoeval as C
    for name, gt, dt in known_cases():
        g = C.CocoGroundTruth(gt)
        cat_ids = g.cat_ids
        sg = _segm_results(gt, dt)
        res = C.evaluate_json(g, cat_ids, bbox_json=dt, segm_json=sg)
        _assert_same(res, {'bbox': R.run(gt, dt, 'bbox'), 'segm': R.run(gt, sg, 'segm')}, name)


def random_dataset(seed, n_img=14, cats=(1, 3, 7), big=False):
    """Polygon / uncompressed / compressed ground truth, crowds, repeated scores, IoUs of exactly 3/4, images without
    ground truth or without detections, more than 100 detections of a category in one image and across images.
    big: 260 false positives of one category in every odd image, so that one category has more than 600 rows after the
    per-image cut at 100 and single images hold more than 256 detections of it (several chunks of every device loop)."""
    from sipmask_b200 import rle
    rng = np.random.default_rng(seed)
    gt = dict(images=[], categories=[dict(id=c) for c in cats], annotations=[])
    bbox, segm = [], []
    scores = [0.9, 0.75, 0.5, 0.5, 0.3, 0.125]
    aid = 0
    for i in range(n_img):
        img = 100 + 3 * i
        h, w = int(rng.integers(60, 120)), int(rng.integers(70, 140))
        gt['images'].append(dict(id=img, height=h, width=w))
        n_gt = 0 if i % 5 == 1 else int(rng.integers(1, 7))
        masks = []
        for g in range(n_gt):
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
            crowd = int(rng.random() < 0.15)
            area = float(m.sum()) if rng.random() < 0.7 else float(rng.integers(10, 12000))
            gt['annotations'].append(dict(id=aid if rng.random() > 0.05 else 0, image_id=img, category_id=cat,
                                          bbox=[x0, y0, x1 - x0, y1 - y0], area=area, iscrowd=crowd, segmentation=seg))
            masks.append((cat, x0, y0, x1, y1))
        if i % 5 == 2:
            continue                                          # no detections
        dets = []
        for cat, x0, y0, x1, y1 in masks:
            for _ in range(int(rng.integers(1, 4))):
                dx, dy = int(rng.integers(-3, 4)), int(rng.integers(-3, 4))
                dets.append((cat, x0 + dx, y0 + dy, x1 + dx + int(rng.integers(-2, 3)), y1 + dy))
            if x1 - x0 >= 8:                                  # IoU 3/4 exactly with the rectangle
                dets.append((cat, x0, y0, x0 + (x1 - x0) * 3 // 4, y1) if (x1 - x0) % 4 == 0 else (cat, x0, y0, x1, y1))
        many = i == 3 or (big and i % 2 == 1)
        n_fp = (260 if big else 130) if many else int(rng.integers(0, 8))
        for _ in range(n_fp):
            x0, y0 = int(rng.integers(0, w - 5)), int(rng.integers(0, h - 5))
            dets.append((int(cats[0]) if many else int(rng.choice(cats)), x0, y0, x0 + int(rng.integers(2, 40)),
                         y0 + int(rng.integers(2, 40))))
        for cat, x0, y0, x1, y1 in dets:
            s = float(rng.choice(scores)) if rng.random() < 0.5 else float(np.float32(rng.random()))
            bbox.append(dict(image_id=img, category_id=cat, bbox=[float(x0), float(y0), float(x1 - x0), float(y1 - y0)],
                             score=s))
            segm.append(dict(image_id=img, category_id=cat, score=s, segmentation=_mask_rle(_rect(h, w, x0, y0, x1, y1))))
    return gt, bbox, segm


@pytest.mark.parametrize('seed,big', [(0, False), (1, False), (2, True)])
def test_evaluate_json_equals_restatement(seed, big):
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = random_dataset(seed, big=big)
    if big:
        per_cat = {}
        for r in bbox:
            per_cat[(r['image_id'], r['category_id'])] = per_cat.get((r['image_id'], r['category_id']), 0) + 1
        assert sum(min(v, 100) for (i, c), v in per_cat.items() if c == 1) > 600 and max(per_cat.values()) > 256
    g = C.CocoGroundTruth(gt)
    res = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, chunk=5)
    _assert_same(res, {'bbox': R.run(gt, bbox, 'bbox'), 'segm': R.run(gt, segm, 'segm')})
    assert res['bbox_mAP'] == float('{:.3f}'.format(res['stats']['bbox'][0]))


# ---------------------------------------------------------------------------------------------------- engine records
def _geom_rows(metas, benchmark):
    from sipmask_b200 import _lib as L
    from sipmask_b200.postproc import image_geometry
    rows = []
    for img_shape, ori_shape, sf in metas:
        g = image_geometry((img_shape[0] // 8, img_shape[1] // 8), img_shape, ori_shape, sf, benchmark=benchmark)
        rows.append(np.frombuffer(bytes(g), dtype=np.int32))
    return torch.from_numpy(np.stack(rows)).cuda()


def fake_records(seed, benchmark=False, rescoring=False, N=3, max_num=100, ncls=4):
    """A batch of engine records (device tensors), its metas and geometry rows, with a ground truth built from it
    (shifted boxes, grown / shrunk planes as RLE, box polygons, crowds, a category without detections)."""
    from sipmask_b200 import rle
    rng = np.random.default_rng(seed)
    oris = [(90, 120), (77, 101), (64, 150)][:N]
    metas = []
    for oh, ow in oris:
        img = (oh * 4, ow * 4) if not benchmark else (oh * 4 + 3, ow * 4 - 5)
        metas.append(((img[0], img[1], 3), (oh, ow, 3), 4.0))
    cap_h, words = 160, 5
    det = np.zeros((N, max_num, 5), np.float32)
    labels = np.zeros((N, max_num), np.int64)
    count = np.zeros(N, np.int32)
    bits = np.zeros((N, max_num, cap_h, words), np.uint32)
    ms = np.zeros((N, max_num), np.float32)
    for n, (oh, ow) in enumerate(oris):
        k = [max_num, 37, 12][n]
        count[n] = k
        ih, iw = metas[n][0][:2]
        sx, sy = (iw / ow, ih / oh) if benchmark else (1.0, 1.0)
        for j in range(k):
            x0, y0 = rng.uniform(0, ow - 12), rng.uniform(0, oh - 12)
            x1, y1 = x0 + rng.uniform(3, 40), y0 + rng.uniform(3, 40)
            det[n, j, :4] = [x0 * sx, y0 * sy, x1 * sx, y1 * sy]
            det[n, j, 4] = rng.choice([0.9, 0.5, 0.25]) if j % 3 == 0 else rng.random()
            labels[n, j] = rng.integers(0, ncls - 1)          # the last label has no detections
            ms[n, j] = rng.random()
            m = _rect(oh, ow, int(x0), int(y0), int(x1), int(y1))
            pk = np.packbits(np.pad(m, ((0, 0), (0, words * 32 - ow))), axis=-1, bitorder='little')
            bits[n, j, :oh] = pk.view(np.uint32)
    rec = dict(det_bboxes=torch.from_numpy(det).cuda(), det_labels=torch.from_numpy(labels).cuda(),
               count=torch.from_numpy(count).cuda(), mask_bits=torch.from_numpy(bits.view(np.int32)).cuda())
    if rescoring:
        rec['mask_scores'] = torch.from_numpy(ms).cuda()
    geom = _geom_rows(metas, benchmark)
    # ground truth from the records
    cat_ids = [2, 4, 9, 11][:ncls]
    gt = dict(images=[dict(id=10 + n, height=o[0], width=o[1]) for n, o in enumerate(oris)],
              categories=[dict(id=c) for c in cat_ids], annotations=[])
    aid = 0
    for n, (oh, ow) in enumerate(oris):
        for j in range(0, int(count[n]), 2):
            aid += 1
            m = np.unpackbits(bits[n, j, :oh].view(np.uint8), axis=-1, bitorder='little')[:, :ow].astype(bool)
            ys, xs = np.nonzero(m)
            x0, y0, x1, y1 = xs.min() + int(rng.integers(-2, 3)), ys.min(), xs.max() + 1, ys.max() + 1 + int(rng.integers(-2, 3))
            kind = aid % 3
            if kind == 0:
                seg = [[float(x0), float(y0), float(x0), float(y1), float(x1), float(y1), float(x1), float(y0)]]
            else:
                grown = _rect(oh, ow, x0, y0, x1, y1)
                seg = _mask_rle(grown) if kind == 1 else {'size': [oh, ow], 'counts': rle.counts(grown).tolist()}
            gt['annotations'].append(dict(id=aid, image_id=10 + n, category_id=cat_ids[int(labels[n, j])],
                                          bbox=[float(x0), float(y0), float(x1 - x0), float(y1 - y0)],
                                          area=float((x1 - x0) * (y1 - y0)), iscrowd=int(aid % 11 == 0), segmentation=seg))
        aid += 1
        gt['annotations'].append(dict(id=aid, image_id=10 + n, category_id=cat_ids[-1], bbox=[1.0, 1.0, 20.0, 20.0],
                                      area=400.0, iscrowd=0, segmentation=[[1, 1, 1, 21, 21, 21, 21, 1]]))
    return rec, metas, geom, gt, cat_ids


def _record_json(rec, metas, cat_ids, benchmark, ids):
    from sipmask_b200 import coco, rle
    bbox, segm = [], []
    for n, i in enumerate(ids):
        k = int(rec['count'][n])
        ori = metas[n][1][:2]
        one = {key: v[n] for key, v in rec.items()}
        one['count'] = rec['count'][n:n + 1]
        segs = rle.encode_planes(rec['mask_bits'][n, :k].cpu().numpy(), ori)
        one['segms'] = [{'size': s['size'], 'counts': s['counts']} for s in segs]
        b, s = coco.coco_json(one, i, cat_ids, benchmark=benchmark,
                              meta=dict(img_shape=metas[n][0], ori_shape=metas[n][1]))
        bbox += b
        segm += s
    return bbox, segm


@pytest.mark.parametrize('flavour', ['mm', 'bm', 'mm_rescoring'])
def test_records_equal_coco_json_and_restatement(flavour):
    from sipmask_b200 import cocoeval as C
    benchmark, rescoring = flavour == 'bm', flavour == 'mm_rescoring'
    rec, metas, geom, gt, cat_ids = fake_records(5, benchmark=benchmark, rescoring=rescoring)
    g = C.CocoGroundTruth(gt)
    ids = [10, 11, 12]
    ev = C.CocoEvaluator(g, cat_ids, benchmark=benchmark)
    ev.add_records(rec, geom, ids, [m[1] for m in metas])
    res = ev.evaluate()
    bbox, segm = _record_json(rec, metas, cat_ids, benchmark, ids)
    # kernel 2a: its rows equal the json the writers produce, field by field
    dets = _record_rows(rec, geom, cat_ids, g, benchmark)
    for n in range(3):
        js = [r for r in bbox if r['image_id'] == ids[n]]
        ss = [r for r in segm if r['image_id'] == ids[n]]
        k = int(rec['count'][n])
        order = (np.argsort(rec['det_labels'][n, :k].cpu().numpy(), kind='stable') if not benchmark else np.arange(k))
        for q, j in enumerate(order):
            d = dets[n * 100 + j]
            assert list(d['box']) == js[q]['bbox'] and d['score'][0] == js[q]['score'] and d['score'][1] == ss[q]['score']
            assert d['area_box'] == js[q]['bbox'][2] * js[q]['bbox'][3]
            assert g.cat_ids[d['cat']] == js[q]['category_id']
            assert d['area_mask'] == int(R.ann_to_mask(ss[q]['segmentation'], *metas[n][1][:2]).sum())
    ref = C.evaluate_json(g, cat_ids, bbox_json=bbox, segm_json=segm)
    for m in ('bbox', 'segm'):
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(res['arrays'][m][key], ref['arrays'][m][key]), (m, key)
    _assert_same(res, {'bbox': R.run(gt, bbox, 'bbox'), 'segm': R.run(gt, segm, 'segm')})


def _record_rows(rec, geom, cat_ids, g, benchmark):
    from sipmask_b200 import _lib as L, cocoeval as C
    N, mx = rec['det_bboxes'].shape[:2]
    rows = torch.empty(N * mx * C.DET_DTYPE.itemsize, dtype=torch.uint8, device='cuda')
    imgs = torch.zeros(N * C.IMG_DTYPE.itemsize, dtype=torch.uint8, device='cuda')
    st = torch.zeros(1, dtype=torch.int32, device='cuda')
    lc = torch.tensor([g.cat_index[c] for c in cat_ids], dtype=torch.int32, device='cuda')
    bits = rec['mask_bits']
    L.check(L.lib().smb_coco_det_from_record_dev(L.ptr(rec['det_bboxes']), L.ptr(rec['det_labels']), L.ptr(rec['count']),
                                                 L.ptr(rec.get('mask_scores')), L.ptr(bits), N, mx, bits.shape[2],
                                                 bits.shape[3], L.ptr(geom), L.ptr(lc), len(cat_ids), int(benchmark),
                                                 L.ptr(rows), L.ptr(imgs), L.ptr(st), L.stream_ptr()), 'det_from_record')
    return rows.cpu().numpy().view(C.DET_DTYPE)


def test_batching_and_order_do_not_matter():
    from sipmask_b200 import cocoeval as C
    rec, metas, geom, gt, cat_ids = fake_records(9, rescoring=True)
    g = C.CocoGroundTruth(gt)
    ids = [10, 11, 12]
    outs = []
    for order in ([0, 1, 2], [2, 0, 1]):
        ev = C.CocoEvaluator(g, cat_ids)
        for n in order:                                       # batch 1, in this order
            one = {k: v[n:n + 1].contiguous() for k, v in rec.items()}
            ev.add_records(one, geom[n:n + 1].contiguous(), [ids[n]], [metas[n][1]])
        outs.append(ev.evaluate())
    ev = C.CocoEvaluator(g, cat_ids)
    ev.add_records(rec, geom, ids, [m[1] for m in metas])
    outs.append(ev.evaluate())
    for o in outs[1:]:
        for m in ('bbox', 'segm'):
            for key in ('precision', 'recall', 'scores'):
                assert np.array_equal(o['arrays'][m][key], outs[0]['arrays'][m][key])


def test_bounds_and_errors():
    from sipmask_b200 import cocoeval as C
    rec, metas, geom, gt, cat_ids = fake_records(3)
    g = C.CocoGroundTruth(gt)
    ids = [10, 11, 12]
    # a count past the capacity is clamped: the same as a full record
    over = dict(rec, count=torch.tensor([1000, 37, 12], dtype=torch.int32, device='cuda'))
    a = C.CocoEvaluator(g, cat_ids)
    a.add_records(over, geom, ids, [m[1] for m in metas])
    b = C.CocoEvaluator(g, cat_ids)
    b.add_records(rec, geom, ids, [m[1] for m in metas])
    ra, rb = a.evaluate(), b.evaluate()
    assert np.array_equal(ra['arrays']['segm']['precision'], rb['arrays']['segm']['precision'])
    # a label outside cat_ids
    bad = dict(rec, det_labels=rec['det_labels'].clone())
    bad['det_labels'][1, 3] = 17
    e = C.CocoEvaluator(g, cat_ids)
    e.add_records(bad, geom, ids, [m[1] for m in metas])
    with pytest.raises(ValueError):
        e.evaluate()
    # ori_shape differs from the annotation, unknown / repeated image ids
    e = C.CocoEvaluator(g, cat_ids)
    with pytest.raises(ValueError):
        e.add_records(rec, geom, ids, [(91, 120, 3)] + [m[1] for m in metas[1:]])
    with pytest.raises(ValueError):
        e.add_records(rec, geom, [10, 11, 99], [m[1] for m in metas])
    e.add_records({k: v[:1].contiguous() for k, v in rec.items()}, geom[:1].contiguous(), [10], [metas[0][1]])
    with pytest.raises(ValueError):
        e.add_records({k: v[:1].contiguous() for k, v in rec.items()}, geom[:1].contiguous(), [10], [metas[0][1]])
    # no detections at all
    empty = dict(rec, count=torch.zeros(3, dtype=torch.int32, device='cuda'))
    e = C.CocoEvaluator(g, cat_ids)
    e.add_records(empty, geom, ids, [m[1] for m in metas])
    with pytest.raises(ValueError):
        e.evaluate()
    with pytest.raises(ValueError):
        C.evaluate_json(g, cat_ids, bbox_json=[dict(image_id=55, category_id=2, bbox=[0, 0, 1, 1], score=0.5)])


def test_evaluate_json_image_subset():
    """Results of ground-truth images outside img_ids are dropped (_prepare), not rejected (loadRes checks the whole
    ground truth)."""
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = random_dataset(4, n_img=6)
    g = C.CocoGroundTruth(gt)
    sub = g.img_ids[1:4]
    res = C.evaluate_json(g, g.cat_ids, bbox_json=bbox, segm_json=segm, img_ids=sub)
    _assert_same(res, {'bbox': R.run(gt, bbox, 'bbox', img_ids=sub), 'segm': R.run(gt, segm, 'segm', img_ids=sub)})


# ---------------------------------------------------------------------------------------------------- CocoEvalRunner
def _runner_images(n, seed):
    from test_gpu_stream import _raw_images
    rs = np.random.RandomState(seed)
    sizes = [(427, 640), (480, 640), (375, 500), (544, 544), (640, 480), (333, 500)]
    return _raw_images([sizes[i] for i in rs.randint(0, len(sizes), n)], seed=seed)


def _runner_kw(batch, masks):
    from test_gpu_stream import _config
    sd, ekw, rule, _ = _config('plusplus')
    return sd, dict(in_flight=2, batch=batch, max_src_hw=(1088, 1920), max_ori_hw=(640, 640), min_mask_up=0.5,
                    masks=masks, **rule, **ekw)


def _first_pass_gt(imgs, cat_ids, seed):
    """Ground truth built from a plain StreamRunner pass over the images: shifted boxes as polygons, grown / shrunk
    planes as compressed and uncompressed RLE, some crowds, and a category without detections."""
    from sipmask_b200 import rle
    from sipmask_b200.serving import StreamRunner
    sd, kw = _runner_kw(1, 'bits')
    runner = StreamRunner(sd, **kw)
    rng = np.random.default_rng(seed)
    gt = dict(images=[], categories=[dict(id=c) for c in sorted(set(cat_ids))] + [dict(id=999)], annotations=[])
    aid = 0
    for n, img in enumerate(imgs):
        k = runner.submit(img.pin_memory())
        r = runner.result(k)
        h, w = img.shape[:2]
        gt['images'].append(dict(id=1000 + n, height=h, width=w))
        cnt = int(r['count'][0])
        for j in range(0, cnt, 2):
            lab = int(r['det_labels'][j])
            m = np.unpackbits(r['mask_bits'][j].numpy().view(np.uint8), axis=-1, bitorder='little')[:h, :w].astype(bool)
            if not m.any():
                continue
            aid += 1
            kind = aid % 4
            if kind == 1:
                m = np.pad(m, 1)[2:, 1:-1] | m                        # grown down by a row
            elif kind == 2:
                m = m & np.pad(m, 1)[1:-1, 2:]                        # shrunk from the right
            ys, xs = np.nonzero(m) if m.any() else (np.array([0]), np.array([0]))
            x0, y0, x1, y1 = float(xs.min()), float(ys.min()), float(xs.max() + 1), float(ys.max() + 1)
            if kind == 0:
                d = float(rng.integers(-3, 4))
                seg = [[x0 + d, y0, x0 + d, y1, x1 + d, y1, x1 + d, y0]]
            elif kind == 3:
                seg = {'size': [h, w], 'counts': rle.counts(m).tolist()}
            else:
                seg = _mask_rle(m)
            gt['annotations'].append(dict(id=aid, image_id=1000 + n, category_id=cat_ids[lab], bbox=[x0, y0, x1 - x0, y1 - y0],
                                          area=float(m.sum()), iscrowd=int(aid % 9 == 0), segmentation=seg))
        aid += 1
        gt['annotations'].append(dict(id=aid, image_id=1000 + n, category_id=999, bbox=[1.0, 1.0, 30.0, 30.0], area=900.0,
                                      iscrowd=0, segmentation=[[1, 1, 1, 31, 31, 31, 31, 1]]))
    return gt


def _run_eval(gt, cat_ids, imgs, order, batch, masks):
    """CocoEvalRunner over the images in `order`; returns evaluate() and the runner's own result json."""
    from sipmask_b200 import cocoeval as C, coco, rle
    from sipmask_b200.serving import CocoEvalRunner
    sd, kw = _runner_kw(batch, masks)
    runner = CocoEvalRunner(sd, C.CocoGroundTruth(gt), cat_ids, **kw)
    bbox, segm, seen = [], [], set()

    def collect():
        for k, images in enumerate(runner.slot_images):
            for m in images:
                if m['ticket'] in seen:
                    continue
                seen.add(m['ticket'])
                r = runner.result(m['ticket'] if batch > 1 else k)
                cnt = int(r['count'][0])
                if masks == 'bits':
                    r['segms'] = rle.encode_planes(r['mask_bits'][:cnt].numpy(), m['ori_shape'][:2])
                b, s = coco.coco_json(r, ids[m['ticket']], cat_ids)
                bbox.extend(b)
                segm.extend(s)
    ids = {}
    for n in order:
        before = runner.dispatched
        ids[runner.i] = 1000 + n
        runner.submit(imgs[n].pin_memory(), 1000 + n)
        if runner.dispatched != before:
            collect()
    res = runner.evaluate()
    torch.cuda.synchronize()
    collect()
    return res, bbox, segm


def test_runner_equals_restatement_and_settings_do_not_matter():
    imgs = _runner_images(7, seed=21)
    cat_ids = [1 + label % 12 for label in range(80)]            # 80 labels onto 12 categories
    gt = _first_pass_gt(imgs, cat_ids, seed=3)
    assert len(gt['annotations']) > 20
    base, bbox, segm = _run_eval(gt, cat_ids, imgs, list(range(7)), 1, 'bits')
    for s in (bbox, segm):
        for r in s:
            if 'segmentation' in r:
                r['segmentation'] = {'size': r['segmentation']['size'], 'counts': r['segmentation']['counts']}
    _assert_same(base, {'bbox': R.run(gt, bbox, 'bbox'), 'segm': R.run(gt, segm, 'segm')}, 'runner')
    shuffled = list(np.random.default_rng(5).permutation(7))
    for batch, masks, order in ((4, 'rle', shuffled), (4, 'bits', list(range(7))), (1, 'rle', shuffled)):
        res = _run_eval(gt, cat_ids, imgs, order, batch, masks)[0]
        for m in ('bbox', 'segm'):
            for key in ('precision', 'recall', 'scores'):
                assert np.array_equal(res['arrays'][m][key], base['arrays'][m][key]), (batch, masks, m, key)


def test_runner_rejects_before_enqueueing():
    from sipmask_b200 import cocoeval as C
    from sipmask_b200.serving import CocoEvalRunner
    imgs = _runner_images(2, seed=22)
    gt = dict(images=[dict(id=1, height=imgs[0].shape[0], width=imgs[0].shape[1])], categories=[dict(id=1)],
              annotations=[])
    sd, kw = _runner_kw(1, 'rle')
    with pytest.raises(ValueError):
        CocoEvalRunner(sd, C.CocoGroundTruth(gt), [1] * 80, vis=True, **kw)
    runner = CocoEvalRunner(sd, C.CocoGroundTruth(gt), [1] * 80, **kw)
    with pytest.raises(ValueError):
        runner.submit(imgs[0].pin_memory(), 2)                                   # not in the ground truth
    bad = torch.zeros((imgs[0].shape[0] + 1, imgs[0].shape[1], 3), dtype=torch.uint8)
    with pytest.raises(ValueError):
        runner.submit(bad.pin_memory(), 1)                                       # ori_shape differs
    assert runner.i == 0
    runner.submit(imgs[0].pin_memory(), 1)
    with pytest.raises(ValueError):
        runner.submit(imgs[0].pin_memory(), 1)                                   # twice
    runner.flush()
