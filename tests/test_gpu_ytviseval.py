"""YouTube-VIS mask AP on the device (sipmask_b200.ytviseval, serving.VideoEvalRunner) against the test restatement of
YTVOSeval (tests/ytviseval_ref.py): the precision / recall / scores arrays must be equal exactly, and so the 12 stats."""
import numpy as np
import pytest
import torch

import ytviseval_ref as R
from test_ytviseval_host import _rect, _rle, known_cases

pytestmark = pytest.mark.gpu


def _same(got, ref):
    a = got['arrays']['segm']
    assert np.array_equal(a['precision'], ref.precision)
    assert np.array_equal(a['recall'], ref.recall)
    assert np.array_equal(a['scores'], ref.scores)
    assert np.array_equal(got['stats']['segm'], ref.stats)


@pytest.mark.parametrize('name', [c[0] for c in known_cases()])
def test_known_cases_equal_restatement(name):
    from sipmask_b200.ytviseval import YtvisGroundTruth, evaluate_json
    _, ann, res = [c for c in known_cases() if c[0] == name][0]
    _same(evaluate_json(YtvisGroundTruth(ann), res), R.run(ann, res))


def _synthetic(seed):
    """Several videos of mixed sizes and lengths, 3 categories, crowds, absent and empty frames, repeated scores, and
    one (video, category) with more than 100 entries."""
    rs = np.random.RandomState(seed)
    videos = [(1, (48, 70), 3), (4, (33, 96), 5), (7, (64, 64), 2)]
    ann = dict(videos=[dict(id=v, height=s[0], width=s[1], length=n) for v, s, n in videos],
               categories=[dict(id=c) for c in (1, 3, 5)], annotations=[])
    res = []
    aid = 1
    for vid, (h, w), n in videos:
        objs = []
        for _ in range(rs.randint(2, 6)):
            y0, x0 = rs.randint(0, h - 8), rs.randint(0, w - 8)
            y1, x1 = y0 + rs.randint(3, min(30, h - y0)), x0 + rs.randint(3, min(30, w - x0))
            masks = []
            for f in range(n):
                if rs.rand() < 0.2:
                    masks.append(None)
                else:
                    dy, dx = rs.randint(-2, 3), rs.randint(-2, 3)
                    masks.append(_rect(h, w, max(y0 + dy, 0), max(x0 + dx, 0), y1 + dy, x1 + dx))
            cat = int(rs.choice([1, 3, 5]))
            objs.append((masks, cat))
            ann['annotations'].append(dict(id=aid, video_id=vid, category_id=cat, iscrowd=int(rs.rand() < 0.15),
                                           segmentations=[None if m is None else _rle(m, compressed=bool(rs.rand() < .5))
                                                          for m in masks],
                                           areas=[None if m is None else float(m.sum()) for m in masks]))
            aid += 1
        n_res = 130 if vid == 4 else rs.randint(3, 12)
        for e in range(n_res):
            masks, cat = objs[rs.randint(len(objs))]
            out = []
            for f in range(n):
                u = rs.rand()
                if u < 0.15:
                    out.append(None)
                elif u < 0.2:
                    out.append(np.zeros((h, w), bool))
                else:
                    base = masks[f] if masks[f] is not None else _rect(h, w, 0, 0, 4, 4)
                    out.append(np.roll(base, (rs.randint(-3, 4), rs.randint(-3, 4)), (0, 1)))
            score = float(np.float32(rs.choice([0.5, 0.25, rs.rand()])))
            res.append(dict(video_id=vid, score=score, category_id=int(cat if (vid == 4 or rs.rand() < .8) else 5),
                            segmentations=[None if m is None else _rle(m) for m in out]))
    rs.shuffle(res)
    return ann, res


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_seeded_datasets_equal_restatement(seed):
    from sipmask_b200.ytviseval import YtvisGroundTruth, evaluate_json
    ann, res = _synthetic(seed)
    assert sum(r['video_id'] == 4 for r in res) > 100
    ref = R.run(ann, res)
    got = evaluate_json(YtvisGroundTruth(ann), res, chunk=2)
    _same(got, ref)
    assert got['segm_mAP'] == float('{:.3f}'.format(ref.stats[0]))
    sub = R.run(ann, res, vid_ids=[4, 7])
    _same(evaluate_json(YtvisGroundTruth(ann), res, vid_ids=[4, 7]), sub)


# --------------------------------------------------------------------------------------------- kernels on crafted rows
def _crafted():
    from sipmask_b200.ytviseval import YtvisEvaluator, YtvisGroundTruth
    H, W, n = 20, 40, 2
    g0, g1 = _rect(H, W, 0, 0, 4, 4), _rect(H, W, 10, 30, 14, 38)
    ann = dict(videos=[dict(id=2, height=H, width=W, length=n)], categories=[dict(id=1)],
               annotations=[dict(id=1, video_id=2, category_id=1, segmentations=[_rle(g0), _rle(g0)], areas=[16, 16]),
                            dict(id=2, video_id=2, category_id=1, segmentations=[None, _rle(g1)], areas=[None, 32])])
    gt = YtvisGroundTruth(ann)
    ev = YtvisEvaluator(gt, slots=2, objects=8, max_gts=2)
    return gt, ev, (H, W, n), (g0, g1)


def _planes(masks, W, mx, H=20):
    """[N, mx, H, pitch] int32 device planes of per-frame detection masks."""
    N = len(masks)
    pitch = (W + 31) // 32
    out = np.zeros((N, mx, H, pitch), np.uint32)
    for n, ms in enumerate(masks):
        for j, m in enumerate(ms):
            out[n, j] = np.packbits(np.pad(m, ((0, 0), (0, pitch * 32 - W))), axis=1, bitorder='little').view(np.uint32)
    return torch.from_numpy(out.view(np.int32)).cuda(), pitch


def _run_frames(ev, video_id, dets, ids, counts, slot=1, mx=4, W=40):
    ev.begin_video(video_id, slot)
    planes, pitch = _planes(dets, W, mx)
    H = planes.shape[2]
    staged = [ev.stage_frame(video_id, f) for f in range(len(dets))]
    count = torch.tensor(counts, dtype=torch.int32, device='cuda')
    ovl = ev.overlap(staged, [planes.data_ptr() + 4 * n * mx * H * pitch for n in range(len(dets))], H * pitch, pitch,
                     mx, count=count)
    ev.scatter(ovl, torch.tensor(ids, dtype=torch.int32, device='cuda'), count=count)
    for s in staged:
        ev.commit_frame(s)
    torch.cuda.synchronize()


def test_kernels_last_detection_wins_and_carried_ids():
    gt, ev, (H, W, n), (g0, g1) = _crafted()
    a = _rect(H, W, 0, 0, 4, 2)                 # 8 pixels, 8 inside g0
    b = _rect(H, W, 1, 1, 3, 3)                 # 4 pixels, 4 inside g0
    c = _rect(H, W, 10, 32, 14, 40)             # 32 pixels, 24 inside g1
    z = np.zeros((H, W), bool)
    # frame 0 has no detections (the lane carries state, so frame 1's ids do not start at 0); frame 1 holds id 5 twice
    # (the last, b, wins), id 6, an id -1 and, past the count, an id that must not be read
    _run_frames(ev, 2, [[], [a, b, c, z]], [[0, 0, 0, 0], [5, 5, 6, -1]], [0, 3])
    s = 1
    assert ev.acc_area[s].tolist() == [0, 0, 0, 0, 0, 4, 32, 0]
    assert ev.acc_nz[s].tolist() == [0, 0, 0, 0, 0, 1, 1, 0]
    assert ev.acc_inter[s, 5].tolist() == [4, 0] and ev.acc_inter[s, 6].tolist() == [0, 24]
    assert int(ev.status.item()) == 0
    # sequence IoUs: id 5 vs g0 = 4 / (4 + 32 - 4), id 6 vs g1 = 24 / (32 + 32 - 24)
    ev.end_video(2, [dict(score=0.9, category_id=1), dict(score=0.8, category_id=1)], [5, 6])
    got = ev.evaluate()
    ref = R.run(dict(videos=[dict(id=2, height=H, width=W, length=n)], categories=[dict(id=1)],
                     annotations=[dict(id=1, video_id=2, category_id=1, segmentations=[_rle(g0), _rle(g0)], areas=[16, 16]),
                                  dict(id=2, video_id=2, category_id=1, segmentations=[None, _rle(g1)],
                                       areas=[None, 32])]),
                [dict(video_id=2, score=0.9, category_id=1, segmentations=[None, _rle(b)]),
                 dict(video_id=2, score=0.8, category_id=1, segmentations=[None, _rle(c)])])
    _same(got, ref)


def test_kernels_bound_counts_and_raise_on_overflow():
    from sipmask_b200._lib import SmbError
    gt, ev, (H, W, n), (g0, g1) = _crafted()
    a = _rect(H, W, 0, 0, 4, 2)
    # a count beyond max_num is clamped; an id beyond the 8 objects sets the status bit, which evaluate() raises
    _run_frames(ev, 2, [[a], [a, a, a, a]], [[0, 0, 0, 0], [1, 2, 3, 9]], [1, 99])
    assert ev.acc_area[1].tolist() == [8, 8, 8, 8, 0, 0, 0, 0]
    assert int(ev.status.item()) == 1
    ev.end_video(2, [dict(score=0.9, category_id=1)], [0])
    with pytest.raises(SmbError, match='capacity of 8 objects'):
        ev.evaluate()
    # a ground-truth column beyond max_gts
    gt, ev, _, _ = _crafted()
    ev.begin_video(2, 0)
    s = ev.stage_frame(2, 1)
    s['rows']['g'][1] = 5
    planes, pitch = _planes([[a]], W, 1)
    ovl = ev.overlap([s], [planes.data_ptr()], H * pitch, pitch, 1, n_det=[1])
    torch.cuda.synchronize()
    assert int(ev.status.item()) == 2
    with pytest.raises(ValueError, match='ended after 0 frames'):
        ev.end_video(2, [], [])
    del ovl


def test_evaluator_checks():
    gt, ev, (H, W, n), _ = _crafted()
    with pytest.raises(ValueError, match='max_gts'):
        type(ev)(gt, max_gts=1).check_frame(2, 0, (H, W))
    ev.begin_video(2, 0)
    with pytest.raises(ValueError, match='evaluated twice'):
        ev.check_frame(2, 0, (H, W))
    with pytest.raises(ValueError, match='ended after 0 frames'):
        ev.end_video(2, [dict(score=1.0, category_id=1)], [0])
    for f in range(n):
        ev.commit_frame(ev.stage_frame(2, f))
    with pytest.raises(ValueError, match='category'):
        ev.end_video(2, [dict(score=1.0, category_id=4)], [0])
    with pytest.raises(ValueError, match='object ids'):
        ev.end_video(2, [dict(score=1.0, category_id=1)], [])


# --------------------------------------------------------------------------------------------- VideoEvalRunner
def _gt_from_json(videos, js, seed=0):
    """A ground truth derived from a first pass's json: masks shifted, frames dropped, objects relabelled, one crowd."""
    from sipmask_b200.cocoeval import segm_plane
    rs = np.random.RandomState(seed)
    ann = dict(videos=[], categories=[dict(id=c) for c in range(1, 41)], annotations=[])
    aid = 1
    for vid, frames in videos:
        h, w = frames[0].shape[:2]
        ann['videos'].append(dict(id=vid, height=h, width=w, length=len(frames)))
        for e, ent in enumerate(js[vid]):
            segs, areas = [], []
            dy, dx = rs.randint(-6, 7), rs.randint(-6, 7)
            for s in ent['segmentations']:
                if s is None or rs.rand() < 0.2:
                    segs.append(None)
                    areas.append(None)
                    continue
                p = segm_plane(s, h, w)
                m = np.unpackbits(p.view(np.uint8), axis=1, bitorder='little')[:, :w].astype(bool)
                m = np.roll(m, (dy, dx), (0, 1))
                segs.append(_rle(m))
                areas.append(int(m.sum()))
            cat = ent['category_id'] if rs.rand() < 0.75 else int(rs.randint(1, 41))
            ann['annotations'].append(dict(id=aid, video_id=vid, category_id=cat, iscrowd=int(e == 1),
                                           segmentations=segs, areas=areas))
            aid += 1
    return ann


def _vis_videos():
    from test_gpu_video import _videos
    return [(n + 1, f) for n, (_, f) in enumerate(_videos())]


def _first_pass(sd, kw, rule, videos, order):
    from sipmask_b200.serving import VideoRunner
    vr = VideoRunner(sd, lanes=4, batch=1, in_flight=2, max_src_hw=(1080, 1920), masks='rle', **rule, **kw)
    for v, f in order:
        vr.submit(videos[v][1][f], videos[v][0], f)
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    vr.flush()
    return {vid: vr.video_json(vid) for vid, _ in videos}


@pytest.fixture(scope='module')
def vis_setup():
    from test_gpu_video import _interleave, _sd
    sd, kw, rule = _sd()
    videos = _vis_videos()
    order = _interleave(videos)
    js = _first_pass(sd, kw, rule, videos, order)
    assert sum(len(v) for v in js.values()) >= 3
    return sd, kw, rule, videos, order, js, _gt_from_json(videos, js)


@pytest.mark.parametrize('batch,lanes,masks', [(1, 1, 'rle'), (4, 1, 'rle'), (4, 4, 'bits'), (1, 4, 'bits')])
def test_video_eval_runner_equals_evaluate_json_and_restatement(vis_setup, batch, lanes, masks):
    from sipmask_b200.serving import VideoEvalRunner
    from sipmask_b200.ytviseval import YtvisGroundTruth, evaluate_json
    sd, kw, rule, videos, order, js, ann = vis_setup
    gt = YtvisGroundTruth(ann)
    if lanes == 1:                              # one lane: each video in turn
        order = [(v, f) for v in range(len(videos)) for f in range(len(videos[v][1]))]
    # eval_slots = lanes forces the runner to match ended videos to free slots for the next ones
    vr = VideoEvalRunner(sd, gt, lanes=lanes, eval_slots=lanes, batch=batch, in_flight=2, max_src_hw=(1080, 1920),
                         masks=masks, **rule, **kw)
    for v, f in order:
        vr.submit(videos[v][1][f], videos[v][0], f)
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    got = vr.evaluate()
    results = []
    for vid, _ in videos:
        j = vr.video_json(vid)
        assert j == js[vid], vid
        results += j
    ref = R.run(ann, results)
    assert 0 < ref.stats[0] < 1, ref.stats
    _same(got, ref)
    _same(evaluate_json(gt, results), ref)


def test_video_eval_runner_rejections(vis_setup):
    from sipmask_b200.serving import VideoEvalRunner
    from sipmask_b200.ytviseval import YtvisGroundTruth
    sd, kw, rule, videos, _, _, ann = vis_setup
    vr = VideoEvalRunner(sd, YtvisGroundTruth(ann), lanes=2, in_flight=2, max_src_hw=(1080, 1920), **rule, **kw)
    f0 = videos[0][1][0]
    with pytest.raises(ValueError, match='not in the ground truth'):
        vr.submit(f0, 99, 0)
    with pytest.raises(ValueError, match='frame of'):
        vr.submit(videos[1][1][0], videos[0][0], 0)
    vr.submit(f0, videos[0][0], 0)
    with pytest.raises(ValueError, match='ends after 1 frames'):
        vr.end_video(videos[0][0])
    with pytest.raises(ValueError, match='has not ended'):
        vr.evaluate()
    assert vr.i == 1
