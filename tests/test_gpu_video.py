"""SipMask-VIS videos on the device: the tracker association kernel (smb_track_assoc_dev, tracker.LaneTracker) and
serving.VideoRunner.

The kernel must give exactly the ids and lane state of the host association.  Its dot products and exp-sum are summed in
another order than the host's, so every random case first shows, with a float64 restatement of the formula, that each
argmax and claim comparison it makes has a margin above the fp32 error bound of its 512-term dot products
(gamma_512 * sum |f * p| per dot product, plus a few ulps for the log terms; comparisons of bit-identical inputs are
exact ties in both): exact equality is then a fair demand."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
GAMMA512 = 512 * U / (1 - 512 * U)
COEF = (1.0, 2.0, 10.0)


def _iou(d, p):
    w = min(d[2], p[2]) - max(d[0], p[0]) + 1
    h = min(d[3], p[3]) - max(d[1], p[1]) + 1
    ov = max(w, 0.0) * max(h, 0.0)
    return ov / ((d[2] - d[0] + 1) * (d[3] - d[1] + 1) + (p[2] - p[0] + 1) * (p[3] - p[1] + 1) - ov)


class Ref64(object):
    """The association in float64 (state as float32 copies), recording the smallest margin over the fp32 error bound of
    every comparison that decides an id."""

    def __init__(self, cap=4096):
        self.cap, self.n, self.worst, self.worst_at = cap, -1, np.inf, None
        self.boxes = np.zeros((cap, 5), np.float32)
        self.labels = np.zeros((cap,), np.int64)
        self.feats = np.zeros((cap, 512), np.float32)
        self.overflow = False

    def _margin(self, a, b, err):
        if abs(a - b) - err < self.worst:
            self.worst, self.worst_at = abs(a - b) - err, (float(a), float(b), float(err))

    def step(self, det, lab, feats, first):
        n, m = det.shape[0], self.n
        if n == 0:
            return np.zeros((0,), np.int32)
        ids = -np.ones(n, np.int32)
        if first or m < 0:
            keep = min(n, self.cap)
            self.boxes[:keep], self.labels[:keep], self.feats[:keep] = det[:keep], lab[:keep], feats[:keep]
            ids[:keep] = np.arange(keep)
            self.overflow |= n > self.cap
            self.n = keep
            return ids
        f64, p64 = feats.astype(np.float64), self.feats[:m].astype(np.float64)
        dots = f64 @ p64.T
        err_dot = GAMMA512 * (np.abs(f64) @ np.abs(p64).T)
        score = np.concatenate([np.zeros((n, 1)), dots], 1)
        mx = score.max(1, keepdims=True)
        comp = score - mx - np.log(np.exp(score - mx).sum(1, keepdims=True)) + COEF[0] * np.log(det[:, 4:5].astype(np.float64))
        for i in range(n):
            comp[i, 0] += COEF[2]
            for j in range(m):
                comp[i, j + 1] += COEF[1] * _iou(det[i].astype(np.float64), self.boxes[j].astype(np.float64))
                comp[i, j + 1] += COEF[2] * (self.labels[j] == lab[i])
        # error bounds: a dot product within err_dot; the row max and log-sum-exp move by at most the row's largest dot
        # error (they cancel between two entries of one row); a few ulps for the fp32 log / IoU / sums
        row_err = err_dot.max(1, initial=0.0)
        ulps = 16 * U * (np.abs(comp) + 20)
        edot = np.concatenate([np.zeros((n, 1)), err_dot], 1)
        same_obj = lambda a, b: a > 0 and b > 0 and np.array_equal(self.feats[a - 1], self.feats[b - 1])   # noqa: E731
        arg = comp.argmax(1)
        for i in range(n):
            a = arg[i]
            for j in range(m + 1):
                if j != a:
                    # equal feature vectors give equal dot products in both implementations: only the exact terms differ
                    if same_obj(a, j):
                        if comp[i, a] == comp[i, j]:
                            continue                 # an exact tie: the first maximum in both
                        e = 0.0
                    else:
                        e = edot[i, a] + edot[i, j]
                    self._margin(comp[i, a], comp[i, j], e + ulps[i, a] + ulps[i, j])
        best, claimant, np_ = {}, {}, m
        same_det = lambda a, b: (np.array_equal(feats[a], feats[b]) and np.array_equal(det[a], det[b])   # noqa: E731
                                 and lab[a] == lab[b])
        for i in range(n):
            if arg[i] == 0:
                if np_ < self.cap:
                    ids[i] = np_
                    self.boxes[np_], self.labels[np_], self.feats[np_] = det[i], lab[i], feats[i]
                    np_ += 1
                else:
                    self.overflow = True
            else:
                o = arg[i] - 1
                b = best.get(o, -100.0)
                if o in claimant:
                    c = claimant[o]
                    if not same_det(i, c):           # identical detections tie exactly: the earlier claimant keeps it
                        self._margin(comp[i, arg[i]], b, 2 * (row_err[i] + row_err[c]) + edot[i, arg[i]] + edot[c, arg[c]]
                                     + ulps[i, arg[i]] + ulps[c, arg[c]])
                if comp[i, arg[i]] > b:
                    ids[i], best[o], claimant[o] = o, comp[i, arg[i]], i
                    self.boxes[o], self.feats[o] = det[i], feats[i]
        self.n = np_
        return ids


def _lane_tracker(lanes, cap=4096):
    from sipmask_b200.tracker import LaneTracker
    return LaneTracker(lanes, cap, COEF, 'cuda', max_rows=64)


def _launch(lt, frames, mx=10, count_override=None, direct=False):
    """frames: list of (lane, is_first, det [n,5], lab [n], feats [n,512]) -> ids [N, mx] numpy (one launch).
    direct: through ops.track_assoc with the rows as given (LaneTracker rejects lanes outside its state on the host)."""
    N = len(frames)
    det = torch.zeros((N, mx, 5), dtype=torch.float32)
    lab = torch.zeros((N, mx), dtype=torch.int64)
    feats = torch.zeros((N, mx, 512), dtype=torch.float32)
    cnt = torch.zeros((N,), dtype=torch.int32)
    for r, (lane, first, d, l, f) in enumerate(frames):
        n = d.shape[0]
        det[r, :n], lab[r, :n], feats[r, :n] = torch.from_numpy(d), torch.from_numpy(l), torch.from_numpy(f)
        cnt[r] = n
    if count_override is not None:
        for r, c in count_override.items():
            cnt[r] = c
    rows = [(a, int(b)) for a, b, _, _, _ in frames]
    if direct:
        from sipmask_b200 import ops
        ids = ops.track_assoc(torch.tensor(rows, dtype=torch.int32).cuda(), det.cuda(), lab.cuda(), cnt.cuda(), feats.cuda(),
                              lt.state, COEF)
    else:
        ids = lt.associate(rows, det.cuda(), lab.cuda(), cnt.cuda(), feats.cuda())
    torch.cuda.synchronize()
    return ids.cpu().numpy()


def _clip_inputs(g):
    """The (det, labels, features, is_first) the reference's tracker saw on ref_vis_clip.npz (oracle head + oracle
    post-processing, pinned to the fixture by tests/test_vis_oracle.py)."""
    from oracle import model as M
    from oracle import postproc as P
    from sipmask_b200 import synth
    from sipmask_b200.tracker import Tracker
    from test_vis_oracle import clip_feats, vis_cfg, vis_meta
    head = M.SipMaskVISHead(num_classes=41, stacked_convs=3)
    head.load_state_dict(synth.head_state_dict(seed=int(g['seed']), prefix='', num_classes=41, stacked_convs=3, gn=True,
                                               cls_bias=-2.0, track=True), strict=True)
    head.eval()
    seen = []

    class Wrap(object):
        t = Tracker(native=True)

        def step(self, det, lab, feats, first):
            seen.append((det.numpy().copy(), lab.numpy().copy(), feats.numpy().copy(), bool(first)))
            return self.t.step(det.numpy(), lab.numpy(), feats.numpy(), first)
    w = Wrap()
    for t, feats in enumerate(clip_feats(g)):
        with torch.no_grad():
            outs = head(feats, feats, False)
        P.vis_get_bboxes(outs, vis_meta(g, t), vis_cfg(g), w, rescale=True)
    return seen


def test_kernel_reproduces_reference_clip(golden_dir):
    g = dict(np.load(os.path.join(golden_dir, 'ref_vis_clip.npz')))
    seen = _clip_inputs(g)
    assert len(seen) == 5 and any(s[3] for s in seen[1:])       # a later frame is flagged is_first again
    lt = _lane_tracker(2)
    ids = _launch(lt, [(1, first, d, l, f) for d, l, f, first in seen])       # the whole clip in one launch, lane 1
    for t, (d, _, _, _) in enumerate(seen):
        assert ids[t, :d.shape[0]].tolist() == g['f%d_ids' % t].tolist(), t
        assert (ids[t, d.shape[0]:] == -1).all()
    assert int(lt.n_obj[0]) == -1                                  # the other lane is untouched


def _video_frame(rs, objs, n_new, drop, p_same=0.15):
    """A frame of a synthetic video: some tracked objects seen again (feature + noise, box moved), some new ones."""
    keep = [o for o in objs if rs.rand() > drop]
    d, l, f = [], [], []
    for o in keep:
        xy = o['box'][:2] + rs.randn(2) * 3
        d.append(np.concatenate([xy, xy + o['box'][2:4] - o['box'][:2], [rs.uniform(0.05, 1)]]))
        l.append(o['label'] if rs.rand() > p_same else rs.randint(0, 40))
        f.append(o['feat'] + rs.randn(512) * 0.05)
    for _ in range(n_new):
        xy = rs.rand(2) * 300
        o = dict(box=np.concatenate([xy, xy + rs.rand(2) * 80 + 8]), label=rs.randint(0, 40), feat=rs.randn(512) * 0.08)
        objs.append(o)
        d.append(np.concatenate([o['box'], [rs.uniform(0.05, 1)]]))
        l.append(o['label'])
        f.append(o['feat'] + rs.randn(512) * 0.05)
    order = rs.permutation(len(d))
    det = np.asarray(d, np.float32).reshape(-1, 5)[order]
    return det, np.asarray(l, np.int64).reshape(-1)[order], np.asarray(f, np.float32).reshape(-1, 512)[order]


def test_kernel_random_lanes_equal_float64_and_host():
    from sipmask_b200.tracker import Tracker
    rs = np.random.RandomState(3)
    lanes, n_launch = 5, 7
    lt = _lane_tracker(lanes)
    refs = [Ref64() for _ in range(lanes)]
    hosts = [Tracker(COEF, native=False) for _ in range(lanes)]
    objs = [[] for _ in range(lanes)]
    for it in range(n_launch):
        frames = []
        for lane in range(lanes):
            for _ in range(rs.randint(0, 4)):                       # 0-3 frames of each lane per launch
                first = not objs[lane] or rs.rand() < 0.05
                if first:
                    objs[lane] = []
                n_new = rs.randint(1, 5) if first else rs.randint(0, 3)
                det, lab, feats = _video_frame(rs, objs[lane], n_new, drop=0.2)
                det, lab, feats = det[:10], lab[:10], feats[:10]
                frames.append((lane, first, det, lab, feats))
        order = rs.permutation(len(frames))                         # interleave the lanes, keep each lane's order
        by_lane = {l: [fr for fr in frames if fr[0] == l] for l in range(lanes)}
        mixed = []
        for o in order:
            mixed.append(by_lane[frames[o][0]].pop(0))
        mixed.insert(rs.randint(0, len(mixed) + 1), (-1, False, np.zeros((3, 5), np.float32), np.zeros(3, np.int64),
                                                    np.zeros((3, 512), np.float32)))           # a filler row
        ids = _launch(lt, mixed)
        for r, (lane, first, det, lab, feats) in enumerate(mixed):
            if lane < 0:
                assert (ids[r] == -1).all()
                continue
            want = refs[lane].step(det, lab, feats, first)
            host = hosts[lane].step(det, lab, feats, first)
            assert ids[r, :det.shape[0]].tolist() == want.tolist() == np.asarray(host).tolist(), (it, r)
    worst = min(r.worst for r in refs)
    assert worst > 0, 'a comparison is within the fp32 error bound: %g' % worst
    n_obj = lt.n_obj.cpu().numpy()
    for lane, r in enumerate(refs):
        assert n_obj[lane] == r.n
        if r.n < 0:
            continue
        assert r.n == hosts[lane].num_objects
        n = r.n
        assert np.array_equal(lt.boxes[lane, :n].cpu().numpy(), r.boxes[:n])
        assert np.array_equal(lt.labels[lane, :n].cpu().numpy(), r.labels[:n])
        assert np.array_equal(lt.feats[lane, :n].cpu().numpy(), r.feats[:n])
        assert np.array_equal(hosts[lane].prev_roi_feats, r.feats[:n])
    assert (lt.status.cpu().numpy() == 0).all()
    assert sum(r.n for r in refs) > 20


def test_kernel_edge_rows():
    rs = np.random.RandomState(9)
    lt = _lane_tracker(3, cap=6)
    objs = []
    d0, l0, f0 = _video_frame(rs, objs, 3, 0.0)
    e = (np.zeros((0, 5), np.float32), np.zeros((0,), np.int64), np.zeros((0, 512), np.float32))
    # lane 0: a first frame; lane 1: is_first with no detections keeps "no state"; filler rows (lane -1 and lane 7)
    ids = _launch(lt, [(0, True) + (d0, l0, f0), (1, True) + e, (-1, False, d0, l0, f0), (7, False, d0, l0, f0)],
                  direct=True)
    assert ids[0].tolist() == [0, 1, 2] + [-1] * 7 and (ids[1:] == -1).all()
    assert lt.n_obj.cpu().tolist() == [3, -1, -1]
    state = [t.clone() for t in (lt.boxes, lt.labels, lt.feats)]
    # lane 0: is_first with zero detections keeps the state; count > max is clamped to max
    ids = _launch(lt, [(0, True) + e], count_override={0: -4})
    assert (ids == -1).all() and lt.n_obj.cpu().tolist() == [3, -1, -1]
    assert all(torch.equal(a, b) for a, b in zip(state, (lt.boxes, lt.labels, lt.feats)))
    d1, l1, f1 = _video_frame(rs, objs, 7, 0.0)                     # 10 detections: 3 known, 7 new
    ids = _launch(lt, [(2, True, d1, l1, f1)], count_override={0: 25})
    assert ids[0].tolist() == list(range(6)) + [-1] * 4 and lt.n_obj.cpu().tolist() == [3, -1, 6]
    assert lt.status.cpu().tolist() == [0, 0, 1]                    # the first frame of lane 2 exceeded capacity 6
    lt.status.zero_()
    # lane 0: a continuation (objects re-identified), then is_first in the middle of the lane, then a continuation that
    # appends beyond capacity
    ref = Ref64(cap=6)
    ref.step(d0, l0, f0, True)
    objs2 = []
    d2, l2, f2 = _video_frame(rs, objs2, 2, 0.0)
    frames = [(0, False, d1[:5], l1[:5], f1[:5]), (0, True, d2, l2, f2)]
    d3, l3, f3 = _video_frame(rs, objs2, 6, 0.0)
    frames.append((0, False, d3, l3, f3))
    ids = _launch(lt, frames)
    for r, (_, first, d, l, f) in enumerate(frames):
        assert ids[r, :d.shape[0]].tolist() == ref.step(d, l, f, first).tolist(), r
    assert ref.overflow and ref.worst > 0
    assert (ids[2] == -1).sum() >= 2 + 10 - d3.shape[0]
    assert lt.status.cpu().tolist() == [1, 0, 0] and int(lt.n_obj[0]) == 6


# --------------------------------------------------------------------------------------------- VideoRunner end to end
def _videos(seed=1):
    """Three interleaved synthetic videos of mixed sizes (moving smooth blobs): (video_id, frames)."""
    rs = np.random.RandomState(seed)
    out = []
    for vid, ((h, w), nf) in enumerate((((720, 1280), 6), ((480, 640), 5), ((1080, 1920), 4))):
        base = rs.randint(0, 256, (h // 16 + 6, w // 16 + 6, 3)).astype(np.float32)
        big = torch.nn.functional.interpolate(torch.from_numpy(base).permute(2, 0, 1)[None], size=(h + 96, w + 96),
                                              mode='bilinear', align_corners=False)[0].permute(1, 2, 0)
        frames = []
        for t in range(nf):
            dy, dx = 8 * t, 12 * t
            img = big[dy:dy + h, dx:dx + w] + torch.from_numpy(rs.randint(-10, 11, (h, w, 3)).astype(np.float32))
            frames.append(img.clamp(0, 255).to(torch.uint8).contiguous().pin_memory())
        out.append(('vid%d' % vid, frames))
    return out


def _interleave(videos):
    order, pos = [], [0] * len(videos)
    rs = np.random.RandomState(0)
    while any(p < len(f) for p, (_, f) in zip(pos, videos)):
        v = rs.choice([i for i, (_, f) in enumerate(videos) if pos[i] < len(f)])
        order.append((v, pos[v]))
        pos[v] += 1
    return order


def _sd():
    """test_gpu_stream's synthetic VIS weights with the 512-d track output scaled by 1/20: its unscaled features give dot
    products in the thousands, whose fp32 error bound (not their actual error) is wider than the gaps between some comp
    values; scaled, every decision has a margin over the bound and the dot products still take part."""
    from test_gpu_stream import _config
    sd, kw, rule, _ = _config('vis')
    sd = dict(sd)
    for k in ('bbox_head.sipmask_track.weight', 'bbox_head.sipmask_track.bias'):
        sd[k] = sd[k] * 0.05
    return sd, kw, rule


def _read_before_reuse(runner, read, done, img=None):
    """Read the frames of the slot the next batch opens in (the other slots keep their associations pending).  A frame
    of another padded shape than the open batch dispatches that batch and opens the next slot in the same submit."""
    d, n = runner.dispatched, runner.n
    slots = [d % n]
    if img is not None and runner._open is not None and runner.check(img.shape[:2])[1][:2] != runner._open['pad']:
        slots.append((d + 1) % n)
    for k in slots:
        for m in runner.slot_images[k]:
            if m['ticket'] not in done:
                done[m['ticket']] = read(m['ticket'])


def _host_path(sd, kw, rule, videos, order, batch, masks):
    """StreamRunner(vis=True) records of the same frames, the host Tracker per video, ytvis.video_json."""
    from sipmask_b200 import rle, ytvis
    from sipmask_b200.serving import StreamRunner
    sr = StreamRunner(sd, in_flight=2, batch=batch, max_src_hw=(1080, 1920), masks=masks, **rule, **kw)
    tickets, done = [], {}

    def read(t):
        k, j = sr._locate(t)
        r = sr.result(k if batch == 1 else t)
        cnt = int(r['count'].reshape(-1)[0])
        out = dict(det=r['det_bboxes'][:cnt].clone(), lab=r['det_labels'][:cnt].clone(), count=r['count'].clone(),
                   trk=r['track_feats'][:cnt].numpy().copy(), ori=sr.slot_images[k][j]['ori_shape'][:2])
        if masks == 'rle':
            out['segms'] = r['segms']
        else:
            out['bits'] = r['mask_bits'][:cnt].clone()
            out['segms'] = rle.encode_planes(out['bits'].numpy(), out['ori'])
        return out
    for v, f in order:
        _read_before_reuse(sr, read, done, videos[v][1][f])
        t = sr.i
        sr.submit(videos[v][1][f])
        tickets.append(t)
    _read_before_reuse(sr, read, done)
    sr.flush()
    for t in tickets:
        if t not in done:
            done[t] = read(t)
    recs = {(v, f): done[t] for (v, f), t in zip(order, tickets)}
    from sipmask_b200.tracker import Tracker
    ref64, js, frames = {}, {}, {}
    for v, (vid, fr) in enumerate(videos):
        tr, r64 = Tracker(COEF, native=False), Ref64()
        pairs = []
        for f in range(len(fr)):
            rec = recs[(v, f)]
            det, lab = rec['det'].numpy(), rec['lab'].numpy()
            ids = tr.step(det, lab, rec['trk'], f == 0)
            assert np.asarray(ids).tolist() == r64.step(det, lab, rec['trk'], f == 0).tolist()
            rec['ids'] = np.asarray(ids, np.int32)
            pairs.append(ytvis.frame_result(det, lab, ids, rec['segms']))
        ref64[vid] = r64
        frames[vid] = pairs
        js[vid] = ytvis.video_json(vid, pairs)
    return recs, js, frames, ref64


@pytest.mark.parametrize('batch,masks', [(1, 'rle'), (4, 'rle'), (4, 'bits')])
def test_video_runner_equals_stream_runner_and_host_tracker(batch, masks):
    from sipmask_b200.serving import VideoRunner
    sd, kw, rule = _sd()
    videos = _videos()
    order = _interleave(videos)
    recs, js, frames, ref64 = _host_path(sd, kw, rule, videos, order, batch, masks)
    assert min(r.worst for r in ref64.values()) > 0, 'a comparison is within the fp32 error bound: %s' % (
        [(v, r.worst, r.worst_at) for v, r in ref64.items()],)
    assert sum(int(r['count']) for r in recs.values()) >= 3 * len(recs)
    assert any((r['ids'] > 0).any() for r in recs.values()) and sum(r.n for r in ref64.values()) > 0
    vr = VideoRunner(sd, lanes=4, batch=batch, in_flight=2, max_src_hw=(1080, 1920), masks=masks, **rule, **kw)
    tickets, done = [], {}

    def read(t):
        r = vr.result(t)
        return dict(r, obj_ids=r['obj_ids'].clone(), det_bboxes=r['det_bboxes'].clone(), det_labels=r['det_labels'].clone(),
                    count=r['count'].clone(), mask_bits=r['mask_bits'].clone() if 'mask_bits' in r else None)
    for v, f in order:
        _read_before_reuse(vr, read, done, videos[v][1][f])
        tickets.append(vr.submit(videos[v][1][f], videos[v][0], f))
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    _read_before_reuse(vr, read, done)
    vr.flush()
    for t in tickets:
        if t not in done:
            done[t] = read(t)
    for (v, f), t in zip(order, tickets):
        got, want = done[t], recs[(v, f)]
        cnt = int(want['count'].reshape(-1)[0])
        assert 'track_feats' not in got
        assert torch.equal(got['count'].reshape(-1), want['count'].reshape(-1))
        assert torch.equal(got['det_bboxes'][:cnt], want['det']) and torch.equal(got['det_labels'][:cnt], want['lab'])
        if masks == 'rle':
            assert got['segms'] == want['segms']
        else:
            assert torch.equal(got['mask_bits'][:cnt], want['bits'])
        assert got['obj_ids'].tolist() == want['ids'].tolist(), (v, f)
        assert _same_frame(got['frame'], frames[videos[v][0]][f])
    for vid, _ in videos:
        assert vr.video_json(vid) == js[vid], vid
    assert len(vr.frames) == 0 and len(vr.book.videos) == 0


def _same_frame(a, b):
    (da, sa), (db, sb) = a, b
    if list(da) != list(db) or (isinstance(sa, list) != isinstance(sb, list)):
        return False
    for o in da:
        if not (np.array_equal(da[o]['bbox'], db[o]['bbox']) and da[o]['label'] == db[o]['label']):
            return False
    return sa == sb


def test_video_runner_rejections():
    from sipmask_b200.serving import VideoRunner
    sd, kw, rule = _sd()
    with pytest.raises(ValueError, match='vis=False'):
        VideoRunner(sd, **rule, **dict(kw, vis=False))
    vr = VideoRunner(sd, lanes=1, batch=2, in_flight=2, max_src_hw=(480, 640), **rule, **kw)
    img = _videos()[1][1][0]
    with pytest.raises(ValueError, match='frame 0'):
        vr.submit(img, 'a', 1)
    t0 = vr.submit(img, 'a', 0)
    with pytest.raises(ValueError, match='follows'):
        vr.submit(img, 'a', 2)
    with pytest.raises(ValueError, match='end_video'):
        vr.submit(img, 'b', 0)
    with pytest.raises(ValueError, match='has not ended'):
        vr.video_json('a')
    vr.end_video('a')
    with pytest.raises(ValueError, match='open batch'):
        vr.video_json('a')
    t1 = vr.submit(img, 'b', 0)                 # lane 0 again: closes the batch holding a's frame first
    assert vr.dispatched == 1 and vr.rows[t1][:2] == (0, True)
    vr.flush()
    assert vr.result(t0)['obj_ids'].tolist() == list(range(int(vr.result(t0)['count'].reshape(-1)[0])))
    assert len(vr.video_json('a')) == int(vr.result(t0)['count'].reshape(-1)[0])


def test_video_runner_reads_slots_before_new_engines():
    """Nothing read by the caller: the runner reads every slot itself before the slot takes a new batch.  Strings capped
    at 64 bytes per frame, so frames fall back to encoding their planes on the host, and frames of different padded shapes
    alternate in two slots, so new bucket engines are built (with a warm-up forward in the slot's arena) in slots that still
    hold unread frames: video_json must still equal the host path's."""
    from sipmask_b200.serving import VideoRunner
    sd, kw, rule = _sd()
    videos = _videos()
    order = _interleave(videos)
    _, js, _, _ = _host_path(sd, kw, rule, videos, order, 1, 'bits')
    per_frame = {}
    for vid, entries in js.items():
        for e in entries:
            for f, s in enumerate(e['segmentations']):
                if s is not None:
                    per_frame[(vid, f)] = per_frame.get((vid, f), 0) + len(s['counts'])
    assert max(per_frame.values()) > 64                   # some frames overflow the string capacity
    vr = VideoRunner(sd, lanes=4, batch=1, in_flight=2, max_src_hw=(1080, 1920), masks='rle', rle_bytes=64, **rule, **kw)
    for v, f in order:
        vr.submit(videos[v][1][f], videos[v][0], f)
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    vr.flush()
    assert all(len(d) >= 2 for d in vr.engines)            # every slot built engines of both padded shapes
    for vid, _ in videos:
        assert vr.video_json(vid) == js[vid], vid


def test_video_runner_overflow_raises_and_forgets_the_video():
    from sipmask_b200._lib import SmbError
    from sipmask_b200.serving import VideoRunner
    sd, kw, rule = _sd()
    img = _videos()[1][1][0]
    vr = VideoRunner(sd, lanes=1, batch=1, in_flight=2, max_src_hw=(480, 640), max_objects=2, **rule, **kw)
    t = vr.submit(img, 'a', 0)
    vr.end_video('a')
    vr.flush()
    with pytest.raises(SmbError, match="'a'"):
        vr.result(t)                                       # more detections than max_objects on the first frame
    with pytest.raises(SmbError, match="'a'"):
        vr.video_json('a')
    assert 'a' not in vr.book.videos and 'a' not in vr.frames and 'a' not in vr.overflowed
    t = vr.submit(img, 'a', 0)                             # the id is served again; the lane's overflow was cleared
    vr.end_video('a')
    vr.flush()
    with pytest.raises(SmbError):
        vr.result(t)                                       # the same frame overflows again, on its own
    vr2 = VideoRunner(sd, lanes=1, batch=1, in_flight=2, max_src_hw=(480, 640), max_objects=64, **rule, **kw)
    t = vr2.submit(img, 'a', 0)
    vr2.flush()
    assert int(vr2.result(t)['count'].reshape(-1)[0]) > 2


def test_track_assoc_rejects_malformed_state():
    from sipmask_b200 import ops
    lt = _lane_tracker(2, cap=8)
    det = torch.zeros((1, 10, 5), device='cuda')
    lab = torch.zeros((1, 10), dtype=torch.int64, device='cuda')
    cnt = torch.zeros((1,), dtype=torch.int32, device='cuda')
    feats = torch.zeros((1, 10, 512), device='cuda')
    rows = torch.zeros((1, 2), dtype=torch.int32, device='cuda')
    bad = [dict(lt.state, boxes=lt.boxes.cpu()), dict(lt.state, labels=lt.labels.int()),
           dict(lt.state, feats=lt.feats.transpose(0, 1).contiguous().transpose(0, 1)),
           dict(lt.state, n_obj=lt.n_obj[:1])]
    for state in bad:
        with pytest.raises(ValueError, match='state'):
            ops.track_assoc(rows, det, lab, cnt, feats, state)
    with pytest.raises(ValueError, match='ids'):
        ops.track_assoc(rows, det, lab, cnt, feats, lt.state, ids=torch.empty((1, 10), dtype=torch.int64, device='cuda'))
    with pytest.raises(ValueError, match='workspace'):
        ops.track_assoc(rows, det, lab, cnt, feats, lt.state, workspace=torch.empty(16, dtype=torch.uint8, device='cuda'))
    ids = ops.track_assoc(rows, det, lab, cnt, feats, lt.state)
    torch.cuda.synchronize()
    assert (ids.cpu() == -1).all()
