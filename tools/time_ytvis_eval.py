"""Time YouTube-VIS mask AP from the stream (serving.VideoEvalRunner) against the offline path.

The videos, weights and interleaved order of tools/time_video_stream.py (--videos videos of --frames frames of
720x1280, 1080x1920 and 480x640); the ground truth comes from one VideoRunner pass's json, each object's masks shifted by a
few pixels and some frames dropped.  Alternating, --reps times, in one process, best of the reps:
  (a) VideoRunner(lanes=8, masks='rle') and then ytviseval.evaluate_json on its json (every present frame's RLE string
      decoded on the host): frames/s from the first submit to the evaluation dict;
  (b) VideoEvalRunner with the same arguments: frames/s from the first submit to evaluate()'s dict;
at batch 1 (in_flight 6) and batch 8 (in_flight 2).  Then (c) each kernel alone on the device: CUDA events around 50
back-to-back launches queued behind a device sleep (so the host's enqueueing is not timed), per launch, median of 5:
overlap for a batch of 8 720x1280 frames of 10 detections and 10 ground-truth objects, scatter for the same batch, and
the sequence match of a video of 10 entries and 10 ground-truth objects.  Prints one JSON line (and writes it to --out)."""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def ground_truth(vids, js, seed=0):
    from sipmask_b200 import rle
    from sipmask_b200.cocoeval import segm_plane
    rs = np.random.RandomState(seed)
    ann = dict(videos=[], categories=[dict(id=c) for c in range(1, 41)], annotations=[])
    for v, frames in enumerate(vids):
        h, w = frames[0].shape[:2]
        ann['videos'].append(dict(id=v + 1, height=h, width=w, length=len(frames)))
        for ent in js[v + 1]:
            segs, areas = [], []
            dy, dx = rs.randint(-6, 7), rs.randint(-6, 7)
            for s in ent['segmentations']:
                if s is None or rs.rand() < 0.1:
                    segs.append(None)
                    areas.append(None)
                    continue
                m = np.unpackbits(segm_plane(s, h, w).view(np.uint8), axis=1, bitorder='little')[:, :w]
                m = np.roll(m, (dy, dx), (0, 1))
                r = rle.encode(m)
                segs.append({'size': r['size'], 'counts': r['counts'].decode()})
                areas.append(int(m.sum()))
            ann['annotations'].append(dict(id=len(ann['annotations']) + 1, video_id=v + 1, category_id=ent['category_id'],
                                           iscrowd=0, segmentations=segs, areas=areas))
    return ann


def run(vr, vids, order, gt=None):
    """Submit every frame; with gt, evaluate the runner's json offline (a), else evaluate() (b).  Returns (s, mAP)."""
    from sipmask_b200.ytviseval import evaluate_json
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for v, t in order:
        vr.submit(vids[v][t], v + 1, t)
        if t == len(vids[v]) - 1:
            vr.end_video(v + 1)
    if gt is None:
        r = vr.evaluate()
    else:
        vr.flush()
        js = [e for v in range(len(vids)) for e in vr.video_json(v + 1)]
        r = evaluate_json(gt, js)
    torch.cuda.synchronize()
    return time.perf_counter() - t0, r['stats']['segm'][0]


def _events(fn, launches=50, reps=5):
    out = []
    for _ in range(reps):
        torch.cuda._sleep(10 ** 7)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(launches):
            fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b) * 1e3 / launches)
    return round(float(np.median(out)), 2)


def kernels_alone():
    import ctypes
    from sipmask_b200 import _lib as L, rle, ytviseval as Y
    from sipmask_b200.ytviseval import YtvisEvaluator, YtvisGroundTruth
    h, w, N, mx, G = 720, 1280, 8, 10, 10
    rs = np.random.RandomState(0)
    pitch = (w + 31) // 32
    masks = []
    for g in range(G):
        m = np.zeros((h, w), np.uint8)
        y, x = rs.randint(0, h - 200), rs.randint(0, w - 200)
        m[y:y + 150, x:x + 180] = 1
        r = rle.encode(m)
        masks.append((m, {'size': r['size'], 'counts': r['counts'].decode()}))
    ann = dict(videos=[dict(id=1, height=h, width=w, length=N)], categories=[dict(id=1)],
               annotations=[dict(id=g + 1, video_id=1, category_id=1, segmentations=[s] * N, areas=[int(m.sum())] * N)
                            for g, (m, s) in enumerate(masks)])
    gt = YtvisGroundTruth(ann)
    ev = YtvisEvaluator(gt, slots=1, objects=mx, max_gts=G)
    ev.begin_video(1, 0)
    det = np.zeros((N, mx, h, pitch), np.uint32)
    for n in range(N):
        for j in range(mx):
            m = np.roll(masks[j][0], (3 * n, 2 * n), (0, 1))
            det[n, j] = np.packbits(np.pad(m, ((0, 0), (0, pitch * 32 - w))), axis=1, bitorder='little').view(np.uint32)
    planes = torch.from_numpy(det.view(np.int32)).cuda()
    staged = [ev.stage_frame(1, f) for f in range(N)]
    for s in staged:
        ev.commit_frame(s)
    count = torch.full((N,), mx, dtype=torch.int32, device='cuda')
    ids = torch.arange(mx, dtype=torch.int32, device='cuda').repeat(N, 1).contiguous()
    dets = [planes.data_ptr() + 4 * n * mx * h * pitch for n in range(N)]
    ovl = ev.overlap(staged, dets, h * pitch, pitch, mx, count=count)
    torch.cuda.synchronize()
    lib = L.lib()
    n_gts = sum(len(s_['rows']) for s_ in staged)

    def overlap():
        L.check(lib.smb_ytvis_overlap_dev(L.ptr(ovl['frames']), N, L.ptr(count), mx, L.ptr(ovl['gts']), n_gts, G,
                                          L.ptr(ovl['inter']), L.ptr(ovl['area']), L.ptr(ev.status), L.stream_ptr()),
                'smb_ytvis_overlap_dev')
    out = dict(overlap_us_8_frames=_events(overlap), scatter_us_8_frames=_events(lambda: ev.scatter(ovl, ids, count=count)))
    ents = np.zeros(mx, Y.ENT_DTYPE)
    ents['score'], ents['obj'], ents['cat'] = 1 - np.arange(mx) / 20, np.arange(mx), 0
    vg, off = gt.video(1)
    vg['sum_area'] = [int(m.sum()) * N for m, _ in masks]
    ents_d, vg_d, off_d = (Y._pinned_to(x, 'cuda') for x in (ents, vg, off))
    ws_bytes = lib.smb_ytvis_match_workspace_bytes(G)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    rows = torch.empty(mx * Y.OUT_DTYPE.itemsize, dtype=torch.uint8, device='cuda')

    def match():
        L.check(lib.smb_ytvis_match_dev(L.ptr(ents_d), mx, L.ptr(vg_d), G, L.ptr(off_d), 1, 0, L.ptr(ev.acc_inter),
                                        L.ptr(ev.acc_area), L.ptr(ev.acc_nz), 1, mx, G, ctypes.c_int64(1),
                                        Y._ptr(ev._iou_thr), Y._ptr(ev._area_rng), L.ptr(rows), ctypes.c_int64(mx),
                                        L.ptr(ev.npig), L.ptr(ev.status), L.ptr(ws), ctypes.c_size_t(ws_bytes),
                                        L.stream_ptr()), 'smb_ytvis_match_dev')
    out['match_us_per_video'] = _events(match)
    # algorithmic bytes of one overlap launch: every detection plane read once over the canvas, plus the ground-truth
    # words inside the overlapping extents (bounded by one more read of each ground-truth plane per detection)
    out['overlap_plane_bytes_8_frames'] = N * mx * h * pitch * 4
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--videos', type=int, default=8)
    ap.add_argument('--frames', type=int, default=12)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from time_video_stream import videos, weights
    from sipmask_b200.serving import VideoEvalRunner, VideoRunner
    from sipmask_b200.ytviseval import YtvisGroundTruth
    sd = weights()
    vids, order = videos(a.videos, a.frames)
    n_frames = len(order)
    kw = dict(lanes=8, resize=(640, 360), max_src_hw=(1080, 1920), masks='rle')
    vr = VideoRunner(sd, batch=1, in_flight=6, **kw)
    for v, t in order:
        vr.submit(vids[v][t], v + 1, t)
        if t == len(vids[v]) - 1:
            vr.end_video(v + 1)
    vr.flush()
    js = {v + 1: vr.video_json(v + 1) for v in range(len(vids))}
    del vr
    gc.collect()
    gt = YtvisGroundTruth(ground_truth(vids, js))
    out = dict(videos=a.videos, frames=n_frames, gt_objects=sum(len(x) for x in gt.anns.values()),
               entries=sum(len(x) for x in js.values()))
    for batch, in_flight in ((1, 6), (8, 2)):
        best = {}
        for _ in range(a.reps):
            for name in ('offline', 'stream'):
                r = (VideoRunner(sd, batch=batch, in_flight=in_flight, **kw) if name == 'offline'
                     else VideoEvalRunner(sd, gt, batch=batch, in_flight=in_flight, **kw))
                for k in range(in_flight):                 # build the bucket engines outside the timed region
                    for frames in vids[:3]:
                        r._engine(k, r.check(frames[0].shape[:2])[1][:2])
                s, ap_ = run(r, vids, order, gt if name == 'offline' else None)
                best[name] = max(best.get(name, 0.0), n_frames / s)
                best[name + '_mAP'] = round(float(ap_), 6)
                del r
                gc.collect()
        out['batch%d' % batch] = {k: (round(v, 1) if not k.endswith('mAP') else v) for k, v in best.items()}
    out['kernels'] = kernels_alone()
    out['gpu'] = torch.cuda.get_device_name()
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
