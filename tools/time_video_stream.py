"""SipMask-VIS video serving: the device tracker association (VideoRunner) against the host association.

Seeded synthetic videos (moving smooth blobs plus noise) of 720x1280, 1080x1920 and 480x640 frames, --videos of them
interleaved frame by frame, and seeded synthetic VIS weights (R50-FPN, 3-conv towers, 40 classes) with the classifier bias
lowered to -1 so that frames fill their max_per_img = 10 detections.  Alternating, --reps times, in one process:
  (a) VideoRunner(lanes=8, masks='rle') at batch=1, in_flight=6 and at batch=8, in_flight=2: frames/s from the first
      submit to the last video's json;
  (b) StreamRunner(vis=True, masks='rle') at batch=1, in_flight=6, the host Tracker per video on the downloaded records
      (with their 512-d features) and ytvis.video_json, on the same frames;
  (c) the association kernel alone with m = 10, 100, 1000 tracked objects per lane and 1, 8, 32 lanes, one frame of 10
      detections per lane: CUDA events around 50 back-to-back launches queued behind a device sleep (so the host's
      enqueueing is not timed), per launch, median of 5.
Also the D2H bytes per frame of (a) and (b), the host microseconds per frame spent in each runner's per-batch steps
(submit, the download / association enqueue, reading a frame), and the device time of the association kernel in one
(a) batch-1 pass under torch.profiler.  Prints one JSON line (and writes it to --out when given)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = ((720, 1280), (1080, 1920), (480, 640))


def weights():
    from sipmask_b200 import synth
    sd = {}
    sd.update(synth.backbone_state_dict(50, 1))
    sd.update(synth.neck_state_dict(2))
    sd.update(synth.head_state_dict(3, num_classes=41, stacked_convs=3, gn=True, cls_bias=-1.0, track=True))
    return sd


def videos(n_videos, n_frames, seed=0):
    rs = np.random.RandomState(seed)
    out = []
    for v in range(n_videos):
        h, w = SIZES[v % len(SIZES)]
        base = rs.randint(0, 256, (h // 16 + 8, w // 16 + 8, 3)).astype(np.float32)
        big = torch.nn.functional.interpolate(torch.from_numpy(base).permute(2, 0, 1)[None], size=(h + 4 * n_frames,
                                                                                                 w + 6 * n_frames),
                                              mode='bilinear', align_corners=False)[0].permute(1, 2, 0)
        frames = []
        for t in range(n_frames):
            img = big[4 * t:4 * t + h, 6 * t:6 * t + w] + torch.from_numpy(rs.randint(-10, 11, (h, w, 3)).astype(np.float32))
            frames.append(img.clamp(0, 255).to(torch.uint8).contiguous().pin_memory())
        out.append(frames)
    order = [(v, t) for t in range(n_frames) for v in range(n_videos)]
    return out, order


def run_device(vr, vids, order):
    """(a): returns (seconds, D2H bytes per frame)."""
    from sipmask_b200 import rle
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for v, t in order:
        vr.submit(vids[v][t], v, t)
        if t == len(vids[v]) - 1:
            vr.end_video(v)
    vr.flush()
    # D2H of the frames still held by the slots (the json reads them): the record without features, ids, status, strings
    d2h, n = 0, 0
    for k in range(vr.n):
        for m in vr.slot_images[k]:
            r = vr.result(m['ticket'])
            d2h += sum(r[f].numel() * r[f].element_size() for f in ('det_bboxes', 'det_labels', 'count', 'idxs_keep'))
            d2h += r['det_labels'].numel() * 4 + vr.tracker.lanes * 4 // vr.B
            d2h += rle.header_bytes(r['det_labels'].numel()) + sum(len(s['counts']) for s in r['segms'])
            n += 1
    for v in range(len(vids)):
        vr.video_json(v)
    return time.perf_counter() - t0, d2h / max(n, 1)


def run_host(sr, vids, order):
    """(b): StreamRunner + host Tracker per video + ytvis.video_json; returns (seconds, D2H bytes per frame)."""
    from sipmask_b200 import rle, ytvis
    from sipmask_b200.tracker import Tracker
    trackers = [Tracker() for _ in vids]
    frames = [[] for _ in vids]
    stats = dict(d2h=0, n=0, read_s=0.0)

    def take(k, v, t):
        t0 = time.perf_counter()
        take_(k, v, t)
        stats['read_s'] += time.perf_counter() - t0

    def take_(k, v, t):
        r = sr.result(k)
        cnt = int(r['count'].reshape(-1)[0])
        det, lab = r['det_bboxes'][:cnt].numpy(), r['det_labels'][:cnt].numpy()
        ids = trackers[v].step(det, lab, r['track_feats'][:cnt].numpy(), t == 0)
        frames[v].append(ytvis.frame_result(det, lab, ids, r['segms']))
        stats['d2h'] += sum(r[f].numel() * r[f].element_size() for f in ('det_bboxes', 'det_labels', 'count', 'idxs_keep',
                                                                          'track_feats'))
        stats['d2h'] += rle.header_bytes(r['det_labels'].numel()) + sum(len(s['counts']) for s in r['segms'])
        stats['n'] += 1
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    pending = []
    for v, t in order:
        if len(pending) >= sr.n:                         # read the oldest frame before its slot is reused
            take(*pending.pop(0))
        pending.append((sr.submit(vids[v][t]), v, t))
    sr.flush()
    for p in pending:
        take(*p)
    for v in range(len(vids)):
        ytvis.video_json(v, frames[v])
    run_host.read_s = getattr(run_host, 'read_s', 0.0) + stats['read_s']
    return time.perf_counter() - t0, stats['d2h'] / stats['n']


def kernel_us(m, lanes, launches=50):
    """(c): the association launch alone with m tracked objects on each of `lanes` lanes, one 10-detection frame each.
    Detection i of a lane carries tracked object i's features, so it claims that object and the state keeps m objects:
    every launch does the same work.  A device sleep queued before the start event covers the host's enqueueing of the
    launches, so the events time `launches` back-to-back kernels; returns microseconds per launch (median of 5)."""
    from sipmask_b200 import ops
    from sipmask_b200.tracker import LaneTracker
    g = torch.Generator(device='cuda').manual_seed(m + lanes)
    lt = LaneTracker(lanes, max(m, 16), device='cuda', max_rows=lanes)
    lt.feats.copy_(torch.randn(lt.feats.shape, generator=g, device='cuda'))
    lt.boxes.copy_(torch.rand(lt.boxes.shape, generator=g, device='cuda') * 100)
    lt.boxes[..., 2:4] += lt.boxes[..., 0:2] + 8
    lt.boxes[..., 4] = 0.5
    lt.labels.copy_(torch.randint(0, 40, lt.labels.shape, generator=g, device='cuda'))
    det = lt.boxes[:, :10].contiguous()
    lab = lt.labels[:, :10].contiguous()
    feats = lt.feats[:, :10].contiguous()
    cnt = torch.full((lanes,), min(10, m), dtype=torch.int32, device='cuda')
    rows = torch.tensor([[l, 0] for l in range(lanes)], dtype=torch.int32, device='cuda')
    ws = torch.empty(ops.track_assoc_workspace_bytes(lanes, 10, lt.capacity), dtype=torch.uint8, device='cuda')
    ids = torch.empty((lanes, 10), dtype=torch.int32, device='cuda')
    lt.n_obj.fill_(m)
    ops.track_assoc(rows, det, lab, cnt, feats, lt.state, ids=ids, workspace=ws)
    torch.cuda.synchronize()
    assert lt.n_obj.cpu().tolist() == [m] * lanes, 'the timed launches must not change the number of objects'
    times = []
    for _ in range(5):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(200_000_000)                   # ~0.1 s of device time: the host enqueues under it
        e0.record()
        for _ in range(launches):
            ops.track_assoc(rows, det, lab, cnt, feats, lt.state, ids=ids, workspace=ws)
        e1.record()
        e1.synchronize()
        times.append(e0.elapsed_time(e1) * 1e3 / launches)
    return float(np.median(times))


class HostTimer(object):
    """Host seconds spent in wrapped methods of one object (tool-side instrumentation)."""

    def __init__(self, obj, names):
        self.t = {n: 0.0 for n in names}
        for n in names:
            f = getattr(obj, n)

            def wrapped(*a, _f=f, _n=n, **k):
                t0 = time.perf_counter()
                try:
                    return _f(*a, **k)
                finally:
                    self.t[_n] += time.perf_counter() - t0
            setattr(obj, n, wrapped)


def profile_device_pass(vr, vids, order):
    """One (a) pass under torch.profiler: the device time of the association kernel and of the whole GPU work."""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        run_device(vr, vids, order)
        torch.cuda.synchronize()
    assoc, calls = 0.0, 0
    for e in prof.key_averages():
        dt = getattr(e, 'device_time_total', None)
        if dt is None:
            dt = getattr(e, 'cuda_time_total', 0.0)
        if 'track_assoc_kernel' in e.key:
            assoc += dt
            calls += e.count
    return dict(assoc_kernel_us_per_launch=round(assoc / max(calls, 1), 2), assoc_launches=calls,
                assoc_kernel_us_per_frame=round(assoc / len(order), 2))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--videos', type=int, default=6)
    ap.add_argument('--frames', type=int, default=24)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    from sipmask_b200.serving import StreamRunner, VideoRunner, VIS_ENGINE_KW
    sd = weights()
    vids, order = videos(a.videos, a.frames)
    kw = dict(max_src_hw=(1080, 1920), masks='rle')
    runners = dict(dev_b1=lambda: VideoRunner(sd, lanes=8, batch=1, in_flight=6, **kw),
                   dev_b8=lambda: VideoRunner(sd, lanes=8, batch=8, in_flight=2, **kw),
                   host_b1=lambda: StreamRunner(sd, in_flight=6, resize=(640, 360), **kw, **VIS_ENGINE_KW))
    built = {k: f() for k, f in runners.items()}
    # warm-up: every bucket engine of every slot built and captured
    for name, r in built.items():
        (run_host if name.startswith('host') else run_device)(r, vids, order)
    # host seconds in the per-batch steps: the download enqueue (VideoRunner: plus the association enqueue), the reading
    # of a frame (VideoRunner: record, ids, frame pair; host path: record, host Tracker step, frame pair) and submit overall
    timers = {k: HostTimer(r, ('submit', '_download') + (('_read',) if k.startswith('dev') else ()))
              for k, r in built.items()}
    run_host.read_s = 0.0
    res = {k: [] for k in built}
    d2h = {}
    for _ in range(a.reps):
        for name, r in built.items():
            secs, b = (run_host if name.startswith('host') else run_device)(r, vids, order)
            res[name].append(len(order) / secs)
            d2h[name] = b
    nf = a.reps * len(order)
    host_us = {k: {n: round(v / nf * 1e6, 1) for n, v in t.t.items()} for k, t in timers.items()}
    host_us['host_b1']['read_and_track'] = round(run_host.read_s / nf * 1e6, 1)
    prof = profile_device_pass(built['dev_b1'], vids, order)
    kern = {'m%d_lanes%d' % (m, l): kernel_us(m, l) for m in (10, 100, 1000) for l in (1, 8, 32)}
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip().splitlines()
    out = dict(card=card[0] if card else torch.cuda.get_device_name(), frames=len(order), videos=a.videos,
               frames_per_s={k: [round(x, 1) for x in v] for k, v in res.items()},
               d2h_bytes_per_frame={k: round(v) for k, v in d2h.items()}, host_us_per_frame=host_us, profile_dev_b1=prof,
               kernel_us={k: round(v, 2) for k, v in kern.items()})
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
