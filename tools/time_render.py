"""Detections drawn on the device: the render kernel alone, and what StreamRunner(render=True) costs a stream.

  kernel : one 800x1333 image with 100 detections (rectangle-and-ellipse masks and boxes of 32-512 px, every score above
           the threshold), the image rule with boxes, drawn out of place (source -> render buffer, as the runner does);
           a CUDA graph of --launches launches, timed with CUDA events.  Reported against the byte floor: the image read
           and written (2 x 3.2 MB) plus every detection's mask words over the image's rows (100 x 800 x 42 x 4 B).
  stream : bench.py workload A's model (R50-FPN-GN, seeded synthetic weights, classifier bias -2.5 so that images fill
           their 100 detections) on a stream of raw 800x1333 images (smooth seeded blobs + noise), batch=1,
           in_flight=6, every record read before its slot is reused; render off and on alternated --reps times each in
           this one process.  images/s from the first submit to the last result().
The card's name and power limit are read in the same run.  Prints one JSON line (and writes it to --out when given)."""
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


def blobs(rs, h, w):
    base = torch.from_numpy(rs.randint(0, 256, (3, h // 16 + 2, w // 16 + 2)).astype(np.float32))[None]
    img = torch.nn.functional.interpolate(base, size=(h, w), mode='bilinear', align_corners=False)[0].permute(1, 2, 0)
    noise = torch.from_numpy(rs.randint(-20, 21, (h, w, 3)).astype(np.float32))
    return (img + noise).clamp(0, 255).to(torch.uint8).contiguous()


def kernel_alone(launches):
    from sipmask_b200 import _lib as L
    from sipmask_b200 import ops, render
    h, w, mx = 800, 1333, 100
    words = (w + 31) // 32
    rs = np.random.RandomState(0)
    yy, xx = np.mgrid[:h, :w]
    px = np.zeros((mx, h, words * 32), np.uint8)
    det = np.zeros((1, mx, 5), np.float32)
    for d in range(mx):
        bh, bw = rs.randint(32, 513, 2)
        y0, x0 = rs.randint(0, h - min(bh, h - 1)), rs.randint(0, w - bw)
        cy, cx = y0 + bh / 2, x0 + bw / 2
        px[d, :h, :w] = ((((yy - cy) / (bh / 2)) ** 2 + ((xx - cx) / (bw / 2)) ** 2 < 1) |
                         ((np.abs(yy - cy) < bh / 4) & (np.abs(xx - cx) < bw / 4)))
        det[0, d] = (x0, y0, x0 + bw, y0 + bh, rs.uniform(0.31, 1))
    bits = torch.from_numpy(np.packbits(px, axis=-1, bitorder='little').view('<i4').copy()).cuda()[None]
    det = torch.from_numpy(det).cuda()
    labels = torch.from_numpy(rs.randint(0, 80, (1, mx))).cuda()
    count = torch.full((1,), mx, dtype=torch.int32, device='cuda')
    src = blobs(rs, h, w).cuda()
    dst = torch.empty_like(src)
    rows = render.rows([(src, dst, h, w)], src.device)
    pal = render.device_palette(render.image_palette(81), src.device)
    run = lambda: ops.render(rows, 1, (h, w), bits, det, count, pal, L.RENDER_IMAGES, 0.3, True, labels=labels)  # noqa: E731
    run()
    torch.cuda.synchronize()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.stream(s):
        with torch.cuda.graph(g, stream=s):
            for _ in range(launches):
                run()
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    reps = 10
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / (reps * launches)
    img_bytes = 2 * h * w * 3
    mask_bytes = mx * h * words * 4
    return dict(image='%dx%d' % (h, w), detections=mx, launches_per_graph=launches, us=us, image_bytes=img_bytes,
                mask_bytes=mask_bytes, gb_per_s=(img_bytes + mask_bytes) / us * 1e-3)


def serve(sr, stream):
    """Submit every image, read each record (render included) before its slot is reused; returns seconds."""
    n = sr.n
    state = dict(next=sr.dispatched)
    drawn = [0]

    def read(b):
        r = sr.result(b % n)
        if 'render' in r:
            drawn[0] += int(r['count'].reshape(-1)[0])
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for img in stream:
        sr.submit(img)
        while state['next'] <= sr.dispatched - n:
            read(state['next'])
            state['next'] += 1
    sr.flush()
    while state['next'] < sr.dispatched:
        read(state['next'])
        state['next'] += 1
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=240, help='images per pass of the stream')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--launches', type=int, default=20, help='render launches per CUDA graph')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_render measures the GPU'
    from sipmask_b200 import synth
    from sipmask_b200.serving import StreamRunner
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    res = dict(card=card, kernel=kernel_alone(a.launches))
    rs = np.random.RandomState(1)
    imgs = [blobs(rs, 800, 1333).pin_memory() for _ in range(8)]
    stream = [imgs[i % len(imgs)] for i in range(a.images)]
    sd = synth.detector_state_dict(50, stacked_convs=4, gn=True, cls_bias=-2.5)
    kw = dict(depth=50, stacked_convs=4, gn=True, test_cfg=dict(nms_pre=1000, score_thr=0.05,
                                                                nms=dict(type='nms', iou_thr=0.5), max_per_img=100),
              resize=(1333, 800), keep_ratio=True, max_src_hw=(800, 1333), max_ori_hw=(800, 1333), batch=1, in_flight=6)
    runners = {on: StreamRunner(sd, render=on, **kw) for on in (False, True)}
    for sr in runners.values():
        serve(sr, stream[:48])                        # build + capture every slot's engine, warm the pinned buffers
    runs = {False: [], True: []}
    for _ in range(a.reps):
        for on, sr in runners.items():
            runs[on].append(len(stream) / serve(sr, stream))
    med = {on: float(np.median(v)) for on, v in runs.items()}
    res['stream'] = dict(images_per_pass=len(stream), image='800x1333', in_flight=6, batch=1,
                         render_off_images_per_s=runs[False], render_on_images_per_s=runs[True],
                         median_off=med[False], median_on=med[True], on_over_off=med[True] / med[False],
                         d2h_render_bytes_per_image=800 * 1333 * 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
