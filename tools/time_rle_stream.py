"""COCO RLE output of the serving runners: bit planes + host encoding against strings encoded on the device.

Two streams, each served by StreamRunner with masks='bits' and with masks='rle' (alternating, --reps times, one process):
  * batch32: BASELINE config 4 (R50-FPN SSD-style head, 544x544 keep_ratio=False), batch=32, in_flight=2, on a seeded
    shuffled stream of tools/time_stream.py's MIX_WH raw sizes (DESIGN.md §6);
  * batch1: the R50-GN model at 1333x800 keep_ratio (800x1344 and smaller padded shapes), batch=1, in_flight=6, same mix.
Seeded synthetic weights with the classifier bias at -2.5 and smooth seeded images (blobs + noise), so that the images
have detections (100 each; uniform noise images give none with config 4's weights).
Per stream and mode: images/s from the first submit to the last image's RLE dicts on the host.  (a) masks='bits': every
returned detection's planes are copied out of the pinned record and encoded with rle.encode on --threads host threads;
(b) masks='rle': the strings are read from the slot's region (fallback_images: images whose strings overflowed and were
encoded on the host).  Also the D2H bytes per image of both modes, the mean
detections per image, and the encoder node alone (CUDA events over 50 launches with 100 detections per image of blob
masks on a 480x640 canvas): its algorithmic bytes (bit planes read once + headers and strings written) and GB/s.
Prints one JSON line (and writes it to --out when given)."""
import argparse
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def serve(sr, stream, pool):
    """One pass: submit every image; read each batch before its slot is reused; returns (seconds, stats)."""
    from sipmask_b200 import rle
    n, B = sr.n, sr.B
    futures, stats = [], dict(dets=0, d2h=0, images=0, fallback=0)
    fixed = None
    state = dict(next=sr.dispatched)

    def read(b):
        nonlocal fixed
        k = b % n
        for m in sr.slot_images[k]:
            r = sr.result(m['ticket'] if B > 1 else k)
            cnt = int(r['count'].reshape(-1)[0])
            if fixed is None:
                fixed = sum(r[f].numel() * r[f].element_size() for f in ('det_bboxes', 'det_labels', 'count', 'idxs_keep'))
            stats['dets'] += cnt
            stats['images'] += 1
            if sr.rle:
                segms = r['segms']
                ib = sr.engines[k][m['pad_shape'][:2]].rle_img_bytes
                j = sr.slot_images[k].index(m)
                stats['fallback'] += rle.read_region(sr.rle_regions[k].numpy()[j * ib:(j + 1) * ib],
                                                     r['det_bboxes'].shape[0])[0] != 0
                stats['d2h'] += fixed + rle.header_bytes(r['det_bboxes'].shape[0]) + sum(len(s['counts']) for s in segms)
            else:
                stats['d2h'] += fixed + r['mask_bits'].numel() * 4
                futures.append(pool.submit(rle.encode_planes, r['mask_bits'][:cnt].numpy().copy(), m['ori_shape'][:2]))

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    first = sr.dispatched
    for img in stream:
        sr.submit(img)
        while state['next'] <= sr.dispatched - n:       # the slot the next dispatch reuses
            read(state['next'])
            state['next'] += 1
    sr.flush()
    while state['next'] < sr.dispatched:
        read(state['next'])
        state['next'] += 1
    for f in futures:
        f.result()
    dt = time.perf_counter() - t0
    assert stats['images'] == len(stream), (stats, len(stream), sr.dispatched - first)
    return dt, stats


def encoder_alone(eng, reps=50):
    """The encoder node on eng's record with every detection slot filled: blob masks on a 480x640 canvas."""
    from sipmask_b200 import ops, rle
    N, mx, cap_h, words = eng.mask_bits.shape
    oh, ow = 480, 640
    eng.set_image_meta([((eng.H, eng.W, 3), (oh, ow, 3), np.array([eng.W / ow, eng.H / oh] * 2, np.float32))] * N)
    rs = np.random.RandomState(0)
    yy, xx = np.mgrid[:oh, :ow]
    px = np.zeros((mx, cap_h, words * 32), np.uint8)
    for d in range(mx):
        cy, cx, ry, rx = rs.uniform(0, oh), rs.uniform(0, ow), rs.uniform(10, 200), rs.uniform(10, 250)
        px[d, :oh, :ow] = (((yy - cy) / ry) ** 2 + ((xx - cx) / rx) ** 2 < 1).astype(np.uint8)
    planes = torch.from_numpy(np.packbits(px, axis=-1, bitorder='little').view('<i4').copy()).cuda()
    eng.mask_bits.copy_(planes.unsqueeze(0).expand(N, -1, -1, -1))
    eng.count.fill_(mx)
    ib = eng.rle_img_bytes
    region = torch.zeros(N * ib, dtype=torch.uint8).pin_memory()
    dst = torch.tensor([ops.host_device_pointer(region)], dtype=torch.int64).cuda()
    ws = torch.empty(ops.rle_encode_workspace_bytes(N, mx, eng.rle_runs), dtype=torch.uint8, device='cuda')
    run = lambda: ops.rle_encode_dev(eng.mask_bits, eng.count, eng.geom, dst, ib, eng.rle_runs, ws)   # noqa: E731
    for _ in range(5):
        run()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        run()
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / reps
    written = 0
    for n in range(N):
        status, k, strings = rle.read_region(region.numpy()[n * ib:(n + 1) * ib], mx)
        assert status == 0 and k == mx, status
        written += rle.header_bytes(mx) + sum(len(s) for s in strings)
    read = N * mx * oh * ((ow + 31) // 32) * 4
    return dict(images=N, detections_per_image=mx, canvas='%dx%d' % (oh, ow), us=us, bytes_read=read, bytes_written=written,
                gb_per_s=(read + written) / us * 1e-3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=448, help='images per pass of the batch-32 stream')
    ap.add_argument('--images-b1', type=int, default=140, help='images per pass of the batch-1 stream')
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--threads', type=int, default=8, help='host threads encoding the planes in masks=bits mode')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_rle_stream measures the GPU'
    import bench
    from time_stream import MIX_WH
    from sipmask_b200 import synth
    from sipmask_b200.serving import StreamRunner
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    rs = np.random.RandomState(0)

    def blobs(w, h):
        # smooth random blobs + noise: with the synthetic weights (cls_bias -2.5) every image fills its 100 detections
        base = torch.from_numpy(rs.randint(0, 256, (3, h // 16 + 2, w // 16 + 2)).astype(np.float32))[None]
        img = torch.nn.functional.interpolate(base, size=(h, w), mode='bilinear', align_corners=False)[0].permute(1, 2, 0)
        noise = torch.from_numpy(rs.randint(-20, 21, (h, w, 3)).astype(np.float32))
        return (img + noise).clamp(0, 255).to(torch.uint8).contiguous().pin_memory()
    imgs = {wh: blobs(*wh) for wh in MIX_WH}

    def stream_of(count):
        sizes = [MIX_WH[i % len(MIX_WH)] for i in range(count)]
        rs.shuffle(sizes)
        return [imgs[wh] for wh in sizes]

    wl = bench.WORKLOADS['B']
    sd_b = synth.detector_state_dict(wl['depth'], stacked_convs=wl['stacked'], gn=wl['gn'], cls_bias=-2.5)
    kw_b = dict(depth=wl['depth'], stacked_convs=wl['stacked'], gn=wl['gn'], ssd_flag=wl['ssd'], test_cfg=bench.test_cfg(wl),
                resize=(wl['W'], wl['H']), keep_ratio=False, max_src_hw=(640, 640), max_ori_hw=(640, 640))
    sd_1 = synth.detector_state_dict(50, stacked_convs=4, gn=True, cls_bias=-2.5)
    kw_1 = dict(max_src_hw=(1333, 1333), max_ori_hw=(640, 640), min_mask_up=0.9)
    setups = {'batch32_in_flight2': (sd_b, dict(kw_b, batch=wl['batch'], in_flight=2), stream_of(a.images)),
              'batch1_in_flight6': (sd_1, dict(kw_1, batch=1, in_flight=6), stream_of(a.images_b1))}
    pool = ThreadPoolExecutor(a.threads)
    res = dict(card=card, threads=a.threads, mix_wh=['%dx%d' % wh for wh in MIX_WH], streams={})
    for name, (sd, kw, stream) in setups.items():
        runners = {m: StreamRunner(sd, masks=m, **kw) for m in ('bits', 'rle')}
        for sr in runners.values():                   # build + capture every bucket of every slot
            serve(sr, stream[:max(len(stream) // 2, kw['batch'] * kw['in_flight'] * 2)] + list(imgs.values()) * kw['in_flight'],
                  pool)
        runs = []
        for _ in range(a.reps):
            r = {}
            for m, sr in runners.items():
                dt, st = serve(sr, stream, pool)
                r[m] = dict(images_per_s=len(stream) / dt, d2h_bytes_per_image=st['d2h'] / st['images'],
                            detections_per_image=st['dets'] / st['images'], fallback_images=st['fallback'])
            runs.append(r)
        med = {m: float(np.median([r[m]['images_per_s'] for r in runs])) for m in runners}
        eng = next(iter(runners['rle'].engines[0].values()))
        res['streams'][name] = dict(images_per_pass=len(stream), images_per_s_median=med, runs=runs,
                                    encoder_alone=encoder_alone(eng))
        del runners, eng
        torch.cuda.empty_cache()
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
