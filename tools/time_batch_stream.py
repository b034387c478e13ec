"""Throughput of a raw uint8 image stream served in batches: BASELINE config 4 (R50-FPN SSD-style head, 544x544
keep_ratio=False, seeded synthetic weights) on a seeded, shuffled stream of the raw sizes in tools/time_stream.py's MIX_WH.

  (a) StreamRunner(batch=32), in_flight 1 and 2: images/s from the first submit to the last record on the host;
  (b) StreamRunner(batch=1, in_flight=6) on the same stream: serving raw images one per forward;
  (c) a batch-32 PipelinedRunner fed one pre-made pinned fp32 batch per step, as bench.py --workload B measures end to
      end (host-side resize / normalisation excluded);
  (d) the host work (c) leaves out: cv2.resize + mean subtraction per image on `--threads` host threads;
  (e) the batched preprocessing kernel alone: CUDA events over 50 launches of one 32-image batch, and GB/s against its
      algorithmic bytes (sum of source bytes read + 32 * (H/2+3) * (W/2+4) * 32 bytes written);
and the D2H bytes per image of (a).  (a)-(c) alternate `--reps` times in one process.  Prints one JSON line (and writes
it to --out when given)."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))

MEAN = (102.9801, 115.9465, 122.7717)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=640, help='images per pass')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--threads', type=int, default=8, help='host threads for (d)')
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_batch_stream measures the GPU'
    import subprocess
    import bench
    from time_stream import MIX_WH
    from sipmask_b200 import _lib as L, conv as C, synth
    from sipmask_b200.serving import PipelinedRunner, StreamRunner, make_engines
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    wl = bench.WORKLOADS['B']
    B, H, W = wl['batch'], wl['H'], wl['W']
    sd = bench.state_dict_for(wl)
    ekw = dict(depth=wl['depth'], stacked_convs=wl['stacked'], gn=wl['gn'], ssd_flag=wl['ssd'], test_cfg=bench.test_cfg(wl))
    rs = np.random.RandomState(0)
    sizes = [MIX_WH[i % len(MIX_WH)] for i in range(a.images)]
    rs.shuffle(sizes)
    imgs = {wh: torch.from_numpy(rs.randint(0, 256, (wh[1], wh[0], 3), dtype=np.uint8)).pin_memory() for wh in MIX_WH}
    stream = [imgs[wh] for wh in sizes]
    rule = dict(resize=(W, H), keep_ratio=False, max_src_hw=(640, 640), max_ori_hw=(640, 640))

    runners = {'batch32_in_flight1': StreamRunner(sd, in_flight=1, batch=B, **rule, **ekw),
               'batch32_in_flight2': StreamRunner(sd, in_flight=2, batch=B, **rule, **ekw),
               'batch1_in_flight6': StreamRunner(sd, in_flight=6, batch=1, **rule, **ekw)}
    for sr in runners.values():                           # build + capture every slot's engine
        for img in stream[:B * sr.n] + stream[:sr.n]:
            sr.step(img)
        sr.flush()
    engs = make_engines(sd, (H, W), in_flight=1, batch=B, img_shape=(H, W, 3), scale_factor=np.ones(4, np.float32),
                        use_graph=True, **ekw)
    batch_host = torch.cat([synth.synthetic_image(H, W, seed=b) for b in range(B)], 0).pin_memory()
    pr = PipelinedRunner(engs)
    torch.cuda.synchronize()

    def run_stream(sr):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for img in stream:
            sr.step(img)
        sr.flush()
        torch.cuda.synchronize()
        return len(stream) / (time.perf_counter() - t0)

    def run_fp32_batches():
        steps = max(1, len(stream) // B)
        for _ in range(2):
            pr.step(batch_host)
        pr.drain()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(steps):
            pr.step(batch_host)
        pr.drain()
        torch.cuda.synchronize()
        return steps * B / (time.perf_counter() - t0)

    runs = []
    for _ in range(a.reps):
        r = {k: run_stream(sr) for k, sr in runners.items()}
        r['fp32_batches_pipelined'] = run_fp32_batches()
        runs.append(r)
    med = {k: float(np.median([r[k] for r in runs])) for k in runs[0]}

    # (d) host preprocessing the pre-made fp32 batches leave out
    host = None
    try:
        import cv2
        from concurrent.futures import ThreadPoolExecutor
        cv2.setNumThreads(1)
        mean = np.asarray(MEAN, np.float32)
        np_imgs = [s.numpy() for s in stream]

        def prep(x):
            return cv2.resize(x, (W, H), interpolation=cv2.INTER_LINEAR).astype(np.float32) - mean
        with ThreadPoolExecutor(a.threads) as ex:
            list(ex.map(prep, np_imgs[:64]))
            t0 = time.perf_counter()
            list(ex.map(prep, np_imgs))
            dt = time.perf_counter() - t0
        host = dict(threads=a.threads, images_per_s=len(np_imgs) / dt, ms_per_image_per_thread=1e3 * dt * a.threads / len(np_imgs))
    except ImportError:
        pass

    # (e) the batched preprocessing kernel alone, on the first 32 images of the stream
    dev = torch.device('cuda', torch.cuda.current_device())
    srcs = [s.cuda() for s in stream[:B]]
    rows = (L.RawSrc * B)(*[C.raw_src_row(s, (H, W), (H, W), MEAN, dev) for s in srcs])
    rows_dev = torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()
    out = torch.empty((B, H // 2 + 3, W // 2 + 4, 16), dtype=torch.float16, device=dev)
    for _ in range(5):
        C.preprocess_u8_rows(rows_dev, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        C.preprocess_u8_rows(rows_dev, out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 50
    nbytes = sum(s.numel() for s in srcs) + out.numel() * out.element_size()
    kernel = dict(us_per_batch=us, bytes=nbytes, gb_per_s=nbytes / us * 1e-3)

    # D2H per image of (a): the record with mask_bits cropped to [max, ori_h, ceil(ori_w / 32)]
    mx = next(iter(runners['batch32_in_flight1'].engines[0].values())).max_num
    fixed = mx * 5 * 4 + mx * 8 + 4 + mx * 8
    d2h = float(np.mean([fixed + mx * wh[1] * ((wh[0] + 31) // 32) * 4 for wh in sizes]))

    res = dict(card=card, workload='config 4: ' + wl['name'], images_per_pass=len(stream),
               mix_wh=['%dx%d' % wh for wh in MIX_WH], batch=B, images_per_s_median=med, runs=runs,
               host_preprocess=host, preprocess_kernel=kernel, d2h_bytes_per_image=d2h,
               arena_bytes_per_slot={k: sr.arena_bytes for k, sr in runners.items()})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
