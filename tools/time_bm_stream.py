"""Throughput of SipMask-benchmark (BM) R50 serving a stream of raw RGB images: seeded synthetic weights
(benchmark.synthetic_state_dict), the benchmark's test rule (min 800, max 1333), and a seeded, shuffled stream of the raw
sizes in tools/time_stream.py's MIX_WH (seven sizes, six padded shapes under the BM rule).

  (a) StreamRunner(benchmark=True, raw=True, batch=1, in_flight=6): the PIL-bilinear preprocessing on the GPU;
  (b) the same with batch=B for each B of --batches (a batch closes early when the next image has another padded shape);
  (c) StreamRunner(benchmark=True, in_flight=6) fed fp32 images that the chain of (d) made before timing: the GPU-side
      rate of serving BM checkpoints without the raw mode (host preprocessing excluded);
  (d) the host work (c) leaves out: the reference-equivalent chain (PIL Image.resize(BILINEAR), BGR, mean, pad) per image
      on `--threads` host threads;
  (e) the preprocessing kernel alone: CUDA events over 50 launches of one batch of --kernel-batch 640x480 images
      (800x1066 in an 800x1088 canvas), and TB/s against its algorithmic bytes (sum of source bytes read +
      N * (H/2+3) * (W/2+4) * 32 bytes written);
and the H2D bytes per image for raw uint8 and for padded fp32 input.  (a)-(c) alternate `--reps` times in one process,
each also on a stream of one size (640x480, one padded shape: "_single_size"), where every batch fills.
Prints one JSON line (and writes it to --out when given)."""
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
    ap.add_argument('--images', type=int, default=210, help='images per pass')
    ap.add_argument('--reps', type=int, default=3)
    ap.add_argument('--batches', default='4', help='comma-separated batch sizes for (b)')
    ap.add_argument('--batch-in-flight', type=int, default=2, help='in_flight of the (b) runners')
    ap.add_argument('--threads', type=int, default=8, help='host threads for (d)')
    ap.add_argument('--kernel-batch', type=int, default=8)
    ap.add_argument('--out', default=None, help='also write the JSON line to this file')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_bm_stream measures the GPU'
    import subprocess
    from time_stream import MIX_WH
    from PIL import Image
    from sipmask_b200 import _lib as L, benchmark as BM, conv as C
    from sipmask_b200.serving import StreamRunner, bm_image_meta
    card = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                          text=True).stdout.strip()
    sd = BM.convert_state_dict(BM.synthetic_state_dict(depth=50))
    ekw = dict(depth=50, benchmark=True)
    rs = np.random.RandomState(0)
    sizes = [MIX_WH[i % len(MIX_WH)] for i in range(a.images)]
    rs.shuffle(sizes)
    rgb = {wh: rs.randint(0, 256, (wh[1], wh[0], 3), dtype=np.uint8) for wh in MIX_WH}
    raw = {wh: torch.from_numpy(x).pin_memory() for wh, x in rgb.items()}
    meta = {wh: bm_image_meta(wh[1], wh[0]) for wh in MIX_WH}
    mean = np.asarray(MEAN, np.float32)

    def prep(x):
        """The reference-equivalent host chain: PIL resize, BGR, minus the mean, zero pad to 32 -> fp32 [3, H, W]."""
        (oh, ow, _), (ph, pw, _), _ = bm_image_meta(x.shape[0], x.shape[1])
        r = np.asarray(Image.fromarray(x, 'RGB').resize((ow, oh), Image.BILINEAR))
        out = np.zeros((3, ph, pw), np.float32)
        out[:, :oh, :ow] = (r[:, :, ::-1].astype(np.float32) - mean).transpose(2, 0, 1)
        return out
    fp32 = {wh: torch.from_numpy(prep(x))[None].pin_memory() for wh, x in rgb.items()}
    stream = list(sizes)
    # 500x375 is the steepest mask resize of the mix (resized 800x1066: masks resized by 0.94)
    rule = dict(max_src_hw=(640, 640), max_ori_hw=(640, 640), min_mask_up=0.9)

    runners = {'raw_batch1_in_flight6': StreamRunner(sd, in_flight=6, raw=True, **rule, **ekw)}
    for B in [int(v) for v in a.batches.split(',')]:
        runners['raw_batch%d_in_flight%d' % (B, a.batch_in_flight)] = StreamRunner(
            sd, in_flight=a.batch_in_flight, batch=B, raw=True, **rule, **ekw)
    runners['fp32_preprocessed_in_flight6'] = StreamRunner(sd, in_flight=6, **rule, **ekw)

    def feed(sr, wh):
        if sr.bm_raw:
            sr.step(raw[wh])
        else:
            img_shape, _, sf = meta[wh]
            sr.step(fp32[wh], meta=(img_shape, (wh[1], wh[0], 3), sf))

    for sr in runners.values():                           # build + capture every bucket of every slot
        for _ in range(sr.n * sr.B):
            for wh in MIX_WH:
                feed(sr, wh)
        sr.flush()
    torch.cuda.synchronize()

    def run(sr, whs):
        torch.cuda.synchronize()
        d0 = sr.dispatched
        t0 = time.perf_counter()
        for wh in whs:
            feed(sr, wh)
        sr.flush()
        torch.cuda.synchronize()
        return len(whs) / (time.perf_counter() - t0), len(whs) / (sr.dispatched - d0)

    runs, per_batch = [], {}
    single = [(640, 480)] * len(stream)
    for _ in range(a.reps):
        r = {}
        for k, sr in runners.items():
            r[k], per_batch[k] = run(sr, stream)
            r[k + '_single_size'], per_batch[k + '_single_size'] = run(sr, single)
        runs.append(r)
    med = {k: float(np.median([r[k] for r in runs])) for k in runs[0]}

    # (d) the host preprocessing (c) leaves out: PIL resize + BGR + mean + pad to 32, per image
    from concurrent.futures import ThreadPoolExecutor
    np_imgs = [rgb[wh] for wh in stream]
    with ThreadPoolExecutor(a.threads) as ex:
        list(ex.map(prep, np_imgs[:32]))
        t0 = time.perf_counter()
        list(ex.map(prep, np_imgs))
        dt = time.perf_counter() - t0
    host = dict(threads=a.threads, images_per_s=len(np_imgs) / dt,
                ms_per_image_per_thread=1e3 * dt * a.threads / len(np_imgs))

    # (e) the preprocessing kernel alone: one batch of 640x480 images, 800x1066 in an 800x1088 canvas
    N = a.kernel_batch
    dev = torch.device('cuda', torch.cuda.current_device())
    (oh, ow, _), (H, W, _), _ = meta[(640, 480)]
    srcs = [torch.from_numpy(rs.randint(0, 256, (480, 640, 3), dtype=np.uint8)).cuda() for _ in range(N)]
    rows = (L.RawSrc * N)(*[C.raw_src_row(s, (oh, ow), (H, W), MEAN, dev, order='RGB', max_downscale=C.PIL_MAX_DOWNSCALE)
                            for s in srcs])
    rows_dev = torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()
    out = torch.empty((N, H // 2 + 3, W // 2 + 4, 16), dtype=torch.float16, device=dev)
    for _ in range(5):
        C.preprocess_pil_rows(rows_dev, out)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(50):
        C.preprocess_pil_rows(rows_dev, out)
    e1.record()
    torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 1e3 / 50
    nbytes = sum(s.numel() for s in srcs) + out.numel() * out.element_size()
    kernel = dict(batch=N, src_hw=(480, 640), resized_hw=(oh, ow), canvas_hw=(H, W), us_per_batch=us, bytes=nbytes,
                  tb_per_s=nbytes / us * 1e-6)

    h2d = dict(raw_uint8=float(np.mean([wh[0] * wh[1] * 3 for wh in stream])),
               fp32_padded=float(np.mean([3 * meta[wh][1][0] * meta[wh][1][1] * 4 for wh in stream])))
    res = dict(card=card, workload='BM R50, min 800 / max 1333, synthetic weights', images_per_pass=len(stream),
               mix_wh=['%dx%d' % wh for wh in MIX_WH], images_per_s_median=med, runs=runs,
               images_per_forward=per_batch, host_pil_preprocess=host, preprocess_kernel=kernel, h2d_bytes_per_image=h2d,
               buckets={k: ['%dx%d' % hw for hw in sr.buckets] for k, sr in runners.items()},
               arena_bytes_per_slot={k: sr.arena_bytes for k, sr in runners.items()})
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or '.', exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
