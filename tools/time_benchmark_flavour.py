"""Time the SipMask-benchmark (BM) engine against the MM workload-A engine, and the two BM post-processing kernels alone.

    python tools/time_benchmark_flavour.py [--rounds 3] [--steps 200] [--out DIR]

- Engines: R50 at 800x1344 (img_shape 800x1333), six images in flight (serving.make_engines + EnginePool), synthetic
  weights that give detections; BM and MM alternate `--rounds` times.  Reports images/s.
- Kernels: smb_pair_decode_topk on the 800x1344 pyramid with normal inputs (logits ~ N(-4, 2)) and saturated inputs (every
  pair passes), and smb_ml_nms_topk on 5000 candidates (1 and 80 labels); CUDA events over many launches.
The card name and power limit are read in the same run and printed with the results (one JSON line).
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from sipmask_b200 import benchmark as B, ops, synth  # noqa: E402
from sipmask_b200.serving import EnginePool, make_engines  # noqa: E402

STRIDES = (8, 16, 32, 64, 128)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else 'unknown'


def engine_rate(engs, steps):
    for e, s in zip(engs, range(len(engs))):
        e.img.copy_(synth.synthetic_image(800, 1344, seed=s).cuda())
    pool = EnginePool(engs)
    for _ in range(20):
        pool.step()
    pool.flush()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        pool.step()
    pool.flush()
    torch.cuda.synchronize()
    return steps / (time.perf_counter() - t0)


def time_ms(fn, iters=50):
    for _ in range(5):
        fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def kernels():
    g = torch.Generator().manual_seed(0)
    sizes = [((800 + s - 1) // s, (1344 + s - 1) // s) for s in STRIDES]
    out = {}
    for name, mean, std in (('normal', -4.0, 2.0), ('saturated', 3.0, 0.5)):
        cls = [(torch.randn(h, w, 80, generator=g) * std + mean).cuda() for h, w in sizes]
        box = [(torch.randn(h, w, 4, generator=g) * 4 * s).abs().cuda() for (h, w), s in zip(sizes, STRIDES)]
        ctr = [torch.randn(h, w, 1, generator=g).cuda() for h, w in sizes]
        res = ops.pair_decode_topk(cls, box, ctr, STRIDES, (800, 1333), 1000, 0.05)
        out['pair_decode_%s_ms' % name] = time_ms(lambda: ops.pair_decode_topk(cls, box, ctr, STRIDES, (800, 1333), 1000, 0.05))
        out['pair_decode_%s_candidates' % name] = int(res[4].item())
        bx, sc, lab, _, n = res
        out['ml_nms_%s_ms' % name] = time_ms(lambda: ops.ml_nms_topk(bx, sc, lab, n, 0.6, 100, out_cap=100))
    for nl in (1, 80):
        rng = torch.Generator().manual_seed(nl)
        xy = torch.rand(5000, 2, generator=rng) * 1200
        bx = torch.cat([xy, xy + 4 + torch.rand(5000, 2, generator=rng) * 200], 1).cuda()
        sc = torch.rand(5000, generator=rng).cuda()
        lab = torch.randint(0, nl, (5000,), generator=rng, dtype=torch.int32).cuda()
        n = torch.tensor([5000], dtype=torch.int32).cuda()
        out['ml_nms_5000_labels%d_ms' % nl] = time_ms(lambda: ops.ml_nms_topk(bx, sc, lab, n, 0.6, 100, out_cap=100))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--in-flight', type=int, default=6)
    a = ap.parse_args()
    res = dict(card=card())
    sd_mm = synth.detector_state_dict(depth=50, seed=1)
    sd_bm = B.convert_state_dict(B.synthetic_state_dict(depth=50, seed=1))
    kw = dict(in_flight=a.in_flight, img_shape=(800, 1333, 3), use_graph=True)
    mm = make_engines(sd_mm, (800, 1344), **kw)
    bm = make_engines(sd_bm, (800, 1344), benchmark=True, **kw)
    res['mm_img_s'], res['bm_img_s'] = [], []
    for _ in range(a.rounds):
        res['mm_img_s'].append(round(engine_rate(mm, a.steps), 1))
        res['bm_img_s'].append(round(engine_rate(bm, a.steps), 1))
    res['bm_kept_total'] = bm[0].kept_total.tolist()
    res.update({k: (round(v, 4) if isinstance(v, float) else v) for k, v in kernels().items()})
    res['card_after'] = card()
    print(json.dumps(res))


if __name__ == '__main__':
    main()
