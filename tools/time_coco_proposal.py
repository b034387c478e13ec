"""Time MM's 'proposal' metric (COCOeval of the bbox results with useCats = 0, maxDets 100 / 300 / 1000) on the device.

Reports, on a seeded synthetic dataset of `--images` images (default 5000) over 80 categories with up to
`--max-results` (default 1000) box results per image:
  - offline: CocoEvaluator.add_results + evaluate() of 'proposal' alone, and of 'bbox' (default Params) on the same
    results for comparison;
  - match2_kernel's device time per image (torch.profiler, CUDA activity) over the first `--profile-images` images;
  - CocoEvalRunner images/s with metrics ('bbox', 'segm') and ('bbox', 'segm', 'proposal') on the same stream of
    `--runner-images` images (config B shapes, synthetic weights), so the difference is the per-batch cost of 'proposal'.
The GPU's name and power limit are printed with the numbers.

    python tools/time_coco_proposal.py --images 5000
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def dataset(n_img, max_results, seed=0, n_cat=80):
    """Ground truth of 0..14 boxes per image; per image a uniform number of results in [max_results / 2, max_results]:
    two jittered copies of each ground truth in its category, the rest random boxes of random categories."""
    rng = np.random.default_rng(seed)
    gt = dict(images=[], categories=[dict(id=c + 1) for c in range(n_cat)], annotations=[])
    per = {}
    aid = 0
    for i in range(n_img):
        h, w = int(rng.integers(360, 481)), int(rng.integers(480, 641))
        gt['images'].append(dict(id=i + 1, height=h, width=w))
        boxes, cats = [], []
        for _ in range(int(rng.integers(0, 15))):
            aid += 1
            cat = int(rng.integers(1, n_cat + 1))
            x0, y0 = float(rng.uniform(0, w - 30)), float(rng.uniform(0, h - 30))
            bw, bh = float(rng.uniform(4, min(200, w - x0))), float(rng.uniform(4, min(200, h - y0)))
            gt['annotations'].append(dict(id=aid, image_id=i + 1, category_id=cat, bbox=[x0, y0, bw, bh], area=bw * bh,
                                          iscrowd=int(rng.random() < 0.01), segmentation=[[x0, y0, x0, y0 + bh,
                                                                                           x0 + bw, y0 + bh, x0 + bw, y0]]))
            boxes += [[x0 + rng.normal(0, 3), y0 + rng.normal(0, 3), bw, bh] for _ in range(2)]
            cats += [cat, cat]
        n = int(rng.integers(max_results // 2, max_results + 1))
        k = max(n - len(boxes), 0)
        xy = rng.uniform(0, 1, (k, 2)) * [w - 40, h - 40]
        wh = rng.uniform(4, 40, (k, 2))
        boxes = (boxes + np.concatenate([xy, wh], 1).tolist())[:n]
        cats = (cats + rng.integers(1, n_cat + 1, k).tolist())[:n]
        scores = rng.random(n).astype(np.float32).astype(np.float64)
        per[i + 1] = [dict(image_id=i + 1, category_id=int(c), bbox=b, score=float(s))
                      for c, b, s in zip(cats, boxes, scores)]
    return gt, per


def offline(g, per, metric, chunk):
    import torch
    from sipmask_b200 import cocoeval as C
    ev = C.CocoEvaluator(g, g.cat_ids, metrics=(metric,))
    ids = sorted(per)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c in range(0, len(ids), chunk):
        ev.add_results([(i, per[i]) for i in ids[c:c + chunk]], metric)
    ev.n_results[metric] += sum(len(v) for v in per.values())
    ev.image_ids = list(ids)
    torch.cuda.synchronize()
    t_add = time.perf_counter() - t0
    t0 = time.perf_counter()
    r = ev.evaluate()
    t_eval = time.perf_counter() - t0
    key = 'AR@1000' if metric == 'proposal' else 'bbox_mAP'
    return dict(add_results_s=round(t_add, 3), evaluate_s=round(t_eval, 4), **{key: r[key]})


def kernel_times(g, per, n, chunk):
    """Device time of every match2_kernel launch of 'proposal' over the first n images (one launch per image)."""
    import torch
    from torch.profiler import profile, ProfilerActivity
    from sipmask_b200 import cocoeval as C
    ev = C.CocoEvaluator(g, g.cat_ids, metrics=('proposal',))
    ids = g.img_ids[:n]
    ev.add_results([(i, per[i]) for i in ids[:chunk]], 'proposal')      # warm-up: module load, smem attribute
    torch.cuda.synchronize()
    ev = C.CocoEvaluator(g, g.cat_ids, metrics=('proposal',))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in range(0, len(ids), chunk):
            ev.add_results([(i, per[i]) for i in ids[c:c + chunk]], 'proposal')
        torch.cuda.synchronize()
    us = [e.device_time for e in prof.events() if 'match2_kernel' in e.name]
    n_res = [len(per[i]) for i in ids]
    return dict(launches=len(us), mean_us=round(float(np.mean(us)), 1), max_us=round(float(np.max(us)), 1),
                mean_results_per_image=round(float(np.mean(n_res)), 1))


def runner(n, batch, in_flight=2, reps=2):
    """Images/s of CocoEvalRunner (masks='rle', evaluate() included) with and without 'proposal'; best of reps,
    alternating the two."""
    import torch
    from sipmask_b200 import cocoeval as C, synth
    from sipmask_b200.serving import CocoEvalRunner
    from time_coco_eval import _images
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, cls_bias=-2.5)
    kw = dict(depth=50, stacked_convs=2, gn=False, ssd_flag=True, resize=(544, 544), keep_ratio=False, batch=batch,
              in_flight=in_flight, max_src_hw=(640, 640), max_ori_hw=(640, 640), masks='rle',
              test_cfg=dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100))
    imgs, gt = _images(n, seed=0)
    g = C.CocoGroundTruth(gt)
    best = {}
    for _ in range(reps):
        for name, metrics in (('bbox_segm', ('bbox', 'segm')), ('bbox_segm_proposal', ('bbox', 'segm', 'proposal'))):
            r = CocoEvalRunner(sd, g, list(range(1, 81)), metrics=metrics, **kw)
            for k in range(in_flight):
                r._engine(k, (544, 544))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i, img in enumerate(imgs):
                r.submit(img, i + 1)
            r.evaluate()
            torch.cuda.synchronize()
            best[name] = max(best.get(name, 0.0), n / (time.perf_counter() - t0))
            del r
            gc.collect()
    out = {k + '_images_per_s': round(v, 1) for k, v in best.items()}
    out['proposal_ms_per_batch'] = round((1 / best['bbox_segm_proposal'] - 1 / best['bbox_segm']) * batch * 1e3, 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--max-results', type=int, default=1000)
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--profile-images', type=int, default=256)
    ap.add_argument('--runner-images', type=int, default=256)
    ap.add_argument('--batch', type=int, default=8)
    a = ap.parse_args()
    import torch
    from sipmask_b200 import cocoeval as C
    if not torch.cuda.is_available():
        raise SystemExit('time_coco_proposal: no CUDA device')
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True)
    out = dict(gpu=q.stdout.strip() or torch.cuda.get_device_name())
    t0 = time.perf_counter()
    gt, per = dataset(a.images, a.max_results)
    g = C.CocoGroundTruth(gt)
    out.update(images=a.images, gt=len(gt['annotations']), results=sum(len(v) for v in per.values()),
               dataset_s=round(time.perf_counter() - t0, 2))
    offline(g, {i: per[i] for i in g.img_ids[:a.chunk]}, 'proposal', a.chunk)          # warm-up
    out['proposal'] = offline(g, per, 'proposal', a.chunk)
    out['bbox'] = offline(g, per, 'bbox', a.chunk)
    if a.profile_images:
        out['match2_kernel'] = kernel_times(g, per, a.profile_images, a.chunk)
    if a.runner_images:
        out['runner'] = dict(images=a.runner_images, batch=a.batch, **runner(a.runner_images, a.batch))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
