"""Time the COCO error analysis on the device (cocoeval.analyze_json / CocoEvaluator(analyze=True)).

Seeded dataset: tools/time_coco_eval.py's (about 7 ground truths and 30 detections per image, `--images` images) with
80 categories in 12 supercategories, like COCO.  Reports:
  - offline, per metric: evaluate_json (the plain evaluation) and analyze_json (the plain evaluation plus the analysis'
    two matches per image and its accumulates), wall time;
  - the match launches alone for one chunk of images: the plain match, then the plain match plus the analysis' two (the
    [.75, .5, .1] / maxDets [100] match behind ps[0:3] and the Sim / Oth match behind ps[3:5]) (CUDA events, launches
    queued behind a device sleep so that the host enqueue time is not measured);
  - CocoEvalRunner images/s with and without analyze=True (time_coco_eval.py's runner configuration);
  - the host time of the restated tool (tests/coco_analysis_ref.py, plain Python, NOT pycocotools) on the first
    `--oracle-images` images.

    python tools/time_coco_analysis.py --images 5000 --oracle-images 20
"""
import argparse
import gc
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tools'))


def dataset(n_img, seed=0):
    from time_coco_eval import dataset as base
    gt, bbox, segm = base(n_img, seed=seed)
    for c in gt['categories']:
        c['name'] = 'c%d' % c['id']
        c['supercategory'] = 's%d' % ((c['id'] - 1) * 12 // 80)
    return gt, bbox, segm


def kernel_times(g, res, metric, chunk, reps=5):
    """Milliseconds of the match launches of one chunk of images, per kind, median of reps."""
    import torch
    from sipmask_b200 import cocoeval as C

    class Capture(C.CocoEvaluator):
        calls = []

        def _match(self, *args):
            Capture.calls.append(args)
            return super(Capture, self)._match(*args)

    ev = Capture(g, g.cat_ids, metrics=(metric,), analyze=True)
    per = {}
    for r in res:
        per.setdefault(r['image_id'], []).append(r)
    ids = g.img_ids[:chunk]
    ev.add_results([(i, per.get(i, [])) for i in ids], metric)
    torch.cuda.synchronize()
    # the first call of each image rasterized its ground truth and cleared gt['raster']: the replays below launch only
    # the matches (they add to npig again, which the timing does not read)
    assert all(args[7]['raster'] is None for args in Capture.calls)
    out = {}
    for kind in ('plain', 'plain+analysis'):
        ev.analyze = kind != 'plain'
        ts = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(200_000_000)
            a.record()
            for args in Capture.calls:
                C.CocoEvaluator._match(ev, *args)
            b.record()
            torch.cuda.synchronize()
            ts.append(a.elapsed_time(b))
        out[kind + '_ms'] = round(sorted(ts)[reps // 2], 3)
    out['analysis_ms'] = round(out['plain+analysis_ms'] - out['plain_ms'], 3)
    out['images'] = len(ids)
    return out


def runner_throughput(n, batch, in_flight, reps=2):
    import torch
    from sipmask_b200 import cocoeval as C, synth
    from sipmask_b200.serving import CocoEvalRunner
    from time_coco_eval import _images
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, cls_bias=-2.5)
    kw = dict(depth=50, stacked_convs=2, gn=False, ssd_flag=True, resize=(544, 544), keep_ratio=False, batch=batch,
              in_flight=in_flight, max_src_hw=(640, 640), max_ori_hw=(640, 640), masks='rle',
              test_cfg=dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100))
    imgs, gt = _images(n, seed=0)
    for c in gt['categories']:
        c['supercategory'] = 's%d' % ((c['id'] - 1) * 12 // 80)
    g = C.CocoGroundTruth(gt)
    out = {}
    for analyze in (False, True):
        best = 0.0
        for _ in range(reps):
            r = CocoEvalRunner(sd, g, list(range(1, 81)), analyze=analyze, **kw)
            for k in range(in_flight):
                r._engine(k, (544, 544))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i, img in enumerate(imgs):
                r.submit(img, i + 1)
            r.evaluate()
            torch.cuda.synchronize()
            best = max(best, n / (time.perf_counter() - t0))
            del r
            gc.collect()
        out[('analyze' if analyze else 'plain') + '_images_per_s'] = round(best, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--oracle-images', type=int, default=20)
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--runner-images', type=int, default=256)
    ap.add_argument('--batch', type=int, default=8)
    a = ap.parse_args()
    import torch
    from sipmask_b200 import cocoeval as C
    gt, bbox, segm = dataset(a.images)
    g = C.CocoGroundTruth(gt)
    out = dict(images=a.images, gt=len(gt['annotations']), dets=len(bbox), categories=80, supercategories=12)
    for metric, res in (('bbox', bbox), ('segm', segm)):
        kw = {metric + '_json': res}
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        C.evaluate_json(g, g.cat_ids, chunk=a.chunk, **kw)
        t_plain = time.perf_counter() - t0
        t0 = time.perf_counter()
        C.analyze_json(g, chunk=a.chunk, **kw)
        t_ana = time.perf_counter() - t0
        out[metric] = dict(evaluate_json_s=round(t_plain, 3), analyze_json_s=round(t_ana, 3),
                           kernels=kernel_times(g, res, metric, a.chunk))
    if a.runner_images:
        out['runner'] = dict(images=a.runner_images, batch=a.batch, **runner_throughput(a.runner_images, a.batch, 2))
    if a.oracle_images:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import coco_analysis_ref as AR
        n = a.oracle_images
        gsub = dict(gt, images=gt['images'][:n], annotations=[x for x in gt['annotations'] if x['image_id'] <= n])
        sub = [x for x in bbox if x['image_id'] <= n]
        t0 = time.perf_counter()
        AR.analyze_results(gsub, sub, 'bbox')
        out['restated_tool_bbox_s_for_%d_images' % n] = round(time.perf_counter() - t0, 2)
        t0 = time.perf_counter()
        C.analyze_json(C.CocoGroundTruth(gsub), bbox_json=sub)
        out['device_bbox_s_for_%d_images' % n] = round(time.perf_counter() - t0, 3)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
