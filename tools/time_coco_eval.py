"""Time the device COCO evaluation on a seeded synthetic dataset.

Reports, for `--images` images (default 5000) with about 7 ground truths and 30 detections per image over 80 categories:
  - add_results: the per-batch path (host ground-truth rasterization + detection decoding + match launches), per metric;
  - evaluate(): the device sort + accumulate + download + summarize;
and the host time of the test restatement (tests/cocoeval_ref.py) on the first `--oracle-images` images.  The
restatement is plain Python, not pycocotools: its time is not pycocotools' time.

    python tools/time_coco_eval.py --images 5000 --oracle-images 100
"""
import argparse
import gc
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _rect_string(h, w, x0, y0, x1, y1):
    """The compressed RLE string of a rectangle, from its column-major runs (no mask is built)."""
    from sipmask_b200 import rle
    x0, x1, y0, y1 = max(x0, 0), min(x1, w), max(y0, 0), min(y1, h)
    if x1 <= x0 or y1 <= y0:
        return rle.to_string([h * w]).decode()
    hh = y1 - y0
    cnts = [x0 * h + y0]
    for _ in range(x1 - x0 - 1):
        cnts += [hh, h - hh]
    cnts += [hh, h * w - sum(cnts) - hh]
    return rle.to_string(cnts).decode()


def dataset(n_img, seed=0, n_cat=80):
    rng = np.random.default_rng(seed)
    gt = dict(images=[], categories=[dict(id=c + 1) for c in range(n_cat)], annotations=[])
    bbox, segm = [], []
    aid = 0
    for i in range(n_img):
        h, w = int(rng.integers(360, 481)), int(rng.integers(480, 641))
        gt['images'].append(dict(id=i + 1, height=h, width=w))
        objs = []
        for _ in range(int(rng.integers(0, 15))):
            aid += 1
            cat = int(rng.integers(1, n_cat + 1))
            x0, y0 = float(rng.uniform(0, w - 30)), float(rng.uniform(0, h - 30))
            bw, bh = float(rng.uniform(4, min(200, w - x0))), float(rng.uniform(4, min(200, h - y0)))
            poly = [x0, y0, x0 + bw * 0.5, y0 - 2, x0 + bw, y0, x0 + bw, y0 + bh, x0, y0 + bh]
            gt['annotations'].append(dict(id=aid, image_id=i + 1, category_id=cat, bbox=[x0, y0, bw, bh], area=bw * bh,
                                          iscrowd=int(rng.random() < 0.01), segmentation=[poly]))
            objs.append((cat, x0, y0, bw, bh))
        dets = [(c, x + rng.normal(0, 3), y + rng.normal(0, 3), bw, bh) for c, x, y, bw, bh in objs for _ in range(2)]
        dets += [(int(rng.integers(1, n_cat + 1)), float(rng.uniform(0, w - 40)), float(rng.uniform(0, h - 40)),
                  float(rng.uniform(4, 40)), float(rng.uniform(4, 40))) for _ in range(int(rng.integers(5, 25)))]
        for c, x, y, bw, bh in dets:
            s = float(np.float32(rng.random()))
            bbox.append(dict(image_id=i + 1, category_id=c, bbox=[x, y, bw, bh], score=s))
            segm.append(dict(image_id=i + 1, category_id=c, score=s, segmentation={
                'size': [h, w], 'counts': _rect_string(h, w, int(x), int(y), int(x + bw), int(y + bh))}))
    return gt, bbox, segm


def _images(n, seed):
    """Smooth random blobs (a plain uniform image gives few detections with synthetic weights), with a ground truth of
    random box polygons per image."""
    import torch
    rs = np.random.RandomState(seed)
    sizes = [(427, 640), (480, 640), (375, 500), (640, 480)]
    imgs, gt = [], dict(images=[], categories=[dict(id=c + 1) for c in range(80)], annotations=[])
    for i in range(n):
        h, w = sizes[i % len(sizes)]
        base = torch.from_numpy(rs.randint(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.float32))
        img = torch.nn.functional.interpolate(base.permute(2, 0, 1)[None], size=(h, w), mode='bilinear',
                                              align_corners=False)[0].permute(1, 2, 0)
        imgs.append(img.clamp(0, 255).to(torch.uint8).contiguous().pin_memory())
        gt['images'].append(dict(id=i + 1, height=h, width=w))
        for _ in range(7):
            x0, y0 = float(rs.uniform(0, w - 40)), float(rs.uniform(0, h - 40))
            bw, bh = float(rs.uniform(8, 40)), float(rs.uniform(8, 40))
            gt['annotations'].append(dict(id=len(gt['annotations']) + 1, image_id=i + 1, category_id=int(rs.randint(1, 81)),
                                          bbox=[x0, y0, bw, bh], area=bw * bh, iscrowd=0,
                                          segmentation=[[x0, y0, x0, y0 + bh, x0 + bw, y0 + bh, x0 + bw, y0]]))
    return imgs, gt


def runner_throughput(n, batch, in_flight, reps=2):
    """Images/s of CocoEvalRunner (masks='rle', both metrics, evaluate() included) against StreamRunner(masks='rle')
    without evaluation, config B shapes (544 x 544 resize, SSD head, R50), synthetic weights; best of reps."""
    import torch
    from sipmask_b200 import cocoeval as C, synth
    from sipmask_b200.serving import CocoEvalRunner, StreamRunner
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, cls_bias=-2.5)
    kw = dict(depth=50, stacked_convs=2, gn=False, ssd_flag=True, resize=(544, 544), keep_ratio=False, batch=batch,
              in_flight=in_flight, max_src_hw=(640, 640), max_ori_hw=(640, 640), masks='rle',
              test_cfg=dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100))
    imgs, gt = _images(n, seed=0)
    g = C.CocoGroundTruth(gt)
    out = {}
    for name in ('rle', 'rle_eval'):
        best = 0.0
        for _ in range(reps):
            r = StreamRunner(sd, **kw) if name == 'rle' else CocoEvalRunner(sd, g, list(range(1, 81)), **kw)
            for k in range(in_flight):                     # build the bucket engines outside the timed region
                r._engine(k, (544, 544))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i, img in enumerate(imgs):
                if name == 'rle':
                    r.submit(img)
                else:
                    r.submit(img, i + 1)
            if name == 'rle':
                r.flush()
            else:
                r.evaluate()
            torch.cuda.synchronize()
            best = max(best, n / (time.perf_counter() - t0))
            del r
            gc.collect()
        out[name + '_images_per_s'] = round(best, 1)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--oracle-images', type=int, default=100)
    ap.add_argument('--chunk', type=int, default=64)
    ap.add_argument('--runner-images', type=int, default=256)
    ap.add_argument('--batch', type=int, default=8)
    a = ap.parse_args()
    import torch
    from sipmask_b200 import cocoeval as C
    t0 = time.perf_counter()
    gt, bbox, segm = dataset(a.images)
    t_data = time.perf_counter() - t0
    g = C.CocoGroundTruth(gt)
    out = dict(images=a.images, gt=len(gt['annotations']), dets=len(bbox), dataset_s=round(t_data, 2))
    for metric, res in (('bbox', bbox), ('segm', segm)):
        ev = C.CocoEvaluator(g, g.cat_ids, metrics=(metric,))
        ids = g.img_ids
        per = {}
        for r in res:
            per.setdefault(r['image_id'], []).append(r)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for c in range(0, len(ids), a.chunk):
            chunk = ids[c:c + a.chunk]
            ev.add_results([(i, per.get(i, [])) for i in chunk], metric)
        ev.n_results[metric] += len(res)
        torch.cuda.synchronize()
        t_add = time.perf_counter() - t0
        t0 = time.perf_counter()
        r = ev.evaluate()
        t_eval = time.perf_counter() - t0
        out[metric] = dict(add_results_s=round(t_add, 3), evaluate_s=round(t_eval, 4),
                           mAP=r['%s_mAP' % metric])
    if a.oracle_images:
        sys.path.insert(0, os.path.join(ROOT, 'tests'))
        import cocoeval_ref as R
        n = a.oracle_images
        gsub = dict(gt, images=gt['images'][:n], annotations=[x for x in gt['annotations'] if x['image_id'] <= n])
        for metric, res in (('bbox', bbox), ('segm', segm)):
            sub = [x for x in res if x['image_id'] <= n]
            t0 = time.perf_counter()
            R.run(gsub, sub, metric)
            out['restatement_%s_s_for_%d_images' % (metric, n)] = round(time.perf_counter() - t0, 2)
    if a.runner_images:
        out['runner'] = dict(images=a.runner_images, batch=a.batch, **runner_throughput(a.runner_images, a.batch, 2))
    print(json.dumps(out))


if __name__ == '__main__':
    main()
