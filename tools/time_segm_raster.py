"""Time the device rasterizer of segmentations (csrc/segm_raster.cu) against the host one, on the seeded synthetic
dataset tools/time_coco_eval.py builds.

  (a) the kernels alone: every ground-truth polygon and every detection string of the first `--images` images in one
      launch each, CUDA events around `--launches` launches queued behind a device sleep (so the host's enqueue is not in
      the window), median of 5; with the bytes the algorithm must move (the scratch bitmap zeroed, then read once; the
      planes zeroed; toggles and set words on top are not counted) over the time;
  (b) the host rasterizer (cocoeval.segm_plane + plane_stats) over the same items.
Needs a GPU; prints the card's name, power limit and maximum SM clock with the numbers, as one JSON line.

    python tools/time_segm_raster.py --images 256
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))


def items_of(gt, segm, n_img):
    """(ground-truth polygon segmentations, detection RLE segmentations, h, w) of the first n_img images, on one canvas
    (the largest; the kernels take a canvas per item, one canvas keeps the host comparison simple)."""
    ids = set(im['id'] for im in gt['images'][:n_img])
    hw = {im['id']: (im['height'], im['width']) for im in gt['images']}
    polys = [(a['segmentation'], hw[a['image_id']]) for a in gt['annotations'] if a['image_id'] in ids]
    runs = [(r['segmentation'], hw[r['image_id']]) for r in segm if r['image_id'] in ids]
    return polys, runs


def algorithmic_bytes(canvases, pitch_words, stride_words):
    """Bytes one launch must move: each item's scratch bitmap written (zeroed) and read once, each plane written once."""
    scratch = sum((h * w + 31) // 32 * 4 for h, w in canvases)
    return 2 * scratch + len(canvases) * stride_words * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=256)
    ap.add_argument('--launches', type=int, default=50)
    a = ap.parse_args()
    from time_coco_eval import dataset
    gt, _, segm = dataset(a.images)
    polys, runs = items_of(gt, segm, a.images)
    out = dict(images=a.images, polygons=len(polys), strings=len(runs))

    import torch
    if not torch.cuda.is_available():
        raise SystemExit('time_segm_raster: no GPU (the host rasterizer alone is not what this tool measures)')
    from sipmask_b200 import cocoeval as C, segm_raster as SR
    out['gpu'] = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                         text=True).strip().splitlines()[0]
    dev = torch.device('cuda', 0)
    for name, segs in (('polygons', polys), ('strings', runs)):
        pack = SR.SegmPack()
        for p, (s, (h, w)) in enumerate(segs):
            pack.add(s, h, w, p)
        n = len(segs)
        pitch = max((w + 31) // 32 for _, (h, w) in segs)
        stride = max(h for _, (h, w) in segs) * pitch
        st, _ = SR.staged(pack, dev)
        planes = torch.empty(n * stride, dtype=torch.int32, device=dev)
        stats = torch.zeros((n, 5), dtype=torch.int32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)

        def launch():
            SR.raster(st, planes, n, stride, pitch, status, area=stats, area_stride=5, ext=stats[:, 1:], ext_stride=5)
        launch()
        torch.cuda.synchronize()
        SR.check_status(status)
        times = []
        for _ in range(5):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda._sleep(20_000_000)
            e0.record()
            for _ in range(a.launches):
                launch()
            e1.record()
            torch.cuda.synchronize()
            times.append(e0.elapsed_time(e1) / a.launches)
        ms = statistics.median(times)
        # which stage bounds it: per-kernel device time of 5 more launches, from a profiled run of its own
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(5):
                launch()
            torch.cuda.synchronize()
        stages = {}
        for e in prof.key_averages():
            stage = [v for k, v in (('segm_toggle', 'toggle'), ('segm_fill', 'fill'), ('segm_stats', 'stats'),
                                    ('emset', 'memset')) if k in e.key]
            if stage:
                t = getattr(e, 'device_time_total', None) or getattr(e, 'cuda_time_total', 0)
                stages[stage[0]] = round(stages.get(stage[0], 0) + t / 5e3, 4)
        nbytes = algorithmic_bytes([hw for _, hw in segs], pitch, stride)
        # the host rasterizer over the same items, and the planes equal
        t0 = time.perf_counter()
        host_area = []
        for s, (h, w) in segs:
            host_area.append(C.plane_stats(C.segm_plane(s, h, w), w)[0])
        host_s = time.perf_counter() - t0
        assert stats[:, 0].cpu().tolist() == host_area
        out[name] = dict(items=n, device_ms_per_launch=round(ms, 4), spread_ms=[round(min(times), 4), round(max(times), 4)],
                         algorithmic_MB=round(nbytes / 1e6, 2), GB_per_s=round(nbytes / ms / 1e6, 1),
                         share_of_3350_GB_per_s=round(nbytes / ms / 1e6 / 3350, 3), host_ms=round(host_s * 1e3, 1),
                         us_per_item_device=round(ms * 1e3 / n, 3), us_per_item_host=round(host_s * 1e6 / n, 1),
                         stage_ms=stages)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
