"""Time SipMask's fused mask loss (forward + backward) against the composition it replaces, with CUDA events.

    python tools/time_mask_loss.py [--window SECONDS] [--rounds N] [--out FILE.json]

The composition (SipMaskHead.loss, sipmask_head.py:446-463): fp32 matmuls with TF32 off, sigmoid, ops.crop_split /
crop_split_gt (bit for bit the reference's CropSplit kernels), F.binary_cross_entropy and the per-instance
normalisation, per image, then backward.  Both run on the same seeded inputs (tests/mask_loss_inputs.py: FCOS-like
clusters of jittered boxes around COCO-sized objects), alternating, one measured call each per round.
Each timed window runs enough calls to last at least --window seconds (0.5 by default); the best of --rounds windows
per path is reported.  A separate torch.profiler pass (3 fused forward+backward calls) gives each kernel's time per call,
and from the work each kernel must do (FLOP from the in-box pairs, minimal HBM bytes from the shapes) its share of the
card's fp32 rate (67 TFLOP/s) and HBM bandwidth (3.35 TB/s, data sheet), and so what bounds it: "latency" when
neither share reaches 30 %.
Cases: the mask maps of MM 1333x800 (400x672, 4 images), SSD 576 (288x288, 4 images) and VIS (180x320, 4 images), each
with 100, 300 and 1000 positives per image.  Per case: mean ms per forward+backward, max_memory_allocated above the
inputs, the in-box (pixel, instance) pairs, the useful FLOP rate (~200 FLOP per pair: three 32-term dot products,
sigmoid, BCE) and the fused path's byte rate (feat read twice, d feat written once, cofs / targets / d cofs).  The
composition is skipped, and said so, where its estimated activations would not fit in the card's memory.
The GPU name and power limit are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'tests'))

from sipmask_b200 import ops  # noqa: E402
import mask_loss_inputs as MI  # noqa: E402

CASES = [(name, 4, H, W, m) for name, H, W in [('mm_1333x800', 400, 672), ('ssd_576', 288, 288), ('vis', 180, 320)]
         for m in (100, 300, 1000)]


class _Crop(torch.autograd.Function):
    @staticmethod
    def forward(ctx, data, rois):
        ctx.save_for_backward(rois)
        return ops.crop_split(data, rois)

    @staticmethod
    def backward(ctx, g):
        (rois,) = ctx.saved_tensors
        return ops.crop_split_backward(g.contiguous(), rois), None


def _card():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                                       text=True).strip()
    except Exception as e:                      # noqa: BLE001
        return 'unknown (%s)' % e


def _pairs(d):
    """in-box (pixel, instance) pairs: integer pixels with x1 <= w < x2, y1 <= h < y2 inside the map"""
    _, _, H, W = d['feat'].shape
    b = d['boxes'].double()
    nx = (torch.ceil(b[:, 2]).clamp(max=W) - torch.ceil(b[:, 0]).clamp(min=0)).clamp(min=0)
    ny = (torch.ceil(b[:, 3]).clamp(max=H) - torch.ceil(b[:, 1]).clamp(min=0)).clamp(min=0)
    return int((nx * ny).sum().item())


def _fused_step(d):
    feat = d['feat'].requires_grad_(True)
    cofs = d['cofs'].requires_grad_(True)
    loss = ops.sipmask_mask_loss(feat, cofs, d['boxes'], d['offsets'], d['bits'], d['rows'], d['weights'])
    loss.sum().backward()
    feat.grad = cofs.grad = None


def _composed_step(d):
    feat = d['feat'].requires_grad_(True)
    cofs = d['cofs'].requires_grad_(True)
    loss = MI.composition(d, feat, cofs, _Crop.apply, ops.crop_split_gt)
    loss.sum().backward()
    feat.grad = cofs.grad = None


def _calls_for(fn, d, window):
    """calls per timed window so that it lasts at least `window` seconds"""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn(d)
    e1.record()
    torch.cuda.synchronize()
    return max(3, int(window * 1e3 / max(e0.elapsed_time(e1), 1e-3)) + 1)


# per kernel: (FLOP per in-box pair, minimal HBM bytes as a function of (feat bytes, M, bits bytes))
KERNELS = {
    'mask_loss_pixel_kernel<false>': (70, lambda fb, M, bb: fb + M * 128 * 4 + bb),
    'mask_loss_pixel_kernel<true>': (130, lambda fb, M, bb: 2 * fb + M * 128 * 4 + bb),
    'mask_loss_inst_kernel': (130, lambda fb, M, bb: fb + M * 128 * 4 * 9 + bb),
    'mask_loss_cof_reduce_kernel': (0, lambda fb, M, bb: M * 128 * 4 * 9),
    'mask_loss_sum_kernel': (0, lambda fb, M, bb: 0),
}


def _kernel_split(d, pairs):
    from torch.profiler import ProfilerActivity, profile
    n = 3
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(n):
            _fused_step(d)
        torch.cuda.synchronize()
    fb = d['feat'].numel() * 4
    M, bb = d['cofs'].shape[0], d['bits'].numel() * 4
    out = {}
    for ev in prof.key_averages():
        name = next((k for k in KERNELS if k in ev.key), None)
        if name is None:
            continue
        t = getattr(ev, 'device_time_total', None) or getattr(ev, 'cuda_time_total', 0)
        ms = t / 1e3 / n
        flop, nbytes = KERNELS[name][0] * pairs, KERNELS[name][1](fb, M, bb)
        fr, br = flop / (ms * 1e-3) / 67e12 if ms else 0, nbytes / (ms * 1e-3) / 3.35e12 if ms else 0
        bound = 'fp32' if fr >= 0.3 and fr >= br else 'HBM' if br >= 0.3 else 'latency'
        out[name] = dict(ms=ms, fp32_share=fr, hbm_share=br, bound=bound)
    return out


def _time(fn, d, iters):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn(d)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters, torch.cuda.max_memory_allocated() - base


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--window', type=float, default=0.5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    torch.backends.cuda.matmul.allow_tf32 = False
    card = _card()
    free = torch.cuda.mem_get_info()[0]
    print('card: %s' % card)
    rows = []
    for name, B, H, W, m in CASES:
        inp = MI.clustered_inputs(B, H, W, m, seed=H + m, grid=False, zmax=12.0)
        d = MI.to_device(inp)
        pairs = _pairs(d)
        M = B * m
        # the composition keeps ~10 [H, W, M_b] fp32 tensors per image alive until backward
        est = 10 * 4 * H * W * M
        run_comp = est < 0.8 * free
        _fused_step(d)                                         # warm-up
        if run_comp:
            try:
                _composed_step(d)
            except torch.cuda.OutOfMemoryError:
                run_comp, est = False, float('nan')
                torch.cuda.empty_cache()
        f_calls = _calls_for(_fused_step, d, a.window)
        c_calls = _calls_for(_composed_step, d, a.window) if run_comp else 0
        f_ms, c_ms, f_mem, c_mem = [], [], 0, 0
        for _ in range(a.rounds):
            t, mem = _time(_fused_step, d, f_calls)
            f_ms.append(t)
            f_mem = max(f_mem, mem)
            if run_comp:
                try:
                    t, mem = _time(_composed_step, d, c_calls)
                except torch.cuda.OutOfMemoryError:
                    run_comp, est = False, float('nan')
                    torch.cuda.empty_cache()
                    continue
                c_ms.append(t)
                c_mem = max(c_mem, mem)
        fms = min(f_ms)
        nbytes = 2 * d['feat'].numel() * 4 + d['feat'].numel() * 4 + M * 128 * 4 * (2 + 8 + 8) + d['bits'].numel() * 4
        r = dict(case=name, B=B, H=H, W=W, per_img=m, pairs=pairs, fused_ms=fms, fused_ms_all=f_ms, fused_peak_mb=f_mem / 2**20,
                 fused_gflops=200.0 * pairs / fms / 1e6, fused_gbs=nbytes / fms / 1e6,
                 composed_ms=min(c_ms) if run_comp else None, composed_peak_mb=c_mem / 2**20 if run_comp else None,
                 composed_skipped=None if run_comp else 'out of memory (estimated %.1f GB of activations, %.1f GB free)' % (est / 1e9, free / 1e9))
        r['fused_calls_per_window'], r['composed_calls_per_window'] = f_calls, c_calls
        r['kernels'] = _kernel_split(d, pairs)
        rows.append(r)
        print('%-12s M/img=%4d pairs=%9d  fused %8.3f ms %8.1f MB (%6.1f GFLOP/s, %6.1f GB/s)  composed %s' % (
            name, m, pairs, fms, f_mem / 2**20, r['fused_gflops'], r['fused_gbs'],
            ('%8.3f ms %8.1f MB' % (r['composed_ms'], r['composed_peak_mb'])) if run_comp else 'skipped: ' + r['composed_skipped']))
        for k, v in r['kernels'].items():
            print('    %-32s %8.3f ms  fp32 %5.1f %%  HBM %5.1f %%  -> %s' % (k, v['ms'], 100 * v['fp32_share'],
                                                                          100 * v['hbm_share'], v['bound']))
        del d
        torch.cuda.empty_cache()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        json.dump(dict(card=card, rows=rows), open(a.out, 'w'), indent=1)


if __name__ == '__main__':
    main()
