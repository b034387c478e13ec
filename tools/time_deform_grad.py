"""Time the DeformConv backward kernels with CUDA events, beside the reference's own path.

    python tools/time_deform_grad.py [--iters N] [--out FILE.json]

Cases: FeatureAlign (batch 2, C = Cout = 256, dg = 4) at the five pyramid levels of an 800x1344 image, and the SipMask++
DCN layers (batch 2, dg = 1: C = 128 at 68x68, 256 at 34x34, 512 at 17x17, the stage sizes of a 544x544 image).
Per case and kernel: mean milliseconds per call; TFLOP/s for the two GEMMs (2 * P * Cout * 9C each); GB/s for col2im, counting
the bytes it must move at least (grad_col read once, x read once, grad_offset and grad_input written once).
The reference path, timed the same way: oracle/_ref's deformable_col2im, deformable_col2im_coord
(libsipmask_ref_train_cuda.so) and deformable_im2col (libsipmask_ref_cuda.so) kernels (MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu, fp32), and torch.mm in fp32 for its two addmm_ calls
(deform_conv_cuda.cpp:333-338, 446-451).  The GPU name and power limit are printed beside the numbers.
"""
import argparse
import ctypes
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from sipmask_b200 import conv  # noqa: E402
from sipmask_b200 import ops  # noqa: E402

CASES = [('feature_align_p%d' % (3 + i), 2, 256, 256, h, w, 4)
         for i, (h, w) in enumerate([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)])] + \
        [('pp_dcn_c128', 2, 128, 128, 68, 68, 1), ('pp_dcn_c256', 2, 256, 256, 34, 34, 1),
         ('pp_dcn_c512', 2, 512, 512, 17, 17, 1)]


def timed(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def gpu_info():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        q = 'nvidia-smi unavailable (%s)' % e
    return {'torch_name': torch.cuda.get_device_name(0), 'nvidia_smi': q}


def run_case(name, B, C, Cout, H, W, dg, iters, ref):
    g = torch.Generator(device='cuda').manual_seed(0)
    x = torch.randn(B, C, H, W, device='cuda', generator=g)
    off = torch.randn(B, dg * 18, H, W, device='cuda', generator=g) * 2.0
    w = torch.randn(Cout, C, 3, 3, device='cuda', generator=g) / 48.0
    gy = torch.randn(B, Cout, H, W, device='cuda', generator=g) * 1e-3
    P, K = B * H * W, 9 * C
    xh, offl = ops._channels_last(x, off)
    g16, scale = conv.deform_grad_scale(gy)
    wt = conv.pack_weight(w)[0].t().contiguous()
    gcol = torch.empty((B, H, W, K), dtype=torch.float32, device='cuda')
    plan = conv.ConvPlan(g16, wt, gcol, 1, 1)
    col = conv.deform_im2col(xh, offl, dg)
    gemm_flop = 2.0 * P * Cout * K
    col2im_bytes = 4 * P * K + 2 * P * C + 4 * P * dg * 18 + 4 * P * C
    r = {'case': name, 'shape': [B, C, Cout, H, W, dg]}
    r['grad_scale_ms'] = timed(lambda: conv.deform_grad_scale(gy), iters)
    r['grad_col_gemm_ms'] = timed(plan.run, iters)
    r['col2im_ms'] = timed(lambda: conv.deform_col2im(gcol, xh, offl, dg, scale), iters)
    r['im2col_ms'] = timed(lambda: conv.deform_im2col(xh, offl, dg, out=col), iters)
    r['weight_grad_ms'] = timed(lambda: conv.deform_weight_grad(g16, col, scale), iters)
    r['grad_col_gemm_tflops'] = gemm_flop / r['grad_col_gemm_ms'] * 1e-9
    r['weight_grad_tflops'] = gemm_flop / r['weight_grad_ms'] * 1e-9
    r['col2im_gbps'] = col2im_bytes / r['col2im_ms'] * 1e-6
    r['smb_backward_ms'] = sum(r[k] for k in ('grad_scale_ms', 'grad_col_gemm_ms', 'col2im_ms', 'im2col_ms',
                                              'weight_grad_ms'))
    if ref is not None:
        train, fwd = ref                                 # col2im / col2im_coord; im2col
        p = lambda t: ctypes.c_void_p(t.data_ptr())     # noqa: E731
        colr = torch.randn(K, B, H, W, device='cuda', generator=g)
        gin, goff = torch.zeros_like(x), torch.zeros_like(off)
        r['ref_col2im_ms'] = timed(lambda: train.ref_deformable_col2im(p(colr), p(off), C, H, W, 3, 1, 1, 1, B, dg, p(gin)),
                                   iters)
        r['ref_col2im_coord_ms'] = timed(lambda: train.ref_deformable_col2im_coord(p(colr), p(x), p(off), C, H, W, 3, 1, 1, 1,
                                                                                  B, dg, p(goff)), iters)
        r['ref_im2col_ms'] = timed(lambda: fwd.ref_deformable_im2col(p(x), p(off), C, H, W, 3, 1, 1, 1, B, dg, p(colr)),
                                   iters)
        w2, g2 = w.view(Cout, K), gy.permute(1, 0, 2, 3).reshape(Cout, P).contiguous()
        r['ref_grad_col_mm_ms'] = timed(lambda: torch.mm(w2.t(), g2), iters)
        cr = colr.view(K, P)
        r['ref_weight_mm_ms'] = timed(lambda: torch.mm(g2, cr.t()), iters)
        r['ref_backward_ms'] = sum(r[k] for k in ('ref_col2im_ms', 'ref_col2im_coord_ms', 'ref_im2col_ms',
                                                  'ref_grad_col_mm_ms', 'ref_weight_mm_ms'))
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'time_deform_grad.py needs a GPU'
    torch.backends.cuda.matmul.allow_tf32 = False
    sos = [os.path.join(ROOT, 'oracle', '_ref', n) for n in ('libsipmask_ref_train_cuda.so', 'libsipmask_ref_cuda.so')]
    ref = tuple(ctypes.CDLL(so) for so in sos) if all(os.path.exists(so) for so in sos) else None
    res = {'gpu': gpu_info(), 'cases': [run_case(*c, iters=a.iters, ref=ref) for c in CASES]}
    if ref is None:
        res['reference'] = 'not measured: oracle/_ref/libsipmask_ref_train_cuda.so or libsipmask_ref_cuda.so not built'
    s = json.dumps(res, indent=1)
    print(s)
    if a.out:
        with open(a.out, 'w') as f:
            f.write(s)


if __name__ == '__main__':
    main()
