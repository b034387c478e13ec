"""Generate tests/golden/ref_train_ops.npz: what the reference's own CUDA kernels compute on the inputs of
tests/train_ops_inputs.py.

Needs a GPU and oracle/_ref/libsipmask_ref_train_cuda.so (built by oracle/build_train.py from the reference sources).
    python tests/golden/gen_golden_ref_train_ops.py OUT_DIR

Arrays of an existing OUT_DIR/ref_train_ops.npz are kept (see main), so adding cases leaves the other keys' bits alone.

  * `deformable_col2im` / `deformable_col2im_coord` (MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:279-465) on each
    COL2IM_CASES input: grad_input [B,C,H,W] and grad_offset [B,dg*18,H,W] as the fp32 values at a fixed, seeded sample of
    flat indices (`train_ops_inputs.sample_index`), as in ref_cuda_kernels.npz;
  * `SigmoidFocalLossForward` / `Backward` (MM/mmdet/ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-100) on
    each FOCAL_CASES input: the whole loss and gradient, fp32.
"""
import ctypes
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))

import train_ops_inputs as T  # noqa: E402

REF_SO = os.path.join(ROOT, 'oracle', '_ref', 'libsipmask_ref_train_cuda.so')


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def ref_col2im(lib, x, off, gcol, dg):
    B, C, H, W = x.shape
    gin = torch.zeros_like(x)
    goff = torch.zeros_like(off)
    torch.cuda.synchronize()
    assert lib.ref_deformable_col2im(_p(gcol), _p(off), C, H, W, 3, 1, 1, 1, B, dg, _p(gin)) == 0
    assert lib.ref_deformable_col2im_coord(_p(gcol), _p(x), _p(off), C, H, W, 3, 1, 1, 1, B, dg, _p(goff)) == 0
    torch.cuda.synchronize()
    return gin, goff


def ref_focal(lib, logits, targets, d_loss, gamma, alpha):
    N, C = logits.shape
    loss = torch.zeros_like(logits)
    grad = torch.zeros_like(logits)
    torch.cuda.synchronize()
    g, a = ctypes.c_float(gamma), ctypes.c_float(alpha)
    assert lib.ref_sigmoid_focal_loss_forward(_p(logits), _p(targets), N, C, g, a, _p(loss)) == 0
    assert lib.ref_sigmoid_focal_loss_backward(_p(logits), _p(targets), _p(d_loss), N, C, g, a, _p(grad)) == 0
    return loss, grad


def main(out_dir):
    lib = ctypes.CDLL(REF_SO)
    os.makedirs(out_dir, exist_ok=True)
    g = {}
    for B, C, H, W, dg in T.COL2IM_CASES:
        x, off, gcol = [t.cuda() for t in T.col2im_inputs(B, C, H, W, dg)]
        gin, goff = ref_col2im(lib, x, off, gcol, dg)
        key = '%d_%d_%d_%d_%d' % (B, C, H, W, dg)
        g['col2im_input_' + key] = gin.cpu().numpy().ravel()[T.sample_index(gin.numel(), 1)]
        g['col2im_offset_' + key] = goff.cpu().numpy().ravel()[T.sample_index(goff.numel(), 2)]
    for C, gamma, alpha in T.FOCAL_CASES:
        logits, targets, d_loss = [t.cuda() for t in T.focal_inputs(C)]
        loss, grad = ref_focal(lib, logits, targets, d_loss, gamma, alpha)
        g[T.focal_key(C, gamma, alpha) + '_loss'] = loss.cpu().numpy()
        g[T.focal_key(C, gamma, alpha) + '_grad'] = grad.cpu().numpy()
    path = os.path.join(out_dir, 'ref_train_ops.npz')
    if os.path.exists(path):
        # deformable_col2im sums grad_input with float atomics, so a second run reproduces it only to rounding: arrays
        # already in the file keep their bits (after checking they agree), and added cases only add keys
        old = np.load(path)
        for k in old.files:
            if k in g:
                tol = 1e-6 * float(np.abs(g[k]).max()) if k.startswith('col2im_input_') else 0.0
                assert old[k].shape == g[k].shape and np.abs(old[k].astype(np.float64) - g[k]).max() <= tol, k
                g[k] = old[k]
        print('kept %d existing arrays' % len([k for k in old.files if k in g]))
    np.savez_compressed(path, **g)
    print('wrote %s (%d arrays)' % (path, len(g)))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
