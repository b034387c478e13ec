"""Generate tests/golden/ref_cuda_kernels.npz: what the reference's own CUDA kernels compute on the inputs of
tests/test_gpu_ref_cuda.py.

Needs a GPU and oracle/_ref/libsipmask_ref_cuda.so (built by oracle/build.py::build_ref_cuda from the reference sources).
    python tests/golden/gen_golden_ref_cuda.py OUT_DIR

The kernels are `CropSplitKernelForward` / backward (MM/mmdet/ops/crop/src/crop_split_cuda_kernel.cu:19-163),
CropSplitGt forward / backward (crop_split_gt_cuda_kernel.cu:19-140) and `deformable_im2col_gpu_kernel`
(MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:84-277).  Their outputs are stored compactly:
  * every CropSplit output element is either 0 or a copy of one input element, so the file stores, per output element,
    WHICH input it copies (0 = none, k + 1 = cell k), checked here to rebuild the reference output bit for bit;
  * im2col columns and the DeformConv GEMM are stored as the fp32 values at a fixed, seeded sample of flat indices
    (`test_gpu_ref_cuda.sample_index`).
Selector codes are stored detection-major, [N, H, W]: long runs, so they compress well.
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

import test_gpu_ref_cuda as T  # noqa: E402

REF_SO = os.path.join(ROOT, 'oracle', '_ref', 'libsipmask_ref_cuda.so')


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


def ref_crop_split(lib, data, rois):
    _, H, W, N = data.shape
    out = torch.zeros((H, W, N), dtype=torch.float32, device=data.device)
    torch.cuda.synchronize()
    assert lib.ref_crop_split_forward(_p(data), _p(rois), _p(out), H, W, 2, N) == 0
    torch.cuda.synchronize()
    return out


def ref_deform_im2col(lib, x, offset, dg, k=3, pad=1, stride=1, dil=1):
    B, C, H, W = x.shape
    Ho = (H + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    Wo = (W + 2 * pad - (dil * (k - 1) + 1)) // stride + 1
    col = torch.zeros((C * k * k, B, Ho, Wo), dtype=torch.float32, device=x.device)
    torch.cuda.synchronize()
    assert lib.ref_deformable_im2col(_p(x), _p(offset), C, H, W, k, pad, stride, dil, B, dg, _p(col)) == 0
    torch.cuda.synchronize()
    return col


def _nhw(code):
    return code.permute(2, 0, 1).contiguous().numpy()


def main(out_dir):
    lib = ctypes.CDLL(REF_SO)
    os.makedirs(out_dir, exist_ok=True)
    g = {}
    for H, W, N in T.CROP_CASES:
        data, rois = T.crop_inputs(H, W, N)
        ref = ref_crop_split(lib, data.cuda(), rois.cuda()).cpu()
        code = T.selector_code(ref, data)
        assert torch.equal(T.from_code(code, data), ref)
        g['crop_%d_%d_%d' % (H, W, N)] = _nhw(code)
    for H, W, N, sf in T.ASSEMBLY_CASES:
        protos, cofs, boxes = T.assembly_inputs(H, W, N, sf)
        maps = T.assembly_maps(protos.cuda(), cofs.cuda())
        rois = (boxes * (sf / 2.0)).contiguous()
        ref = ref_crop_split(lib, maps, rois.cuda()).cpu()
        code = T.selector_code(ref, maps.cpu())
        assert torch.equal(T.from_code(code, maps.cpu()), ref)
        g['assembly_%d_%d_%d' % (H, W, N)] = _nhw(code)
    for B, C, H, W, dg in T.IM2COL_CASES:
        x, off = T.im2col_inputs(B, C, H, W, dg)
        ref = ref_deform_im2col(lib, x.cuda(), off.cuda(), dg)
        ref_bkhw = ref.permute(1, 0, 2, 3).reshape(B, C * 9, H * W).cpu().contiguous().view(-1)
        idx = T.sample_index(ref_bkhw.numel(), B * C + H)
        g['im2col_%d_%d_%d_%d_%d' % (B, C, H, W, dg)] = ref_bkhw.numpy()[idx]
    x, off, w = T.deform_conv_inputs()
    B, C, H, W, dg, Cout = T.DEFORM_CONV_SHAPE
    col = ref_deform_im2col(lib, x.cuda(), off.cuda(), dg)
    want = (w.cuda().view(Cout, -1).double() @ col.view(C * 9, -1).double()).view(Cout, B, H, W).permute(1, 0, 2, 3)
    want = want.contiguous().view(-1).cpu()
    g['deform_conv'] = want.numpy()[T.sample_index(want.numel(), 5)].astype(np.float32)
    for H, W, N in T.BACKWARD_CASES:
        rois, top, d = T.backward_inputs(H, W, N)
        rc, tc, dc = rois.cuda(), top.cuda(), d.cuda()
        grad = torch.zeros((4, H, W, N), dtype=torch.float32, device='cuda')
        gt_f = torch.zeros_like(dc)
        gt_b = torch.zeros_like(dc)
        torch.cuda.synchronize()
        assert lib.ref_crop_split_backward(_p(tc), _p(rc), _p(grad), H, W, 2, N) == 0
        assert lib.ref_crop_split_gt_forward(_p(dc), _p(rc), _p(gt_f), H, W, 2, N) == 0
        assert lib.ref_crop_split_gt_backward(_p(tc), _p(rc), _p(gt_b), H, W, 2, N) == 0
        torch.cuda.synchronize()
        grad, gt_f, gt_b = grad.cpu(), gt_f.cpu(), gt_b.cpu()
        # backward scatters top[y, x, n] into cell k of the gradient: the cell index is the selector
        code = T.selector_code(grad.sum(0), top, grad)
        assert torch.equal(T.scatter_from_code(code, top), grad)
        g['backward_%d_%d_%d' % (H, W, N)] = _nhw(code)
        for name, t, src in (('gt_forward', gt_f, d), ('gt_backward', gt_b, top)):
            c = T.selector_code(t, src[None])
            assert torch.equal(T.from_code(c, src[None]), t)
            g['%s_%d_%d_%d' % (name, H, W, N)] = _nhw(c)
    path = os.path.join(out_dir, 'ref_cuda_kernels.npz')
    np.savez_compressed(path, **g)
    print(path, os.path.getsize(path))


if __name__ == '__main__':
    main(sys.argv[1] if len(sys.argv) > 1 else HERE)
