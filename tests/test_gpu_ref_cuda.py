"""Pins for the two CUDA-only reference operators, against what the reference's OWN kernels compute.

`CropSplitKernelForward` / backward (MM/mmdet/ops/crop/src/crop_split_cuda_kernel.cu:19-163), CropSplitGt
(crop_split_gt_cuda_kernel.cu:19-140) and `deformable_im2col_gpu_kernel` (MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:84-277)
were run on the seeded inputs below by tests/golden/gen_golden_ref_cuda.py; their outputs are stored in
tests/golden/ref_cuda_kernels.npz (CropSplit outputs exactly, as "which input element each output copies"; im2col columns
and the DeformConv GEMM as a fixed, seeded sample of elements).  Each test compares three things on the same inputs:
    reference kernel  ==  oracle restatement (oracle/ops.py)  ==  smb kernel through the C ABI
which removes the circularity of tests/golden/gen_golden.py (there the reference python's two native calls are bound to
the oracle, because neither has a CPU build).
"""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_cuda_kernels.npz')

CROP_CASES = [(40, 56, 16), (100, 168, 37), (272, 272, 100)]
ASSEMBLY_CASES = [(100, 168, 40, 1.0), (136, 136, 100, 1.0), (75, 125, 33, 1.6666)]
IM2COL_CASES = [(1, 256, 13, 21, 4), (2, 256, 25, 42, 4), (1, 128, 17, 17, 1), (1, 64, 7, 11, 1)]
DEFORM_CONV_SHAPE = (1, 256, 25, 42, 4, 256)
BACKWARD_CASES = [(40, 56, 16), (100, 168, 37)]
SAMPLE = 4096                     # sampled elements per im2col / DeformConv case


def _golden():
    return np.load(GOLDEN)


def _code(gold, key):
    """selector codes are stored detection-major [N,H,W] (long runs: compact); the outputs are [H,W,N]"""
    return np.ascontiguousarray(gold[key].transpose(1, 2, 0))


def _rois(N, H, W, g):
    cx, cy = torch.rand(N, generator=g) * W, torch.rand(N, generator=g) * H
    bw, bh = torch.rand(N, generator=g) * W * 0.8 + 0.3, torch.rand(N, generator=g) * H * 0.8 + 0.3
    r = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1)
    fixed = torch.tensor([[0, 0, W, H], [-5, -7, W + 9, H + 3], [3.2, 4.1, 30.7, 35.2], [10, 10, 10.5, 10.5],
                          [0.5, 0.5, 1.5, 1.5], [20, 20, 19, 19], [W - 1, H - 1, W, H], [7, 3, 8, H - 1],
                          [4, 4, 12, 12], [4.0, 4.0, 11.9, 11.9]], dtype=torch.float32)
    r[:fixed.shape[0]] = fixed[:N]
    return r.contiguous()


# ---- seeded inputs (shared with tests/golden/gen_golden_ref_cuda.py)
def crop_inputs(H, W, N):
    g = torch.Generator().manual_seed(H * 7 + N)
    data = torch.rand(4, H, W, N, generator=g) + 0.01            # strictly positive: zeros mark "outside the box"
    return data, _rois(N, H, W, g)


def assembly_inputs(H, W, N, sf=1.0):
    from sipmask_b200 import synth
    g = torch.Generator().manual_seed(N)
    protos = synth.prototypes(H, W, seed=N)                       # [32,H,W]
    cofs = torch.randn(N, 128, generator=g)
    boxes = _rois(N, H, W, g) * 2.0 / sf                          # image space; rois = boxes * sf / 2
    return protos, cofs, boxes


def assembly_maps(protos, cofs):
    """sipmask_head.py:615-620: 4x sigmoid(P @ cof_k^T) -> [4,H,W,N] (fp32, on the device of the inputs)."""
    P = protos.permute(1, 2, 0).contiguous()
    return torch.stack([torch.sigmoid(P @ cofs[:, 32 * k:32 * k + 32].t()) for k in range(4)], 0).contiguous()


def im2col_inputs(B, C, H, W, dg):
    g = torch.Generator().manual_seed(C + H)
    x = torch.randn(B, C, H, W, generator=g).half().float()       # fp16-representable so the smb (fp16 storage) path reads the same values
    off = torch.randn(B, dg * 18, H, W, generator=g) * 2.5
    off[:, :, 0, 0] = 0.0                                         # integer sampling points (bilinear weights exactly 0 / 1)
    off[:, :, -1, -1] = torch.round(off[:, :, -1, -1])
    off[:, 0::2, 1, :] = -3.7                                     # rows far outside the map (the `h_im > -1` predicate)
    return x, off


def deform_conv_inputs():
    B, C, H, W, dg, Cout = DEFORM_CONV_SHAPE
    g = torch.Generator().manual_seed(5)
    x = torch.randn(B, C, H, W, generator=g).half().float()
    off = torch.randn(B, dg * 18, H, W, generator=g) * 2.0
    w = (torch.randn(Cout, C, 3, 3, generator=g) / 48.0).half().float()
    return x, off, w


def backward_inputs(H, W, N):
    g = torch.Generator().manual_seed(H + N)
    rois = _rois(N, H, W, g)
    top = torch.rand(H, W, N, generator=g) + 0.01
    torch.rand(4, H, W, N, generator=g)                           # (the forward input of the autograd check: values unused)
    d = torch.rand(H, W, N, generator=g) + 0.01
    return rois, top, d


# ---- compact forms of the reference outputs
def selector_code(out, src, scattered=None):
    """CropSplit-style outputs copy input elements: code = 0 where the output is 0, else k + 1 for the source plane k
    (out == src[k] elementwise).  With `scattered` [K,...] (a backward pass), k is the plane that received the value."""
    code = torch.zeros(out.shape, dtype=torch.uint8)
    planes = scattered if scattered is not None else src
    for k in range(planes.shape[0]):
        hit = (planes[k] != 0) if scattered is not None else (out == src[k]) & (out != 0)
        code[(code == 0) & hit] = k + 1
    return code


def from_code(code, src):
    """inverse of selector_code for a gather: out = src[code - 1] where code > 0, else 0."""
    code = torch.as_tensor(np.asarray(code)).long().to(src.device)
    idx = (code - 1).clamp(min=0).unsqueeze(0)
    return torch.where(code > 0, torch.gather(src, 0, idx).squeeze(0), torch.zeros((), dtype=src.dtype, device=src.device))


def scatter_from_code(code, top):
    """inverse of selector_code for a scatter: plane k holds top where code == k + 1."""
    code = torch.as_tensor(np.asarray(code)).to(top.device)
    return torch.stack([torch.where(code == k + 1, top, torch.zeros((), dtype=top.dtype, device=top.device)) for k in range(4)], 0)


def sample_index(n, seed):
    """the fixed sample of flat output indices whose reference values are stored"""
    return np.sort(np.random.RandomState(seed).choice(n, size=min(SAMPLE, n), replace=False)).astype(np.int64)


@pytest.mark.parametrize('H,W,N', CROP_CASES)
def test_crop_split_reference_kernel_vs_oracle_vs_smb(H, W, N):
    from oracle import ops as O
    from sipmask_b200 import ops
    data, rois = crop_inputs(H, W, N)
    ref = from_code(_code(_golden(), 'crop_%d_%d_%d' % (H, W, N)), data).numpy()
    orc = O.crop_split(data, rois, 2).numpy()
    np.testing.assert_array_equal(orc, ref)                       # the restatement IS the reference kernel, bit for bit
    got = ops.crop_split(data.cuda(), rois.cuda()).cpu().numpy()
    np.testing.assert_array_equal(got, ref)                       # and so is the drop-in operator


@pytest.mark.parametrize('H,W,N,sf', ASSEMBLY_CASES)
def test_mask_assembly_vs_reference_pipeline(H, W, N, sf):
    """sipmask_head.py:615-627 with the reference's own CropSplit kernel:  4x (P @ cof_k^T) -> sigmoid -> stack ->
    CropSplitKernelForward -> permute, all fp32 on the GPU, versus the fused smb_mask_assemble."""
    from sipmask_b200 import ops
    protos, cofs, boxes = assembly_inputs(H, W, N, sf)
    protos, cofs, boxes = protos.cuda(), cofs.cuda(), boxes.cuda()
    maps = assembly_maps(protos, cofs)                            # [4,H,W,N]
    ref = from_code(_code(_golden(), 'assembly_%d_%d_%d' % (H, W, N)), maps).permute(2, 0, 1).contiguous().cpu().numpy()
    got = ops.mask_assemble(protos, cofs, boxes, sf / 2.0, layout='chw').cpu().numpy()
    assert ((got == 0) == (ref == 0)).all()                       # crop + cell geometry identical to the reference kernel
    np.testing.assert_allclose(got, ref, atol=5e-6, rtol=0)       # 32-term fp32 dot + sigmoid: summation order only


@pytest.mark.parametrize('B,C,H,W,dg', IM2COL_CASES)
def test_deformable_im2col_reference_kernel_vs_oracle_vs_smb(B, C, H, W, dg):
    from oracle import ops as O
    from sipmask_b200 import conv
    x, off = im2col_inputs(B, C, H, W, dg)
    idx = sample_index(B * C * 9 * H * W, B * C + H)
    ref = _golden()['im2col_%d_%d_%d_%d_%d' % (B, C, H, W, dg)]
    orc, _, _ = O.deform_im2col(x, off, 3, 3, 1, 1, 1, dg)        # [B, C*9, HW]
    # identical predicates / gather indices; the reference is compiled with FMA contraction, torch CPU is not
    orc_s = orc.reshape(-1).numpy()[idx]
    np.testing.assert_allclose(orc_s, ref, atol=2e-6, rtol=1e-6)
    assert ((orc_s == 0) == (ref == 0)).mean() > 0.9999
    # smb kernel: NHWC fp16 in, [N,H,W,tap*C + c] fp16 out
    x_nhwc = x.permute(0, 2, 3, 1).contiguous().half().cuda()
    off_nhwc = off.permute(0, 2, 3, 1).contiguous().cuda()
    col = conv.deform_im2col(x_nhwc, off_nhwc, dg).float().cpu()  # [B,H,W,9*C]
    col_bkhw = col.view(B, H * W, 9, C).permute(0, 3, 2, 1).reshape(-1)
    err = np.abs(col_bkhw.numpy()[idx] - ref).max()
    assert err <= 2e-3 * (np.abs(ref).max() + 1.0), err           # one fp16 rounding of the output
    want = orc.view(B, C, 9, H * W).permute(0, 3, 2, 1).reshape(B, H, W, 9 * C)
    err = (col - want).abs().max().item()
    assert err <= 2e-3 * (want.abs().max().item() + 1.0), err


def test_deform_conv_operator_vs_reference_im2col_gemm():
    """ops.DeformConv (drop-in for mmdet.ops.DeformConv, dcn/deform_conv.py:192-255) against the reference's
    im2col kernel followed by the weight GEMM (deform_conv_cuda.cpp:231-236), fp32 on the GPU."""
    from oracle import ops as O
    from sipmask_b200 import ops
    B, C, H, W, dg, Cout = DEFORM_CONV_SHAPE
    x, off, w = deform_conv_inputs()
    m = ops.DeformConv(C, Cout, 3, stride=1, padding=1, deformable_groups=dg).cuda()
    with torch.no_grad():
        m.weight.copy_(w)
    got = m(x.cuda(), off.cuda())
    assert got.shape == (B, Cout, H, W) and got.dtype == x.dtype
    want_s = _golden()['deform_conv'].astype(np.float64)
    got_s = got.double().reshape(-1).cpu().numpy()[sample_index(B * Cout * H * W, 5)]
    err = np.abs(got_s - want_s).max()
    assert err <= 4e-3 * (np.abs(want_s).max() + 1.0), err        # fp16 column + fp16 output storage, fp32 accumulate
    col, _, _ = O.deform_im2col(x, off, 3, 3, 1, 1, 1, dg)        # [B, C*9, HW], pinned to the reference kernel above
    want = (w.view(Cout, -1).double() @ col[0].double()).view(1, Cout, H, W)
    err = (got.double().cpu() - want).abs().max().item()
    assert err <= 4e-3 * (want.abs().max().item() + 1.0), err


@pytest.mark.parametrize('H,W,N', BACKWARD_CASES)
def test_crop_split_backward_and_gt_vs_reference_kernels(H, W, N):
    """Training-side companions (SURVEY 8f-4): CropSplit backward and CropSplitGt forward / backward against the reference's
    own kernels (crop_split_cuda_kernel.cu:90-163, crop_split_gt_cuda_kernel.cu:19-140), bit for bit, incl. autograd."""
    from sipmask_b200 import ops
    gold = _golden()
    rois, top, d = backward_inputs(H, W, N)
    want = scatter_from_code(_code(gold, 'backward_%d_%d_%d' % (H, W, N)), top).cuda()
    rois, top, d = rois.cuda(), top.cuda(), d.cuda()
    got = ops.crop_split_backward(top, rois)
    assert torch.equal(got, want)
    data = (torch.rand(4, H, W, N) + 0.01).cuda().requires_grad_(True)
    out = ops.CropSplit(2)(data, rois)
    out.backward(top)
    assert torch.equal(data.grad, want)
    # CropSplitGt
    want_f = from_code(_code(gold, 'gt_forward_%d_%d_%d' % (H, W, N)), d[None])
    assert torch.equal(ops.CropSplitGt(2)(d, rois), want_f)
    want_b = from_code(_code(gold, 'gt_backward_%d_%d_%d' % (H, W, N)), top[None])
    dg = d.clone().requires_grad_(True)
    ops.CropSplitGt(2)(dg, rois).backward(top)
    assert torch.equal(dg.grad, want_b)
