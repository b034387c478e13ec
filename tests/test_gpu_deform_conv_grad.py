"""The DeformConv backward (ops.DeformConvFunction / deform_conv, TrainableDeformConv, DeformConvPack) on sm_90a.

  * kernel level, three ways on the same fp32 grad_col and fp16-representable x: the reference's own
    deformable_col2im / deformable_col2im_coord (MM/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu:279-465, fixture
    tests/golden/ref_train_ops.npz), the float64 autograd of the oracle's im2col restatement, and smb_deform_col2im;
  * module level against the float64 autograd of oracle.ops.deform_conv at the FeatureAlign and SipMask++ DCN sizes;
  * the gradient scaling, determinism, needs_input_grad, a FeatureAlign step, DeformConvPack.
"""
import math
import os

import numpy as np
import pytest
import torch

import train_ops_inputs as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_train_ops.npz')

# Module-level bound on ||g - g64|| / ||g64||.  The tensor cores see each operand rounded to fp16 once: the scaled
# grad_out (both GEMMs) and the recomputed columns (the weight GEMM); x and the weights are fp16-representable here.
# fp16's unit roundoff is 2^-11 = 4.9e-4; the rounding errors are independent with random signs, so the relative error
# of a gradient's norm stays near 2^-11 * sqrt(2) = 7e-4 for two rounded operands.  3e-3 leaves 4x for cancellation in
# the sums (accumulation is fp32 throughout, 2^-24 per addition, negligible beside that).
REL = 3e-3

FEATURE_ALIGN = [(2, 256, 256, h, w, 4) for h, w in [(100, 168), (50, 84), (25, 42), (13, 21), (7, 11), (2, 2)]]
PP_DCN = [(2, 128, 128, 68, 68, 1), (2, 256, 256, 34, 34, 1), (2, 512, 512, 17, 17, 1)]
# shapes the API accepts beyond the models': ragged M and N tiles in both GEMMs, Cin != Cout, dg up to Cin / 8, and maps
# smaller than the kernel (TrainableDeformConv pads them to 3 x 3 and crops the output)
EDGES = [(1, 64, 64, 13, 21, 1), (3, 64, 128, 9, 11, 8), (2, 256, 64, 25, 42, 4), (1, 1024, 64, 7, 9, 128)] + \
    [(1, 256, 256, h, w, 4) for h, w in [(1, 1), (1, 5), (5, 1), (2, 1)]]


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _module_inputs(B, C, Cout, H, W, dg, seed=0):
    g = torch.Generator().manual_seed(seed + C + H)
    x = torch.randn(B, C, H, W, generator=g).half().float()
    # offsets on a 2^-10 grid: every sampling position h + offset is then exact in fp32, so the float64 reference samples
    # the same points (a position within fp32 rounding of an integer would otherwise pick other corners in one of them)
    off = torch.round(torch.randn(B, dg * 18, H, W, generator=g) * 2.0 * 1024) / 1024
    w = (torch.randn(Cout, C, 3, 3, generator=g) / (3 * C ** 0.5)).half().float()
    gy = torch.randn(B, Cout, H, W, generator=g) * 1e-3
    return x.cuda(), off.cuda(), w.cuda(), gy.cuda()


def _smb_grads(x, off, w, gy, dg):
    from sipmask_b200 import ops
    m = ops.TrainableDeformConv(x.shape[1], w.shape[0], 3, padding=1, deformable_groups=dg).cuda()
    m.weight.data.copy_(w)
    xr, offr = x.clone().requires_grad_(True), off.clone().requires_grad_(True)
    m(xr, offr).backward(gy)
    return xr.grad, offr.grad, m.weight.grad


def _ref64_grads(x, off, w, gy, dg):
    from oracle import ops as O
    x64, off64, w64 = [t.double().requires_grad_(True) for t in (x, off, w)]
    with torch.device('cuda'):                       # the oracle's index grids are made on the device too
        O.deform_conv(x64, off64, w64, padding=1, deformable_groups=dg).backward(gy.double())
    return x64.grad, off64.grad, w64.grad


# ---------------------------------------------------------------------------------------------------- kernel level
@pytest.mark.parametrize('B,C,H,W,dg', T.COL2IM_CASES)
def test_col2im_reference_kernel_vs_float64_autograd_vs_smb(B, C, H, W, dg):
    from oracle import ops as O
    from sipmask_b200 import conv
    gold = np.load(GOLDEN)
    key = '%d_%d_%d_%d_%d' % (B, C, H, W, dg)
    x, off, gcol = T.col2im_inputs(B, C, H, W, dg)
    # float64 autograd of the im2col restatement: d/dx, d/doffset of sum(cols * grad_col)
    x64, off64 = x.double().cuda().requires_grad_(True), off.double().cuda().requires_grad_(True)
    with torch.device('cuda'):
        cols, _, _ = O.deform_im2col(x64, off64, 3, 3, 1, 1, 1, dg)            # [B, C*9, HW], row c*9 + tap
    g64 = gcol.double().cuda().permute(1, 0, 2, 3).reshape(B, C * 9, H * W)
    (cols * g64).sum().backward()
    # smb: grad_col in the channel-last column layout [B, H, W, tap * C + c], scale {1, 1}
    gcl = gcol.view(C, 9, B, H, W).permute(2, 3, 4, 1, 0).reshape(B, H, W, 9 * C).contiguous().cuda()
    one = torch.ones(2, device='cuda')
    gin, goff = conv.deform_col2im(gcl, x.permute(0, 2, 3, 1).contiguous().half().cuda(),
                                   off.permute(0, 2, 3, 1).contiguous().cuda(), dg, one)
    smb_in = gin.permute(0, 3, 1, 2).cpu().numpy().ravel()
    smb_off = goff.permute(0, 3, 1, 2).cpu().numpy().ravel()
    for name, smb, auto, sample in (('input', smb_in, x64.grad, T.sample_index(x.numel(), 1)),
                                    ('offset', smb_off, off64.grad, T.sample_index(off.numel(), 2))):
        ref = gold['col2im_%s_%s' % (name, key)].astype(np.float64)
        auto = auto.cpu().numpy().ravel()
        scale = np.abs(ref).max()
        assert scale > 0
        assert np.abs(auto[sample] - ref).max() <= 1e-5 * scale, name
        assert np.abs(smb[sample] - ref).max() <= 1e-5 * scale, name
        assert np.abs(smb - auto).max() <= 1e-5 * np.abs(auto).max(), name


# ---------------------------------------------------------------------------------------------------- module level
def _wgrad_split(cout, kc, P):
    """smb_deform_weight_grad's split of the P pixels (wgrad_split in csrc/train_ops.cu): 128 x 128 tiles, 64-pixel
    blocks, about 264 CTAs -> (blocks, blocks per split, splits)."""
    tiles = -(-cout // 128) * -(-kc // 128)
    kb_total = -(-P // 64)
    want = max(1, min(-(-264 // tiles), kb_total))
    kps = -(-kb_total // want)
    return kb_total, kps, -(-kb_total // kps)


def _dw_bound(x, off, gy, dg, splits_cfg):
    """Per-element bound on |dW - dW64| [Cout, Cin, 3, 3]: the weight GEMM's accumulation (gamma of the pixels in one
    split, one fp32 rounding per split added) over m = sum_p |g| |col|, plus the fp16 rounding of s * g and of the columns
    (2^-11 each, their product 2^-22, fp16's subnormal spacing 2^-25 in absolute terms) and the fp32 interpolation of the
    columns (2^-20).  |col| is bounded by the columns of |x| (the bilinear weights are non-negative)."""
    from oracle import ops as O
    from oracle import numerics as NU
    kb_total, kps, splits = splits_cfg
    B, Cout, H, W = gy.shape
    C = x.shape[1]
    with torch.device('cuda'):
        ph, pw = max(3 - H, 0), max(3 - W, 0)                    # TrainableDeformConv's padding of small maps
        xa = torch.nn.functional.pad(x.double().abs(), (0, pw, 0, ph))
        oa = torch.nn.functional.pad(off.double(), (0, pw, 0, ph))
        cols, _, _ = O.deform_im2col(xa, oa, 3, 3, 1, 1, 1, dg)             # [B, C*9, Hp*Wp], row c*9 + tap
    ga = torch.nn.functional.pad(gy.double().abs(), (0, pw, 0, ph)).reshape(B, Cout, -1)
    m = torch.einsum('bop,bkp->ok', ga, cols).view(Cout, C, 3, 3)
    amax = float(gy.abs().max())
    e = math.frexp(amax)[1] - 1 if amax > 0 else 0
    s = 2.0 ** min(max(14 - e, -126), 126) if amax > 0 else 1.0
    g_sum = ga.sum((0, 2)).view(Cout, 1, 1, 1)
    c_sum = cols.sum((0, 2)).view(1, C, 3, 3)
    u = 2.0 ** -11
    rel = NU.gamma_k(64 * kps) + (splits - 1) * 2.0 ** -24 + 2 * u + u * u + 2.0 ** -20
    return rel * m + 2.0 ** -25 * (c_sum / s + g_sum)


@pytest.mark.parametrize('B,C,Cout,H,W,dg', FEATURE_ALIGN + PP_DCN + EDGES)
def test_module_gradients_vs_float64(B, C, Cout, H, W, dg):
    x, off, w, gy = _module_inputs(B, C, Cout, H, W, dg)
    cfg = _wgrad_split(Cout, 9 * C, B * max(H, 3) * max(W, 3))
    print('module B %d Cin %4d Cout %4d map %3dx%-3d dg %3d: weight GEMM %d x %d tiles, %d blocks, %d per split, %d splits'
          % (B, C, Cout, H, W, dg, -(-Cout // 128), -(-9 * C // 128), cfg[0], cfg[1], cfg[2]))
    got = _smb_grads(x, off, w, gy, dg)
    want = _ref64_grads(x, off, w, gy, dg)
    errs = {}
    for name, a, b in zip(('grad_input', 'grad_offset', 'grad_weight'), got, want):
        assert a.shape == b.shape and a.dtype == torch.float32, name
        errs[name] = _rel(a, b)
    assert max(errs.values()) <= REL, errs
    err = (got[2].double() - want[2]).abs()
    bound = _dw_bound(x, off, gy, dg, cfg)
    worst = float((err / bound).max())
    assert worst <= 1.0, ('grad_weight per-element bound', worst)


def test_gradient_scaling_is_exact():
    """grad_out * 2^-24 (far below fp16's normal range: cast to fp16 it would mostly flush to zero) and grad_out * 2^25
    (amax above fp16's 65504, so the scale s < 1) give dW and grad_offset of exactly 2^e times the unscaled ones;
    grad_input (float atomics, any order) agrees to rounding."""
    x, off, w, gy = _module_inputs(1, 256, 256, 25, 42, 4)
    a = _smb_grads(x, off, w, gy, 4)
    assert a[2].abs().max() > 0 and a[1].abs().max() > 0
    for e in (-24, 25):
        scaled = gy * 2.0 ** e
        if e < 0:
            assert (scaled.half() == 0).float().mean().item() > 0.9
        else:
            assert scaled.abs().max().item() > 65504
        b = _smb_grads(x, off, w, scaled, 4)
        assert torch.equal(b[2], a[2] * 2.0 ** e), e
        assert torch.equal(b[1], a[1] * 2.0 ** e), e
        assert _rel(b[0] * 2.0 ** -e, a[0]) <= 1e-6, e


def test_backward_is_deterministic():
    x, off, w, gy = _module_inputs(2, 256, 256, 50, 84, 4)
    a = _smb_grads(x, off, w, gy, 4)
    b = _smb_grads(x, off, w, gy, 4)
    assert torch.equal(a[2], b[2]) and torch.equal(a[1], b[1])


def test_needs_input_grad(monkeypatch):
    from sipmask_b200 import conv, ops
    calls = []
    for name in ('deform_col2im', 'deform_weight_grad'):
        fn = getattr(conv, name)
        monkeypatch.setattr(conv, name, lambda *a, _n=name, _f=fn, **k: calls.append(_n) or _f(*a, **k))
    x, off, w, gy = _module_inputs(1, 256, 256, 13, 21, 4)
    # frozen weight: no weight gradient, no weight-gradient work
    xr, offr = x.clone().requires_grad_(True), off.clone().requires_grad_(True)
    ops.deform_conv(xr, offr, w, 1, 1, 1, 1, 4).backward(gy)
    assert calls == ['deform_col2im'] and xr.grad is not None and offr.grad is not None
    # frozen x and offsets: only dW
    del calls[:]
    wr = w.clone().requires_grad_(True)
    ops.deform_conv(x, off, wr, 1, 1, 1, 1, 4).backward(gy)
    assert calls == ['deform_weight_grad'] and wr.grad is not None


class FeatureAlign(torch.nn.Module):
    """FeatureAlign of MM/mmdet/models/anchor_heads/sipmask_head.py:21-55 (flag_norm=False), with the DeformConv class
    as a parameter."""

    def __init__(self, dcn, c, dg=4):
        super().__init__()
        self.conv_offset = torch.nn.Conv2d(4, dg * 18, 1, bias=False)
        self.conv_adaption = dcn(c, c, kernel_size=3, padding=1, deformable_groups=dg)
        self.relu = torch.nn.ReLU(inplace=True)

    def forward(self, x, shape):
        offset = self.conv_offset(shape.detach())
        return self.relu(self.conv_adaption(x, offset))


def test_feature_align_step_trains_conv_offset():
    from oracle import ops as O
    from sipmask_b200 import ops
    torch.manual_seed(0)
    x, _, w, _ = _module_inputs(2, 256, 256, 25, 42, 4)
    shape = torch.rand(2, 4, 25, 42, device='cuda') * 4.0
    gy = torch.randn(2, 256, 25, 42, device='cuda') * 1e-3
    m = FeatureAlign(ops.TrainableDeformConv, 256).cuda()
    torch.nn.init.normal_(m.conv_offset.weight, std=0.1)
    m.conv_adaption.weight.data.copy_(w)
    y = m(x, shape)
    y.backward(gy)
    g = m.conv_offset.weight.grad
    assert g is not None and g.abs().max() > 0 and m.conv_adaption.weight.grad is not None
    # float64: the same step through the oracle
    wo = m.conv_offset.weight.detach().double().requires_grad_(True)
    off = torch.nn.functional.conv2d(shape.double(), wo)
    # sample where the fp32 step sampled (the fp32 offsets), with the float64 offsets' gradient path
    off = off + (m.conv_offset(shape).detach().double() - off).detach()
    with torch.device('cuda'):
        y64 = O.deform_conv(x.double(), off, w.double(), padding=1, deformable_groups=4)
    # the ReLU mask of the step itself: outputs within rounding of 0 must not pass the gradient in one and not the other
    y64.backward(gy.double() * (y > 0))
    assert _rel(g, wo.grad) <= REL
    # the known trap: ops.DeformConv runs under no_grad, so conv_offset never learns
    m0 = FeatureAlign(ops.DeformConv, 256).cuda()
    m0.conv_adaption.weight.data.copy_(w)
    y0 = m0(x, shape)
    assert not y0.requires_grad
    assert m0.conv_offset.weight.grad is None and m0.conv_adaption.weight.grad is None


def test_deform_conv_pack_keys_and_forward():
    from sipmask_b200 import ops
    m = ops.DeformConvPack(256, 256, 3, padding=1).cuda()
    assert list(m.state_dict().keys()) == ['weight', 'conv_offset.weight', 'conv_offset.bias']
    assert m.conv_offset.bias is not None and not m.conv_offset.weight.detach().any()
    torch.nn.init.normal_(m.conv_offset.weight, std=0.05)
    x = torch.randn(1, 256, 17, 17, device='cuda').half().float()
    y = m(x)
    want = ops.deform_conv(x, m.conv_offset(x), m.weight, m.stride, m.padding, m.dilation, m.groups, m.deformable_groups)
    assert torch.equal(y, want)
    # the module's own keys load strictly; a version-1 state dict's `_offset.*` keys are renamed, as the reference does
    m2 = ops.DeformConvPack(256, 256, 3, padding=1)
    m2.load_state_dict({k: v.detach().cpu() for k, v in m.state_dict().items()}, strict=True)
    assert torch.equal(m2.conv_offset.weight, m.conv_offset.weight.detach().cpu())
    m3 = ops.DeformConvPack(256, 256, 3, padding=1)
    m3.load_state_dict({'weight': m.weight.detach().cpu(), '_offset.weight': m.conv_offset.weight.detach().cpu(),
                        '_offset.bias': m.conv_offset.bias.detach().cpu()}, strict=True)
    assert torch.equal(m3.conv_offset.weight, m.conv_offset.weight.detach().cpu())
