"""SipMask's fused mask loss (ops.sipmask_mask_targets / sipmask_mask_loss / sipmask_head_mask_loss) on sm_90a.

The composition it replaces (tests/mask_loss_inputs.py::composition) runs on the device with fp32 matmuls (TF32 off),
torch's sigmoid, the reference's own CropSplit / CropSplitGt kernels (oracle/_ref/libsipmask_ref_cuda.so, compiled from the
reference sources by oracle/build.py) and F.binary_cross_entropy; its dZ is read with retain_grad and contracted in
float64.  Where the reference sources were absent at build time the compiled kernels are too, and the composition uses
ops.crop_split / crop_split_backward / crop_split_gt, which tests/test_gpu_ref_cuda.py pins bit for bit to them.
`sipmask_head_mask_loss` is compared with the unmodified reference head's `loss_mask` and gradients
(tests/golden/ref_mask_loss.npz, tests/golden/gen_golden_mask_loss.py).
"""
import ctypes
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mask_loss_inputs as MI

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _fp32_matmul():
    old = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32 = old


def _rel(a, b):
    a, b = a.double(), b.double()
    n = b.norm()
    return ((a - b).norm() / n).item() if n > 0 else (a - b).norm().item()


ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_SO = os.path.join(ROOT, 'oracle', '_ref', 'libsipmask_ref_cuda.so')
GOLDEN = os.path.join(ROOT, 'tests', 'golden', 'ref_mask_loss.npz')
_REF = []


def _ref_lib():
    if not _REF:
        _REF.append(ctypes.CDLL(REF_SO) if os.path.exists(REF_SO) else None)
    return _REF[0]


def _p(t):
    return ctypes.c_void_p(t.data_ptr())


class _Crop(torch.autograd.Function):
    """CropSplitFunction (ops/crop/crop_split.py:12-38): zero-initialised outputs, the reference kernels when built"""

    @staticmethod
    def forward(ctx, data, rois):
        from sipmask_b200 import ops
        ctx.save_for_backward(rois)
        lib = _ref_lib()
        if lib is None:
            return ops.crop_split(data, rois)
        _, H, W, N = data.shape
        out = data.new_zeros(H, W, N)
        assert lib.ref_crop_split_forward(_p(data), _p(rois), _p(out), H, W, 2, N) == 0
        return out

    @staticmethod
    def backward(ctx, g):
        from sipmask_b200 import ops
        (rois,) = ctx.saved_tensors
        g = g.contiguous()
        lib = _ref_lib()
        if lib is None:
            return ops.crop_split_backward(g, rois), None
        H, W, N = g.shape
        grad = g.new_zeros(4, H, W, N)
        assert lib.ref_crop_split_backward(_p(g), _p(rois), _p(grad), H, W, 2, N) == 0
        return grad, None


def _crop_gt(data, rois):
    from sipmask_b200 import ops
    lib = _ref_lib()
    if lib is None:
        return ops.crop_split_gt(data, rois)
    H, W, N = data.shape
    out = data.new_zeros(H, W, N)
    assert lib.ref_crop_split_gt_forward(_p(data), _p(rois), _p(out), H, W, 2, N) == 0
    return out


def _fused(d, g=None, need=(True, True)):
    from sipmask_b200 import ops
    feat = d['feat'].clone().requires_grad_(need[0])
    cofs = d['cofs'].clone().requires_grad_(need[1])
    loss = ops.sipmask_mask_loss(feat, cofs, d['boxes'], d['offsets'], d['bits'], d['rows'], d['weights'])
    if need[0] or need[1]:
        (loss * (1.0 if g is None else g)).sum().backward()
    torch.cuda.synchronize()
    return loss.detach(), feat.grad, cofs.grad


def _composed(d):
    feat = d['feat'].clone().requires_grad_(True)
    cofs = d['cofs'].clone().requires_grad_(True)
    zs = []
    loss = MI.composition(d, feat, cofs, _Crop.apply, _crop_gt, keep_dz=zs)
    loss.sum().backward()
    # float64 contraction of the composition's own fp32 dZ
    B, _, H, W = feat.shape
    offs = d['offsets'].tolist()
    dX = torch.zeros(B, 32, H, W, dtype=torch.float64, device='cuda')
    dC = torch.zeros(d['cofs'].shape, dtype=torch.float64, device='cuda')
    it = iter(zs)
    for b in range(B):
        n0, n1 = offs[b], offs[b + 1]
        if n1 == n0:
            continue
        dz = next(it).grad.double().reshape(4, H * W, n1 - n0)
        X = d['feat'][b].double().reshape(32, -1).t()
        C = d['cofs'][n0:n1].double().view(-1, 4, 32)
        dX[b] = sum(dz[q] @ C[:, q] for q in range(4)).t().reshape(32, H, W)
        dC[n0:n1] = torch.stack([dz[q].t() @ X for q in range(4)], 1).reshape(-1, 128)
    return loss.detach(), feat.grad, cofs.grad, dX, dC


REGIMES = [20.0, 40.0, -110.0, -120.0, -20.0, -40.0]


def _regime_inputs():
    """Two clustered images plus one whose features are e_0 at every pixel, so that z = cof[32 * cell] exactly: its
    instances' cells carry the logits of REGIMES, over a checkerboard target (t = 0 and 1 in every cell).
      z = 20, 40: p rounds to exactly 1; z = -110, -120: expf(-z) overflows, p = 0.  There the term is 100 (wrong
      target) or 0 and dz is exactly 0.  z = -40: p ~ 4e-18, (1 - p) p below the 1e-12 clamp of the BCE backward;
      z = -20: p ~ 2e-9 just above it.
    Every other logit has |z| <= 14 (|feat| <= 1, |cof| <= 14 / 32): away from z ~ 17, where fp32's sigmoid rounds to 1
    and a one-ulp difference would move a term between ~17 and 100."""
    inp = MI.clustered_inputs(3, 40, 72, 24, seed=11)
    H, W = 40, 72
    inp['feat'][2] = 0
    inp['feat'][2, 0] = 1
    n0, n1 = inp['offsets'][2].item(), inp['offsets'][3].item()
    yy, xx = np.mgrid[0:H, 0:W]
    for i, n in enumerate(range(n0, n1)):
        for q in range(4):
            inp['cofs'][n, 32 * q] = REGIMES[(i + q) % len(REGIMES)]
        inp['planes'][inp['rows'][n]] = torch.from_numpy(((xx + yy) % 2).astype(np.float32))
    return inp


def test_bce_uses_log1p():
    """torch's CUDA binary_cross_entropy takes log1p(-p) for the (1 - t) term (not log(1 - p)), which the kernel
    restates; p where the two differ in fp32."""
    p = torch.tensor([1e-5, 3e-4, 0.01, 0.3, 0.77], device='cuda')
    got = F.binary_cross_entropy(p, torch.zeros_like(p), reduction='none')
    assert torch.equal(got, -torch.log1p(-p))
    assert not torch.equal(-torch.log(1 - p), -torch.log1p(-p))


def test_exact_logit_parity_with_composition():
    """Grid inputs: z, p, every loss term and every dz are the same in both paths.  loss[b] differs only by summation
    order (1e-6 relative); d feat and d cofs are compared with the float64 contraction of the composition's own dZ
    (1e-5 relative norm: the fused path's fp32 sums of exact products, against exact sums)."""
    d = MI.to_device(_regime_inputs())
    loss, dX, dC = _fused(d)
    rloss, _, _, dX64, dC64 = _composed(d)
    assert torch.allclose(loss.double(), rloss.double(), rtol=1e-6, atol=0), (loss, rloss)
    assert rloss[2].item() > 10 * rloss[0].item()         # the saturated, wrong regime terms (100 each) dominate
    assert _rel(dX, dX64) < 1e-5 and _rel(dC, dC64) < 1e-5, (_rel(dX, dX64), _rel(dC, dC64))
    # the regime image: d cofs of the saturated cells' channel 0 only come from the non-saturated cells
    n0 = d['offsets'][2].item()
    assert torch.isfinite(dC).all() and torch.isfinite(dX).all()
    assert _rel(dC[n0:], dC64[n0:]) < 1e-5


GEOM_BOXES = [
    (2.0, 3.0, 20.0, 17.0),            # integer edges
    (2.3, 4.7, 19.6, 15.2),            # fractional edges
    (0.0, 0.0, 9.9, 9.9),              # roi = 5.0: (pw - x1) / roi_w is exactly 1 at pw = 5
    (1.0, 1.0, 6.9, 6.9),              # roi = 3.0: (pw - x1) / roi_w is exactly 1 at pw = 4
    (-5.0, -3.0, 10.0, 12.0),          # partly outside
    (35.0, 20.0, 50.0, 30.0),          # partly outside, right / bottom
    (100.0, 100.0, 120.0, 130.0),      # fully outside
    (-20.0, -20.0, -5.0, -5.0),        # fully outside
    (3.0, 2.0, 3.6, 12.0),             # narrower than a pixel, area 6
    (0.0, 0.0, 40.0, 24.0),            # the whole map
    (-0.5, -0.5, 40.3, 24.7),          # beyond the whole map
]


def test_geometry_bits_single_instance_images():
    """One instance per image with four distinct coefficient blocks: d feat[pix] = dz * C[n, cell] is one product, so it
    must be the composition's bits; the boxes cover the cell geometry's edge cases."""
    H, W = 24, 40
    B = len(GEOM_BOXES)
    rs = np.random.RandomState(5)
    inp = dict(feat=torch.tensor(np.round(rs.uniform(-1, 1, (B, 32, H, W)) * 256) / 256, dtype=torch.float32),
               cofs=torch.tensor(np.round(rs.uniform(-0.4, 0.4, (B, 128)) * 256) / 256, dtype=torch.float32),
               boxes=torch.tensor(GEOM_BOXES, dtype=torch.float32), offsets=torch.arange(B + 1, dtype=torch.int32),
               planes=torch.tensor(rs.rand(B, H, W) < 0.5, dtype=torch.float32),
               rows=torch.arange(B, dtype=torch.int64), weights=torch.tensor(rs.uniform(0.5, 1.5, B), dtype=torch.float32))
    d = MI.to_device(inp)
    loss, dX, dC = _fused(d)
    rloss, rX, rC, _, dC64 = _composed(d)
    assert torch.equal(dX, rX)
    assert torch.allclose(loss.double(), rloss.double(), rtol=1e-6, atol=0)
    assert _rel(dC, dC64) < 1e-5
    assert (loss[6] == 0) and (loss[7] == 0) and (dC[6] == 0).all() and (dC[7] == 0).all()


@pytest.mark.parametrize('B,H,W,per_img', [(2, 400, 672, 60), (2, 288, 288, 80), (3, 180, 320, 40)])
def test_general_inputs_against_float64(B, H, W, per_img):
    """Unrounded fp32 inputs with |z| <= 12 against float64.  Each z carries a relative error of at most ~32 * 2^-24
    (fp32 fma chain) times sum |x c| <= 12, i.e. |dz_err| <= 2.3e-5 absolute in z; sigmoid's derivative p (1 - p) <= 1/4
    turns that into <= 6e-6 in p; the BCE term and dz = c (p - t) inherit it against values of order c, and the sums
    (fp32, fixed order, up to ~10^5 terms of one sign per image in the loss, mixed signs in the gradients) add ~1e-6 in
    norm.  Measured errors sit far below; 1e-5 (loss: relative, gradients: relative norm) bounds them with margin."""
    inp = MI.clustered_inputs(B, H, W, per_img, seed=B * 7 + H, grid=False, zmax=12.0)
    d = MI.to_device(inp)
    loss, dX, dC = _fused(d)
    ref = MI.reference64({k: v.cuda() for k, v in inp.items()})
    assert torch.allclose(loss.double().cpu(), ref[0].cpu(), rtol=1e-5, atol=0), (loss, ref[0])
    assert _rel(dX, ref[1]) < 1e-5 and _rel(dC, ref[2]) < 1e-5, (_rel(dX, ref[1]), _rel(dC, ref[2]))


def test_edges_empty_and_stacked():
    """M = 0; an image without instances; instances whose gt object has an empty mask; > 1000 instances stacked over one
    region of one image (several instance chunks and staging batches per tile)."""
    from sipmask_b200 import ops
    H, W = 64, 96
    # M = 0
    feat = torch.randn(2, 32, H, W, device='cuda', requires_grad=True)
    cofs = torch.zeros(0, 128, device='cuda', requires_grad=True)
    z = lambda *s, dt=torch.float32: torch.zeros(*s, dtype=dt, device='cuda')          # noqa: E731
    loss = ops.sipmask_mask_loss(feat, cofs, z(0, 4), z(3, dt=torch.int32), z(0, H, 3, dt=torch.int32),
                                 z(0, dt=torch.int64), z(0))
    loss.sum().backward()
    assert (loss == 0).all() and (feat.grad == 0).all() and cofs.grad.shape == (0, 128)
    # an empty image between two, empty gt masks, and 1100 stacked instances
    inp = MI.clustered_inputs(3, H, W, 1100, seed=3, objs_per_img=2)
    keep = torch.cat([torch.arange(0, 1100), torch.arange(2200, 2300)])
    for k in ('cofs', 'boxes', 'rows', 'weights'):
        inp[k] = inp[k][keep]
    inp['offsets'] = torch.tensor([0, 1100, 1100, 1200], dtype=torch.int32)
    inp['planes'][1] = 0
    d = MI.to_device(inp)
    loss, dX, dC = _fused(d)
    ref = MI.reference64({k: v.cuda() for k, v in inp.items()})
    assert loss[1] == 0 and (dX[1] == 0).all()
    assert torch.allclose(loss.double().cpu(), ref[0].cpu(), rtol=1e-5, atol=0)
    assert _rel(dX, ref[1]) < 1e-5 and _rel(dC, ref[2]) < 1e-5


def test_behaviour_determinism_needs_input_grad_and_scaling():
    d = MI.to_device(MI.clustered_inputs(2, 96, 160, 120, seed=9, grid=False, zmax=12.0))
    a, b = _fused(d), _fused(d)
    for x, y in zip(a, b):
        assert torch.equal(x, y)
    lx, gx, gc = _fused(d, need=(True, False))
    assert gc is None and torch.equal(gx, a[1]) and torch.equal(lx, a[0])
    lc, gx, gc = _fused(d, need=(False, True))
    assert gx is None and torch.equal(gc, a[2])
    s = 2.0 ** -20
    _, sx, sc = _fused(d, g=s)
    assert torch.equal(sx, a[1] * s) and torch.equal(sc, a[2] * s)


@pytest.mark.parametrize('hf,wf', [(96, 128), (97, 129), (50, 61), (131, 170), (3, 5)])
def test_targets_equal_interpolate_pad_threshold(hf, wf):
    """sipmask_mask_targets == F.interpolate(0.5, bilinear, align_corners=False) -> zero pad / crop -> gt(0.5), bit for
    bit, for even and odd sources smaller and larger than 2 * (H, W), from uint8, bool and float masks."""
    from sipmask_b200 import ops
    H, W = 48, 64
    rs = np.random.RandomState(hf * 1000 + wf)
    masks = [torch.from_numpy(rs.rand(3, hf, wf) < 0.6).cuda(), torch.from_numpy((rs.rand(2, hf, wf) < 0.4).astype(np.uint8)).cuda(),
             torch.from_numpy((rs.rand(4, hf, wf) < 0.5).astype(np.float32)).cuda()]
    bits, offs = ops.sipmask_mask_targets(masks, (H, W))
    want = []
    for m in masks:
        gm = F.interpolate(m.float().unsqueeze(0), scale_factor=0.5, mode='bilinear', align_corners=False).squeeze(0)
        new = gm.new_zeros(gm.shape[0], H, W)
        h, w = min(H, gm.shape[1]), min(W, gm.shape[2])
        new[:, :h, :w] = gm[:, :h, :w]
        want.append(new.gt(0.5).cpu().numpy())
    assert torch.equal(bits.cpu(), MI.pack_bits(np.concatenate(want)))
    assert offs.tolist() == [0, 3, 5, 9]


def test_head_mask_loss_against_reference_block():
    """sipmask_head_mask_loss on head-shaped intermediates (two images, one without positives after the area filter)
    against the reference block restated with torch ops and the crop kernels (sipmask_head.py:407-484, rescoring off):
    loss to 1e-5 relative and the gradients of feat_masks and the cof predictions to 1e-4 relative norm (fp32 cuBLAS sums
    against the fused path's fixed-order sums, |z| <= 14)."""
    from sipmask_b200 import ops
    torch.manual_seed(0)
    B, H, W, P, C = 3, 48, 80, 600, 80
    rs = np.random.RandomState(2)
    feat = torch.tensor(rs.uniform(-1, 1, (B, 32, H, W)), dtype=torch.float32, device='cuda')
    cof = torch.tensor(rs.uniform(-0.4, 0.4, (B, P, 128)), dtype=torch.float32, device='cuda')
    cls = torch.tensor(rs.randn(B, P, C), dtype=torch.float32, device='cuda')
    gt_bboxes, gt_masks, det, labels, gt_inds = [], [], [], [], []
    for b in range(B):
        G = 3
        xy = rs.uniform(0, [2 * W - 40, 2 * H - 40], (G, 2))
        wh = rs.uniform(16, 60, (G, 2))
        gb = np.concatenate([xy, xy + wh], 1)
        gt_bboxes.append(torch.tensor(gb, dtype=torch.float32, device='cuda'))
        m = np.zeros((G, 2 * H + 3, 2 * W - 5), dtype=np.uint8)
        for g_ in range(G):
            x1, y1, x2, y2 = gb[g_].astype(int)
            m[g_, y1:y2, x1:x2] = 1
        gt_masks.append(m)
        lab = np.where(rs.rand(P) < 0.05, rs.randint(1, C + 1, P), 0)
        if b == 1:
            lab[:] = 0
        gi = rs.randint(0, G, P)
        bx = gb[gi] + rs.uniform(-6, 6, (P, 4))
        if b == 2:
            bx[:, 2:] = bx[:, :2] + 0.5          # every positive has area <= 1 after / 2
        det.append(torch.tensor(bx, dtype=torch.float32, device='cuda'))
        labels.append([torch.tensor(lab[:400], device='cuda'), torch.tensor(lab[400:], device='cuda')])
        gt_inds.append(torch.tensor(gi[lab > 0], device='cuda'))

    def run(fused):
        f = feat.clone().requires_grad_(True)
        c = cof.clone().requires_grad_(True)
        if fused:
            loss = ops.sipmask_head_mask_loss(f, c, cls, det, labels, gt_inds, gt_bboxes, gt_masks)
        else:
            loss = 0
            for i in range(B):
                lab = torch.cat([lv.flatten() for lv in labels[i]])
                bbox_dt = (det[i] / 2).detach()
                pos = (lab > 0).nonzero().view(-1)
                cp = c[i][pos]
                idx_gt = gt_inds[i]
                bbox_dt = bbox_dt[pos, :4]
                area = (bbox_dt[:, 2] - bbox_dt[:, 0]) * (bbox_dt[:, 3] - bbox_dt[:, 1])
                bbox_dt, idx_gt, cp = bbox_dt[area > 1.0], idx_gt[area > 1.0], cp[area > 1.0]
                if bbox_dt.shape[0] == 0:
                    loss += area.sum() * 0
                    continue
                score = cls[i, pos, lab[pos] - 1].sigmoid().detach()[area > 1.0]
                b1 = gt_bboxes[i][idx_gt] / 2                  # bbox_overlaps(is_aligned=True), geometry.py:57-69
                lt = torch.max(b1[:, :2], bbox_dt[:, :2])
                rb = torch.min(b1[:, 2:], bbox_dt[:, 2:])
                wh = (rb - lt + 1).clamp(min=0)
                ov = wh[:, 0] * wh[:, 1]
                a1 = (b1[:, 2] - b1[:, 0] + 1) * (b1[:, 3] - b1[:, 1] + 1)
                a2 = (bbox_dt[:, 2] - bbox_dt[:, 0] + 1) * (bbox_dt[:, 3] - bbox_dt[:, 1] + 1)
                ious = ov / (a1 + a2 - ov)
                wgt = score * ious
                wgt = wgt / (wgt.sum() + 0.0001) * len(wgt)
                gm = F.interpolate(torch.from_numpy(gt_masks[i]).float().cuda().unsqueeze(0), scale_factor=0.5,
                                   mode='bilinear', align_corners=False).squeeze(0)
                new = gm.new_zeros(gm.shape[0], H, W)
                h, w = min(H, gm.shape[1]), min(W, gm.shape[2])
                new[:, :h, :w] = gm[:, :h, :w]
                new = new.gt(0.5).float().index_select(0, idx_gt).permute(1, 2, 0).contiguous()
                X = f[i].permute(1, 2, 0)
                P_ = torch.stack([torch.sigmoid(X @ cp[:, 32 * q:32 * q + 32].t()) for q in range(4)])
                pred = _Crop.apply(P_.contiguous(), bbox_dt)
                gtc = ops.crop_split_gt(new, bbox_dt)
                pre = F.binary_cross_entropy(pred, gtc, reduction='none')
                pre = pre.sum(dim=(0, 1)) / (bbox_dt[:, 2] - bbox_dt[:, 0]) / (bbox_dt[:, 3] - bbox_dt[:, 1]) / bbox_dt.shape[0]
                loss += torch.sum(pre * wgt.detach())
            loss = loss / B
        loss.backward()
        return loss.detach(), f.grad, c.grad

    lf, gf, cf = run(True)
    lr, gr, cr = run(False)
    assert abs(lf.item() - lr.item()) <= 1e-5 * abs(lr.item()), (lf, lr)
    assert _rel(gf, gr) < 1e-4 and _rel(cf, cr) < 1e-4, (_rel(gf, gr), _rel(cf, cr))


def test_head_mask_loss_against_reference_head_golden():
    """sipmask_head_mask_loss on the intermediates of the unmodified reference SipMaskHead.loss (run on the CPU by
    tests/golden/gen_golden_mask_loss.py, rescoring off) against its loss_mask and the gradients of feat_masks and every
    level of cof_preds.  Bound 1e-4 relative (norm for the gradients): both sides compute the same fp32 expressions, but
    the reference on the CPU (its own sum orders, matmul blocking and libm logf / expf) and the fused kernels on the GPU
    (fixed-order sums, CUDA's logf / expf) differ by a few ulp per term, which sums over ~10^4 terms keep near 1e-6."""
    from sipmask_b200 import ops
    z = np.load(GOLDEN)
    L, B = int(z['num_levels']), int(z['num_imgs'])
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()         # noqa: E731
    feat = cuda(z['feat_masks']).requires_grad_(True)
    cof_preds = [cuda(z['cof_preds_%d' % lv]).requires_grad_(True) for lv in range(L)]
    cls_scores = [cuda(z['cls_scores_%d' % lv]) for lv in range(L)]
    # sipmask_head.py:392-406, as the reference builds them
    flatten_cls_scores1 = torch.cat([c.permute(0, 2, 3, 1).reshape(B, -1, 80) for c in cls_scores], dim=1)
    flatten_cof_preds = torch.cat([c.permute(0, 2, 3, 1).reshape(c.shape[0], -1, 32 * 4) for c in cof_preds], dim=1)
    det = [cuda(z['det_bboxes_%d' % i]) for i in range(B)]
    labels = [[cuda(z['labels_%d_%d' % (i, lv)]) for lv in range(L)] for i in range(B)]
    gt_inds = [cuda(z['gt_inds_%d' % i]) for i in range(B)]
    gt_bboxes = [cuda(z['gt_bboxes_%d' % i]) for i in range(B)]
    gt_masks = [z['gt_masks_%d' % i] for i in range(B)]
    loss = ops.sipmask_head_mask_loss(feat, flatten_cof_preds, flatten_cls_scores1, det, labels, gt_inds, gt_bboxes,
                                      gt_masks)
    loss.backward()
    ref = float(z['loss_mask'])
    assert ref > 0 and abs(loss.item() - ref) <= 1e-4 * ref, (loss.item(), ref)
    assert _rel(feat.grad, cuda(z['d_feat_masks'])) < 1e-4
    for lv in range(L):
        want = cuda(z['d_cof_preds_%d' % lv])
        assert _rel(cof_preds[lv].grad, want) < 1e-4 or want.norm() == 0, lv


def test_mask_loss_rejects_non_contiguous_device_tensors(monkeypatch):
    """Non-contiguous CUDA inputs raise before anything is launched."""
    from sipmask_b200 import _lib, ops
    d = MI.to_device(MI.clustered_inputs(1, 16, 40, 3, seed=1))

    def fail():
        raise AssertionError('the library was called')
    monkeypatch.setattr(_lib, 'lib', fail)
    args = dict(feat_masks=d['feat'], cofs=d['cofs'], boxes=d['boxes'], img_offsets=d['offsets'], targets=d['bits'],
                gt_rows=d['rows'], weights=d['weights'])
    bad = dict(feat_masks=d['feat'].transpose(2, 3).contiguous().transpose(2, 3),
               cofs=d['cofs'].t().contiguous().t(), boxes=d['boxes'].t().contiguous().t(),
               weights=torch.stack([d['weights'], d['weights']], 1)[:, 0])
    for k, v in bad.items():
        assert not v.is_contiguous() and v.is_cuda
        a = dict(args)
        a[k] = v
        with pytest.raises(_lib.SmbError, match='contiguous'):
            ops.sipmask_mask_loss(**a)
