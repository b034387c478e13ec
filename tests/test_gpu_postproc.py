"""GPU parity tests (run with -m gpu on an H100): CUDA post-processing kernels, called through the
C ABI, against the CPU oracle on the same seeded inputs and against the reference-generated fixtures."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _oracle():
    from oracle import ops as O
    from oracle import postproc as P
    from oracle import cbind
    return O, P, cbind


@pytest.fixture(params=[False, True], ids=['scalar_dot', 'tensor_dot'])
def mask_dot(request):
    """Both families of mask kernels for fp16 prototypes: scalar fmaf and mma.sync (smb_mask_set_tensor_dot)."""
    from sipmask_b200 import ops
    prev = ops.set_mask_tensor_dot(request.param)
    yield request.param
    ops.set_mask_tensor_dot(prev)


def _rand_dets(n, seed, size=200.0):
    rng = np.random.RandomState(seed)
    xy = rng.rand(n, 2) * size
    wh = rng.rand(n, 2) * size * 0.4 + 1
    return np.concatenate([xy, xy + wh, rng.rand(n, 1)], 1).astype(np.float32)


@pytest.mark.parametrize('n', [1, 5, 63, 64, 65, 300, 1000, 4097, 8192])
@pytest.mark.parametrize('cmp_ge', [False, True])
def test_nms_matches_oracle(n, cmp_ge):
    from sipmask_b200 import ops
    O, P, cbind = _oracle()
    dets = _rand_dets(n, n, size=60.0 if n > 1000 else 200.0)
    keep_ref = cbind.nms(dets, 0.5, int(cmp_ge))
    d, inds = ops.nms(torch.from_numpy(dets).cuda(), 0.5, cmp_ge=cmp_ge)
    assert inds.dtype == torch.long
    assert inds.cpu().numpy().tolist() == keep_ref.tolist()
    np.testing.assert_array_equal(d.cpu().numpy(), dets[keep_ref])


def test_nms_known_answers(golden_dir):
    from sipmask_b200 import ops
    g = np.load(os.path.join(golden_dir, 'nms_known_answers.npz'))
    d, inds = ops.nms(g['mm4_dets'], float(g['mm4_thr']), device_id=0)        # numpy in -> numpy out
    assert isinstance(inds, np.ndarray) and len(inds) == int(g['mm4_num_keep']) and inds.tolist() == [0, 2, 3]
    d, inds = ops.nms(g['mm7_dets'], float(g['mm7_thr']), device_id=0)
    assert len(inds) == int(g['mm7_num_keep'])
    d, inds = ops.nms(torch.zeros(0, 5).cuda(), 0.5)
    assert inds.numel() == 0


def test_nms_ties_are_stable():
    from sipmask_b200 import ops
    O, P, cbind = _oracle()
    dets = _rand_dets(500, 7, size=80.0)
    dets[:, 4] = np.round(dets[:, 4] * 4) / 4          # many exact score ties
    keep_ref = cbind.nms(dets, 0.4, 0)
    _, inds = ops.nms(torch.from_numpy(dets).cuda(), 0.4)
    assert inds.cpu().tolist() == keep_ref.tolist()


@pytest.mark.parametrize('seed,n,C,thr,max_num', [(0, 3350, 80, 0.05, 100), (1, 500, 80, 0.05, 100), (2, 200, 5, 0.3, 1000),
                                                  (3, 64, 80, 0.9999, 100), (4, 4096, 3, 0.05, 10), (5, 5000, 6, 0.05, 100)])
def test_multiclass_nms_matches_oracle(seed, n, C, thr, max_num):
    from sipmask_b200 import ops
    O, P, cbind = _oracle()
    g = torch.Generator().manual_seed(seed)
    dets = _rand_dets(n, seed, size=400.0)
    boxes = torch.from_numpy(dets[:, :4].copy())
    scores = torch.sigmoid(torch.randn(n, C, generator=g) * 2 - 4)
    ctr = torch.sigmoid(torch.randn(n, generator=g))
    bg = torch.cat([scores.new_zeros(n, 1), scores], 1)
    rb, rl, ri = O.multiclass_nms_idx(boxes, bg, thr, 0.5, max_num, score_factors=ctr)
    db, dl, di = ops.multiclass_nms_idx(boxes.cuda(), bg.cuda(), thr, dict(type='nms', iou_thr=0.5), max_num,
                                        score_factors=ctr.cuda())
    assert dl.cpu().tolist() == rl.tolist()
    assert di.cpu().tolist() == ri.tolist()
    np.testing.assert_array_equal(db.cpu().numpy(), rb.numpy())


@pytest.mark.parametrize('seed,n,C', [(0, 2395, 80), (1, 300, 40), (2, 150, 3)])
def test_fast_nms_matches_oracle(seed, n, C):
    from sipmask_b200 import ops
    O, P, cbind = _oracle()
    g = torch.Generator().manual_seed(seed)
    dets = _rand_dets(n, seed + 10, size=300.0)
    boxes = torch.from_numpy(dets[:, :4].copy())
    scores = torch.sigmoid(torch.randn(n, C, generator=g) * 2 - 2)
    ctr = torch.sigmoid(torch.randn(n, generator=g))
    cofs = torch.randn(n, 128, generator=g)
    s = (scores * ctr.view(-1, 1)).transpose(1, 0).contiguous()
    rb, rl, rc, ri = O.fast_nms(boxes, s, cofs, 0.5, 200, 0.1, 100)
    db, dl, di = ops.fast_nms(boxes.cuda(), scores.cuda(), ctr.cuda(), 0.5, 200, 0.1, 100)
    assert dl.cpu().tolist() == rl.tolist()
    assert di.cpu().tolist() == ri.tolist()
    np.testing.assert_array_equal(db.cpu().numpy(), rb.numpy())


@pytest.mark.parametrize('sizes,img_shape,nms_pre', [
    ([(100, 168), (50, 84), (25, 42), (13, 21), (7, 11)], (800, 1333), 1000),
    ([(12, 16), (6, 8), (3, 4), (2, 2), (1, 1)], (96, 125), 60)])
def test_decode_topk_matches_oracle(sizes, img_shape, nms_pre):
    from sipmask_b200 import ops, synth
    O, P, cbind = _oracle()
    strides = (8, 16, 32, 64, 128)
    cls, box, ctr, cof = synth.head_level_inputs(sizes, seed=3)
    rb, rs, rc, rcof, ridx = P.decode_candidates(cls, box, ctr, cof, strides, img_shape + (3,), nms_pre)
    cl = [c.permute(1, 2, 0).contiguous().cuda() for c in cls]
    bl = [b.permute(1, 2, 0).contiguous().cuda() for b in box]
    tl = [t.permute(1, 2, 0).contiguous().cuda() for t in ctr]
    db, ds, dc, dloc = ops.decode_topk(cl, bl, tl, strides, img_shape, nms_pre, scale_factor=1.0)
    assert dloc.cpu().tolist() == ridx.tolist()                       # bit-exact candidate selection and order
    np.testing.assert_array_equal(db.cpu().numpy(), rb.numpy())        # box arithmetic is exact
    np.testing.assert_allclose(ds.cpu().numpy(), rs.numpy(), rtol=2e-6, atol=1e-7)   # sigmoid: expf vs torch CPU
    np.testing.assert_allclose(dc.cpu().numpy(), rc.numpy(), rtol=2e-6, atol=1e-7)


def _iou(a, b):
    inter = np.logical_and(a, b).sum((1, 2)).astype(np.float64)
    union = np.logical_or(a, b).sum((1, 2)).astype(np.float64)
    return (inter + 1e-9) / (union + 1e-9)


@pytest.mark.parametrize('H,W,N,layout,dtype', [(100, 168, 17, 'chw', torch.float32), (100, 168, 17, 'hwc', torch.float16),
                                                (37, 53, 5, 'chw', torch.float16), (37, 53, 70, 'hwc', torch.float32),
                                                (400, 672, 100, 'hwc', torch.float16)])
def test_mask_assemble_matches_oracle(H, W, N, layout, dtype, mask_dot):
    from sipmask_b200 import ops, synth
    if mask_dot and dtype != torch.float16:
        pytest.skip('the tensor-core kernels take fp16 prototypes only (fp32 prototypes always run the scalar kernels)')
    O, P, cbind = _oracle()
    g = torch.Generator().manual_seed(H + N)
    protos = synth.prototypes(H, W, seed=N)
    protos_in = protos.to(dtype)
    cofs = torch.randn(N, 128, generator=g)
    cx = torch.rand(N, generator=g) * W * 2
    cy = torch.rand(N, generator=g) * H * 2
    bw = torch.rand(N, generator=g) * W * 1.2 + 2
    bh = torch.rand(N, generator=g) * H * 1.2 + 2
    boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).clamp(min=0)
    boxes[0] = torch.tensor([0.0, 0.0, 2.0 * W, 2.0 * H])              # whole image
    ref = cbind.mask_assemble(protos_in.float().numpy(), cofs.numpy(), (boxes * 0.5).numpy())
    p_dev = (protos_in if layout == 'chw' else protos_in.permute(1, 2, 0)).contiguous().cuda()
    out = ops.mask_assemble(p_dev, cofs.cuda(), boxes.cuda(), 0.5, layout=layout, out_dtype=torch.float32)
    got = out.cpu().numpy()
    assert ((got == 0) == (ref == 0)).all()                              # crop geometry is exact
    # scalar kernels: sequential fp32 fmaf like the oracle; tensor-core kernels: fp16 hi + lo coefficients (2^-22 relative
    # per term) and the tensor core's own fp32 summation order
    np.testing.assert_allclose(got, ref, atol=5e-6 if mask_dot else 3e-6, rtol=0)
    # x2 upsample + threshold
    m_ref = cbind.upsample2_thresh(ref, 0.4)
    m_dev = ops.mask_upsample2_threshold(out, (2 * H - 3, 2 * W - 1), 0.4).cpu().numpy()
    assert _iou(m_dev, m_ref[:, :2 * H - 3, :2 * W - 1]).min() >= 0.999
    # bit-packed variant and the fully fused kernel must agree with the two-step path bit for bit
    oh, ow = 2 * H - 3, 2 * W - 1
    packed = ops.unpack_mask_bits(ops.mask_upsample2_threshold_pack(out, (oh, ow), 0.4), ow).cpu().numpy()
    assert _iou(packed, m_ref[:, :oh, :ow]).min() >= 0.999
    fused = ops.unpack_mask_bits(ops.mask_assemble_pack(p_dev, cofs.cuda(), boxes.cuda(), 0.5, (oh, ow), 0.4, layout=layout), ow).cpu().numpy()
    assert _iou(fused, m_ref[:, :oh, :ow]).min() >= 0.999
    assert (fused != packed).mean() < 1e-5
    fused_full = ops.unpack_mask_bits(ops.mask_assemble_pack(p_dev, cofs.cuda(), boxes.cuda(), 0.5, (2 * H + 5, 2 * W + 40), 0.4,
                                                             layout=layout), 2 * W + 40).cpu().numpy()
    assert fused_full[:, 2 * H:].sum() == 0 and fused_full[:, :, 2 * W:].sum() == 0       # beyond the x2 frame: zeros
    assert _iou(fused_full[:, :2 * H, :2 * W], m_ref).min() >= 0.999
    # fp16 output variant
    out16 = ops.mask_assemble(p_dev, cofs.cuda(), boxes.cuda(), 0.5, layout=layout, out_dtype=torch.float16)
    np.testing.assert_allclose(out16.float().cpu().numpy(), ref, atol=1e-3, rtol=0)


@pytest.mark.parametrize('H,W,N,layout', [(400, 672, 100, 'hwc'), (37, 53, 9, 'chw'), (64, 64, 150, 'hwc'), (9, 70, 6, 'hwc'),
                                          (100, 168, 33, 'chw')])
def test_mask_tensor_dot_matches_scalar_kernels(H, W, N, layout):
    """mma.sync kernels vs the scalar-fmaf kernels on the same fp16 prototypes: identical crop geometry (which pixels are
    non-zero), values within 2e-6, packed masks equal up to pixels sitting on the threshold.  Boxes include whole-image,
    sub-pixel, integer-aligned and tile-straddling rois; N = 150 needs two list passes per tile."""
    from sipmask_b200 import ops, synth
    g = torch.Generator().manual_seed(7 * H + N)
    protos = synth.prototypes(H, W, seed=N).half()
    p_dev = (protos if layout == 'chw' else protos.permute(1, 2, 0)).contiguous().cuda()
    cofs = torch.randn(N, 128, generator=g)
    cofs[1] *= 40.0                                                     # large logits (both families lose ~1e-5 there)
    cofs[2] *= 1e-3                                                     # tiny coefficients (fp16 lo part underflows)
    cx, cy = torch.rand(N, generator=g) * W * 2, torch.rand(N, generator=g) * H * 2
    bw, bh = torch.rand(N, generator=g) * W * 1.2 + 0.2, torch.rand(N, generator=g) * H * 1.2 + 0.2
    boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).clamp(min=0)
    boxes[0] = torch.tensor([0.0, 0.0, 2.0 * W, 2.0 * H])              # whole image
    boxes[3] = torch.tensor([16.0, 8.0, 48.0, 24.0])                    # integer-aligned in prototype space (x0.5)
    boxes[4] = torch.tensor([30.2, 14.6, 30.9, 15.3])                   # smaller than one prototype pixel
    boxes[5] = torch.tensor([2.0 * W - 40.0, 2.0 * H - 9.0, 2.0 * W + 50.0, 2.0 * H + 50.0])   # hangs over the corner
    oh, ow = 2 * H - 1, 2 * W - 3
    res = {}
    prev = ops.set_mask_tensor_dot(None)
    try:
        for mode in (False, True):
            ops.set_mask_tensor_dot(mode)
            pos = ops.mask_assemble(p_dev, cofs.cuda(), boxes.cuda(), 0.5, layout=layout, out_dtype=torch.float32)
            pos16 = ops.mask_assemble(p_dev, cofs.cuda(), boxes.cuda(), 0.5, layout=layout, out_dtype=torch.float16)
            two = ops.unpack_mask_bits(ops.mask_upsample2_threshold_pack(pos, (oh, ow), 0.4), ow)
            fused = ops.unpack_mask_bits(ops.mask_assemble_pack(p_dev, cofs.cuda(), boxes.cuda(), 0.5, (oh, ow), 0.4, layout=layout), ow)
            fused_sf = ops.unpack_mask_bits(ops.mask_assemble_pack(p_dev, cofs.cuda(), boxes.cuda(), 0.5, (oh, ow), 0.4,
                                                                   layout=layout, up=2.0 / 1.6667), ow)
            res[mode] = [x.cpu().numpy() for x in (pos, pos16.float(), two, fused, fused_sf)]
    finally:
        ops.set_mask_tensor_dot(prev)
    s_pos, s_pos16, s_two, s_fused, s_sf = res[False]
    t_pos, t_pos16, t_two, t_fused, t_sf = res[True]
    # crop geometry is exact (the tensor kernels' sigmoid flushes values below 1.2e-38 to 0, the scalar one keeps denormals)
    assert (t_pos[s_pos == 0] == 0).all() and (t_pos[s_pos > 1e-30] > 0).all()
    big = np.zeros(N, bool)
    big[1] = True
    np.testing.assert_allclose(t_pos[~big], s_pos[~big], atol=3e-6, rtol=0)
    np.testing.assert_allclose(t_pos[big], s_pos[big], atol=2e-4, rtol=0)
    np.testing.assert_allclose(t_pos16, s_pos16, atol=1.5e-3, rtol=0)
    assert (t_fused != t_two).mean() < 1e-5                              # fused == two-step within the tensor family
    assert (t_fused != s_fused).mean() < 2e-5                            # and across families up to threshold ties
    assert (t_sf != s_sf).mean() < 2e-5
    assert t_fused.any() and t_sf.any()


def test_crop_split_operator_matches_oracle():
    from sipmask_b200 import ops
    O, P, cbind = _oracle()
    g = torch.Generator().manual_seed(0)
    data = torch.rand(4, 40, 56, 9, generator=g)
    rois = torch.tensor([[3.2, 4.1, 30.7, 35.2], [0, 0, 56, 40], [10, 10, 10.5, 10.5], [-5, -5, 20, 20], [50, 30, 80, 90],
                         [7, 3, 8, 39], [0.5, 0.5, 1.5, 1.5], [20, 20, 19, 19], [55, 39, 56, 40]])
    ref = O.crop_split(data, rois, 2)
    got = ops.CropSplit(2)(data.cuda(), rois.cuda())
    np.testing.assert_array_equal(got.cpu().numpy(), ref.numpy())
    with pytest.raises(Exception):
        ops.crop_split(data.cuda().permute(0, 2, 1, 3), rois.cuda())       # non-contiguous input raises


@pytest.mark.parametrize('name', ['ref_head_gn4.npz', 'ref_head_ssd2.npz', 'ref_head_gn4_sf.npz', 'ref_head_ssd2_sf.npz'])
def test_postproc_reproduces_reference_fixture(golden_dir, name):
    """Head outputs captured from the unmodified reference python -> device post-processing must give the
    reference's detections (labels / kept boxes bit-exact, masks IoU >= 0.999)."""
    from sipmask_b200 import postproc
    g = dict(np.load(os.path.join(golden_dir, name)))
    nl = len(g['sizes'])
    ssd = bool(g['ssd_flag'])
    cfg = dict(nms_pre=int(g['nms_pre']), score_thr=float(g['score_thr']), nms=dict(type='nms', iou_thr=0.5),
               max_per_img=int(g['max_per_img']))
    sf = g['scale_factor']
    sf = float(sf[0]) if sf.size == 1 else sf
    res = postproc.get_bboxes_single(
        [torch.from_numpy(g['cls%d' % i][0]).cuda() for i in range(nl)],
        [torch.from_numpy(g['bbox%d' % i][0]).cuda() for i in range(nl)],
        [torch.from_numpy(g['ctr%d' % i][0]).cuda() for i in range(nl)],
        [torch.from_numpy(g['cof%d' % i][0]).cuda() for i in range(nl)],
        torch.from_numpy(g['feat_masks'][0]).cuda(), (8, 16, 32, 64, 128),
        tuple(g['img_shape']), tuple(g['ori_shape']), sf, cfg, rescale=True, ssd_flag=ssd,
        cmp_ge=True)    # the fixture was produced on CPU -> nms_cpu.cpp comparator (>=)
    k = int(res['count'])
    assert res['det_labels'][:k].cpu().tolist() == g['det_labels'].tolist()
    np.testing.assert_allclose(res['det_bboxes'][:k].cpu().numpy(), g['det_bboxes'], rtol=1e-6, atol=1e-6)
    masks = res['masks'][:k].cpu().numpy()
    assert masks.shape == g['masks'].shape
    assert _iou(masks, g['masks']).min() >= 0.999


@pytest.mark.parametrize('H,W,up', [(48, 62, 2.0), (48, 62, 2.0 / 1.6667), (50, 64, (2 / 1.3, 2 / 1.7)), (60, 41, 2.0 / 3.1),
                                    (37, 53, 2.0 / 0.8), (272, 272, 2.0)])
def test_mask_resize_matches_torch_interpolate(H, W, up, mask_dot):
    """The general resize (scale_factor != 1, ADVICE r1 high): two-step kernels and the fused kernel against
    F.interpolate(pos_masks, scale_factor=2/scale_factor, mode='bilinear', align_corners=False) > 0.4
    (sipmask_head.py:629-633), both coordinate rules (PyTorch >= 1.6 given-factor, and recompute_scale_factor=True)."""
    import torch.nn.functional as F
    from sipmask_b200 import ops, synth
    O, P, cbind = _oracle()
    g = torch.Generator().manual_seed(H + W)
    N = 23
    protos = synth.prototypes(H, W, seed=3)
    cofs = torch.randn(N, 128, generator=g)
    cx, cy = torch.rand(N, generator=g) * W * 2, torch.rand(N, generator=g) * H * 2
    bw, bh = torch.rand(N, generator=g) * W * 1.5 + 2, torch.rand(N, generator=g) * H * 1.5 + 2
    boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).clamp(min=0)
    boxes[0] = torch.tensor([0.0, 0.0, 2.0 * W, 2.0 * H])
    pos_ref = torch.from_numpy(cbind.mask_assemble(protos.numpy(), cofs.numpy(), (boxes * 0.5).numpy()))
    pos = ops.mask_assemble(protos.cuda(), cofs.cuda(), boxes.cuda(), 0.5, layout='chw')
    sf = tuple(float(u) for u in up) if isinstance(up, tuple) else float(up)
    for legacy in (False, True):
        want = (F.interpolate(pos_ref.unsqueeze(0), scale_factor=sf, mode='bilinear', align_corners=False,
                              recompute_scale_factor=True if legacy else None).squeeze(0) > 0.4).numpy()
        fh, fw = want.shape[1:]
        for (oh, ow) in ((fh, fw), (fh - 3, fw - 5), (fh + 4, fw + 37)):
            canvas = np.zeros((N, oh, ow), bool)
            canvas[:, :min(oh, fh), :min(ow, fw)] = want[:, :min(oh, fh), :min(ow, fw)]
            a = ops.mask_resize_threshold(pos, up, (oh, ow), 0.4, legacy_interp=legacy).cpu().numpy().astype(bool)
            b = ops.unpack_mask_bits(ops.mask_resize_threshold_pack(pos, up, (oh, ow), 0.4, legacy_interp=legacy), ow).cpu().numpy().astype(bool)
            c = ops.unpack_mask_bits(ops.mask_assemble_pack(protos.cuda(), cofs.cuda(), boxes.cuda(), 0.5, (oh, ow), 0.4,
                                                            layout='chw', up=up, legacy_interp=legacy), ow).cpu().numpy().astype(bool)
            c16 = ops.unpack_mask_bits(ops.mask_assemble_pack(protos.half().permute(1, 2, 0).contiguous().cuda(), cofs.cuda(),
                                                              boxes.cuda(), 0.5, (oh, ow), 0.4, layout='hwc', up=up,
                                                              legacy_interp=legacy), ow).cpu().numpy().astype(bool)
            assert _iou(a, canvas).min() >= 0.999, (legacy, oh, ow)
            assert (a != canvas).mean() < 2e-5                      # only pixels whose value sits on the threshold may flip
            assert (a == b).all()                                   # byte and bit-packed outputs are the same kernel math
            assert (c != b).mean() < 1e-5                           # fused == two-step
            assert (c16 != canvas).mean() < 2e-3                    # fp16 prototypes (engine storage type)
