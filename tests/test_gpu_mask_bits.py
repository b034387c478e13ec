"""Every mask bit of every mask entry point against the float64 reference of oracle/numerics.py (run with -m gpu).

A bit may differ from the reference only where the reference value lies within its proven error bound of the threshold;
those ambiguous pixels are counted and capped.  Every dense value must lie within its bound.  The planes past the valid
frame, past out_w inside the last word and past the detection count must be zero."""
import numpy as np
import pytest
import torch

from oracle import numerics as NU

pytestmark = pytest.mark.gpu

THR = 0.4


def _quotient_rois(rng):
    """Two float32 rois found by search: one with an in-map pixel w where float32(w - x1) == roi_w exactly (cell quotient
    exactly 1), one where float32(w - x1) / roi_w rounds to 2 (x1 far left, where float32 spacing exceeds the +0.1 of
    roi_w): the tensor-core kernels' cold path."""
    f32 = np.float32
    one = None
    for c in (f32(2.25), f32(3.5), f32(5.125), f32(7.75)):
        w = f32(9.0)
        x1 = f32(w - c)
        d = f32(2.0 * c - 0.1)
        for _ in range(64):
            x2 = f32(x1 + d)
            rw = f32((np.float64(f32(x2 - x1)) + 0.1) / 2)
            if rw == c and f32(w - x1) == c and w < x2:
                one = (x1, x2)
                break
            d = np.nextafter(d, f32(1e9)) if rw < c else np.nextafter(d, f32(0))
        if one is not None:
            break
    assert one is not None
    x1 = -rng.uniform(2.0 ** 21, 2.0 ** 23, 4096).astype(np.float32)
    x2 = rng.uniform(3.0, 30.0, 4096).astype(np.float32)
    rw = ((np.float64(1) * (x2 - x1).astype(np.float32) + 0.1) / 2).astype(np.float32)
    a = ((np.ceil(x2) - 1).astype(np.float32) - x1).astype(np.float32)
    k = int(np.nonzero((a / rw).astype(np.float32) >= 2)[0][0])
    return one, (x1[k], x2[k])


def _boxes(H, W, N, g, rng):
    """Image-space boxes (rois = boxes * 0.5): random ones plus the edge cases, zero rows at the end like the engine's
    rows past the count, and with N > 128 a cluster of up to 130 boxes over the first 8 x 64 tile."""
    cx, cy = torch.rand(N, generator=g) * W * 2, torch.rand(N, generator=g) * H * 2
    bw, bh = torch.rand(N, generator=g) * W * 1.3 + 0.2, torch.rand(N, generator=g) * H * 1.3 + 0.2
    b = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1)
    if N > 128:
        k = torch.arange(min(130, N - 10), dtype=torch.float32)
        b[8:8 + k.numel()] = torch.stack([4 + k % 7, 2 + k % 5, 2.0 * min(W, 60) - k % 11, 2.0 * min(H, 14) - k % 3], 1)
    (q1x1, q1x2), (q2x1, q2x2) = _quotient_rois(rng)
    seam = 64.0 if W > 70 else 8.0
    special = [[0.0, 0.0, 2.0 * W, 2.0 * H],                                      # whole image
               [2.0 * (W // 3) - 0.6, 2.0 * (H // 2) - 0.5, 2.0 * (W // 3) + 0.4, 2.0 * (H // 2) + 0.3],   # sub-pixel
               [2.0 * seam, 16.0, 2.0 * min(W, seam + 64), 2.0 * max(H - 1, 9)],  # integer roi edges on tile seams
               [2.0 * W - 40.0, 2.0 * H - 9.0, 2.0 * W + 50.0, 2.0 * H + 50.0],  # hangs over the far corner
               [-30.0, -11.0, 0.7 * W, 25.0],                                     # negative
               [40.0, 10.0, 40.0, 30.0],                                         # x2 == x1
               [2.0 * q1x1, 0.0, 2.0 * q1x2, 2.0 * H],                           # cell quotient exactly 1
               [2.0 * q2x1, -3.0, 2.0 * q2x2, 2.0 * H + 3.0]]                    # cell quotient 2: cold path
    for i, s in enumerate(special[:N]):
        b[i] = torch.tensor(s)
    if N > 10:
        b[-2:] = 0.0                                                            # the engine's rows past the count
    return b


def _cofs(N, g, kind):
    c = torch.randn(N, 128, generator=g)
    if N > 2:
        c[1] *= 40.0                                                           # steep logits
        c[2] *= 1e-3                                                           # tiny coefficients (fp16 lo underflows)
    if kind == 'big':
        c[0] = (torch.randn(128, generator=g) * 3e4).clamp(-1e5, 1e5)           # beyond the fp16 range
    return c


def _canvas(fh, fw, kind, rem):
    oh = {'eq': fh, 'small': fh - 3, 'big': fh + 5}[kind]
    if kind == 'eq':
        return oh, fw
    ow = fw - 1 if kind == 'small' else fw + 1
    while ow % 32 != rem:
        ow += -1 if kind == 'small' else 1
    return oh, ow


F16, F32 = torch.float16, torch.float32
# (H, W, N, prototype dtype, layout, up, legacy interpolation, canvas, out_w % 32, coefficients)
CASES = [
    (2, 40, 3, F16, 'hwc', 2.0, False, 'eq', 0, 'mix'),
    (9, 70, 5, F32, 'chw', 2.0 / 1.6667, True, 'small', 31, 'mix'),
    (9, 70, 4, F16, 'chw', 2.5, False, 'big', 1, 'mix'),
    (37, 53, 129, F16, 'hwc', (2 / 1.3, 2 / 1.7), False, 'small', 1, 'mix'),
    (37, 53, 1, F32, 'hwc', 2.0 / 3.1, True, 'big', 0, 'mix'),
    (100, 168, 128, F16, 'hwc', 0.25, False, 'big', 31, 'mix'),
    (100, 168, 127, F32, 'chw', 2.0, True, 'small', 0, 'mix'),
    (136, 136, 200, F16, 'chw', 2.0 / 1.6667, False, 'big', 0, 'mix'),
    (136, 136, 3, F16, 'hwc', 0.25, True, 'small', 1, 'mix'),
    (400, 672, 20, F16, 'hwc', 2.0, False, 'small', 31, 'mix'),
    (400, 672, 5, F32, 'chw', (2 / 1.3, 2 / 1.7), True, 'eq', 0, 'mix'),
    (37, 53, 5, F16, 'hwc', 2.0 / 3.1, True, 'eq', 0, 'big'),
    (40, 64, 5, F16, 'chw', 2.0, False, 'small', 1, 'big'),
]


def _ids(c):
    H, W, N, dt, lay, up, leg, cv, rem, ck = c
    return '%dx%d-N%d-%s-%s-up%s-%s-%s%d-%s' % (H, W, N, 'f16' if dt == F16 else 'f32', lay,
                                                'x'.join('%.3g' % u for u in (up if isinstance(up, tuple) else (up,))),
                                                'legacy' if leg else 'given', cv, rem, ck)


def _geom_row(H, W, full, r, out_hw, dev):
    from sipmask_b200 import _lib as L, ops
    g = L.ImgGeom()
    g.roi_scale[:] = [0.5] * 4
    g.full_h, g.full_w = full
    g.ry, g.rx = r
    g.out_h, g.out_w = out_hw
    return ops.geom_row(g, dev)


@pytest.mark.parametrize('case', CASES, ids=[_ids(c) for c in CASES])
def test_mask_bits_equal_the_float64_reference(case):
    from sipmask_b200 import ops
    from sipmask_b200.postproc import fused_mask_tile
    H, W, N, dt, layout, up, legacy, cv, rem, ck = case
    g = torch.Generator().manual_seed(H * 1000 + W + N)
    rng = np.random.RandomState(H + N)
    protos = torch.relu(torch.randn(32, H, W, generator=g))
    if ck == 'big':
        protos *= 0.01                                                         # small prototypes: finite logits
    protos = protos.to(dt)
    cofs, boxes = _cofs(N, g, ck), _boxes(H, W, N, g, rng)
    p_dev = (protos if layout == 'chw' else protos.permute(1, 2, 0)).contiguous().cuda()
    c_dev, b_dev = cofs.cuda(), boxes.cuda()
    fh, fw, ry, rx = ops.resize_spec(H, W, up, legacy)
    r = (NU.resize_step(H, fh, ry), NU.resize_step(W, fw, rx))
    oh, ow = _canvas(fh, fw, cv, rem)
    assert ow % 32 == (rem if cv != 'eq' else fw % 32)
    words = (ow + 31) // 32
    cap = (oh + 3, ow + 40)
    steep = (max(r[0], 2.0), max(r[1], 2.0))
    fused_mask_tile(*steep, proto_bytes=64 if dt == F16 else 128)
    prev = ops.set_mask_tensor_dot(None)
    lines = []
    try:
        for family in (('scalar', 'tensor') if dt == F16 else ('scalar',)):
            ops.set_mask_tensor_dot(family == 'tensor')
            what = '%s %s' % (_ids(case), family)
            vals = NU.mask_values(protos, cofs, boxes, 0.5, family)
            pos = ops.mask_assemble(p_dev, c_dev, b_dev, 0.5, layout=layout, out_dtype=torch.float32)
            pos16 = ops.mask_assemble(p_dev, c_dev, b_dev, 0.5, layout=layout, out_dtype=torch.float16)
            v32 = NU.check_mask_values(pos, vals, what + ' mask_assemble fp32')
            v16 = NU.check_mask_values(pos16, vals, what + ' mask_assemble fp16')
            ref = NU.resize_reference(vals, H, W, (fh, fw), r, (oh, ow), THR, proto_bytes=64 if dt == F16 else 128)
            fused = ops.mask_assemble_pack(p_dev, c_dev, b_dev, 0.5, (oh, ow), THR, layout=layout, up=up, legacy_interp=legacy)
            st = NU.check_mask_bits(fused, ref, N, what=what + ' mask_assemble_pack')
            row = _geom_row(H, W, (fh, fw), r, (oh, ow), p_dev.device)
            dev_bits = [ops.mask_assemble_pack_dev(p_dev, c_dev, b_dev, row, t, cap, THR, layout=layout) for t in (r, steep)]
            assert torch.equal(dev_bits[0], dev_bits[1]), what + ': the device-row bits depend on the tile'
            NU.check_mask_bits(dev_bits[0], ref, N, what=what + ' mask_assemble_pack_dev', tile_r=r)
            assert torch.equal(dev_bits[0][:, :oh, :words], fused), what + ': device row and host arguments differ'
            # two-step: the resize kernels on the dense masks they are given (teacher forcing)
            for p in ((pos, pos16) if H * W <= 20000 else (pos,)):
                ref2 = NU.resize_reference(NU.dense_values(p), H, W, (fh, fw), r, (oh, ow), THR)
                packed = ops.mask_resize_threshold_pack(p, up, (oh, ow), THR, legacy_interp=legacy)
                s2 = NU.check_mask_bits(packed, ref2, N, what='%s mask_resize_threshold_pack %s' % (what, p.dtype))
                u8 = ops.mask_resize_threshold(p, up, (oh, ow), THR, legacy_interp=legacy).cpu().numpy().astype(bool)
                pad = np.zeros((N, oh, words * 32), bool)
                pad[:, :, :ow] = u8
                as_bits = np.packbits(pad, axis=-1, bitorder='little').view(np.int32).reshape(N, oh, words)
                NU.check_mask_bits(as_bits, ref2, N, what='%s mask_resize_threshold %s' % (what, p.dtype))
            lines.append('%s: dense err/bound fp32 %.3f fp16 %.3f; fused ambiguous %.2e of %d px (margin %.3g); two-step '
                         'ambiguous %.2e' % (what, v32, v16, st['ambiguous'], st['pixels'], st['margin'], s2['ambiguous']))
    finally:
        ops.set_mask_tensor_dot(prev)
    print('\n'.join(lines))


def test_engine_batch_with_three_image_metas():
    """One batch-3 SSD engine, three images of different original sizes and per-axis scale factors, the fused mask tile
    sized for a steeper resize than any of them: each image's bit planes, over the whole capacity of the record, against
    the reference computed from the engine's own prototypes, coefficients, rois, geometry row and count."""
    from sipmask_b200 import _lib as L, ops, synth
    from sipmask_b200.engine import SipMaskEngine
    from sipmask_b200.serving import image_meta
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, cls_bias=-2.5)
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
    metas = []
    for h, w in ((427, 640), (640, 480), (300, 353)):
        img_shape, _, sf = image_meta(h, w, (544, 544), keep_ratio=False)
        metas.append((img_shape, (h, w, 3), sf))
    eng = SipMaskEngine(sd, (544, 544), batch=3, depth=50, stacked_convs=2, gn=False, ssd_flag=True, test_cfg=cfg,
                        max_ori_hw=(640, 640), min_mask_up=0.4, use_graph=True)
    eng.set_image_meta(metas)
    imgs = torch.cat([synth.synthetic_image(544, 544, seed=60 + i) for i in range(3)]).cuda()
    eng.forward(imgs)
    torch.cuda.synchronize()
    family = 'tensor' if ops.set_mask_tensor_dot(None) else 'scalar'
    total = 0
    for n in range(3):
        gm = L.ImgGeom.from_buffer_copy(eng.geom[n].cpu().numpy().tobytes())
        assert gm.ry < eng.mask_tile_r[0] and gm.rx < eng.mask_tile_r[1]
        k = int(eng.count[n])
        total += k
        protos = eng.protos[n].permute(2, 0, 1).cpu()
        ref = NU.mask_reference(protos, eng.det_cofs[n, :k].cpu(), eng.det_boxes4[n, :k].cpu(), list(gm.roi_scale),
                                (gm.full_h, gm.full_w), (gm.ry, gm.rx), (gm.out_h, gm.out_w), eng.mask_thr, family)
        st = NU.check_mask_bits(eng.mask_bits[n], ref, k, what='engine image %d' % n, tile_r=eng.mask_tile_r)
        print('image %d (%dx%d, %d masks): ambiguous %.2e, margin %.3g' % (n, gm.out_h, gm.out_w, k, st['ambiguous'],
                                                                        st['margin']))
    assert total > 0
