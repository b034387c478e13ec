"""GPU tests (run with -m gpu on an H100): the selection and gather kernels of nms.cu on constructed inputs where such
kernels go wrong (IoU exactly at the threshold, clipped and degenerate boxes, ties at every cut, capacity limits, empty
outputs, extreme logits, the device geometry rows), each checked by oracle/postproc_check.py."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import postproc_check as PC

pytestmark = pytest.mark.gpu
STRIDES = (8, 16, 32, 64, 128)


def _levels_dev(sizes, C, seed, cls_fn=None):
    g = torch.Generator().manual_seed(seed)
    cls, box, ctr = [], [], []
    for (h, w), s in zip(sizes, STRIDES):
        c = torch.randn(h, w, C, generator=g) * 2 - 2
        if cls_fn is not None:
            c = cls_fn(c)
        cls.append(c.cuda())
        box.append(((torch.randn(h, w, 4, generator=g) * 4 * s).abs()).cuda())
        ctr.append(torch.randn(h, w, 1, generator=g).cuda())
    return cls, box, ctr


def _host_levels(cls, box, ctr, box_scales=None):
    return [PC.level_inputs(c, b, t, s, 1.0 if box_scales is None else box_scales[l], 1.0 if box_scales is None else s)
            for l, (c, b, t, s) in enumerate(zip(cls, box, ctr, STRIDES))]


def _record(det, lab, idx, cnt):
    return det.cpu().numpy(), lab.cpu().numpy(), idx.cpu().numpy(), cnt.cpu().numpy()


# ------------------------------------------------------------------------------------------------ IoU at threshold
@pytest.mark.parametrize('thr', [0.5, 0.45, 0.6])
def test_iou_exactly_at_the_threshold(thr):
    from sipmask_b200 import ops
    a, b = PC.threshold_pairs(thr, 1)
    for j, (keep_gt, keep_ge) in enumerate(((True, True), (True, False), (False, False))):   # IoU below, at, above
        d = np.concatenate([np.stack([a[j], b[j]]), [[0.9], [0.8]]], 1).astype(np.float32)
        for ge, want in ((False, keep_gt), (True, keep_ge)):
            _, inds = ops.nms(torch.from_numpy(d).cuda(), thr, cmp_ge=ge)
            assert inds.cpu().tolist() == ([0, 1] if want else [0]), (j, ge)
            boxes, scores, ctr = d[:, :4].copy(), d[:, 4:5].copy(), np.ones(2, np.float32)
            rec = ops.multiclass_nms_idx(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), 0.05, thr, 10,
                                         score_factors=torch.from_numpy(ctr).cuda(), has_bg_column=False, cmp_ge=ge,
                                         return_count_tensor=True)
            assert PC.check_multiclass_nms(boxes, scores, ctr, 2, 0.05, thr, 10, ge, *_record(*rec)) == 1 + int(want)
        # label-aware NMS suppresses at IoU > thr
        rec = ops.ml_nms_topk(torch.from_numpy(d[:, :4].copy()).cuda(), torch.from_numpy(d[:, 4].copy()).cuda(),
                              torch.zeros(2, dtype=torch.int32).cuda(), torch.tensor([2], dtype=torch.int32).cuda(), thr,
                              100, 4)
        assert PC.check_ml_nms(d[:, :4], d[:, 4], np.zeros(2), 2, thr, 100, 4, *_record(*rec[:4]), rec[4].cpu().numpy()) \
            == 1 + int(keep_gt)
    a, b = PC.threshold_pairs(thr, 0)                          # fast NMS keeps IoU <= thr (no +1 in its jaccard)
    for j, want in enumerate((True, True, False)):
        boxes = np.stack([a[j], b[j]]).astype(np.float32)
        scores, ctr = np.float32([[0.9], [0.8]]), np.ones(2, np.float32)
        rec = ops.fast_nms(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(), torch.from_numpy(ctr).cuda(), thr,
                           200, 0.1, 100, return_count_tensor=True)
        assert PC.check_fast_nms(boxes, scores, ctr, 2, 0.1, thr, 200, 100, *_record(*rec)) == 1 + int(want)


# --------------------------------------------------------------------------------------- degenerate and clipped boxes
def test_degenerate_and_clipped_boxes():
    """Boxes outside a 100 x 80 image clamp to its border: fast NMS's jaccard of two of them is 0 / 0 = NaN, and NaN
    drops the later box (torch.max propagates it, the comparison is false); zero-width and zero-area boxes elsewhere."""
    from sipmask_b200 import ops
    lv = PC.level_inputs(np.zeros((1, 4, 1), np.float32), np.float32([[[-500, 10, 500, 10], [-900, -900, 900, 900],
                                                                        [1, 1, 1, 1], [0, 0, 0, 0]]]), np.zeros((1, 4)), 8)
    boxes = PC.decode_boxes(lv, np.arange(4), PC.geometry(80, 100))
    assert (boxes[0, [0, 2]] == 99).all() and (boxes[1] == [99, 79, 99, 79]).all()        # flattened onto the border
    boxes = np.concatenate([boxes, boxes[1:2], [[10, 10, 10, 40], [30, 30, 30, 30], [29, 29, 31, 31]]]).astype(np.float32)
    n = boxes.shape[0]
    scores = np.linspace(0.9, 0.5, n, dtype=np.float32)[:, None].repeat(3, 1)
    ctr = np.ones(n, np.float32)
    with np.errstate(invalid='ignore'):
        assert np.isnan(PC.iou_f32(boxes[1], boxes[4], 0))
    bt, st, ct = (torch.from_numpy(x).cuda() for x in (boxes, scores, ctr))
    rec = ops.fast_nms(bt, st, ct, 0.5, 200, 0.1, 100, return_count_tensor=True)
    PC.check_fast_nms(boxes, scores, ctr, n, 0.1, 0.5, 200, 100, *_record(*rec))
    for ge in (False, True):
        rec = ops.multiclass_nms_idx(bt, st, 0.05, 0.5, 100, score_factors=ct, has_bg_column=False, cmp_ge=ge,
                                     return_count_tensor=True)
        PC.check_multiclass_nms(boxes, scores, ctr, n, 0.05, 0.5, 100, ge, *_record(*rec))
    rec = ops.ml_nms_topk(bt, st[:, 0].contiguous(), torch.zeros(n, dtype=torch.int32).cuda(),
                          torch.tensor([n], dtype=torch.int32).cuda(), 0.6, 100, 16)
    PC.check_ml_nms(boxes, scores[:, 0], np.zeros(n), n, 0.6, 100, 16, *_record(*rec[:4]), rec[4].cpu().numpy())


# ------------------------------------------------------------------------------------------------- ties at the cuts
def test_ties_at_max_num_and_top_k():
    """Equal scores across classes at the max_num cut (radix select of finalize_kernel), at fast NMS's top_k = 200 and its
    final max_num: ties go to the class-major / lower-index entry, as the stable sorts of the oracle order them."""
    from sipmask_b200 import ops
    rng = np.random.RandomState(3)
    n, C = 700, 6
    xy = rng.rand(n, 2).astype(np.float32) * 2000
    boxes = np.concatenate([xy, xy + 8], 1).astype(np.float32)           # sparse: NMS keeps most of them
    scores = np.float32(rng.choice([0.25, 0.5, 0.75], size=(n, C)))
    ctr = np.ones(n, np.float32)
    bt, st, ct = (torch.from_numpy(x).cuda() for x in (boxes, scores, ctr))
    for max_num in (1, 100, 333, 1024):
        rec = ops.multiclass_nms_idx(bt, st, 0.05, 0.5, max_num, score_factors=ct, has_bg_column=False,
                                     return_count_tensor=True)
        PC.check_multiclass_nms(boxes, scores, ctr, n, 0.05, 0.5, max_num, False, *_record(*rec))
    for max_num in (1, 100, 1024):
        rec = ops.fast_nms(bt, st, ct, 0.5, 200, 0.1, max_num, return_count_tensor=True)
        PC.check_fast_nms(boxes, scores, ctr, n, 0.1, 0.5, 200, max_num, *_record(*rec))


def test_capacity_one_class_5120_candidates_max_num_1024():
    from sipmask_b200 import ops
    rng = np.random.RandomState(4)
    n = 5120
    xy = rng.rand(n, 2).astype(np.float32) * 3000
    boxes = np.concatenate([xy, xy + rng.rand(n, 2).astype(np.float32) * 60 + 1], 1).astype(np.float32)
    scores = np.float32(np.round(rng.rand(n, 1) * 64) / 64)              # many ties
    ctr = np.float32(rng.rand(n))
    bt, st, ct = (torch.from_numpy(x).cuda() for x in (boxes, scores, ctr))
    rec = ops.multiclass_nms_idx(bt, st, 0.05, 0.5, 1024, score_factors=ct, has_bg_column=False, return_count_tensor=True)
    assert PC.check_multiclass_nms(boxes, scores, ctr, n, 0.05, 0.5, 1024, False, *_record(*rec), use_c=True) == 1024
    rec = ops.ml_nms_topk(bt, st[:, 0].contiguous(), torch.zeros(n, dtype=torch.int32).cuda(),
                          torch.tensor([n], dtype=torch.int32).cuda(), 0.6, 1000, 1024)
    PC.check_ml_nms(boxes, scores[:, 0], np.zeros(n), n, 0.6, 1000, 1024, *_record(*rec[:4]), rec[4].cpu().numpy())


def test_nothing_above_the_score_threshold():
    """A count of 0: the whole record is the zero / -1 tail."""
    from sipmask_b200 import ops
    boxes = np.float32([[0, 0, 10, 10], [5, 5, 20, 20], [40, 40, 50, 60]])
    scores, ctr = np.full((3, 4), 0.04, np.float32), np.ones(3, np.float32)
    bt, st, ct = (torch.from_numpy(x).cuda() for x in (boxes, scores, ctr))
    rec = ops.multiclass_nms_idx(bt, st, 0.05, 0.5, 100, score_factors=ct, has_bg_column=False, return_count_tensor=True)
    assert PC.check_multiclass_nms(boxes, scores, ctr, 3, 0.05, 0.5, 100, False, *_record(*rec)) == 0
    rec = ops.fast_nms(bt, st, ct, 0.5, 200, 0.1, 100, return_count_tensor=True)
    assert PC.check_fast_nms(boxes, scores, ctr, 3, 0.1, 0.5, 200, 100, *_record(*rec)) == 0
    rec = ops.ml_nms_topk(bt, st[:, 0].contiguous(), torch.zeros(3, dtype=torch.int32).cuda(),
                          torch.tensor([0], dtype=torch.int32).cuda(), 0.6, 100, 8)
    assert PC.check_ml_nms(boxes, scores[:, 0], np.zeros(3), 0, 0.6, 100, 8, *_record(*rec[:4]), rec[4].cpu().numpy()) == 0
    cls, box, ctr_l = _levels_dev([(9, 7), (5, 4)], 3, 0, cls_fn=lambda c: c * 0 - 30.0)
    out = ops.pair_decode_topk(cls, box, ctr_l, STRIDES[:2], (70, 55), nms_pre=1000, score_thr=0.05)
    PC.check_pair_decode(_host_levels(cls, box, ctr_l), 3, 0.05, 1000, PC.geometry(70, 55),
                         *[t.cpu().numpy() for t in out])


# ----------------------------------------------------------------------------------------- candidates: nms_pre, logits
@pytest.mark.parametrize('sizes,nms_pre', [([(40, 36), (32, 32), (20, 51), (1, 1)], 1024),      # larger, equal, smaller
                                           ([(25, 41), (13, 21), (7, 11), (4, 6), (1, 3)], 100)])
def test_decode_topk_at_nms_pre(sizes, nms_pre):
    from sipmask_b200 import ops
    for C in (1, 80):
        cls, box, ctr = _levels_dev(sizes, C, C)
        out = ops.decode_topk(cls, box, ctr, STRIDES[:len(sizes)], (sizes[0][0] * 8 - 5, sizes[0][1] * 8 - 3), nms_pre)
        st = PC.check_candidates(_host_levels(cls, box, ctr), nms_pre,
                                 PC.geometry(sizes[0][0] * 8 - 5, sizes[0][1] * 8 - 3), *[t.cpu().numpy() for t in out])
        print('decode_topk C=%d nms_pre=%d: %d of %d locations of cut levels ambiguous' % (C, nms_pre, st['ambiguous'],
                                                                                          st['cut_locations']))


def test_decode_topk_extreme_and_tied_logits():
    """+-large and +-inf logits, and several classes sharing the maximum logit: the ranking key sigmoid(max) * sigmoid(ctr)
    must equal the max over classes of the products, and equal keys must be listed by ascending location (every key of
    the tied level is equal, so the nms_pre cut takes the first locations)."""
    from sipmask_b200 import ops
    sizes = [(20, 30), (10, 15), (5, 8)]

    def extreme(c):
        c = c.clone()
        c[::3, :, 0] = 1e4
        c[1::3, :, 1] = -1e4
        c[2::7, ::2, 2] = float('inf')
        c[2::5, 1::2, :] = float('-inf')
        c[1::4, :, 3] = c[1::4, :, 4] = c[1::4, :].max(-1).values + 1.0      # two classes share the maximum
        return c
    cls, box, ctr = _levels_dev(sizes, 8, 11, cls_fn=extreme)
    out = ops.decode_topk(cls, box, ctr, STRIDES[:3], (150, 230), 100)
    PC.check_candidates(_host_levels(cls, box, ctr), 100, PC.geometry(150, 230), *[t.cpu().numpy() for t in out], cap=1.0)
    tied = [torch.full_like(c, 1.5) for c in cls]
    ctr_t = [torch.zeros_like(t) for t in ctr]
    out = ops.decode_topk(tied, box, ctr_t, STRIDES[:3], (150, 230), 100)
    PC.check_candidates(_host_levels(tied, box, ctr_t), 100, PC.geometry(150, 230), *[t.cpu().numpy() for t in out], cap=1.0)
    loc = out[3].cpu().numpy()
    assert loc[:100].tolist() == list(range(100)) and loc[100:200].tolist() == list(range(600, 700))


def test_decode_topk_nan_logit():
    """A NaN logit: the kernel's fmaxf skips it when ranking (the location ranks by its other classes) and its score is
    NaN.  The oracle's torch max of products would propagate the NaN into the key instead; the kernel is left as it is,
    and this records what it does."""
    from sipmask_b200 import ops
    cls, box, ctr = _levels_dev([(6, 5)], 4, 2)
    cls[0][0, 0, 2] = float('nan')
    cls[0][0, 0, 1] = 20.0                       # with the NaN skipped, location 0 has the largest key
    ctr[0][0, 0, 0] = 20.0
    out = ops.decode_topk(cls, box, ctr, STRIDES[:1], (48, 40), 10)
    s, loc = out[1].cpu().numpy(), out[3].cpu().numpy()
    q = int(np.flatnonzero(loc == 0)[0])
    assert np.isnan(s[q, 2]) and np.isfinite(np.delete(s, 2, axis=1)).all() and np.isfinite(s[:, 2][loc != 0]).all()
    assert loc[0] == 0


# ------------------------------------------------------------------------------------------------------- entry points
def test_dev_and_host_entry_points_agree_bit_for_bit():
    """smb_decode_topk_dev / smb_pair_decode_topk_dev read the geometry row on the device: same bits as the host-value
    entry points, with an anisotropic scale and an image smaller than the padded input."""
    from sipmask_b200 import _lib as L, ops
    from sipmask_b200.postproc import image_geometry
    sizes = [(24, 32), (12, 16), (6, 8), (3, 4), (2, 2)]
    cls, box, ctr = _levels_dev(sizes, 80, 9)
    sf = np.float32([1.25, 0.8, 1.25, 0.8])
    img = (150, 201)                                              # padded input 192 x 256
    host = ops.decode_topk(cls, box, ctr, STRIDES, img, 200, scale_factor=sf, box_scales=[1.1, 0.9, 1.0, 1.2, 0.7])
    g = image_geometry((48, 64), img + (3,), (120, 161, 3), sf)
    row = ops.geom_row(g, 'cuda')
    lv, keep = ops.level_descs(cls, box, ctr, STRIDES, [1.1, 0.9, 1.0, 1.2, 0.7])
    lib = L.lib()
    ws_bytes = lib.smb_decode_workspace_bytes(5, lv, 200)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    dev = [torch.full_like(t, -1) for t in host]
    L.check(lib.smb_decode_topk_dev(5, lv, 80, 200, L.ptr(row), *[L.ptr(t) for t in dev], L.ptr(ws),
                                    ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_decode_topk_dev')
    for a, b in zip(host, dev):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    PC.check_candidates(_host_levels(cls, box, ctr, [1.1, 0.9, 1.0, 1.2, 0.7]), 200, PC.geometry_from_row(g),
                        *[t.cpu().numpy() for t in dev])
    # the BM pair path
    hostp = ops.pair_decode_topk(cls, box, ctr, STRIDES, img, nms_pre=300, score_thr=0.05, box_scales=[1.1, 0.9, 1.0, 1.2, 0.7])
    n = hostp[0].shape[0]
    ws_bytes = lib.smb_pair_decode_workspace_bytes(5, lv, 80, 300)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device='cuda')
    devp = [torch.full_like(t, -1) for t in hostp]
    L.check(lib.smb_pair_decode_topk_dev(5, lv, 80, ctypes.c_float(0.05), 300, L.ptr(row), *[L.ptr(t) for t in devp], n,
                                         L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_pair_decode_topk_dev')
    for a, b in zip(hostp, devp):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    PC.check_pair_decode(_host_levels(cls, box, ctr, [1.1, 0.9, 1.0, 1.2, 0.7]), 80, 0.05, 300, PC.geometry(*img),
                         *[t.cpu().numpy() for t in devp])


# ------------------------------------------------------------------------------------------------------------ gathers
def test_gather_det_inputs_three_images_odd_levels():
    from sipmask_b200 import _lib as L
    rng = np.random.RandomState(5)
    level_hw = [7 * 9, 5 * 3, 3 * 1, 1 * 5, 1]
    N, tot, pitch, max_rows = 3, sum(level_hw), 144, 40
    src = torch.from_numpy(rng.randn(N * tot, pitch).astype(np.float32)).cuda()
    cof = src[:, 9:9 + 128]
    cand_loc = torch.from_numpy(rng.randint(0, tot, 60).astype(np.int32)).cuda()
    hw = (ctypes.c_int * 5)(*level_hw)
    lib = L.lib()
    for img in range(N):
        for k in (0, 17, max_rows):
            idx = torch.full((max_rows,), -1, dtype=torch.long)
            idx[:k] = torch.from_numpy(rng.choice(60, k, replace=False))
            idx = idx.cuda()
            det = torch.from_numpy(rng.rand(max_rows, 5).astype(np.float32)).cuda()
            cnt = torch.tensor([k], dtype=torch.int32).cuda()
            det_cofs = torch.full((max_rows, 128), float('nan'), device='cuda')
            boxes = torch.full((max_rows, 4), float('nan'), device='cuda')
            loc_kept = torch.full((max_rows,), -7, dtype=torch.long, device='cuda')
            L.check(lib.smb_gather_det_inputs(L.ptr(cof), cof.stride(0), L.ptr(cand_loc), L.ptr(idx), L.ptr(det), L.ptr(cnt),
                                              max_rows, 128, L.ptr(det_cofs), L.ptr(boxes), L.ptr(loc_kept), 5, hw, N, img,
                                              L.stream_ptr()), 'smb_gather_det_inputs')
            PC.check_gather_cofs(cof.cpu().numpy(), cand_loc.cpu().numpy(), idx.cpu().numpy(), det.cpu().numpy(), k,
                                 level_hw, N, img, det_cofs.cpu().numpy(), boxes.cpu().numpy(), loc_kept.cpu().numpy())


def test_gather_track_feats_on_cell_edges_and_off_the_map():
    from sipmask_b200 import _lib as L, ops
    from sipmask_b200.postproc import image_geometry
    h, w, C = 9, 13, 512
    track = torch.randn(h, w, C, generator=torch.Generator().manual_seed(6)).cuda()
    e = np.nextafter(np.float32(24), np.float32(0))
    det = np.float32([[8, 8, 24, 24, 1], [8, 8, e, e, 1], [-90, -90, -70, -70, 1], [500, 500, 900, 900, 1],
                      [0, 0, 0, 0, 1], [103, 71, 105, 72, 1], [np.inf, 0, np.inf, 0, 1], [4, 4, 4, 4, 1]])
    sf = np.float32([1.25, 0.8, 1.25, 0.8])
    g = image_geometry((36, 52), (100, 130, 3), (125, 104, 3), sf)
    row = ops.geom_row(g, 'cuda')
    dt = torch.from_numpy(det).cuda()
    for k in (0, 5, 8):
        cnt = torch.tensor([k], dtype=torch.int32).cuda()
        out = torch.full((8, C), float('nan'), device='cuda')
        L.check(L.lib().smb_gather_track_feats_dev(L.ptr(track), h, w, C, L.ptr(dt), L.ptr(cnt), 8, L.ptr(row),
                                                   ctypes.c_float(8.0), L.ptr(out), L.stream_ptr()), 'smb_gather_track_feats_dev')
        PC.check_gather_track(track.cpu().numpy(), det, k, g.track_sx, g.track_sy, 8.0, out.cpu().numpy())
        host = ops.gather_track_feats(track, dt, cnt, scale_factor=sf[:2], feat_stride=8.0)
        assert torch.equal(host.view(torch.int32), out.view(torch.int32))
