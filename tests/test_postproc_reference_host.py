"""Host tests of the post-processing checkers (oracle/postproc_check.py): the restatements agree with the oracle, the
constructed edge inputs hit their edges, and every checker rejects deliberately wrong outputs with a message that names
the field and the index."""
import numpy as np
import pytest
import torch

from oracle import postproc_check as PC

SIZES = [(12, 16), (6, 8), (3, 4), (2, 2), (1, 1)]
STRIDES = (8, 16, 32, 64, 128)


def _levels(seed=3, sizes=SIZES, C=80):
    from sipmask_b200 import synth
    cls, box, ctr, _ = synth.head_level_inputs(sizes, num_classes=C, seed=seed)
    return [PC.level_inputs(c.permute(1, 2, 0), b.permute(1, 2, 0), t.permute(1, 2, 0), s)
            for c, b, t, s in zip(cls, box, ctr, STRIDES)], (cls, box, ctr)


def test_sigmoid_interval_holds_the_float64_sigmoid_and_is_tight():
    x = np.float32(np.concatenate([np.linspace(-110, 110, 44001), [0.0, 87.0, 88.7, 89.0, -87.0, -88.7, -89.0, -104.0,
                                                                   1e-30, -1e-30, 3e38, -3e38]]))
    lo, hi = PC.sigmoidf_interval(x)
    for s in (PC.sigmoid_f32(x), torch.sigmoid(torch.from_numpy(x)).numpy().astype(np.float64)):
        assert ((s >= lo) & (s <= hi)).all()
    inner = np.abs(x) <= 85                                  # beyond, the float64 value is below the float32 range
    s = PC.sigmoid64(x[inner])
    assert ((s >= lo[inner]) & (s <= hi[inner])).all()
    mid = np.abs(x) <= 20
    s = PC.sigmoid64(x[mid])
    assert ((hi[mid] - lo[mid]) / s).max() < 60 * 2.0 ** -23            # (2 + 1.173 * 20) ulp plus the two roundings
    lo, hi = PC.sigmoidf_interval(np.float32([np.inf, -np.inf, np.nan]))
    assert lo[0] == hi[0] == 1.0 and lo[1] == hi[1] == 0.0 and np.isnan(lo[2]) and np.isnan(hi[2])


@pytest.mark.parametrize('thr,one', [(0.5, 1), (0.5, 0), (0.6, 1), (0.45, 1)])
def test_threshold_pairs_hit_the_threshold(thr, one):
    a, b = PC.threshold_pairs(thr, one)
    t = np.float32(thr)
    v = PC.iou_f32(a, b, one)
    assert v[1] == t and v[0] == np.nextafter(t, np.float32(0)) and v[2] == np.nextafter(t, np.float32(1))
    # and the oracle's own NMS sees the same three IoUs: kept / suppressed flips at the comparator
    from oracle import ops as O
    if one == 1:
        for j, (gt, ge) in enumerate(((1, 1), (1, 0), (0, 0))):
            d = np.concatenate([np.stack([a[j], b[j]]), [[0.9], [0.8]]], 1).astype(np.float32)
            assert len(O.nms(d, thr, cmp_ge=False)) == 1 + gt
            assert len(O.nms(d, thr, cmp_ge=True)) == 1 + ge


def test_decode_reference_agrees_with_the_oracle():
    """The oracle's decode (torch sigmoid, max of products, stable sort) passes check_candidates, and the host emulation
    of the kernels selects the same locations with the same boxes."""
    from oracle import postproc as P
    levels, (cls, box, ctr) = _levels()
    img = (90, 125)
    rb, rs, rc, _, ridx = P.decode_candidates(cls, box, ctr, [torch.zeros(128, h, w) for h, w in SIZES], STRIDES,
                                              img + (3,), 60)
    geom = PC.geometry(*img)
    st = PC.check_candidates(levels, 60, geom, rb.numpy(), rs.numpy(), rc.numpy(), ridx.numpy())
    assert st['cut_locations'] == 12 * 16 and st['ambiguous'] <= 2
    eb, es, ec, el = PC.emulate_decode_topk(levels, 60, geom)
    assert el.tolist() == ridx.tolist()
    assert (eb.view(np.uint32) == rb.numpy().view(np.uint32)).all()


def _emulated(scale=(1.0, 1.0, 1.0, 1.0)):
    levels, _ = _levels()
    geom = PC.geometry(90, 125, scale)
    return levels, geom, [x.copy() for x in PC.emulate_decode_topk(levels, 60, geom)]


def test_check_candidates_accepts_the_emulation_with_anisotropic_scale():
    levels, geom, (b, s, c, l) = _emulated((1.25, 0.8, 1.25, 0.8))
    PC.check_candidates(levels, 60, geom, b, s, c, l)


def test_check_candidates_rejects_a_swap_of_disjoint_neighbours():
    levels, geom, (b, s, c, l) = _emulated()
    klo, khi = PC.key_intervals(levels[0])
    sel = l[:60]
    j = next(j for j in range(59) if klo[sel[j]] > khi[sel[j + 1]])
    for t in (b, s, c, l):
        t[[j, j + 1]] = t[[j + 1, j]]
    with pytest.raises(PC.CheckError, match=r'decode_topk: loc\[%d\]' % (j + 1)):
        PC.check_candidates(levels, 60, geom, b, s, c, l)


def test_check_candidates_rejects_a_candidate_one_past_the_cut():
    levels, geom, (b, s, c, l) = _emulated()
    lv = levels[0]
    key = PC.f32(PC.sigmoid_f32(lv['cls'].max(1)) * PC.sigmoid_f32(lv['ctr']))
    order = np.lexsort((np.arange(key.size), -key.astype(np.float64)))
    klo, khi = PC.key_intervals(lv)
    assert khi[order[60]] < klo[order[58]]            # the 61st is surely below the 59th: dropping the 60th is a choice
    nb, ns, nc, nl = PC.emulate_decode_topk([lv], 0, geom)
    i = order[60]
    b[59], s[59], c[59], l[59] = nb[i], ns[i], nc[i], i
    with pytest.raises(PC.CheckError, match=r'decode_topk: loc\[\d+\] .*(cut|order)'):
        PC.check_candidates(levels, 60, geom, b, s, c, l)


def test_check_candidates_rejects_x_divided_by_the_y_scale():
    levels, geom, (b, s, c, l) = _emulated((1.25, 0.8, 1.25, 0.8))
    wrong = PC.geometry(90, 125, (0.8, 0.8, 1.25, 0.8))
    b0 = PC.emulate_decode_topk(levels, 60, wrong)[0]
    q = int(np.flatnonzero(b0[:, 0] != b[:, 0])[0])
    with pytest.raises(PC.CheckError, match=r'decode_topk: boxes\[%d\]' % q):
        PC.check_candidates(levels, 60, geom, b0, s, c, l)


def test_check_candidates_rejects_a_score_outside_the_sigmoid_bound():
    levels, geom, (b, s, c, l) = _emulated()
    s[7, 3] = np.nextafter(np.nextafter(s[7, 3], np.float32(2)), np.float32(2)) * np.float32(1 + 2 ** -10)
    with pytest.raises(PC.CheckError, match=r'decode_topk: scores\[\(7, 3\)\]'):
        PC.check_candidates(levels, 60, geom, b, s, c, l)


def _gather_case():
    rng = np.random.RandomState(0)
    level_hw = [35, 12, 6, 2, 1]
    tot, N, img = sum(level_hw), 3, 1
    cof_src = rng.randn(N * tot, 40).astype(np.float32)
    cand_loc = rng.randint(0, tot, size=50).astype(np.int32)
    idx = np.full(16, -1, np.int64)
    idx[:9] = rng.choice(50, 9, replace=False)
    det = rng.rand(16, 5).astype(np.float32)
    det[9:] = 0
    k = np.int32(9)
    loc = cand_loc[idx[:9]].astype(np.int64)
    rows = PC.cof_row(loc, level_hw, N, img)
    det_cofs = np.zeros((16, 40), np.float32)
    det_cofs[:9] = cof_src[rows]
    boxes = np.zeros((16, 4), np.float32)
    boxes[:9] = det[:9, :4]
    loc_kept = np.full(16, -1, np.int64)
    loc_kept[:9] = loc
    return cof_src, cand_loc, idx, det, k, level_hw, N, img, det_cofs, boxes, loc_kept


def test_cof_row_is_the_level_major_image_inside_level_layout():
    level_hw, N = [35, 12, 6, 2, 1], 3
    table = np.arange(N * sum(level_hw))                   # row r of the buffer
    off = 0
    for l, hw in enumerate(level_hw):
        for img in range(N):
            for i in range(hw):
                loc = sum(level_hw[:l]) + i
                assert PC.cof_row(loc, level_hw, N, img) == table[off + img * hw + i]
        off += N * hw
    assert PC.cof_row(17, None, 1, 0) == 17


def test_check_gather_cofs_rejects_the_neighbouring_image_and_a_nonzero_tail():
    case = _gather_case()
    PC.check_gather_cofs(*case)
    cof_src, cand_loc, idx, det, k, level_hw, N, img, det_cofs, boxes, loc_kept = case
    wrong = det_cofs.copy()
    wrong[4] = cof_src[PC.cof_row(int(cand_loc[idx[4]]), level_hw, N, img + 1)]
    with pytest.raises(PC.CheckError, match=r'gather_cofs: det_cofs\[\(4, 0\)\]'):
        PC.check_gather_cofs(cof_src, cand_loc, idx, det, k, level_hw, N, img, wrong, boxes, loc_kept)
    tail = boxes.copy()
    tail[12, 2] = 1.0
    with pytest.raises(PC.CheckError, match=r'gather_cofs: det_boxes\[\(12, 2\)\]'):
        PC.check_gather_cofs(cof_src, cand_loc, idx, det, k, level_hw, N, img, det_cofs, tail, loc_kept)
    lk = loc_kept.copy()
    lk[10] = 0
    with pytest.raises(PC.CheckError, match=r'gather_cofs: loc_kept\[10\]'):
        PC.check_gather_cofs(cof_src, cand_loc, idx, det, k, level_hw, N, img, det_cofs, boxes, lk)


def test_track_cells_on_cell_edges_and_off_the_map():
    # centre exactly on a cell edge (x = 16: cell 2), just below it, and off the map on every side
    det = np.float32([[8, 8, 24, 24, 1], [8, 8, np.nextafter(np.float32(24), np.float32(0)), 24, 1],
                      [-90, -90, -70, -70, 1], [500, 500, 900, 900, 1], [0, 0, 0, 0, 1]])
    cy, cx = PC.track_cells(det, 1.0, 1.0, 8.0, 10, 12)
    assert cx.tolist() == [2, 1, 0, 11, 0] and cy.tolist() == [2, 2, 0, 9, 0]
    cy, cx = PC.track_cells(det[:1], 2.0, 0.5, 8.0, 10, 12)          # per-axis scale factors
    assert cx.tolist() == [4] and cy.tolist() == [1]


def test_check_gather_track_rejects_a_wrong_cell_and_a_nonzero_tail():
    rng = np.random.RandomState(1)
    track = rng.randn(10, 12, 6).astype(np.float32)
    det = (rng.rand(8, 5) * 100).astype(np.float32)
    cy, cx = PC.track_cells(det[:5], 1.5, 0.75, 8.0, 10, 12)
    out = np.zeros((8, 6), np.float32)
    out[:5] = track[cy, cx]
    PC.check_gather_track(track, det, 5, 1.5, 0.75, 8.0, out)
    with pytest.raises(PC.CheckError, match=r'gather_track: out\[\(\d, 0\)\]'):
        PC.check_gather_track(track, det, 5, 0.75, 1.5, 8.0, out)    # the axes' factors swapped
    out[6, 1] = 1.0
    with pytest.raises(PC.CheckError, match=r'gather_track: out\[\(6, 1\)\]'):
        PC.check_gather_track(track, det, 5, 1.5, 0.75, 8.0, out)


def _record(d, lab, idx, cap):
    k = d.shape[0]
    det = np.zeros((cap, 5), np.float32)
    det[:k] = d
    L = np.full(cap, -1, np.int64)
    L[:k] = lab
    I = np.full(cap, -1, np.int64)
    I[:k] = idx
    return det, L, I, np.int32(k)


def test_check_multiclass_nms_rejects_gt_for_ge_and_a_nonzero_tail():
    from oracle import ops as O
    a, b = PC.threshold_pairs(0.5, 1)
    boxes = np.concatenate([a[1:2], b[1:2], [[200, 200, 240, 230]]]).astype(np.float32)
    scores = np.float32([[0.9, 0.01], [0.8, 0.7], [0.6, 0.2]])
    ctr = np.float32([1.0, 1.0, 0.5])
    bg = torch.from_numpy(np.concatenate([np.zeros((3, 1), np.float32), scores], 1))
    rec = {}
    for ge in (False, True):
        rb, rl, ri = O.multiclass_nms_idx(torch.from_numpy(boxes), bg, 0.05, 0.5, 10, score_factors=torch.from_numpy(ctr),
                                          cmp_ge=ge)
        rec[ge] = _record(rb.numpy(), rl.numpy(), ri.numpy(), 10)
    assert int(rec[False][3]) == int(rec[True][3]) + 1              # the at-threshold pair decides one detection
    PC.check_multiclass_nms(boxes, scores, ctr, 3, 0.05, 0.5, 10, True, *rec[True])
    with pytest.raises(PC.CheckError, match=r'nms: count is 5, expected 4'):
        PC.check_multiclass_nms(boxes, scores, ctr, 3, 0.05, 0.5, 10, True, *rec[False])
    det, lab, idx, k = rec[True]
    det = det.copy()
    det[7, 4] = 0.5
    with pytest.raises(PC.CheckError, match=r'nms: det\[7\] past the count'):
        PC.check_multiclass_nms(boxes, scores, ctr, 3, 0.05, 0.5, 10, True, det, lab, idx, k)
    lab = lab.copy()
    lab[9] = 0
    with pytest.raises(PC.CheckError, match=r'nms: labels\[9\] past the count'):
        PC.check_multiclass_nms(boxes, scores, ctr, 3, 0.05, 0.5, 10, True, rec[True][0], lab, idx, k)


def test_check_fast_and_ml_nms_accept_their_oracles_and_reject_a_swap():
    from oracle import benchmark as B, ops as O
    rng = np.random.RandomState(2)
    n = 300
    xy = rng.rand(n, 2) * 100
    boxes = np.concatenate([xy, xy + rng.rand(n, 2) * 40 + 1], 1).astype(np.float32)
    scores = rng.rand(n, 4).astype(np.float32)
    ctr = rng.rand(n).astype(np.float32)
    s = torch.from_numpy(PC.f32(scores * ctr[:, None]).T.copy())
    rd, rl, _, ri = O.fast_nms(torch.from_numpy(boxes), s, torch.zeros(n, 1), 0.5, 200, 0.1, 100)
    rec = _record(rd.numpy(), rl.numpy(), ri.numpy(), 100)
    PC.check_fast_nms(boxes, scores, ctr, n, 0.1, 0.5, 200, 100, *rec)
    det, lab, idx, k = (x.copy() for x in rec)
    idx[[3, 4]] = idx[[4, 3]]
    with pytest.raises(PC.CheckError, match=r'nms: idx\[3\]'):
        PC.check_fast_nms(boxes, scores, ctr, n, 0.1, 0.5, 200, 100, det, lab, idx, k)
    labels = rng.randint(0, 3, n).astype(np.int32)
    sc = rng.rand(n).astype(np.float32)
    keep = B.kth_value_cut(sc, B.ml_nms(boxes, sc, labels, 0.6), 50)
    rec = _record(np.concatenate([boxes[keep], sc[keep, None]], 1)[:50], labels[keep][:50], keep[:50], 50)
    PC.check_ml_nms(boxes, sc, labels, n, 0.6, 50, 50, *rec, len(keep))
    with pytest.raises(PC.CheckError, match=r'nms: kept_total'):
        PC.check_ml_nms(boxes, sc, labels, n, 0.6, 50, 50, *rec, len(keep) + 1)


def test_pair_reference_matches_the_benchmark_oracle():
    """pair_reference on relu'd, stride-scaled distances (box_scale = 1, box_mul = 1) is oracle.benchmark.pair_candidates."""
    from oracle import benchmark as B
    sizes = [(9, 11), (5, 6), (3, 3)]
    levels, (cls, box, ctr) = _levels(seed=4, sizes=sizes, C=6)
    for lv in levels:
        lv['cls'] = lv['cls'] + np.float32(3.0)                     # many pairs pass, so the nms_pre cut is exercised
    cls = [c + 3.0 for c in cls]
    rb, rs, rl, rloc = PC.pair_reference(levels, 6, 0.05, 40, PC.geometry(70, 85))
    ob, os_, ol, oloc = B.pair_candidates(cls, box, ctr, STRIDES[:3], (70, 85), 0.05, 40)
    assert rloc.tolist() == oloc.tolist() and rl.tolist() == ol.tolist()
    assert (rb.view(np.uint32) == ob.view(np.uint32)).all() and (rs.view(np.uint32) == os_.view(np.uint32)).all()
    slots = rb.shape[0] + 5
    boxes = np.zeros((slots, 4), np.float32)
    boxes[:rb.shape[0]] = rb
    scores = np.zeros(slots, np.float32)
    scores[:rb.shape[0]] = rs
    labels = np.full(slots, -1, np.int32)
    labels[:rb.shape[0]] = rl
    loc = np.full(slots, -1, np.int32)
    loc[:rb.shape[0]] = rloc
    PC.check_pair_decode(levels, 6, 0.05, 40, PC.geometry(70, 85), boxes, scores, labels, loc, rb.shape[0])
    scores[-1] = 1.0
    with pytest.raises(PC.CheckError, match=r'decode_topk: scores\[4\]'):
        PC.check_pair_decode(levels, 6, 0.05, 40, PC.geometry(70, 85), boxes, scores, labels, loc, rb.shape[0])
