"""SipMask-benchmark path on the GPU (-m gpu): the pair selection and label-aware NMS kernels bit-exact against
oracle/benchmark.py, and the BM engine against the oracle network and post-processor.

Tolerances: network outputs as tests/test_gpu_engine.py (fp16 storage, relative L2 <= 2e-2); post-processing given the
engine's own head outputs: kept indices / labels exact, boxes within 1e-5, mask IoU >= 0.999."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

STRIDES = (8, 16, 32, 64, 128)


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _pyramid(H, W):
    sizes = []
    for s in STRIDES:
        sizes.append(((H + s - 1) // s, (W + s - 1) // s))
    return sizes


def _decode_both(cls, box, ctr, img_hw, nms_pre, thr=0.05):
    from oracle import benchmark as OB
    from sipmask_b200 import ops
    dev = lambda ts: [t.permute(1, 2, 0).contiguous().cuda() for t in ts]          # noqa: E731
    b, s, lab, loc, n = ops.pair_decode_topk(dev(cls), dev(box), dev(ctr), STRIDES, img_hw, nms_pre, thr)
    k = int(n.item())
    got = (b[:k].cpu().numpy(), s[:k].cpu().numpy(), lab[:k].cpu().numpy(), loc[:k].cpu().numpy())
    assert (lab[k:] == -1).all() and (loc[k:] == -1).all()
    want = OB.pair_candidates(cls, box, ctr, STRIDES, img_hw, thr, nms_pre)
    return got, want


def _assert_same_candidates(got, want):
    assert got[2].tolist() == want[2].tolist()
    assert got[3].tolist() == want[3].tolist()
    assert np.array_equal(got[1], want[1])
    assert np.array_equal(got[0], want[0])


def test_pair_decode_random_matches_oracle_bit_exact():
    g = torch.Generator().manual_seed(0)
    sizes = _pyramid(256, 384)
    cls = [torch.randn(80, h, w, generator=g) * 2 - 4 for h, w in sizes]
    box = [(torch.randn(4, h, w, generator=g) * 4 * s).abs() for (h, w), s in zip(sizes, STRIDES)]
    ctr = [torch.randn(1, h, w, generator=g) for h, w in sizes]
    got, want = _decode_both(cls, box, ctr, (250, 370), 1000)
    _assert_same_candidates(got, want)


def test_pair_decode_saturated_800x1344_gives_nms_pre_per_level():
    """Every pair of an 800x1344 pyramid passes (1.34 M pairs at P3): exactly nms_pre per level, the oracle's pairs."""
    g = torch.Generator().manual_seed(1)
    sizes = _pyramid(800, 1344)
    cls = [torch.randn(80, h, w, generator=g) * 0.5 + 3 for h, w in sizes]
    box = [(torch.randn(4, h, w, generator=g) * 4 * s).abs() for (h, w), s in zip(sizes, STRIDES)]
    ctr = [torch.randn(1, h, w, generator=g) for h, w in sizes]
    got, want = _decode_both(cls, box, ctr, (800, 1333), 1000)
    assert got[0].shape[0] == 5000
    _assert_same_candidates(got, want)


def test_pair_decode_few_passes_and_equal_scores():
    sizes = _pyramid(64, 96)
    g = torch.Generator().manual_seed(2)
    cls = [torch.full((80, h, w), -6.0) for h, w in sizes]
    cls[0][3, 1, 2] = 0.5                                          # P3: two passing pairs, fewer than nms_pre
    cls[0][7, 0, 0] = 0.25
    cls[1][:] = 1.0                                               # P4: 4*6*80 = 1920 equal scores -> the lowest pair indices
    box = [(torch.randn(4, h, w, generator=g) * 4 * s).abs() for (h, w), s in zip(sizes, STRIDES)]
    ctr = [torch.zeros(1, h, w) for h, w in sizes]
    got, want = _decode_both(cls, box, ctr, (60, 90), 1000)
    _assert_same_candidates(got, want)
    lv = got[3]
    assert (lv < 8 * 12).sum() == 2
    p4 = (lv >= 8 * 12) & (lv < 8 * 12 + 4 * 6)
    assert p4.sum() == 1000 and ((lv[p4] - 8 * 12) * 80 + got[2][p4]).tolist() == list(range(1000))


def _nms_case(n, n_labels, seed, tie_sqrt=False):
    rng = np.random.default_rng(seed)
    xy = rng.uniform(0, 1200, (n, 2)).astype(np.float32)
    wh = rng.uniform(4, 200, (n, 2)).astype(np.float32)
    boxes = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    prod = rng.uniform(0.0025, 1, n).astype(np.float32)
    if tie_sqrt:        # distinct products whose float32 sqrt coincides
        prod[1::2] = np.nextafter(prod[0::2], np.float32(2))[: len(prod[1::2])]
    scores = np.sqrt(prod).astype(np.float32)
    labels = rng.integers(0, n_labels, n).astype(np.int32)
    return boxes, scores, labels


@pytest.mark.parametrize('n_labels,tie_sqrt', [(1, False), (80, False), (80, True)])
def test_ml_nms_matches_oracle_bit_exact(n_labels, tie_sqrt):
    from oracle import benchmark as OB
    from sipmask_b200 import ops
    boxes, scores, labels = _nms_case(5000, n_labels, n_labels, tie_sqrt)
    if tie_sqrt:
        assert len(np.unique(scores)) < len(scores)
    n = torch.tensor([5000], dtype=torch.int32).cuda()
    det, lab, idx, cnt, total = ops.ml_nms_topk(torch.from_numpy(boxes).cuda(), torch.from_numpy(scores).cuda(),
                                                torch.from_numpy(labels).cuda(), n, 0.6, 100, out_cap=5000)
    keep = OB.kth_value_cut(scores, OB.ml_nms(boxes, scores, labels, 0.6), 100)
    k = int(cnt.item())
    assert k == int(total.item()) == len(keep) and k >= 100
    assert idx[:k].cpu().tolist() == keep.tolist()
    assert lab[:k].cpu().tolist() == labels[keep].tolist()
    assert np.array_equal(det[:k].cpu().numpy(), np.concatenate([boxes[keep], scores[keep, None]], 1))
    assert (idx[k:] == -1).all()


def test_ml_nms_kth_value_tie_beyond_capacity():
    """150 disjoint boxes with equal scores all survive the k-th-value cut at 100: count stays at the capacity (100, the
    first rows in candidate order) and the full kept count is reported."""
    from sipmask_b200 import ops
    n = 150
    x = torch.arange(n, dtype=torch.float32) * 20
    boxes = torch.stack([x, torch.zeros(n), x + 10, torch.full((n,), 10.0)], 1)
    scores = torch.full((n,), 0.5)
    labels = torch.zeros(n, dtype=torch.int32)
    cap = 160                                  # slots past n_cand are ignored
    bb = torch.cat([boxes, torch.zeros(cap - n, 4)]).cuda()
    ss = torch.cat([scores, torch.ones(cap - n)]).cuda()
    ll = torch.cat([labels, torch.zeros(cap - n, dtype=torch.int32)]).cuda()
    det, lab, idx, cnt, total = ops.ml_nms_topk(bb, ss, ll, torch.tensor([n], dtype=torch.int32).cuda(), 0.6, 100,
                                                out_cap=100)
    assert int(cnt.item()) == 100 and int(total.item()) == 150
    assert idx.cpu().tolist() == list(range(100))


def test_invalid_sizes_rejected():
    from sipmask_b200 import ops, _lib
    z = torch.zeros(6000, 4).cuda()
    with pytest.raises(_lib.SmbError):
        ops.ml_nms_topk(z, z[:, 0], z[:, 0].int(), torch.zeros(1, dtype=torch.int32).cuda())


# ----------------------------------------------------------------------------------------------------- engine
def _engine_case(depth, H, W, img_shape, ori_shape, batch=1, use_graph=False):
    from oracle import benchmark as OB
    from sipmask_b200 import benchmark as B, synth
    from sipmask_b200.engine import SipMaskEngine
    sd = B.convert_state_dict(B.synthetic_state_dict(depth=depth, cls_bias=-2.5))
    img = synth.synthetic_image(H, W, batch=batch, seed=0)
    net = OB.SipMaskDetector(depth)
    net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        feats = net.extract_feat(img[:1])
        ref = net.bbox_head(feats)
    eng = SipMaskEngine(sd, (H, W), batch=batch, depth=depth, img_shape=img_shape, ori_shape=ori_shape, use_graph=use_graph,
                        benchmark=True)
    out = eng.forward(img.cuda())
    torch.cuda.synchronize()
    return dict(eng=eng, out=out, feats=feats, ref=ref, img=img, sd=sd)


def _check_network(c):
    eng, feats, ref = c['eng'], c['feats'], c['ref']
    for l, (p, r) in enumerate(zip(eng.fpn_outs, feats)):
        assert _rel(p[:1].float().cpu().permute(0, 3, 1, 2), r) < 1e-2, l
    ho = eng.head_outputs()
    cls, bbox, ctr, cof, fm = ref
    for l in range(5):
        assert _rel(ho['cls'][l][:1].cpu(), cls[l]) < 2e-2, l
        assert _rel(ho['bbox'][l][:1].cpu(), bbox[l]) < 2e-2, l
        assert _rel(ho['cof'][l][:1].cpu(), cof[l]) < 2e-2, l
        assert (ho['ctr'][l][:1].cpu() - ctr[l]).abs().max().item() < 5e-2 * (ctr[l].abs().max().item() + 1), l
    assert _rel(ho['feat_masks'][:1].float().cpu(), fm) < 2e-2


def _check_postproc(c, img_shape, ori_shape, image=0):
    from oracle import benchmark as OB
    from sipmask_b200 import ops
    eng, out = c['eng'], c['out']
    ho = eng.head_outputs()
    outs = ([t.cpu() for t in ho['cls']], [t.cpu() for t in ho['bbox']], [t.cpu() for t in ho['ctr']],
            [t.cpu() for t in ho['cof']], ho['feat_masks'].float().cpu())
    res = OB.postprocess(outs, img_shape[:2], ori_shape[:2], image=image)
    k = int(out['count'][image])
    keep = res['keep']
    assert int(eng.kept_total[image]) == len(keep) and k == min(len(keep), 100) and k > 0
    assert out['idxs_keep'][image, :k].cpu().tolist() == keep[:k].tolist()
    assert out['det_labels'][image, :k].cpu().tolist() == res['det_labels'][:k].tolist()
    np.testing.assert_allclose(out['det_bboxes'][image, :k].cpu().numpy(), res['det_bboxes'][:k], rtol=1e-5, atol=1e-5)
    masks = ops.unpack_mask_bits(out['mask_bits'][image, :k].cpu(), ori_shape[1]).numpy().astype(bool)
    ref = res['masks'][:k].astype(bool)
    iou = (np.logical_and(masks, ref).sum((1, 2)) + 1e-9) / (np.logical_or(masks, ref).sum((1, 2)) + 1e-9)
    assert iou.min() >= 0.999, iou
    return res


@pytest.fixture(scope='module')
def small_r50():
    return _engine_case(50, 128, 192, (120, 187, 3), (180, 280, 3))


def test_engine_r50_small_network_parity(small_r50):
    _check_network(small_r50)


def test_engine_r50_small_postproc_exact(small_r50):
    res = _check_postproc(small_r50, (120, 187, 3), (180, 280, 3))
    assert len(res['keep']) > 0


def test_engine_r101_small():
    c = _engine_case(101, 128, 192, (128, 192, 3), (128, 192, 3))
    _check_network(c)
    _check_postproc(c, (128, 192, 3), (128, 192, 3))


def test_engine_r50_800x1344():
    c = _engine_case(50, 800, 1344, (800, 1333, 3), (427, 711, 3))
    _check_network(c)
    res = _check_postproc(c, (800, 1333, 3), (427, 711, 3))
    from oracle import benchmark as OB
    b, s, lab, _ = res['cand']
    assert len(OB.ml_nms(b, s, lab, 0.6)) > 100        # more than 100 survive NMS: the k-th-value cut is exercised


def test_engine_graph_replay_and_batch(small_r50):
    from sipmask_b200.engine import SipMaskEngine
    sd, img = small_r50['sd'], small_r50['img']
    want = small_r50['out']
    g = SipMaskEngine(sd, (128, 192), img_shape=(120, 187, 3), ori_shape=(180, 280, 3), use_graph=True, benchmark=True)
    for _ in range(2):
        o = g.forward(img.cuda())
        torch.cuda.synchronize()
        for k in ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'mask_bits'):
            assert torch.equal(o[k], want[k]), k
    from sipmask_b200 import synth
    img2 = torch.cat([img, synth.synthetic_image(128, 192, seed=5)])
    b = SipMaskEngine(sd, (128, 192), batch=2, img_shape=(120, 187, 3), ori_shape=(180, 280, 3), use_graph=True,
                      benchmark=True)
    ob = {k: v.clone() for k, v in b.forward(img2.cuda()).items()}
    torch.cuda.synchronize()
    for i in range(2):
        o = g.forward(img2[i:i + 1].cuda())
        torch.cuda.synchronize()
        for k in ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'mask_bits'):
            assert torch.equal(ob[k][i], o[k][0]), (i, k)


def test_engine_rejects_options_before_touching_gpu():
    from sipmask_b200.engine import SipMaskEngine
    with pytest.raises(ValueError, match='vis'):
        SipMaskEngine({}, (128, 192), benchmark=True, vis=True, device='cuda:0')
    with pytest.raises(ValueError, match='rescoring'):
        SipMaskEngine({}, (128, 192), benchmark=True, rescoring_flag=True, device='cuda:0')


def test_pipelined_runner_returns_the_engine_record(small_r50):
    from sipmask_b200.serving import PipelinedRunner, make_engines
    sd, img = small_r50['sd'], small_r50['img']
    want = small_r50['out']
    engs = make_engines(sd, (128, 192), in_flight=2, img_shape=(120, 187, 3), ori_shape=(180, 280, 3), use_graph=True,
                        benchmark=True)
    runner = PipelinedRunner(engs)
    seen, slots = [], []
    for _ in range(3):
        slots.append(runner.step(img.pin_memory(), lambda rec: seen.append({k: v.clone() for k, v in rec.items()})))
    runner.flush(lambda rec: seen.append({k: v.clone() for k, v in rec.items()}))
    torch.cuda.synchronize()
    assert len(seen) == 3
    for rec in seen:                           # the runner's record: boxes, labels, count, mask bits
        for k in ('det_bboxes', 'det_labels', 'count', 'mask_bits'):
            assert torch.equal(rec[k].to(want[k].device), want[k]), k
    host = runner.result(slots[-1])
    assert torch.equal(host['det'], want['det_bboxes'].cpu()) and torch.equal(host['bits'], want['mask_bits'].cpu())


class _BoxList(object):
    """Stand-in for fcos_core.structures.bounding_box.BoxList (pure python in the reference; not installed here)."""

    def __init__(self, bbox, image_size, mode='xyxy'):
        self.bbox, self.size, self.mode, self.extra_fields = bbox, image_size, mode, {}

    def add_field(self, k, v):
        self.extra_fields[k] = v

    def get_field(self, k):
        return self.extra_fields[k]

    def __len__(self):
        return self.bbox.shape[0]


def test_dropin_module_matches_oracle_postprocessor(monkeypatch):
    import sys
    import types
    from oracle import benchmark as OB
    from sipmask_b200 import benchmark as B
    mods = {n: types.ModuleType(n) for n in ('fcos_core', 'fcos_core.structures', 'fcos_core.structures.bounding_box')}
    mods['fcos_core.structures.bounding_box'].BoxList = _BoxList
    for n, m in mods.items():
        monkeypatch.setitem(sys.modules, n, m)
    s = types.SimpleNamespace(NUM_CLASSES=81, FPN_STRIDES=list(STRIDES), NORM_REG_TARGETS=True, CENTERNESS_ON_REG=True,
                              USE_DCN_IN_TOWER=False, INFERENCE_TH=0.05, PRE_NMS_TOP_N=1000, NMS_TH=0.6, NUM_CONVS=4)
    cfg = types.SimpleNamespace(MODEL=types.SimpleNamespace(SIPMASK=s), TEST=types.SimpleNamespace(DETECTIONS_PER_IMG=100))
    mod = B.SipMaskModule(cfg, 256).eval()
    bm = B.synthetic_state_dict(depth=50, cls_bias=-2.5)
    mod.load_state_dict({'head.' + k[len('rpn.head.'):]: v for k, v in bm.items() if k.startswith('rpn.head.')}, strict=True)
    mod = mod.cuda()
    g = torch.Generator().manual_seed(3)
    feats = [torch.randn(2, 256, (128 + st - 1) // st, (192 + st - 1) // st, generator=g).cuda() for st in STRIDES]
    images = types.SimpleNamespace(image_sizes=[(120, 187), (128, 192)])
    metas = [(280, 180), (192, 128)]
    boxlists, losses = mod(images, feats, img_metas=metas)
    assert losses == {} and len(boxlists) == 2
    ho = next(iter(mod._engines.values())).head_outputs()
    outs = ([t.cpu() for t in ho['cls']], [t.cpu() for t in ho['bbox']], [t.cpu() for t in ho['ctr']],
            [t.cpu() for t in ho['cof']], ho['feat_masks'].float().cpu())
    for n, bl in enumerate(boxlists):
        (h, w), (ow, oh) = images.image_sizes[n], metas[n]
        res = OB.postprocess(outs, (h, w), (oh, ow), image=n)
        k = len(res['keep'])
        assert len(bl) == k > 0 and bl.size == (w, h)
        assert bl.get_field('labels').cpu().tolist() == (res['det_labels'] + 1).tolist()
        np.testing.assert_allclose(bl.bbox.cpu().numpy(), res['det_bboxes'][:, :4], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(bl.get_field('scores').cpu().numpy(), res['det_bboxes'][:, 4], rtol=1e-6, atol=1e-7)
        m = bl.get_field('mask')
        assert m.dtype == torch.uint8 and tuple(m.shape) == (k, 1, oh, ow)
        mm, ref = m[:, 0].cpu().numpy().astype(bool), res['masks'].astype(bool)
        iou = (np.logical_and(mm, ref).sum((1, 2)) + 1e-9) / (np.logical_or(mm, ref).sum((1, 2)) + 1e-9)
        assert iou.min() >= 0.999, iou
    mod.train()
    with pytest.raises(NotImplementedError):
        mod(images, feats, img_metas=metas)
