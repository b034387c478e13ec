"""End-to-end parity of the engine against the fp32 CPU oracle on the same seeded weights and image (-m gpu).

Tolerances (stated per BASELINE.json north_star):
  * head outputs (fp16 storage / fp32 accumulate through ~70 conv layers vs fp32 oracle): relative L2 error <= 2e-2
  * post-processing given the engine's own head outputs: kept indices / labels bit-exact vs the oracle run on the
    same head outputs; masks IoU >= 0.999."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


@pytest.fixture(scope='module')
def small_case():
    from oracle import model as M
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    H, W = 128, 192
    sd = synth.detector_state_dict(depth=50, seed=1, cls_bias=-2.5)
    img = synth.synthetic_image(H, W, seed=0)
    net = M.SipMaskDetector(50)
    net.load_state_dict(sd, strict=True)
    net.eval()
    with torch.no_grad():
        feats = net.extract_feat(img)
        ref = net.bbox_head(feats)
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    eng = SipMaskEngine(sd, (H, W), test_cfg=cfg, img_shape=(H, W - 5, 3), use_graph=False)
    out = eng.forward(img.cuda())
    torch.cuda.synchronize()
    return dict(eng=eng, out=out, ref=ref, feats=feats, cfg=cfg, img=img, sd=sd, H=H, W=W)


def test_backbone_fpn_parity(small_case):
    eng, feats = small_case['eng'], small_case['feats']
    for l, (p, r) in enumerate(zip(eng.fpn_outs, feats)):
        e = _rel(p.float().cpu().permute(0, 3, 1, 2), r)
        assert e < 1e-2, 'FPN level %d rel err %g' % (l, e)


def test_head_outputs_parity(small_case):
    eng, ref = small_case['eng'], small_case['ref']
    ho = eng.head_outputs()
    cls, bbox, ctr, cof, fm = ref
    for l in range(5):
        assert _rel(ho['cls'][l].cpu(), cls[l]) < 2e-2, l
        assert _rel(ho['bbox'][l].cpu(), bbox[l]) < 2e-2, l
        assert _rel(ho['cof'][l].cpu(), cof[l]) < 2e-2, l
        assert (ho['ctr'][l].cpu() - ctr[l]).abs().max().item() < 5e-2 * (ctr[l].abs().max().item() + 1), l
    assert _rel(ho['feat_masks'].float().cpu(), fm) < 2e-2


def test_postproc_bit_exact_given_engine_head_outputs(small_case):
    from oracle import postproc as P
    from sipmask_b200 import ops
    eng, out, cfg, H, W = small_case['eng'], small_case['out'], small_case['cfg'], small_case['H'], small_case['W']
    ho = eng.head_outputs()
    img_shape = (H, W - 5, 3)
    res = P.get_bboxes_single([t[0].cpu() for t in ho['cls']], [t[0].cpu() for t in ho['bbox']],
                              [t[0].cpu() for t in ho['ctr']], [t[0].cpu() for t in ho['cof']],
                              ho['feat_masks'][0].float().cpu(), eng.strides, img_shape, img_shape, 1.0, cfg, rescale=True)
    k = int(out['count'][0])
    assert k == res['det_bboxes'].shape[0] and k > 0
    assert out['det_labels'][0, :k].cpu().tolist() == res['det_labels'].tolist()
    assert out['idxs_keep'][0, :k].cpu().tolist() == res['idxs_keep'].tolist()
    np.testing.assert_allclose(out['det_bboxes'][0, :k].cpu().numpy(), res['det_bboxes'].numpy(), rtol=1e-5, atol=1e-5)
    masks = ops.unpack_mask_bits(out['mask_bits'][0, :k].cpu(), img_shape[1]).numpy().astype(bool)
    ref = res['masks'].astype(bool)
    iou = (np.logical_and(masks, ref).sum((1, 2)) + 1e-9) / (np.logical_or(masks, ref).sum((1, 2)) + 1e-9)
    assert iou.min() >= 0.999, iou


def test_graph_replay_matches_eager(small_case):
    from sipmask_b200.engine import SipMaskEngine
    sd, cfg, H, W, img = small_case['sd'], small_case['cfg'], small_case['H'], small_case['W'], small_case['img']
    eng = SipMaskEngine(sd, (H, W), test_cfg=cfg, img_shape=(H, W - 5, 3), use_graph=True)
    a = eng.forward(img.cuda())
    torch.cuda.synchronize()
    first = {k: v.clone() for k, v in a.items()}
    b = eng.forward(img.cuda())
    torch.cuda.synchronize()
    ref = small_case['out']
    for k in ('det_labels', 'count', 'idxs_keep', 'mask_bits'):
        assert torch.equal(first[k], b[k]), k
        assert torch.equal(b[k], ref[k]), k


def test_images_in_flight_match_serial(small_case):
    """Three engines (shared weights, capped grids, different planner tiling) replayed concurrently on three streams give,
    for every image, exactly the record the single serial engine gives: boxes, labels, kept indices and mask bits."""
    from sipmask_b200 import synth
    from sipmask_b200.serving import make_engines, EnginePool, PipelinedRunner
    sd, cfg, H, W = small_case['sd'], small_case['cfg'], small_case['H'], small_case['W']
    serial = make_engines(sd, (H, W), in_flight=1, test_cfg=cfg, img_shape=(H, W - 5, 3), use_graph=True)[0]
    # 7 images over 3 slots: consecutive uses of a slot get different images, so a stale input or record shows
    imgs = [synth.synthetic_image(H, W, seed=s) for s in range(7)]
    want = []
    for im in imgs:
        o = serial.forward(im.cuda())
        torch.cuda.synchronize()
        want.append({k: v.clone() for k, v in o.items()})
    assert torch.equal(want[0]['mask_bits'], small_case['out']['mask_bits'])
    engs = make_engines(sd, (H, W), in_flight=3, test_cfg=cfg, img_shape=(H, W - 5, 3), use_graph=True)
    assert engs[1]._wcache is engs[0]._wcache
    for e, im in zip(engs, imgs):
        e.img.copy_(im)
    pool = EnginePool(engs)
    for _ in range(7):
        pool.step()
    pool.flush()
    torch.cuda.synchronize()
    for e, w in zip(engs, want):
        assert torch.equal(e.det, w['det_bboxes'])
        assert torch.equal(e.labels, w['det_labels'])
        assert torch.equal(e.count, w['count'])
        assert torch.equal(e.mask_bits, w['mask_bits'])
    # the same through the host <-> device pipeline (pinned host in, pinned host out), lagged consumer included
    runner = PipelinedRunner(engs)
    pinned = [im.pin_memory() for im in imgs]
    seen = []
    slots = []

    def check(i):                                      # image i % 7, read before its slot takes image i + 3
        host = runner.result(slots[i])
        w = want[i % 7]
        assert torch.equal(host['det'], w['det_bboxes'].cpu()), i
        assert torch.equal(host['lab'], w['det_labels'].cpu()), i
        assert torch.equal(host['cnt'], w['count'].cpu()), i
        assert torch.equal(host['bits'], w['mask_bits'].cpu()), i
    for i in range(10):
        if i >= 3:
            check(i - 3)
        slots.append(runner.step(pinned[i % 7], lambda rec: seen.append(int(rec['count'][0]))))
    runner.flush(lambda rec: seen.append(int(rec['count'][0])))
    torch.cuda.synchronize()
    for i in (7, 8, 9):
        check(i)
    assert seen == [int(want[i % 7]['count'][0]) for i in range(10)]


def _engine_vs_oracle(depth, stacked, gn, ssd, H, W, cfg, cls_bias, scale_factor=1.0, tol=2e-2):
    from oracle import model as M
    from oracle import postproc as P
    from sipmask_b200 import ops, synth
    from sipmask_b200.engine import SipMaskEngine
    sd = synth.detector_state_dict(depth=depth, stacked_convs=stacked, gn=gn, seed=1, cls_bias=cls_bias)
    img = synth.synthetic_image(H, W, seed=0)
    net = M.SipMaskDetector(depth, stacked_convs=stacked, gn=gn, ssd_flag=ssd)
    net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        ref = net(img)
    img_shape = (H, W, 3)
    eng = SipMaskEngine(sd, (H, W), depth=depth, stacked_convs=stacked, gn=gn, ssd_flag=ssd, test_cfg=cfg, img_shape=img_shape,
                        scale_factor=scale_factor, use_graph=True)
    out = eng.forward(img.cuda())
    torch.cuda.synchronize()
    ho = eng.head_outputs()
    cls, bbox, ctr, cof, fm = ref
    for l in range(5):
        assert _rel(ho['cls'][l].cpu(), cls[l]) < tol, l
        assert _rel(ho['bbox'][l].cpu(), bbox[l]) < tol, l
        assert _rel(ho['cof'][l].cpu(), cof[l]) < tol, l
    assert _rel(ho['feat_masks'].float().cpu(), fm) < tol
    res = P.get_bboxes_single([t[0].cpu() for t in ho['cls']], [t[0].cpu() for t in ho['bbox']],
                              [t[0].cpu() for t in ho['ctr']], [t[0].cpu() for t in ho['cof']],
                              ho['feat_masks'][0].float().cpu(), eng.strides, img_shape, img_shape, scale_factor, cfg,
                              rescale=True, ssd_flag=ssd)
    k = int(out['count'][0])
    assert k == res['det_bboxes'].shape[0] and k > 0
    assert out['det_labels'][0, :k].cpu().tolist() == res['det_labels'].tolist()
    np.testing.assert_allclose(out['det_bboxes'][0, :k].cpu().numpy(), res['det_bboxes'].numpy(), rtol=1e-5, atol=1e-5)
    masks = ops.unpack_mask_bits(out['mask_bits'][0, :k].cpu(), img_shape[1]).numpy().astype(bool)
    want = res['masks'].astype(bool)
    iou = (np.logical_and(masks, want).sum((1, 2)) + 1e-9) / (np.logical_or(masks, want).sum((1, 2)) + 1e-9)
    assert iou.min() >= 0.999, iou


def test_config_b_ssd_two_convs_no_gn_fast_nms():
    """SURVEY §8 config B at reduced size: stacked_convs=2, norm_cfg=None, ssd_flag (fast_nms, per-axis scale_factor),
    sipmask_r50_caffe_fpn_ssd_6x.py.  Head outputs within 2e-2 of the fp32 oracle; detections equal to the oracle's on the
    engine's own head outputs; masks IoU >= 0.999."""
    cfg = dict(nms_pre=200, score_thr=0.1, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
    _engine_vs_oracle(50, 2, False, True, 160, 160, cfg, cls_bias=-2.5, scale_factor=np.ones(4, dtype=np.float32))


def test_r101_backbone():
    """SURVEY §8 config A with the R101 backbone ((3,4,23,3) bottlenecks, resnet.py:312-324) at reduced size."""
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    _engine_vs_oracle(101, 4, True, False, 128, 160, cfg, cls_bias=-2.5, tol=3e-2)


def test_backbone_dcn_sipmask_pp():
    """SipMask++ backbone (SURVEY 8a-1 / 8f-4): DeformConvPack dg=1 as conv2 of every third block of stages 2-4
    (resnet.py:146-168,288-291).  FPN outputs within 2e-2 relative L2 of the fp32 oracle."""
    from oracle import model as M
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    H, W = 128, 160
    sd = synth.detector_state_dict(depth=50, backbone_dcn=True, seed=1, cls_bias=-2.5)
    img = synth.synthetic_image(H, W, seed=0)
    net = M.SipMaskDetector(50, backbone_dcn=True)
    net.load_state_dict(sd, strict=True)
    with torch.no_grad():
        feats = net.extract_feat(img)
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    eng = SipMaskEngine(sd, (H, W), test_cfg=cfg, img_shape=(H, W, 3), use_graph=True, backbone_dcn=True)
    assert eng.op_names.count('deform_im2col') == 1 + 2 + 2 + 1          # head + stage 2 (blocks 0,3) + stage 3 (0,3) + stage 4 (0)
    out = eng.forward(img.cuda())
    torch.cuda.synchronize()
    for l, (p, r) in enumerate(zip(eng.fpn_outs, feats)):
        e = _rel(p.float().cpu().permute(0, 3, 1, 2), r)
        assert e < 2e-2, 'FPN level %d rel err %g' % (l, e)
    assert int(out['count'][0]) > 0


@pytest.mark.parametrize('stacked,gn,ssd', [(4, True, False), (2, False, True)])
def test_batched_forward_matches_single_image_engines(stacked, gn, ssd):
    """batch > 1 per forward (BASELINE config 4 is bs=32; get_bboxes loops over images, sipmask_head.py:517-540): every image
    of a 3-image batch gives exactly the record the batch-1 engine gives for it (detections, labels, kept indices, masks)."""
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    H, W = 96, 128
    sd = synth.detector_state_dict(depth=50, stacked_convs=stacked, gn=gn, seed=1, cls_bias=-2.5)
    cfg = dict(nms_pre=200, score_thr=0.1 if ssd else 0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    sf = np.ones(4, dtype=np.float32) if ssd else 1.0
    imgs = torch.cat([synth.synthetic_image(H, W, seed=s) for s in range(3)], 0)
    one = SipMaskEngine(sd, (H, W), stacked_convs=stacked, gn=gn, ssd_flag=ssd, test_cfg=cfg, img_shape=(H, W - 3, 3),
                        scale_factor=sf, use_graph=True)
    want = []
    for i in range(3):
        o = one.forward(imgs[i:i + 1].cuda())
        torch.cuda.synchronize()
        want.append({k: v.clone() for k, v in o.items()})
    many = SipMaskEngine(sd, (H, W), batch=3, stacked_convs=stacked, gn=gn, ssd_flag=ssd, test_cfg=cfg, img_shape=(H, W - 3, 3),
                         scale_factor=sf, use_graph=True, share_weights=one)
    for _ in range(2):                                   # second pass = graph replay
        got = many.forward(imgs.cuda())
        torch.cuda.synchronize()
        for i in range(3):
            k = int(want[i]['count'][0])
            assert int(got['count'][i]) == k and k > 0
            assert torch.equal(got['det_labels'][i, :k], want[i]['det_labels'][0, :k])
            assert torch.equal(got['idxs_keep'][i, :k], want[i]['idxs_keep'][0, :k])
            assert torch.equal(got['det_bboxes'][i, :k], want[i]['det_bboxes'][0, :k])
            assert torch.equal(got['mask_bits'][i, :k], want[i]['mask_bits'][0, :k])
    ho1, hoN = one.head_outputs(), many.head_outputs()     # `one` holds image 2 now
    for l in range(5):
        assert torch.equal(hoN['cls'][l][2:3], ho1['cls'][l])


def test_engine_rescale_into_ori_shape():
    """scale_factor != 1 (ADVICE r1 high): boxes are divided by the scale factor and the masks are resized by 2/scale_factor
    into the ori_shape canvas, like SingleStageDetector.simple_test(rescale=True) - engine vs the oracle on the engine's own
    head outputs."""
    from oracle import postproc as P
    from sipmask_b200 import ops, synth
    from sipmask_b200.engine import SipMaskEngine
    H, W, sf = 128, 160, 1.6667
    img_shape, ori_shape = (H, W - 4, 3), (77, 94, 3)
    sd = synth.detector_state_dict(depth=50, seed=1, cls_bias=-2.5)
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    eng = SipMaskEngine(sd, (H, W), test_cfg=cfg, img_shape=img_shape, ori_shape=ori_shape, scale_factor=sf, use_graph=True)
    out = eng.forward(synth.synthetic_image(H, W, seed=0).cuda())
    torch.cuda.synchronize()
    ho = eng.head_outputs()
    res = P.get_bboxes_single([t[0].cpu() for t in ho['cls']], [t[0].cpu() for t in ho['bbox']], [t[0].cpu() for t in ho['ctr']],
                              [t[0].cpu() for t in ho['cof']], ho['feat_masks'][0].float().cpu(), eng.strides, img_shape,
                              ori_shape, sf, cfg, rescale=True)
    k = int(out['count'][0])
    assert k == res['det_bboxes'].shape[0] and k > 0
    assert out['det_labels'][0, :k].cpu().tolist() == res['det_labels'].tolist()
    np.testing.assert_allclose(out['det_bboxes'][0, :k].cpu().numpy(), res['det_bboxes'].numpy(), rtol=1e-5, atol=1e-5)
    assert tuple(out['mask_bits'].shape[2:]) == (ori_shape[0], (ori_shape[1] + 31) // 32)
    masks = ops.unpack_mask_bits(out['mask_bits'][0, :k].cpu(), ori_shape[1]).numpy().astype(bool)
    want = res['masks'].astype(bool)
    assert masks.shape == want.shape
    iou = (np.logical_and(masks, want).sum((1, 2)) + 1e-9) / (np.logical_or(masks, want).sum((1, 2)) + 1e-9)
    assert iou.min() >= 0.999, iou
