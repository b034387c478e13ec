"""SipMask++ mask rescoring on tensor cores (ops.mask_rescore_f16, SipMaskEngine(rescoring_flag=True)).

Numerics: fp16 masks, weights and activations with fp32 accumulation.  Scores are compared with the fp32 chain
(ops.mask_rescore on the same fp16-rounded masks, or the oracle head) to |d| <= 1e-2 |want| + 2e-3 max|want|, the max taken
over the compared rows; the CPU emulation below pins that bound without a GPU.  Everything else in the engine's record is
bit-identical to the engine without rescoring."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

RTOL, ATOL_OF_MAX = 1e-2, 2e-3
SHAPES = [(272, 272), (400, 672), (127, 131)]


def _assert_scores_close(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    bound = RTOL * np.abs(want) + ATOL_OF_MAX * np.abs(want).max()
    err = np.abs(got - want)
    assert (err <= bound).all(), 'max excess %g (err %s, want %s)' % ((err - bound).max(), err, want)


def _scoring_weights(seed=3):
    from sipmask_b200 import synth
    sd = synth.head_state_dict(seed, stacked_convs=2, gn=False, rescoring_flag=True, prefix='')
    cw = [sd['convs_scoring.%d.conv.weight' % i] for i in range(6)]
    cb = [sd['convs_scoring.%d.conv.bias' % i] for i in range(6)]
    return cw, cb, sd['mask_scoring.weight'], sd['mask_scoring.bias']


def _cropped_masks(n, H, W, seed):
    """Seeded cropped stride-2 masks: a smooth sigmoid field inside a random roi, 0 outside."""
    g = torch.Generator().manual_seed(seed)
    field = F.interpolate(torch.randn(n, 1, H // 16 + 2, W // 16 + 2, generator=g) * 4.0, size=(H, W), mode='bilinear',
                          align_corners=False)[:, 0]
    pos = torch.sigmoid(field)
    out = torch.zeros(n, H, W)
    for i in range(n):
        y0, x0 = int(torch.randint(0, H // 2, (1,), generator=g)), int(torch.randint(0, W // 2, (1,), generator=g))
        y1, x1 = y0 + int(torch.randint(H // 4, H - y0 + 1, (1,), generator=g)), x0 + int(torch.randint(W // 4, W - x0 + 1, (1,), generator=g))
        out[i, y0:y1, x0:x1] = pos[i, y0:y1, x0:x1]
    return out.half()


def _chain(pos, cw, cb, w1, b1, labels, det, fp16):
    """The rescoring chain on the CPU: float64 throughout (fp16=False), or fp16-rounded weights and activations with fp32
    accumulation (fp16=True), the numerics of smb_mask_rescore_f16."""
    r = (lambda t: t.half().float()) if fp16 else (lambda t: t.double())
    b = (lambda t: t.float()) if fp16 else (lambda t: t.double())
    x = r(pos.float()).unsqueeze(1)
    for w, bb in zip(cw, cb):
        x = r(F.relu(F.conv2d(x, r(w), b(bb), stride=2)))
    s = F.relu(F.conv2d(x, r(w1).view(w1.shape[0], -1, 1, 1), b(b1))).amax((2, 3))
    return s[torch.arange(pos.shape[0]), labels] * b(det[:, 4])


@pytest.mark.parametrize('hw', SHAPES)
def test_fp16_emulation_within_bound(hw):
    """CPU: the fp16-storage / fp32-accumulate model of the kernels stays within the stated bound of the float64 chain on the
    same fp16 masks, for the synthetic scoring weights."""
    cw, cb, w1, b1 = _scoring_weights()
    g = torch.Generator().manual_seed(hw[1])
    n = 6
    pos = _cropped_masks(n, hw[0], hw[1], seed=hw[0])
    labels = torch.randint(0, 80, (n,), generator=g)
    det = torch.rand(n, 5, generator=g)
    with torch.no_grad():
        want = _chain(pos, cw, cb, w1, b1, labels, det, fp16=False)
        got = _chain(pos, cw, cb, w1, b1, labels, det, fp16=True)
    assert want.abs().max() > 0
    _assert_scores_close(got.numpy(), want.numpy())


def _kernel_inputs(hw, seed=0):
    g = torch.Generator().manual_seed(seed)
    n_img, max_rows = 2, 7
    pos = _cropped_masks(n_img * max_rows, hw[0], hw[1], seed=hw[0] + 1).view(n_img, max_rows, hw[0], hw[1])
    labels = torch.randint(0, 80, (n_img, max_rows), generator=g)
    labels[0, 5:] = torch.tensor([-3, 1000])                   # rows past the count: never read as labels
    labels[1] = 10 ** 6
    det = torch.rand(n_img, max_rows, 5, generator=g)
    count = torch.tensor([5, 0], dtype=torch.int32)
    return pos, labels, det, count


@pytest.mark.gpu
@pytest.mark.parametrize('hw', SHAPES)
def test_mask_rescore_f16_matches_fp32_chain(hw):
    from sipmask_b200 import ops
    cw, cb, w1, b1 = _scoring_weights()
    from oracle import numerics as NU
    wt = ops.RescoreWeights(cw, cb, w1, b1, 'cuda')
    pos, labels, det, count = _kernel_inputs(hw)
    R = pos.shape[0] * pos.shape[1]
    need = ops.mask_rescore_f16_workspace_bytes(R, hw[0], hw[1])
    ws = torch.full((need,), 0xFF, dtype=torch.uint8, device='cuda')        # unwritten fp16 reads back as 0xFFFF
    layers = ops.mask_rescore_f16_layers(ws, R, hw[0], hw[1])
    assert [t.shape[3] for t in layers] == [16, 16, 32, 64] and all(t.data_ptr() % 256 == 0 for t in layers)
    end = layers[-1].data_ptr() + layers[-1].numel() * 2 - ws.data_ptr()          # the views tile the whole workspace
    assert (end + 255) // 256 * 256 == need
    gotd = ops.mask_rescore_f16(pos.cuda(), count.cuda(), wt, labels.cuda(), det.cuda(), workspace=ws)
    # layer by layer: layer 2 from float64 layer 1, layers 3-5 and the score teacher-forced from the device's layers
    res = NU.check_rescore_chain(pos.cuda(), count.cuda(), wt.conv_w, wt.conv_b, wt.score_w, wt.score_b, labels.cuda(),
                                 det.cuda(), layers, gotd)
    print('rescore %dx%d: %s' % (hw[0], hw[1], ', '.join('%s %.3g' % kv for kv in res.items())))
    got = gotd.cpu()
    want = ops.mask_rescore(pos[0, :5].float().cuda(), [w.cuda() for w in cw], [b.cuda() for b in cb], w1.cuda(), b1.cuda(),
                            labels[0, :5].cuda(), det[0, :5].cuda()).cpu()
    assert (got[0, :5] != 0).any()
    _assert_scores_close(got[0, :5].numpy(), want.numpy())
    assert (got[0, 5:] == 0).all() and (got[1] == 0).all()


@pytest.mark.gpu
def test_mask_rescore_f16_label_out_of_range_scores_zero():
    from sipmask_b200 import ops
    cw, cb, w1, b1 = _scoring_weights()
    wt = ops.RescoreWeights(cw, cb, w1, b1, 'cuda')
    pos = _cropped_masks(3, 127, 131, seed=5).view(1, 3, 127, 131)
    labels = torch.tensor([[4, 80, -1]])
    det = torch.ones(1, 3, 5)
    got = ops.mask_rescore_f16(pos.cuda(), torch.tensor([3], dtype=torch.int32).cuda(), wt, labels.cuda(), det.cuda()).cpu()
    assert got[0, 0] > 0 and got[0, 1] == 0 and got[0, 2] == 0


@pytest.mark.gpu
def test_mask_rescore_f16_rejects_small_masks_and_workspace():
    from sipmask_b200 import _lib as L, ops
    cw, cb, w1, b1 = _scoring_weights()
    wt = ops.RescoreWeights(cw, cb, w1, b1, 'cuda')
    labels, det, count = torch.zeros(1, 2, dtype=torch.long).cuda(), torch.ones(1, 2, 5).cuda(), torch.ones(1, dtype=torch.int32).cuda()
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device='cuda')
    with pytest.raises(L.SmbError, match=r'\(-1\)'):
        ops.mask_rescore_f16(torch.zeros(1, 2, 126, 131, dtype=torch.float16, device='cuda'), count, wt, labels, det, workspace=ws)
    assert ops.mask_rescore_f16_workspace_bytes(2, 126, 131) == 0
    need = ops.mask_rescore_f16_workspace_bytes(2, 127, 131)
    assert need > 0
    pos = torch.zeros(1, 2, 127, 131, dtype=torch.float16, device='cuda')
    with pytest.raises(L.SmbError, match=r'\(-1\)'):
        ops.mask_rescore_f16(pos, count, wt, labels, det, workspace=torch.zeros(need - 1, dtype=torch.uint8, device='cuda'))
    ops.mask_rescore_f16(pos, count, wt, labels, det, workspace=torch.zeros(need, dtype=torch.uint8, device='cuda'))


# ---------------------------------------------------------------------------------------------------------- engine
H = W = 256                                 # prototypes 128 x 128
CFG = dict(nms_pre=200, score_thr=0.1, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
PP_KW = dict(depth=50, stacked_convs=2, gn=False, ssd_flag=True, backbone_dcn=True, test_cfg=CFG)


@pytest.fixture(scope='module')
def pp():
    from oracle import model as M
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    sd = synth.detector_state_dict(depth=50, stacked_convs=2, gn=False, rescoring_flag=True, backbone_dcn=True, seed=1,
                                   cls_bias=-2.5)
    head = M.SipMaskHead(stacked_convs=2, gn=False, ssd_flag=True, rescoring_flag=True)
    head.load_state_dict({k[len('bbox_head.'):]: v for k, v in sd.items() if k.startswith('bbox_head.')}, strict=True)
    sf = np.ones(4, dtype=np.float32)
    off = SipMaskEngine(sd, (H, W), scale_factor=sf, use_graph=True, **PP_KW)
    on = SipMaskEngine(sd, (H, W), scale_factor=sf, use_graph=True, rescoring_flag=True, share_weights=off, **PP_KW)
    imgs = [synth.synthetic_image(H, W, seed=s) for s in range(3)]
    want = []
    for im in imgs:
        o = on.forward(im.cuda())
        torch.cuda.synchronize()
        want.append({k: v.clone() for k, v in o.items()})
    return dict(sd=sd, head=head.eval(), off=off, on=on, imgs=imgs, want=want, sf=sf)


def _oracle_scores(eng, head, img_shape, ori_shape, sf):
    from oracle import postproc as P
    ho = eng.head_outputs()
    with torch.no_grad():
        return P.get_bboxes_single([t[0].cpu() for t in ho['cls']], [t[0].cpu() for t in ho['bbox']],
                                   [t[0].cpu() for t in ho['ctr']], [t[0].cpu() for t in ho['cof']],
                                   ho['feat_masks'][0].float().cpu(), eng.strides, img_shape, ori_shape, sf, CFG, rescale=True,
                                   ssd_flag=True, head=head)


@pytest.mark.gpu
def test_engine_rescoring_keeps_the_record_bit_identical(pp):
    for im, w in zip(pp['imgs'], pp['want']):
        o = pp['off'].forward(im.cuda())
        torch.cuda.synchronize()
        assert 'mask_scores' not in o
        assert int(w['count'][0]) > 0
        for k in ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'mask_bits'):
            assert torch.equal(o[k], w[k]), k
        k = int(w['count'][0])
        assert (w['mask_scores'][0, k:] == 0).all() and (w['mask_scores'][0, :k] != 0).any()
    assert pp['on'].op_names.count('rescore') == 1 and pp['on'].op_names.count('mask_dense') == 1
    assert pp['on'].rescore_flops > 0 and pp['on'].conv_flops == pp['off'].conv_flops


@pytest.mark.gpu
def test_engine_mask_scores_match_oracle_head(pp):
    on = pp['on']
    on.forward(pp['imgs'][0].cuda())
    torch.cuda.synchronize()
    res = _oracle_scores(on, pp['head'], (H, W, 3), (H, W, 3), pp['sf'])
    k = int(on.count[0])
    assert k == res['det_bboxes'].shape[0] and k > 0
    assert on.labels[0, :k].cpu().tolist() == res['det_labels'].tolist()
    _assert_scores_close(on.mask_scores[0, :k].cpu().numpy(), res['mask_scores'].numpy())


@pytest.mark.gpu
def test_engine_mask_scores_match_oracle_head_rescaled(pp):
    """Per-axis scale_factor (w, h, w, h) != 1: rois = boxes * scale_factor / 2, boxes and masks in the ori_shape canvas."""
    from sipmask_b200.engine import SipMaskEngine
    sf = np.array([1.25, 1.2, 1.25, 1.2], dtype=np.float32)
    img_shape, ori_shape = (H, W - 6, 3), (213, 200, 3)
    eng = SipMaskEngine(pp['sd'], (H, W), img_shape=img_shape, ori_shape=ori_shape, scale_factor=sf, use_graph=True,
                        rescoring_flag=True, share_weights=pp['off'], **PP_KW)
    eng.forward(pp['imgs'][1].cuda())
    torch.cuda.synchronize()
    res = _oracle_scores(eng, pp['head'], img_shape, ori_shape, sf)
    k = int(eng.count[0])
    assert k == res['det_bboxes'].shape[0] and k > 0
    assert eng.labels[0, :k].cpu().tolist() == res['det_labels'].tolist()
    np.testing.assert_allclose(eng.det[0, :k].cpu().numpy(), res['det_bboxes'].numpy(), rtol=1e-5, atol=1e-5)
    _assert_scores_close(eng.mask_scores[0, :k].cpu().numpy(), res['mask_scores'].numpy())


@pytest.mark.gpu
def test_engine_rescoring_graph_replay_matches_eager(pp):
    from sipmask_b200.engine import SipMaskEngine
    eager = SipMaskEngine(pp['sd'], (H, W), scale_factor=pp['sf'], use_graph=False, rescoring_flag=True,
                          share_weights=pp['off'], **PP_KW)
    for im, w in zip(pp['imgs'], pp['want']):
        o = eager.forward(im.cuda())
        torch.cuda.synchronize()
        for k in w:
            assert torch.equal(o[k], w[k]), k


@pytest.mark.gpu
def test_engine_rescoring_batch_matches_single_image(pp):
    from sipmask_b200.engine import SipMaskEngine
    many = SipMaskEngine(pp['sd'], (H, W), batch=3, scale_factor=pp['sf'], use_graph=True, rescoring_flag=True,
                         share_weights=pp['off'], **PP_KW)
    assert many.op_names.count('rescore') == 1 and many.op_names.count('mask_dense') == 3
    for _ in range(2):                                          # second pass = graph replay
        got = many.forward(torch.cat(pp['imgs'], 0).cuda())
        torch.cuda.synchronize()
        for i, w in enumerate(pp['want']):
            for k in w:
                assert torch.equal(got[k][i], w[k][0]), (i, k)


@pytest.mark.gpu
def test_pipelined_runner_carries_mask_scores(pp):
    from sipmask_b200.serving import PipelinedRunner
    runner = PipelinedRunner(pp['on'])
    seen, slots = [], []
    for i in range(4):
        slots.append(runner.step(pp['imgs'][i % 3].pin_memory(), lambda rec: seen.append(rec['mask_scores'].clone())))
    runner.flush(lambda rec: seen.append(rec['mask_scores'].clone()))
    torch.cuda.synchronize()
    assert len(seen) == 4
    for i in range(4):
        assert torch.equal(seen[i], pp['want'][i % 3]['mask_scores'])
    for i in (2, 3):                                            # the last use of each slot
        assert torch.equal(runner.result(slots[i])['msc'], pp['want'][i % 3]['mask_scores'].cpu())


@pytest.mark.gpu
def test_engine_rescoring_constructor_errors():
    """Validation before anything is built: VIS, missing scoring weights, prototypes below 127 x 127."""
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    sd = synth.detector_state_dict(depth=50, stacked_convs=2, gn=False, rescoring_flag=True, seed=1)
    with pytest.raises(ValueError, match='VIS'):
        SipMaskEngine(sd, (H, W), vis=True, rescoring_flag=True, **PP_KW)
    with pytest.raises(ValueError, match='mask_scoring.weight'):
        SipMaskEngine({k: v for k, v in sd.items() if 'mask_scoring.weight' not in k}, (H, W), rescoring_flag=True, **PP_KW)
    with pytest.raises(ValueError, match='127'):
        SipMaskEngine(sd, (224, 256), rescoring_flag=True, **PP_KW)
