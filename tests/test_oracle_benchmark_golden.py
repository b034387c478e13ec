"""oracle/benchmark.py against fixtures produced by the unmodified SipMask-benchmark python (tests/golden/gen_golden_bm.py):
backbone + FPN, head and post-processor at three sizes.  Post-processing is run by the oracle on the reference's own head
outputs: labels exact, boxes and scores within 1e-4, masks exact.  When a level has more than PRE_NMS_TOP_N passing pairs
the reference's order is implementation-defined (`topk(sorted=False)`), so detections are compared in a canonical order."""
import os

import numpy as np
import pytest
import torch

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')


def _load(name):
    return dict(np.load(os.path.join(GOLD, name)))


def _rel(a, b):
    a, b = np.asarray(a, np.float64).ravel(), np.asarray(b, np.float64).ravel()
    return np.linalg.norm(a - b) / (np.linalg.norm(b) + 1e-12)


def _features(pad_hw, seed):
    g = torch.Generator().manual_seed(int(seed))
    return [torch.randn(1, 256, (int(pad_hw[0]) + s - 1) // s, (int(pad_hw[1]) + s - 1) // s, generator=g)
            for s in (8, 16, 32, 64, 128)]


def _oracle_net():
    from oracle import benchmark as OB
    return OB.SipMaskDetector(50)


def test_backbone_fpn_matches_reference():
    from sipmask_b200 import benchmark as B
    g = _load('ref_bm_backbone_r50_64x96.npz')
    net = _oracle_net()
    net.load_state_dict(B.convert_state_dict(B.synthetic_state_dict(depth=50, seed=int(g['seed']))), strict=True)
    with torch.no_grad():
        outs = net.extract_feat(torch.from_numpy(g['image']))
    for l, o in enumerate(outs):
        assert _rel(o.numpy(), g['p%d' % (l + 3)]) < 1e-5, l


@pytest.mark.parametrize('name', ['head_s1', 'head_sizes', 'head_many'])
def test_head_and_postprocessor_match_reference(name):
    from oracle import benchmark as OB
    from sipmask_b200 import benchmark as B
    g = _load('ref_bm_%s.npz' % name)
    net = _oracle_net()
    net.load_state_dict(B.convert_state_dict(B.synthetic_state_dict(depth=50, seed=1, cls_bias=float(g['cls_bias']))),
                        strict=True)
    with torch.no_grad():
        head = net.bbox_head(_features(g['pad_hw'], g['feat_seed']))
    keys = ('logits', 'bbox_reg', 'centerness', 'cofs')
    for k, outs in zip(keys, head[:4]):
        for l in range(5):
            assert _rel(outs[l].numpy(), g['%s%d' % (k, l)]) < 1e-5, (k, l)
    assert _rel(head[4].numpy(), g['feat_masks']) < 1e-5
    ref_head = tuple([torch.from_numpy(g['%s%d' % (k, l)]) for l in range(5)] for k in keys) + (torch.from_numpy(g['feat_masks']),)
    res = OB.postprocess(ref_head, g['img_hw'], g['ori_hw'])
    assert len(OB.ml_nms(*res['cand'][:3], 0.6)) == int(g['n_survivors'])
    det, lab = res['det_bboxes'], res['det_labels'] + 1                  # BoxList labels are 1-based
    assert det.shape[0] == g['bbox'].shape[0]
    o_mine = np.lexsort((det[:, 3], det[:, 2], det[:, 1], det[:, 0], lab))
    o_ref = np.lexsort((g['bbox'][:, 3], g['bbox'][:, 2], g['bbox'][:, 1], g['bbox'][:, 0], g['labels']))
    assert lab[o_mine].tolist() == g['labels'][o_ref].tolist()
    np.testing.assert_allclose(det[o_mine, :4], g['bbox'][o_ref], atol=1e-4, rtol=0)
    np.testing.assert_allclose(det[o_mine, 4], g['scores'][o_ref], atol=1e-4, rtol=0)
    assert np.array_equal(res['masks'][o_mine], g['mask'][o_ref, 0])


def test_fixtures_cover_the_kth_value_cut():
    for name in ('head_s1', 'head_sizes', 'head_many'):
        g = _load('ref_bm_%s.npz' % name)
        assert int(g['n_survivors']) > 100 and g['bbox'].shape[0] >= 100
    g = _load('ref_bm_head_sizes.npz')
    assert tuple(g['pad_hw']) != tuple(g['img_hw']) != tuple(g['ori_hw'])
