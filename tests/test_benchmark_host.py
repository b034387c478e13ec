"""CPU checks of the SipMask-benchmark support: checkpoint key conversion and the oracle's label-aware NMS."""
import numpy as np
import pytest
import torch


def test_convert_state_dict_maps_every_key_once_and_strips_module():
    from sipmask_b200 import benchmark as B
    for depth in (50, 101):
        bm = B.synthetic_state_dict(depth=depth)
        assert any(k.startswith('rpn.head.cls_tower.3.') for k in bm) and any(k.startswith('backbone.body.stem.') for k in bm)
        plain = B.convert_state_dict(bm)
        ddp = B.convert_state_dict({'module.' + k: v for k, v in bm.items()})
        assert sorted(plain) == sorted(ddp) == sorted(B.expected_keys(depth))
        assert len(plain) == len(bm)                      # one engine key per BM key
        assert all(ddp[k] is plain[k] for k in plain)
        for k in ('bbox_head.cls_convs.0.conv.bias', 'bbox_head.reg_convs.3.conv.bias', 'bbox_head.feat_align.conv_adaption.bias',
                  'bbox_head.cls_convs.2.gn.weight', 'neck.lateral_convs.0.conv.bias', 'neck.fpn_convs.4.conv.weight'):
            assert k in plain, k
        assert plain['neck.lateral_convs.0.conv.weight'] is bm['backbone.fpn.fpn_inner2.weight']
        assert plain['bbox_head.reg_convs.1.gn.bias'] is bm['rpn.head.bbox_tower.4.bias']


def test_convert_state_dict_rejects_unknown_and_missing_keys_and_ignores_training_buffers():
    from sipmask_b200 import benchmark as B
    bm = B.synthetic_state_dict(depth=50)
    extra = dict(bm)
    extra['rpn.head.cls_tower.2.weight'] = torch.zeros(1)          # index 3i+2 is the ReLU: no parameters
    extra['rpn.head.something_new.weight'] = torch.zeros(1)
    with pytest.raises(KeyError, match='something_new'):
        B.convert_state_dict(extra)
    short = {k: v for k, v in bm.items() if k != 'rpn.head.feat_align.conv_adaption.bias'}
    with pytest.raises(KeyError, match='feat_align.conv_adaption.bias'):
        B.convert_state_dict(short)
    buf = dict(bm)
    buf['backbone.body.layer1.0.bn1.num_batches_tracked'] = torch.tensor(0)
    assert sorted(B.convert_state_dict(buf)) == sorted(B.expected_keys(50))


def test_oracle_detector_loads_converted_dict_strictly():
    from oracle import benchmark as OB
    from sipmask_b200 import benchmark as B
    net = OB.SipMaskDetector(50)
    net.load_state_dict(B.convert_state_dict(B.synthetic_state_dict(depth=50)), strict=True)
    bn = net.backbone.bn1
    x = torch.randn(1, 64, 3, 3)
    want = x * (bn.weight / bn.running_var.sqrt()).view(1, -1, 1, 1) + (bn.bias - bn.running_mean * bn.weight /
                                                                          bn.running_var.sqrt()).view(1, -1, 1, 1)
    torch.testing.assert_close(bn(x), want, rtol=1e-5, atol=1e-5)     # FrozenBatchNorm2d: no eps


@pytest.mark.parametrize('n_labels', [1, 3, 80])
def test_ml_nms_is_union_of_per_label_nms(n_labels):
    """ml_nms_kernel's devIoU differs from the pinned nms_kernel's only by the label test, so the label-aware NMS must keep
    exactly the union over labels of the per-label (+1, `>`) NMS."""
    from oracle import benchmark as OB
    from oracle import ops as O
    rng = np.random.default_rng(n_labels)
    n = 600
    xy = rng.uniform(0, 200, (n, 2)).astype(np.float32)
    wh = rng.uniform(4, 60, (n, 2)).astype(np.float32)
    boxes = np.concatenate([xy, xy + wh], 1).astype(np.float32)
    scores = rng.uniform(0, 1, n).astype(np.float32)
    scores[::7] = scores[1::7][:len(scores[::7])]                  # score ties
    labels = rng.integers(0, n_labels, n)
    got = OB.ml_nms(boxes, scores, labels, 0.6)
    want = []
    for c in range(n_labels):
        idx = np.nonzero(labels == c)[0]
        keep = O.nms(np.concatenate([boxes[idx], scores[idx, None]], 1), 0.6)
        want += idx[keep].tolist()
    assert got.tolist() == sorted(want)


def test_kth_value_cut_keeps_ties():
    from oracle import benchmark as OB
    scores = np.array([0.9, 0.5, 0.5, 0.5, 0.1], np.float32)
    assert OB.kth_value_cut(scores, np.arange(5), 2).tolist() == [0, 1, 2, 3]
    assert OB.kth_value_cut(scores, np.arange(5), 5).tolist() == [0, 1, 2, 3, 4]


def test_pair_candidates_topk_ties_and_order():
    """More passing pairs than nms_pre: the largest products are kept, ties go to the lower pair index, and the kept
    pairs are listed by ascending pair index."""
    from oracle import benchmark as OB
    C, h, w = 3, 2, 2
    cls = torch.full((C, h, w), 2.0)
    cls[1, 0, 1] = 3.0
    cls[2, 1, 1] = -10.0                                           # below the threshold
    box = torch.ones(4, h, w)
    ctr = torch.zeros(1, h, w)
    b, s, lab, loc = OB.pair_candidates([cls], [box], [ctr], [8], (16, 16), nms_pre=4)
    # pair index = loc * C + c; the largest is (loc 1, c 1) = 4, then ties 0, 1, 2 (lowest indices)
    assert (loc * C + lab).tolist() == [0, 1, 2, 4]
    assert s[3] > s[0] and s[0] == s[1] == s[2]


def test_rejected_options_raise_value_error():
    from sipmask_b200 import benchmark as B
    for kw, word in ((dict(centerness_on_reg=False), 'CENTERNESS_ON_REG'), (dict(norm_reg_targets=False), 'NORM_REG_TARGETS'),
                     (dict(use_dcn_in_tower=True), 'USE_DCN_IN_TOWER'), (dict(vis=True), 'vis'),
                     (dict(rescoring=True), 'rescoring')):
        with pytest.raises(ValueError, match=word):
            B.check_options(**kw)
