"""Generate tests/golden/ref_bm_*.npz from the UNMODIFIED SipMask-benchmark python (fcos_core), imported through
_ref_import_bm.py.  Run from the repository root where /root/reference exists:  python tests/golden/gen_golden_bm.py

Weights: sipmask_b200.benchmark.synthetic_state_dict(depth=50, seed=1, cls_bias) in BM keys and shapes, loaded strictly into
the reference modules.  The backbone image is stored; the head cases store the seed of
their features (torch.randn with a seeded CPU generator, see `features`).
  ref_bm_backbone_r50_64x96.npz : image -> backbone.body + backbone.fpn (P3..P7)
  ref_bm_head_s1.npz            : features -> SipMaskHead -> SipMaskPostProcessor, resized = padded = original (64x96)
  ref_bm_head_sizes.npz         : padded 128x192, resized 120x187, original 180x280
  ref_bm_head_many.npz          : more than DETECTIONS_PER_IMG survive ml_nms (the k-th-value cut)
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from _ref_import_bm import CropSplitOracle, load  # noqa: E402
from sipmask_b200 import benchmark as B, synth  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def _sub(sd, prefix):
    return {k[len(prefix):]: v for k, v in sd.items() if k.startswith(prefix)}


def backbone_case(cfg, BB):
    sd = B.synthetic_state_dict(depth=50, seed=1)
    net = BB.build_resnet_fpn_p3p7_backbone(cfg).eval()
    net.load_state_dict(_sub(sd, 'backbone.'), strict=True)
    img = synth.synthetic_image(64, 96, seed=0)
    with torch.no_grad():
        outs = net(img)
    d = dict(image=img.numpy(), seed=np.int64(1))
    for l, o in enumerate(outs):
        d['p%d' % (l + 3)] = o.numpy()
    np.savez_compressed(os.path.join(OUT, 'ref_bm_backbone_r50_64x96.npz'), **d)
    print('backbone', [o.shape for o in outs])


def features(pad_hw, seed):
    g = torch.Generator().manual_seed(int(seed))
    return [torch.randn(1, 256, (pad_hw[0] + s - 1) // s, (pad_hw[1] + s - 1) // s, generator=g) for s in (8, 16, 32, 64, 128)]


def head_case(cfg, S, name, pad_hw, img_hw, ori_hw, cls_bias, feat_seed, min_dets=1):
    sd = B.synthetic_state_dict(depth=50, seed=1, cls_bias=cls_bias)
    mod = S.SipMaskModule(cfg, 256).eval()
    mod.load_state_dict({'head.' + k: v for k, v in _sub(sd, 'rpn.head.').items()}, strict=True)
    mod.box_selector_test.crop_cuda = CropSplitOracle()
    feats = features(pad_hw, feat_seed)
    images = types.SimpleNamespace(image_sizes=[tuple(img_hw)])
    with torch.no_grad():
        head = mod.head(feats)
        # SipMaskModule._forward_test (sipmask.py:254-259) with the per-level maps in channels_last memory: the values are
        # the same, and `candidate_inds.view(N, -1)` (inference.py:91) then works on current PyTorch, where the permuted
        # reshape of an NCHW map stays a non-contiguous view
        cl = [[t.contiguous(memory_format=torch.channels_last) for t in lst] for lst in head[:4]]
        res, = mod.box_selector_test(mod.compute_locations(feats), *cl, head[4], images.image_sizes,
                                     [(ori_hw[1], ori_hw[0])])
    d = dict(cls_bias=np.float32(cls_bias), feat_seed=np.int64(feat_seed), pad_hw=np.array(pad_hw), img_hw=np.array(img_hw),
             ori_hw=np.array(ori_hw), bbox=res.bbox.numpy(), scores=res.get_field('scores').numpy(),
             labels=res.get_field('labels').numpy(),
             mask=res.get_field('mask').numpy().astype(np.uint8))
    for l in range(5):
        for k, t in zip(('logits', 'bbox_reg', 'centerness', 'cofs'), head[:4]):
            d['%s%d' % (k, l)] = t[l].numpy()
    d['feat_masks'] = head[4].numpy()
    # survivors of ml_nms before the k-th-value cut, from the reference's own candidate stage
    cands = mod.box_selector_test.forward_for_single_feature_map
    from fcos_core.structures.boxlist_ops import boxlist_ml_nms, cat_boxlist
    locs = mod.compute_locations(feats)
    per = [cands(locs[l], cl[0][l], cl[1][l], cl[2][l], cl[3][l], images.image_sizes)[0] for l in range(5)]
    d['n_survivors'] = np.int64(len(boxlist_ml_nms(cat_boxlist(per), cfg.MODEL.SIPMASK.NMS_TH)))
    assert len(res) >= min_dets, (name, len(res))
    np.savez_compressed(os.path.join(OUT, 'ref_bm_%s.npz' % name), **d)
    print(name, 'detections', len(res), 'survivors', int(d['n_survivors']))
    return d


if __name__ == '__main__':
    cfg, BB, S = load()
    backbone_case(cfg, BB)
    head_case(cfg, S, 'head_s1', (64, 96), (64, 96), (64, 96), -2.5, 11)
    head_case(cfg, S, 'head_sizes', (128, 192), (120, 187), (180, 280), -2.5, 12)
    d = head_case(cfg, S, 'head_many', (128, 192), (128, 192), (128, 192), 0.0, 13, min_dets=100)
    assert d['n_survivors'] > 100
