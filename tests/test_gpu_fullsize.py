"""End-to-end image -> detections parity at the BASELINE shapes (VERDICT r1 item 1a).

The engine (fp16 storage / fp32 accumulate, all kernels through the C ABI) and the fp32 CPU oracle run on the SAME seeded
synthetic image and weights at full size:
    config A  R50  800 x 1344   (BASELINE config 2, the bench workload)
    config A  R101 800 x 1344   (BASELINE config 3)
    config B  R50  544 x 544    (SSD-style head: 2 convs, no GN, fast_nms; BASELINE config 4)
and the two detection lists are compared directly (NOT the oracle re-run on the engine's head outputs, which
tests/test_gpu_engine.py covers):
  * detections are matched one-to-one: equal label, box IoU >= 0.9, best IoU first;
  * reported (gpurun_out/parity_fullsize_<case>.json) and bounded: fraction of reference detections matched, box L-inf and
    score difference over matches, min / mean mask IoU over matches, head-output relative L2.
Stated tolerance: labels of matched pairs are equal by construction; matched fraction >= 0.95; box L-inf <= 1.0 px; score
|diff| <= 2e-3; head outputs relative L2 <= 5e-3; mask IoU over matches: pooled (sum of intersections / sum of unions) >= 0.995,
mean >= 0.99, min >= 0.80 (the minimum is set by masks of a few dozen pixels, where one threshold flip costs several percent).
(The post-processing's "mask IoU >= 0.999, indices
bit-exact" holds for the post-processing given identical head outputs - tests/test_gpu_postproc.py, test_gpu_engine.py; an
fp16 backbone cannot reproduce an fp32 one bit for bit, so near-tie candidates at the max_per_img / NMS boundaries differ.)
"""
import json
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rel(a, b):
    a, b = a.double().flatten(), b.double().flatten()
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def _box_iou(a, b):
    """a [n,4], b [m,4] -> [n,m]"""
    x1 = np.maximum(a[:, None, 0], b[None, :, 0]); y1 = np.maximum(a[:, None, 1], b[None, :, 1])
    x2 = np.minimum(a[:, None, 2], b[None, :, 2]); y2 = np.minimum(a[:, None, 3], b[None, :, 3])
    inter = np.clip(x2 - x1, 0, None) * np.clip(y2 - y1, 0, None)
    aa = (a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]); ab = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    return inter / (aa[:, None] + ab[None, :] - inter + 1e-9)


def match_detections(det_a, lab_a, det_b, lab_b, iou_thr=0.9):
    iou = _box_iou(det_a[:, :4], det_b[:, :4]) * (lab_a[:, None] == lab_b[None, :])
    pairs, used_a, used_b = [], set(), set()
    for flat in np.argsort(-iou, axis=None):
        i, j = divmod(int(flat), iou.shape[1])
        if iou[i, j] < iou_thr:
            break
        if i in used_a or j in used_b:
            continue
        used_a.add(i); used_b.add(j)
        pairs.append((i, j))
    return pairs


def run_case(name, depth, stacked, gn, ssd, H, W, img_w, cfg, cls_bias, scale_factor=1.0):
    from oracle import model as M
    from oracle import ops as O
    from oracle import postproc as P
    from sipmask_b200 import ops, synth
    from sipmask_b200.engine import SipMaskEngine
    torch.set_num_threads(max(1, len(os.sched_getaffinity(0))))
    O.USE_TORCHVISION_DCN = True            # same arithmetic as the restatement (tests/test_oracle_golden.py), C++ speed
    O.USE_C_CROP_SPLIT = True
    try:
        sd = synth.detector_state_dict(depth=depth, stacked_convs=stacked, gn=gn, seed=1, cls_bias=cls_bias)
        img = synth.synthetic_image(H, W, seed=0)
        net = M.SipMaskDetector(depth, stacked_convs=stacked, gn=gn, ssd_flag=ssd)
        net.load_state_dict(sd, strict=True)
        img_shape = (H, img_w, 3)
        with torch.no_grad():
            cls, box, ctr, cof, fm = net(img)
            ref = P.get_bboxes_single([t[0] for t in cls], [t[0] for t in box], [t[0] for t in ctr], [t[0] for t in cof], fm[0],
                                      (8, 16, 32, 64, 128), img_shape, img_shape, scale_factor, cfg, rescale=True, ssd_flag=ssd)
    finally:
        O.USE_TORCHVISION_DCN = False
        O.USE_C_CROP_SPLIT = False
    eng = SipMaskEngine(sd, (H, W), depth=depth, stacked_convs=stacked, gn=gn, ssd_flag=ssd, test_cfg=cfg, img_shape=img_shape,
                        scale_factor=scale_factor, use_graph=True)
    out = eng.forward(img.cuda())
    torch.cuda.synchronize()
    ho = eng.head_outputs()
    rep = dict(case=name, H=H, W=W)
    rep['head_rel_l2'] = dict(
        cls=max(_rel(ho['cls'][l].cpu(), cls[l]) for l in range(5)), bbox=max(_rel(ho['bbox'][l].cpu(), box[l]) for l in range(5)),
        cof=max(_rel(ho['cof'][l].cpu(), cof[l]) for l in range(5)), protos=_rel(ho['feat_masks'].float().cpu(), fm))
    k = int(out['count'][0])
    det_e = out['det_bboxes'][0, :k].cpu().numpy()
    lab_e = out['det_labels'][0, :k].cpu().numpy()
    det_r, lab_r = ref['det_bboxes'].numpy(), ref['det_labels'].numpy()
    masks_e = ops.unpack_mask_bits(out['mask_bits'][0, :k].cpu(), img_shape[1]).numpy().astype(bool)
    masks_r = ref['masks'].astype(bool)
    pairs = match_detections(det_e, lab_e, det_r, lab_r)
    ie = np.array([p[0] for p in pairs], int); ir = np.array([p[1] for p in pairs], int)
    miou = (np.logical_and(masks_e[ie], masks_r[ir]).sum((1, 2)) + 1e-9) / (np.logical_or(masks_e[ie], masks_r[ir]).sum((1, 2)) + 1e-9)
    rep.update(n_engine=int(k), n_oracle=int(det_r.shape[0]), matched=len(pairs),
               matched_frac=len(pairs) / max(1, det_r.shape[0]),
               box_linf=float(np.abs(det_e[ie, :4] - det_r[ir, :4]).max()) if pairs else None,
               score_absdiff=float(np.abs(det_e[ie, 4] - det_r[ir, 4]).max()) if pairs else None,
               mask_iou_min=float(miou.min()) if pairs else None, mask_iou_mean=float(miou.mean()) if pairs else None,
               mask_iou_pooled=float(np.logical_and(masks_e[ie], masks_r[ir]).sum() / max(1, np.logical_or(masks_e[ie], masks_r[ir]).sum()))
               if pairs else None,
               mask_iou_ge_0999=float((miou >= 0.999).mean()) if pairs else None,
               oracle_score_at_cut=float(det_r[:, 4].min()), oracle_score_max=float(det_r[:, 4].max()))
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    json.dump(rep, open(os.path.join(ROOT, 'gpurun_out', 'parity_fullsize_%s.json' % name), 'w'), indent=1)
    print(json.dumps(rep))
    return rep


def check(rep):
    h = rep['head_rel_l2']
    assert max(h['cls'], h['bbox'], h['cof'], h['protos']) < 5e-3, h
    assert rep['n_oracle'] > 0 and rep['n_engine'] > 0
    assert rep['matched_frac'] >= 0.95, rep
    assert rep['box_linf'] <= 1.0, rep
    assert rep['score_absdiff'] <= 2e-3, rep
    assert rep['mask_iou_pooled'] >= 0.995 and rep['mask_iou_mean'] >= 0.99 and rep['mask_iou_min'] >= 0.80, rep


CFG_A = dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
CFG_B = dict(nms_pre=1000, score_thr=0.1, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)


def test_fullsize_config_a_r50_800x1344():
    check(run_case('A_r50_800x1344', 50, 4, True, False, 800, 1344, 1333, CFG_A, cls_bias=-5.0))


def test_fullsize_config_a_r101_800x1344():
    check(run_case('A_r101_800x1344', 101, 4, True, False, 800, 1344, 1333, CFG_A, cls_bias=-5.0))


def test_fullsize_config_b_r50_544x544():
    check(run_case('B_r50_544x544', 50, 2, False, True, 544, 544, 544, CFG_B, cls_bias=-5.0,
                   scale_factor=np.ones(4, dtype=np.float32)))
