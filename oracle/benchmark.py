"""Oracle restatement of the SipMask-benchmark (BM) inference path (CPU, fp32).

TEST INFRASTRUCTURE ONLY - see oracle/__init__.py.
Paths are relative to /root/reference/SipMask-benchmark/fcos_core/.  Parameter names are the engine's (the output of
sipmask_b200.benchmark.convert_state_dict), so one converted dict loads into this oracle and the engine alike.

Orders the reference leaves to the implementation are fixed here, as the GPU kernels fix them:
- per level, when more than PRE_NMS_TOP_N pairs pass, the top-k keeps the largest sigmoid(cls) * sigmoid(ctr) with ties
  going to the lower pair index, and lists the kept pairs by ascending pair index loc * C + c (`topk(sorted=False)`,
  inference.py:116-118);
- ml_nms sorts by descending score with ties by ascending index (`scores.sort(0, descending=True)`, ml_nms.cu:78-80).
Sigmoids are 1 / (1 + exp(-x)) with exp evaluated in float64 and rounded to float32, the arithmetic of the kernels.
"""
import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import model as M
from . import ops as O
from .postproc import assemble_masks


# ------------------------------------------------------------------------------------------------ network
class FrozenBatchNorm2d(nn.Module):
    """layers/batch_norm.py:6-24: scale = weight * running_var.rsqrt() (no eps), bias = bias - running_mean * scale."""

    def __init__(self, n):
        super().__init__()
        for k, v in (('weight', torch.ones(n)), ('bias', torch.zeros(n)), ('running_mean', torch.zeros(n)),
                     ('running_var', torch.ones(n))):
            self.register_buffer(k, v)

    def forward(self, x):
        scale = self.weight * self.running_var.rsqrt()
        bias = self.bias - self.running_mean * scale
        return x * scale.reshape(1, -1, 1, 1) + bias.reshape(1, -1, 1, 1)


def _freeze_bn(module):
    for name, child in module.named_children():
        if isinstance(child, nn.BatchNorm2d):
            setattr(module, name, FrozenBatchNorm2d(child.num_features))
        else:
            _freeze_bn(child)


class FeatureAlign(nn.Module):
    """rpn/sipmask/sipmask.py:14-45: 1x1 offset conv on the ReLU'd regression, DCN (dg=4) WITH bias, GN, ReLU."""

    def __init__(self, c, dg=4):
        super().__init__()
        self.conv_offset = nn.Conv2d(4, dg * 18, 1, bias=False)
        self.conv_adaption = M._DeformConvW(c, c, dg)
        self.conv_adaption.bias = nn.Parameter(torch.zeros(c))
        self.norm = nn.GroupNorm(32, c)

    def forward(self, x, shape):
        offset = self.conv_offset(shape)
        y = self.conv_adaption(x, offset) + self.conv_adaption.bias.view(1, -1, 1, 1)
        return F.relu(self.norm(y))


class Scale(nn.Module):
    """layers/scale.py:5-11: a one-element parameter (shape [1], not a 0-d tensor as in MM)."""

    def __init__(self, init_value=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.FloatTensor([init_value]))

    def forward(self, x):
        return x * self.scale


class SipMaskHead(nn.Module):
    """rpn/sipmask/sipmask.py:48-214 with NORM_REG_TARGETS = CENTERNESS_ON_REG = True, USE_DCN_IN_TOWER = False: tower
    convs with bias AND GN, bbox = relu(scale * bbox_pred) (x stride for the output, unscaled into FeatureAlign)."""

    def __init__(self, num_classes=81, c=256, num_convs=4, strides=(8, 16, 32, 64, 128)):
        super().__init__()
        self.strides = strides
        self.cls_convs = nn.ModuleList([M.ConvModule(c, c, gn=True, bias=True) for _ in range(num_convs - 1)])
        self.reg_convs = nn.ModuleList([M.ConvModule(c, c, gn=True, bias=True) for _ in range(num_convs)])
        self.fcos_cls = nn.Conv2d(c, num_classes - 1, 3, padding=1)
        self.fcos_reg = nn.Conv2d(c, 4, 3, padding=1)
        self.fcos_centerness = nn.Conv2d(c, 1, 3, padding=1)
        self.scales = nn.ModuleList([Scale(1.0) for _ in strides])
        self.feat_align = FeatureAlign(c)
        self.sip_cof = nn.Conv2d(c, 128, 3, padding=1)
        self.sip_mask_lat = nn.Conv2d(512, 32, 3, padding=1)
        self.sip_mask_lat0 = nn.Conv2d(768, 512, 1)

    def forward(self, feats):
        logits, bbox_reg, centerness, cofs, feat_masks = [], [], [], [], []
        for l, x in enumerate(feats):
            cls_tower, box_tower = x, x
            for m in self.cls_convs:
                cls_tower = m(cls_tower)
            for m in self.reg_convs:
                box_tower = m(box_tower)
            centerness.append(self.fcos_centerness(box_tower))                     # :158-159
            bbox_pred = F.relu(self.scales[l](self.fcos_reg(box_tower)))           # :161-163
            bbox_reg.append(bbox_pred * self.strides[l])                           # :167
            cls_tower1 = self.feat_align(cls_tower, bbox_pred)                     # :171
            logits.append(self.fcos_cls(cls_tower1))
            cofs.append(self.sip_cof(cls_tower1))
            if l < 3:
                feat_masks.append(F.interpolate(box_tower, scale_factor=(2 ** l), mode='bilinear', align_corners=False))
        fm = torch.cat(feat_masks, dim=1)
        fm = F.relu(self.sip_mask_lat(F.relu(self.sip_mask_lat0(fm))))
        fm = F.interpolate(fm, scale_factor=4, mode='bilinear', align_corners=False)
        return logits, bbox_reg, centerness, cofs, fm


class SipMaskDetector(nn.Module):
    """ResNet (FrozenBatchNorm2d, stride in the 1x1, modeling/backbone/resnet.py) + FPN with P6 from P5 and ReLU before P7
    (modeling/backbone/fpn.py:51-100, backbone.py:50-72) + the head above."""

    def __init__(self, depth=50, num_classes=81):
        super().__init__()
        self.backbone = M.ResNet(depth)
        _freeze_bn(self.backbone)
        self.neck = M.FPN()
        self.bbox_head = SipMaskHead(num_classes)
        self.eval()

    def extract_feat(self, img):
        return self.neck(self.backbone(img))

    def forward(self, img):
        return self.bbox_head(self.extract_feat(img))


# ------------------------------------------------------------------------------------------- post-processor
def sigmoid_rn(x):
    x = np.asarray(x, dtype=np.float32)
    e = np.exp(-x.astype(np.float64)).astype(np.float32)
    return (np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32)


def pair_candidates(cls_scores, bbox_reg, centerness, strides, img_hw, thr=0.05, nms_pre=1000):
    """forward_for_single_feature_map (inference.py:66-141) for one image over all levels, concatenated
    (cat_boxlist).  Inputs per level CHW: logits [C,h,w], distances [4,h,w] (already relu'd and x stride), centerness
    [1,h,w].  Returns boxes [n,4] f32, scores [n] f32 (sqrt), labels [n] int64 (0-based), loc [n] int64 (level-concatenated
    location)."""
    out_b, out_s, out_l, out_loc = [], [], [], []
    base = 0
    h_img, w_img = int(img_hw[0]), int(img_hw[1])
    for cls, box, ctr, stride in zip(cls_scores, bbox_reg, centerness, strides):
        C, h, w = cls.shape
        s_cls = sigmoid_rn(cls.detach().permute(1, 2, 0).reshape(-1, C).numpy())
        s_ctr = sigmoid_rn(ctr.detach().reshape(-1).numpy())
        reg = box.detach().permute(1, 2, 0).reshape(-1, 4).numpy().astype(np.float32)
        cand = s_cls > np.float32(thr)                                          # :90
        prod = (s_cls * s_ctr[:, None]).astype(np.float32)                     # :93
        pairs = np.nonzero(cand.reshape(-1))[0]                                 # nonzero order = ascending loc*C + c
        if pairs.size > nms_pre:                                                # :116-123
            order = np.argsort(-prod.reshape(-1)[pairs], kind='stable')[:nms_pre]
            pairs = np.sort(pairs[order])
        loc, c = pairs // C, pairs % C
        points = O.get_points_single(h, w, stride).numpy()[loc]
        d = reg[loc]
        x1 = np.clip(points[:, 0] - d[:, 0], 0, w_img - 1)                      # :125-130, clip_to_image
        y1 = np.clip(points[:, 1] - d[:, 1], 0, h_img - 1)
        x2 = np.clip(points[:, 0] + d[:, 2], 0, w_img - 1)
        y2 = np.clip(points[:, 1] + d[:, 3], 0, h_img - 1)
        out_b.append(np.stack([x1, y1, x2, y2], 1).astype(np.float32))
        out_s.append(np.sqrt(prod.reshape(-1)[pairs]).astype(np.float32))      # :136
        out_l.append(c.astype(np.int64))
        out_loc.append((loc + base).astype(np.int64))
        base += h * w
    return (np.concatenate(out_b).reshape(-1, 4), np.concatenate(out_s), np.concatenate(out_l), np.concatenate(out_loc))


def ml_nms(boxes, scores, labels, iou_thr):
    """ml_nms_cuda (csrc/cuda/ml_nms.cu:13-135): greedy NMS in descending score order (ties: ascending index), IoU with
    +1 areas and 0 across labels, suppress when IoU > thr; kept indices ascending."""
    b = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    s = np.asarray(scores, dtype=np.float32)
    lab = np.asarray(labels)
    n = b.shape[0]
    one = np.float32(1.0)
    x1, y1, x2, y2 = b[:, 0], b[:, 1], b[:, 2], b[:, 3]
    areas = ((x2 - x1 + one) * (y2 - y1 + one)).astype(np.float32)
    order = np.argsort(-s, kind='stable')
    suppressed = np.zeros(n, dtype=bool)
    for _i in range(n):
        i = order[_i]
        if suppressed[i]:
            continue
        rest = order[_i + 1:]
        rest = rest[(lab[rest] == lab[i]) & ~suppressed[rest]]
        w = np.maximum(np.float32(0), (np.minimum(x2[i], x2[rest]) - np.maximum(x1[i], x1[rest]) + one).astype(np.float32))
        h = np.maximum(np.float32(0), (np.minimum(y2[i], y2[rest]) - np.maximum(y1[i], y1[rest]) + one).astype(np.float32))
        inter = (w * h).astype(np.float32)
        ovr = (inter / ((areas[i] + areas[rest]).astype(np.float32) - inter).astype(np.float32)).astype(np.float32)
        suppressed[rest[ovr > np.float32(iou_thr)]] = True
    return np.nonzero(~suppressed)[0].astype(np.int64)


def kth_value_cut(scores, keep, max_per_img):
    """select_over_all_levels (inference.py:182-190): with more than max_per_img survivors, keep the scores >= the
    max_per_img-th largest (ties can keep more), in survivor order."""
    k = keep.shape[0]
    if k > max_per_img > 0:
        sc = scores[keep]
        thr = np.sort(sc)[k - max_per_img]                                      # kthvalue(k - max_per_img + 1)
        keep = keep[sc >= thr]
    return keep


def select_over_all_levels(boxes, scores, labels, feat_mask, cofs, img_hw, ori_hw, nms_thr=0.6, max_per_img=100,
                           mask_thr=0.4):
    """inference.py:168-222 for one image.  cofs [n,128] of the candidates, feat_mask [32,Hm,Wm].  Returns dict(keep
    [k] candidate rows, det_bboxes [k,5], det_labels [k] 0-based, masks [k,ori_h,ori_w] uint8)."""
    keep = ml_nms(boxes, scores, labels, nms_thr)
    keep = kth_value_cut(scores, keep, max_per_img)
    det = np.concatenate([boxes[keep], scores[keep, None]], 1).astype(np.float32)
    oh, ow = int(ori_hw[0]), int(ori_hw[1])
    out = dict(keep=keep, det_bboxes=det, det_labels=labels[keep], masks=np.zeros((len(keep), oh, ow), np.uint8))
    if len(keep):
        sf = np.minimum(img_hw[0] / ori_hw[0], img_hw[1] / ori_hw[1])          # :196
        _, masks = assemble_masks(feat_mask.float(), torch.as_tensor(cofs[keep]).float(), torch.from_numpy(det[:, :4]),
                                  torch.tensor(0.5), up=float(2 / sf), thr=mask_thr)
        hh, ww = min(masks.shape[1], oh), min(masks.shape[2], ow)
        out['masks'][:, :hh, :ww] = masks.numpy()[:, :hh, :ww]
    return out


def postprocess(head_outs, img_hw, ori_hw, strides=(8, 16, 32, 64, 128), thr=0.05, nms_pre=1000, nms_thr=0.6,
                max_per_img=100, image=0):
    """SipMaskPostProcessor.forward (inference.py:143-166) for image `image` of the head outputs."""
    logits, bbox_reg, ctr, cofs, fm = head_outs
    b, s, lab, loc = pair_candidates([t[image] for t in logits], [t[image] for t in bbox_reg], [t[image] for t in ctr],
                                     strides, img_hw, thr, nms_pre)
    cof_all = torch.cat([c[image].detach().permute(1, 2, 0).reshape(-1, 128) for c in cofs], 0).numpy()
    res = select_over_all_levels(b, s, lab, fm[image].detach(), cof_all[loc], img_hw, ori_hw, nms_thr, max_per_img)
    res['cand'] = (b, s, lab, loc)
    return res
