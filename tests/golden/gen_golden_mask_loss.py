"""Generate tests/golden/ref_mask_loss.npz by running the UNMODIFIED reference `SipMaskHead.loss` (SipMask-mmdetection,
rescoring off) on the CPU.

Run in the build container only (needs /root/reference):
    python tests/golden/gen_golden_mask_loss.py

The reference python is imported through tests/golden/_ref_import.py.  What is bound in place of native code or stubbed
(no arithmetic of the mask loss lives in any of it):
  * `crop_split_cuda.crop_split_cuda_forward` -> oracle.ops.crop_split (restatement of crop_split_cuda_kernel.cu:19-59);
  * `crop_split_cuda.crop_split_cuda_backward` -> the same cell geometry (oracle.ops.crop_split of planes holding their
    cell index + 1) scattering grad_output into its cell (crop_split_cuda_kernel.cu:90-133), so the golden carries
    gradients;
  * `crop_split_gt_cuda.crop_split_gt_cuda_forward` -> the inside-the-box copy (crop_split_gt_cuda_kernel.cu:19-50), with
    the inside test of the same restatement;
  * `six.moves.map` / `zip` in mmdet/core/utils/misc.py (six is an inert mock under the shim) -> the builtins, which
    is what six.moves gives on Python 3;
  * `loss_cls`, `loss_bbox`, `loss_centerness` -> zero (they are not under test; loss_cls would need the CUDA focal loss).
The head's intermediates (`det_bboxes`, `label_list`, `gt_inds`, from its own fcos_target / get_points / distance2bbox),
`loss_mask` and its gradients with respect to `feat_masks` and every level of `cof_preds` are stored.
"""
import os
import sys

import numpy as np
import torch
import torch.nn as nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import _ref_import  # noqa: E402

_ref_import.install()

from oracle import ops as O  # noqa: E402

OUT = os.path.join(HERE, 'ref_mask_loss.npz')
IMG = (64, 128)                               # padded image; feat_masks at stride 2
STRIDES = [8, 16, 32, 64, 128]


def _cell_plus_one(rois, H, W, N):
    """[H, W, N] int64: CropSplit's cell + 1 inside roi n, 0 outside (oracle.ops.crop_split on planes holding q + 1)"""
    planes = torch.arange(1, 5, dtype=torch.float32).view(4, 1, 1, 1).expand(4, H, W, N).contiguous()
    return O.crop_split(planes, rois.float(), 2).long()


def bind_crop():
    import mmdet.ops  # noqa: F401
    cs = sys.modules['mmdet.ops.crop.crop_split']
    csg = sys.modules['mmdet.ops.crop.crop_split_gt']

    def forward(data, rois, output, height, width, c, n):
        output.copy_(O.crop_split(data.detach(), rois.detach(), c))

    def backward(grad_output, rois, grad_input, height, width, c, n):
        if isinstance(rois, tuple):              # CropSplitFunction keeps _pair(rois): a tuple of the box rows
            rois = torch.stack(list(rois))
        cell = _cell_plus_one(rois, height, width, n)
        g = grad_output * (cell > 0)
        grad_input.scatter_add_(0, (cell - 1).clamp(min=0).unsqueeze(0), g.unsqueeze(0))

    def gt_forward(data, rois, output, height, width, c, n):
        output.copy_(torch.where(_cell_plus_one(rois, height, width, n) > 0, data, torch.zeros_like(data)))

    import mmdet.core.utils.misc as misc
    misc.map, misc.zip = map, zip
    cs.crop_split_cuda.crop_split_cuda_forward = forward
    cs.crop_split_cuda.crop_split_cuda_backward = backward
    csg.crop_split_gt_cuda.crop_split_gt_cuda_forward = gt_forward


class _Zero(nn.Module):
    def forward(self, x, *a, **k):
        return x.sum() * 0


def main():
    bind_crop()
    from mmdet.models.anchor_heads import sipmask_head as sh
    from mmdet.core import distance2bbox

    torch.manual_seed(0)
    rs = np.random.RandomState(0)
    head = sh.SipMaskHead(num_classes=81, in_channels=256, stacked_convs=1, strides=STRIDES, rescoring_flag=False)
    head.loss_cls, head.loss_bbox, head.loss_centerness = _Zero(), _Zero(), _Zero()
    B = 2
    sizes = [(-(-IMG[0] // s), -(-IMG[1] // s)) for s in STRIDES]
    cls_scores = [torch.tensor(rs.randn(B, 80, h, w), dtype=torch.float32) for h, w in sizes]
    bbox_preds = [torch.tensor(rs.uniform(4, 24, (B, 4, h, w)) * (s / 8), dtype=torch.float32)
                  for (h, w), s in zip(sizes, STRIDES)]
    centernesses = [torch.zeros(B, 1, h, w) for h, w in sizes]
    cof_preds = [torch.tensor(rs.uniform(-0.5, 0.5, (B, 128, h, w)), dtype=torch.float32).requires_grad_(True)
                 for h, w in sizes]
    feat_masks = torch.tensor(np.round(rs.uniform(-1, 1, (B, 32, IMG[0] // 2, IMG[1] // 2)) * 256) / 256,
                              dtype=torch.float32)
    feat_masks.requires_grad_(True)
    gt_bboxes, gt_labels, gt_masks = [], [], []
    for b in range(B):
        G = 4 - b
        xy = rs.uniform(0, [IMG[1] - 44, IMG[0] - 44], (G, 2))
        wh = rs.uniform(16, 42, (G, 2))
        gb = np.concatenate([xy, xy + wh], 1).astype(np.float32)
        m = np.zeros((G,) + IMG, dtype=np.uint8)
        yy, xx = np.mgrid[0:IMG[0], 0:IMG[1]]
        for g_ in range(G):
            cx, cy = (gb[g_, 0] + gb[g_, 2]) / 2, (gb[g_, 1] + gb[g_, 3]) / 2
            rx, ry = (gb[g_, 2] - gb[g_, 0]) / 2, (gb[g_, 3] - gb[g_, 1]) / 2
            m[g_] = ((xx - cx) / rx) ** 2 + ((yy - cy) / ry) ** 2 <= 1
        gt_bboxes.append(torch.from_numpy(gb))
        gt_labels.append(torch.from_numpy(rs.randint(1, 81, G)).long())
        gt_masks.append(m)

    captured = {}
    fcos_target = head.fcos_target

    def spy(*a, **k):
        r = fcos_target(*a, **k)
        captured['t'] = r
        return r
    head.fcos_target = spy
    img_metas = [dict(img_shape=IMG + (3,), pad_shape=IMG + (3,))] * B
    losses = head.loss(cls_scores, bbox_preds, centernesses, cof_preds, feat_masks, gt_bboxes, gt_labels, img_metas,
                       None, gt_masks_list=gt_masks)
    loss_mask = losses['loss_mask']
    loss_mask.backward()

    _, _, label_list, _, gt_inds = captured['t']
    points, _ = head.get_points([c.size()[-2:] for c in cls_scores], torch.float32, 'cpu')
    out = dict(feat_masks=feat_masks.detach().numpy(), loss_mask=np.float32(loss_mask.item()),
               d_feat_masks=feat_masks.grad.numpy(), num_levels=np.int64(len(STRIDES)), num_imgs=np.int64(B))
    for lv in range(len(STRIDES)):
        out['cls_scores_%d' % lv] = cls_scores[lv].numpy()
        out['cof_preds_%d' % lv] = cof_preds[lv].detach().numpy()
        out['d_cof_preds_%d' % lv] = cof_preds[lv].grad.numpy()
    for i in range(B):
        det = torch.cat([distance2bbox(points[lv], bbox_preds[lv][i].permute(1, 2, 0).reshape(-1, 4))
                         for lv in range(len(STRIDES))])
        out['det_bboxes_%d' % i] = det.numpy()
        out['gt_inds_%d' % i] = gt_inds[i].numpy()
        out['gt_bboxes_%d' % i] = gt_bboxes[i].numpy()
        out['gt_masks_%d' % i] = gt_masks[i]
        for lv in range(len(STRIDES)):
            out['labels_%d_%d' % (i, lv)] = label_list[i][lv].numpy()
    np.savez_compressed(OUT, **out)
    print('wrote %s: loss_mask %.6f, positives %s' % (OUT, loss_mask.item(), [int(len(g)) for g in gt_inds]))


if __name__ == '__main__':
    main()
