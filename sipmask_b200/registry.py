"""Registry hook: make `type='SipMaskHead'` / `type='FCOSHead'` in an mmdetection config build the sm_90a heads.

The reference registers its heads with `@HEADS.register_module` (MM/mmdet/models/anchor_heads/sipmask_head.py:107-108,
MM/mmdet/utils/registry.py:24-48); duplicate names raise KeyError unless `force=True` (registry.py:39-42).
`register(force=True)` therefore *replaces* the two entries in an importable mmdet; configs, detectors
(`SingleStageDetector`), checkpoints and test scripts stay unchanged.
"""


def register(force=True):
    from mmdet.models.registry import HEADS       # raises ImportError when mmdet is not installed
    from .head import FCOSHead, SipMaskHead
    for cls in (SipMaskHead, FCOSHead):
        HEADS._register_module(cls, force=force) if hasattr(HEADS, '_register_module') else HEADS.register_module(cls)
    return HEADS


def register_ops(force=True, train=False):
    """Point `mmdet.ops.{CropSplit, DeformConv, nms}` at the sm_90a operators (same call signatures;
    MM/mmdet/ops/__init__.py:5-22 exports).

    train=True also binds the operators a fine-tuning step needs, with autograd on the device:
      * in mmdet.ops and its `dcn` / `sigmoid_focal_loss` submodules: DeformConv -> ops.TrainableDeformConv (ops.DeformConv
        runs without gradients), DeformConvPack, deform_conv, sigmoid_focal_loss, SigmoidFocalLoss;
      * mmdet.ops.conv.conv_cfg['DCN'] (the SipMask++ backbone builds its DCN blocks from it, ops/conv.py:9);
      * names bound at import time by modules already loaded: mmdet.models.losses.focal_loss._sigmoid_focal_loss and
        DeformConv / CropSplit / CropSplitGt in mmdet.models.anchor_heads.sipmask_head."""
    import sys
    import mmdet.ops as mmops
    from . import ops
    mmops.CropSplit = ops.CropSplit
    mmops.CropSplitGt = ops.CropSplitGt
    mmops.DeformConv = ops.TrainableDeformConv if train else ops.DeformConv
    mmops.nms = ops.nms
    for sub in ('crop', 'dcn', 'nms'):          # `from mmdet.ops.dcn import DeformConv` style imports
        m = getattr(mmops, sub, None)
        if m is not None:
            for name in ('CropSplit', 'CropSplitGt', 'DeformConv', 'nms'):
                if hasattr(m, name):
                    setattr(m, name, getattr(mmops, name))
    if train:
        bound = {'DeformConvPack': ops.DeformConvPack, 'deform_conv': ops.deform_conv,
                 'sigmoid_focal_loss': ops.sigmoid_focal_loss, 'SigmoidFocalLoss': ops.SigmoidFocalLoss}
        for name, obj in bound.items():
            setattr(mmops, name, obj)
        for sub, names in (('dcn', ('DeformConv', 'DeformConvPack', 'deform_conv')),
                           ('sigmoid_focal_loss', ('sigmoid_focal_loss', 'SigmoidFocalLoss'))):
            for mod in (getattr(mmops, sub, None), sys.modules.get('mmdet.ops.' + sub)):
                if mod is not None and not isinstance(mod, type(ops.sigmoid_focal_loss)):
                    for name in names:
                        setattr(mod, name, getattr(mmops, name))
        conv = sys.modules.get('mmdet.ops.conv')
        if conv is not None and hasattr(conv, 'conv_cfg'):
            conv.conv_cfg['DCN'] = ops.DeformConvPack
        focal = sys.modules.get('mmdet.models.losses.focal_loss')
        if focal is not None:
            focal._sigmoid_focal_loss = ops.sigmoid_focal_loss
        head = sys.modules.get('mmdet.models.anchor_heads.sipmask_head')
        if head is not None:
            head.DeformConv, head.CropSplit, head.CropSplitGt = ops.TrainableDeformConv, ops.CropSplit, ops.CropSplitGt
    return mmops
