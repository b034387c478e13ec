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


def register_ops(force=True):
    """Point `mmdet.ops.{CropSplit, DeformConv, nms}` at the sm_90a operators (same call signatures;
    MM/mmdet/ops/__init__.py:5-22 exports)."""
    import mmdet.ops as mmops
    from . import ops
    mmops.CropSplit = ops.CropSplit
    mmops.CropSplitGt = ops.CropSplitGt
    mmops.DeformConv = ops.DeformConv
    mmops.nms = ops.nms
    for sub in ('crop', 'dcn', 'nms'):          # `from mmdet.ops.dcn import DeformConv` style imports
        m = getattr(mmops, sub, None)
        if m is not None:
            for name in ('CropSplit', 'CropSplitGt', 'DeformConv', 'nms'):
                if hasattr(m, name):
                    setattr(m, name, getattr(ops, name))
    return mmops
