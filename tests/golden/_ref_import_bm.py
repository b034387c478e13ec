"""Import shim that lets the *unmodified* SipMask-benchmark python (fcos_core) be imported in the build container, where
yacs, pycocotools and the compiled `fcos_core._C` extension are absent.

Test infrastructure only (used by tests/golden/gen_golden_bm.py to produce the committed ref_bm_*.npz fixtures).

What is stubbed or bound (no arithmetic of the inference path lives in the stubs):
  * yacs.config.CfgNode -> a dict with attribute access (enough for config/defaults.py to build its tree)
  * pycocotools, fcos_core._C -> inert mocks
  * DeformConv's `deform_conv` and the post-processor's CropSplit -> oracle.ops (both pinned against the reference's own
    CUDA kernels by tests/golden/ref_cuda_kernels.npz)
  * `ml_nms` -> oracle.benchmark.ml_nms (pinned separately: it equals the union over labels of the pinned `nms`)
"""
import importlib.abc
import importlib.machinery
import sys
import types
from unittest import mock

import torch

REF_BM = '/root/reference/SipMask-benchmark'


class CfgNode(dict):
    def __getattr__(self, k):
        try:
            return self[k]
        except KeyError:
            raise AttributeError(k)

    def __setattr__(self, k, v):
        self[k] = v


class _MockLoader(importlib.abc.Loader):
    def create_module(self, spec):
        m = mock.MagicMock(name=spec.name)
        m.__name__, m.__path__, m.__spec__, m.__loader__ = spec.name, [], spec, self
        return m

    def exec_module(self, module):
        pass


class _MockFinder(importlib.abc.MetaPathFinder):
    def find_spec(self, name, path, target=None):
        if name.split('.')[0] == 'pycocotools' or name == 'fcos_core._C':
            return importlib.machinery.ModuleSpec(name, _MockLoader(), is_package=True)
        return None


def load():
    """Returns (cfg, backbone module, sipmask module) of the reference with the bindings above."""
    if REF_BM not in sys.path:
        sys.path.insert(0, REF_BM)
    yacs, yc = types.ModuleType('yacs'), types.ModuleType('yacs.config')
    yc.CfgNode, yacs.config = CfgNode, yc
    sys.modules.setdefault('yacs', yacs)
    sys.modules.setdefault('yacs.config', yc)
    sys.meta_path.insert(0, _MockFinder())
    from oracle import benchmark as OB
    from oracle import ops as O
    from fcos_core.config import cfg
    from fcos_core.layers.dcn import deform_conv_module
    from fcos_core.modeling.backbone import backbone as BB
    from fcos_core.modeling.rpn.sipmask import sipmask as S
    from fcos_core.structures import boxlist_ops

    def deform_conv(x, offset, weight, stride, padding, dilation, groups, deformable_groups):
        one = lambda v: v[0] if isinstance(v, (tuple, list)) else v      # noqa: E731  (_pair'd by the module)
        assert groups == 1
        return O.deform_conv(x, offset, weight, one(stride), one(padding), one(dilation), deformable_groups)

    def ml_nms(boxes, scores, labels, thr):
        return torch.from_numpy(OB.ml_nms(boxes.numpy(), scores.numpy(), labels.numpy(), thr))

    deform_conv_module.deform_conv = deform_conv
    boxlist_ops._box_ml_nms = ml_nms
    # configs/sipmask/sipmask_R_50_FPN_1x.yaml
    cfg.MODEL.BACKBONE.CONV_BODY = 'R-50-FPN-RETINANET'
    cfg.MODEL.RESNETS.BACKBONE_OUT_CHANNELS = 256
    cfg.MODEL.RETINANET.USE_C5 = False
    cfg.MODEL.SIPMASK.NORM_REG_TARGETS = True
    cfg.MODEL.SIPMASK.CENTERNESS_ON_REG = True
    return cfg, BB, S


class CropSplitOracle(torch.nn.Module):
    def forward(self, data, rois):
        from oracle import ops as O
        return O.crop_split(data, rois, 2)
