"""Host-side checks of the training-side operators: register_ops(train=True) on a stub mmdet tree, and the argument
checks of deform_conv / sigmoid_focal_loss, which raise before anything is launched (no GPU needed)."""
import sys
import types

import pytest
import torch


def _stub_mmdet(monkeypatch):
    """The module layout of MM/VIS mmdet that register_ops touches: mmdet.ops re-exports its submodules' names (so
    `mmdet.ops.sigmoid_focal_loss` is the function, shadowing the submodule), conv.py keeps conv_cfg, focal_loss.py and
    sipmask_head.py bound their names at import time."""
    sentinel = {}

    def mod(name, **attrs):
        m = types.ModuleType(name)
        for k, v in attrs.items():
            setattr(m, k, v)
        monkeypatch.setitem(sys.modules, name, m)
        return m

    def orig(name):
        sentinel[name] = type('Orig' + name, (), {}) if name[0].isupper() else (lambda *a: None)
        return sentinel[name]

    names = ('DeformConv', 'DeformConvPack', 'deform_conv', 'CropSplit', 'CropSplitGt', 'nms', 'sigmoid_focal_loss',
             'SigmoidFocalLoss')
    for n in names:
        orig(n)
    mod('mmdet')
    dcn = mod('mmdet.ops.dcn', **{n: sentinel[n] for n in ('DeformConv', 'DeformConvPack', 'deform_conv')})
    sfl = mod('mmdet.ops.sigmoid_focal_loss', **{n: sentinel[n] for n in ('sigmoid_focal_loss', 'SigmoidFocalLoss')})
    conv = mod('mmdet.ops.conv', conv_cfg={'Conv': torch.nn.Conv2d, 'DCN': sentinel['DeformConvPack']})
    crop = mod('mmdet.ops.crop', CropSplit=sentinel['CropSplit'], CropSplitGt=sentinel['CropSplitGt'])
    mod('mmdet.ops.nms', nms=sentinel['nms'])
    ops = mod('mmdet.ops', dcn=dcn, conv=conv, crop=crop, **{n: sentinel[n] for n in names})
    sys.modules['mmdet'].ops = ops
    focal = mod('mmdet.models.losses.focal_loss', _sigmoid_focal_loss=sentinel['sigmoid_focal_loss'])
    head = mod('mmdet.models.anchor_heads.sipmask_head', DeformConv=sentinel['DeformConv'],
               CropSplit=sentinel['CropSplit'], CropSplitGt=sentinel['CropSplitGt'])
    return sentinel, dict(ops=ops, dcn=dcn, sfl=sfl, conv=conv, focal=focal, head=head)


def test_register_ops_train_binds_every_name(monkeypatch):
    from sipmask_b200 import ops, registry
    _, m = _stub_mmdet(monkeypatch)
    registry.register_ops(train=True)
    want = {'DeformConv': ops.TrainableDeformConv, 'DeformConvPack': ops.DeformConvPack, 'deform_conv': ops.deform_conv,
            'sigmoid_focal_loss': ops.sigmoid_focal_loss, 'SigmoidFocalLoss': ops.SigmoidFocalLoss}
    for name, obj in want.items():
        assert getattr(m['ops'], name) is obj, name
    for name in ('DeformConv', 'DeformConvPack', 'deform_conv'):
        assert getattr(m['dcn'], name) is want[name], name
    for name in ('sigmoid_focal_loss', 'SigmoidFocalLoss'):
        assert getattr(m['sfl'], name) is want[name], name
    assert m['conv'].conv_cfg['DCN'] is ops.DeformConvPack and m['conv'].conv_cfg['Conv'] is torch.nn.Conv2d
    assert m['focal']._sigmoid_focal_loss is ops.sigmoid_focal_loss
    assert m['head'].DeformConv is ops.TrainableDeformConv
    assert m['head'].CropSplit is ops.CropSplit and m['head'].CropSplitGt is ops.CropSplitGt
    assert m['ops'].CropSplit is ops.CropSplit and m['ops'].nms is ops.nms


def test_register_ops_default_leaves_training_names(monkeypatch):
    from sipmask_b200 import ops, registry
    orig, m = _stub_mmdet(monkeypatch)
    registry.register_ops()
    assert m['ops'].DeformConv is ops.DeformConv and m['dcn'].DeformConv is ops.DeformConv
    assert m['ops'].CropSplit is ops.CropSplit and m['ops'].nms is ops.nms
    for name in ('DeformConvPack', 'deform_conv', 'sigmoid_focal_loss', 'SigmoidFocalLoss'):
        assert getattr(m['ops'], name) is orig[name], name
    assert m['dcn'].DeformConvPack is orig['DeformConvPack'] and m['dcn'].deform_conv is orig['deform_conv']
    assert m['sfl'].sigmoid_focal_loss is orig['sigmoid_focal_loss']
    assert m['conv'].conv_cfg['DCN'] is orig['DeformConvPack']
    assert m['focal']._sigmoid_focal_loss is orig['sigmoid_focal_loss']
    assert m['head'].DeformConv is orig['DeformConv'] and m['head'].CropSplit is orig['CropSplit']


@pytest.fixture
def no_launch(monkeypatch):
    from sipmask_b200 import _lib

    def fail():
        raise AssertionError('the library was called')
    monkeypatch.setattr(_lib, 'lib', fail)


def test_deform_conv_rejects_before_launch(no_launch):
    from sipmask_b200 import ops, _lib
    x, off, w = torch.zeros(1, 64, 8, 8), torch.zeros(1, 18, 8, 8), torch.zeros(64, 64, 3, 3)
    with pytest.raises(_lib.SmbError, match='CUDA'):
        ops.deform_conv(x, off, w, 1, 1)
    with pytest.raises(_lib.SmbError, match='fp32'):
        ops.deform_conv(x.double(), off, w, 1, 1)
    with pytest.raises(_lib.SmbError, match='fp32'):
        ops.deform_conv(x, off, w.half(), 1, 1)
    for kw in (dict(stride=2), dict(padding=0), dict(dilation=2)):
        args = dict(stride=1, padding=1, dilation=1)
        args.update(kw)
        with pytest.raises(NotImplementedError):
            ops.deform_conv(x, off, w, args['stride'], args['padding'], args['dilation'])
    with pytest.raises(NotImplementedError):
        ops.deform_conv(x, off, torch.zeros(64, 64, 1, 1), 1, 1)
    with pytest.raises(NotImplementedError):                       # out_channels % 64
        ops.deform_conv(x, off, torch.zeros(48, 64, 3, 3), 1, 1)
    with pytest.raises(NotImplementedError):                       # (in_channels / deformable_groups) % 8
        ops.deform_conv(x, torch.zeros(1, 16 * 18, 8, 8), w, 1, 1, 1, 1, 16)
    with pytest.raises(_lib.SmbError, match='offset shape'):
        ops.deform_conv(x, torch.zeros(1, 36, 8, 8), w, 1, 1)
    with pytest.raises(AssertionError, match='im2col step'):
        ops.deform_conv(torch.zeros(3, 64, 8, 8), torch.zeros(3, 18, 8, 8), w, 1, 1, 1, 1, 1, 2)
    m = ops.DeformConvPack(64, 64, 3, padding=1)
    with pytest.raises(_lib.SmbError, match='CUDA'):
        m(x)


def test_sigmoid_focal_loss_rejects_before_launch(no_launch):
    from sipmask_b200 import ops, _lib
    t = torch.ones(4, dtype=torch.int64)
    for dt in (torch.float16, torch.float64, torch.bfloat16):
        with pytest.raises(_lib.SmbError, match='fp32'):
            ops.sigmoid_focal_loss(torch.zeros(4, 80, dtype=dt), t)
    with pytest.raises(_lib.SmbError, match='int64'):
        ops.sigmoid_focal_loss(torch.zeros(4, 80), t.int())
    with pytest.raises(_lib.SmbError, match='int64'):
        ops.sigmoid_focal_loss(torch.zeros(4, 80), torch.ones(5, dtype=torch.int64))
    with pytest.raises(_lib.SmbError, match='CUDA'):
        ops.sigmoid_focal_loss(torch.zeros(4, 80), t)
    with pytest.raises(_lib.SmbError, match='CUDA'):
        ops.SigmoidFocalLoss(2.0, 0.25)(torch.zeros(4, 80), t)
