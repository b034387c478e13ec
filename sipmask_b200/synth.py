"""Seeded synthetic weights and inputs for the SipMask inference hot path.

There are no checkpoints or datasets in the build/measure environment, and the
reference's own `init_weights` produces a degenerate forward (all scores ~0.01
< score_thr, zero DCN offsets, dead residual branches; SURVEY.md §7 "Synthetic
weights").  This module generates a reference-keyed `state_dict`
(MM/mmdet/models/anchor_heads/sipmask_head.py:159-224,
 MM/mmdet/models/backbones/resnet.py:132-177,258-267,449-458,
 MM/mmdet/models/necks/fpn.py:86-129) whose forward exercises every branch:
non-trivial BN statistics, non-zero DCN offsets, and >= max_per_img detections.
The same dict loads into the reference modules, the oracle and the engine.
"""
import math

import torch

ARCH = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}
IMG_MEAN = (102.9801, 115.9465, 122.7717)   # MM/configs/sipmask/sipmask_r50_caffe_fpn_gn_1x.py:60-61


def _kaiming(g, cout, cin, k, gain=math.sqrt(2.0)):
    fan_in = cin * k * k
    return torch.randn(cout, cin, k, k, generator=g) * (gain / math.sqrt(fan_in))


def _bn(sd, prefix, c, g, gamma_scale=1.0):
    sd[prefix + '.weight'] = (0.5 + 0.5 * torch.rand(c, generator=g)) * gamma_scale
    sd[prefix + '.bias'] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + '.running_mean'] = 0.1 * torch.randn(c, generator=g)
    sd[prefix + '.running_var'] = 0.5 + torch.rand(c, generator=g)
    sd[prefix + '.num_batches_tracked'] = torch.tensor(0, dtype=torch.long)


def backbone_state_dict(depth=50, seed=1, prefix='backbone.', stage_with_dcn=(False,) * 4):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    sd[prefix + 'conv1.weight'] = _kaiming(g, 64, 3, 7) * 0.02      # inputs are 0..255-scale pixels
    _bn(sd, prefix + 'bn1', 64, g)
    inplanes = 64
    for i, nb in enumerate(ARCH[depth]):
        planes = 64 * 2 ** i
        for j in range(nb):
            p = '%slayer%d.%d.' % (prefix, i + 1, j)
            sd[p + 'conv1.weight'] = _kaiming(g, planes, inplanes, 1)
            _bn(sd, p + 'bn1', planes, g)
            sd[p + 'conv2.weight'] = _kaiming(g, planes, planes, 3)
            if stage_with_dcn[i] and j % 3 == 0:
                sd[p + 'conv2.conv_offset.weight'] = 0.02 * torch.randn(18, planes, 3, 3, generator=g)
                sd[p + 'conv2.conv_offset.bias'] = 0.1 * torch.randn(18, generator=g)
            _bn(sd, p + 'bn2', planes, g)
            sd[p + 'conv3.weight'] = _kaiming(g, planes * 4, planes, 1)
            _bn(sd, p + 'bn3', planes * 4, g, gamma_scale=0.25)
            if j == 0:
                sd[p + 'downsample.0.weight'] = _kaiming(g, planes * 4, inplanes, 1, gain=1.0)
                _bn(sd, p + 'downsample.1', planes * 4, g)
            inplanes = planes * 4
    return sd


def neck_state_dict(seed=2, prefix='neck.', in_channels=(512, 1024, 2048), out_channels=256, num_extra=2):
    g = torch.Generator().manual_seed(seed)
    sd = {}
    for i, c in enumerate(in_channels):
        sd['%slateral_convs.%d.conv.weight' % (prefix, i)] = _kaiming(g, out_channels, c, 1, gain=1.0)
        sd['%slateral_convs.%d.conv.bias' % (prefix, i)] = 0.05 * torch.randn(out_channels, generator=g)
    for i in range(len(in_channels) + num_extra):
        sd['%sfpn_convs.%d.conv.weight' % (prefix, i)] = _kaiming(g, out_channels, out_channels, 3, gain=1.0)
        sd['%sfpn_convs.%d.conv.bias' % (prefix, i)] = 0.05 * torch.randn(out_channels, generator=g)
    return sd


def head_state_dict(seed=3, prefix='bbox_head.', num_classes=81, feat=256, stacked_convs=4, gn=True,
                    rescoring_flag=False, cls_bias=-3.0, num_levels=5, track=False):
    g = torch.Generator().manual_seed(seed)
    sd = {}

    def convmod(name, cin, cout, k=3):
        sd[name + '.conv.weight'] = _kaiming(g, cout, cin, k)
        if gn:
            sd[name + '.gn.weight'] = 0.5 + torch.rand(cout, generator=g)
            sd[name + '.gn.bias'] = 0.2 * torch.randn(cout, generator=g)
        else:
            sd[name + '.conv.bias'] = 0.05 * torch.randn(cout, generator=g)

    for i in range(stacked_convs - 1):
        convmod('%scls_convs.%d' % (prefix, i), feat, feat)
    for i in range(stacked_convs):
        convmod('%sreg_convs.%d' % (prefix, i), feat, feat)
    ncls = num_classes - 1
    sd[prefix + 'fcos_cls.weight'] = _kaiming(g, ncls, feat, 3, gain=1.0)
    sd[prefix + 'fcos_cls.bias'] = torch.full((ncls,), float(cls_bias)) + 0.3 * torch.randn(ncls, generator=g)
    sd[prefix + 'fcos_reg.weight'] = _kaiming(g, 4, feat, 3, gain=1.0)
    sd[prefix + 'fcos_reg.bias'] = torch.full((4,), 2.0)           # positive distances -> non-empty boxes
    sd[prefix + 'fcos_centerness.weight'] = _kaiming(g, 1, feat, 3, gain=1.0)
    sd[prefix + 'fcos_centerness.bias'] = torch.zeros(1)
    for i in range(num_levels):
        sd['%sscales.%d.scale' % (prefix, i)] = torch.tensor(1.0 + 0.1 * i)
    sd[prefix + 'feat_align.conv_offset.weight'] = 0.05 * torch.randn(72, 4, 1, 1, generator=g)
    sd[prefix + 'feat_align.conv_adaption.weight'] = _kaiming(g, feat, feat, 3)
    sd[prefix + 'feat_align.norm.weight'] = 0.5 + torch.rand(feat, generator=g)
    sd[prefix + 'feat_align.norm.bias'] = 0.2 * torch.randn(feat, generator=g)
    sd[prefix + 'sip_cof.weight'] = _kaiming(g, 128, feat, 3, gain=1.0)
    sd[prefix + 'sip_cof.bias'] = 0.1 * torch.randn(128, generator=g)
    sd[prefix + 'sip_mask_lat.weight'] = _kaiming(g, 32, 512, 3)
    sd[prefix + 'sip_mask_lat.bias'] = 0.1 * torch.randn(32, generator=g)
    sd[prefix + 'sip_mask_lat0.weight'] = _kaiming(g, 512, 768, 1)
    sd[prefix + 'sip_mask_lat0.bias'] = 0.1 * torch.randn(512, generator=g)
    if rescoring_flag:
        ch = [1, 16, 16, 16, 32, 64, 128]
        for i in range(6):
            sd['%sconvs_scoring.%d.conv.weight' % (prefix, i)] = _kaiming(g, ch[i + 1], ch[i], 3)
            sd['%sconvs_scoring.%d.conv.bias' % (prefix, i)] = 0.05 * torch.randn(ch[i + 1], generator=g)
        sd[prefix + 'mask_scoring.weight'] = _kaiming(g, ncls, 128, 1)
        sd[prefix + 'mask_scoring.bias'] = 0.1 * torch.randn(ncls, generator=g)
    if track:                      # SipMask-VIS tracking branch (VIS/.../sipmask_head.py:274-287), drawn last: older seeds keep their values
        for i in range(stacked_convs - 1):
            convmod('%strack_convs.%d' % (prefix, i), feat, feat)
        sd[prefix + 'sipmask_track.weight'] = _kaiming(g, 512, 3 * feat, 1, gain=1.0)
        sd[prefix + 'sipmask_track.bias'] = 0.1 * torch.randn(512, generator=g)
    return sd


def detector_state_dict(depth=50, stacked_convs=4, gn=True, num_classes=81, rescoring_flag=False,
                        backbone_dcn=False, seed=1, cls_bias=-3.0):
    sd = {}
    sd.update(backbone_state_dict(depth, seed, stage_with_dcn=(False, backbone_dcn, backbone_dcn, backbone_dcn)))
    sd.update(neck_state_dict(seed + 1))
    sd.update(head_state_dict(seed + 2, num_classes=num_classes, stacked_convs=stacked_convs, gn=gn,
                              rescoring_flag=rescoring_flag, cls_bias=cls_bias))
    return sd


def detector_keys(depth=50, stacked_convs=4, gn=True, rescoring_flag=False, backbone_dcn=False, track=False,
                  num_levels=5):
    """The parameter / buffer names of an MM (track=True: SipMask-VIS) detector's state dict: the keys
    backbone_state_dict + neck_state_dict + head_state_dict write, without making the tensors."""
    bn = ('weight', 'bias', 'running_mean', 'running_var', 'num_batches_tracked')
    keys = ['backbone.conv1.weight'] + ['backbone.bn1.' + s for s in bn]
    for i, nb in enumerate(ARCH[depth]):
        for j in range(nb):
            p = 'backbone.layer%d.%d.' % (i + 1, j)
            keys += [p + 'conv1.weight', p + 'conv2.weight', p + 'conv3.weight']
            if backbone_dcn and i > 0 and j % 3 == 0:
                keys += [p + 'conv2.conv_offset.weight', p + 'conv2.conv_offset.bias']
            keys += [p + 'bn%d.%s' % (c, s) for c in (1, 2, 3) for s in bn]
            if j == 0:
                keys += [p + 'downsample.0.weight'] + [p + 'downsample.1.' + s for s in bn]
    keys += ['neck.lateral_convs.%d.conv.%s' % (i, s) for i in range(3) for s in ('weight', 'bias')]
    keys += ['neck.fpn_convs.%d.conv.%s' % (i, s) for i in range(5) for s in ('weight', 'bias')]
    h = 'bbox_head.'
    conv = ('conv.weight', 'gn.weight', 'gn.bias') if gn else ('conv.weight', 'conv.bias')
    towers = [('cls_convs', stacked_convs - 1), ('reg_convs', stacked_convs)]
    towers += [('track_convs', stacked_convs - 1)] if track else []
    for name, n in towers:
        keys += ['%s%s.%d.%s' % (h, name, i, c) for i in range(n) for c in conv]
    for m in ('fcos_cls', 'fcos_reg', 'fcos_centerness', 'sip_cof', 'sip_mask_lat', 'sip_mask_lat0', 'feat_align.norm'):
        keys += [h + m + '.weight', h + m + '.bias']
    keys += [h + 'feat_align.conv_offset.weight', h + 'feat_align.conv_adaption.weight']
    keys += [h + 'scales.%d.scale' % i for i in range(num_levels)]
    if rescoring_flag:
        keys += ['%sconvs_scoring.%d.conv.%s' % (h, i, s) for i in range(6) for s in ('weight', 'bias')]
        keys += [h + 'mask_scoring.weight', h + 'mask_scoring.bias']
    if track:
        keys += [h + 'sipmask_track.weight', h + 'sipmask_track.bias']
    return keys


def synthetic_image(h=800, w=1344, batch=1, seed=0):
    """uniform [0,255) BGR minus mean (SURVEY.md §8d); NCHW fp32."""
    g = torch.Generator().manual_seed(seed)
    img = torch.rand(batch, 3, h, w, generator=g) * 255.0
    return img - torch.tensor(IMG_MEAN).view(1, 3, 1, 1)


def img_meta(h=800, w=1333, pad_h=800, pad_w=1344, scale_factor=1.0):
    return dict(img_shape=(h, w, 3), ori_shape=(h, w, 3), pad_shape=(pad_h, pad_w, 3),
                scale_factor=scale_factor, flip=False)


def head_level_inputs(sizes, num_classes=80, seed=0, strides=(8, 16, 32, 64, 128)):
    """Head-output-level synthetic tensors for the post-processing kernels (SURVEY.md §8d):
    cls logits ~ N(-4,2), ctr ~ N(0,1), distances ~ |N(0, 4*stride)|, cofs ~ N(0,1)."""
    g = torch.Generator().manual_seed(seed)
    cls, box, ctr, cof = [], [], [], []
    for (h, w), s in zip(sizes, strides):
        cls.append(torch.randn(num_classes, h, w, generator=g) * 2.0 - 4.0)
        ctr.append(torch.randn(1, h, w, generator=g))
        box.append((torch.randn(4, h, w, generator=g) * 4.0 * s).abs())
        cof.append(torch.randn(128, h, w, generator=g))
    return cls, box, ctr, cof


def prototypes(h, w, seed=0):
    g = torch.Generator().manual_seed(seed + 100)
    return torch.relu(torch.randn(32, h, w, generator=g))
