"""Reference configs -> engine and runner settings, checkpoints -> engine state dicts.

Three config trees are read:
  - 'mmdet'     : SipMask-mmdetection (mmdetection v1.1) `.py` configs, `data.test.type = 'CocoDataset'`;
  - 'vis'       : SipMask-VIS (mmdetection v1.0rc0) `.py` configs, `data.test.type = 'YTVOSDataset'`;
  - 'benchmark' : SipMask-benchmark `.yaml` configs, laid over the fcos_core defaults the engine depends on.
Everything the engine cannot run raises ValueError naming the config key: a config is either understood completely or
refused.  No file of the reference is read at run time.
"""
import os
import runpy
import types

import numpy as np

CAFFE_MEAN = [102.9801, 115.9465, 122.7717]
CAFFE_STD = [1.0, 1.0, 1.0]
STRIDES = (8, 16, 32, 64, 128)
# SipMaskHead's own default when a config does not set bbox_head.strides (SipMask-mmdetection sipmask_head.py:113,
# SipMask-VIS sipmask_head.py:130): a detector the engine does not build, refused like any other value
HEAD_DEFAULT_STRIDES = (4, 8, 16, 32, 64)

# SipMask-benchmark: the fcos_core/config/defaults.py values the engine depends on (a `.yaml` config overrides them)
BM_DEFAULTS = {
    'INPUT.MIN_SIZE_TEST': 800,                                  # defaults.py:53
    'INPUT.MAX_SIZE_TEST': 1333,                                 # defaults.py:55
    'INPUT.PIXEL_MEAN': [102.9801, 115.9465, 122.7717],          # defaults.py:57
    'INPUT.PIXEL_STD': [1., 1., 1.],                             # defaults.py:59
    'INPUT.TO_BGR255': True,                                     # defaults.py:61
    'DATALOADER.SIZE_DIVISIBILITY': 0,                           # defaults.py:81
    'MODEL.BACKBONE.CONV_BODY': 'R-50-C4',                       # defaults.py:97
    'MODEL.RESNETS.STAGE_WITH_DCN': (False, False, False, False),    # defaults.py:284
    'MODEL.SIPMASK.NUM_CLASSES': 81,                             # defaults.py:292
    'MODEL.SIPMASK.FPN_STRIDES': [8, 16, 32, 64, 128],           # defaults.py:293
    'MODEL.SIPMASK.INFERENCE_TH': 0.05,                          # defaults.py:295
    'MODEL.SIPMASK.NMS_TH': 0.6,                                 # defaults.py:296
    'MODEL.SIPMASK.PRE_NMS_TOP_N': 1000,                         # defaults.py:297
    'MODEL.SIPMASK.NUM_CONVS': 4,                                # defaults.py:305
    'MODEL.SIPMASK.NORM_REG_TARGETS': False,                     # defaults.py:312
    'MODEL.SIPMASK.CENTERNESS_ON_REG': False,                    # defaults.py:313
    'MODEL.SIPMASK.USE_DCN_IN_TOWER': False,                     # defaults.py:314
    'TEST.DETECTIONS_PER_IMG': 100,                              # defaults.py:487
    'TEST.BBOX_AUG.ENABLED': False,                              # defaults.py:497
    # the rest of the detector's structure: only the values of the shipped configs are run (BM_SHIPPED)
    'MODEL.RPN_ONLY': False,                                     # defaults.py:24
    'MODEL.MASK_ON': False,                                      # defaults.py:25
    'MODEL.FCOS_ON': False,                                      # defaults.py:26
    'MODEL.SIPMASK_ON': True,                                    # defaults.py:27
    'MODEL.RETINANET_ON': False,                                 # defaults.py:29
    'MODEL.META_ARCHITECTURE': 'GeneralizedRCNN',                # defaults.py:32
    'MODEL.FPN.USE_GN': False,                                   # defaults.py:109
    'MODEL.FPN.USE_RELU': False,                                 # defaults.py:110
    'MODEL.RESNETS.NUM_GROUPS': 1,                               # defaults.py:262
    'MODEL.RESNETS.WIDTH_PER_GROUP': 64,                         # defaults.py:265
    'MODEL.RESNETS.STRIDE_IN_1X1': True,                         # defaults.py:269
    'MODEL.RESNETS.TRANS_FUNC': 'BottleneckWithFixedBatchNorm',  # defaults.py:272
    'MODEL.RESNETS.STEM_FUNC': 'StemWithFixedBatchNorm',         # defaults.py:274
    'MODEL.RESNETS.RES5_DILATION': 1,                            # defaults.py:277
    'MODEL.RESNETS.BACKBONE_OUT_CHANNELS': 256 * 4,              # defaults.py:279
    'MODEL.RESNETS.RES2_OUT_CHANNELS': 256,                      # defaults.py:280
    'MODEL.RESNETS.STEM_OUT_CHANNELS': 64,                       # defaults.py:281
    'MODEL.RESNETS.WITH_MODULATED_DCN': False,                   # defaults.py:285
    'MODEL.RETINANET.USE_C5': True,                              # defaults.py:366
}
# the structure both shipped SipMask-benchmark configs give the detector (configs/sipmask/*.yaml over the defaults)
BM_SHIPPED = {
    'MODEL.RPN_ONLY': (True,), 'MODEL.MASK_ON': (False,), 'MODEL.FCOS_ON': (False,), 'MODEL.SIPMASK_ON': (True,),
    'MODEL.RETINANET_ON': (False,), 'MODEL.META_ARCHITECTURE': ('GeneralizedRCNN',), 'MODEL.FPN.USE_GN': (False,),
    'MODEL.FPN.USE_RELU': (False,), 'MODEL.RESNETS.NUM_GROUPS': (1,), 'MODEL.RESNETS.WIDTH_PER_GROUP': (64,),
    'MODEL.RESNETS.STRIDE_IN_1X1': (True,), 'MODEL.RESNETS.TRANS_FUNC': ('BottleneckWithFixedBatchNorm',),
    'MODEL.RESNETS.STEM_FUNC': ('StemWithFixedBatchNorm',), 'MODEL.RESNETS.RES5_DILATION': (1,),
    'MODEL.RESNETS.BACKBONE_OUT_CHANNELS': (256,), 'MODEL.RESNETS.RES2_OUT_CHANNELS': (256,),
    'MODEL.RESNETS.STEM_OUT_CHANNELS': (64,), 'MODEL.RESNETS.WITH_MODULATED_DCN': (False,),
    'MODEL.RETINANET.USE_C5': (False,),
}
BM_BODIES = {'R-50-FPN-RETINANET': 50, 'R-101-FPN-RETINANET': 101}


def load_config(path):
    """The config at `path` as a nested dict, with 'filename' set to the path.  `.py` configs (mmdetection v1.1 / v1.0rc0:
    flat files without `_base_`) are executed as mmcv.Config.fromfile executes them, so they must be trusted files, like
    any Python program; every module-level name not starting with '__' (and not a module) is kept.  `.yaml` configs
    (SipMask-benchmark) are read with PyYAML and laid over BM_DEFAULTS, as dotted keys under 'bm'."""
    path = os.fspath(path)
    if path.endswith('.py'):
        g = runpy.run_path(path)
        cfg = {k: v for k, v in g.items() if not k.startswith('__') and not isinstance(v, types.ModuleType)}
    elif path.endswith(('.yaml', '.yml')):
        import yaml
        with open(path) as f:
            raw = yaml.safe_load(f) or {}
        flat = dict(BM_DEFAULTS)

        def walk(d, prefix):
            for k, v in d.items():
                key = prefix + str(k)
                if isinstance(v, dict):
                    walk(v, key + '.')
                else:
                    flat[key] = v
        walk(raw, '')
        cfg = {'bm': flat}
    else:
        raise ValueError('config %s: a .py (mmdetection) or .yaml (SipMask-benchmark) file is needed' % path)
    cfg['filename'] = path
    return cfg


def tree(cfg):
    """'mmdet', 'vis' or 'benchmark'."""
    if 'bm' in cfg:
        return 'benchmark'
    kind = _get(cfg, 'data.test.type')
    if kind == 'CocoDataset':
        return 'mmdet'
    if kind == 'YTVOSDataset':
        return 'vis'
    raise ValueError("data.test.type %r: 'CocoDataset' (SipMask-mmdetection) or 'YTVOSDataset' (SipMask-VIS) is "
                     "supported" % (kind,))


_MISSING = object()


def _get(cfg, key, default=_MISSING):
    d = cfg
    for part in key.split('.'):
        if not isinstance(d, dict) or part not in d:
            if default is _MISSING:
                raise ValueError('config key %s is missing' % key)
            return default
        d = d[part]
    return d


def _want(key, value, allowed):
    if value not in allowed:
        raise ValueError('config key %s = %r is not supported (supported: %s)' % (key, value,
                                                                                 ' / '.join(repr(a) for a in allowed)))
    return value


def _same_floats(a, b):
    try:
        return len(a) == len(b) and np.allclose(np.asarray(a, np.float64), b, rtol=0, atol=1e-6)
    except TypeError:
        return False


def _test_cfg(tc, key='test_cfg'):
    if not isinstance(tc, dict):
        raise ValueError('config key %s must be a dict' % key)
    extra = sorted(set(tc) - {'nms_pre', 'min_bbox_size', 'score_thr', 'nms', 'max_per_img'})
    if extra:
        raise ValueError('config key %s.%s is not supported' % (key, extra[0]))
    nms = _get(tc, 'nms') if 'nms' in tc else None
    if not isinstance(nms, dict):
        raise ValueError('config key %s.nms must be a dict' % key)
    _want(key + '.nms.type', nms.get('type', 'nms'), ('nms', 'soft_nms'))
    out = {k: _get(tc, k) for k in ('nms_pre', 'score_thr', 'max_per_img')}
    out['nms'] = dict(nms)
    return out


# ------------------------------------------------------------------------------------------------ mmdet / vis models
def _model_kwargs(cfg):
    m = _get(cfg, 'model')
    _want('model.type', m.get('type'), ('SipMask',))
    b = _get(cfg, 'model.backbone')
    _want('model.backbone.type', b.get('type'), ('ResNet',))
    depth = _want('model.backbone.depth', b.get('depth'), (50, 101))
    _want('model.backbone.style', b.get('style', 'pytorch'), ('caffe',))
    _want('model.backbone.num_stages', b.get('num_stages', 4), (4,))
    _want('model.backbone.out_indices', tuple(b.get('out_indices', (0, 1, 2, 3))), ((0, 1, 2, 3),))
    _want('model.backbone.norm_cfg.type', (b.get('norm_cfg') or dict(type='BN')).get('type'), ('BN',))
    dcn = b.get('dcn')
    if dcn is None:
        backbone_dcn = False
        if any(b.get('stage_with_dcn', ())):
            raise ValueError('config key model.backbone.stage_with_dcn needs model.backbone.dcn')
    else:
        # mmdet's build_conv_layer: 'DCN' -> DeformConvPack, 'DCNv2' -> ModulatedDeformConvPack
        _want('model.backbone.dcn.type', dcn.get('type'), ('DCN',))
        _want('model.backbone.dcn.deformable_groups', dcn.get('deformable_groups', 1), (1,))
        _want('model.backbone.dcn.fallback_on_stride', dcn.get('fallback_on_stride', False), (False,))
        _want('model.backbone.stage_with_dcn', tuple(b.get('stage_with_dcn', (False,) * 4)), ((False, True, True, True),))
        backbone_dcn = True
    n = _get(cfg, 'model.neck')
    for k, v in (('type', 'FPN'), ('in_channels', [256, 512, 1024, 2048]), ('out_channels', 256), ('start_level', 1),
                 ('add_extra_convs', True), ('extra_convs_on_inputs', False), ('num_outs', 5),
                 ('relu_before_extra_convs', True)):
        got = list(n.get(k)) if isinstance(n.get(k), (list, tuple)) else n.get(k)
        _want('model.neck.' + k, got, (v,))
    h = _get(cfg, 'model.bbox_head')
    _want('model.bbox_head.type', h.get('type'), ('SipMaskHead',))
    _want('model.bbox_head.in_channels', h.get('in_channels', 256), (256,))
    _want('model.bbox_head.feat_channels', h.get('feat_channels', 256), (256,))
    norm = h.get('norm_cfg', dict(type='GN', num_groups=32))          # SipMaskHead's default
    if norm is not None:
        _want('model.bbox_head.norm_cfg.type', norm.get('type'), ('GN',))
        _want('model.bbox_head.norm_cfg.num_groups', norm.get('num_groups'), (32,))
    strides = tuple(h.get('strides', HEAD_DEFAULT_STRIDES))
    _want('model.bbox_head.strides', strides, (STRIDES,))
    return dict(depth=depth, backbone_dcn=backbone_dcn, stacked_convs=int(h.get('stacked_convs', 4)), gn=norm is not None,
                ssd_flag=bool(h.get('ssd_flag', False)), rescoring_flag=bool(h.get('rescoring_flag', False)),
                num_classes=int(_get(cfg, 'model.bbox_head.num_classes')), strides=strides,
                test_cfg=_test_cfg(_get(cfg, 'test_cfg')))


def _check_norm(norm, key):
    if not isinstance(norm, dict):
        raise ValueError('config key %s must be a dict' % key)
    if not _same_floats(norm.get('mean'), CAFFE_MEAN):
        raise ValueError('config key %s.mean = %r is not supported (the caffe mean %r)' % (key, norm.get('mean'), CAFFE_MEAN))
    if not _same_floats(norm.get('std'), CAFFE_STD):
        raise ValueError('config key %s.std = %r is not supported (%r)' % (key, norm.get('std'), CAFFE_STD))
    _want(key + '.to_rgb', norm.get('to_rgb', True), (False,))


def _one_scale(scale, key):
    if isinstance(scale, list):
        if len(scale) != 1:
            raise ValueError('config key %s holds %d test scales: multi-scale testing (aug_test) is not supported'
                             % (key, len(scale)))
        scale = scale[0]
    if not (isinstance(scale, tuple) and len(scale) == 2):
        raise ValueError('config key %s = %r: one (long, short) scale is needed' % (key, scale))
    return tuple(int(v) for v in scale)


def _mm_pipeline(cfg):
    """resize / keep_ratio of a v1.1 test pipeline: LoadImageFromFile, MultiScaleFlipAug(Resize, RandomFlip, Normalize, Pad,
    ImageToTensor, Collect)."""
    pipe = _get(cfg, 'data.test.pipeline')
    if len(pipe) != 2 or pipe[0].get('type') != 'LoadImageFromFile' or pipe[1].get('type') != 'MultiScaleFlipAug':
        raise ValueError('config key data.test.pipeline: LoadImageFromFile followed by MultiScaleFlipAug is supported, got %r'
                         % ([t.get('type') for t in pipe],))
    load = pipe[0]
    _want('data.test.pipeline.LoadImageFromFile.to_float32', load.get('to_float32', False), (False,))
    _want('data.test.pipeline.LoadImageFromFile.color_type', load.get('color_type', 'color'), ('color',))
    aug = pipe[1]
    _want('data.test.pipeline.MultiScaleFlipAug.flip', aug.get('flip', False), (False,))
    scale = _one_scale(aug.get('img_scale'), 'data.test.pipeline.MultiScaleFlipAug.img_scale')
    keep_ratio, divisor = None, None
    for t in aug.get('transforms', []):
        kind = t.get('type')
        key = 'data.test.pipeline.MultiScaleFlipAug.transforms.' + str(kind)
        extra = sorted(set(t) - {'type', 'keep_ratio', 'flip_ratio', 'size_divisor', 'mean', 'std', 'to_rgb', 'keys'})
        if extra:
            raise ValueError('config key %s.%s is not supported' % (key, extra[0]))
        if kind == 'Resize':
            keep_ratio = bool(t.get('keep_ratio', True))
        elif kind == 'RandomFlip':
            _want(key + '.flip_ratio', t.get('flip_ratio'), (None, 0, 0.0))
        elif kind == 'Normalize':
            _check_norm(t, key)
        elif kind == 'Pad':
            divisor = _want(key + '.size_divisor', t.get('size_divisor'), (32,))
        elif kind not in ('ImageToTensor', 'Collect'):
            raise ValueError('config key %s: transform %r is not supported' % (key, kind))
    if keep_ratio is None:
        raise ValueError('config key data.test.pipeline.MultiScaleFlipAug.transforms needs a Resize')
    if divisor is None and (keep_ratio or scale[0] % 32 or scale[1] % 32):
        raise ValueError('config key data.test.pipeline.MultiScaleFlipAug.transforms has no Pad(size_divisor=32) and '
                         'the resize does not give multiples of 32')
    return dict(resize=scale, keep_ratio=keep_ratio)


def _vis_pipeline(cfg):
    """resize / keep_ratio of a v1.0rc0 YTVOSDataset test entry (img_scale, img_norm_cfg, size_divisor, flip_ratio)."""
    t = _get(cfg, 'data.test')
    _want('data.test.flip_ratio', t.get('flip_ratio', 0), (0, 0.0))
    scale = _one_scale(t.get('img_scale'), 'data.test.img_scale')
    _check_norm(t.get('img_norm_cfg'), 'data.test.img_norm_cfg')
    _want('data.test.size_divisor', t.get('size_divisor'), (32,))
    return dict(resize=scale, keep_ratio=bool(t.get('resize_keep_ratio', True)))


# ------------------------------------------------------------------------------------------------ benchmark
def _bm_engine(cfg):
    from .benchmark import check_options
    c = cfg['bm']
    for k, allowed in BM_SHIPPED.items():
        _want(k, c[k], allowed)
    _want('DATALOADER.SIZE_DIVISIBILITY', c['DATALOADER.SIZE_DIVISIBILITY'], (32,))
    _want('TEST.BBOX_AUG.ENABLED', c['TEST.BBOX_AUG.ENABLED'], (False,))
    _want('INPUT.TO_BGR255', c['INPUT.TO_BGR255'], (True,))
    for k, ref in (('INPUT.PIXEL_MEAN', CAFFE_MEAN), ('INPUT.PIXEL_STD', CAFFE_STD)):
        if not _same_floats(c[k], ref):
            raise ValueError('config key %s = %r is not supported (%r)' % (k, c[k], ref))
    body = _want('MODEL.BACKBONE.CONV_BODY', c['MODEL.BACKBONE.CONV_BODY'], tuple(BM_BODIES))
    _want('MODEL.RESNETS.STAGE_WITH_DCN', tuple(c['MODEL.RESNETS.STAGE_WITH_DCN']), ((False,) * 4,))
    strides = tuple(c['MODEL.SIPMASK.FPN_STRIDES'])
    _want('MODEL.SIPMASK.FPN_STRIDES', strides, (STRIDES,))
    try:
        check_options(centerness_on_reg=c['MODEL.SIPMASK.CENTERNESS_ON_REG'],
                      norm_reg_targets=c['MODEL.SIPMASK.NORM_REG_TARGETS'],
                      use_dcn_in_tower=c['MODEL.SIPMASK.USE_DCN_IN_TOWER'])
    except ValueError as e:
        raise ValueError('config key MODEL.SIPMASK.%s' % str(e).split(': ', 1)[1])
    return dict(benchmark=True, depth=BM_BODIES[body], stacked_convs=int(c['MODEL.SIPMASK.NUM_CONVS']),
                num_classes=int(c['MODEL.SIPMASK.NUM_CLASSES']), strides=strides,
                test_cfg=dict(nms_pre=int(c['MODEL.SIPMASK.PRE_NMS_TOP_N']), score_thr=float(c['MODEL.SIPMASK.INFERENCE_TH']),
                              nms=dict(type='nms', iou_thr=float(c['MODEL.SIPMASK.NMS_TH'])),
                              max_per_img=int(c['TEST.DETECTIONS_PER_IMG'])))


# ------------------------------------------------------------------------------------------------ public mapping
def engine_kwargs(cfg):
    """SipMaskEngine keyword arguments of the config's detector (every value explicit, none left to the engine's
    defaults): depth, backbone_dcn, stacked_convs, gn, ssd_flag, rescoring_flag, vis, num_classes, strides and test_cfg
    for 'mmdet' / 'vis'; benchmark, depth, stacked_convs, num_classes, strides and test_cfg for 'benchmark'."""
    t = tree(cfg)
    if t == 'benchmark':
        return _bm_engine(cfg)
    kw = _model_kwargs(cfg)
    kw['vis'] = t == 'vis'
    if kw['vis'] and (kw['ssd_flag'] or kw['rescoring_flag']):
        raise ValueError('config key model.bbox_head: ssd_flag / rescoring_flag are not SipMask-VIS head options')
    return kw


def runner_kwargs(cfg):
    """The test transform as StreamRunner / VideoRunner keyword arguments: resize, keep_ratio (and raw=True, the PIL
    transform of SipMask-benchmark, with resize = (MAX_SIZE_TEST, MIN_SIZE_TEST))."""
    t = tree(cfg)
    if t == 'benchmark':
        c = cfg['bm']
        return dict(resize=(int(c['INPUT.MAX_SIZE_TEST']), int(c['INPUT.MIN_SIZE_TEST'])), keep_ratio=True, raw=True)
    return _vis_pipeline(cfg) if t == 'vis' else _mm_pipeline(cfg)


def expected_keys(cfg):
    """Every parameter / buffer name a checkpoint of the configured detector may hold (engine key scheme)."""
    from . import benchmark as B, synth
    kw = engine_kwargs(cfg)
    if kw.get('benchmark'):
        return set(B.expected_keys(kw['depth'], kw['stacked_convs']))
    return set(synth.detector_keys(kw['depth'], kw['stacked_convs'], kw['gn'], kw['rescoring_flag'], kw['backbone_dcn'],
                                   kw['vis']))


def load_checkpoint(path_or_dict, cfg):
    """(state_dict in the engine's key scheme, CLASSES or None) of a checkpoint of the configured detector.
      mmdet / vis: an mmcv checkpoint ({'state_dict', 'meta'}) or a bare state dict; a `module.` prefix is stripped and
                   meta['CLASSES'] returned when present.
      benchmark  : a SipMask-benchmark checkpoint ({'model', ...}) through benchmark.convert_state_dict.
    A path is read with torch.load, which unpickles: load trusted files only, as mmcv does.  Raises KeyError naming the
    keys the configured detector does not have (num_batches_tracked buffers excepted)."""
    import torch
    ck = torch.load(os.fspath(path_or_dict), map_location='cpu', weights_only=False) \
        if not isinstance(path_or_dict, dict) else path_or_dict
    kw = engine_kwargs(cfg)
    if kw.get('benchmark'):
        from .benchmark import convert_state_dict
        sd = convert_state_dict(ck['model'] if 'model' in ck else ck)
        classes = None
    else:
        sd = ck['state_dict'] if 'state_dict' in ck else ck
        sd = {(k[len('module.'):] if k.startswith('module.') else k): v for k, v in sd.items()}
        classes = (ck.get('meta') or {}).get('CLASSES') if 'state_dict' in ck else None
    known = expected_keys(cfg)
    unknown = sorted(k for k in sd if k not in known and not k.endswith('num_batches_tracked'))
    if unknown:
        raise KeyError('checkpoint keys the configured detector (%s) does not have: %s'
                       % (os.path.basename(cfg.get('filename', '')), ', '.join(unknown[:8])))
    return sd, (list(classes) if classes is not None else None)


RUNNERS = {'stream': 'StreamRunner', 'coco_eval': 'CocoEvalRunner', 'video': 'VideoRunner',
           'video_eval': 'VideoEvalRunner'}


def batch_defaults(cfg):
    """The runner's batching for the config: batch=32 for fixed-size resizes (the 544 x 544 configs), batch=1 with 6
    images in flight for keep-ratio resizes (800 x 1333), VideoRunner's own defaults for SipMask-VIS."""
    if tree(cfg) == 'vis':
        return {}
    return dict(batch=32) if not runner_kwargs(cfg)['keep_ratio'] else dict(batch=1, in_flight=6)


def from_config(cfg, checkpoint, kind='stream', **overrides):
    """The runner `kind` ('stream', 'coco_eval', 'video' or 'video_eval') of the config, serving `checkpoint` (a path,
    a checkpoint dict or, as load_checkpoint returns it, a (state_dict, classes) pair).  The engine settings are
    engine_kwargs(cfg), the transform runner_kwargs(cfg), the batching batch_defaults(cfg); `overrides` win, and carry
    the runner's own arguments (gt and cat_ids for 'coco_eval', gt for 'video_eval', max_src_hw, masks, ...)."""
    from . import serving
    if kind not in RUNNERS:
        raise ValueError('kind %r: one of %s' % (kind, ', '.join(RUNNERS)))
    if (tree(cfg) == 'vis') != kind.startswith('video'):
        raise ValueError("kind %r does not serve a %s config" % (kind, tree(cfg)))
    sd = checkpoint[0] if isinstance(checkpoint, tuple) else load_checkpoint(checkpoint, cfg)[0]
    kw = dict(engine_kwargs(cfg), **runner_kwargs(cfg))
    kw.update(batch_defaults(cfg))
    kw.update(overrides)
    cls = getattr(serving, RUNNERS[kind])
    if kind == 'coco_eval':
        return cls(sd, kw.pop('gt'), kw.pop('cat_ids'), **kw)
    if kind == 'video_eval':
        return cls(sd, kw.pop('gt'), **kw)
    return cls(sd, **kw)
