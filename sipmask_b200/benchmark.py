"""SipMask-benchmark (the FCOS / maskrcnn-benchmark tree of the reference) checkpoints on the engine.

A BM checkpoint names its parameters `backbone.body.*`, `backbone.fpn.*` and `rpn.head.*`
(SipMask-benchmark/fcos_core/modeling/backbone/{resnet,fpn,backbone}.py, modeling/rpn/sipmask/sipmask.py).
`convert_state_dict` is the one place that knows that format: it returns the engine's key scheme, which the engine
(`SipMaskEngine(..., benchmark=True)`) and `oracle/benchmark.py` read.
"""
import re

import torch

from . import synth

# BM key (after the `module.` prefix is stripped) -> engine key
_RULES = [
    (r'backbone\.body\.stem\.(conv1\.weight|bn1\.(?:weight|bias|running_mean|running_var))$', r'backbone.\1'),
    (r'backbone\.body\.(layer\d\.\d+\.(?:conv\d\.weight|bn\d\.(?:weight|bias|running_mean|running_var)|downsample\.0\.weight'
     r'|downsample\.1\.(?:weight|bias|running_mean|running_var)))$', r'backbone.\1'),
    (r'backbone\.fpn\.fpn_inner([234])\.(weight|bias)$', lambda m: 'neck.lateral_convs.%d.conv.%s' % (int(m[1]) - 2, m[2])),
    (r'backbone\.fpn\.fpn_layer([234])\.(weight|bias)$', lambda m: 'neck.fpn_convs.%d.conv.%s' % (int(m[1]) - 2, m[2])),
    (r'backbone\.fpn\.top_blocks\.p6\.(weight|bias)$', r'neck.fpn_convs.3.conv.\1'),
    (r'backbone\.fpn\.top_blocks\.p7\.(weight|bias)$', r'neck.fpn_convs.4.conv.\1'),
    (r'rpn\.head\.(cls|bbox)_tower\.(\d+)\.(weight|bias)$', None),           # conv at 3i, GroupNorm at 3i+1
    (r'rpn\.head\.cls_logits\.(weight|bias)$', r'bbox_head.fcos_cls.\1'),
    (r'rpn\.head\.bbox_pred\.(weight|bias)$', r'bbox_head.fcos_reg.\1'),
    (r'rpn\.head\.centerness\.(weight|bias)$', r'bbox_head.fcos_centerness.\1'),
    (r'rpn\.head\.(feat_align\.conv_offset\.weight|feat_align\.conv_adaption\.(?:weight|bias)|feat_align\.norm\.(?:weight|bias)'
     r'|sip_cof\.(?:weight|bias)|sip_mask_lat0?\.(?:weight|bias)|scales\.\d\.scale)$', r'bbox_head.\1'),
]
_TRAINING_ONLY = re.compile(r'.*num_batches_tracked$')


def _tower(m):
    kind, idx, what = m[1], int(m[2]), m[3]
    name = 'cls_convs' if kind == 'cls' else 'reg_convs'
    if idx % 3 == 0:
        return 'bbox_head.%s.%d.conv.%s' % (name, idx // 3, what)
    if idx % 3 == 1:
        return 'bbox_head.%s.%d.gn.%s' % (name, idx // 3, what)
    return None


def _map_key(k):
    for pat, repl in _RULES:
        m = re.match(pat, k)
        if m is None:
            continue
        if repl is None:
            return _tower(m)
        return repl(m) if callable(repl) else m.expand(repl)
    return None


def expected_keys(depth=50, num_convs=4, num_levels=5):
    """Every engine key a BM detector of this depth needs."""
    keys = ['backbone.conv1.weight'] + ['backbone.bn1.' + s for s in ('weight', 'bias', 'running_mean', 'running_var')]
    for i, nb in enumerate(synth.ARCH[depth]):
        for j in range(nb):
            p = 'backbone.layer%d.%d.' % (i + 1, j)
            for c in (1, 2, 3):
                keys.append(p + 'conv%d.weight' % c)
                keys += [p + 'bn%d.%s' % (c, s) for s in ('weight', 'bias', 'running_mean', 'running_var')]
            if j == 0:
                keys.append(p + 'downsample.0.weight')
                keys += [p + 'downsample.1.' + s for s in ('weight', 'bias', 'running_mean', 'running_var')]
    for i in range(3):
        keys += ['neck.lateral_convs.%d.conv.%s' % (i, s) for s in ('weight', 'bias')]
    for i in range(5):
        keys += ['neck.fpn_convs.%d.conv.%s' % (i, s) for s in ('weight', 'bias')]
    h = 'bbox_head.'
    for name, n in (('cls_convs', num_convs - 1), ('reg_convs', num_convs)):
        for i in range(n):
            keys += ['%s%s.%d.%s.%s' % (h, name, i, m, s) for m in ('conv', 'gn') for s in ('weight', 'bias')]
    for m in ('fcos_cls', 'fcos_reg', 'fcos_centerness', 'feat_align.conv_adaption', 'feat_align.norm', 'sip_cof',
              'sip_mask_lat', 'sip_mask_lat0'):
        keys += [h + m + '.weight', h + m + '.bias']
    keys.append(h + 'feat_align.conv_offset.weight')
    keys += [h + 'scales.%d.scale' % i for i in range(num_levels)]
    return keys


def convert_state_dict(sd):
    """BM state dict (with or without the DDP `module.` prefix, utils/model_serialization.py:76) -> engine keys.
    Raises KeyError naming keys that have no mapping, that map twice, or that an inference key set lacks."""
    out, unknown = {}, []
    for k, v in sd.items():
        kk = k[len('module.'):] if k.startswith('module.') else k
        if _TRAINING_ONLY.match(kk):
            continue
        mk = _map_key(kk)
        if mk is None:
            unknown.append(k)
        elif mk in out:
            raise KeyError('BM checkpoint: %s maps to %s twice' % (k, mk))
        else:
            out[mk] = v
    if unknown:
        raise KeyError('BM checkpoint: keys without a mapping: %s' % ', '.join(sorted(unknown)))
    depth = 101 if 'backbone.layer3.22.conv1.weight' in out else 50
    num_convs = 1 + max([int(m[1]) for m in (re.match(r'bbox_head\.reg_convs\.(\d+)\.', k) for k in out) if m] + [-1])
    want = expected_keys(depth, num_convs)
    missing = [k for k in want if k not in out]
    if missing:
        raise KeyError('BM checkpoint: missing keys: %s' % ', '.join(missing))
    extra = sorted(set(out) - set(want))
    if extra:
        raise KeyError('BM checkpoint: keys outside a depth-%d, %d-conv detector: %s' % (depth, num_convs, ', '.join(
            k for k, v in sd.items() if _map_key(k[len('module.'):] if k.startswith('module.') else k) in extra)))
    return out


def to_bm_keys(sd_engine):
    """Inverse of convert_state_dict (engine keys -> BM keys); used to build BM-format dicts for tests and tools."""
    out = {}
    for k, v in sd_engine.items():
        m = re.match(r'bbox_head\.(cls|reg)_convs\.(\d+)\.(conv|gn)\.(weight|bias)$', k)
        if m:
            kind = 'cls' if m[1] == 'cls' else 'bbox'
            out['rpn.head.%s_tower.%d.%s' % (kind, 3 * int(m[2]) + (m[3] == 'gn'), m[4])] = v
            continue
        for a, b in (('backbone.conv1.', 'backbone.body.stem.conv1.'), ('backbone.bn1.', 'backbone.body.stem.bn1.'),
                     ('backbone.layer', 'backbone.body.layer'), ('bbox_head.fcos_cls.', 'rpn.head.cls_logits.'),
                     ('bbox_head.fcos_reg.', 'rpn.head.bbox_pred.'), ('bbox_head.fcos_centerness.', 'rpn.head.centerness.'),
                     ('neck.fpn_convs.3.conv.', 'backbone.fpn.top_blocks.p6.'),
                     ('neck.fpn_convs.4.conv.', 'backbone.fpn.top_blocks.p7.'), ('bbox_head.', 'rpn.head.')):
            if k.startswith(a):
                out[b + k[len(a):]] = v
                break
        else:
            m = re.match(r'neck\.(lateral|fpn)_convs\.(\d)\.conv\.(weight|bias)$', k)
            if not m:
                raise KeyError(k)
            out['backbone.fpn.fpn_%s%d.%s' % ('inner' if m[1] == 'lateral' else 'layer', int(m[2]) + 2, m[3])] = v
    return out


def synthetic_state_dict(depth=50, seed=1, cls_bias=-3.0):
    """Seeded BM-format detector dict (FrozenBatchNorm buffers, tower conv biases, DCN bias) whose forward gives
    detections, like synth.detector_state_dict for the MM tree."""
    sd = synth.detector_state_dict(depth=depth, seed=seed, cls_bias=cls_bias)
    sd = {k: v for k, v in sd.items() if not k.endswith('num_batches_tracked')}
    g = torch.Generator().manual_seed(seed + 10)
    for k in [k for k in sd if re.match(r'bbox_head\.(cls|reg)_convs\.\d+\.conv\.weight$', k)]:
        sd[k[:-len('weight')] + 'bias'] = 0.05 * torch.randn(sd[k].shape[0], generator=g)
    sd['bbox_head.feat_align.conv_adaption.bias'] = 0.05 * torch.randn(256, generator=g)
    for k in [k for k in sd if k.endswith('.scale')]:
        sd[k] = sd[k].reshape(1)                       # layers/scale.py:8: FloatTensor([init_value])
    return to_bm_keys(sd)


def check_options(centerness_on_reg=True, norm_reg_targets=True, use_dcn_in_tower=False, vis=False, rescoring=False):
    """The engine runs the two shipped BM configs (configs/sipmask/*.yaml); other head options raise ValueError."""
    if not centerness_on_reg:
        raise ValueError('benchmark: CENTERNESS_ON_REG=False is not supported (both shipped configs set it True)')
    if not norm_reg_targets:
        raise ValueError('benchmark: NORM_REG_TARGETS=False is not supported (both shipped configs set it True)')
    if use_dcn_in_tower:
        raise ValueError('benchmark: USE_DCN_IN_TOWER=True is not supported')
    if vis:
        raise ValueError('benchmark: vis=True is not supported (the BM tree has no tracking head)')
    if rescoring:
        raise ValueError('benchmark: rescoring_flag=True is not supported (the BM tree has no mask rescoring)')


# --------------------------------------------------------------------------------------------- drop-in module
class _Scale(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.scale = torch.nn.Parameter(torch.ones(1))          # layers/scale.py:8


class _FeatureAlign(torch.nn.Module):
    def __init__(self, c):
        super().__init__()
        self.conv_offset = torch.nn.Conv2d(4, 72, 1, bias=False)
        self.conv_adaption = torch.nn.Module()
        self.conv_adaption.weight = torch.nn.Parameter(torch.zeros(c, c, 3, 3))
        self.conv_adaption.bias = torch.nn.Parameter(torch.zeros(c))
        self.norm = torch.nn.GroupNorm(32, c)


class _Head(torch.nn.Module):
    """The reference SipMaskHead's parameters under its names (sipmask.py:48-125), so its state dict loads strictly."""

    def __init__(self, num_classes, c, num_convs):
        super().__init__()
        nn = torch.nn

        def tower(n):
            mods = []
            for _ in range(n):
                mods += [nn.Conv2d(c, c, 3, padding=1), nn.GroupNorm(32, c), nn.ReLU()]
            return nn.Sequential(*mods)
        self.cls_tower, self.bbox_tower = tower(num_convs - 1), tower(num_convs)
        self.cls_logits = nn.Conv2d(c, num_classes - 1, 3, padding=1)
        self.bbox_pred = nn.Conv2d(c, 4, 3, padding=1)
        self.centerness = nn.Conv2d(c, 1, 3, padding=1)
        self.feat_align = _FeatureAlign(c)
        self.sip_cof = nn.Conv2d(c, 128, 3, padding=1)
        self.sip_mask_lat = nn.Conv2d(512, 32, 3, padding=1)
        self.sip_mask_lat0 = nn.Conv2d(768, 512, 1)
        self.scales = nn.ModuleList([_Scale() for _ in range(5)])


class SipMaskModule(torch.nn.Module):
    """Drop-in for SipMask-benchmark's `SipMaskModule` (fcos_core/modeling/rpn/sipmask/sipmask.py:217-288), bound at
    `rpn.py:211-212` (`build_sipmask`).  Parameters carry the reference's names (`head.cls_tower.{0,1,3,4,...}`, ...).
    forward(images, features, img_metas) returns (boxlists, {}) like `_forward_test`: per image a BoxList in resized-image
    coordinates with fields labels (1-based), scores (sqrt), cofs and mask [k,1,ori_h,ori_w] uint8 (inference.py:143-222).
    The head runs on a head-only engine per feature-map size; the post-processing keeps every survivor of the k-th-value
    cut (no record capacity), so ties are kept as the reference keeps them."""

    MAX_ENGINES = 8

    def __init__(self, cfg, in_channels):
        super().__init__()
        s = cfg.MODEL.SIPMASK
        check_options(bool(s.CENTERNESS_ON_REG), bool(s.NORM_REG_TARGETS), bool(s.USE_DCN_IN_TOWER))
        if in_channels != 256:
            raise ValueError('benchmark.SipMaskModule: in_channels must be 256, got %d' % in_channels)
        self.num_classes, self.strides = int(s.NUM_CLASSES), tuple(int(v) for v in s.FPN_STRIDES)
        self.thr, self.nms_pre, self.nms_thr = float(s.INFERENCE_TH), int(s.PRE_NMS_TOP_N), float(s.NMS_TH)
        self.max_per_img = int(cfg.TEST.DETECTIONS_PER_IMG)
        self.head = _Head(self.num_classes, in_channels, int(s.NUM_CONVS))
        self._engines, self._wver = {}, None

    def _engine(self, features):
        from .engine import SipMaskEngine
        ver = tuple((p.data_ptr(), p._version) for p in self.parameters())
        if ver != self._wver:
            self._engines, self._wver = {}, ver
        sizes = tuple((f.shape[2], f.shape[3]) for f in features)
        key = (sizes, features[0].shape[0], features[0].device)
        if key not in self._engines:
            sd = convert_head_state_dict(self.head.state_dict())
            self._engines[key] = SipMaskEngine(sd, (8 * sizes[0][0], 8 * sizes[0][1]), batch=features[0].shape[0],
                                               num_classes=self.num_classes, strides=self.strides, head_only=True,
                                               feat_sizes=list(sizes), build_postproc=False, device=features[0].device,
                                               use_graph=False, benchmark=True)
            while len(self._engines) > self.MAX_ENGINES:
                self._engines.pop(next(iter(self._engines)))
        return self._engines[key]

    @torch.no_grad()
    def forward(self, images, features, img_metas=None, targets=None):
        if self.training or targets is not None:
            raise NotImplementedError('benchmark.SipMaskModule: training is not supported (inference only)')
        import numpy as np
        from fcos_core.structures.bounding_box import BoxList
        from . import ops
        eng = self._engine(features)
        eng.load_features(features)
        eng._run_ops()
        out = []
        for n, (h, w) in enumerate(images.image_sizes):
            views = [{k: t[n] for k, t in v.items()} for v in eng.level_views]
            b, sc, lab, loc, nc = ops.pair_decode_topk([v['cls'] for v in views], [v['box'] for v in views],
                                                       [v['ctr'] for v in views], self.strides, (h, w), self.nms_pre, self.thr,
                                                       box_scales=eng.scales)
            det, dl, idx, cnt, _ = ops.ml_nms_topk(b, sc, lab, nc, self.nms_thr, self.max_per_img)
            k = int(cnt.item())
            det, dl, idx = det[:k], dl[:k], idx[:k]
            cof_all = torch.cat([v['cof'].reshape(-1, 128) for v in views])
            cofs = cof_all[loc.long()[idx]]
            ow, oh = (img_metas[n] if img_metas is not None else (w, h))
            sf = np.minimum(h / oh, w / ow)                                  # inference.py:196
            bits = ops.mask_assemble_pack(eng.protos[n], cofs, det[:, :4], 0.5, (oh, ow), thr=0.4, layout='hwc',
                                          up=float(2 / sf)) if k else None
            mask = (ops.unpack_mask_bits(bits, ow)[:, None] if k else
                    torch.zeros((0, 1, oh, ow), dtype=torch.uint8, device=det.device))
            bl = BoxList(det[:, :4].clone(), (int(w), int(h)), mode='xyxy')
            bl.add_field('labels', dl + 1)
            bl.add_field('scores', det[:, 4].clone())
            bl.add_field('cofs', cofs)
            bl.add_field('mask', mask)
            out.append(bl)
        return out, {}


def convert_head_state_dict(head_sd):
    """The reference SipMaskHead's state dict (`cls_tower.0.weight`, ...) -> the head keys of the engine."""
    out = {}
    for k, v in head_sd.items():
        mk = _map_key('rpn.head.' + k)
        if mk is None:
            raise KeyError('SipMaskHead: key without a mapping: %s' % k)
        out[mk] = v
    return out
