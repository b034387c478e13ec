"""Drop-in heads with the reference's registry / module API, computed by the sm_90a kernels.

    SipMaskHead  <- MM/mmdet/models/anchor_heads/sipmask_head.py:107-287,500-662
    FCOSHead     <- MM/mmdet/models/anchor_heads/fcos_head.py:15-135,190-291

Same constructor keywords, same parameter names (a reference checkpoint `load_state_dict`s unchanged:
`cls_convs.{i}.conv.weight`, `cls_convs.{i}.gn.{weight,bias}`, `fcos_cls`, `scales.{i}.scale`,
`feat_align.conv_offset/conv_adaption/norm`, `sip_cof`, `sip_mask_lat`, `sip_mask_lat0`), same
`forward(feats)` / `get_bboxes(*outs, img_metas, cfg, rescale)` signatures and return structure as used by
`SingleStageDetector.simple_test` (MM/mmdet/models/detectors/single_stage.py:75-93).

The nn.Conv2d / nn.GroupNorm members only hold parameters; nothing here calls their forward.  Inference only:
`loss()` raises (training stays with the reference implementation).  CUDA sm_90 required - no CPU path.
"""
import numpy as np
import torch
import torch.nn as nn

from . import ops, postproc, rle
from .engine import SipMaskEngine

INF = 1e8


class _ConvModule(nn.Module):
    """Parameter container with the reference ConvModule's attribute names (`conv`, `gn`; ops/conv_module.py:68-100)."""

    def __init__(self, cin, cout, k=3, stride=1, padding=1, gn=True):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, k, stride=stride, padding=padding, bias=not gn)
        if gn:
            self.gn = nn.GroupNorm(32, cout)


class _Scale(nn.Module):
    def __init__(self, scale=1.0):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(scale, dtype=torch.float))


class _DeformConvParams(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(cout, cin, 3, 3))


class _FeatureAlign(nn.Module):
    def __init__(self, c, dg=4):
        super().__init__()
        self.conv_offset = nn.Conv2d(4, dg * 18, 1, bias=False)
        self.conv_adaption = _DeformConvParams(c, c)
        self.norm = nn.GroupNorm(32, c)


class _HeadBase(nn.Module):
    fcos = False
    MAX_ENGINES = 8          # COCO evaluation sees a handful of padded shapes; each engine owns ~0.3 GB of activations

    def _engine(self, feats):
        """Engine (launch plans + activation buffers) for this set of feature-map sizes.  Packed weights are cached once
        per parameter version and shared by all engines; engines live in a small LRU keyed by (sizes, device), so a change
        of input resolution does not repack / re-upload the weights, and a repeated resolution re-uses its plans."""
        from collections import OrderedDict
        sizes = tuple((f.shape[2], f.shape[3]) for f in feats)
        dev = feats[0].device
        ver = (self._param_version(), dev)
        if getattr(self, '_wver', None) != ver:
            self._wver, self._wcache, self._engines = ver, {}, OrderedDict()
        key = (sizes, dev)
        eng = self._engines.get(key)
        if eng is None:
            sd = {k: v.detach() for k, v in self.state_dict().items()}
            eng = SipMaskEngine(sd, (0, 0), batch=1, stacked_convs=self.stacked_convs,
                                gn=self.norm_cfg is not None, ssd_flag=getattr(self, 'ssd_flag', False),
                                num_classes=self.num_classes, strides=self.strides, device=dev,
                                use_graph=False, head_only=True, feat_sizes=sizes, in_channels=self.in_channels,
                                fcos=self.fcos, prefix_head='', build_postproc=False, share_weights=self._wcache,
                                vis=getattr(self, 'vis', False))
            self._engines[key] = eng
            while len(self._engines) > self.MAX_ENGINES:
                self._engines.popitem(last=False)
        else:
            self._engines.move_to_end(key)
        return eng

    def _run_images(self, feats, collect):
        """The engine processes one image per pass (imgs_per_gpu = 1 at test time, detectors/base.py:118-119); a batched
        call loops over the images.  `collect(eng)` returns the outputs of one image; they are CLONED because the engine's
        buffers are overwritten by the next pass."""
        eng = self._engine(feats)
        per_img = []
        for i in range(feats[0].shape[0]):
            eng.load_features([f[i:i + 1] for f in feats])
            eng._run_ops()
            per_img.append([[t.clone() for t in lst] if isinstance(lst, (list, tuple)) else lst.clone() for lst in collect(eng)])
        if len(per_img) == 1:
            return per_img[0]
        out = []
        for j in range(len(per_img[0])):
            col = [p[j] for p in per_img]
            out.append([torch.cat([c[l] for c in col], 0) for l in range(len(col[0]))] if isinstance(col[0], list)
                       else torch.cat(col, 0))
        return out

    def _param_version(self):
        return tuple(p._version for p in self.parameters())

    def loss(self, *args, **kwargs):
        raise NotImplementedError('sipmask_b200 heads are inference-only; train with the reference head '
                                  '(same parameter names, so checkpoints move both ways)')


class _ScoringConv(nn.Module):
    """Parameter holder with the reference's names: convs_scoring.{i}.conv.{weight,bias} (ConvModule, bias=True, no norm)."""

    def __init__(self, cin, cout):
        super().__init__()
        self.conv = nn.Conv2d(cin, cout, 3, stride=2, padding=0, bias=True)


class SipMaskHead(_HeadBase):
    def __init__(self, num_classes, in_channels, feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64),
                 regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)), center_sampling=False,
                 center_sample_radius=1.5, ssd_flag=False, rescoring_flag=False, loss_cls=None, loss_bbox=None,
                 loss_centerness=None, conv_cfg=None, norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)):
        super().__init__()
        if in_channels % 64 != 0 or feat_channels != 256:
            raise NotImplementedError('in_channels must be a multiple of 64 (one 128-byte K row of the implicit GEMM) and '
                                      'feat_channels 256 (GroupNorm-statistics epilogue: 8 channels per group; the prototype '
                                      'branch concatenates 3 x 256 channels, sipmask_head.py:197-198)')
        self.num_classes, self.cls_out_channels = num_classes, num_classes - 1
        self.in_channels, self.feat_channels, self.stacked_convs = in_channels, feat_channels, stacked_convs
        self.strides, self.regress_ranges = tuple(strides), regress_ranges
        self.ssd_flag, self.rescoring_flag = ssd_flag, rescoring_flag
        self.conv_cfg, self.norm_cfg = conv_cfg, norm_cfg
        self.fp16_enabled = False
        gn = norm_cfg is not None
        self.cls_convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else feat_channels, feat_channels, gn=gn)
                                        for i in range(stacked_convs - 1)])
        self.reg_convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else feat_channels, feat_channels, gn=gn)
                                        for i in range(stacked_convs)])
        self.fcos_cls = nn.Conv2d(feat_channels, self.cls_out_channels, 3, padding=1)
        self.fcos_reg = nn.Conv2d(feat_channels, 4, 3, padding=1)
        self.fcos_centerness = nn.Conv2d(feat_channels, 1, 3, padding=1)
        self.scales = nn.ModuleList([_Scale(1.0) for _ in self.strides])
        self.nc = 32
        self.feat_align = _FeatureAlign(feat_channels)
        self.sip_cof = nn.Conv2d(feat_channels, self.nc * 4, 3, padding=1)
        self.sip_mask_lat = nn.Conv2d(512, self.nc, 3, padding=1)
        self.sip_mask_lat0 = nn.Conv2d(768, 512, 1, padding=0)
        if rescoring_flag:                             # SipMask++ mask rescoring (sipmask_head.py:200-219)
            ch = [1, 16, 16, 16, 32, 64, 128]
            self.convs_scoring = nn.Sequential(*[_ScoringConv(ch[i], ch[i + 1]) for i in range(6)])
            self.mask_scoring = nn.Conv2d(128, self.cls_out_channels, 1)
        self.init_weights()

    def init_weights(self):
        """sipmask_head.py:226-239 (normal std 0.01, cls bias = -log(99), zero DCN offsets)."""
        for m in list(self.cls_convs) + list(self.reg_convs):
            nn.init.normal_(m.conv.weight, 0, 0.01)
        for m, std in ((self.fcos_cls, 0.01), (self.fcos_reg, 0.01), (self.fcos_centerness, 0.01), (self.sip_cof, 0.001),
                       (self.sip_mask_lat, 0.01), (self.sip_mask_lat0, 0.01)):
            nn.init.normal_(m.weight, 0, std)
            nn.init.constant_(m.bias, 0)
        nn.init.constant_(self.fcos_cls.bias, float(-np.log((1 - 0.01) / 0.01)))
        nn.init.constant_(self.feat_align.conv_offset.weight, 0.0)
        nn.init.normal_(self.feat_align.conv_adaption.weight, 0, 0.01)
        if self.rescoring_flag:
            for m in self.convs_scoring:
                nn.init.kaiming_normal_(m.conv.weight, mode='fan_out', nonlinearity='relu')
                nn.init.constant_(m.conv.bias, 0)
            nn.init.normal_(self.mask_scoring.weight, 0, 0.001)
            nn.init.constant_(self.mask_scoring.bias, 0)

    @torch.no_grad()
    def forward(self, feats):
        """feats: tuple of 5 NCHW CUDA tensors -> (cls_scores, bbox_preds, centernesses, cof_preds: lists of 5 NCHW
        fp32 tensors; feat_masks [N,32,4*h3,4*w3] fp16) - sipmask_head.py:241-287.  The returned tensors are the caller's
        (copies of the engine buffers); batches are processed image by image."""
        def collect(eng):
            o = eng.head_outputs()
            return o['cls'], o['bbox'], o['ctr'], o['cof'], o['feat_masks']
        return tuple(self._run_images(feats, collect))

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, centernesses, cof_preds, feat_masks, img_metas, cfg, rescale=None):
        """-> list over images of (det_bboxes [k,5], det_labels [k], cls_segms: list[num_classes-1] of RLE dicts),
        sipmask_head.py:500-541,645-662."""
        results = []
        for i in range(len(img_metas)):
            meta = img_metas[i]
            res = postproc.get_bboxes_single(
                [t[i] for t in cls_scores], [t[i] for t in bbox_preds], [t[i] for t in centernesses],
                [t[i] for t in cof_preds], feat_masks[i], self.strides, meta['img_shape'], meta['ori_shape'],
                meta['scale_factor'], cfg, rescale=rescale, ssd_flag=self.ssd_flag, pack=True,
                rescoring=self._rescoring_weights())
            k = int(res['count'])
            det_bboxes, det_labels = res['det_bboxes'][:k], res['det_labels'][:k]
            # RLE run lengths are computed on the device; the host receives a few KB of counts per detection (the
            # reference copies k dense masks, one synchronous 4.3 MB D2H each, and encodes them single-threaded)
            mh, mw = res['mask_hw']
            rles = ops.masks_to_rle(res['mask_bits'], mh, mw, k)
            labels = det_labels.cpu().numpy()
            cls_segms = [[] for _ in range(self.num_classes - 1)]
            for j in range(k):
                cls_segms[int(labels[j])].append(rles[j])
            if self.rescoring_flag:                      # (cls_segms, mask_scores) like sipmask_head.py:641-643,659-660
                ms = res['mask_scores'][:k].cpu().numpy()
                mask_scores = [ms[labels == c] for c in range(self.num_classes - 1)]
                results.append((det_bboxes, det_labels, (cls_segms, mask_scores)))
            else:
                results.append((det_bboxes, det_labels, cls_segms))
        return results

    def _rescoring_weights(self):
        if not self.rescoring_flag:
            return None
        return dict(conv_w=[m.conv.weight for m in self.convs_scoring], conv_b=[m.conv.bias for m in self.convs_scoring],
                    w1x1=self.mask_scoring.weight, b1x1=self.mask_scoring.bias)


class SipMaskVISHead(SipMaskHead):
    """Drop-in for the SipMask-VIS head (SipMask-VIS/mmdet/models/anchor_heads/sipmask_head.py:131-317,565-682; registered
    there under the same name `SipMaskHead`): tracking branch parameters `track_convs.{i}.conv/gn`, `sipmask_track`,
    `forward(feats, feats_x, flag_train)` -> 7-tuple, `get_bboxes(..., track_feats, track_feats_ref, img_metas, cfg, rescale)`
    -> [det_bboxes, det_labels, obj_segms {obj_id: RLE}, det_obj_ids] with the tracker state (`prev_*`) kept in the module
    like the reference keeps it.  Inference only (flag_train=True raises)."""
    vis = True

    def __init__(self, num_classes, in_channels, feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64),
                 regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)), center_sampling=False,
                 center_sample_radius=1.5, loss_cls=None, loss_bbox=None, loss_centerness=None, conv_cfg=None,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)):
        super().__init__(num_classes, in_channels, feat_channels=feat_channels, stacked_convs=stacked_convs, strides=strides,
                         regress_ranges=regress_ranges, center_sampling=center_sampling, center_sample_radius=center_sample_radius,
                         conv_cfg=conv_cfg, norm_cfg=norm_cfg)
        gn = norm_cfg is not None
        self.track_convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else feat_channels, feat_channels, gn=gn)
                                          for i in range(stacked_convs - 1)])
        self.sipmask_track = nn.Conv2d(feat_channels * 3, 512, 1, padding=0)
        self.match_coeff = [1.0, 2.0, 10]
        for m in self.track_convs:
            nn.init.normal_(m.conv.weight, 0, 0.01)
        from .tracker import Tracker
        self.tracker = Tracker(self.match_coeff)

    @torch.no_grad()
    def forward(self, feats, feats_x=None, flag_train=False):
        if flag_train:
            raise NotImplementedError('sipmask_b200 heads are inference-only (flag_train=False, single_stage.py:71)')

        def collect(eng):
            o = eng.head_outputs()
            return o['cls'], o['bbox'], o['ctr'], o['cof'], o['feat_masks'], o['track_feats']
        out = self._run_images(feats, collect)
        return tuple(out) + (out[5],)                       # track_feats_ref is track_feats at test time (VIS/...:317)

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, centernesses, cof_preds, feat_masks, track_feats, track_feats_ref, img_metas,
                   cfg, rescale=None):
        results = []
        for i in range(len(img_metas)):
            meta = img_metas[i]
            res = postproc.get_bboxes_single(
                [t[i] for t in cls_scores], [t[i] for t in bbox_preds], [t[i] for t in centernesses],
                [t[i] for t in cof_preds], feat_masks[i], self.strides, meta['img_shape'], meta['ori_shape'],
                meta['scale_factor'], cfg, rescale=bool(rescale), pack=True, vis=True, mask_thr=0.5, track_feats=track_feats[i])
            k = int(res['count'])
            det_bboxes, det_labels = res['det_bboxes'][:k], res['det_labels'][:k]
            if k == 0:                                       # VIS/...:605-608
                results.append([det_bboxes, det_labels, [[] for _ in range(self.num_classes - 1)], []])
                return results
            ids = self.tracker.step(det_bboxes.cpu().numpy(), det_labels.cpu().numpy(), res['track_feats'][:k].cpu().numpy(),
                                    bool(meta['is_first']))
            # the VIS reference always pastes into the ori_shape canvas (:669-674), also without rescale
            oh, ow = int(meta['ori_shape'][0]), int(meta['ori_shape'][1])
            mh, mw = res['mask_hw']
            rles = ops.masks_to_rle(res['mask_bits'], min(oh, mh), min(ow, mw), k) if (oh, ow) == (mh, mw) else \
                [rle.encode(_paste(ops.unpack_mask_bits(res['mask_bits'][j:j + 1], mw)[0].cpu().numpy(), oh, ow)) for j in range(k)]
            obj_segms = {}
            for j in range(k):
                if ids[j] >= 0:
                    obj_segms[int(ids[j])] = rles[j]
            results.append([det_bboxes, det_labels, obj_segms, ids])
        return results


def _paste(mask, oh, ow):
    im = np.zeros((oh, ow), np.uint8)
    hh, ww = min(mask.shape[0], oh), min(mask.shape[1], ow)
    im[:hh, :ww] = mask[:hh, :ww]
    return im


class FCOSHead(_HeadBase):
    fcos = True

    def __init__(self, num_classes, in_channels, feat_channels=256, stacked_convs=4, strides=(4, 8, 16, 32, 64),
                 regress_ranges=((-1, 64), (64, 128), (128, 256), (256, 512), (512, INF)), center_sampling=False,
                 center_sample_radius=1.5, loss_cls=None, loss_bbox=None, loss_centerness=None, conv_cfg=None,
                 norm_cfg=dict(type='GN', num_groups=32, requires_grad=True)):
        super().__init__()
        if in_channels % 64 != 0 or feat_channels != 256:
            raise NotImplementedError('in_channels must be a multiple of 64 and feat_channels 256 (GroupNorm-statistics epilogue)')
        self.num_classes, self.cls_out_channels = num_classes, num_classes - 1
        self.in_channels, self.feat_channels, self.stacked_convs = in_channels, feat_channels, stacked_convs
        self.strides, self.regress_ranges = tuple(strides), regress_ranges
        self.conv_cfg, self.norm_cfg = conv_cfg, norm_cfg
        self.fp16_enabled = False
        gn = norm_cfg is not None
        self.cls_convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else feat_channels, feat_channels, gn=gn)
                                        for i in range(stacked_convs)])
        self.reg_convs = nn.ModuleList([_ConvModule(in_channels if i == 0 else feat_channels, feat_channels, gn=gn)
                                        for i in range(stacked_convs)])
        self.fcos_cls = nn.Conv2d(feat_channels, self.cls_out_channels, 3, padding=1)
        self.fcos_reg = nn.Conv2d(feat_channels, 4, 3, padding=1)
        self.fcos_centerness = nn.Conv2d(feat_channels, 1, 3, padding=1)
        self.scales = nn.ModuleList([_Scale(1.0) for _ in self.strides])
        self.init_weights()

    def init_weights(self):
        for m in list(self.cls_convs) + list(self.reg_convs):
            nn.init.normal_(m.conv.weight, 0, 0.01)
        for m in (self.fcos_cls, self.fcos_reg, self.fcos_centerness):
            nn.init.normal_(m.weight, 0, 0.01)
            nn.init.constant_(m.bias, 0)
        nn.init.constant_(self.fcos_cls.bias, float(-np.log((1 - 0.01) / 0.01)))

    @torch.no_grad()
    def forward(self, feats):
        """-> (cls_scores, bbox_preds, centernesses), lists of 5 NCHW fp32 tensors (fcos_head.py:118-135)."""
        def collect(eng):
            cls, box, ctr = [], [], []
            for l, v in enumerate(eng.level_views):
                cls.append(v['cls'].permute(0, 3, 1, 2))
                ctr.append(v['ctr'].permute(0, 3, 1, 2))
                box.append((v['box'] * eng.scales[l]).exp().permute(0, 3, 1, 2))     # scale(x).float().exp() (:134)
            return cls, box, ctr
        return tuple(self._run_images(feats, collect))

    @torch.no_grad()
    def get_bboxes(self, cls_scores, bbox_preds, centernesses, img_metas, cfg, rescale=None):
        """-> list over images of (det_bboxes [k,5], det_labels [k]) - fcos_head.py:190-291."""
        from . import ops
        results = []
        for i in range(len(img_metas)):
            meta = img_metas[i]
            cl = [t[i].float().permute(1, 2, 0).contiguous() for t in cls_scores]
            bl = [t[i].float().permute(1, 2, 0).contiguous() for t in bbox_preds]
            tl = [t[i].float().permute(1, 2, 0).contiguous() for t in centernesses]
            sf = np.atleast_1d(np.asarray(meta['scale_factor'], dtype=np.float32))
            boxes, scores, ctr, _ = ops.decode_topk(cl, bl, tl, self.strides, meta['img_shape'], cfg.get('nms_pre', -1),
                                                    scale_factor=(sf if rescale else None))
            iou_thr = cfg['nms']['iou_thr'] if isinstance(cfg['nms'], dict) else cfg['nms'].iou_thr
            det, lab, _ = ops.multiclass_nms_idx(boxes, scores, cfg['score_thr'], dict(iou_thr=iou_thr),
                                                 int(cfg.get('max_per_img', 100)), score_factors=ctr, has_bg_column=False)
            results.append((det, lab))
        return results
