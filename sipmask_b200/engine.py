"""SipMask inference engine: the whole per-image hot path as a fixed sequence of sm_90a kernel launches.

    image (NCHW fp32) -> space-to-depth fp16 -> ResNet-50/101 (caffe, folded BN) -> FPN P3..P7 -> FCOS towers
    (conv+GN+ReLU) -> FeatureAlign (DCN) -> cls/centerness/reg/coefficient heads -> prototype branch -> decode/top-k ->
    NMS -> mask assembly -> x2 upsample + threshold (bit-packed)

Reference call stack replaced (SipMask-mmdetection/mmdet/): detectors/single_stage.py:75-93,
backbones/resnet.py:501-512, necks/fpn.py:138-178, anchor_heads/sipmask_head.py:241-287,500-662.
Weights come from a reference-keyed state_dict (SURVEY.md §8b); all buffers are allocated once, TMA descriptors
are baked into per-layer plans, and the launch sequence can be replayed as one CUDA graph.  Independent branches run on
side streams: the projection shortcut of residual stages 2-4, P5 -> P6 -> P7, the reg tower next to the cls tower, the
prototype branch next to FeatureAlign / the cls heads, and (batch > 1) the per-image post-processing chains.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from . import conv as C
from . import ops

ARCH = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}


class SipMaskEngine(object):
    def __init__(self, state_dict, img_hw, batch=1, depth=50, stacked_convs=4, gn=True, ssd_flag=False, num_classes=81,
                 strides=(8, 16, 32, 64, 128), test_cfg=None, img_shape=None, scale_factor=1.0, device='cuda',
                 mask_thr=0.4, use_graph=True, head_only=False, feat_sizes=None, in_channels=256,
                 fcos=False, prefix_head='bbox_head.', build_postproc=True, share_weights=None,
                 max_ctas=None, head_max_ctas=None, backbone_dcn=False, ori_shape=None, legacy_interp=False, vis=False,
                 rescoring_flag=False):
        self.dev = torch.device(device)
        if self.dev.index is None:
            self.dev = torch.device('cuda', torch.cuda.current_device())
        with torch.cuda.device(self.dev):
            L.check(L.lib().smb_check_device(), 'smb_check_device')
        self.N, (self.H, self.W) = batch, img_hw
        self.head_only, self.feat_sizes, self.in_channels, self.fcos = head_only, feat_sizes, in_channels, fcos
        self.hp, self.build_post = prefix_head, build_postproc
        # batch > 1: N images per forward (the reference's forward_test asserts imgs_per_gpu == 1, base.py:118-119, but
        # get_bboxes loops over images, sipmask_head.py:517-540; BASELINE config 4 is a bs=32 throughput mode)
        assert head_only or (self.H % 32 == 0 and self.W % 32 == 0), 'images are padded to a multiple of 32 (Pad size_divisor=32)'
        self.depth, self.stacked, self.gn, self.ssd = depth, stacked_convs, gn, ssd_flag
        # SipMask-VIS head (SipMask-VIS/mmdet/models/anchor_heads/sipmask_head.py): tracking branch, fast_nms with
        # cfg.score_thr / cfg.max_per_img, masks > 0.5, per-detection 512-d box-centre features in the result record
        self.vis = vis
        self.backbone_dcn = backbone_dcn           # SipMask++: DeformConvPack (dg=1) as conv2 of every 3rd block of stages 2-4
        self.ncls = num_classes - 1
        self.strides = tuple(strides)
        self.cfg = dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
        if test_cfg:
            self.cfg.update(test_cfg)
        self.img_shape = tuple(img_shape) if img_shape is not None else (self.H, self.W, 3)
        self.scale_factor = scale_factor
        # rescale=True semantics (SingleStageDetector.simple_test): boxes / scale_factor, masks resized by 2 / scale_factor and
        # pasted into the ori_shape canvas (sipmask_head.py:587-588,629-633,648-654)
        self.ori_shape = tuple(ori_shape) if ori_shape is not None else self.img_shape
        self.legacy_interp = legacy_interp
        self.mask_thr = 0.5 if (vis and mask_thr == 0.4) else mask_thr      # VIS thresholds at 0.5 (VIS/...:764), MM at 0.4
        self.sd = {k: v for k, v in state_dict.items()}
        # SipMask++ mask rescoring (sipmask_head.py:200-219,635-643): a mask score per detection in the result record
        self.rescoring = rescoring_flag
        if rescoring_flag:
            self._check_rescoring()
        self.ops = []            # list of zero-argument callables = the launch sequence
        self.op_names = []
        self.op_tags = []        # 0 = main stream, 1 = side stream, 'fork' / 'join' = stream dependencies
        self._tag = 0
        self._max_ctas = max_ctas
        self.side_stream = None
        self.n_launch = 0
        self._keep = []
        # packed weights; `share_weights=<engine>` makes several engines (images in flight) read ONE copy, so the weights'
        # L2 footprint does not grow with the number of images in flight
        self._wcache = ({} if share_weights is None else share_weights if isinstance(share_weights, dict)
                        else share_weights._wcache)
        self.max_ctas = max_ctas                   # persistent-grid cap of every conv (None: all SMs)
        self.head_max_ctas = head_max_ctas         # cap inside the two-stream head section (None: 100)
        self.conv_plans = []
        self.conv_meta = []
        self.conv_flops = 0.0
        self.rescore_flops = 0.0                   # mask rescoring, kept apart from the convolution roofline
        with torch.cuda.device(self.dev):
            self._build()
        self.graph = None
        self.use_graph = use_graph

    def _check_rescoring(self):
        if self.vis:
            raise ValueError('rescoring_flag=True: the SipMask-VIS head has no mask rescoring')
        keys = ['%sconvs_scoring.%d.conv.%s' % (self.hp, i, k) for i in range(6) for k in ('weight', 'bias')]
        missing = [k for k in keys + [self.hp + 'mask_scoring.weight', self.hp + 'mask_scoring.bias'] if k not in self.sd]
        if missing:
            raise ValueError('rescoring_flag=True needs the SipMask++ scoring weights; missing: %s' % ', '.join(missing))
        h3, w3 = self.feat_sizes[0] if self.head_only else (self.H // 8, self.W // 8)
        if min(4 * h3, 4 * w3) < 127:               # prototypes are 4x P3; six valid stride-2 3x3 convs need 127 pixels
            raise ValueError('rescoring_flag=True needs prototypes of at least 127 x 127, got %d x %d' % (4 * h3, 4 * w3))

    # ------------------------------------------------------------------------------------------ helpers
    def _t(self, *shape, dtype=torch.float16, zero=False):
        t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=self.dev)
        self._keep.append(t)
        return t

    def _w(self, key):
        return self.sd[key].detach().float().cpu()

    def _bn(self, prefix):
        return (self._w(prefix + '.weight'), self._w(prefix + '.bias'), self._w(prefix + '.running_mean'),
                self._w(prefix + '.running_var'))

    def _add(self, fn, launches=1, name=None):
        self.ops.append(fn)
        self.op_names.append(name or getattr(fn, '__name__', 'op'))
        self.op_tags.append(self._tag)
        self.n_launch += launches

    def _marker(self, kind):
        self.ops.append(None)
        self.op_names.append(kind)
        self.op_tags.append(kind)

    def _conv(self, x, wkey, k, stride=1, relu=False, bn=None, bias_key=None, residual=None, residual_upsample=False,
              gn_stats=None, out=None, out_dtype=torch.float16, cout_pad=None, weight=None, bias=None, cin=None,
              cout_real=None):
        if weight is None:
            ck = (wkey, bn, bias_key, cout_pad)
            if ck not in self._wcache:           # tower weights are shared by the five pyramid levels
                weight, b = C.pack_weight(self._w(wkey), bn=self._bn(bn) if bn else None, cout_pad=cout_pad, device=self.dev)
                if bias_key is not None:
                    b = self._w(bias_key)
                    if cout_pad and cout_pad != b.numel():
                        b = torch.cat([b, b.new_zeros(cout_pad - b.numel())])
                    b = b.to(self.dev).contiguous()
                self._wcache[ck] = (weight, b)
            weight, bias = self._wcache[ck]
        N, H, W, _ = x.shape
        Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
        if out is None:
            out = self._t(N, Ho, Wo, weight.shape[0], dtype=out_dtype)
        plan = C.ConvPlan(x, weight, out, k, stride, relu=relu, bias=bias, residual=residual,
                          residual_upsample=residual_upsample, gn_stats=gn_stats, cin=cin)
        if self._max_ctas:
            plan.set_max_ctas(self._max_ctas)
        self._keep.append(plan)
        self.conv_plans.append(plan)
        fl = 2.0 * N * Ho * Wo * (cout_real or weight.shape[0]) * weight.shape[1]                 # algorithmic FLOPs
        self.conv_flops += fl
        self.conv_meta.append(dict(name=wkey or 'shared', M=N * Ho * Wo, N=weight.shape[0], K=weight.shape[1], k=k, stride=stride,
                                   flops=fl, res=residual is not None, gn=gn_stats is not None))
        self._add(plan.run, name='conv')
        return out

    # -------------------------------------------------------------------------------------------- build
    def _build(self):
        N, H, W = self.N, self.H, self.W
        if self.head_only:
            # drop-in head: the five FPN levels come from the caller (reference backbone/neck), NHWC fp16 copies
            self.fpn_outs = [self._t(N, h, w, self.in_channels) for (h, w) in self.feat_sizes]
            if self.fcos:
                self._build_fcos_head(self.fpn_outs)
            else:
                self._build_head(self.fpn_outs)
            return
        self.img = self._t(N, 3, H, W, dtype=torch.float32)
        # ---- stem: space-to-depth input [N,H/2+3,W/2+4,16], K = 256
        img8 = self._t(N, H // 2 + 3, W // 2 + 4, 16)
        self.img8 = img8
        self._add(lambda: C.image_to_s2d16(self.img, img8), name='image_to_s2d16')
        wk, b = self._once('stem_s2d', lambda: C.pack_stem_weight_s2d(self._w('backbone.conv1.weight'), self._bn('backbone.bn1'),
                                                                      device=self.dev))
        s1 = self._t(N, H // 2, W // 2, 64)
        stem = C.StemPlan(img8, wk, b, s1, N, H, W)
        self._keep += [stem, wk, b]
        self.conv_plans.append(stem)
        fl = 2.0 * N * (H // 2) * (W // 2) * 64 * 147                                 # algorithmic 7x7x3 (executed K is 256)
        self.conv_flops += fl
        self.conv_meta.append(dict(name='stem', M=N * (H // 2) * (W // 2), N=64, K=256, k=7, stride=2, flops=fl,
                                   res=False, gn=False))
        self._add(stem.run, name='conv')
        x = self._t(N, H // 4, W // 4, 64)
        self._add(lambda s1=s1, x=x: C.maxpool3x3s2(s1, x), name='maxpool')
        # ---- residual stages (caffe style: stride on conv1, resnet.py:125-130)
        feats = []
        for i, nb in enumerate(ARCH[self.depth]):
            for j in range(nb):
                p = 'backbone.layer%d.%d.' % (i + 1, j)
                stride = 2 if (j == 0 and i > 0) else 1
                # the projection shortcut only depends on the block input: it runs on the side stream next to conv1/conv2
                # (layers 2-4 are short latency-bound launches that leave most SMs idle)
                side = j == 0 and i >= 1
                if side:
                    self._marker('fork')
                    self._tag = 1
                    idn = self._conv(x, p + 'downsample.0.weight', 1, stride, relu=False, bn=p + 'downsample.1')
                    self._tag = 0
                t1 = self._conv(x, p + 'conv1.weight', 1, stride, relu=True, bn=p + 'bn1')
                if self.backbone_dcn and i >= 1 and j % 3 == 0:
                    # DeformConvPack (resnet.py:146-168,288-291; dcn/deform_conv.py:258-296): 18 offsets from a 3x3 conv
                    # with bias (fp32 out), dg=1 bilinear gather into the column layout, then the 3x3 weights as a GEMM
                    off = self._conv(t1, p + 'conv2.conv_offset.weight', 3, 1, bias_key=p + 'conv2.conv_offset.bias',
                                     out_dtype=torch.float32, cout_pad=32, cout_real=18)
                    col = self._t(N, t1.shape[1], t1.shape[2], 9 * t1.shape[3])
                    self._add(lambda t1=t1, off=off, col=col: C.deform_im2col(t1, off, 1, out=col), name='deform_im2col')
                    t2 = self._conv(col, p + 'conv2.weight', 1, 1, relu=True, bn=p + 'bn2')
                else:
                    t2 = self._conv(t1, p + 'conv2.weight', 3, 1, relu=True, bn=p + 'bn2')
                if side:
                    self._marker('join')
                elif j == 0:
                    idn = self._conv(x, p + 'downsample.0.weight', 1, stride, relu=False, bn=p + 'downsample.1')
                else:
                    idn = x
                x = self._conv(t2, p + 'conv3.weight', 1, 1, relu=True, bn=p + 'bn3', residual=idn)
            feats.append(x)
        c3, c4, c5 = feats[1], feats[2], feats[3]
        # ---- FPN (fpn.py:138-178): laterals top-down with the nearest-upsample add fused into the epilogue
        lat5 = self._conv(c5, 'neck.lateral_convs.2.conv.weight', 1, bias_key='neck.lateral_convs.2.conv.bias')
        # P5 -> P6 -> P7 is a chain of tiny convolutions (9 / 3 / 1 M-tiles): side stream, next to the P4 / P3 laterals
        self._marker('fork')
        self._tag = 1
        p5, p6, p7 = self._fpn_top(lat5)
        self._tag = 0
        lat4 = self._conv(c4, 'neck.lateral_convs.1.conv.weight', 1, bias_key='neck.lateral_convs.1.conv.bias',
                          residual=lat5, residual_upsample=True)
        lat3 = self._conv(c3, 'neck.lateral_convs.0.conv.weight', 1, bias_key='neck.lateral_convs.0.conv.bias',
                          residual=lat4, residual_upsample=True)
        p3 = self._conv(lat3, 'neck.fpn_convs.0.conv.weight', 3, bias_key='neck.fpn_convs.0.conv.bias')
        p4 = self._conv(lat4, 'neck.fpn_convs.1.conv.weight', 3, bias_key='neck.fpn_convs.1.conv.bias')
        self._marker('join')
        self.fpn_outs = [p3, p4, p5, p6, p7]
        self._build_head(self.fpn_outs)

    def _fpn_top(self, lat5):
        p5 = self._conv(lat5, 'neck.fpn_convs.2.conv.weight', 3, bias_key='neck.fpn_convs.2.conv.bias')
        p6 = self._conv(p5, 'neck.fpn_convs.3.conv.weight', 3, 2, bias_key='neck.fpn_convs.3.conv.bias')
        p6r = self._t(*p6.shape)
        self._add(lambda: C.upsample_bilinear(p6, 1, out=p6r, relu=True), name='relu_copy')   # F.relu(outs[-1]) (fpn.py:175)
        p7 = self._conv(p6r, 'neck.fpn_convs.4.conv.weight', 3, 2, bias_key='neck.fpn_convs.4.conv.bias')
        return p5, p6, p7

    def _once(self, key, fn):
        if key not in self._wcache:
            self._wcache[key] = fn()
        return self._wcache[key]

    def _packed(self, wkey, bias_key=None, cout_pad=None):
        ck = (wkey, None, bias_key, cout_pad)
        if ck not in self._wcache:
            weight, b = C.pack_weight(self._w(wkey), cout_pad=cout_pad, device=self.dev)
            if bias_key is not None:
                b = self._w(bias_key).to(self.dev).contiguous()
            self._wcache[ck] = (weight, b)
        return self._wcache[ck]

    def _conv_multi(self, xs, weight, k, outs=None, relu=False, bias=None, gn_stats=None, out_dtype=torch.float16,
                    cout_real=None):
        N = xs[0].shape[0]
        if outs is None:
            outs = [self._t(N, x.shape[1], x.shape[2], weight.shape[0], dtype=out_dtype) for x in xs]
        plan = C.ConvPlanMulti(xs, weight, outs, k, relu=relu, bias=bias, gn_stats=gn_stats)
        if self._max_ctas:
            plan.set_max_ctas(self._max_ctas)
        self._keep.append(plan)
        self.conv_plans.append(plan)
        npix = sum(x.shape[1] * x.shape[2] for x in xs)
        fl = 2.0 * N * npix * (cout_real or weight.shape[0]) * weight.shape[1]
        self.conv_flops += fl
        self.conv_meta.append(dict(name='multi-level x%d' % len(xs), M=N * npix, N=weight.shape[0], K=weight.shape[1], k=k, stride=1,
                                   flops=fl, res=False, gn=gn_stats is not None))
        self._add(plan.run, name='conv')
        return outs

    def _tower_conv(self, xs, wkey, gn_prefix, bias_key, stats):
        """ConvModule: conv3x3 -> GN(32) -> ReLU (conv_module.py:124-132) for all pyramid levels in one launch;
        GN statistics come out of the GEMM epilogue (per level, per image)."""
        if self.gn:
            w, _ = self._packed(wkey)
            ys = self._conv_multi(xs, w, 3, gn_stats=stats)
            gamma = self._w(gn_prefix + '.weight').to(self.dev)
            beta = self._w(gn_prefix + '.bias').to(self.dev)
            self._keep += [gamma, beta]
            self._add(lambda: C.groupnorm_relu_apply_multi(ys, stats, gamma, beta, 1e-5, True), name='gn_apply')
            return ys
        w, b = self._packed(wkey, bias_key)
        return self._conv_multi(xs, w, 3, relu=True, bias=b)

    def _build_head(self, feats):
        N = self.N
        hp = self.hp
        sizes = [(f.shape[1], f.shape[2]) for f in feats]
        self.level_sizes = sizes
        tot = sum(h * w for h, w in sizes)
        nl = len(feats)
        n_tower = (self.stacked - 1) + self.stacked + 1 + ((self.stacked - 1) if self.vis else 0)
        # one int64 fixed-point statistics arena for every (conv, level) GroupNorm, zeroed once per forward
        self.gn_arena = self._t(n_tower, nl, N, 32, 2, dtype=torch.int64, zero=True)
        self._add(lambda: self.gn_arena.zero_(), 0, name='memset')
        ncls, CC = self.ncls, self.ncls + 128
        CCp = (CC + 15) // 16 * 16
        w_cls = torch.cat([self._w(hp + 'fcos_cls.weight'), self._w(hp + 'sip_cof.weight')], 0)
        b_cls = torch.cat([self._w(hp + 'fcos_cls.bias'), self._w(hp + 'sip_cof.bias')], 0)
        wk_cls = self._once('head.wk_cls', lambda: C.pack_weight(w_cls, cout_pad=CCp, device=self.dev)[0])
        b_cls = self._once('head.b_cls', lambda: torch.cat([b_cls, b_cls.new_zeros(CCp - CC)]).to(self.dev))
        w_reg = torch.cat([self._w(hp + 'fcos_reg.weight'), self._w(hp + 'fcos_centerness.weight')], 0)
        b_reg = torch.cat([self._w(hp + 'fcos_reg.bias'), self._w(hp + 'fcos_centerness.bias')], 0)
        wk_reg = self._once('head.wk_reg', lambda: C.pack_weight(w_reg, cout_pad=16, device=self.dev)[0])
        b_reg = self._once('head.b_reg', lambda: torch.cat([b_reg, b_reg.new_zeros(16 - 5)]).to(self.dev))
        wk_dcn = self._once('head.wk_dcn', lambda: C.pack_weight(self._w(hp + 'feat_align.conv_adaption.weight'),
                                                                   device=self.dev)[0])
        w_off = self._once('head.w_off',
                           lambda: self._w(hp + 'feat_align.conv_offset.weight').view(72, 4).contiguous().to(self.dev))
        self._keep += [wk_cls, b_cls, wk_reg, b_reg, wk_dcn, w_off]
        self.scales = [float(self._w(hp + 'scales.%d.scale' % i)) for i in range(nl)]
        # fp32 head outputs, channel-last, ONE allocation in level-major order [level][image][h*w][C] with C = 80+128 (-> 208)
        # and 16 = 4 reg | 1 ctr | pad: every level is a contiguous [N,h,w,C] tensor for the GEMM epilogue, and with N == 1
        # the buffer is the level-concatenated [tot, C] table a candidate's location index addresses directly
        self.clscof = self._t(N * tot, CCp, dtype=torch.float32)
        self.regctr = self._t(N * tot, 16, dtype=torch.float32)
        offs0 = [sum(h * w for h, w in sizes[:l]) for l in range(nl)]
        clscof_l = [self.clscof[N * offs0[l]:N * (offs0[l] + sizes[l][0] * sizes[l][1])].view(N, sizes[l][0], sizes[l][1], CCp)
                    for l in range(nl)]
        regctr_l = [self.regctr[N * offs0[l]:N * (offs0[l] + sizes[l][0] * sizes[l][1])].view(N, sizes[l][0], sizes[l][1], 16)
                    for l in range(nl)]
        self.level_views = list(zip(clscof_l, regctr_l))
        si = 0
        cls_feats, reg_feats = list(feats), list(feats)
        # The cls and reg towers are independent chains of 202-tile GEMMs (1.5 waves each on 132 SMs).  They are
        # captured on two streams with their persistent grids capped at half the GPU, so together they keep every SM
        # busy (3.06 waves for a pair instead of 2 + 2).
        self._marker('fork')
        cap = self.head_max_ctas if self.head_max_ctas is not None else 100
        if self.max_ctas:
            cap = min(cap, self.max_ctas) if cap else self.max_ctas
        self._max_ctas = cap or None
        self._tag = 0
        for i in range(self.stacked - 1):
            cls_feats = self._tower_conv(cls_feats, hp + 'cls_convs.%d.conv.weight' % i, hp + 'cls_convs.%d.gn' % i,
                                         hp + 'cls_convs.%d.conv.bias' % i, [self.gn_arena[si, l] for l in range(nl)])
            si += 1
        self._tag = 1
        for i in range(self.stacked):
            reg_feats = self._tower_conv(reg_feats, hp + 'reg_convs.%d.conv.weight' % i, hp + 'reg_convs.%d.gn' % i,
                                         hp + 'reg_convs.%d.conv.bias' % i, [self.gn_arena[si, l] for l in range(nl)])
            si += 1
        # fcos_reg | fcos_centerness on the reg tower (sipmask_head.py:261,265), raw fp32 (Scale applied by consumers)
        self._conv_multi(reg_feats, wk_reg, 3, outs=regctr_l, bias=b_reg, cout_real=5)
        self._marker('join')
        self._marker('fork')
        self._tag = 0
        # FeatureAlign: offsets from scale*fcos_reg, DCN 3x3 dg=4, GN, ReLU (sipmask_head.py:49-55)
        offs = [self._t(N, h, w, 72, dtype=torch.float32) for h, w in sizes]
        self._add(lambda: C.offset_conv1x1_multi(regctr_l, self.scales, w_off, offs), name='offset_conv')
        cols = [self._t(N, h, w, 2304) for h, w in sizes]
        self._add(lambda: C.deform_im2col_multi(cls_feats, offs, 4, cols), name='deform_im2col')
        if self.gn:
            stats = [self.gn_arena[si, l] for l in range(nl)]
            aligned = self._conv_multi(cols, wk_dcn, 1, gn_stats=stats)
            gamma = self._w(hp + 'feat_align.norm.weight').to(self.dev)
            beta = self._w(hp + 'feat_align.norm.bias').to(self.dev)
            self._keep += [gamma, beta]
            self._add(lambda: C.groupnorm_relu_apply_multi(aligned, stats, gamma, beta, 1e-5, True), name='gn_apply')
        else:
            aligned = self._conv_multi(cols, wk_dcn, 1, relu=True)
        # fcos_cls | sip_cof on the aligned feature (sipmask_head.py:264,271)
        self._conv_multi(aligned, wk_cls, 3, outs=clscof_l, bias=b_cls)
        # prototype branch on the side stream, next to FeatureAlign / the cls heads
        self._tag = 1
        # prototype input: reg feature of levels 0..2 at P3 resolution (sipmask_head.py:275-281)
        h3, w3 = sizes[0]
        cat = self._t(N, h3, w3, 768)
        for l in range(3):
            self._add(lambda l=l: C.upsample_bilinear(reg_feats[l], 2 ** l, out=cat, out_choff=256 * l), name='upsample')
        # prototype branch (sipmask_head.py:283-285)
        m0 = self._conv(cat, hp + 'sip_mask_lat0.weight', 1, relu=True, bias_key=hp + 'sip_mask_lat0.bias')
        m1 = self._conv(m0, hp + 'sip_mask_lat.weight', 3, relu=True, bias_key=hp + 'sip_mask_lat.bias')
        self.protos = self._t(N, 4 * h3, 4 * w3, 32)
        self._add(lambda: C.upsample_bilinear(m1, 4, out=self.protos), name='upsample')
        self._marker('join')
        self._tag = 0
        if self.vis:
            # tracking branch (VIS/...:274-287,296-312): track_convs on levels 0..2 -> bilinear x1 / x2 / x4 to P3 resolution ->
            # concat 768 -> sipmask_track 1x1 -> 512, fp32 (the features enter dot products of the association)
            tfe = list(feats[:3])
            for i in range(self.stacked - 1):
                tfe = self._tower_conv(tfe, hp + 'track_convs.%d.conv.weight' % i, hp + 'track_convs.%d.gn' % i,
                                       hp + 'track_convs.%d.conv.bias' % i, [self.gn_arena[si + 1 + i, l] for l in range(3)])
            cat_t = self._t(N, h3, w3, 768)
            for l in range(3):
                self._add(lambda l=l, tfe=tfe, cat_t=cat_t: C.upsample_bilinear(tfe[l], 2 ** l, out=cat_t, out_choff=256 * l),
                          name='upsample')
            self.track_feats = self._conv(cat_t, hp + 'sipmask_track.weight', 1, bias_key=hp + 'sipmask_track.bias',
                                          out_dtype=torch.float32)
        self._max_ctas = self.max_ctas
        if self.build_post:
            self._build_postproc()

    def _build_fcos_head(self, feats):
        """Plain FCOS head (MM/mmdet/models/anchor_heads/fcos_head.py:118-135): 4+4 tower ConvModules, fcos_cls and
        fcos_centerness on the cls tower, fcos_reg on the reg tower (exp(scale * x) is applied by the caller)."""
        N, hp = self.N, self.hp
        sizes = [(f.shape[1], f.shape[2]) for f in feats]
        self.level_sizes = sizes
        nl = len(feats)
        tot = sum(h * w for h, w in sizes)
        self.gn_arena = self._t(2 * self.stacked, nl, N, 32, 2, dtype=torch.int64, zero=True)
        self._add(lambda: self.gn_arena.zero_(), 0, name='memset')
        ncls = self.ncls
        CCp = (ncls + 1 + 15) // 16 * 16
        w_cls = torch.cat([self._w(hp + 'fcos_cls.weight'), self._w(hp + 'fcos_centerness.weight')], 0)
        b_cls = torch.cat([self._w(hp + 'fcos_cls.bias'), self._w(hp + 'fcos_centerness.bias')], 0)
        wk_cls, _ = C.pack_weight(w_cls, cout_pad=CCp, device=self.dev)
        b_cls = torch.cat([b_cls, b_cls.new_zeros(CCp - ncls - 1)]).to(self.dev)
        wk_reg, _ = C.pack_weight(self._w(hp + 'fcos_reg.weight'), cout_pad=16, device=self.dev)
        b_reg = torch.cat([self._w(hp + 'fcos_reg.bias'), torch.zeros(12)]).to(self.dev)
        self._keep += [wk_cls, b_cls, wk_reg, b_reg]
        self.scales = [float(self._w(hp + 'scales.%d.scale' % i)) for i in range(nl)]
        self.clscof = self._t(N * tot, CCp, dtype=torch.float32)      # [cls(80) | centerness(1) | pad], level-major
        self.regctr = self._t(N * tot, 16, dtype=torch.float32)       # [reg(4) | pad]
        offs0 = [sum(h * w for h, w in sizes[:l]) for l in range(nl)]
        cls_l = [self.clscof[N * offs0[l]:N * (offs0[l] + sizes[l][0] * sizes[l][1])].view(N, sizes[l][0], sizes[l][1], CCp) for l in range(nl)]
        reg_l = [self.regctr[N * offs0[l]:N * (offs0[l] + sizes[l][0] * sizes[l][1])].view(N, sizes[l][0], sizes[l][1], 16) for l in range(nl)]
        self.level_views = list(zip(cls_l, reg_l))
        si = 0
        cls_feats, reg_feats = list(feats), list(feats)
        for i in range(self.stacked):
            cls_feats = self._tower_conv(cls_feats, hp + 'cls_convs.%d.conv.weight' % i, hp + 'cls_convs.%d.gn' % i,
                                         hp + 'cls_convs.%d.conv.bias' % i, [self.gn_arena[si, l] for l in range(nl)])
            si += 1
        for i in range(self.stacked):
            reg_feats = self._tower_conv(reg_feats, hp + 'reg_convs.%d.conv.weight' % i, hp + 'reg_convs.%d.gn' % i,
                                         hp + 'reg_convs.%d.conv.bias' % i, [self.gn_arena[si, l] for l in range(nl)])
            si += 1
        self._conv_multi(cls_feats, wk_cls, 3, outs=cls_l, bias=b_cls, cout_real=ncls + 1)
        self._conv_multi(reg_feats, wk_reg, 3, outs=reg_l, bias=b_reg, cout_real=4)

    def load_features(self, feats):
        """feats: five NCHW tensors (fp16/fp32, CUDA) from the caller's neck -> the engine's NHWC fp16 buffers."""
        for buf, f in zip(self.fpn_outs, feats):
            buf.copy_(f.permute(0, 2, 3, 1))

    # ------------------------------------------------------------------------------- post-processing
    def _build_postproc(self):
        """decode -> NMS -> coefficient gather -> mask assembly -> x2 upsample/threshold/bit-pack, image by image
        (get_bboxes loops over images, sipmask_head.py:517-540), all on device with fixed-shape outputs."""
        N, dev = self.N, self.dev
        cfg = self.cfg
        nl = len(self.level_sizes)
        CCp = self.clscof.shape[-1]
        ncls = self.ncls
        nms_pre = int(cfg['nms_pre'])
        self.max_num = 100 if self.ssd else int(cfg['max_per_img'])      # MM's fast_nms hard-codes 100 (sipmask_head.py:903)
        fast = self.ssd or self.vis                                         # VIS: fast_nms with cfg.max_per_img (VIS/...:986)
        ncand = sum(min(h * w, nms_pre) if nms_pre > 0 else h * w for h, w in self.level_sizes)
        self.ncand = ncand
        lib = L.lib()
        sf = np.atleast_1d(np.asarray(self.scale_factor, dtype=np.float32))
        s4 = (sf if sf.size == 4 else np.repeat(sf, 4)).astype(np.float32)
        self._sf4 = L.f4(s4)
        self._box_scale4 = L.f4(s4 / 2.0)
        Hm, Wm = self.protos.shape[1], self.protos.shape[2]
        oh, ow = int(self.ori_shape[0]), int(self.ori_shape[1])        # rescale=True: masks live in the ori_shape canvas
        self.mask_hw = (oh, ow)
        from .postproc import mask_up_factors
        fh, fw, ry, rx = ops.resize_spec(Hm, Wm, mask_up_factors(self.scale_factor, self.ssd), self.legacy_interp)
        words = (ow + 31) // 32
        self.det = self._t(N, self.max_num, 5, dtype=torch.float32)
        self.labels = self._t(N, self.max_num, dtype=torch.long)
        self.idx = self._t(N, self.max_num, dtype=torch.long)
        self.count = self._t(N, dtype=torch.int32, zero=True)
        self.mask_bits = self._t(N, self.max_num, oh, words, dtype=torch.int32)
        self.cand_boxes = self._t(N, ncand, 4, dtype=torch.float32)
        self.cand_scores = self._t(N, ncand, ncls, dtype=torch.float32)
        self.cand_ctr = self._t(N, ncand, dtype=torch.float32)
        self.cand_loc = self._t(N, ncand, dtype=torch.int32)
        self.loc_kept = self._t(N, self.max_num, dtype=torch.long)
        self.det_cofs = self._t(N, self.max_num, 128, dtype=torch.float32)
        self.det_boxes4 = self._t(N, self.max_num, 4, dtype=torch.float32)
        self.det_track = self._t(N, self.max_num, 512, dtype=torch.float32) if self.vis else None
        if self.rescoring:
            # dense fp16 cropped masks of every detection slot, for the one batched rescoring op after the per-image chains
            self.pos_masks = self._t(N, self.max_num, Hm, Wm)
            self.mask_scores = self._t(N, self.max_num, dtype=torch.float32, zero=True)
            hp = self.hp
            self._rescore_w = self._once('rescore', lambda: ops.RescoreWeights(
                [self._w('%sconvs_scoring.%d.conv.weight' % (hp, i)) for i in range(6)],
                [self._w('%sconvs_scoring.%d.conv.bias' % (hp, i)) for i in range(6)],
                self._w(hp + 'mask_scoring.weight'), self._w(hp + 'mask_scoring.bias'), self.dev))
            self._rescore_ws = self._t(ops.mask_rescore_f16_workspace_bytes(N * self.max_num, Hm, Wm), dtype=torch.uint8)
            self.rescore_flops = float(N * self.max_num * ops.rescore_flops_per_row(Hm, Wm))    # at full detection counts
        level_hw = (ctypes.c_int * nl)(*[h * w for h, w in self.level_sizes])
        self._keep.append(level_hw)
        # the per-image decode -> NMS -> gather -> mask chains are independent (get_bboxes loops over images,
        # sipmask_head.py:517-540): with a batch they are spread over a few streams of the captured graph
        pp_streams = min(N, 4) if N > 1 else 0
        if pp_streams:
            self._marker('fork')
        for n in range(N):
            self._tag = (n % pp_streams) + 1 if pp_streams else 0
            lv = (L.Level * nl)()
            for l, (h, w) in enumerate(self.level_sizes):
                cc = self.level_views[l][0][n]                 # [h,w,CCp] of image n (contiguous)
                rc = self.level_views[l][1][n]
                lv[l] = L.Level(cc.data_ptr(), rc.data_ptr() + 4 * 4, rc.data_ptr(), CCp, 16, 16, h, w, int(self.strides[l]),
                                float(self.scales[l]), float(self.strides[l]))
            ws_bytes = lib.smb_decode_workspace_bytes(nl, lv, nms_pre)
            ws = self._t(ws_bytes, dtype=torch.uint8)
            self._keep.append(lv)

            def decode(n=n, lv=lv, ws=ws, ws_bytes=ws_bytes):
                L.check(lib.smb_decode_topk(nl, lv, ncls, nms_pre, int(self.img_shape[0]), int(self.img_shape[1]), self._sf4,
                                            L.ptr(self.cand_boxes[n]), L.ptr(self.cand_scores[n]), L.ptr(self.cand_ctr[n]),
                                            L.ptr(self.cand_loc[n]), L.ptr(ws), ctypes.c_size_t(ws_bytes), L.stream_ptr()),
                        'smb_decode_topk')
            self._add(decode, 3, name='decode_topk')
            iou_thr = float(cfg['nms']['iou_thr'])
            if not fast:
                nws_bytes = lib.smb_multiclass_nms_workspace_bytes(ncand, ncls)
                nws = self._t(nws_bytes, dtype=torch.uint8)

                def nms(n=n, nws=nws, nws_bytes=nws_bytes):
                    L.check(lib.smb_multiclass_nms(L.ptr(self.cand_boxes[n]), L.ptr(self.cand_scores[n]), L.ptr(self.cand_ctr[n]),
                                                   ncand, ncls, ctypes.c_float(cfg['score_thr']), ctypes.c_float(iou_thr),
                                                   self.max_num, 0, L.ptr(self.det[n]), L.ptr(self.labels[n]), L.ptr(self.idx[n]),
                                                   L.ptr(self.count[n:n + 1]), L.ptr(nws), ctypes.c_size_t(nws_bytes),
                                                   L.stream_ptr()), 'smb_multiclass_nms')
            else:
                nws_bytes = lib.smb_fast_nms_workspace_bytes(ncand, ncls, 200)
                nws = self._t(nws_bytes, dtype=torch.uint8)

                def nms(n=n, nws=nws, nws_bytes=nws_bytes):
                    L.check(lib.smb_fast_nms(L.ptr(self.cand_boxes[n]), L.ptr(self.cand_scores[n]), L.ptr(self.cand_ctr[n]), ncand,
                                             ncls, ctypes.c_float(cfg['score_thr']), ctypes.c_float(iou_thr), 200, self.max_num,
                                             L.ptr(self.det[n]), L.ptr(self.labels[n]), L.ptr(self.idx[n]),
                                             L.ptr(self.count[n:n + 1]), L.ptr(nws), ctypes.c_size_t(nws_bytes), L.stream_ptr()),
                            'smb_fast_nms')
            self._add(nms, 4 if not fast else 2, name='nms')
            cof_src = self.clscof[:, ncls:ncls + 128]                          # coefficient columns, row pitch CCp

            def gather(n=n, cof_src=cof_src):
                # candidate row -> level-concatenated location -> coefficient row (mlvl_cofs[idxs_keep], sipmask_head.py:612)
                # and det[:, :4] -> contiguous rois input, one launch (was index_select + gather + copy_)
                L.check(lib.smb_gather_det_inputs(L.ptr(cof_src), CCp, L.ptr(self.cand_loc[n]), L.ptr(self.idx[n]),
                                                  L.ptr(self.det[n]), L.ptr(self.count[n:n + 1]), self.max_num, 128,
                                                  L.ptr(self.det_cofs[n]), L.ptr(self.det_boxes4[n]), L.ptr(self.loc_kept[n]),
                                                  nl if N > 1 else 0, level_hw, N, n, L.stream_ptr()), 'smb_gather_det_inputs')
            self._add(gather, 1, name='gather_cofs')

            def masks(n=n):
                # fused: prototypes -> sub-region dot/sigmoid/crop -> x2 bilinear -> threshold -> bit-pack (no pos_masks tensor)
                L.check(lib.smb_mask_assemble_pack(L.ptr(self.protos[n]), L.F16, 1, L.ptr(self.det_cofs[n]), L.ptr(self.det_boxes4[n]),
                                                   self._box_scale4, L.ptr(self.mask_bits[n]), Hm, Wm, self.max_num, fh, fw,
                                                   ctypes.c_float(ry), ctypes.c_float(rx), oh, ow,
                                                   ctypes.c_float(self.mask_thr), L.stream_ptr()), 'smb_mask_assemble_pack')
            self._add(masks, 2, name='mask_fused')
            if self.rescoring:
                def dense(n=n):
                    # the same rois as mask_fused; rows past the count have zero boxes and are skipped by the rescoring
                    L.check(lib.smb_mask_assemble(L.ptr(self.protos[n]), L.F16, 1, L.ptr(self.det_cofs[n]),
                                                  L.ptr(self.det_boxes4[n]), self._box_scale4, L.ptr(self.pos_masks[n]), L.F16,
                                                  Hm, Wm, self.max_num, L.stream_ptr()), 'smb_mask_assemble')
                self._add(dense, 1, name='mask_dense')
            if self.vis:
                th, tw = self.track_feats.shape[1], self.track_feats.shape[2]

                def track(n=n, th=th, tw=tw):
                    L.check(lib.smb_gather_track_feats(L.ptr(self.track_feats[n]), th, tw, 512, L.ptr(self.det[n]),
                                                       L.ptr(self.count[n:n + 1]), self.max_num, ctypes.c_float(float(s4[0])),
                                                       ctypes.c_float(float(s4[1])), ctypes.c_float(8.0),
                                                       L.ptr(self.det_track[n]), L.stream_ptr()), 'smb_gather_track_feats')
                self._add(track, 1, name='gather_track')
        if pp_streams:
            self._marker('join')
        self._tag = 0
        if self.rescoring:
            self._add(lambda: ops.mask_rescore_f16(self.pos_masks, self.count, self._rescore_w, self.labels, self.det,
                                                   workspace=self._rescore_ws, out=self.mask_scores), 5, name='rescore')

    # ---------------------------------------------------------------------------------------------- run
    def _run_ops(self, only=None):
        """Issue the launch sequence on the current stream (+ the side stream between fork / join markers).
        `only`: optional set of op names to issue (markers are always honoured), e.g. {'conv'} for the roofline graph."""
        if torch.cuda.current_device() != self.dev.index:       # every launch goes to the engine's device and its streams
            with torch.cuda.device(self.dev):
                return self._run_ops(only)
        s0 = torch.cuda.current_stream(self.dev)
        ntag = max([t for t in self.op_tags if isinstance(t, int)] + [1])
        if self.side_stream is None:
            self.side_stream = torch.cuda.Stream(device=self.dev)
            self.side_streams = [self.side_stream] + [torch.cuda.Stream(device=self.dev) for _ in range(ntag - 1)]
        side = self.side_streams
        entries = [(f, tag) for f, tag, name in zip(self.ops, self.op_tags, self.op_names)
                   if not (only is not None and f is not None and name not in only)]
        used = set()
        for i, (f, tag) in enumerate(entries):
            if tag == 'fork':
                # only the side streams that get work before the next join enter the capture (an unjoined stream is an error)
                used = set()
                for f2, t2 in entries[i + 1:]:
                    if t2 == 'join':
                        break
                    if isinstance(t2, int) and t2 >= 1:
                        used.add(t2 - 1)
                for k in sorted(used):
                    side[k].wait_stream(s0)
            elif tag == 'join':
                for k in sorted(used):
                    s0.wait_stream(side[k])
                used = set()
            elif isinstance(tag, int) and tag >= 1:
                with torch.cuda.stream(side[tag - 1]):
                    f()
            else:
                f()

    def forward(self, img=None):
        """img: NCHW fp32 CUDA tensor (or None to reuse the resident input).  Returns the device result record."""
        if torch.cuda.current_device() != self.dev.index:
            with torch.cuda.device(self.dev):
                return self.forward(img)
        if img is not None:
            self.img.copy_(img, non_blocking=True)
        if self.use_graph:
            if self.graph is None:
                self._run_ops()                      # warm-up: cudaFuncSetAttribute etc. must not happen under capture
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._run_ops()
                self.graph = g
            self.graph.replay()
        else:
            self._run_ops()
        return self._result()

    def _result(self):
        r = dict(det_bboxes=self.det, det_labels=self.labels, count=self.count, mask_bits=self.mask_bits, idxs_keep=self.idx)
        if self.vis:
            r['track_feats'] = self.det_track          # [N,max,512] box-centre tracking features (zeros after count)
        if self.rescoring:
            r['mask_scores'] = self.mask_scores        # [N,max] fp32 SipMask++ mask scores (zeros after count)
        return r

    def forward_raw(self, img_u8, mean=(102.9801, 115.9465, 122.7717)):
        """img_u8: uint8 BGR HWC CUDA image straight from the decoder.  Resize (keep ratio, mmcv.imrescale rule towards this
        engine's img_shape) + mean subtraction + padding + layout run in ONE kernel that writes the stem's input
        (SURVEY.md 8f-3); the rest of the step is the CUDA graph without its `image_to_s2d16` node.  The resized size must
        equal the engine's img_shape (one engine per input resolution); batch 1."""
        assert self.N == 1, 'forward_raw preprocesses one image'
        if torch.cuda.current_device() != self.dev.index:
            with torch.cuda.device(self.dev):
                return self.forward_raw(img_u8, mean)
        C.preprocess_u8(img_u8, self.img_shape[:2], self.img8, mean)
        if self.use_graph:
            if getattr(self, 'graph_raw', None) is None:
                names = set(self.op_names) - {'image_to_s2d16', 'fork', 'join'}
                self._run_ops(only=names)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._run_ops(only=names)
                self.graph_raw = g
            self.graph_raw.replay()
        else:
            self._run_ops(only=set(self.op_names) - {'image_to_s2d16', 'fork', 'join'})
        return self._result()

    # head outputs in the reference's layout (for parity tests / the drop-in head)
    def head_outputs(self):
        outs = dict(cls=[], bbox=[], ctr=[], cof=[])
        ncls = self.ncls
        for l, (cc, rc) in enumerate(self.level_views):
            outs['cls'].append(cc[..., :ncls].permute(0, 3, 1, 2))
            outs['cof'].append(cc[..., ncls:ncls + 128].permute(0, 3, 1, 2))
            outs['bbox'].append((rc[..., :4] * self.scales[l]).permute(0, 3, 1, 2) * self.strides[l])
            outs['ctr'].append(rc[..., 4:5].permute(0, 3, 1, 2))
        outs['feat_masks'] = self.protos.permute(0, 3, 1, 2)
        if self.vis:
            outs['track_feats'] = self.track_feats.permute(0, 3, 1, 2)
        return outs
