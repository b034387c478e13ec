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
                 rescoring_flag=False, benchmark=False, max_ori_hw=None, min_mask_up=None, arena=None, rle_bytes=0,
                 rle_runs=None):
        # SipMask-benchmark checkpoints (keys from sipmask_b200.benchmark.convert_state_dict): FrozenBatchNorm without eps,
        # tower / DCN convs with bias before GN, relu'd regression, pair candidates, label-aware NMS, k-th-value cut
        self.benchmark = benchmark
        if benchmark:
            from .benchmark import check_options
            check_options(vis=vis, rescoring=rescoring_flag)
        self.bn_eps = 0.0 if benchmark else 1e-5
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
        # BM: INFERENCE_TH, PRE_NMS_TOP_N, NMS_TH, DETECTIONS_PER_IMG (fcos_core/config/defaults.py:295-297,487)
        self.cfg = dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.6 if benchmark else 0.5), max_per_img=100)
        if test_cfg:
            self.cfg.update(test_cfg)
        # MM non-SSD heads pick hard or soft NMS by test_cfg.nms.type (bbox_nms.py:108-109); SSD / VIS heads use fast_nms and
        # SipMask-benchmark ml_nms whatever the type says
        self.soft_nms = None
        if not (benchmark or ssd_flag or vis):
            kind = ops.nms_type(self.cfg['nms'])
            if kind == 'soft_nms':
                self.soft_nms = ops.soft_nms_args(self.cfg['nms'])
            elif kind != 'nms':
                raise ValueError("test_cfg nms type %r: this head supports 'nms' and 'soft_nms'" % (kind,))
        self.img_shape = tuple(img_shape) if img_shape is not None else (self.H, self.W, 3)
        self.scale_factor = scale_factor
        # rescale=True semantics (SingleStageDetector.simple_test): boxes / scale_factor, masks resized by 2 / scale_factor and
        # pasted into the ori_shape canvas (sipmask_head.py:587-588,629-633,648-654)
        self.ori_shape = tuple(ori_shape) if ori_shape is not None else self.img_shape
        # mask record capacity [N, max, cap_h, ceil(cap_w / 32)]: images of any ori_shape up to it (set_image_meta)
        self.mask_cap = tuple(int(v) for v in (max_ori_hw if max_ori_hw is not None else self.ori_shape[:2]))
        # the steepest mask resize the fused mask kernel's tile is sized for (None: this engine's own scale_factor)
        self.min_mask_up = min_mask_up
        # COCO RLE strings of every detection, encoded on the device at the end of each forward (rle_bytes > 0: the string
        # bytes per image of the destination region; rle_runs: the runs one mask may have, default 4 * max width + 2)
        self.rle_bytes = int(rle_bytes)
        self.rle_runs = None if rle_runs is None else int(rle_runs)
        if self.rle_bytes < 0 or (self.rle_runs is not None and self.rle_runs < 1):
            raise ValueError('rle_bytes must be >= 0 and rle_runs >= 1')
        if self.rle_bytes and (fcos or not build_postproc):
            raise ValueError('rle_bytes > 0 encodes the post-processing record: it needs build_postproc=True')
        # activations, workspaces and outputs carved from a caller-owned uint8 device tensor (engines that share one never
        # run concurrently); arena_bytes is what this engine needs of it (counted without an arena too)
        self._arena = arena
        if arena is not None and (arena.dtype != torch.uint8 or arena.dim() != 1 or not arena.is_cuda):
            raise ValueError('arena must be a 1-D uint8 CUDA tensor')
        self.arena_bytes = 0
        self.image_metas = [(self.img_shape, self.ori_shape, self.scale_factor)] * batch
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
        nbytes = int(np.prod(shape, dtype=np.int64)) * torch.empty((), dtype=dtype).element_size()
        off = (self.arena_bytes + 255) // 256 * 256
        self.arena_bytes = off + nbytes
        if self._arena is None:
            t = (torch.zeros if zero else torch.empty)(shape, dtype=dtype, device=self.dev)
        else:
            # every buffer in an arena is rewritten by each forward before it is read (the zeroed ones too: the GroupNorm
            # statistics by a memset node, count / kept_total / mask_scores by their kernels), so another engine
            # using the same bytes between two forwards changes nothing
            if self.arena_bytes > self._arena.numel():
                raise ValueError('arena of %d bytes is too small for this engine (%d bytes needed so far)'
                                 % (self._arena.numel(), self.arena_bytes))
            t = self._arena[off:off + nbytes].view(dtype).view(shape)
            if zero:
                t.zero_()
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

    def _once(self, key, fn):
        if key not in self._wcache:
            self._wcache[key] = fn()
        return self._wcache[key]

    def _packed(self, wkey, bn=None, bias_key=None, cout_pad=None):
        """(packed weight, fp32 bias) of one convolution, once per weight cache: BN `bn` folded in, or the bias `bias_key`
        zero-padded to cout_pad."""
        def pack():
            weight, b = C.pack_weight(self._w(wkey), bn=self._bn(bn) if bn else None, eps=self.bn_eps, cout_pad=cout_pad,
                                      device=self.dev)
            if bias_key is not None:
                b = self._w(bias_key)
                if cout_pad and cout_pad != b.numel():
                    b = torch.cat([b, b.new_zeros(cout_pad - b.numel())])
                b = b.to(self.dev).contiguous()
            return weight, b
        return self._once((wkey, bn, bias_key, cout_pad), pack)

    def _add_conv(self, plan, weight, name, M, k, stride=1, res=False, gn=False, cout_real=None, k_real=None, cap=True):
        """Registers a convolution plan: CTA cap (`cap`), kept alive, its launch, its algorithmic FLOPs in conv_flops and
        its GEMM shape in conv_meta."""
        if cap and self._max_ctas:
            plan.set_max_ctas(self._max_ctas)
        self._keep.append(plan)
        self.conv_plans.append(plan)
        fl = 2.0 * M * (cout_real or weight.shape[0]) * (k_real or weight.shape[1])
        self.conv_flops += fl
        self.conv_meta.append(dict(name=name, M=M, N=weight.shape[0], K=weight.shape[1], k=k, stride=stride, flops=fl,
                                   res=res, gn=gn))
        self._add(plan.run, name='conv')

    def _conv(self, x, wkey, k, stride=1, relu=False, bn=None, bias_key=None, residual=None, residual_upsample=False,
              out_dtype=torch.float16, cout_pad=None, cout_real=None):
        weight, bias = self._packed(wkey, bn, bias_key, cout_pad)
        N, H, W, _ = x.shape
        Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
        out = self._t(N, Ho, Wo, weight.shape[0], dtype=out_dtype)
        plan = C.ConvPlan(x, weight, out, k, stride, relu=relu, bias=bias, residual=residual,
                          residual_upsample=residual_upsample)
        self._add_conv(plan, weight, wkey, N * Ho * Wo, k, stride, res=residual is not None, cout_real=cout_real)
        return out

    def _conv_multi(self, xs, weight, k, outs=None, relu=False, bias=None, gn_stats=None, cout_real=None):
        """One stride-1 convolution over several pyramid levels (one launch)."""
        N = xs[0].shape[0]
        if outs is None:
            outs = [self._t(N, x.shape[1], x.shape[2], weight.shape[0]) for x in xs]
        plan = C.ConvPlanMulti(xs, weight, outs, k, relu=relu, bias=bias, gn_stats=gn_stats)
        self._add_conv(plan, weight, 'multi-level x%d' % len(xs), N * sum(x.shape[1] * x.shape[2] for x in xs), k,
                       gn=gn_stats is not None, cout_real=cout_real)
        return outs

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
                                                                      eps=self.bn_eps, device=self.dev))
        s1 = self._t(N, H // 2, W // 2, 64)
        # algorithmic K is 7x7x3 (executed K is 256); the stem runs on all SMs
        self._add_conv(C.StemPlan(img8, wk, b, s1, N, H, W), wk, 'stem', N * (H // 2) * (W // 2), 7, 2, k_real=147, cap=False)
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

    def _tower(self, xs, name, n, slot):
        """ConvModules <hp><name>.0 .. n-1: conv3x3 -> GN(32) -> ReLU (conv_module.py:124-132), each for all pyramid levels
        in one launch; the GN statistics of conv i come out of the GEMM epilogue into gn_arena[slot + i] (per level, per
        image)."""
        for i in range(n):
            p = '%s%s.%d.' % (self.hp, name, i)
            if self.gn:
                # BM towers keep the conv bias before GN (sipmask.py:71-82); the epilogue adds it before the statistics
                w, b = self._packed(p + 'conv.weight', bias_key=p + 'conv.bias' if self.benchmark else None)
                stats = [self.gn_arena[slot + i, l] for l in range(len(xs))]
                xs = self._conv_multi(xs, w, 3, bias=b, gn_stats=stats)
                self._gn_relu(xs, stats, p + 'gn')
            else:
                w, b = self._packed(p + 'conv.weight', bias_key=p + 'conv.bias')
                xs = self._conv_multi(xs, w, 3, relu=True, bias=b)
        return xs

    def _gn_relu(self, xs, stats, prefix):
        gamma = self._w(prefix + '.weight').to(self.dev)
        beta = self._w(prefix + '.bias').to(self.dev)
        self._keep += [gamma, beta]
        self._add(lambda: C.groupnorm_relu_apply_multi(xs, stats, gamma, beta, 1e-5, True), name='gn_apply')

    def _head_buffers(self, feats, n_stats, cls_pitch):
        """What both heads allocate: one int64 fixed-point statistics arena for every (conv, level) GroupNorm, zeroed once per
        forward; the Scale values; the fp32 head outputs, channel-last, ONE allocation each in level-major order
        [level][image][h*w][C]: clscof (C = cls_pitch) and regctr (C = 16).  Every level is a contiguous [N,h,w,C] tensor
        for the GEMM epilogue, and with N == 1 the buffer is the level-concatenated [tot, C] table a candidate's location
        index addresses directly.  Returns the per-level [N,h,w,C] views of clscof and of regctr."""
        N = self.N
        sizes = self.level_sizes = [(f.shape[1], f.shape[2]) for f in feats]
        self.gn_arena = self._t(n_stats, len(sizes), N, 32, 2, dtype=torch.int64, zero=True)
        self._add(lambda: self.gn_arena.zero_(), 0, name='memset')
        self.scales = [float(self._w(self.hp + 'scales.%d.scale' % i)) for i in range(len(sizes))]
        tot = sum(h * w for h, w in sizes)
        self.clscof = self._t(N * tot, cls_pitch, dtype=torch.float32)
        self.regctr = self._t(N * tot, 16, dtype=torch.float32)
        cls_l, reg_l, o = [], [], 0
        for h, w in sizes:
            cls_l.append(self.clscof[N * o:N * (o + h * w)].view(N, h, w, cls_pitch))
            reg_l.append(self.regctr[N * o:N * (o + h * w)].view(N, h, w, 16))
            o += h * w
        return cls_l, reg_l

    def _build_head(self, feats):
        N, hp, ncls = self.N, self.hp, self.ncls
        CC = ncls + 128
        CCp = (CC + 15) // 16 * 16
        si = 2 * self.stacked - 1                        # GN statistics slot of FeatureAlign, after the cls and reg towers
        cls_l, reg_l = self._head_buffers(feats, si + 1 + ((self.stacked - 1) if self.vis else 0), CCp)
        # clscof = [cls | 128 coefficients | pad], regctr = [4 raw box distances | centerness | pad]
        self.level_views = [dict(cls=c[..., :ncls], cof=c[..., ncls:CC], box=r[..., :4], ctr=r[..., 4:5])
                            for c, r in zip(cls_l, reg_l)]
        self.cof_src = self.clscof[:, ncls:CC]          # coefficients of every location, row pitch CCp
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
        # The cls and reg towers are independent chains of 202-tile GEMMs (1.5 waves each on 132 SMs).  They are
        # captured on two streams with their persistent grids capped at half the GPU, so together they keep every SM
        # busy (3.06 waves for a pair instead of 2 + 2).
        self._marker('fork')
        cap = self.head_max_ctas if self.head_max_ctas is not None else 100
        if self.max_ctas:
            cap = min(cap, self.max_ctas) if cap else self.max_ctas
        self._max_ctas = cap or None
        self._tag = 0
        cls_feats = self._tower(feats, 'cls_convs', self.stacked - 1, 0)
        self._tag = 1
        reg_feats = self._tower(feats, 'reg_convs', self.stacked, self.stacked - 1)
        # fcos_reg | fcos_centerness on the reg tower (sipmask_head.py:261,265), raw fp32 (Scale applied by consumers)
        self._conv_multi(reg_feats, wk_reg, 3, outs=reg_l, bias=b_reg, cout_real=5)
        self._marker('join')
        self._marker('fork')
        self._tag = 0
        # FeatureAlign: offsets from scale*fcos_reg, DCN 3x3 dg=4, GN, ReLU (sipmask_head.py:49-55)
        offs = [self._t(N, h, w, 72, dtype=torch.float32) for h, w in self.level_sizes]
        boxes = [v['box'] for v in self.level_views]
        # BM: offsets from relu(scale * bbox_pred) (sipmask.py:161-171)
        self._add(lambda: C.offset_conv1x1_multi(boxes, self.scales, w_off, offs, relu=self.benchmark), name='offset_conv')
        cols = [self._t(N, h, w, 2304) for h, w in self.level_sizes]
        self._add(lambda: C.deform_im2col_multi(cls_feats, offs, 4, cols), name='deform_im2col')
        if self.gn:
            stats = [self.gn_arena[si, l] for l in range(len(feats))]
            b_dcn = None
            if self.benchmark:            # DeformConv(bias=True) before GN (sipmask.py:26-30,44)
                b_dcn = self._once('head.b_dcn', lambda: self._w(hp + 'feat_align.conv_adaption.bias').to(self.dev))
            aligned = self._conv_multi(cols, wk_dcn, 1, bias=b_dcn, gn_stats=stats)
            self._gn_relu(aligned, stats, hp + 'feat_align.norm')
        else:
            aligned = self._conv_multi(cols, wk_dcn, 1, relu=True)
        # fcos_cls | sip_cof on the aligned feature (sipmask_head.py:264,271)
        self._conv_multi(aligned, wk_cls, 3, outs=cls_l, bias=b_cls)
        # prototype branch on the side stream, next to FeatureAlign / the cls heads
        self._tag = 1
        # prototype input: reg feature of levels 0..2 at P3 resolution (sipmask_head.py:275-281)
        h3, w3 = self.level_sizes[0]
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
            tfe = self._tower(feats[:3], 'track_convs', self.stacked - 1, si + 1)
            cat_t = self._t(N, h3, w3, 768)
            for l in range(3):
                self._add(lambda l=l: C.upsample_bilinear(tfe[l], 2 ** l, out=cat_t, out_choff=256 * l), name='upsample')
            self.track_feats = self._conv(cat_t, hp + 'sipmask_track.weight', 1, bias_key=hp + 'sipmask_track.bias',
                                          out_dtype=torch.float32)
        self._max_ctas = self.max_ctas
        if self.build_post:
            self._build_postproc()

    def _build_fcos_head(self, feats):
        """Plain FCOS head (MM/mmdet/models/anchor_heads/fcos_head.py:118-135): 4+4 tower ConvModules, fcos_cls and
        fcos_centerness on the cls tower, fcos_reg on the reg tower (exp(scale * x) is applied by the caller)."""
        hp, ncls = self.hp, self.ncls
        CCp = (ncls + 1 + 15) // 16 * 16
        cls_l, reg_l = self._head_buffers(feats, 2 * self.stacked, CCp)
        # clscof = [cls | centerness | pad], regctr = [4 raw box distances | pad]
        self.level_views = [dict(cls=c[..., :ncls], ctr=c[..., ncls:ncls + 1], box=r[..., :4]) for c, r in zip(cls_l, reg_l)]
        w_cls = torch.cat([self._w(hp + 'fcos_cls.weight'), self._w(hp + 'fcos_centerness.weight')], 0)
        b_cls = torch.cat([self._w(hp + 'fcos_cls.bias'), self._w(hp + 'fcos_centerness.bias')], 0)
        wk_cls, _ = C.pack_weight(w_cls, cout_pad=CCp, device=self.dev)
        b_cls = torch.cat([b_cls, b_cls.new_zeros(CCp - ncls - 1)]).to(self.dev)
        wk_reg, _ = C.pack_weight(self._w(hp + 'fcos_reg.weight'), cout_pad=16, device=self.dev)
        b_reg = torch.cat([self._w(hp + 'fcos_reg.bias'), torch.zeros(12)]).to(self.dev)
        self._keep += [wk_cls, b_cls, wk_reg, b_reg]
        cls_feats = self._tower(feats, 'cls_convs', self.stacked, 0)
        reg_feats = self._tower(feats, 'reg_convs', self.stacked, self.stacked)
        self._conv_multi(cls_feats, wk_cls, 3, outs=cls_l, bias=b_cls, cout_real=ncls + 1)
        self._conv_multi(reg_feats, wk_reg, 3, outs=reg_l, bias=b_reg, cout_real=4)

    def load_features(self, feats):
        """feats: five NCHW tensors (fp16/fp32, CUDA) from the caller's neck -> the engine's NHWC fp16 buffers."""
        for buf, f in zip(self.fpn_outs, feats):
            buf.copy_(f.permute(0, 2, 3, 1))

    # ------------------------------------------------------------------------------- post-processing
    def _build_postproc(self):
        """candidates -> NMS -> coefficient gather -> mask assembly -> resize / threshold / bit-pack into the ori_shape
        canvas, image by image (get_bboxes loops over images, sipmask_head.py:517-540), all on device with fixed-shape
        outputs.  Only the candidates and the NMS depend on the checkpoint tree (_mm_candidates, _bm_candidates).
        MM: rescale=True semantics, boxes / scale_factor and masks resized by 2 / scale_factor (sipmask_head.py:587-588,
        629-633,648-654).  BM (SipMask-benchmark/fcos_core/modeling/rpn/sipmask/inference.py:66-222): boxes stay in
        resized-image coordinates, rois = boxes / 2, masks are resized by 2 / sf with sf = min(h / ori_h, w / ori_w)."""
        N, cfg = self.N, self.cfg
        nl, ncls = len(self.level_sizes), self.ncls
        nms_pre = int(cfg['nms_pre'])
        Hm, Wm = self.protos.shape[1], self.protos.shape[2]
        # per-image geometry rows [N, smb_img_geom_t]: the only per-image values the post-processing graph reads.  Kept out
        # of the arena (they persist between forwards); written here from the constructor arguments, later by set_image_meta
        self._geom_words = ctypes.sizeof(L.ImgGeom) // 4
        self.geom = torch.empty((N, self._geom_words), dtype=torch.int32, device=self.dev)
        self._geom_host = torch.empty((N, self._geom_words), dtype=torch.int32).pin_memory()
        self._geom_copied = None
        g0 = self._geometry(self.img_shape, self.ori_shape, self.scale_factor)
        if self.min_mask_up is None:
            self.mask_tile_r = (g0.ry, g0.rx)
        else:
            r = float(np.float32(1.0 / float(self.min_mask_up)))
            self.mask_tile_r = (max(r, g0.ry), max(r, g0.rx))
        from .postproc import fused_mask_tile
        fused_mask_tile(*self.mask_tile_r, sizes=(Hm, Wm, g0.full_h, g0.full_w))
        self.set_image_meta([(self.img_shape, self.ori_shape, self.scale_factor)] * N)
        torch.cuda.current_stream(self.dev).synchronize()
        # per image: its (cls, box, ctr) head outputs, level by level; every image has image 0's level sizes
        heads = [[[v[k][n] for v in self.level_views] for k in ('cls', 'box', 'ctr')] for n in range(N)]
        lv, _ = ops.level_descs(*heads[0], self.strides, self.scales)
        if self.benchmark:
            self.max_num = int(cfg['max_per_img'])
            self.ncand = L.lib().smb_pair_decode_slots(nl, lv, ncls, nms_pre)
            if self.ncand < 0 or self.ncand > 5120:
                raise ValueError('benchmark: %d candidate slots (nms_pre=%d) exceed the NMS capacity 5120' % (self.ncand, nms_pre))
            self.cand_scores = self._t(N, self.ncand, dtype=torch.float32)
            self.cand_labels = self._t(N, self.ncand, dtype=torch.int32)
            self.n_cand = self._t(N, dtype=torch.int32)
            # the number the reference keeps; the record holds the first max_per_img (ties at the k-th value keep more)
            self.kept_total = self._t(N, dtype=torch.int32, zero=True)
            candidates = self._bm_candidates
        else:
            self.max_num = 100 if self.ssd else int(cfg['max_per_img'])      # MM's fast_nms hard-codes 100 (sipmask_head.py:903)
            self.ncand = sum(min(h * w, nms_pre) if nms_pre > 0 else h * w for h, w in self.level_sizes)
            self.cand_scores = self._t(N, self.ncand, ncls, dtype=torch.float32)
            self.cand_ctr = self._t(N, self.ncand, dtype=torch.float32)
            candidates = self._mm_candidates
        self.cand_boxes = self._t(N, self.ncand, 4, dtype=torch.float32)
        self.cand_loc = self._t(N, self.ncand, dtype=torch.int32)
        cap_h, cap_w = self.mask_cap
        words = (cap_w + 31) // 32
        self.det = self._t(N, self.max_num, 5, dtype=torch.float32)
        self.labels = self._t(N, self.max_num, dtype=torch.long)
        self.idx = self._t(N, self.max_num, dtype=torch.long)
        self.count = self._t(N, dtype=torch.int32, zero=True)
        self.mask_bits = self._t(N, self.max_num, cap_h, words, dtype=torch.int32)
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
        level_hw = [h * w for h, w in self.level_sizes] if N > 1 else None
        # the per-image chains are independent (get_bboxes loops over images, sipmask_head.py:517-540): with a batch they
        # are spread over a few streams of the captured graph
        pp_streams = min(N, 4) if N > 1 else 0
        if pp_streams:
            self._marker('fork')
        for n in range(N):
            self._tag = (n % pp_streams) + 1 if pp_streams else 0
            cand_loc = candidates(n, heads[n], lv)

            def gather(n=n, cand_loc=cand_loc):
                # candidate row -> level-concatenated location -> coefficient row (mlvl_cofs[idxs_keep], sipmask_head.py:612)
                # and det[:, :4] -> contiguous rois input, one launch
                ops.gather_det_inputs(self.cof_src, cand_loc, self.idx[n], self.det[n], self.count[n:n + 1], self.det_cofs[n],
                                      self.det_boxes4[n], self.loc_kept[n], level_hw, N, n)
            self._add(gather, 1, name='gather_cofs')

            def masks(n=n):
                # fused: prototypes -> sub-region dot/sigmoid/crop -> resize -> threshold -> bit-pack (no pos_masks tensor)
                ops.mask_assemble_pack_dev(self.protos[n], self.det_cofs[n], self.det_boxes4[n], self.geom[n], self.mask_tile_r,
                                           (cap_h, cap_w), self.mask_thr, out=self.mask_bits[n])
            self._add(masks, 2, name='mask_fused')
            if self.rescoring:
                def dense(n=n):
                    # the same rois as mask_fused; rows past the count have zero boxes and are skipped by the rescoring
                    ops.mask_assemble(self.protos[n], self.det_cofs[n], self.det_boxes4[n], None, layout='hwc',
                                      out=self.pos_masks[n], geom=self.geom[n])
                self._add(dense, 1, name='mask_dense')
            if self.vis:
                def track(n=n):
                    ops.gather_track_feats(self.track_feats[n], self.det[n], self.count[n:n + 1], geom=self.geom[n],
                                           out=self.det_track[n])
                self._add(track, 1, name='gather_track')
        if pp_streams:
            self._marker('join')
        self._tag = 0
        if self.rescoring:
            self._add(lambda: ops.mask_rescore_f16(self.pos_masks, self.count, self._rescore_w, self.labels, self.det,
                                                   workspace=self._rescore_ws, out=self.mask_scores), 5, name='rescore')
        if self.rle_bytes:
            self._build_rle(cap_h, cap_w)

    def _build_rle(self, cap_h, cap_w):
        """The encoder node after the per-image chains: every detection's pycocotools string, written per image into the
        region the destination word points at (smb_rle_encode_dev).  The workspace lives in the arena (rewritten each
        forward before it is read); the destination word and the default region persist between forwards, outside it."""
        from . import rle as R
        N, mx = self.N, self.max_num
        if mx > 1024:
            raise ValueError('rle_bytes > 0 supports at most 1024 detections per image, got max_per_img=%d' % mx)
        if self.rle_runs is None:
            self.rle_runs = 4 * cap_w + 2
        self.rle_img_bytes = R.image_bytes(mx, self.rle_bytes)
        ws = self._t(ops.rle_encode_workspace_bytes(N, mx, self.rle_runs), dtype=torch.uint8)
        self._rle_dst = torch.zeros(1, dtype=torch.int64, device=self.dev)
        self._rle_stage = {}                         # region address -> (pinned word holding its device address, region)
        self.rle_region = torch.zeros(N * self.rle_img_bytes, dtype=torch.uint8).pin_memory()
        self.set_rle_dest(self.rle_region)
        torch.cuda.current_stream(self.dev).synchronize()
        geom = self.geom

        def encode():
            ops.rle_encode_dev(self.mask_bits, self.count, geom, self._rle_dst, self.rle_img_bytes, self.rle_runs, ws)
        self._add(encode, 2, name='rle_encode')

    def set_rle_dest(self, region):
        """Points the next forwards on the current stream at `region`, a pinned uint8 host tensor of at least
        N * rle_img_bytes bytes (image n's region at n * rle_img_bytes).  Stream-ordered like set_image_meta: the device
        word the encoder reads is written by an H2D copy on the current stream, from a pinned word that holds the region's
        device address and never changes, so no host wait is needed and the region stays referenced by the engine."""
        if not self.rle_bytes:
            raise ValueError('set_rle_dest: this engine was built without rle_bytes')
        if (region.dtype != torch.uint8 or region.dim() != 1 or region.is_cuda or not region.is_pinned()
                or region.numel() < self.N * self.rle_img_bytes or region.data_ptr() % 16):
            raise ValueError('set_rle_dest: need a 16-byte aligned, pinned 1-D uint8 host tensor of at least %d bytes'
                             % (self.N * self.rle_img_bytes))
        key = region.data_ptr()
        if key not in self._rle_stage:
            with torch.cuda.device(self.dev):
                addr = ops.host_device_pointer(region)
            self._rle_stage[key] = (torch.tensor([addr], dtype=torch.int64).pin_memory(), region)
        self._rle_dst.copy_(self._rle_stage[key][0], non_blocking=True)
        self._rle_region_cur = region

    def rle_results(self):
        """Per image, the list of its count RLE dicts {'size': [ori_h, ori_w], 'counts': bytes} in detection order (the
        layout pycocotools.mask.encode returns), read from the region the last forward wrote.  Valid once the stream has
        passed that forward.  An image whose strings did not fit (rle_runs / rle_bytes) is encoded on the host from this
        engine's mask_bits instead."""
        from . import rle as R
        ib, out = self.rle_img_bytes, []
        region = self._rle_region_cur.numpy()
        for n, (_, ori, _) in enumerate(self.image_metas):
            out.append(R.image_segms(region[n * ib:(n + 1) * ib], self.max_num, ori[:2],
                                     lambda k, n=n: self.mask_bits[n, :k].cpu().numpy()))
        return out

    def _geometry(self, img_shape, ori_shape, scale_factor):
        from .postproc import image_geometry
        return image_geometry(self.protos.shape[1:3], img_shape, ori_shape, scale_factor, ssd_flag=self.ssd,
                              benchmark=self.benchmark, legacy_interp=self.legacy_interp)

    def set_image_meta(self, metas):
        """metas: one (img_shape, ori_shape, scale_factor) per image of the batch, as the reference's img_meta holds them.
        Validates them against this engine (the image fits the padded input, ori_shape fits the mask record's capacity,
        the mask resize is no steeper than the tile was sized for) and writes the geometry rows with a stream-ordered
        H2D copy on the current stream: legal between graph replays, and the next forward on this stream uses them.
        For image n only mask_bits[n, :count, :ori_h, :ceil(ori_w / 32)] is meaningful; the rest of the record is zero."""
        from .postproc import fused_mask_tile
        if len(metas) != self.N:
            raise ValueError('set_image_meta: %d metas for a batch of %d' % (len(metas), self.N))
        rows = []
        Hm, Wm = self.protos.shape[1], self.protos.shape[2]
        for img_shape, ori_shape, scale_factor in metas:
            ih, iw = int(img_shape[0]), int(img_shape[1])
            oh, ow = int(ori_shape[0]), int(ori_shape[1])
            if not (0 < ih <= self.H and 0 < iw <= self.W):
                raise ValueError('set_image_meta: image %dx%d does not fit the padded input %dx%d' % (ih, iw, self.H, self.W))
            if not (0 < oh <= self.mask_cap[0] and 0 < ow <= self.mask_cap[1]):
                raise ValueError('set_image_meta: ori_shape %dx%d exceeds the mask capacity %dx%d (max_ori_hw)'
                                 % (oh, ow, self.mask_cap[0], self.mask_cap[1]))
            g = self._geometry(img_shape, ori_shape, scale_factor)
            fused_mask_tile(g.ry, g.rx, sizes=(Hm, Wm, g.full_h, g.full_w))
            if g.ry > self.mask_tile_r[0] or g.rx > self.mask_tile_r[1]:
                raise ValueError('set_image_meta: mask resize step (%g, %g) is steeper than the (%g, %g) this engine was built '
                                 'for (min_mask_up)' % (g.ry, g.rx, self.mask_tile_r[0], self.mask_tile_r[1]))
            rows.append(np.frombuffer(bytes(g), dtype=np.int32))
        if self._geom_copied is not None:
            self._geom_copied.synchronize()          # the previous copy has left the pinned staging rows
        self._geom_host.copy_(torch.from_numpy(np.stack(rows)))
        self.geom.copy_(self._geom_host, non_blocking=True)
        if self._geom_copied is None:
            self._geom_copied = torch.cuda.Event()
        self._geom_copied.record(torch.cuda.current_stream(self.dev))
        self.image_metas = [tuple(m) for m in metas]

    def _mm_candidates(self, n, head, lv):
        """MM candidates of image n (head: its (cls, box, ctr) level lists, lv: their level_descs): decode + per-level
        top-k (decode_topk), then multi-class NMS (soft-NMS when the nms type is soft_nms), or fast NMS for SSD and VIS
        (fast_nms with cfg.max_per_img, VIS/...:986).  Returns the candidate -> location table."""
        cfg, ncls, ncand, nms_pre = self.cfg, self.ncls, self.ncand, int(self.cfg['nms_pre'])
        boxes, scores, ctr, loc = self.cand_boxes[n], self.cand_scores[n], self.cand_ctr[n], self.cand_loc[n]
        rec = (self.det[n], self.labels[n], self.idx[n], self.count[n:n + 1])
        ws = self._t(ops.decode_workspace_bytes(lv, nms_pre), dtype=torch.uint8)

        def decode(n=n):
            ops.decode_topk(*head, self.strides, None, nms_pre, box_scales=self.scales, geom=self.geom[n],
                            out=(boxes, scores, ctr, loc), workspace=ws)
        self._add(decode, 3, name='decode_topk')
        if self.ssd or self.vis:
            iou_thr = float(cfg['nms']['iou_thr'])
            nws = self._t(ops.fast_nms_workspace_bytes(ncand, ncls, 200), dtype=torch.uint8)

            def nms(n=n):
                ops.fast_nms(boxes, scores, ctr, iou_thr, 200, cfg['score_thr'], self.max_num, out=rec, workspace=nws)
            self._add(nms, 2, name='nms')
            return loc
        soft = self.soft_nms is not None
        if soft and ncand > ops.SOFT_NMS_MAX:
            raise ValueError('soft_nms: %d candidates (nms_pre=%d) exceed the soft-NMS capacity %d'
                             % (ncand, nms_pre, ops.SOFT_NMS_MAX))
        nms_cfg = cfg['nms'] if soft else float(cfg['nms']['iou_thr'])
        nws = self._t(ops.multiclass_nms_workspace_bytes(ncand, ncls, soft), dtype=torch.uint8)

        def nms(n=n):
            ops.multiclass_nms_idx(boxes, scores, cfg['score_thr'], nms_cfg, self.max_num, score_factors=ctr,
                                   has_bg_column=False, out=rec, workspace=nws)
        self._add(nms, 2 if soft else 4, name='nms')
        return loc

    def _bm_candidates(self, n, head, lv):
        """BM candidates of image n (head, lv as _mm_candidates): (location, class) pairs above score_thr, the top nms_pre
        per level (pair_decode_topk), then label-aware NMS and the k-th-value cut (ml_nms_topk), which also writes
        kept_total[n].  Returns the candidate -> location table."""
        cfg, ncls, ncand, nms_pre = self.cfg, self.ncls, self.ncand, int(self.cfg['nms_pre'])
        boxes, scores, labels, loc = self.cand_boxes[n], self.cand_scores[n], self.cand_labels[n], self.cand_loc[n]
        n_cand = self.n_cand[n:n + 1]
        ws = self._t(ops.pair_decode_workspace_bytes(lv, ncls, nms_pre), dtype=torch.uint8)

        def decode(n=n):
            ops.pair_decode_topk(*head, self.strides, None, nms_pre, cfg['score_thr'], box_scales=self.scales,
                                 geom=self.geom[n], out=(boxes, scores, labels, loc, n_cand), workspace=ws)
        self._add(decode, 3, name='decode_topk')
        nws = self._t(ops.ml_nms_workspace_bytes(ncand), dtype=torch.uint8)

        def nms(n=n):
            ops.ml_nms_topk(boxes, scores, labels, n_cand, cfg['nms']['iou_thr'], self.max_num, self.max_num,
                            out=(self.det[n], self.labels[n], self.idx[n], self.count[n:n + 1], self.kept_total[n:n + 1]),
                            workspace=nws)
        self._add(nms, 4, name='nms')
        return loc

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

    def forward_raw(self, imgs, mean=(102.9801, 115.9465, 122.7717), pipeline='mmdet'):
        """imgs: N uint8 HWC CUDA images straight from the decoder (a list; one tensor when N == 1).  Image n is resized
        to its own img_shape (the constructor's, or the one set_image_meta set), mean-subtracted, zero-padded and written
        in the stem's layout by ONE kernel for the whole batch (SURVEY.md 8f-3), captured in place of the
        `image_to_s2d16` node.  A None entry is a filler image: an all-zero canvas, for a partial batch.  Per call: the
        source rows are written with a stream-ordered H2D copy on the current stream, then one graph replay.  The images
        must stay alive and unchanged until the forward has consumed them.
        pipeline='mmdet': BGR images, cv2 INTER_LINEAR (bit-exact), graph `graph_raw`.
        pipeline='benchmark' (benchmark=True engines only): RGB images as PIL decodes them, SipMask-benchmark's test
        transform (PIL bilinear, bit-exact; BGR x 255 - mean), graph `graph_raw_bm`; a downscale steeper than
        conv.PIL_MAX_DOWNSCALE on either axis raises ValueError.  mean is in BGR order for both."""
        if pipeline not in ('mmdet', 'benchmark'):
            raise ValueError("forward_raw: pipeline is 'mmdet' or 'benchmark', got %r" % (pipeline,))
        if pipeline == 'benchmark' and not self.benchmark:
            raise ValueError("forward_raw: pipeline='benchmark' needs a benchmark=True engine")
        rows = self._raw_src_rows(imgs, mean, pipeline)   # host validation: ValueError before anything is enqueued
        if torch.cuda.current_device() != self.dev.index:
            with torch.cuda.device(self.dev):
                return self._forward_raw_rows(rows, pipeline)
        return self._forward_raw_rows(rows, pipeline)

    def _raw_src_rows(self, imgs, mean, pipeline='mmdet'):
        srcs = [imgs] if isinstance(imgs, torch.Tensor) else list(imgs)
        if len(srcs) != self.N:
            raise ValueError('forward_raw: %d images for a batch of %d' % (len(srcs), self.N))
        kw = dict(order='RGB', max_downscale=C.PIL_MAX_DOWNSCALE) if pipeline == 'benchmark' else {}
        return (L.RawSrc * self.N)(*[C.raw_src_row(s, m[0][:2], (self.H, self.W), mean, self.dev, **kw)
                                     for s, m in zip(srcs, self.image_metas)])

    def _forward_raw_rows(self, rows, pipeline='mmdet'):
        """Writes the source rows the way set_image_meta writes the geometry (pinned staging -> one H2D copy on the current
        stream, the staging reused only after that copy has run), then replays the pipeline's graph.  The rows live
        outside the arena: they persist between forwards, and both pipelines' graphs read the same rows."""
        nbytes = ctypes.sizeof(rows)
        if getattr(self, '_raw_rows', None) is None:
            self._raw_rows = torch.empty(nbytes, dtype=torch.uint8, device=self.dev)
            self._raw_host = torch.empty(nbytes, dtype=torch.uint8).pin_memory()
            self._raw_copied = torch.cuda.Event()
        else:
            self._raw_copied.synchronize()           # the previous copy has left the pinned staging rows
        ctypes.memmove(self._raw_host.data_ptr(), ctypes.addressof(rows), nbytes)
        self._raw_rows.copy_(self._raw_host, non_blocking=True)
        self._raw_copied.record(torch.cuda.current_stream(self.dev))
        names = set(self.op_names) - {'image_to_s2d16', 'fork', 'join'}
        pre = C.preprocess_pil_rows if pipeline == 'benchmark' else C.preprocess_u8_rows
        attr = 'graph_raw_bm' if pipeline == 'benchmark' else 'graph_raw'
        if self.use_graph:
            if getattr(self, attr, None) is None:
                pre(self._raw_rows, self.img8)
                self._run_ops(only=names)
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    pre(self._raw_rows, self.img8)
                    self._run_ops(only=names)
                setattr(self, attr, g)
            getattr(self, attr).replay()
        else:
            pre(self._raw_rows, self.img8)
            self._run_ops(only=names)
        return self._result()

    # head outputs in the reference's layout (for parity tests / the drop-in head)
    def head_outputs(self):
        outs = dict(cls=[], bbox=[], ctr=[], cof=[])
        for l, v in enumerate(self.level_views):
            outs['cls'].append(v['cls'].permute(0, 3, 1, 2))
            outs['cof'].append(v['cof'].permute(0, 3, 1, 2))
            d = v['box'] * self.scales[l]
            if self.benchmark:
                d = torch.relu(d)                     # NORM_REG_TARGETS (sipmask.py:161-167)
            outs['bbox'].append(d.permute(0, 3, 1, 2) * self.strides[l])
            outs['ctr'].append(v['ctr'].permute(0, 3, 1, 2))
        outs['feat_masks'] = self.protos.permute(0, 3, 1, 2)
        if self.vis:
            outs['track_feats'] = self.track_feats.permute(0, 3, 1, 2)
        return outs
