"""Layer audit of the engine (run with -m gpu): every op of the launch sequence, one at a time, against a float64
reference of the operands it was actually given (teacher forcing), with the per-element bounds of oracle/numerics.py.

Around every op: its output region is NaN-filled first (a tile the op no longer writes cannot pass on a previous
forward's values), and every other CUDA tensor the engine owns (activations, plan operands, packed weights) must be
bitwise unchanged afterwards.  After the stepped forward the same engine replays as a CUDA graph (two streams) and must
reproduce every activation buffer and the record bit for bit.  An op name without a rule fails the audit."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import numerics as NU

pytestmark = pytest.mark.gpu

POSTPROC = {'gather_cofs', 'mask_fused', 'mask_dense', 'gather_track', 'decode_topk', 'nms'}      # bit-exact elsewhere
PATCHED = ('image_to_s2d16', 'maxpool3x3s2', 'upsample_bilinear', 'groupnorm_relu_apply_multi', 'offset_conv1x1_multi',
           'deform_im2col', 'deform_im2col_multi')


def _collect(obj, out):
    from sipmask_b200 import conv as C, ops
    if isinstance(obj, torch.Tensor):
        if obj.is_cuda:
            out.append(obj)
    elif isinstance(obj, (list, tuple)):
        for o in obj:
            _collect(o, out)
    elif isinstance(obj, dict):
        for o in obj.values():
            _collect(o, out)
    elif isinstance(obj, C.ConvPlan):
        _collect(obj._keep, out)
    elif isinstance(obj, ops.RescoreWeights):
        _collect([obj.conv_w, obj.conv_b, obj.score_w, obj.score_b], out)


def _u8(storage, dev):
    return torch.empty(0, dtype=torch.uint8, device=dev).set_(storage)


class Guard(object):
    """Bitwise guard over every storage the engine holds: prepare(outputs) NaN-fills the outputs and snapshots the rest;
    verify() checks that only the declared outputs changed."""

    def __init__(self, eng):
        ts = []
        _collect([eng._keep, eng._wcache], ts)
        self.storages = {}
        for t in ts:
            s = t.untyped_storage()
            self.storages.setdefault(s.data_ptr(), s)
        self.dev = eng.dev
        self.snap, self.outs = None, []
        self.written = []                   # every region an op wrote or added to, for the graph replay

    def prepare(self, outs, fill=True, accumulators=()):
        """outs: written by the op (NaN-filled unless fill=False); accumulators: added to by the op (not filled)."""
        for o in outs:
            if fill and o.dtype in (torch.float16, torch.float32):
                o.fill_(float('nan'))
        self.outs = list(outs) + list(accumulators)
        self.written += self.outs
        self.snap = {p: _u8(s, self.dev).clone() for p, s in self.storages.items()}

    def verify(self, what):
        for o in self.outs:
            p = o.untyped_storage().data_ptr()
            if p in self.snap:
                sv = torch.empty(0, dtype=o.dtype, device=o.device).set_(self.snap[p].untyped_storage(), o.storage_offset(),
                                                                         o.shape, o.stride())
                sv.copy_(o)
        for p, s in self.storages.items():
            now = _u8(s, self.dev)
            if not torch.equal(now, self.snap[p]):
                first = int(torch.nonzero(now != self.snap[p])[0])
                raise AssertionError('%s wrote outside its outputs: storage of %d bytes changed at byte %d'
                                     % (what, now.numel(), first))
        self.snap = None


def _u(v):
    return NU.fp16_spacing(v)


# ------------------------------------------------------------------------------------------------ per-op references
def _check_conv_plan(plan):
    from sipmask_b200 import conv as C
    d = plan.desc if not isinstance(plan, C.StemPlan) else None
    res = []
    if isinstance(plan, C.StemPlan):
        img8, wk, bias, out = plan._keep
        y, m = NU.conv_reference(img8, wk, 4, 1, bias=bias, pad=0, out_hw=out.shape[1:3])
        res.append(('stem', tuple(out.shape), 256, NU.check_conv(out, y, m, 256, relu=True, what='stem'), None))
        return res
    if isinstance(plan, C.ConvPlanMulti):
        xs, wk, outs, bias, gn = plan._keep[:5]
    else:
        x, wk, out, bias, residual, g1 = plan._keep
        xs, outs, gn = [x], [out], [g1] if g1 is not None else None
    K = wk.shape[1]
    for l, (x, out) in enumerate(zip(xs, outs)):
        r = plan.residual if not isinstance(plan, C.ConvPlanMulti) else None
        y, m = NU.conv_reference(x[..., :d.Cin], wk, d.kh, d.stride, bias=bias, alpha=plan.alpha, residual=r,
                                 residual_upsample=bool(d.residual_upsample))
        what = 'level %d' % l
        st = NU.check_conv(out, y, m, K, relu=bool(d.relu), what=what, patch=NU.conv_patch(out.shape[1], out.shape[2]))
        gr = NU.check_gn_stats(gn[l], y, m, K, what=what) if gn is not None else None
        res.append((what, tuple(out.shape), K, st, gr))
    return res


def _check_upsample(x, factor, out, choff, relu):
    N, H, W, C = x.shape
    o = out[..., choff:choff + C]
    if factor == 1:
        want = x.clamp(min=0) if relu else x
        assert torch.equal(o, want), 'copy / relu_copy is not bit-exact'
        return dict(ratio=0.0, misrounded=0.0)
    Ho, Wo = o.shape[1], o.shape[2]
    assert (Ho, Wo) == (H * factor, W * factor)
    xd = x.double()
    ref = F.interpolate(xd.permute(0, 3, 1, 2), scale_factor=factor, mode='bilinear', align_corners=False).permute(0, 2, 3, 1)
    if relu:
        ref = ref.clamp(min=0)

    def idx(n_out, n_in):
        s = ((torch.arange(n_out, dtype=torch.float64) + 0.5) / factor - 0.5).clamp(min=0)
        i0 = s.floor().long().clamp(max=n_in - 1)
        return i0.to(x.device), (i0 + 1).clamp(max=n_in - 1).to(x.device)
    y0, y1 = idx(Ho, H)
    x0, x1 = idx(Wo, W)
    a = xd.abs()
    nb = torch.maximum(torch.maximum(a[:, y0][:, :, x0], a[:, y0][:, :, x1]), torch.maximum(a[:, y1][:, :, x0], a[:, y1][:, :, x1]))
    bound = _u(torch.maximum(ref.abs(), o.double().abs().nan_to_num(0.0))) + 2.0 ** -20 * nb
    return NU.check_bound(o, ref, bound, 'upsample x%d' % factor, max_misrounded=0.01)


def _check_offsets(bboxes, scales, w, offs, relu):
    worst = 0.0
    wd = w.double()
    for l, (b, s, o) in enumerate(zip(bboxes, scales, offs)):
        bs = b[..., :4].double() * float(np.float32(s))
        if relu:
            bs = bs.clamp(min=0)
        ref = bs @ wd.t()
        bound = 2.0 ** -21 * (bs.abs() @ wd.abs().t())
        worst = max(worst, NU.check_bound(o, ref, bound, 'offset_conv level %d' % l, fp16=False)['ratio'])
    return dict(ratio=worst)


def _deform_reference(x, off, dg):
    """Float64 deformable im2col col [N,H,W,9C] (tap-major) with fp32 sample coordinates, and sum |corner * weight|."""
    N, H, W, C = x.shape
    cpg = C // dg
    dev = x.device
    hh, ww = torch.meshgrid(torch.arange(H, device=dev), torch.arange(W, device=dev), indexing='ij')
    xf = x.double().reshape(N, H * W, dg, cpg)
    col = torch.zeros(N, H, W, 9 * C, dtype=torch.float64, device=dev)
    mag = torch.zeros_like(col)
    for tap in range(9):
        i, j = tap // 3, tap % 3
        for g in range(dg):
            h_im = (hh - 1 + i).float() + off[..., g * 18 + 2 * tap]          # fp32, as the kernel adds them
            w_im = (ww - 1 + j).float() + off[..., g * 18 + 2 * tap + 1]
            inside = (h_im > -1) & (w_im > -1) & (h_im < H) & (w_im < W)
            hl, wl = torch.floor(h_im), torch.floor(w_im)
            lh, lw = (h_im - hl).double(), (w_im - wl).double()
            hl, wl = hl.long(), wl.long()
            xg = xf[:, :, g, :]
            acc = torch.zeros(N, H, W, cpg, dtype=torch.float64, device=dev)
            am = torch.zeros_like(acc)
            for dy, dx, wt in ((0, 0, (1 - lh) * (1 - lw)), (0, 1, (1 - lh) * lw), (1, 0, lh * (1 - lw)), (1, 1, lh * lw)):
                yy, xx = hl + dy, wl + dx
                ok = inside & (yy >= 0) & (xx >= 0) & (yy <= H - 1) & (xx <= W - 1)
                flat = (yy.clamp(0, H - 1) * W + xx.clamp(0, W - 1)).reshape(N, H * W, 1).expand(-1, -1, cpg)
                v = torch.gather(xg, 1, flat).view(N, H, W, cpg)
                t = (wt * ok.double()).unsqueeze(-1) * v
                acc += t
                am += t.abs()
            c0 = tap * C + g * cpg
            col[..., c0:c0 + cpg] = acc
            mag[..., c0:c0 + cpg] = am
    return col, mag


def _check_deform(xs, offs, dg, cols):
    worst = dict(ratio=0.0, misrounded=0.0)
    for l, (x, off, col) in enumerate(zip(xs, offs, cols)):
        ref, mag = _deform_reference(x, off, dg)
        bound = _u(torch.maximum(ref.abs(), col.double().abs().nan_to_num(0.0))) + 2.0 ** -20 * mag
        st = NU.check_bound(col, ref, bound, 'deform_im2col level %d' % l, max_misrounded=0.01)
        worst = dict(ratio=max(worst['ratio'], st['ratio']), misrounded=max(worst['misrounded'], st['misrounded']))
    return worst


def _check_gn_apply(before, xs, stats, gamma, beta, eps, relu):
    worst = dict(ratio=0.0, misrounded=0.0)
    g, b = gamma.double(), beta.double()
    for l, (x0, x, st) in enumerate(zip(before, xs, stats)):
        N, H, W, C = x0.shape
        cnt = H * W * (C // 32)
        s = st[..., 0].double() / NU.GN_SUM_SCALE
        ss = st[..., 1].double() / NU.GN_SQ_SCALE
        mean = s / cnt
        var = (ss / cnt - mean * mean).clamp(min=0)
        rstd = 1.0 / torch.sqrt(var + eps)
        mu = mean.repeat_interleave(C // 32, 1).view(N, 1, 1, C)
        rs = rstd.repeat_interleave(C // 32, 1).view(N, 1, 1, C)
        xd = x0.double()
        ref = (xd - mu) * rs * g + b
        if relu:
            ref = ref.clamp(min=0)
        bound = _u(torch.maximum(ref.abs(), x.double().abs().nan_to_num(0.0))) + 2.0 ** -16 * ((xd - mu).abs() * rs * g.abs()
                                                                                               + b.abs())
        st_ = NU.check_bound(x, ref, bound, 'gn_apply level %d' % l, max_misrounded=0.01)
        worst = dict(ratio=max(worst['ratio'], st_['ratio']), misrounded=max(worst['misrounded'], st_['misrounded']))
    return worst


def _check_rescore(eng, pos, count, labels, det, out):
    """Scores of live rows against the fp32 chain (ops.mask_rescore) on the same fp16 masks, to 1e-2 |want| + 2e-3 max|want|;
    rows past the count exactly 0."""
    from sipmask_b200 import ops
    hp = eng.hp
    cw = [eng._w('%sconvs_scoring.%d.conv.weight' % (hp, i)).to(eng.dev) for i in range(6)]
    cb = [eng._w('%sconvs_scoring.%d.conv.bias' % (hp, i)).to(eng.dev) for i in range(6)]
    w1, b1 = eng._w(hp + 'mask_scoring.weight').to(eng.dev), eng._w(hp + 'mask_scoring.bias').to(eng.dev)
    n_img, max_rows, Hm, Wm = pos.shape
    layers = ops.mask_rescore_f16_layers(eng._rescore_ws, n_img * max_rows, Hm, Wm)
    rw = eng._rescore_w
    res = NU.check_rescore_chain(pos, count, rw.conv_w, rw.conv_b, rw.score_w, rw.score_b, labels, det, layers, out)
    worst, live = 0.0, 0
    for n in range(pos.shape[0]):
        k = int(count[n])
        assert (out[n, k:] == 0).all(), 'rescore: rows past the count of image %d are not 0' % n
        if k == 0:
            continue
        live += k
        want = ops.mask_rescore(pos[n, :k].float(), cw, cb, w1, b1, labels[n, :k], det[n, :k]).double()
        bound = 1e-2 * want.abs() + 2e-3 * want.abs().max()
        worst = max(worst, NU.check_bound(out[n, :k].view(1, 1, k, 1), want.view(1, 1, k, 1), bound.view(1, 1, k, 1),
                                          'rescore image %d' % n, fp16=False)['ratio'])
    assert live > 0, 'rescore: no live rows to check'
    return dict(ratio=max(worst, max(v for k, v in res.items() if k != 'score bound / 1e-2 bound')),
                tight=res['score bound / 1e-2 bound'])


# ------------------------------------------------------------------------------------------------------- the audit
def audit(eng, log=print):
    """Steps through eng.ops; returns {kind: [ratio, misrounded, count]} and checks the graph replay afterwards."""
    from sipmask_b200 import conv as C, ops
    guard = Guard(eng)
    calls = []
    orig = {n: getattr(C, n) for n in PATCHED}
    orig_rescore = ops.mask_rescore_f16

    def outputs(name, a, kw):
        if name == 'image_to_s2d16':
            return [a[1]]
        if name == 'maxpool3x3s2':
            return [a[1]]
        if name == 'upsample_bilinear':
            out, choff, C_ = kw['out'], kw.get('out_choff', 0), a[0].shape[3]
            return [out[..., choff:choff + C_]]
        if name == 'groupnorm_relu_apply_multi':
            return list(a[0])
        if name == 'offset_conv1x1_multi':
            return list(a[3])
        if name == 'deform_im2col':
            return [kw['out']]
        if name == 'deform_im2col_multi':
            return list(a[3])
        raise AssertionError(name)

    def wrap(name):
        def f(*a, **kw):
            before = [x.clone() for x in a[0]] if name == 'groupnorm_relu_apply_multi' else None
            guard.prepare(outputs(name, a, kw), fill=name != 'groupnorm_relu_apply_multi')
            r = orig[name](*a, **kw)
            calls.append((name, a, kw, before))
            return r
        return f

    def rescore(pos, count, wt, labels, det, workspace=None, out=None):
        workspace.fill_(0xFF)
        guard.prepare([out, workspace])
        r = orig_rescore(pos, count, wt, labels, det, workspace=workspace, out=out)
        calls.append(('rescore', (pos, count, wt, labels, det, out), {}, None))
        return r

    summary = {}

    by_k = summary.setdefault('misrounded by K', {})

    def note(kind, i, label, shape, K, st, gn=None, new_op=True):
        e = summary.setdefault(kind, [0.0, 0.0, 0, 0.0])
        e[0] = max(e[0], st.get('ratio', 0.0))
        e[1] = max(e[1], st.get('misrounded', 0.0))
        e[2] += int(new_op)
        if K and 'misrounded' in st:
            by_k[K] = max(by_k.get(K, 0.0), st['misrounded'])
        if gn is not None:
            e[3] = max(e[3], gn)
        log('%4d %-34s %-22s K=%-5s err/bound %.3f  misrounded %.4f%s' % (
            i, label[:34], shape, K if K else '-', st.get('ratio', 0.0), st.get('misrounded', 0.0),
            '  gn %.3f' % gn if gn is not None else ''))

    for n in PATCHED:
        setattr(C, n, wrap(n))
    ops.mask_rescore_f16 = rescore
    try:
        wkey = {id(p): meta['name'] for p, meta in zip(eng.conv_plans, eng.conv_meta)}
        for i, (f, name) in enumerate(zip(eng.ops, eng.op_names)):
            if f is None:
                continue
            if name in POSTPROC:
                f()
                continue
            if name == 'conv':
                plan = f.__self__
                outs = plan._keep[2] if not isinstance(plan, C.StemPlan) else plan._keep[3]
                stats = [] if isinstance(plan, C.StemPlan) else plan._keep[4] if isinstance(plan, C.ConvPlanMulti) else \
                    [plan.gn_stats]
                guard.prepare(outs if isinstance(outs, list) else [outs], accumulators=[t for t in stats or [] if t is not None])
                f()
                torch.cuda.synchronize()
                guard.verify('op %d conv %s' % (i, wkey[id(plan)]))
                for j, (lvl, shape, K, st, gn) in enumerate(_check_conv_plan(plan)):
                    out0 = plan.out[0] if isinstance(plan.out, list) else plan.out
                    kind = 'stem' if isinstance(plan, C.StemPlan) else 'conv fp32 out' if out0.dtype == torch.float32 else 'conv'
                    note(kind, i, '%s %s' % (wkey[id(plan)], lvl), shape, K, st, gn, new_op=j == 0)
                continue
            if name == 'memset':
                eng.gn_arena.fill_(-1)
                guard.prepare([eng.gn_arena])
                f()
                torch.cuda.synchronize()
                guard.verify('op %d memset' % i)
                assert (eng.gn_arena == 0).all()
                note('memset', i, name, tuple(eng.gn_arena.shape), None, dict(ratio=0.0))
                continue
            n0 = len(calls)
            if name not in ('image_to_s2d16', 'maxpool', 'relu_copy', 'upsample', 'offset_conv', 'deform_im2col', 'gn_apply',
                            'rescore'):
                raise AssertionError('op %d: no audit rule for %r' % (i, name))
            f()
            torch.cuda.synchronize()
            guard.verify('op %d %s' % (i, name))
            assert len(calls) == n0 + 1, 'op %d %s: expected one recorded call, got %d' % (i, name, len(calls) - n0)
            cn, a, kw, before = calls[-1]
            if cn == 'image_to_s2d16':
                img, out = a
                N, _, H, W = img.shape
                p = torch.zeros(N, H + 6, W + 8, 4, device=img.device, dtype=torch.float16)
                p[:, 3:3 + H, 3:3 + W, :3] = img.half().permute(0, 2, 3, 1)
                want = p.view(N, H // 2 + 3, 2, W // 2 + 4, 2, 4).permute(0, 1, 3, 2, 4, 5).reshape(out.shape)
                assert torch.equal(out, want), 'image_to_s2d16 is not bit-exact'
                note('image_to_s2d16', i, name, tuple(out.shape), None, dict(ratio=0.0))
            elif cn == 'maxpool3x3s2':
                x, out = a
                want = F.max_pool2d(x.float().permute(0, 3, 1, 2), 3, 2, 1).permute(0, 2, 3, 1).half()
                assert torch.equal(out, want), 'maxpool is not bit-exact'
                note('maxpool', i, name, tuple(out.shape), None, dict(ratio=0.0))
            elif cn == 'upsample_bilinear':
                x, factor = a[0], a[1]
                st = _check_upsample(x, factor, kw['out'], kw.get('out_choff', 0), kw.get('relu', False))
                note(name if factor > 1 else name + ' x1', i, '%s x%d' % (name, factor), tuple(kw['out'].shape), None, st)
            elif cn == 'offset_conv1x1_multi':
                note('offset_conv', i, name, tuple(a[3][0].shape), 4,
                     _check_offsets(a[0], a[1], a[2], a[3], kw.get('relu', False)))
            elif cn == 'deform_im2col':
                note('deform_im2col dg%d' % a[2], i, name, tuple(kw['out'].shape), None,
                     _check_deform([a[0]], [a[1]], a[2], [kw['out']]))
            elif cn == 'deform_im2col_multi':
                note('deform_im2col dg%d' % a[2], i, name, tuple(a[3][0].shape), None, _check_deform(a[0], a[1], a[2], a[3]))
            elif cn == 'groupnorm_relu_apply_multi':
                xs, stats, gamma, beta, eps, relu = a
                note('gn_apply', i, name, tuple(xs[0].shape), None, _check_gn_apply(before, xs, stats, gamma, beta, eps, relu))
            elif cn == 'rescore':
                pos, count, wt, labels, det, out = a
                st = _check_rescore(eng, pos, count, labels, det, out)
                log('     rescore score bound / fp32-chain tolerance %.3f' % st['tight'])
                note('rescore', i, name, tuple(pos.shape), None, st)
    finally:
        for n in PATCHED:
            setattr(C, n, orig[n])
        ops.mask_rescore_f16 = orig_rescore
    torch.cuda.synchronize()
    # the same engine replayed as a CUDA graph over its two-stream schedule: every buffer bit-identical
    ts = []
    _collect(eng._keep, ts)
    ts = [t for t in ts if t.dtype != torch.uint8]          # workspaces are scratch
    stepped = [t.clone() for t in ts]
    # capture first (capturing runs nothing), then poison every region the audited ops write, then replay: a node that
    # the graph no longer runs, or a tile it no longer writes, cannot pass on the stepped run's values
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        eng._run_ops()
    for t in guard.written:
        t.fill_(float('nan') if t.is_floating_point() else -1)
    graph.replay()
    torch.cuda.synchronize()
    for j, (t, s) in enumerate(zip(ts, stepped)):
        assert torch.equal(t, s) or (torch.isnan(t) == torch.isnan(s)).all() and torch.equal(t.nan_to_num(0), s.nan_to_num(0)), \
            'graph replay differs from the stepped run in buffer %d %s' % (j, tuple(t.shape))
    return summary


# -------------------------------------------------------------------------------------------------- configurations
def _engine(cfg):
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    if cfg == 'mm_r50_b2':
        sd = synth.detector_state_dict(50, 4, gn=True, seed=1, cls_bias=-2.5)
        return SipMaskEngine(sd, (128, 192), batch=2, img_shape=(128, 187, 3), use_graph=False), (128, 192, 2)
    if cfg == 'workload_a':
        sd = synth.detector_state_dict(50, 4, gn=True, seed=1, cls_bias=-2.5)
        return SipMaskEngine(sd, (800, 1344), batch=1, img_shape=(800, 1333, 3), use_graph=False), (800, 1344, 1)
    if cfg == 'pp':
        sd = synth.detector_state_dict(depth=50, stacked_convs=2, gn=False, rescoring_flag=True, backbone_dcn=True, seed=1,
                                       cls_bias=-2.5)
        cfg_ = dict(nms_pre=200, score_thr=0.1, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
        return SipMaskEngine(sd, (256, 256), batch=2, depth=50, stacked_convs=2, gn=False, ssd_flag=True, backbone_dcn=True,
                             test_cfg=cfg_, rescoring_flag=True, scale_factor=np.ones(4, dtype=np.float32),
                             use_graph=False), (256, 256, 2)
    if cfg == 'bm':
        from sipmask_b200 import benchmark as B
        sd = B.convert_state_dict(B.synthetic_state_dict())
        return SipMaskEngine(sd, (128, 192), batch=2, img_shape=(120, 187, 3), use_graph=False, benchmark=True), (128, 192, 2)
    if cfg == 'vis':
        sd = {}
        sd.update(synth.backbone_state_dict(50, 1))
        sd.update(synth.neck_state_dict(2))
        sd.update(synth.head_state_dict(3, num_classes=41, stacked_convs=3, gn=True, cls_bias=-2.5, track=True))
        cfg_ = dict(nms_pre=200, score_thr=0.03, nms=dict(type='nms', iou_thr=0.5), max_per_img=10)
        return SipMaskEngine(sd, (384, 640), stacked_convs=3, num_classes=41, test_cfg=cfg_, img_shape=(360, 640, 3),
                             use_graph=False, vis=True), (384, 640, 1)
    if cfg == 'fcos_head':
        sd = synth.head_state_dict(3, prefix='', stacked_convs=5, gn=True)
        sizes = ((25, 37), (13, 19), (7, 10), (4, 5), (1, 3))
        return SipMaskEngine(sd, (0, 0), batch=2, stacked_convs=4, gn=True, use_graph=False, head_only=True, feat_sizes=sizes,
                             fcos=True, prefix_head='', build_postproc=False), None
    if cfg == 'workload_b':
        sd = synth.detector_state_dict(50, 2, gn=False, seed=1, cls_bias=-2.5)
        return SipMaskEngine(sd, (544, 544), batch=3, stacked_convs=2, gn=False, ssd_flag=True,
                             scale_factor=np.ones(4, dtype=np.float32), use_graph=False), (544, 544, 3)
    raise KeyError(cfg)


CONFIGS = ['mm_r50_b2', 'workload_a', 'pp', 'bm', 'vis', 'fcos_head', 'workload_b']


@pytest.mark.parametrize('cfg', CONFIGS)
def test_every_engine_layer_within_its_bound(cfg):
    from sipmask_b200 import synth
    eng, shp = _engine(cfg)
    if shp is None:
        g = torch.Generator().manual_seed(5)
        for t in eng.fpn_outs:
            t.copy_((torch.randn(t.shape, generator=g) * 2).half())
    else:
        H, W, N = shp
        eng.img.copy_(torch.cat([synth.synthetic_image(H, W, seed=s) for s in range(N)], 0))
    lines = []
    summary = audit(eng, log=lines.append)
    print('\n'.join(lines))
    by_k = summary.pop('misrounded by K')
    print('%s ops audited: ' % cfg + ', '.join('%s x%d (worst err/bound %.3f, misrounded %.4f)' % (k, v[2], v[0], v[1])
                                               for k, v in sorted(summary.items())))
    print('%s misrounded fp16 outputs by K: ' % cfg + ', '.join('K=%d %.4f' % kv for kv in sorted(by_k.items())))
    assert summary['conv'][2] > 0 and summary['conv fp32 out'][2] > 0
