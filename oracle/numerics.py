"""Per-element error bounds for the engine's layers (test infrastructure only).

Every bound compares a kernel's output with the float64 value of the same operation on the operands the kernel was
given (teacher forcing), so a layer's bound does not depend on the layers before it.

Convolution model.  A wgmma convolution multiplies fp16 operands exactly and accumulates them in fp32, 16 K terms per
instruction.  With K the executed reduction length (kh * kw * Cin; 256 for the space-to-depth stem), the fp32 value before
output rounding differs from the exact one by at most

    gamma_K * m,   gamma_K = (ceil(K / 16) + 2) * 2^-22,   m = sum_k |x_k w_k| * |alpha| + |bias * alpha| + |residual|

(one rounding of the running sum per 16-term step, bounded by the running magnitude <= m, with two spare steps for the
bias, alpha and residual operations of the epilogue).  `m` is computed by a second convolution on absolute values.
  fp16 output:  |out - y| <= u + gamma_K * m, u the fp16 spacing at max(|y|, |out|) (rounding is half of that);
  fp32 output:  |out - y| <= 2^-23 |y| + gamma_K * m.
One dropped K term is about m / K, far above gamma_K * m for every K the engine runs (K <= 4608: gamma_K * K < 0.0013).

The fraction of fp16 outputs that are not the correctly rounded float64 value is reported as well, and must stay below
max(1 %, 2^9 gamma_K) = max(1 %, (ceil(K / 16) + 2) * 2^-13).  An output is misrounded when the accumulation error
carries the fp32 value across an fp16 rounding midpoint, so the fraction is about the typical error over the fp16
spacing u ~ 2^-10 |y|.  The tensor cores do not round each 16-term step to nearest: the error drifts with the number
of steps (up to ~2^-23 of the running sum per step) rather than growing like its square root, so for running sums of
the size of |y| the fraction grows like ceil(K / 16) * 2^-13.  Measured on an H100 (80 GB): 1.02-1.05 % at
K = 2304 (3x3 x 256, unit-variance operands), where the limit is 1.78 %; a flat 1 % would fail every 3x3 x 256 layer of
a correct kernel, and the per-element bound above is what catches defects.

GroupNorm statistics.  The epilogue sums each (image, group) over the 16 pixel rows of one consumer warp in fp32, stores
the partial as int64 fixed point (sum * 2^20, sum of squares * 2^16) and adds the partials with integer atomics.  The
device sum S_d then satisfies
    |S_d - S| <= sum gamma_K m + 2^-17 sum |y| + P * 2^-21,
    |Q_d - Q| <= sum (2 |y| gamma_K m + (gamma_K m)^2) + 2^-17 sum y^2 + P * 2^-17,
the 2^-17 terms covering the fp32 summation tree inside a warp (at most ten roundings) and P * half a fixed-point unit
the rounding of each partial.  P counts the partials that hold at least one valid pixel.  P = ceil(HW / 16) would
assume every warp covers 16 valid pixels; with ragged tiles a warp may cover fewer (a 21-wide map tiled 16 wide has
two partials per pixel row), so P here is H * ceil(W / 8): every patch is at
least 8 pixels wide and starts on a multiple of its width, so each partial covers whole (row, aligned 8-pixel) cells
and no two partials share one.

Tiles.  Failures name the worst element and its tile: the kernel's output patch (BH x BW = 128 pixels, chosen per map
by `conv_patch` exactly as the planner does) and its 64-channel N block.
"""
import math

import torch
import torch.nn.functional as F

GN_SUM_SCALE, GN_SQ_SCALE = 2.0 ** 20, 2.0 ** 16


def gamma_k(K):
    return (math.ceil(K / 16) + 2) * 2.0 ** -22


def fp16_spacing(v):
    """Spacing of fp16 numbers at |v| (float64 tensor): 2^(e - 10) in binade [2^e, 2^(e+1)), 2^-24 below 2^-14."""
    a = v.abs().clamp(min=2.0 ** -14, max=65504.0)
    _, e = torch.frexp(a)                       # a = mant * 2^e, mant in [0.5, 1): binade exponent e - 1
    return torch.ldexp(torch.ones_like(a), (e - 11).to(torch.int32))


def round_to_fp16(v):
    """float64 -> nearest fp16 value (ties to even), rounded once (tensor.half() on a double tensor rounds twice)."""
    s = fp16_spacing(v)
    return torch.round(v / s) * s


def conv_patch(H, W):
    """The convolution planner's 128-pixel output patch (BH, BW) for an H x W map."""
    best = None
    for bh, bw in ((1, 128), (2, 64), (4, 32), (8, 16), (16, 8)):
        t = -(-H // bh) * -(-W // bw)
        if best is None or t < best[0]:
            best = (t, bh, bw)
    return best[1], best[2]


def _pad_nhwc(x, p):
    if p == 0:
        return x
    return F.pad(x, (0, 0, p, p, p, p))


def conv_reference(x16, w16, k, stride=1, bias=None, alpha=1.0, residual=None, residual_upsample=False, pad=None,
                   out_hw=None, chunk_bytes=1 << 29):
    """Float64 (y, m) of one convolution as the kernel is told to compute it, NHWC [N, Ho, Wo, Cout], before ReLU.

    x16 NHWC fp16 (any pitch); w16 packed [Cout, k*k*Cin] fp16 with K index (r*k + s)*Cin + ci; bias fp32 [Cout];
    y = (conv + bias) * alpha + residual, the residual nearest-upsampled from its own size when residual_upsample (index
    min(floor(dst * in / out), in - 1) in fp32, as the epilogue computes it).  m = sum|x w| |alpha| + |bias alpha| +
    |residual|.  out_hw crops the output (the stem's space-to-depth input is 4 columns wider than its 4x4 valid
    convolution needs).  Runs on x16's device, in chunks of output rows so the im2col matrix stays below chunk_bytes."""
    x = x16.double()
    N, H, W, Cin = x.shape
    Cout = w16.shape[0]
    assert w16.shape[1] == k * k * Cin, (tuple(w16.shape), k, Cin)
    p = k // 2 if pad is None else pad
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    if out_hw is not None:
        assert out_hw[0] <= Ho and out_hw[1] <= Wo, (out_hw, Ho, Wo)
        Ho, Wo = out_hw
    xp = _pad_nhwc(x, p)
    w = w16.double().t().contiguous()
    wa = w.abs()
    y = torch.empty((N, Ho, Wo, Cout), dtype=torch.float64, device=x.device)
    m = torch.empty_like(y)
    rows = max(1, min(Ho, chunk_bytes // max(1, N * Wo * k * k * Cin * 8)))
    for r0 in range(0, Ho, rows):
        r1 = min(Ho, r0 + rows)
        taps = []
        for r in range(k):
            for s in range(k):
                taps.append(xp[:, r0 * stride + r:(r1 - 1) * stride + r + 1:stride, s:(Wo - 1) * stride + s + 1:stride, :])
        col = torch.cat(taps, 3).reshape(-1, k * k * Cin)
        y[:, r0:r1] = (col @ w).view(N, r1 - r0, Wo, Cout)
        m[:, r0:r1] = (col.abs() @ wa).view(N, r1 - r0, Wo, Cout)
        del col, taps
    a = float(alpha)
    if bias is not None:
        b = bias.double().view(1, 1, 1, -1)
        y = (y + b) * a
        m = m * abs(a) + (b * a).abs()
    elif a != 1.0:
        y, m = y * a, m * abs(a)
    if residual is not None:
        r = residual.double()
        if residual_upsample:
            def src(n_out, n_in):            # fp32 arithmetic of the epilogue: floor(dst * (in / out)), clamped
                f = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
                return torch.floor(torch.arange(n_out, dtype=torch.float32) * f).long().clamp(max=n_in - 1).to(r.device)
            r = r[:, src(Ho, r.shape[1])][:, :, src(Wo, r.shape[2])]
        assert r.shape == y.shape, (tuple(r.shape), tuple(y.shape))
        y = y + r
        m = m + r.abs()
    return y, m


class BoundError(AssertionError):
    pass


def _where(idx, shape, patch):
    """'image n, y, x, channel c, tile (ty, tx) of BHxBW, N block nb' of a flat index into an NHWC shape."""
    N, H, W, C = shape
    c = idx % C
    q = idx // C
    x = q % W
    q //= W
    yy = q % H
    n = q // H
    bh, bw = patch if patch is not None else conv_patch(H, W)
    return 'image %d, y %d, x %d, channel %d (tile %d,%d of %dx%d pixels, N block %d)' % (
        n, yy, x, c, yy // bh, x // bw, bh, bw, c // 64)


def check_bound(out, want, bound, what='', patch=None, fp16=None, max_misrounded=None):
    """|out - want| <= bound element by element (all float64-able tensors of one NHWC shape).  Returns a dict with the
    worst error / bound ratio and, for fp16 outputs, the fraction not equal to want rounded once to fp16; raises
    BoundError naming the worst element and its tile if the bound is broken (or a non-finite value appears where want is
    finite, or the misrounded fraction exceeds max_misrounded)."""
    o = out.double()
    shape = tuple(o.shape)
    if len(shape) != 4:
        o, want, bound = o.reshape(1, 1, -1, shape[-1]), want.reshape(1, 1, -1, shape[-1]), bound.reshape(1, 1, -1, shape[-1])
    err = (o - want).abs()
    err = torch.where(torch.isfinite(err), err, torch.full_like(err, float('inf')))
    ratio = torch.where(err == 0, torch.zeros_like(err), err / bound)
    worst = int(torch.argmax(ratio))
    r = float(ratio.view(-1)[worst])
    res = dict(ratio=r, n=o.numel())
    if fp16 is None:
        fp16 = out.dtype == torch.float16
    if fp16:
        res['misrounded'] = float((o != round_to_fp16(want)).double().mean())
    if not r <= 1.0:
        raise BoundError('%s: |out - ref| / bound = %.3g at %s: out %r, ref %r, bound %.3g' % (
            what, r, _where(worst, tuple(o.shape), patch), float(o.view(-1)[worst]), float(want.reshape(-1)[worst]),
            float(bound.reshape(-1)[worst])))
    if max_misrounded is not None and fp16 and res['misrounded'] > max_misrounded:
        bad = int(torch.argmax((o != round_to_fp16(want)).double()))
        raise BoundError('%s: %.3g%% of fp16 outputs are not the correctly rounded value (first at %s)' % (
            what, 100 * res['misrounded'], _where(bad, tuple(o.shape), patch)))
    return res


def max_misrounded(K):
    """Largest fraction of fp16 outputs allowed to differ from the correctly rounded value (module docstring)."""
    return max(0.01, (math.ceil(K / 16) + 2) * 2.0 ** -13)


def check_conv(out, y, m, K, relu=False, what='conv', patch=None):
    """The convolution bound (module docstring) of an fp16 or fp32 output against conv_reference's (y, m)."""
    want = y.clamp(min=0) if relu else y
    g = gamma_k(K)
    if out.dtype == torch.float16:
        bound = fp16_spacing(torch.maximum(want.abs(), out.double().abs().nan_to_num(0.0))) + g * m
    else:
        bound = 2.0 ** -23 * want.abs() + g * m
    return check_bound(out, want, bound, what, patch, max_misrounded=max_misrounded(K))


def check_gn_stats(stats, y, m, K, what='gn stats'):
    """Device GroupNorm statistics [N, 32, 2] int64 (sum * 2^20, sum of squares * 2^16) against the float64 pre-activation
    y [N, H, W, C] of the same convolution (module docstring).  Returns the worst ratio; raises naming image and group."""
    N, H, W, C = y.shape
    g = gamma_k(K)
    P = H * -(-W // 8)
    yg = y.reshape(N, H * W, 32, C // 32)
    eg = (g * m).reshape(N, H * W, 32, C // 32)
    S = yg.sum((1, 3))
    Q = (yg * yg).sum((1, 3))
    bs = eg.sum((1, 3)) + 2.0 ** -17 * yg.abs().sum((1, 3)) + P * 2.0 ** -21
    bq = (2 * yg.abs() * eg + eg * eg).sum((1, 3)) + 2.0 ** -17 * (yg * yg).sum((1, 3)) + P * 2.0 ** -17
    st = stats.double()
    worst = 0.0
    for name, dev, ref, b in (('sum', st[..., 0] / GN_SUM_SCALE, S, bs), ('sum of squares', st[..., 1] / GN_SQ_SCALE, Q, bq)):
        ratio = (dev - ref).abs() / b
        i = int(torch.argmax(ratio))
        r = float(ratio.view(-1)[i])
        if not r <= 1.0:
            raise BoundError('%s: GroupNorm %s of image %d, group %d: device %r, ref %r, |diff| / bound = %.3g' % (
                what, name, i // 32, i % 32, float(dev.view(-1)[i]), float(ref.view(-1)[i]), r))
        worst = max(worst, r)
    return worst


def check_rescore_chain(pos, count, conv_w, conv_b, score_w, score_b, labels, det, layers, scores, what='rescore'):
    """SipMask++ mask rescoring on tensor cores (smb_mask_rescore_f16), layer by layer, on the live rows.

    pos [n_img, max_rows, H, W] fp16 masks; count [n_img]; conv_w / conv_b the six packed fp16 [Cout, 9 Cin] weights and
    fp32 biases; score_w [classes, 128] fp16, score_b fp32; labels, det [n_img, max_rows(, 5)]; layers the layer-2..5
    fp16 activations [n_img * max_rows, h, w, C] the kernels left in a workspace that was filled with 0xFF; scores
    [n_img, max_rows] fp32.
      layer 2: float64 layer 1 rounded once to fp16, then the conv bound, plus sum |w2| (u(a1) + gamma_9 m1) for a
               layer-1 value that the fp32 kernel rounds the other way;
      layers 3-5: teacher-forced from the device's previous layer, conv bound;
      score: conv 6 on the device's layer 5 in float64, ReLU, rounded to fp16 as the kernel does, the label's 1x1 row,
             max over positions, x det.  A conv-6 value can round differently on the device only if its interval
             [y - gamma m, y + gamma m] reaches an fp16 rounding midpoint (or zero); such channels contribute their full
             possible difference, the others none.  The fp32 dot adds at most 14 roundings: 2^-20 (|b| + sum |w h|).
             Its ratio to the fp32-chain tolerance 1e-2 |want| + 2e-3 max |want| is returned, not asserted: the
             bound cannot be made 100x tighter than that tolerance without assuming less accumulation error than
             gamma_K.  gamma_576 m is a sizeable fraction of the fp16 spacing of a conv-6 value, so many of the 128
             channels may legitimately round either way on the device, each worth |w| times one fp16 ulp; with the
             synthetic scoring weights that alone is 0.4 to 4 times the old tolerance.  The defects the layer checks
             exist for (a wrong pixel in layers 2-5, hidden by the max-pool) are caught per element above.
    Rows past the count must be left as 0xFFFF in every layer, and live rows must hold no 0xFFFF (NaN) at all.
    Returns {name: worst error / bound}, plus 'score bound / 1e-2 bound'."""
    n_img, max_rows, H, W = pos.shape
    dev = pos.device
    cnt = [min(max(int(c), 0), max_rows) for c in count.tolist()]
    alive = torch.zeros(n_img * max_rows, dtype=torch.bool, device=dev)
    for n, c in enumerate(cnt):
        alive[n * max_rows:n * max_rows + c] = True
    for l, a in enumerate(layers, 2):
        ff = (a.view(torch.int16) == -1).reshape(a.shape[0], -1)
        if ff[alive].any():
            r = int(torch.nonzero(ff.any(1) & alive)[0])
            raise BoundError('%s layer %d: live row %d (image %d) holds unwritten 0xFFFF' % (what, l, r, r // max_rows,))
        if not ff[~alive].all():
            r = int(torch.nonzero(~ff.all(1) & ~alive)[0])
            raise BoundError('%s layer %d: row %d past the count of image %d was written' % (what, l, r, r // max_rows))
    res = {}
    idx = torch.nonzero(alive).view(-1)
    if idx.numel() == 0:
        return res
    x0 = pos.reshape(-1, H, W)[idx].unsqueeze(-1)
    y1, m1 = conv_reference(x0, conv_w[0], 3, 2, bias=conv_b[0], pad=0)
    a1 = y1.clamp(min=0)
    a1r = round_to_fp16(a1)
    y2, m2 = conv_reference(a1r, conv_w[1], 3, 2, bias=conv_b[1], pad=0)
    _, extra = conv_reference(fp16_spacing(a1) + gamma_k(9) * m1, conv_w[1], 3, 2, pad=0)
    out2 = layers[0][idx]
    want2 = y2.clamp(min=0)
    bound2 = fp16_spacing(torch.maximum(want2.abs(), out2.double().abs().nan_to_num(0.0))) + gamma_k(144) * m2 + extra
    res['layer 2'] = check_bound(out2, want2, bound2, '%s layer 2' % what)['ratio']
    for l in (3, 4, 5):
        x, out = layers[l - 3][idx], layers[l - 2][idx]
        y, m = conv_reference(x, conv_w[l - 1], 3, 2, bias=conv_b[l - 1], pad=0)
        res['layer %d' % l] = check_conv(out, y, m, conv_w[l - 1].shape[1], relu=True, what='%s layer %d' % (what, l))['ratio']
    y6, m6 = conv_reference(layers[3][idx], conv_w[5], 3, 2, bias=conv_b[5], pad=0)
    g6 = gamma_k(conv_w[5].shape[1]) * m6
    ry = y6.clamp(min=0)
    h = round_to_fp16(ry)
    safe = (y6 - g6 > 0) & ((ry - h).abs() + g6 < fp16_spacing(h) / 4)
    delta = torch.where(y6 + g6 <= 0, torch.zeros_like(y6),
                        torch.where(safe, torch.zeros_like(y6), (ry - h).abs() + g6 + fp16_spacing(ry + g6)))
    lab = labels.reshape(-1)[idx].long()
    ok = (lab >= 0) & (lab < score_w.shape[0])
    labc = lab.clamp(0, score_w.shape[0] - 1)
    wl = score_w.double()[labc].view(-1, 1, 1, score_w.shape[1])
    bl = score_b.double()[labc].view(-1, 1, 1)
    s = bl + (h * wl).sum(-1)
    ds = (delta * wl.abs()).sum(-1) + 2.0 ** -20 * (bl.abs() + (h * wl).abs().sum(-1))
    d4 = det.reshape(-1, 5)[idx, 4].double()
    want = torch.where(ok, d4 * s.clamp(min=0).amax((1, 2)), torch.zeros_like(d4))
    bound = torch.where(ok, d4.abs() * ds.amax((1, 2)) + 2.0 ** -23 * want.abs(), torch.zeros_like(d4))
    got = scores.reshape(-1)[idx]
    v = lambda t: t.view(1, 1, -1, 1)
    res['score'] = check_bound(v(got), v(want), v(bound), '%s score' % what, fp16=False)['ratio']
    old = 1e-2 * want.abs() + 2e-3 * want.abs().max()
    tight = float((bound / old).max()) if float(old.max()) > 0 else 0.0
    res['score bound / 1e-2 bound'] = tight
    return res
