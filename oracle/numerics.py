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

import numpy as np
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


# ------------------------------------------------------------------------------------------------------------ masks
# Mask chain model (mask_assemble.cu).  Per detection the kernels evaluate, at every prototype pixel inside the roi, the
# sigmoid of ONE 32-term dot product (the CropSplit cell of the pixel), bilinearly resize those values and threshold them.
#   crop geometry: exact float32 arithmetic (rois = boxes * roi_scale, roi_w = float32((float64(x2 - x1) + 0.1) / 2),
#                  inside on integer pixel coordinates, cell = trunc(float32(float32(w - x1) / roi_w)), clamped to [0, 3]);
#   logit z:       float64 dot product of the prototypes as the kernel reads them with the fp32 coefficients;
#     scalar family (sequential fmaf): |z_dev - z| <= gamma_32 sum|p c|;
#     tensor family (fp16 hi + lo coefficients, four m16n8k16 fp32 accumulations): the split costs 2^-22 sum|p c| +
#                  2^-25 sum|p| (lo is an fp16 subnormal below 2^-14), each of the four MMA steps at most 2^-22 of the
#                  running magnitude: |z_dev - z| <= 2^-20 sum|p c| + 2^-24 sum|p|.  Pixels the kernels send to their
#                  scalar cold path (a cell quotient >= 2, or a detection with a coefficient beyond the fp16 range) are
#                  bounded by the larger of the two models;
#   value:         sigmoid over [z - dz, z + dz], plus the sigmoid's own fp32 error (< 3e-7 for __expf + IEEE division
#                  and for ex2.approx + rcp.approx);
#   resize:        source index and lambda by torch's float32 rule s = r * (d + 0.5) - 0.5 (r = float32(1 / up), or
#                  in / out in float32 for recompute_scale_factor=True), evaluated both as written and FMA-contracted; where
#                  the two forms disagree the value is their midpoint and the bound grows by half the difference.  The
#                  bilinear value is float64 with the fp32 weights; its bound is the weights applied to the tap bounds plus
#                  4 * 2^-24 of the weighted tap magnitudes (three roundings deep in fp32).
# A pixel is ambiguous when |v - thr| <= bound: the kernel may decide it either way.  Every other bit is determined.
# Measured on an H100 (80 GB): at most 1.7e-6 of the in-frame pixels are ambiguous over the kernel matrix of
# tests/test_gpu_mask_bits.py and the engine configurations of the layer audit; the cap is 1e-4.
# The float64 work is restricted to each roi's extent (prototype pixels) and the output pixels whose taps reach it.
U32 = 2.0 ** -24
GAMMA32 = 32 * U32 / (1 - 32 * U32)
SIGMOID_ERR = 3e-7
COF_FP16_LIMIT = 65000.0            # the tensor family's fp16 hi part holds coefficients up to this magnitude
BILINEAR_ERR = 4 * U32
MASK_AMBIGUOUS_CAP = 1e-4


def _sigmoid(z):
    return 0.5 * (1.0 + np.tanh(0.5 * z))


class MaskVals(object):
    """One detection's prototype-resolution values: window [y0, y1) x [x0, x1) of the map (the roi's pixels), value v
    and bound b (0 outside the crop), inside mask, cell, roi (float32 x1, y1, x2, y2)."""

    def __init__(self, win, v, b, inside=None, cell=None, roi=None):
        self.win, self.v, self.b, self.inside, self.cell, self.roi = win, v, b, inside, cell, roi


def crop_rois(boxes, roi_scale4):
    """float32 rois [N, 4] = boxes * roi_scale and cell sizes roi_w, roi_h [N] exactly as the kernels compute them."""
    b = np.asarray(boxes, np.float32).reshape(-1, 4)
    s = np.atleast_1d(np.asarray(roi_scale4, np.float32))
    s = s if s.size == 4 else np.repeat(s[:1], 4)
    roi = (b * s[None, :]).astype(np.float32)
    rw = (((roi[:, 2] - roi[:, 0]).astype(np.float64) + 0.1) / 2).astype(np.float32)
    rh = (((roi[:, 3] - roi[:, 1]).astype(np.float64) + 0.1) / 2).astype(np.float32)
    return roi, rw, rh


def _crop_axis(lo, hi, cell, n):
    """Pixels p of [0, n) with lo <= p < hi (float32 compare on integers) and trunc(float32(float32(p - lo) / cell))."""
    lo, hi, cell = np.float32(lo), np.float32(hi), np.float32(cell)
    if not (np.isfinite(lo) and np.isfinite(hi)) or not hi > lo:
        return 0, 0, np.zeros(0, np.int64)
    p0 = int(min(max(np.ceil(np.float64(lo)), 0), n))
    p1 = int(min(max(np.ceil(np.float64(hi)), 0), n))
    p = np.arange(p0, max(p0, p1), dtype=np.float32)
    with np.errstate(divide='ignore', invalid='ignore', over='ignore'):
        q = ((p - lo).astype(np.float32) / cell).astype(np.float32)
    return p0, max(p0, p1), np.minimum(q, np.float32(64.0)).astype(np.int64)


def crop_geometry(boxes, roi_scale4, H, W):
    """Per detection: (window (y0, y1, x0, x1), idx_h [h], idx_w [w]) of the CropSplit crop on an H x W map; every pixel
    of the window is inside the roi, cell = clip(2 idx_h + idx_w, 0, 3)."""
    roi, rw, rh = crop_rois(boxes, roi_scale4)
    out = []
    for n in range(roi.shape[0]):
        y0, y1, ih = _crop_axis(roi[n, 1], roi[n, 3], rh[n], H)
        x0, x1, iw = _crop_axis(roi[n, 0], roi[n, 2], rw[n], W)
        if y1 == y0 or x1 == x0:
            y0 = y1 = x0 = x1 = 0
            ih, iw = ih[:0], iw[:0]
        out.append(((y0, y1, x0, x1), ih, iw))
    return out, roi


def mask_values(protos, cofs, boxes, roi_scale4, family='scalar'):
    """Float64 values and bounds of the cropped sigmoid masks (module comment above), one MaskVals per detection.
    protos [32, H, W] as the kernel receives them (numpy or torch, fp16 or fp32), cofs [N, 128] fp32, boxes [N, 4]
    image space, family 'scalar' (sequential fmaf) or 'tensor' (mma.sync, fp16 prototypes)."""
    assert family in ('scalar', 'tensor'), family
    P = protos.detach().cpu().numpy() if hasattr(protos, 'detach') else np.asarray(protos)
    C = cofs.detach().cpu().numpy() if hasattr(cofs, 'detach') else np.asarray(cofs)
    C = C.astype(np.float32).astype(np.float64).reshape(-1, 4, 32)
    _, H, W = P.shape
    geo, roi = crop_geometry(boxes.detach().cpu().numpy() if hasattr(boxes, 'detach') else boxes, roi_scale4, H, W)
    res = []
    for n, ((y0, y1, x0, x1), ih, iw) in enumerate(geo):
        h, w = y1 - y0, x1 - x0
        if h == 0:
            res.append(MaskVals((0, 0, 0, 0), np.zeros((0, 0)), np.zeros((0, 0)), np.zeros((0, 0), bool),
                                np.zeros((0, 0), np.int64), roi[n]))
            continue
        win = P[:, y0:y1, x0:x1].astype(np.float64).reshape(32, -1)
        cell = np.clip(2 * ih[:, None] + iw[None, :], 0, 3)
        sel = cell.reshape(1, -1)
        z = np.take_along_axis(C[n] @ win, sel, 0)[0]
        m = np.take_along_axis(np.abs(C[n]) @ np.abs(win), sel, 0)[0]
        if family == 'scalar':
            dz = GAMMA32 * m
        else:
            dz = 2.0 ** -20 * m + 2.0 ** -24 * np.abs(win).sum(0)
            cold = ((ih[:, None] >= 2) | (iw[None, :] >= 2)).reshape(-1)
            if np.abs(C[n]).max() > COF_FP16_LIMIT:
                cold[:] = True
            dz = np.where(cold, np.maximum(dz, GAMMA32 * m), dz)
        v = _sigmoid(z)
        b = np.maximum(_sigmoid(z + dz) - v, v - _sigmoid(z - dz)) + SIGMOID_ERR
        res.append(MaskVals((y0, y1, x0, x1), v.reshape(h, w), b.reshape(h, w), np.ones((h, w), bool), cell, roi[n]))
    return res


def dense_values(pos):
    """MaskVals of given [N, H, W] values (a kernel's pos_masks), exact: the window is each plane's non-zero extent."""
    a = pos.detach().cpu().numpy() if hasattr(pos, 'detach') else np.asarray(pos)
    res = []
    for n in range(a.shape[0]):
        nz = np.nonzero(a[n])
        if nz[0].size == 0:
            res.append(MaskVals((0, 0, 0, 0), np.zeros((0, 0)), np.zeros((0, 0))))
            continue
        y0, y1, x0, x1 = int(nz[0].min()), int(nz[0].max()) + 1, int(nz[1].min()), int(nz[1].max()) + 1
        v = a[n, y0:y1, x0:x1].astype(np.float64)
        res.append(MaskVals((y0, y1, x0, x1), v, np.zeros_like(v), v != 0))
    return res


def src_index(r, n_out, n_in):
    """[(i0, i1, lam) as written, (i0, i1, lam) FMA-contracted] of the float32 rule s = r * (d + 0.5) - 0.5, clamped at 0,
    i0 = min(trunc(s), n_in - 1), i1 = i0 + (i0 < n_in - 1), lam = float32(s - i0), for d = 0 .. n_out - 1."""
    r = np.float32(r)
    d = np.arange(n_out, dtype=np.float32) + np.float32(0.5)
    plain = (r * d).astype(np.float32) - np.float32(0.5)
    fma = (np.float64(r) * d.astype(np.float64) - 0.5).astype(np.float32)
    out = []
    for s in (plain, fma):
        s = np.maximum(s.astype(np.float32), np.float32(0.0))
        i0 = np.minimum(s.astype(np.int64), n_in - 1)
        i1 = i0 + (i0 < n_in - 1)
        lam = (s - i0.astype(np.float32)).astype(np.float32)
        out.append((i0, i1, lam))
    return out


def resize_step(n_in, full, r):
    """The source step the kernels use: r when positive, else float32(n_in) / float32(full) (recompute_scale_factor)."""
    return float(np.float32(r)) if r > 0 else float(np.float32(n_in) / np.float32(full))


class MaskRef(object):
    """Bilinear-resized reference of every detection (resize_reference)."""

    def __init__(self, dets, vals, H, W, full_hw, r_yx, out_hw, thr, proto_bytes):
        self.dets, self.vals, self.H, self.W = dets, vals, H, W
        self.full_hw, self.r_yx, self.out_hw = tuple(full_hw), tuple(r_yx), tuple(out_hw)
        self.thr = float(np.float32(thr))
        self.frame = (min(out_hw[0], full_hw[0]), min(out_hw[1], full_hw[1]))
        self.proto_bytes = proto_bytes


def _axis_range(forms, w0, w1):
    """Output indices whose taps (either form) reach source window [w0, w1): (o0, o1), empty as (0, 0)."""
    hit = np.zeros(forms[0][0].size, bool)
    for i0, i1, _ in forms:
        hit |= ((i0 >= w0) & (i0 < w1)) | ((i1 >= w0) & (i1 < w1))
    idx = np.nonzero(hit)[0]
    return (int(idx[0]), int(idx[-1]) + 1) if idx.size else (0, 0)


def resize_reference(vals, H, W, full_hw, r_yx, out_hw, thr, proto_bytes=64):
    """Per detection, the float64 bilinear values and bounds over the output pixels its window reaches, inside the valid
    frame min(out, full); all other output pixels are exactly 0.  r_yx: source steps (<= 0: in / out)."""
    fh, fw = int(full_hw[0]), int(full_hw[1])
    ry, rx = resize_step(H, fh, r_yx[0]), resize_step(W, fw, r_yx[1])
    vh, vw = min(int(out_hw[0]), fh), min(int(out_hw[1]), fw)
    fy, fx = src_index(ry, vh, H), src_index(rx, vw, W)
    same = all(np.array_equal(a, b) for f in (fy, fx) for a, b in zip(f[0], f[1]))     # FMA contraction changes nothing
    dets = []
    for d in vals:
        y0, y1, x0, x1 = d.win
        oy = _axis_range(fy, y0, y1) if y1 > y0 else (0, 0)
        ox = _axis_range(fx, x0, x1) if x1 > x0 else (0, 0)
        if oy[1] == oy[0] or ox[1] == ox[0]:
            dets.append(((0, 0), (0, 0), np.zeros((0, 0)), np.zeros((0, 0))))
            continue
        res = []
        for k, ((yi0, yi1, ly), (xi0, xi1, lx)) in enumerate(zip(fy, fx)):
            if k == 1 and same:
                res.append(res[0])
                break
            yi0, yi1, ly = yi0[oy[0]:oy[1]], yi1[oy[0]:oy[1]], ly[oy[0]:oy[1]]
            xi0, xi1, lx = xi0[ox[0]:ox[1]], xi1[ox[0]:ox[1]], lx[ox[0]:ox[1]]
            hy, hx = (np.float32(1) - ly).astype(np.float64), (np.float32(1) - lx).astype(np.float64)
            ly, lx = ly.astype(np.float64), lx.astype(np.float64)

            def tap(a, iy, ix):
                oky = ((iy >= y0) & (iy < y1)).astype(np.float64)
                okx = ((ix >= x0) & (ix < x1)).astype(np.float64)
                t = a[np.clip(iy - y0, 0, y1 - y0 - 1)][:, np.clip(ix - x0, 0, x1 - x0 - 1)]
                return t * oky[:, None] * okx[None, :]
            wts = ((hy[:, None] * hx[None, :], yi0, xi0), (hy[:, None] * lx[None, :], yi0, xi1),
                   (ly[:, None] * hx[None, :], yi1, xi0), (ly[:, None] * lx[None, :], yi1, xi1))
            v = np.zeros((oy[1] - oy[0], ox[1] - ox[0]))
            b = np.zeros_like(v)
            mag = np.zeros_like(v)
            for wt, iy, ix in wts:
                tv, tb = tap(d.v, iy, ix), tap(d.b, iy, ix)
                v += wt * tv
                b += np.abs(wt) * tb
                mag += np.abs(wt) * (np.abs(tv) + tb)
            res.append((v, b + BILINEAR_ERR * mag))
        (va, ba), (vb, bb) = res
        dets.append((oy, ox, 0.5 * (va + vb), np.maximum(ba, bb) + 0.5 * np.abs(va - vb)))
    return MaskRef(dets, vals, H, W, (fh, fw), (ry, rx), out_hw, thr, proto_bytes)


def mask_reference(protos, cofs, boxes, roi_scale4, full_hw, r_yx, out_hw, thr, family='scalar'):
    """The whole mask chain of the fused kernel (mask_values, then resize_reference)."""
    P = protos.detach().cpu() if hasattr(protos, 'detach') else protos
    vals = mask_values(P, cofs, boxes, roi_scale4, family)
    pb = 64 if str(getattr(P, 'dtype', '')).endswith('float16') else 128
    return resize_reference(vals, P.shape[1], P.shape[2], full_hw, r_yx, out_hw, thr, proto_bytes=pb)


def reference_bits(ref, n_planes, plane_h, words):
    """int32 bit planes [n_planes, plane_h, words] holding the reference's decision v > thr (ambiguous pixels included):
    what a correct kernel writes up to the ambiguous pixels."""
    px = np.zeros((n_planes, plane_h, words * 32), bool)
    for n, (oy, ox, v, _) in enumerate(ref.dets[:n_planes]):
        if oy[1] > oy[0]:
            px[n, oy[0]:oy[1], ox[0]:ox[1]] = v > ref.thr
    return np.packbits(px, axis=-1, bitorder='little').view(np.int32).reshape(n_planes, plane_h, words)


def _tile_of(ref, y, x, tile_r):
    from sipmask_b200.postproc import fused_mask_tile
    TY, TW, _ = fused_mask_tile(*(tile_r or ref.r_yx), proto_bytes=ref.proto_bytes)
    sy = int(src_index(ref.r_yx[0], y + 1, ref.H)[0][0][y])
    sx = int(src_index(ref.r_yx[1], x + 1, ref.W)[0][0][x])
    return 'fused tile (%d,%d) of %dx%d words, source pixel (%d,%d) in 8x64 dense tile (%d,%d)' % (
        y // TY, x // (32 * TW), TY, TW, sy, sx, sy // 8, sx // 64)


def check_mask_bits(bits, ref, count, cap=MASK_AMBIGUOUS_CAP, what='masks', tile_r=None):
    """Bit planes int32 [N, plane_h, words] (pixel x = bit x & 31 of word x >> 5) against a MaskRef of (at least) the first
    `count` detections: every non-ambiguous bit equals the reference, the ambiguous fraction of in-frame pixels stays
    below `cap`, everything outside the frame min(out, full) (bits past out_w of the last word included) and every plane
    at or past `count` is 0.  Returns dict(ambiguous=fraction, margin=smallest |v - thr| / bound of a decided pixel,
    pixels=in-frame pixels checked); raises BoundError naming the first wrong bit."""
    a = bits.detach().cpu().numpy() if hasattr(bits, 'detach') else np.asarray(bits)
    a = np.ascontiguousarray(a).view(np.uint32)
    Np, ph, words = a.shape
    count = min(max(int(count), 0), Np)
    if a[count:].any():
        n, y, wq = (int(i[0]) for i in np.nonzero(a[count:]))
        raise BoundError('%s: plane %d at or past the count %d is not zero (row %d, word %d = %#x)' % (
            what, count + n, count, y, wq, int(a[count + n, y, wq])))
    vh, vw = ref.frame
    assert vh <= ph and vw <= 32 * words, (ref.frame, a.shape)
    thr = ref.thr
    amb_total, margin = 0, float('inf')
    for n in range(count):
        px = np.unpackbits(a[n].view(np.uint8), axis=-1, bitorder='little').reshape(ph, 32 * words).astype(bool)
        outside = px.copy()
        outside[:vh, :vw] = False
        if outside.any():
            y, x = (int(i[0]) for i in np.nonzero(outside))
            raise BoundError('%s: detection %d has a set bit outside the %dx%d frame at (y %d, x %d)' % (what, n, vh, vw, y, x))
        oy, ox, v, b = ref.dets[n]
        got = px[:vh, :vw]
        bad = got.copy()
        if oy[1] > oy[0]:
            bad[oy[0]:oy[1], ox[0]:ox[1]] = False
            g = got[oy[0]:oy[1], ox[0]:ox[1]]
            d = np.abs(v - thr)
            amb = d <= b
            wrong = (g != (v > thr)) & ~amb
            amb_total += int(amb.sum())
            dec = ~amb & (b > 0)
            if dec.any():
                margin = min(margin, float((d[dec] / b[dec]).min()))
            if wrong.any():
                i, j = (int(t[0]) for t in np.nonzero(wrong))
                raise BoundError('%s: detection %d, y %d, x %d: bit %d, reference %.9g %s thr %.9g with bound %.3g '
                                 '(%.3g bounds away); %s' % (
                                     what, n, oy[0] + i, ox[0] + j, int(g[i, j]), v[i, j], '>' if v[i, j] > thr else '<=', thr,
                                     b[i, j], d[i, j] / b[i, j] if b[i, j] > 0 else float('inf'),
                                     _tile_of(ref, oy[0] + i, ox[0] + j, tile_r)))
        if bad.any():
            y, x = (int(i[0]) for i in np.nonzero(bad))
            raise BoundError('%s: detection %d, y %d, x %d: bit set where the reference is exactly 0; %s' % (
                what, n, y, x, _tile_of(ref, y, x, tile_r)))
    pixels = count * vh * vw
    frac = amb_total / pixels if pixels else 0.0
    if frac > cap:
        raise BoundError('%s: %.3g of the in-frame pixels are ambiguous (cap %.3g): the bound is too loose' % (what, frac, cap))
    return dict(ambiguous=frac, margin=margin, pixels=pixels)


def check_mask_values(out, vals, what='pos_masks'):
    """Dense cropped masks [N, H, W] (fp32 or fp16) against mask_values: |out - v| <= bound (plus half an fp16 spacing for
    fp16 outputs) inside the crop, exactly 0 outside it.  Returns the worst |out - v| / bound."""
    o = out.detach().cpu() if hasattr(out, 'detach') else out
    fp16 = str(o.dtype).endswith('float16')
    a = np.asarray(o.float().numpy() if hasattr(o, 'numpy') else o, np.float64)
    assert a.shape[0] >= len(vals), (a.shape, len(vals))
    worst = 0.0
    for n, d in enumerate(vals):
        y0, y1, x0, x1 = d.win
        rest = a[n].copy()
        rest[y0:y1, x0:x1] = 0.0
        if rest.any():
            y, x = (int(i[0]) for i in np.nonzero(rest))
            raise BoundError('%s: detection %d, y %d, x %d: %r outside the crop (must be 0)' % (what, n, y, x, a[n, y, x]))
        if y1 == y0:
            continue
        g = a[n, y0:y1, x0:x1]
        bound = d.b.copy()
        if fp16:
            bound += 0.5 * fp16_spacing(torch.from_numpy(d.v + d.b)).numpy()
        err = np.abs(g - d.v)
        ratio = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))
        i = int(np.argmax(ratio))
        r = float(ratio.reshape(-1)[i])
        if not r <= 1.0:
            y, x = divmod(i, x1 - x0)
            raise BoundError('%s: detection %d, y %d, x %d (8x64 tile %d,%d): out %r, ref %r, bound %.3g' % (
                what, n, y0 + y, x0 + x, (y0 + y) // 8, (x0 + x) // 64, g[y, x], d.v[y, x], bound[y, x]))
        worst = max(worst, r)
    return worst
