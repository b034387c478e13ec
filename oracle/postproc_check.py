"""Checkers for the selection and gather kernels of the post-processing (nms.cu), teacher-forced on the operands each
kernel was given (test infrastructure only).

Every check raises CheckError naming the field and the index of the first wrong element.

Sigmoid bound.  The MM candidate kernels compute sigmoidf_(x) = 1.0f / (1.0f + __expf(-x)) with IEEE round-to-nearest
add and divide (no fast-math).  The CUDA Programming Guide gives __expf(y) a maximum error of 2 + floor(|1.173 y|) ulp,
and one ulp of a normal float32 v is at most 2^-23 |v|, so for e = exp(y)

    e_dev in [e (1 - k 2^-23), e (1 + k 2^-23)],   k = 2 + floor(1.173 |y|).

__expf flushes results below 2^-126 to zero, so the lower end drops to 0 there; where the upper end reaches the float32
overflow threshold it may return inf (s = 0), and where the lower end does it does.
Then t = 1 + e_dev and s = 1 / t are each rounded once: t in [(1 + e_lo)(1 - u), (1 + e_hi)(1 + u)], u = 2^-24, and
s in [(1 / t_hi)(1 - u) - 2^-149, (1 / t_lo)(1 + u) + 2^-149] clipped to [0, 1] (the 2^-149 covers a subnormal
quotient; t = inf gives s = 0).  x = +inf gives exactly 1, x = -inf exactly 0.  Products of two such values
(__fmul_rn) widen by one more rounding.  The float64 arithmetic that evaluates the interval is widened by 2^-50 per step.
Because every bound is monotone in x, sigmoidf_(max_c x_c) and max_c sigmoidf_(x_c) lie in the same interval: the
ranking key sigmoid(max_c cls) * sigmoid(ctr) of level_score_kernel is checked against it, and, exactly, against the
max over classes of the products of the scores the kernel wrote.

Candidate selection.  Per level with more than nms_pre locations, a location whose key interval lies above the
intervals of all but fewer than nms_pre others must be selected; one with at least nms_pre intervals entirely above it
must not be.  The rest are ambiguous: the kernel's sigmoid error can decide them either way.  Their number is reported
and capped (CANDIDATE_AMBIGUOUS_CAP, a fraction of the locations of levels that are cut).

Everything else (boxes, the BM pair path, every NMS, the gathers) is IEEE round-to-nearest arithmetic and is restated
in float32 numpy with the kernels' operation order: bit-exact, nothing ambiguous.
"""
import numpy as np

U = 2.0 ** -24
SLACK = 2.0 ** -50
TINY = 2.0 ** -149
FLT_MIN = 2.0 ** -126
FLT_OVF = 2.0 ** 128 * (1 - 2.0 ** -25)           # values from here on round to inf
# measured on an H100 (80 GB): no ambiguous location in the ~53,000 of cut levels of the layer audit's configurations
CANDIDATE_AMBIGUOUS_CAP = 1e-4


class CheckError(AssertionError):
    pass


def _fail(what, field, i, msg):
    raise CheckError('%s: %s[%s] %s' % (what, field, i, msg))


def _first(bad):
    return int(np.flatnonzero(np.asarray(bad).reshape(-1))[0])


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype == np.float32:
        return a.view(np.uint32) == b.astype(np.float32).view(np.uint32)
    return a == b


def expect_equal(what, field, got, want):
    """Bitwise equality of two arrays of the same shape; the first differing element is named (row index for 2-D)."""
    got, want = np.asarray(got), np.asarray(want)
    if got.shape != want.shape:
        raise CheckError('%s: %s has shape %s, expected %s' % (what, field, got.shape, want.shape))
    eq = _bits_equal(got, want.astype(got.dtype))
    if not eq.all():
        j = _first(~eq)
        idx = np.unravel_index(j, got.shape)
        i = idx[0] if len(idx) == 1 else tuple(int(v) for v in idx)
        _fail(what, field, i, 'is %r, expected %r' % (got.reshape(-1)[j], want.reshape(-1)[j]))


# -------------------------------------------------------------------------------------------------------- sigmoid
def sigmoid64(x):
    x = np.asarray(x, np.float64)
    with np.errstate(over='ignore'):
        return np.where(x >= 0, 1.0 / (1.0 + np.exp(-np.abs(x))), np.exp(-np.abs(x)) / (1.0 + np.exp(-np.abs(x))))


def sigmoidf_interval(x):
    """[lo, hi] (float64) holding the device's sigmoidf_(x) for float32 x (module comment).  NaN gives NaN bounds."""
    x = np.asarray(x, np.float32).astype(np.float64)
    y = -x
    fin = np.isfinite(y)
    yf = np.where(fin, y, 0.0)
    with np.errstate(over='ignore', invalid='ignore'):
        e = np.exp(yf)
        k = 2.0 + np.floor(1.173 * np.abs(yf))
        rel = k * 2.0 ** -23
        e_lo = np.maximum(e * (1 - rel) * (1 - SLACK), 0.0)
        e_hi = e * (1 + rel) * (1 + SLACK)
        e_lo = np.where(e_lo < FLT_MIN, 0.0, e_lo)
        e_hi = np.where(e_hi < FLT_MIN, FLT_MIN, e_hi)
        t_lo = (1.0 + e_lo) * (1 - U) * (1 - SLACK)
        t_hi = (1.0 + e_hi) * (1 + U) * (1 + SLACK)
        lo = np.clip((1.0 / t_hi) * (1 - U) * (1 - SLACK) - TINY, 0.0, 1.0)
        hi = np.clip((1.0 / t_lo) * (1 + U) * (1 + SLACK) + TINY, 0.0, 1.0)
        lo = np.where(e_hi >= FLT_OVF, 0.0, lo)             # __expf may return inf: s = 0
        hi = np.where(e_lo >= FLT_OVF, 0.0, hi)             # __expf returns inf
    lo = np.where(x == np.inf, 1.0, np.where(x == -np.inf, 0.0, lo))
    hi = np.where(x == np.inf, 1.0, np.where(x == -np.inf, 0.0, hi))
    nan = np.isnan(x)
    return np.where(nan, np.nan, lo), np.where(nan, np.nan, hi)


def product_interval(a, b):
    """Interval of __fmul_rn(p, q) for p in a = (lo, hi), q in b, all non-negative."""
    lo = a[0] * b[0] * (1 - U) * (1 - SLACK) - TINY
    hi = a[1] * b[1] * (1 + U) * (1 + SLACK) + TINY
    return np.maximum(lo, 0.0), hi


def sigmoid_f32(x):
    """A float32 sigmoid with one rounding per step (float64 exp rounded to float32): within sigmoidf_interval, used to
    emulate the kernels on the host."""
    x = np.asarray(x, np.float32)
    with np.errstate(over='ignore'):
        e = np.exp(-x.astype(np.float64)).astype(np.float32)
    return (np.float32(1.0) / (np.float32(1.0) + e)).astype(np.float32)


def f32(v):
    return np.asarray(v, dtype=np.float32)


# ----------------------------------------------------------------------------------------- MM decode + top-k
def level_inputs(cls, box, ctr, stride, box_scale=1.0, box_mul=1.0):
    """One level as the candidate kernels read it: cls [h, w, C], box [h, w, 4], ctr [h, w(, 1)] (numpy or torch)."""
    def np_(t):
        return t.detach().cpu().numpy() if hasattr(t, 'detach') else np.asarray(t)
    c = np_(cls).astype(np.float32)
    h, w, C = c.shape
    return dict(cls=c.reshape(h * w, C), box=np_(box).astype(np.float32).reshape(h * w, 4),
                ctr=np_(ctr).astype(np.float32).reshape(h * w), h=h, w=w, stride=int(stride),
                box_scale=np.float32(box_scale), box_mul=np.float32(box_mul))


def geometry(img_h, img_w, scale=(1.0, 1.0, 1.0, 1.0), track_sx=1.0, track_sy=1.0):
    return dict(img_h=int(img_h), img_w=int(img_w), scale=f32(np.broadcast_to(np.asarray(scale, np.float32), (4,))),
                track_sx=np.float32(track_sx), track_sy=np.float32(track_sy))


def geometry_from_row(row):
    """geometry() of an smb_img_geom_t (sipmask_b200._lib.ImgGeom)."""
    return geometry(row.img_h, row.img_w, list(row.scale), row.track_sx, row.track_sy)


def decode_boxes(lv, sel, geom, divide=True):
    """gather_decode_kernel's boxes of locations `sel` in float32: distance = (d * box_scale) * box_mul, point - / +
    distance, clamp to [0, img_w - 1] x [0, img_h - 1], then x1, y1, x2, y2 divided by scale[0..3] (divide=False: the
    BM pair path, relu'd distances, no division)."""
    sel = np.asarray(sel, np.int64)
    y, x = sel // lv['w'], sel % lv['w']
    s = lv['stride']
    px, py = f32(x * s + s // 2), f32(y * s + s // 2)
    d = lv['box'][sel]
    d = f32(d * lv['box_scale'])
    if not divide:
        d = np.fmax(d, np.float32(0))
    d = f32(d * lv['box_mul'])
    mw, mh = np.float32(geom['img_w'] - 1), np.float32(geom['img_h'] - 1)
    z = np.float32(0)
    x1 = np.fmin(np.fmax(f32(px - d[:, 0]), z), mw)
    y1 = np.fmin(np.fmax(f32(py - d[:, 1]), z), mh)
    x2 = np.fmin(np.fmax(f32(px + d[:, 2]), z), mw)
    y2 = np.fmin(np.fmax(f32(py + d[:, 3]), z), mh)
    if divide:
        sc = geom['scale']
        x1, y1, x2, y2 = f32(x1 / sc[0]), f32(y1 / sc[1]), f32(x2 / sc[2]), f32(y2 / sc[3])
    return np.stack([x1, y1, x2, y2], 1).astype(np.float32)


def _level_max(cls):
    with np.errstate(invalid='ignore'):
        return np.fmax.reduce(cls, axis=1) if cls.shape[1] else np.full(cls.shape[0], -np.inf, np.float32)


def key_intervals(lv):
    """Interval of level_score_kernel's key sigmoidf_(max_c cls) * sigmoidf_(ctr) at every location of the level."""
    return product_interval(sigmoidf_interval(_level_max(lv['cls'])), sigmoidf_interval(lv['ctr']))


def emulate_decode_topk(levels, nms_pre, geom):
    """The candidate kernels with sigmoid_f32 in place of sigmoidf_: (boxes, scores, ctr, loc).  A stand-in kernel for
    the host tests of check_candidates."""
    out_b, out_s, out_c, out_l, off = [], [], [], [], 0
    for lv in levels:
        hw = lv['h'] * lv['w']
        key = f32(sigmoid_f32(_level_max(lv['cls'])) * sigmoid_f32(lv['ctr']))
        if nms_pre > 0 and hw > nms_pre:
            sel = np.lexsort((np.arange(hw), -key.astype(np.float64)))[:nms_pre]
        else:
            sel = np.arange(hw)
        out_b.append(decode_boxes(lv, sel, geom))
        out_s.append(sigmoid_f32(lv['cls'][sel]))
        out_c.append(sigmoid_f32(lv['ctr'][sel]))
        out_l.append((sel + off).astype(np.int32))
        off += hw
    return np.concatenate(out_b), np.concatenate(out_s), np.concatenate(out_c), np.concatenate(out_l)


def check_candidates(levels, nms_pre, geom, boxes, scores, ctr, loc, what='decode_topk',
                     cap=CANDIDATE_AMBIGUOUS_CAP):
    """smb_decode_topk(_dev) outputs (boxes [n, 4], scores [n, C], ctr [n], loc [n]) against the level inputs (list of
    level_inputs()), nms_pre and the geometry row (geometry()).  Returns dict(locations, cut_locations, ambiguous)."""
    boxes, scores = np.asarray(boxes, np.float32), np.asarray(scores, np.float32)
    ctr, loc = np.asarray(ctr, np.float32), np.asarray(loc).astype(np.int64)
    q0, loc0 = 0, 0
    n_cut, n_amb, n_loc = 0, 0, 0
    for l, lv in enumerate(levels):
        hw = lv['h'] * lv['w']
        k = min(hw, nms_pre) if nms_pre > 0 else hw
        q = np.arange(q0, q0 + k)
        if q0 + k > loc.shape[0]:
            raise CheckError('%s: level %d needs candidates %d..%d, only %d written' % (what, l, q0, q0 + k - 1, loc.shape[0]))
        sel = loc[q] - loc0
        bad = (sel < 0) | (sel >= hw)
        if bad.any():
            j = _first(bad)
            _fail(what, 'loc', q0 + j, '= %d is outside level %d (locations %d..%d)' % (loc[q0 + j], l, loc0, loc0 + hw - 1))
        n_loc += hw
        # scores and centerness within the sigmoid bound, boxes bit-exact
        lo, hi = sigmoidf_interval(lv['cls'][sel])
        s = scores[q].astype(np.float64)
        bad = ~((s >= lo) & (s <= hi))
        if bad.any():
            j = _first(bad)
            r, c = divmod(j, s.shape[1])
            _fail(what, 'scores', (q0 + r, c), '= %r outside the sigmoid bound [%r, %r] of logit %r'
                  % (float(s[r, c]), lo[r, c], hi[r, c], float(lv['cls'][sel[r], c])))
        lo, hi = sigmoidf_interval(lv['ctr'][sel])
        t = ctr[q].astype(np.float64)
        bad = ~((t >= lo) & (t <= hi))
        if bad.any():
            j = _first(bad)
            _fail(what, 'ctr', q0 + j, '= %r outside the sigmoid bound [%r, %r]' % (float(t[j]), lo[j], hi[j]))
        want = decode_boxes(lv, sel, geom)
        eq = _bits_equal(boxes[q], want).all(1)
        if not eq.all():
            j = _first(~eq)
            _fail(what, 'boxes', q0 + j, '= %s, expected %s (location %d of level %d)'
                  % (boxes[q0 + j].tolist(), want[j].tolist(), sel[j], l))
        if k == hw:
            if not (sel == np.arange(hw)).all():
                j = _first(sel != np.arange(hw))
                _fail(what, 'loc', q0 + j, '= %d: an uncut level lists its locations in order (expected %d)'
                      % (loc[q0 + j], loc0 + j))
        else:
            n_cut += hw
            if np.unique(sel).size != k:
                _fail(what, 'loc', q0, 'level %d selects a location twice' % l)
            # the kernel's own keys: sigmoidf_(max logit) is the score it wrote for the max-logit class
            cs = _level_max(lv['cls'][sel])
            cstar = np.argmax(lv['cls'][sel] == cs[:, None], axis=1)
            key = f32(scores[q, cstar] * ctr[q])
            prod = f32(scores[q] * ctr[q][:, None]).max(1)
            bad = ~_bits_equal(key, prod)
            if bad.any():
                j = _first(bad)
                _fail(what, 'scores', q0 + j, 'sigmoid(max logit) * ctr = %r is not the max over classes of the products '
                      '(%r): the device sigmoid is not monotone' % (float(key[j]), float(prod[j])))
            klo, khi = key_intervals(lv)
            kk = key.astype(np.float64)
            bad = ~((kk >= klo[sel]) & (kk <= khi[sel]))
            if bad.any():
                j = _first(bad)
                _fail(what, 'scores', q0 + j, 'ranking key %r outside its bound [%r, %r]' % (kk[j], klo[sel[j]], khi[sel[j]]))
            # output order: descending key, ties by ascending location, exactly
            if k > 1:
                a, b = kk[:-1], kk[1:]
                bad = (a < b) | ((a == b) & (sel[:-1] >= sel[1:]))
                if bad.any():
                    j = _first(bad)
                    _fail(what, 'loc', q0 + j + 1, '= %d (key %r) is listed after location %d (key %r): not in descending '
                          'key / ascending index order' % (loc[q0 + j + 1], b[j], loc[q0 + j], a[j]))
            # selection against the intervals of every location of the level
            hs, ls = np.sort(khi), np.sort(klo)
            maybe_above = hw - np.searchsorted(hs, klo, 'left') - 1        # others whose key may reach i's
            surely_above = hw - np.searchsorted(ls, khi, 'right')          # others whose key is surely above i's
            must_in, must_out = maybe_above < k, surely_above >= k
            chosen = np.zeros(hw, bool)
            chosen[sel] = True
            bad = must_in & ~chosen
            if bad.any():
                i = _first(bad)
                _fail(what, 'loc', loc0 + i, 'is certainly above the nms_pre cut of level %d but not selected' % l)
            bad = must_out & chosen
            if bad.any():
                i = _first(bad)
                j = int(np.flatnonzero(sel == i)[0])
                _fail(what, 'loc', q0 + j, '= %d is certainly below the nms_pre cut of level %d but selected' % (loc0 + i, l))
            n_amb += int((~must_in & ~must_out).sum())
        q0 += k
        loc0 += hw
    if q0 != loc.shape[0]:
        raise CheckError('%s: %d candidates written, the levels give %d' % (what, loc.shape[0], q0))
    if n_cut and n_amb > cap * n_cut:
        raise CheckError('%s: %d of %d locations of cut levels are ambiguous (cap %g)' % (what, n_amb, n_cut, cap))
    return dict(locations=n_loc, cut_locations=n_cut, ambiguous=n_amb)


# ---------------------------------------------------------------------------------------- NMS, teacher-forced
def _check_record(what, det, labels, idx, count, want_det, want_labels, want_idx):
    det, labels, idx = np.asarray(det, np.float32), np.asarray(labels), np.asarray(idx)
    k = int(np.asarray(count).reshape(-1)[0])
    n = want_det.shape[0]
    if k != n:
        raise CheckError('%s: count is %d, expected %d' % (what, k, n))
    expect_equal(what, 'labels', labels[:n].astype(np.int64), np.asarray(want_labels, np.int64))
    expect_equal(what, 'idx', idx[:n].astype(np.int64), np.asarray(want_idx, np.int64))
    expect_equal(what, 'det', det[:n], np.asarray(want_det, np.float32).reshape(n, 5))
    tail = det[n:]
    if (tail.view(np.uint32) != 0).any():
        j = _first((tail.view(np.uint32) != 0).any(1))
        _fail(what, 'det', n + j, 'past the count is %s, expected zeros' % tail[j].tolist())
    for field, v in (('labels', labels[n:]), ('idx', idx[n:])):
        if (v != -1).any():
            j = _first(v != -1)
            _fail(what, field, n + j, 'past the count is %d, expected -1' % v[j])
    return n


def _nms_fn(use_c):
    if use_c:
        from . import cbind
        return lambda d, thr, cmp_ge=False: cbind.nms(d, thr, int(cmp_ge))
    return None


def check_multiclass_nms(boxes, scores, ctr, n, score_thr, iou_thr, max_num, cmp_ge, det, labels, idx, count,
                         what='nms', use_c=False):
    """smb_multiclass_nms over the first n candidates against oracle.ops.multiclass_nms_idx on the same buffers."""
    import torch
    from . import ops as O
    b = torch.from_numpy(np.ascontiguousarray(boxes[:n], np.float32))
    s = np.ascontiguousarray(scores[:n], np.float32)
    bg = torch.from_numpy(np.concatenate([np.zeros((n, 1), np.float32), s], 1))
    rb, rl, ri = O.multiclass_nms_idx(b, bg, float(np.float32(score_thr)), float(np.float32(iou_thr)), max_num,
                                      score_factors=torch.from_numpy(np.ascontiguousarray(ctr[:n], np.float32)),
                                      cmp_ge=cmp_ge, nms_fn=_nms_fn(use_c))
    return _check_record(what, det, labels, idx, count, rb.numpy(), rl.numpy(), ri.numpy())


def check_fast_nms(boxes, scores, ctr, n, score_thr, iou_thr, top_k, max_num, det, labels, idx, count, what='nms'):
    """smb_fast_nms against oracle.ops.fast_nms on the same buffers (scores multiplied by ctr in float32 first)."""
    import torch
    from . import ops as O
    b = torch.from_numpy(np.ascontiguousarray(boxes[:n], np.float32))
    s = torch.from_numpy(f32(np.asarray(scores[:n], np.float32) * np.asarray(ctr[:n], np.float32)[:, None]).T.copy())
    rd, rl, _, ri = O.fast_nms(b, s, torch.zeros(n, 1), float(np.float32(iou_thr)), top_k, float(np.float32(score_thr)),
                               max_num)
    return _check_record(what, det, labels, idx, count, rd.numpy(), rl.numpy(), ri.numpy())


def check_ml_nms(boxes, scores, labels_in, n_cand, iou_thr, max_per_img, out_cap, det, labels, idx, count, kept_total,
                 what='nms'):
    """smb_ml_nms_topk against oracle.benchmark.ml_nms + kth_value_cut on the same candidate buffers."""
    from . import benchmark as B
    n = int(np.asarray(n_cand).reshape(-1)[0])
    b, s = np.asarray(boxes[:n], np.float32), np.asarray(scores[:n], np.float32)
    lab = np.asarray(labels_in[:n]).astype(np.int64)
    keep = B.kth_value_cut(s, B.ml_nms(b, s, lab, float(np.float32(iou_thr))), max_per_img)
    kt = int(np.asarray(kept_total).reshape(-1)[0])
    if kt != keep.shape[0]:
        raise CheckError('%s: kept_total is %d, expected %d' % (what, kt, keep.shape[0]))
    keep = keep[:out_cap]
    want = np.concatenate([b[keep], s[keep, None]], 1).astype(np.float32)
    return _check_record(what, det, labels, idx, count, want, lab[keep], keep)


# ------------------------------------------------------------------------------------------------ BM pair decode
def pair_reference(levels, C, score_thr, nms_pre, geom):
    """smb_pair_decode_topk's candidates (boxes, scores, labels, loc): pairs with sigmoid_rn(cls) > thr, per level the
    nms_pre largest sigmoid_rn(cls) * sigmoid_rn(ctr) (ties: lower pair index) listed by ascending pair index; box from
    relu(d * box_scale) * box_mul clipped to the image, score sqrt of the product.  sigmoid_rn is exactly
    oracle.benchmark.sigmoid_rn."""
    from .benchmark import sigmoid_rn
    out_b, out_s, out_l, out_loc, off = [], [], [], [], 0
    thr = np.float32(score_thr)
    for lv in levels:
        hw = lv['h'] * lv['w']
        sc = sigmoid_rn(lv['cls'])
        st = sigmoid_rn(lv['ctr'])
        prod = f32(sc * st[:, None]).reshape(-1)
        pairs = np.flatnonzero((sc > thr).reshape(-1))
        if pairs.size > nms_pre:
            order = np.argsort(-prod[pairs].astype(np.float64), kind='stable')[:nms_pre]
            pairs = np.sort(pairs[order])
        loc, c = pairs // C, pairs % C
        out_b.append(decode_boxes(lv, loc, geom, divide=False))
        out_s.append(np.sqrt(prod[pairs]).astype(np.float32))
        out_l.append(c.astype(np.int64))
        out_loc.append((loc + off).astype(np.int64))
        off += hw
    return (np.concatenate(out_b).reshape(-1, 4), np.concatenate(out_s), np.concatenate(out_l), np.concatenate(out_loc))


def check_pair_decode(levels, C, score_thr, nms_pre, geom, boxes, scores, labels, loc, n_cand, what='decode_topk'):
    """smb_pair_decode_topk(_dev) outputs (every slot) against pair_reference: bit-exact, zero / -1 slots after."""
    rb, rs, rl, rloc = pair_reference(levels, C, score_thr, nms_pre, geom)
    n = rb.shape[0]
    got = int(np.asarray(n_cand).reshape(-1)[0])
    if got != n:
        raise CheckError('%s: n_cand is %d, expected %d' % (what, got, n))
    expect_equal(what, 'loc', np.asarray(loc[:n]).astype(np.int64), rloc)
    expect_equal(what, 'labels', np.asarray(labels[:n]).astype(np.int64), rl)
    expect_equal(what, 'boxes', np.asarray(boxes[:n], np.float32), rb)
    expect_equal(what, 'scores', np.asarray(scores[:n], np.float32), rs)
    m = np.asarray(loc).shape[0] - n
    expect_equal(what, 'boxes', np.asarray(boxes[n:], np.float32), np.zeros((m, 4), np.float32))
    expect_equal(what, 'scores', np.asarray(scores[n:], np.float32), np.zeros(m, np.float32))
    expect_equal(what, 'labels', np.asarray(labels[n:]).astype(np.int64), np.full(m, -1))
    expect_equal(what, 'loc', np.asarray(loc[n:]).astype(np.int64), np.full(m, -1))
    return n


# ------------------------------------------------------------------------------------------------------- gathers
def cof_row(loc, level_hw, n_img, img):
    """Row of the coefficient source of level-concatenated location `loc` of image `img`: the level-major,
    image-inside-level layout [level][image][hw_l] (LocMap in nms.cu); no level table: row = loc."""
    loc = np.asarray(loc, np.int64)
    if not level_hw:
        return loc
    off = np.concatenate([[0], np.cumsum(level_hw)]).astype(np.int64)
    l = np.searchsorted(off[1:], loc, 'right')
    hw = off[l + 1] - off[l]
    return off[l] * n_img + img * hw + (loc - off[l])


def check_gather_cofs(cof_src, cand_loc, idx, det, count, level_hw, n_img, img, det_cofs, det_boxes, loc_kept,
                      what='gather_cofs'):
    """smb_gather_det_inputs: det_cofs[r] = cof_src[row(cand_loc[idx[r]])], det_boxes[r] = det[r, :4], loc_kept[r] =
    cand_loc[idx[r]] for r < count; zeros / -1 after."""
    k = int(np.asarray(count).reshape(-1)[0])
    cof_src, det = np.asarray(cof_src, np.float32), np.asarray(det, np.float32)
    max_rows = np.asarray(det_cofs).shape[0]
    loc = np.asarray(cand_loc).astype(np.int64)[np.asarray(idx[:k]).astype(np.int64)]
    rows = cof_row(loc, level_hw, n_img, img)
    E = np.asarray(det_cofs).shape[1]
    want = np.zeros((max_rows, E), np.float32)
    want[:k] = cof_src[rows, :E]
    expect_equal(what, 'det_cofs', np.asarray(det_cofs, np.float32), want)
    wb = np.zeros((max_rows, 4), np.float32)
    wb[:k] = det[:k, :4]
    expect_equal(what, 'det_boxes', np.asarray(det_boxes, np.float32), wb)
    if loc_kept is not None:
        wl = np.full(max_rows, -1, np.int64)
        wl[:k] = loc
        expect_equal(what, 'loc_kept', np.asarray(loc_kept).astype(np.int64), wl)
    return k


def track_cells(det, sx, sy, stride, h, w):
    """gather_track_feats_kernel's map cell of each row: centre of det * (sx, sy) over the stride, floored, clamped."""
    det = np.asarray(det, np.float32)
    sx, sy, st, two = np.float32(sx), np.float32(sy), np.float32(stride), np.float32(2.0)
    x1, y1, x2, y2 = f32(det[:, 0] * sx), f32(det[:, 1] * sy), f32(det[:, 2] * sx), f32(det[:, 3] * sy)
    with np.errstate(invalid='ignore'):
        cx = np.floor(f32(f32(f32(x2 + x1) / two) / st)).astype(np.float64)
        cy = np.floor(f32(f32(f32(y2 + y1) / two) / st)).astype(np.float64)
    cx = np.clip(np.nan_to_num(cx, nan=0.0, posinf=w - 1, neginf=0), 0, w - 1).astype(np.int64)
    cy = np.clip(np.nan_to_num(cy, nan=0.0, posinf=h - 1, neginf=0), 0, h - 1).astype(np.int64)
    return cy, cx


def check_gather_track(track, det, count, sx, sy, stride, out, what='gather_track'):
    """smb_gather_track_feats(_dev): out[r] = track[cy, cx] for r < count (track [h, w, C]), zeros after."""
    track = np.asarray(track, np.float32)
    h, w, C = track.shape
    k = int(np.asarray(count).reshape(-1)[0])
    out = np.asarray(out, np.float32)
    cy, cx = track_cells(np.asarray(det)[:k], sx, sy, stride, h, w)
    want = np.zeros_like(out)
    want[:k] = track[cy, cx]
    expect_equal(what, 'out', out, want)
    return k


# ------------------------------------------------------------------------------------------- constructed inputs
def iou_f32(a, b, one):
    """iou_ref (one = 1, the MM / BM NMS) or jaccard_ref (one = 0, fast NMS) of float32 boxes [.., 4], in float32."""
    a, b, one = f32(a), f32(b), np.float32(one)
    z = np.float32(0)
    iw = np.maximum(f32(f32(np.minimum(a[..., 2], b[..., 2]) - np.maximum(a[..., 0], b[..., 0])) + one), z)
    ih = np.maximum(f32(f32(np.minimum(a[..., 3], b[..., 3]) - np.maximum(a[..., 1], b[..., 1])) + one), z)
    inter = f32(iw * ih)
    sa = f32(f32(f32(a[..., 2] - a[..., 0]) + one) * f32(f32(a[..., 3] - a[..., 1]) + one))
    sb = f32(f32(f32(b[..., 2] - b[..., 0]) + one) * f32(f32(b[..., 3] - b[..., 1]) + one))
    with np.errstate(invalid='ignore', divide='ignore'):
        return f32(inter / f32(f32(sa + sb) - inter))


def threshold_pairs(thr, one):
    """Three box pairs (a, b) whose float32 IoU (iou_f32 with `one`) is the float32 just below thr, thr itself, and just
    above: a [3, 4], b [3, 4].  a is 64 x 32 (with +one); b is a shifted right by about the width that gives thr, its
    left and right edges nudged independently in steps of 2^-19 until the quotient rounds to each target."""
    t = np.float32(thr)
    want = [np.nextafter(t, np.float32(0)), t, np.nextafter(t, np.float32(1))]
    W, H = np.float32(64.0), np.float32(32.0)
    a = f32([0.0, 0.0, W - np.float32(one), H - np.float32(one)])
    dx = float(W) * (1 - float(t)) / (1 + float(t))
    steps = np.arange(-256, 256, dtype=np.float64) * 2.0 ** -19
    x1 = f32(dx + steps)[:, None]
    x2 = f32(float(a[2]) + dx + steps)[None, :]
    x1, x2 = np.broadcast_arrays(x1, x2)
    b = np.stack([x1, np.zeros_like(x1), x2, np.full_like(x1, a[3])], -1).reshape(-1, 4)
    v = iou_f32(a[None], b, one)
    out_b = []
    for target in want:
        hit = np.flatnonzero(v == target)
        assert hit.size, 'no pair with IoU %r' % target
        out_b.append(b[hit[hit.size // 2]])
    return np.stack([a] * 3).astype(np.float32), np.stack(out_b).astype(np.float32)
