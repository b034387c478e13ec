"""Raw-image preprocessing at the edges of its size rules, on the host: the restatements of OpenCV's INTER_LINEAR
(oracle/preprocess.py: resize_linear_u8) and Pillow's BILINEAR (bm_transform_ref.resize_pil_bilinear_u8) against the
installed libraries over a systematic sweep of shapes, and a model of the PIL kernel's tile bounds that proves its
shared-memory and tap clamps never bind for a row raw_src_row(..., max_downscale=8) admits.

The sweeps are also the shapes tests/test_gpu_preprocess_edges.py runs through the device kernels (the pairs that fit
its canvases), so the host and device tests cover the same cases."""
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PREPROCESS_CU = os.path.join(ROOT, 'sipmask_b200', 'csrc', 'preprocess.cu')

# Pillow runs the vertical pass first for sources more than 100 times taller than wide whose height shrinks
TALL = [((2001, 20), (1300, 13)), ((1401, 14), (1300, 13)), ((1500, 14), (1285, 12)), ((3000, 20), (1350, 9)),
        ((10000, 12), (1344, 2))]


def pil_sweep():
    """{group: [((h, w), (dh, dw))]} for the PIL restatement against Pillow; every pair shrinks at most 8x per axis."""
    from sipmask_b200.serving import bm_resize_size
    g = {}
    bands = (1.01, 1.5, 2.0, 2.49, 3.0, 3.7, 4.0, 4.5, 5.0, 5.99, 6.0, 7.0, 7.5, 7.99, 8.0)
    g['shrink_bands'] = ([((int(round(o * s)), 37), (o, 41)) for o in (7, 30, 61) for s in bands] +
                         [((29, int(round(o * s))), (23, o)) for o in (7, 64, 126) for s in bands] +
                         [((8 * o, 8 * o - 3), (o, o)) for o in (1, 2, 16, 31, 32)] +
                         [((240, 1008), (30, 126))])         # the widest tile spans of the kernel (rows and columns)
    g['one_axis'] = [((61, 83), (61, 40)), ((61, 83), (30, 83)), ((700, 900), (300, 900)), ((600, 333), (600, 1000)),
                     ((17, 512), (17, 64)), ((512, 17), (64, 17)), ((201, 2), (100, 2)), ((5, 1), (5, 9))]
    g['upscale_thin'] = [((1, 1), (1, 2)), ((1, 1), (13, 7)), ((1, 1), (256, 256)), ((1, 9), (4, 300)),
                         ((1, 200), (3, 400)), ((9, 1), (300, 4)), ((200, 1), (400, 3)), ((1, 2048), (1, 1333))]
    g['wide'] = [((20, 2001), (13, 1300)), ((14, 1401), (13, 1300)), ((3, 400), (2, 300)), ((20, 3000), (9, 1350)),
                 ((2, 201), (1, 100))]
    # the benchmark rule around its max-size switch (long / short = 1333 / 800) and around Pillow's 100:1 threshold,
    # with the height shrinking and growing
    near = [(480, 799), (480, 800), (480, 801), (600, 999), (600, 1000), (600, 1001), (799, 480), (800, 480),
            (801, 480), (1333, 800), (1334, 800), (2000, 20), (2001, 20), (2100, 21), (2101, 21), (1400, 14),
            (1401, 14), (1399, 14), (1501, 15), (1500, 15), (300, 3), (301, 3), (200, 2), (201, 2), (101, 1),
            (100, 1), (1001, 10), (1000, 10), (3000, 20)]
    g['bm_rule'] = [((h, w), bm_resize_size(h, w)) for h, w in near]
    g['tall'] = TALL + [((2000, 20), (1300, 13)), ((2001, 20), (1999, 19)), ((1001, 10), (1000, 9)),
                        ((1001, 10), (1000, 10)), ((1001, 10), (500, 30)), ((301, 3), (1304, 13)),
                        ((300, 3), (1300, 13)), ((2001, 20), (2002, 20)), ((2001, 20), (2500, 13))]
    rs = np.random.RandomState(11)
    rnd = []
    for _ in range(200):
        h, w = (int(v) for v in rs.randint(1, 257, 2))
        rnd.append(((h, w), (int(rs.randint(-(-h // 8), 2 * h + 2)), int(rs.randint(-(-w // 8), 2 * w + 2)))))
    g['random'] = rnd
    return g


def cv2_sweep():
    """{group: [((h, w), (dh, dw))]} for the cv2 restatement against OpenCV."""
    from oracle.preprocess import rescale_size
    g = {}
    extreme = [(2048, 9), (9, 2048), (1, 1), (1, 2048), (2048, 1), (2, 3), (5, 1999), (1999, 5), (100, 3000),
               (3000, 100), (1, 7), (7, 1), (800, 1333), (1333, 800)]
    g['rescale'] = [((h, w), rescale_size(h, w, scale)[:2]) for scale in ((1333, 800), (544, 544)) for h, w in extreme]
    g['rescale'] = [p for p in g['rescale'] if min(p[1]) > 0]      # 1x2048 at 544: rounds to 0 rows, nothing to resize
    g['integer_shrink'] = [((2 * h, 2 * w), (h, w)) for h, w in ((240, 320), (1, 1), (3, 5), (17, 9))] + \
                          [((4 * h, 4 * w), (h, w)) for h, w in ((120, 160), (1, 1), (3, 5), (17, 9))] + \
                          [((4 * 75, 2 * 50), (75, 50)), ((2 * 75, 4 * 50), (75, 50))]
    g['one_axis'] = [((61, 83), (61, 40)), ((61, 83), (30, 83)), ((480, 640), (480, 1066)), ((480, 640), (800, 640)),
                     ((9, 2048), (9, 1333)), ((2048, 9), (1333, 9))]
    g['one_pixel'] = [((1, 1), (5, 7)), ((1, 9), (4, 3)), ((9, 1), (2, 6)), ((1, 1), (1, 1)), ((1, 5), (1, 1)),
                      ((5, 1), (1, 1)), ((7, 5), (1, 1))]
    return g


def _flat(sweep):
    return [(name, p) for name, pairs in sweep.items() for p in pairs]


def _img(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3), dtype=np.uint8)


def test_pil_sweep_is_what_it_claims():
    from sipmask_b200.conv import PIL_MAX_DOWNSCALE
    import bm_transform_ref as P
    flat = _flat(pil_sweep())
    assert len(flat) > 300
    for _, ((h, w), (dh, dw)) in flat:
        assert h <= PIL_MAX_DOWNSCALE * dh and w <= PIL_MAX_DOWNSCALE * dw, ((h, w), (dh, dw))
    # the 100:1 threshold is met from both sides, shrinking and growing; wide images never take the branch
    tall = [p for _, p in flat if P.pil_height_first(p[0][0], p[0][1], p[1][0])]
    assert len(tall) >= 10
    assert any(h == 100 * w + 1 for (h, w), _ in tall)
    assert any(h == 100 * w and dh < h for _, ((h, w), (dh, _dw)) in flat)
    assert any(h > 100 * w and dh > h for _, ((h, w), (dh, _dw)) in flat)
    assert not any(P.pil_height_first(h, w, dh) for (h, w), (dh, _dw) in pil_sweep()['wide'])


@pytest.mark.parametrize('group', ['shrink_bands', 'one_axis', 'upscale_thin', 'wide', 'bm_rule', 'tall', 'random'])
def test_pil_restatement_sweep_equals_pillow(group):
    Image = pytest.importorskip('PIL.Image')
    import bm_transform_ref as P
    for i, ((h, w), (dh, dw)) in enumerate(pil_sweep()[group]):
        src = _img(h, w, 1000 + i)
        want = np.asarray(Image.fromarray(src, 'RGB').resize((dw, dh), Image.BILINEAR))
        got = P.resize_pil_bilinear_u8(src, dh, dw)
        assert got.shape == want.shape and np.array_equal(got, want), ((h, w), (dh, dw), int((got != want).sum()))


@pytest.mark.parametrize('group', ['rescale', 'integer_shrink', 'one_axis', 'one_pixel'])
def test_cv2_restatement_sweep_equals_cv2(group):
    cv2 = pytest.importorskip('cv2')
    from oracle.preprocess import resize_linear_u8
    for i, ((h, w), (dh, dw)) in enumerate(cv2_sweep()[group]):
        src = _img(h, w, 2000 + i)
        want = cv2.resize(src, (dw, dh), interpolation=cv2.INTER_LINEAR)
        if want.ndim == 2:                       # cv2 drops a channel axis it never had; never for 3 channels
            want = want[:, :, None]
        assert np.array_equal(resize_linear_u8(src, dh, dw), want), ((h, w), (dh, dw))


# ------------------------------------------------------------------------------------------------ PIL kernel tile bounds
def kernel_constants():
    """PIL_* constexpr ints of preprocess.cu, evaluated in order, so the model follows the source."""
    env = {}
    for line in open(PREPROCESS_CU):
        m = re.match(r'\s*constexpr int (.*?);', line)
        if not m:
            continue
        for decl in m.group(1).split(','):
            name, expr = (s.strip() for s in decl.split('=', 1))
            expr = re.sub(r'^(.+)\?(.+):(.+)$', r'(\2) if (\1) else (\3)', expr)      # c ? a : b
            env[name] = int(eval(expr, {}, dict(env)))
    return env


def _tile_spans(ins, out, tile):
    """For axes ins[i] -> out: the most taps of any output index and the most source indices any kernel tile of `tile`
    outputs reads.  Tiles start at output 2 * T0 - 3 (T0 a multiple of tile / 2, the halo of the stem's space-to-depth
    layout); the kernel reads source [lo[first], lo[last] + cnt[last]) of a tile's first and last output inside the image,
    which holds every tap of the tile because the first tap and the end are nondecreasing in the output index."""
    import bm_transform_ref as P
    lo, cnt, _, _, _ = P._pil_bounds(np.asarray(ins, np.int64)[:, None], out)
    end = lo + cnt
    assert (np.diff(lo, axis=1) >= 0).all() and (np.diff(end, axis=1) >= 0).all()
    p0 = np.arange(-3, out, tile)
    first, last = np.maximum(p0, 0), np.minimum(p0 + tile, out) - 1
    return cnt.max(1), (end[:, last] - lo[:, first]).max(1)


# the PIL kernel's edge launch in tests/test_gpu_preprocess_edges.py (a 1408 x 1408 canvas): exact 8x on both axes, the
# widest tile spans, 8x on one axis with an upscale on the other, one axis unchanged, the tall images Pillow resizes
# vertically first next to 2000x20 (h = 100 w), resizes to the full canvas height, a wide image
PIL_EDGES = [((2048, 1024), (256, 128)), ((240, 1008), (30, 126)), ((2048, 100), (256, 300)), ((100, 2048), (300, 256)),
             ((700, 900), (300, 900)), ((600, 333), (600, 1000)), ((2001, 20), (1300, 13)), ((1401, 14), (1300, 13)),
             ((1500, 14), (1285, 12)), ((2000, 20), (1300, 13)), ((10000, 12), (1408, 2)), ((704, 200), (1408, 400)),
             ((20, 2001), (13, 1300))]


def gpu_pil_pairs():
    """Every PIL (in, out) pair the device tests run."""
    return [p for _, p in _flat(pil_sweep())] + PIL_EDGES


def test_pil_kernel_tile_bounds_model():
    """Every (in, out) with 1 <= out <= 256 and out <= in <= 8 * out, plus the device tests' pairs: no output index has
    more than PIL_KMAX taps, the width-first tile's source rows fit PIL_RMAX and the height-first tile's source columns
    PIL_CMAX, so the kernel's min(..., PIL_KMAX) / PIL_RMAX / PIL_CMAX clamps never bind."""
    import bm_transform_ref as P
    k = kernel_constants()
    ty, tx, s = k['PIL_TY'], k['PIL_TX'], k['PIL_MAX_SCALE']
    assert (2 * ty, 2 * tx) == (k['PIL_OY'], k['PIL_OX'])
    from sipmask_b200.conv import PIL_MAX_DOWNSCALE
    assert s == PIL_MAX_DOWNSCALE
    worst = {'taps': (0, None), 'rows': (0, None), 'cols': (0, None)}

    def take(key, vals, ins, out):
        i = int(np.argmax(vals))
        if vals[i] > worst[key][0]:
            worst[key] = (int(vals[i]), (int(ins[i]), out))

    for out in range(1, 257):
        ins = np.arange(1, s * out + 1)
        taps, rows = _tile_spans(ins, out, 2 * ty)
        _, cols = _tile_spans(ins, out, 2 * tx)
        take('taps', taps, ins, out)
        take('rows', rows, ins, out)
        take('cols', cols, ins, out)
    axes = {(h, dh) for (h, _), (dh, _) in gpu_pil_pairs()} | {(w, dw) for (_, w), (_, dw) in gpu_pil_pairs()}
    for n_in, out in sorted(axes):
        taps, rows = _tile_spans([n_in], out, 2 * ty)
        _, cols = _tile_spans([n_in], out, 2 * tx)
        take('taps', taps, [n_in], out)
        take('rows', rows, [n_in], out)
        take('cols', cols, [n_in], out)
        # the device's tap count is the restatement's (the kernel computes the same bounds in the same arithmetic)
        assert (P._pil_taps(n_in, out)[1] == P._pil_bounds(n_in, out)[1]).all()
    print('largest tap count %d at %s, tile source rows %d at %s, tile source columns %d at %s'
          % (worst['taps'] + worst['rows'] + worst['cols']))
    assert worst['taps'][0] <= k['PIL_KMAX'], (worst['taps'], k['PIL_KMAX'])
    assert worst['rows'][0] <= k['PIL_RMAX'], (worst['rows'], k['PIL_RMAX'])
    assert worst['cols'][0] <= k['PIL_CMAX'], (worst['cols'], k['PIL_CMAX'])
    # the buffer the kernel sizes holds either intermediate image
    assert k['PIL_PASS_BYTES'] >= max(k['PIL_RMAX'] * k['PIL_OX'], k['PIL_OY'] * k['PIL_CMAX']) * 3
    # and the spans are reached: an exact 8x shrink fills a whole tile
    assert worst['rows'][0] == (2 * ty - 1) * s + 2 * s and worst['cols'][0] == (2 * tx - 1) * s + 2 * s
