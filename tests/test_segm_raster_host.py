"""CPU checks of the device rasterizer's host side: the packing of segmentations (pools, item ranges, the four input
kinds, every validation error segm_plane raises, with its type and message), and the parity claim the kernels rest on,
in numpy: rleFrPoly's boundary positions left unsorted, toggled and filled by a cumulative XOR equal the plane
segm_plane fills."""
import numpy as np
import pytest

from test_cocoeval_host import random_polys

INT_MIN = -2 ** 31


def plane_bits(plane, w):
    return np.unpackbits(np.ascontiguousarray(plane).view(np.uint8), axis=-1, bitorder='little')[:, :w].astype(bool)


def seeded_polys(seed, n, h, w, kmin=3, kmax=200):
    """Random rings of kmin..kmax vertices around a centre inside or near the canvas, some far outside it."""
    rng = np.random.default_rng(seed)
    out = []
    for i in range(n):
        k = int(rng.integers(kmin, kmax + 1))
        cx, cy = rng.uniform(-0.1 * w, 1.1 * w), rng.uniform(-0.1 * h, 1.1 * h)
        ang = np.sort(rng.uniform(0, 2 * np.pi, k))
        rad = rng.uniform(0.05, 0.6) * min(h, w) * rng.uniform(0.5, 1.5, k)
        xy = np.stack([cx + rad * np.cos(ang), cy + rad * np.sin(ang)], 1)
        if i % 3 == 0:
            xy = np.round(xy * 2) / 2                         # integer and half-pixel vertices
        out.append(xy.reshape(-1).tolist())
    return out


def hard_cases():
    """(name, segmentation, h, w): one plane each."""
    c = []
    c.append(('outside_every_side', [[-20, -10, 70, -15, 80, 60, -5, 55]], 37, 45))
    c.append(('half_pixel', [[2.5, 3.5, 20.5, 3.5, 20.5, 15.5, 2.5, 15.5]], 37, 45))
    c.append(('integer', [[2, 3, 20, 3, 20, 15, 2, 15]], 37, 45))
    c.append(('repeated_vertex', [[3, 3, 3, 3, 20, 3, 20, 3, 20, 15, 3, 15]], 37, 45))
    c.append(('horizontal_vertical', [[5, 5, 30, 5, 30, 5.2, 30, 30, 5, 30]], 37, 45))
    c.append(('zero_area', [[4, 4, 30, 20, 4, 4, 30, 20]], 37, 45))
    c.append(('two_and_a_half_vertices', [[4, 4, 30, 20, 9]], 37, 45))
    c.append(('y_clamped_to_h', [[3, 30, 20, 50, 40, 30, 40, 80, 3, 80]], 37, 45))
    c.append(('last_column', [[40, 2, 44.9, 2, 45, 30, 44, 36.9, 40, 30]], 37, 45))
    c.append(('beyond_last_column', [[40, 2, 60, 2, 60, 30, 40, 30]], 37, 45))
    c.append(('self_intersecting', [[0, 0, 30, 30, 30, 0, 0, 30]], 37, 45))
    c.append(('merged_overlapping', [[2, 2, 25, 2, 25, 25, 2, 25], [10, 10, 40, 12, 38, 33, 12, 30], [0, 0, 44, 36, 0, 36]],
              37, 45))
    c.append(('boxes', [[2.5, 3.2, 10, 12], [20, 5, 7.7, 30]], 40, 50))
    c.append(('full_box', [[0, 0, 49.9, 39.9]], 40, 50))
    c.append(('w_64', [[1, 1, 63, 2, 60, 30, 2, 31]], 33, 64))
    c.append(('h_32', [[1, 1, 40, 2, 44, 31, 2, 30]], 32, 45))
    c.append(('h_over_1024', [[1, 1, 18, 500, 10, 1099, 2, 800]], 1100, 20))
    c.append(('canvas_1x1', [[0, 0, 1, 0, 1, 1, 0, 1]], 1, 1))
    c.append(('canvas_1xw', [[3, 0, 30, 0, 30, 1, 3, 1]], 1, 45))
    c.append(('canvas_hx1', [[0, 3, 1, 3, 1, 30, 0, 30]], 37, 1))
    return c


# ---------------------------------------------------------------------------------------------------- the parity claim
def _scaled(v):
    return int(np.float64(5.0) * np.float64(v) + .5)         # C's (int): truncation


def boundaries_unsorted(p, h, w):
    """rleFrPoly's boundary positions of polygon p in generation order: every point against the point before it, edge by
    edge, each point from its (edge, offset) alone.  No sort, no differences, no merging of zero-length runs."""
    xy = np.asarray(p, np.float64)[:len(p) // 2 * 2]
    k = xy.size // 2
    x = [_scaled(xy[2 * j]) for j in range(k)]
    y = [_scaled(xy[2 * j + 1]) for j in range(k)]

    def point(j, d):
        xs, ys, xe, ye = x[j], y[j], x[(j + 1) % k], y[(j + 1) % k]
        dx, dy = abs(xe - xs), abs(ys - ye)
        flip = (dx >= dy and xs > xe) or (dx < dy and ys > ye)
        if flip:
            xs, xe, ys, ye = xe, xs, ye, ys
        if dx == 0 and dy == 0:
            return xs, INT_MIN
        t = max(dx, dy) - d if flip else d
        if dx >= dy:
            s = np.float64(ye - ys) / np.float64(dx)
            return t + xs, int(np.float64(ys) + s * np.float64(t) + .5)
        s = np.float64(xe - xs) / np.float64(dy)
        return int(np.float64(xs) + s * np.float64(t) + .5), t + ys

    def length(j):
        return max(abs(x[(j + 1) % k] - x[j]), abs(y[(j + 1) % k] - y[j]))

    out = []
    for j in range(k):
        for d in range(length(j) + 1):
            if j == 0 and d == 0:
                continue
            u0, v0 = point(j, d - 1) if d > 0 else point(j - 1, length(j - 1))
            u1, v1 = point(j, d)
            if u1 == u0:
                continue
            xd = np.float64(u1 if u1 < u0 else u1 - 1)
            xd = (xd + .5) / 5.0 - .5
            if np.floor(xd) != xd or xd < 0 or xd > w - 1:
                continue
            yd = np.float64(min(v1, v0))
            yd = (yd + .5) / 5.0 - .5
            yd = np.ceil(min(max(yd, 0.0), float(h)))
            out.append(int(xd) * h + int(yd))
    return out


def fill_by_parity(positions, h, w):
    """Toggle one bit per position (positions at h * w fall off the canvas) and take the cumulative XOR in column-major
    order: the mask [h, w]."""
    t = np.zeros(h * w + 1, np.int64)
    np.add.at(t, np.asarray(positions, np.int64), 1)
    return (np.cumsum(t[:h * w]) & 1).astype(bool).reshape(w, h).T


def runs_by_parity(counts, h, w):
    pos = np.cumsum(np.asarray(counts, np.int64))
    return fill_by_parity(pos[pos <= h * w], h, w)


def test_parity_of_unsorted_boundaries_equals_segm_plane():
    from sipmask_b200 import cocoeval as C
    cases = [(str(i), [p], 37, 45) for i, p in enumerate(random_polys(0, h=37, w=45))]
    cases += [('ring%d' % i, [p], 60, 83) for i, p in enumerate(seeded_polys(5, 12, 60, 83, kmax=40))]
    cases += [c for c in hard_cases() if c[2] * c[3] <= 4000 and len(c[1][0]) != 4]
    for name, segm, h, w in cases:
        got = np.zeros((h, w), bool)
        for p in segm:                                         # merge: the union of the polygons' fills
            got |= fill_by_parity(boundaries_unsorted(p, h, w), h, w)
        assert np.array_equal(got, plane_bits(C.segm_plane(segm, h, w), w)), name


def test_parity_of_run_lengths_equals_segm_plane():
    from sipmask_b200 import cocoeval as C
    h, w = 7, 9
    for counts in ([63], [0, 63], [5, 0, 0, 10, 48], [0, 3, 0, 0, 4, 56], [10, 5, 0, 5, 43], [62, 1], [3, 4, 56, 0]):
        got = runs_by_parity(counts, h, w)
        assert np.array_equal(got, plane_bits(C.segm_plane({'size': [h, w], 'counts': counts}, h, w), w)), counts


# ---------------------------------------------------------------------------------------------------- packing
def test_pack_pools_and_item_ranges():
    from sipmask_b200 import rle, segm_raster as SR
    h, w = 20, 30
    m = np.zeros((h, w), bool)
    m[3:9, 4:20] = True
    c = rle.counts(m)
    pack = SR.SegmPack()
    pack.add([[1, 2, 9, 2, 9, 8, 1, 8.5, 77], [3, 3, 5, 3, 5, 5]], h, w, 0)         # two polygons (one with an odd tail)
    pack.add([[2.5, 3, 10, 12], [1, 1, 2, 2]], h, w, 1)                              # a first element of 4: boxes
    pack.add({'size': [h, w], 'counts': [int(v) for v in c]}, h, w, 2)               # uncompressed
    pack.add({'size': [h, w], 'counts': rle.to_string(c).decode()}, h, w, 3)         # compressed str
    pack.add({'size': [h, w], 'counts': rle.to_string(c)}, 20, 30, 4)                # compressed bytes
    items, xy, counts = pack.arrays()
    assert items.dtype == SR.ITEM_DTYPE and items['kind'].tolist() == [0, 0, 0, 0, 1, 1, 1]
    assert items['plane'].tolist() == [0, 0, 1, 1, 2, 3, 4]
    assert items['off'].tolist() == [0, 4, 7, 11, 0, len(c), 2 * len(c)]
    assert items['n'].tolist() == [4, 3, 4, 4, len(c), len(c), len(c)]
    assert (items['h'] == h).all() and (items['w'] == w).all()
    assert xy.dtype == np.float64 and xy.size == 2 * pack.n_xy == 30
    assert xy[:8].tolist() == [1, 2, 9, 2, 9, 8, 1, 8.5]
    assert xy[14:22].tolist() == [2.5, 3, 2.5, 15, 12.5, 15, 12.5, 3]                # frBbox's four vertices
    assert counts.dtype == np.uint32 and counts.tolist() == c.tolist() * 3
    assert (pack.max_hw, pack.max_w) == (h * w, w)
    empty = SR.SegmPack().arrays()
    assert [a.size for a in empty] == [0, 0, 0]


BAD = [
    ([[1, 2]], 'input type is not supported'),
    ([], 'polygon list needs lists'),
    ([3, 4, 5, 6, 7, 8], 'polygon list needs lists'),
    ([[1, 2, 3, 4], [1, 2, 3]], 'boxes must have 4 numbers'),
    ({'size': [4, 4], 'counts': [3, 20]}, 'do not cover'),
    ({'size': [4, 4], 'counts': [3, 12]}, 'do not cover'),
    ({'size': [4, 4], 'counts': [20, -4]}, 'non-negative'),
    ({'size': [4, 4], 'counts': [[16]]}, 'non-negative'),
    ({'size': [4, 5], 'counts': [20]}, 'differs from the image canvas'),
    ({'size': [4, 4], 'counts': '0#'}, 'malformed RLE string'),
    ({'size': [4, 4], 'counts': 'o'}, 'malformed RLE string'),
    ({'size': [4, 4], 'counts': 3.5}, 'counts must be a list or a string'),
    ({'counts': 'abc'}, 'not a polygon list or an RLE dict'),
    ('abc', 'not a polygon list or an RLE dict'),
]


@pytest.mark.parametrize('segm,match', BAD, ids=[str(i) for i in range(len(BAD))])
def test_pack_raises_what_segm_plane_raises(segm, match):
    from sipmask_b200 import cocoeval as C, segm_raster as SR
    with pytest.raises(ValueError, match=match) as host:
        C.segm_plane(segm, 4, 4, 'annotation 7')
    with pytest.raises(ValueError) as packed:
        SR.SegmPack().add(segm, 4, 4, 0, 'annotation 7')
    assert str(packed.value) == str(host.value)


def test_pack_bounds_coordinates():
    from sipmask_b200 import segm_raster as SR
    for v in (float('nan'), float('inf'), 1e9, -1.1e8):
        with pytest.raises(ValueError, match='coordinates'):
            SR.SegmPack().add([[1, 2, 3, 4, v, 6]], 10, 10, 0)
    SR.SegmPack().add([[1, 2, 3, 4, 1e8, -1e8]], 10, 10, 0)
    with pytest.raises(ValueError, match='canvas'):
        SR.SegmPack().add([[1, 2, 3, 4, 5, 6]], 65536, 32768, 0)


def test_ground_truth_packed_forms():
    """CocoGroundTruth.packed / YtvisGroundTruth.packed_frame: image()'s / frame()'s rows in the same order, masks as
    items, and their errors at the same call."""
    from sipmask_b200 import cocoeval as C, ytviseval as Y
    ann = dict(images=[dict(id=3, height=30, width=40)], categories=[dict(id=2), dict(id=1)], annotations=[
        dict(id=1, image_id=3, category_id=2, bbox=[1, 1, 5, 5], area=25, iscrowd=0, segmentation=[[1, 1, 6, 1, 6, 6, 1, 6]]),
        dict(id=2, image_id=3, category_id=1, bbox=[2, 2, 8, 8], area=64, iscrowd=1,
             segmentation={'size': [30, 40], 'counts': [100, 50, 1050]}),
        dict(id=3, image_id=3, category_id=2, bbox=[0, 0, 9, 9], area=81, iscrowd=0,
             segmentation=[[0, 0, 9, 0, 9, 9], [3, 3, 20, 3, 20, 20]])])
    g = C.CocoGroundTruth(ann)
    rows, off, planes = g.image(3)
    prow, poff, pack = g.packed(3)
    assert poff.tolist() == off.tolist() and prow['id'].tolist() == rows['id'].tolist() == [2, 1, 3]
    assert (prow['area_mask'] == 0).all() and (prow['ext'] == 0).all()
    items, xy, counts = pack.arrays()
    assert items['plane'].tolist() == [0, 1, 2, 2] and items['kind'].tolist() == [1, 0, 0, 0]
    bad = dict(ann, annotations=ann['annotations'] + [dict(ann['annotations'][0], id=9, segmentation=[[1, 2]])])
    gb = C.CocoGroundTruth(bad)                                # the constructor does not look at segmentations
    with pytest.raises(ValueError) as a:
        gb.image(3)
    with pytest.raises(ValueError) as b:
        gb.packed(3)
    assert str(a.value) == str(b.value) and 'annotation 9' in str(a.value)
    nos = C.CocoGroundTruth(dict(ann, annotations=[{k: v for k, v in ann['annotations'][0].items() if k != 'segmentation'}]))
    with pytest.raises(ValueError, match='has no segmentation'):
        nos.packed(3)

    vann = dict(videos=[dict(id=5, height=30, width=40, length=2)], categories=[dict(id=1)], annotations=[
        dict(id=1, video_id=5, category_id=1, segmentations=[None, [[1, 1, 6, 1, 6, 6]]], areas=[None, 12]),
        dict(id=2, video_id=5, category_id=1, segmentations=[{'size': [30, 40], 'counts': [7, 3, 1190]},
                                                             {'size': [30, 41], 'counts': [1230]}], areas=[3, 0])])
    yg = Y.YtvisGroundTruth(vann)
    rows, planes, areas = yg.frame(5, 0)
    prow, pack = yg.packed_frame(5, 0)
    assert prow['g'].tolist() == rows['g'].tolist() == [1] and pack.arrays()[2].tolist() == [7, 3, 1190]
    with pytest.raises(ValueError) as a:
        yg.frame(5, 1)
    with pytest.raises(ValueError) as b:
        yg.packed_frame(5, 1)
    assert str(a.value) == str(b.value) and 'annotation 2 frame 1' in str(a.value)
