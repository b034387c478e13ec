"""Host side of SipMask-benchmark raw-image serving: the benchmark's test size rule and PIL bilinear resize restated
(serving.bm_resize_size; bm_transform_ref.resize_pil_bilinear_u8 / bm_preprocess) against data the reference's own
transforms produced (tests/golden/ref_bm_transforms.npz) and against the installed Pillow, and the rejections
StreamRunner(benchmark=True, raw=True) / forward_raw(pipeline='benchmark') make before anything is enqueued."""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_bm_transforms.npz')
MEAN = (102.9801, 115.9465, 122.7717)


def test_size_rule_equals_the_reference():
    import bm_transform_ref as P
    from sipmask_b200.serving import bm_resize_size
    d = np.load(GOLDEN)
    src, want = d['sizes_src'], d['sizes_out']
    assert len(src) > 400
    for (h, w), (oh, ow) in zip(src.tolist(), want.tolist()):
        assert bm_resize_size(h, w) == (oh, ow), (h, w)
        assert P.bm_resize_size(h, w) == (oh, ow), (h, w)
    # the long side is not bounded: extreme aspect ratios keep their size
    assert bm_resize_size(56, 1345) == (56, 1345) and bm_resize_size(1, 2048) == (1, 2048)


def test_bm_preprocess_equals_the_reference_transform():
    import bm_transform_ref as P
    d = np.load(GOLDEN)
    for i in range(int(d['count'])):
        img, want, (oh, ow), rule = d['img_%d' % i], d['out_%d' % i], d['size_%d' % i].tolist(), d['rule_%d' % i].tolist()
        assert want.shape == (3, oh, ow)
        if rule == [0, 0]:        # an explicit one-axis resize: the resize and the normalisation without the size rule
            assert oh == img.shape[0] and ow != img.shape[1]
            x = P.resize_pil_bilinear_u8(img, oh, ow)[:, :, ::-1].astype(np.float32) - np.asarray(MEAN, np.float32)
            assert torch.equal(torch.from_numpy(np.ascontiguousarray(x.transpose(2, 0, 1))), torch.from_numpy(want)), i
            continue
        x = P.bm_preprocess(img, *rule)
        assert x.dtype == torch.float32 and x.shape[:2] == (1, 3)
        assert x.shape[2] == -(-oh // 32) * 32 and x.shape[3] == -(-ow // 32) * 32
        assert torch.equal(x[0, :, :oh, :ow], torch.from_numpy(want)), i
        assert (x[0, :, oh:] == 0).all() and (x[0, :, :, ow:] == 0).all()


def _pil_pairs():
    """(h, w) -> (dh, dw): 1-pixel sources, odd sizes, upscale x20, downscale to 8x, one axis only."""
    pairs = [((1, 1), (5, 7)), ((1, 9), (4, 3)), ((9, 1), (2, 6)), ((7, 5), (140, 100)), ((3, 4), (60, 80)),
             ((480, 640), (800, 1066)), ((1080, 1920), (750, 1333)), ((2048, 1536), (1066, 800)), ((333, 17), (800, 40)),
             ((64, 64), (8, 8)), ((65, 63), (9, 8)), ((800, 96), (100, 12)), ((100, 37), (100, 11)), ((37, 100), (11, 100)),
             ((61, 83), (61, 40)), ((61, 83), (30, 83)), ((17, 23), (340, 460)), ((513, 257), (97, 301)),
             ((99, 101), (13, 13)), ((56, 1345), (56, 1345)), ((640, 427), (1199, 800)), ((31, 29), (31, 29)),
             # more than 100x taller than wide: Pillow runs the vertical pass first when the height shrinks (h = 100 w
             # + 1), not at h = 100 w, and not when the height grows
             ((2001, 20), (1300, 13)), ((1401, 14), (1300, 13)), ((1500, 14), (1285, 12)), ((3000, 20), (1350, 9)),
             ((2000, 20), (1300, 13)), ((1001, 10), (1000, 9)), ((1000, 10), (999, 9)), ((301, 3), (1304, 13)),
             ((300, 3), (1300, 13)), ((2001, 20), (2500, 13))]
    rs = np.random.RandomState(7)
    for _ in range(6):
        h, w = rs.randint(1, 300, 2)
        pairs.append(((int(h), int(w)), (int(rs.randint(max(1, -(-h // 8)), 400)), int(rs.randint(max(1, -(-w // 8)), 400)))))
    return pairs


def test_pil_resize_restatement_equals_pillow():
    Image = pytest.importorskip('PIL.Image')
    import bm_transform_ref as P
    pairs = _pil_pairs()
    assert len(pairs) >= 20
    rs = np.random.RandomState(3)
    for (h, w), (dh, dw) in pairs:
        src = rs.randint(0, 256, (h, w, 3), dtype=np.uint8)
        want = np.asarray(Image.fromarray(src, 'RGB').resize((dw, dh), Image.BILINEAR))
        assert np.array_equal(P.resize_pil_bilinear_u8(src, dh, dw), want), ((h, w), (dh, dw))


def _bm_runner(**kw):
    """A benchmark=True, raw=True StreamRunner's host state (validation only; the device is never touched)."""
    from sipmask_b200.serving import StreamRunner
    r = StreamRunner.__new__(StreamRunner)
    r.resize, r.keep_ratio = kw.get('resize', (1333, 800)), True
    r.max_src_hw, r.max_ori_hw = kw.get('max_src_hw', (2048, 2048)), kw.get('max_ori_hw', (2048, 2048))
    r.min_mask_up, r.benchmark, r.bm_raw = kw.get('min_mask_up', 0.5), True, True
    r.kw = dict(benchmark=True)
    r.n, r.B = 1, kw.get('batch', 1)
    r._init_queue()
    return r


def test_runner_check_applies_the_benchmark_rule():
    from sipmask_b200.serving import bm_image_meta
    r = _bm_runner()
    for (h, w), img, pad in [((480, 640), (800, 1066), (800, 1088)), ((1080, 1920), (750, 1333), (768, 1344)),
                             ((2048, 1536), (1066, 800), (1088, 800)), ((800, 1000), (800, 1000), (800, 1024)),
                             ((427, 640), (800, 1199), (800, 1216))]:
        img_shape, pad_shape, sf, ori = r.check((h, w))
        assert img_shape == img + (3,) and pad_shape == pad + (3,) and ori == (h, w, 3), (h, w)
        assert (img_shape, pad_shape, sf) == bm_image_meta(h, w)


def test_runner_rejections_before_anything_is_enqueued():
    from sipmask_b200.serving import StreamRunner
    r = _bm_runner()
    with pytest.raises(ValueError, match='size rule'):
        r.check((56, 1345))                         # stays 56x1345: padded 64x1376 is outside 800x1344 / 1344x800
    with pytest.raises(ValueError, match='size rule'):
        r.check((1, 2048))
    small = _bm_runner(resize=(166, 100))
    assert small.check((500, 600))[0] == (100, 120, 3)
    with pytest.raises(ValueError, match='more than 8x'):
        small.check((900, 1000))                    # 900x1000 -> 100x111: 9x
    with pytest.raises(ValueError, match='uint8 HWC RGB'):
        r.submit(torch.zeros((480, 640, 3), dtype=torch.float32))
    with pytest.raises(ValueError, match='raw=True'):
        r.submit(torch.zeros((1, 3, 800, 1088)), meta=((800, 1066, 3), (480, 640, 3), 1.0))
    assert r.i == 0 and r._open is None
    with pytest.raises(ValueError, match='keep_ratio'):
        StreamRunner({}, benchmark=True, raw=True, keep_ratio=False)
    with pytest.raises(ValueError, match='benchmark=True'):
        StreamRunner({}, raw=True)
    with pytest.raises(ValueError, match='batch=1'):
        StreamRunner({}, batch=2, benchmark=True)     # without raw: one preprocessed image per forward, as before


def _host_engine(N, hw, metas, benchmark=True):
    from sipmask_b200.engine import SipMaskEngine
    e = SipMaskEngine.__new__(SipMaskEngine)
    e.N, (e.H, e.W), e.dev, e.benchmark = N, hw, torch.device('cpu'), benchmark
    e.image_metas = metas
    return e


def test_forward_raw_benchmark_pipeline_rejections():
    img = torch.zeros((900, 1000, 3), dtype=torch.uint8)
    with pytest.raises(ValueError, match='benchmark=True engine'):
        _host_engine(1, (128, 128), [((100, 111, 3), (900, 1000, 3), 1.0)], benchmark=False).forward_raw(
            img, pipeline='benchmark')
    e = _host_engine(1, (128, 128), [((100, 111, 3), (900, 1000, 3), 1.0)])
    with pytest.raises(ValueError, match="'mmdet' or 'benchmark'"):
        e.forward_raw(img, pipeline='pil')
    with pytest.raises(ValueError, match='more than 8x'):
        e.forward_raw(img, pipeline='benchmark')
    with pytest.raises(ValueError, match='uint8 HWC RGB'):
        e.forward_raw(img.float(), pipeline='benchmark')
    # the same shrink is accepted by the cv2 pipeline, whose kernel has no tap limit
    rows = e._raw_src_rows([img], MEAN)
    assert (rows[0].src_h, rows[0].dst_h, rows[0].dst_w) == (900, 100, 111)
    ok = _host_engine(2, (128, 128), [((113, 128, 3), (900, 1000, 3), 1.0)] * 2)._raw_src_rows([img, None], MEAN,
                                                                                            'benchmark')
    assert (ok[0].dst_h, ok[0].dst_w) == (113, 128) and not ok[1].src and list(ok[1].mean) == list(np.float32(MEAN))
