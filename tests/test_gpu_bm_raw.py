"""SipMask-benchmark checkpoints served from raw RGB images: the PIL-bilinear preprocessing kernel
(smb_preprocess_pil_u8_s2d_dev), SipMaskEngine.forward_raw(pipeline='benchmark') and StreamRunner(benchmark=True, raw=True).

The kernel restates the benchmark's test transform bit for bit, so its canvas must EQUAL the oracle's, and every record
field of a raw forward must EQUAL (torch.equal) the field of the same engine fed the oracle's fp32 image."""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_stream import _check, _config, _raw_images

pytestmark = pytest.mark.gpu

MEAN = (102.9801, 115.9465, 122.7717)


def _oracle_s2d(rgb, dh, dw, H, W):
    """The oracle's benchmark input (PIL bilinear resize, BGR, minus the mean, zero padding) in the stem's space-to-depth
    layout [H/2+3, W/2+4, 16]."""
    import bm_transform_ref as P
    x = P.resize_pil_bilinear_u8(rgb, dh, dw)[:, :, ::-1].astype(np.float32) - np.asarray(MEAN, np.float32)
    p = np.zeros((H + 6, W + 8, 4), np.float16)
    p[3:3 + dh, 3:3 + dw, :3] = x
    return p.reshape(H // 2 + 3, 2, W // 2 + 4, 2, 4).transpose(0, 2, 1, 3, 4).reshape(H // 2 + 3, W // 2 + 4, 16)


def test_pil_kernel_equals_oracle():
    """One batch-8 launch: an upscale, a 7x5 -> 200x150 upscale, two downscales (the 2048x1536 one with 7 taps), a
    no-resize source, a source whose row pitch exceeds 3 * w and two fillers; the output starts as a sentinel so an
    unwritten cell fails."""
    from sipmask_b200 import _lib as L, conv as C
    H, W = 1088, 1344
    rs = np.random.RandomState(21)
    wide = torch.from_numpy(rs.randint(0, 256, (500, 900, 3), dtype=np.uint8)).cuda()
    cases = [(rs.randint(0, 256, (480, 640, 3), dtype=np.uint8), (800, 1066)),
             (rs.randint(0, 256, (7, 5, 3), dtype=np.uint8), (200, 150)),
             None,
             (rs.randint(0, 256, (1080, 1920, 3), dtype=np.uint8), (750, 1333)),
             (rs.randint(0, 256, (2048, 1536, 3), dtype=np.uint8), (1066, 800)),
             (rs.randint(0, 256, (800, 1000, 3), dtype=np.uint8), (800, 1000)),                  # not resized
             (wide[:, :700], (600, 840)),                                                       # row pitch 2700 > 3 * 700
             None]
    srcs = [None if c is None else (c[0] if torch.is_tensor(c[0]) else torch.from_numpy(c[0]).cuda()) for c in cases]
    assert srcs[6].stride(0) == 2700
    dev = torch.device('cuda', torch.cuda.current_device())
    rows = (L.RawSrc * 8)(*[C.raw_src_row(s, (0, 0) if c is None else c[1], (H, W), MEAN, dev, order='RGB',
                                          max_downscale=C.PIL_MAX_DOWNSCALE) for s, c in zip(srcs, cases)])
    rows_dev = torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()
    assert rows_dev.numel() == 8 * ctypes.sizeof(L.RawSrc)
    out = torch.full((8, H // 2 + 3, W // 2 + 4, 16), 7.0, dtype=torch.float16, device='cuda')
    C.preprocess_pil_rows(rows_dev, out)
    torch.cuda.synchronize()
    for n, (s, c) in enumerate(zip(srcs, cases)):
        if c is None:
            assert (out[n] == 0).all(), 'filler canvas %d is not zero' % n
            continue
        want = _oracle_s2d(s.cpu().numpy(), c[1][0], c[1][1], H, W)
        assert np.array_equal(out[n].cpu().numpy(), want), n


# padded 800x1088 under the default rule (800 / 1333); 800x1000 is not resized (padded 800x1024)
SIZES = [(480, 640), (600, 800), (375, 500), (720, 960), (240, 320), (800, 1000), (810, 1010)]


def _rgb(sizes, seed):
    return [im.numpy() for im in _raw_images(sizes, seed)]


def _meta(h, w):
    from sipmask_b200.serving import bm_image_meta
    img_shape, pad, sf = bm_image_meta(h, w)
    return (img_shape, (h, w, 3), sf), pad[:2]


def _rec(out, i=0):
    return {k: v[i].cpu().clone() for k, v in out.items()}


def test_engine_forward_raw_equals_forward_on_bm_preprocess():
    """batch 1 for an upscale, a downscale and a no-resize image, then batch 4 with a filler: the raw forward of each
    image equals the same engine's forward of bm_preprocess(image)."""
    import bm_transform_ref as P
    from sipmask_b200.engine import SipMaskEngine
    sd, kw, _, _ = _config('bm_r50')
    wc = {}
    imgs = _rgb([(480, 640), (1080, 1920), (800, 1000)], seed=5)
    total = 0
    for rgb in imgs:
        meta, pad = _meta(*rgb.shape[:2])
        eng = SipMaskEngine(sd, pad, img_shape=meta[0], ori_shape=meta[1], scale_factor=meta[2], use_graph=True,
                            share_weights=wc, **kw)
        raw = _rec(eng.forward_raw([torch.from_numpy(rgb).cuda()], pipeline='benchmark'))
        ref = _rec(eng.forward(P.bm_preprocess(rgb).cuda()))
        torch.cuda.synchronize()
        _check(raw, ref, meta[1])
        total += int(ref['count'])
        del eng
    four = _rgb(SIZES[:3], seed=6)
    metas = [_meta(*im.shape[:2]) for im in four]
    pad = metas[0][1]
    assert all(m[1] == pad for m in metas)
    metas = [m[0] for m in metas]
    eng = SipMaskEngine(sd, pad, batch=4, img_shape=metas[0][0], ori_shape=metas[0][1], scale_factor=metas[0][2],
                        max_ori_hw=(600, 800), min_mask_up=0.5, use_graph=True, share_weights=wc, **kw)
    eng.set_image_meta(metas + [metas[-1]])
    raw = {k: v.cpu().clone() for k, v in eng.forward_raw([torch.from_numpy(im).cuda() for im in four] + [None],
                                                          MEAN, pipeline='benchmark').items()}
    x = torch.cat([P.bm_preprocess(im) for im in four] + [torch.zeros((1, 3) + pad)]).cuda()
    ref = {k: v.cpu().clone() for k, v in eng.forward(x).items()}
    torch.cuda.synchronize()
    for i in range(4):
        _check({k: v[i] for k, v in raw.items()}, {k: v[i] for k, v in ref.items()}, (metas + [metas[-1]])[i][1])
        total += int(ref['count'][i])
    assert total > 0
    # the benchmark pipeline captured its own graph; the mmdet pipeline's was never built
    assert eng.graph_raw_bm is not None and getattr(eng, 'graph_raw', None) is None


def _stream(sd, kw, imgs, order, **rk):
    from sipmask_b200.serving import StreamRunner
    runner = StreamRunner(sd, max_src_hw=(810, 1024), max_ori_hw=(810, 1010), min_mask_up=0.5, **rk, **kw)
    got = []

    def take(rec):
        got.append({k: v.cpu() for k, v in rec.items()})
    for i in order:
        if rk.get('raw'):
            runner.step(imgs[i][0], take)                         # uint8 RGB
        else:
            runner.step(imgs[i][1], take, meta=imgs[i][2])        # bm_preprocess's fp32 image and its meta
    runner.flush(take)
    torch.cuda.synchronize()
    return runner, got


def test_raw_runner_equals_preprocessed_runner():
    """A shuffled mix over two padded buckets (800x1088, 800x1024) with a no-resize image and a partial last batch:
    StreamRunner(benchmark=True, raw=True) at batch 4 and at batch 1 with 2 in flight equals the fp32 runner fed
    bm_preprocess outputs with their metas."""
    import bm_transform_ref as P
    sd, kw, _, _ = _config('bm_r50')
    imgs = []
    for rgb in _rgb(SIZES, seed=8):
        meta, pad = _meta(*rgb.shape[:2])
        imgs.append((torch.from_numpy(rgb).pin_memory(), P.bm_preprocess(rgb).pin_memory(), meta))
    assert imgs[5][2][0][:2] == (800, 1000)                       # the no-resize image
    order = list(range(len(imgs)))
    np.random.RandomState(3).shuffle(order)
    order += order[:2]                                            # 9 images
    _, ref = _stream(sd, kw, imgs, order)
    assert len(ref) == len(order) and sum(int(r['count']) for r in ref) > 0
    for rk in (dict(batch=4), dict(batch=1, in_flight=2)):
        runner, got = _stream(sd, kw, imgs, order, raw=True, **rk)
        assert len(got) == len(order)
        assert set(runner.buckets) == {(800, 1088), (800, 1024)}
        for rec, want, i in zip(got, ref, order):
            _check(rec, want, imgs[i][2][1])
        if rk['batch'] == 4:
            assert runner.dispatched > 3                          # shape changes and the end close partial batches
            last = runner.slot_images[(runner.dispatched - 1) % runner.n]
            host = runner.result(last[-1]['ticket'])
            i = order[last[-1]['ticket']]
            assert host['meta']['ori_shape'] == imgs[i][2][1] and host['meta']['img_shape'] == imgs[i][2][0]
            _check(host, ref[-1], imgs[i][2][1])
