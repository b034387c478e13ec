"""Batched raw-image streams: the batched preprocessing kernel (smb_preprocess_u8_s2d_dev), SipMaskEngine.forward_raw with
N images and StreamRunner(batch=B).

Every per-image quantity depends only on that image (GroupNorm statistics per image, one post-processing chain per image,
one geometry row and one source row per image), so a batch of N images must EQUAL (torch.equal) N batch-1 engines."""
import numpy as np
import pytest
import torch

from test_gpu_stream import _check, _config, _raw_images, _reference

pytestmark = pytest.mark.gpu

MEAN = (102.9801, 115.9465, 122.7717)


def _oracle_s2d(img, dh, dw, H, W):
    """The oracle's resized, mean-subtracted, zero-padded image in the stem's space-to-depth layout [H/2+3, W/2+4, 16]."""
    from oracle import preprocess as P
    x = P.resize_linear_u8(img, dh, dw).astype(np.float32) - np.asarray(MEAN, np.float32)
    p = np.zeros((H + 6, W + 8, 4), np.float16)
    p[3:3 + dh, 3:3 + dw, :3] = x
    return p.reshape(H // 2 + 3, 2, W // 2 + 4, 2, 4).transpose(0, 2, 1, 3, 4).reshape(H // 2 + 3, W // 2 + 4, 16)


def test_batch_kernel_equals_single_image_entry_point():
    """One batch-8 launch: the cv2 copy path, a 7x5 upscale, a 1080x1920 downscale, a source whose row pitch exceeds
    3 * w, two filler rows; every canvas equals the single-image entry point and the oracle."""
    import ctypes
    from sipmask_b200 import _lib as L, conv as C
    H, W = 544, 800
    rs = np.random.RandomState(11)
    wide = torch.from_numpy(rs.randint(0, 256, (500, 900, 3), dtype=np.uint8)).cuda()
    cases = [(rs.randint(0, 256, (300, 400, 3), dtype=np.uint8), (300, 400)),        # same size: cv2 copies
             (rs.randint(0, 256, (7, 5, 3), dtype=np.uint8), (200, 150)),
             None,
             (rs.randint(0, 256, (1080, 1920, 3), dtype=np.uint8), (450, 800)),
             (wide[:, :700], (544, 640)),                                             # row pitch 2700 > 3 * 700
             (rs.randint(0, 256, (480, 640, 3), dtype=np.uint8), (544, 544)),
             None,
             (rs.randint(0, 256, (427, 640, 3), dtype=np.uint8), (544, 800))]
    srcs = [None if c is None else (c[0] if torch.is_tensor(c[0]) else torch.from_numpy(c[0]).cuda()) for c in cases]
    assert srcs[4].stride(0) == 2700
    dev = torch.device('cuda', torch.cuda.current_device())
    rows = (L.RawSrc * 8)(*[C.raw_src_row(s, (0, 0) if c is None else c[1], (H, W), MEAN, dev)
                            for s, c in zip(srcs, cases)])
    rows_dev = torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()
    assert rows_dev.numel() == 8 * ctypes.sizeof(L.RawSrc)
    out = torch.full((8, H // 2 + 3, W // 2 + 4, 16), 7.0, dtype=torch.float16, device='cuda')
    C.preprocess_u8_rows(rows_dev, out)
    torch.cuda.synchronize()
    for n, (s, c) in enumerate(zip(srcs, cases)):
        if c is None:
            assert (out[n] == 0).all(), 'filler canvas %d is not zero' % n
            continue
        one = torch.full((1, H // 2 + 3, W // 2 + 4, 16), 7.0, dtype=torch.float16, device='cuda')
        C.preprocess_u8(s, c[1], one, MEAN)
        assert torch.equal(out[n], one[0]), n
        want = _oracle_s2d(s.cpu().numpy(), c[1][0], c[1][1], H, W)
        assert np.array_equal(out[n].cpu().numpy(), want), n


# per config: two batches of four images of one padded shape (sizes h, w)
BATCHES = {
    'ssd': ([(427, 640), (640, 480), (375, 500), (544, 544)], [(600, 800), (360, 640), (480, 640), (426, 640)]),
    'plusplus': ([(427, 640), (640, 480), (375, 500), (544, 544)], [(600, 800), (360, 640), (480, 640), (426, 640)]),
    'vis': ([(720, 1280), (719, 1280), (540, 960), (1080, 1920)], [(360, 640), (1080, 1920), (450, 800), (720, 1280)]),
}


def _metas(sizes, rule):
    from sipmask_b200.serving import image_meta
    out = [image_meta(h, w, rule['resize'], rule['keep_ratio']) for h, w in sizes]
    assert len(set(m[1] for m in out)) == 1, 'one padded shape per batch'
    return [(m[0], (h, w, 3), m[2]) for m, (h, w) in zip(out, sizes)], out[0][1][:2]


@pytest.mark.parametrize('name', ['ssd', 'plusplus', 'vis'])
def test_batched_forward_raw_equals_batch_one_engines(name):
    from sipmask_b200.engine import SipMaskEngine
    sd, kw, rule, _ = _config(name)
    wc = {}
    sets = [(_raw_images(sizes, seed=40 + i), _metas(sizes, rule)[0]) for i, sizes in enumerate(BATCHES[name])]
    pad = _metas(BATCHES[name][0], rule)[1]
    assert all(_metas(sizes, rule)[1] == pad for sizes in BATCHES[name])
    refs = []
    for imgs, metas in sets:
        refs.append([])
        for im, m in zip(imgs, metas):
            one = SipMaskEngine(sd, pad, img_shape=m[0], ori_shape=m[1], scale_factor=m[2], use_graph=True, share_weights=wc,
                                **kw)
            refs[-1].append({k: v[0].cpu().clone() for k, v in one.forward_raw(im.cuda()).items()})
            del one
    assert sum(int(r['count']) for rr in refs for r in rr) > 0
    many = SipMaskEngine(sd, pad, batch=4, max_ori_hw=(1080, 1920), min_mask_up=0.5, use_graph=True, share_weights=wc,
                         **kw)
    # the second replay takes different images and sizes: nothing about the first batch is baked into the graph
    for (imgs, metas), rr in zip(sets, refs):
        many.set_image_meta(metas)
        out = {k: v.cpu().clone() for k, v in many.forward_raw([im.cuda() for im in imgs], MEAN).items()}
        for i, m in enumerate(metas):
            _check({k: v[i] for k, v in out.items()}, rr[i], m[1])
    # a partial batch: the two real images do not depend on what fills the other two rows (filler rows, then images)
    (imgs, metas), (others, ometas) = sets
    for fill, fmetas in (([None, None], [metas[1]] * 2), ([o.cuda() for o in others[2:]], ometas[2:])):
        many.set_image_meta(metas[:2] + fmetas)
        out = {k: v.cpu().clone() for k, v in many.forward_raw([imgs[0].cuda(), imgs[1].cuda()] + fill).items()}
        for i in range(2):
            _check({k: v[i] for k, v in out.items()}, refs[0][i], metas[i][1])


def _run_batched_stream(name, in_flight, order):
    from sipmask_b200.serving import StreamRunner
    sd, kw, rule, refs = _reference(name)
    max_ori = (max(r['meta'][1][0] for r in refs), max(r['meta'][1][1] for r in refs))
    runner = StreamRunner(sd, in_flight=in_flight, batch=4, max_src_hw=(1088, 1920), max_ori_hw=max_ori, min_mask_up=0.5,
                          **rule, **kw)
    got = []
    tickets = []

    def take(rec):
        got.append({k: v.clone() for k, v in rec.items()})
    for i in order:
        tickets.append(runner.step(refs[i]['img'].pin_memory(), take))
    runner.flush(take)
    torch.cuda.synchronize()
    return runner, tickets, got


@pytest.mark.parametrize('in_flight', [1, 2])
@pytest.mark.parametrize('name', ['ssd', 'plusplus', 'vis', 'mm_gn_r50'])
def test_batched_stream_equals_fixed_shape_engines(name, in_flight):
    sd, kw, rule, refs = _reference(name)
    order = list(range(len(refs)))
    np.random.RandomState(5 + in_flight).shuffle(order)
    order += order[:2]                                    # 10 images: the last batch is partial
    runner, tickets, got = _run_batched_stream(name, in_flight, order)
    assert tickets == list(range(len(order)))
    assert len(got) == len(order)
    for rec, i in zip(got, order):
        _check(rec, refs[i]['rec'], refs[i]['meta'][1])
    if rule['keep_ratio']:
        # shape changes close batches early: more batches than ceil(10 / 4)
        assert runner.dispatched > 3 and len(runner.buckets) >= 3
    else:
        assert runner.dispatched == 3
    # the host records of the last batch, by ticket
    last = runner.slot_images[(runner.dispatched - 1) % in_flight]
    assert last and last[-1]['ticket'] == len(order) - 1
    for m in last:
        host = runner.result(m['ticket'])
        i = order[m['ticket']]
        assert host['meta']['ori_shape'] == refs[i]['meta'][1]
        _check(host, refs[i]['rec'], refs[i]['meta'][1])
