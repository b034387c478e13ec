"""Host side of batched raw-image streams (StreamRunner(batch=B), SipMaskEngine.forward_raw with N images): the rule that
closes a batch and the rejections that must happen before anything is enqueued, checked without a device."""
import ctypes

import pytest
import torch


def _queue_runner(batch, in_flight=1, **kw):
    """A StreamRunner's host state (validation + batch bookkeeping) whose device steps only record what they were asked."""
    from sipmask_b200.serving import StreamRunner
    r = StreamRunner.__new__(StreamRunner)
    r.resize, r.keep_ratio = kw.get('resize', (1333, 800)), kw.get('keep_ratio', True)
    r.max_src_hw, r.max_ori_hw = kw.get('max_src_hw', (2048, 2048)), kw.get('max_ori_hw', (2048, 2048))
    r.min_mask_up, r.benchmark = kw.get('min_mask_up', 0.5), False
    r.kw = dict(ssd_flag=kw.get('ssd_flag', False))
    r.n, r.B = in_flight, batch
    r._init_queue()
    log = []
    r._begin = lambda k, hw: log.append(('open', k, hw))
    r._stage = lambda k, j, img: log.append(('stage', k, j, tuple(img.shape[:2])))
    r._launch = lambda k, pad, images: log.append(('launch', k, pad, [m['ticket'] for m in images]))
    return r, log


def _img(h, w):
    return torch.zeros((h, w, 3), dtype=torch.uint8)


def _launches(log):
    return [e[1:] for e in log if e[0] == 'launch']


def test_full_batches_dispatch_in_submission_order():
    r, log = _queue_runner(3, in_flight=2, resize=(544, 544), keep_ratio=False, ssd_flag=True)
    tickets = [r.submit(_img(h, w)) for h, w in [(480, 640), (640, 480), (375, 500), (427, 640), (500, 375), (600, 800)]]
    assert tickets == list(range(6))
    assert _launches(log) == [(0, (544, 544), [0, 1, 2]), (1, (544, 544), [3, 4, 5])]
    # an image is staged in its batch's slot at its position, before its batch is dispatched
    assert [e[1:3] for e in log if e[0] == 'stage'] == [(0, 0), (0, 1), (0, 2), (1, 0), (1, 1), (1, 2)]
    assert log.index(('stage', 0, 2, (375, 500))) < log.index(('launch', 0, (544, 544), [0, 1, 2]))
    assert [m['ticket'] for m in r.slot_images[1]] == [3, 4, 5] and r.meta[1]['ticket'] == 5
    assert r._locate(4) == (1, 1)


def test_padded_shape_change_closes_the_batch_before_staging():
    r, log = _queue_runner(4, in_flight=2)
    # (800, 1088) x2, then (800, 1216) closes it, then back to (800, 1088)
    for h, w in [(480, 640), (600, 800), (427, 640), (426, 640), (480, 640)]:
        r.submit(_img(h, w))
    assert _launches(log) == [(0, (800, 1088), [0, 1]), (1, (800, 1216), [2, 3])]
    i = log.index(('launch', 0, (800, 1088), [0, 1]))
    assert log[i + 1] == ('open', 1, (800, 1216)) and log[i + 2] == ('stage', 1, 0, (427, 640))
    assert r._open['slot'] == 0 and [m['ticket'] for m in r._open['images']] == [4]
    with pytest.raises(ValueError, match='open batch'):
        r._locate(4)
    assert r._locate(1) == (0, 1)                       # slot 0 still holds its first batch until the open one is dispatched
    with pytest.raises(ValueError, match='not held'):
        r._locate(7)


def test_flush_and_partial_batches():
    r, log = _queue_runner(4, in_flight=2, resize=(640, 360))
    r.consume = lambda k, fn: log.append(('consume', k, [m['ticket'] for m in r.slot_images[k]]))
    r._join = lambda: log.append(('join',))
    fn = object()
    # VIS rule: 720x1280, 540x960, 1080x1920 pad to 384x640; 480x640 and 360x480 to 384x480
    sizes = [(720, 1280), (540, 960), (1080, 1920), (720, 1280), (720, 1280), (480, 640), (360, 480), (720, 1280)]
    for h, w in sizes:
        r.step(_img(h, w), fn)
    assert _launches(log) == [(0, (384, 640), [0, 1, 2, 3]), (1, (384, 640), [4]), (0, (384, 480), [5, 6])]
    # two batches in flight: the first is handed over once the second is dispatched, the second once the third is
    assert [e for e in log if e[0] == 'consume'] == [('consume', 0, [0, 1, 2, 3]), ('consume', 1, [4])]
    r.flush(fn)
    assert _launches(log)[-1] == (1, (384, 640), [7])
    assert log[-3:] == [('consume', 0, [5, 6]), ('consume', 1, [7]), ('join',)]
    assert r._open is None and r.pending == [] and r.dispatched == 4
    # every image is handed over exactly once, in submission order
    handed = [t for e in log if e[0] == 'consume' for t in e[2]]
    assert handed == list(range(len(sizes)))


def test_batch_one_returns_slots_and_dispatches_every_image():
    r, log = _queue_runner(1, in_flight=3)
    slots = [r.submit(_img(h, w)) for h, w in [(480, 640), (427, 640), (480, 640), (600, 800)]]
    assert slots == [0, 1, 2, 0]
    assert _launches(log) == [(0, (800, 1088), [0]), (1, (800, 1216), [1]), (2, (800, 1088), [2]), (0, (800, 1088), [3])]
    assert r._open is None and r.meta[0]['ticket'] == 3 and r.meta[0]['ori_shape'] == (600, 800, 3)


def test_rejections_before_anything_is_enqueued():
    from sipmask_b200.serving import StreamRunner
    r, log = _queue_runner(4, max_src_hw=(1080, 1920))
    r.submit(_img(480, 640))
    with pytest.raises(ValueError, match='max_src_hw'):
        r.submit(_img(1200, 1600))
    with pytest.raises(ValueError, match='uint8 HWC'):
        r.submit(torch.zeros((480, 640, 3), dtype=torch.float32))
    # a rejected image neither closes the open batch nor takes a ticket
    assert _launches(log) == [] and r.i == 1 and len(r._open['images']) == 1
    with pytest.raises(ValueError, match='at least 1'):
        StreamRunner({}, batch=0)
    with pytest.raises(ValueError, match='benchmark'):
        StreamRunner({}, batch=2, benchmark=True)


def _host_engine(N, hw=(544, 544), metas=None):
    """A SipMaskEngine's host state for forward_raw's validation (nothing built; the device is never touched)."""
    from sipmask_b200.engine import SipMaskEngine
    e = SipMaskEngine.__new__(SipMaskEngine)
    e.N, (e.H, e.W), e.dev = N, hw, torch.device('cpu')
    e.image_metas = metas or [((hw[0], hw[1], 3), (hw[0], hw[1], 3), 1.0)] * N
    return e


def test_forward_raw_rejections():
    e = _host_engine(4)
    ok = _img(480, 640)
    with pytest.raises(ValueError, match='3 images for a batch of 4'):
        e.forward_raw([ok] * 3)
    with pytest.raises(ValueError, match='1 images for a batch of 4'):
        e.forward_raw(ok)
    chw = torch.zeros((3, 480, 640), dtype=torch.uint8).permute(1, 2, 0)         # HWC shape, CHW memory
    with pytest.raises(ValueError, match='HWC strides'):
        e.forward_raw([ok, chw, ok, ok])
    with pytest.raises(ValueError, match='HWC strides'):
        e.forward_raw([ok, ok, ok[:, ::2], ok])
    with pytest.raises(ValueError, match='uint8 HWC'):
        e.forward_raw([ok, ok, ok, torch.zeros((480, 640, 4), dtype=torch.uint8)])
    with pytest.raises(ValueError, match='uint8 HWC'):
        e.forward_raw([ok.float(), ok, ok, ok])
    big = _host_engine(2, metas=[((544, 544, 3), (480, 640, 3), 1.0), ((576, 544, 3), (480, 640, 3), 1.0)])
    with pytest.raises(ValueError, match='does not fit the 544x544 canvas'):
        big.forward_raw([ok, ok])
    on_gpu = _host_engine(1)
    on_gpu.dev = torch.device('cuda', 0)
    with pytest.raises(ValueError, match='engine on cuda'):
        on_gpu.forward_raw(ok)


def test_source_rows_of_a_valid_batch():
    """Row n holds image n's pointer, size, pitch, its img_shape and the mean; None is a filler row."""
    e = _host_engine(3, metas=[((544, 544, 3), (480, 640, 3), 1.0), ((512, 300, 3), (512, 300, 3), 1.0),
                               ((544, 544, 3), (480, 640, 3), 1.0)])
    a = _img(480, 640)
    wide = torch.zeros((512, 400, 3), dtype=torch.uint8)[:, :300]                # row pitch 1200 > 3 * 300
    rows = e._raw_src_rows([a, wide, None], mean=(1.5, 2.5, 3.5))
    assert (rows[0].src, rows[0].src_h, rows[0].src_w, rows[0].src_pitch_bytes) == (a.data_ptr(), 480, 640, 1920)
    assert (rows[0].dst_h, rows[0].dst_w) == (544, 544)
    assert (rows[1].src_pitch_bytes, rows[1].dst_h, rows[1].dst_w) == (1200, 512, 300)
    assert not rows[2].src and (rows[2].dst_h, rows[2].dst_w) == (0, 0)
    assert all(list(r.mean) == [1.5, 2.5, 3.5] for r in rows)


def test_source_row_layout_matches_the_header():
    from sipmask_b200 import _lib as L
    # include/sipmask_b200.h, smb_raw_src_t: a pointer, five ints, three floats
    assert ctypes.sizeof(L.RawSrc) == 40
    offs = [getattr(L.RawSrc, f).offset for f in ('src', 'src_h', 'src_w', 'src_pitch_bytes', 'dst_h', 'dst_w', 'mean')]
    assert offs == [0, 8, 12, 16, 20, 24, 28]
