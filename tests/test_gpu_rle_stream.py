"""COCO RLE strings encoded on the device (smb_rle_encode_dev), in the engine (rle_bytes > 0) and in both runners
(masks='rle').

Every string must be byte-identical to sipmask_b200.rle.encode (pycocotools' layout) of the same bit planes, the option
must leave every other record field torch.equal to an engine built without it, and an overflow of either capacity must be
reported in the image's status, never truncated."""
import numpy as np
import pytest
import torch

from test_gpu_stream import _config, _raw_images

pytestmark = pytest.mark.gpu

MEAN = (102.9801, 115.9465, 122.7717)


def _planes_segms(bits, n, ori):
    """rle.encode of the first n planes of one image's record, cropped to its ori canvas."""
    from sipmask_b200 import rle
    return rle.encode_planes(bits[:n].cpu().numpy(), ori)


def _geom_rows(canvases):
    from sipmask_b200 import _lib as L
    rows = []
    for h, w in canvases:
        g = L.ImgGeom()
        g.out_h, g.out_w = h, w
        rows.append(np.frombuffer(bytes(g), dtype=np.int32))
    return torch.from_numpy(np.stack(rows)).cuda()


def _encode(bits, count, canvases, run_cap, rle_bytes):
    """One batched launch -> (per image: the raw region as numpy uint8, region bytes per image)."""
    from sipmask_b200 import ops, rle
    N, mx = bits.shape[:2]
    ib = rle.image_bytes(mx, rle_bytes)
    region = torch.full((N * ib,), 0xAB, dtype=torch.uint8).pin_memory()
    dst = torch.tensor([ops.host_device_pointer(region)], dtype=torch.int64).cuda()
    ws = torch.empty(ops.rle_encode_workspace_bytes(N, mx, run_cap), dtype=torch.uint8, device='cuda')
    ops.rle_encode_dev(bits, count, _geom_rows(canvases), dst, ib, run_cap, ws)
    torch.cuda.synchronize()
    r = region.numpy().copy()
    return [r[i * ib:(i + 1) * ib] for i in range(N)], ib


def _kernel_case():
    """Four images of one record [4, 100, 70, 66 words]: a 70 x 2100 canvas with 100 masks (empty, full, the four corner
    pixels, blobs, column stripes), a 1 x 37 canvas with one mask, count -3 (clamped to 0), and a 33 x 45 canvas of noise
    masks whose count 150 is clamped to 100.  Every bit outside the canvases is random: the encoder crops."""
    rs = np.random.RandomState(3)
    N, mx, ch, cw = 4, 100, 70, 2100
    words = (cw + 31) // 32
    canvases = [(70, 2100), (1, 37), (33, 45), (33, 45)]
    counts = [100, 1, -3, 150]
    px = rs.randint(0, 2, (N, mx, ch, words * 32)).astype(np.uint8)      # junk everywhere, then the canvases
    for n, (h, w) in enumerate(canvases):
        for d in range(mx):
            if n == 0:
                m = np.zeros((h, w), np.uint8)
                if d == 1:
                    m[:] = 1
                elif 2 <= d < 6:
                    m[(0, 0, h - 1, h - 1)[d - 2], (0, w - 1, 0, w - 1)[d - 2]] = 1
                elif d == 6:
                    m[:, ::2] = 1
                elif d >= 7:
                    y0, x0 = rs.randint(0, h), rs.randint(0, w)
                    m[y0:y0 + rs.randint(1, h), x0:x0 + rs.randint(1, 400)] = 1
                    m[rs.randint(0, h, 20), rs.randint(0, w, 20)] ^= 1
            elif n == 1:
                m = rs.randint(0, 2, (h, w)).astype(np.uint8)
            else:
                m = (rs.rand(h, w) < (d % 5) / 4.0).astype(np.uint8)
            px[n, d, :h, :w] = m
    packed = np.packbits(px, axis=-1, bitorder='little').view('<i4').reshape(N, mx, ch, words)
    return torch.from_numpy(packed.copy()).cuda(), torch.tensor(counts, dtype=torch.int32).cuda(), canvases, px


def test_kernel_strings_equal_host_encoder():
    from sipmask_b200 import rle
    bits, count, canvases, px = _kernel_case()
    regions, ib = _encode(bits, count, canvases, run_cap=4 * 2100 + 2, rle_bytes=1 << 20)
    for n, ((h, w), c) in enumerate(zip(canvases, count.tolist())):
        status, k, strings = rle.read_region(regions[n], 100)
        assert status == 0 and k == min(max(c, 0), 100), (n, status, k)
        for d in range(k):
            assert strings[d] == rle.encode(px[n, d, :h, :w])['counts'], (n, d)
        # the device's planes -> host encoder agrees too (the record as the fallback reads it)
        assert [s['counts'] for s in _planes_segms(bits[n], k, (h, w))] == strings


@pytest.mark.parametrize('run_cap,rle_bytes', [(3, 1 << 20), (60, 1 << 20), (8402, 600), (8402, 16), (40, 3000)])
def test_kernel_status_flags_exactly_the_overflows(run_cap, rle_bytes):
    from sipmask_b200 import rle
    bits, count, canvases, px = _kernel_case()
    regions, ib = _encode(bits, count, canvases, run_cap, rle_bytes)
    str_bytes = ib - rle.header_bytes(100)
    for n, ((h, w), c) in enumerate(zip(canvases, count.tolist())):
        k = min(max(c, 0), 100)
        runs = [len(rle.counts(px[n, d, :h, :w])) for d in range(k)]
        lens = [len(rle.encode(px[n, d, :h, :w])['counts']) for d in range(k)]
        want = (rle.RUNS_OVERFLOW if any(r > run_cap for r in runs) else 0)
        if sum(l for l, r in zip(lens, runs) if r <= run_cap) > str_bytes:
            want |= rle.BYTES_OVERFLOW
        status, kk, strings = rle.read_region(regions[n], 100)
        assert (status, kk) == (want, k), (n, status, want)
        if status == 0:
            assert strings == [rle.encode(px[n, d, :h, :w])['counts'] for d in range(k)]
        # nothing past the used bytes of the region was touched
        used = rle.header_bytes(100) + (0 if status else (sum(lens) + 3) // 4 * 4)
        assert (regions[n][used:] == 0xAB).all(), n


def _metas(name, batch):
    from sipmask_b200.serving import image_meta
    oris = [(427, 640), (640, 480), (375, 500), (544, 544)][:batch] if batch > 1 else [(480, 631)]
    if name == 'bm_r50':
        return [((544, 544, 3), (h, w, 3), 1.0) for h, w in oris]
    return [(image_meta(h, w, (544, 544), keep_ratio=False)[0], (h, w, 3), image_meta(h, w, (544, 544), keep_ratio=False)[2])
            for h, w in oris]


def _config_544(name):
    if name == 'bm_r50':
        return _config('bm_r50')[:2]
    sd, kw, _, _ = _config(name)
    return sd, kw


def _check_engine_pair(plain, enc, out_plain, out_enc, metas):
    for key in out_plain:
        assert torch.equal(out_plain[key].cpu(), out_enc[key].cpu()), key
    torch.cuda.synchronize()
    segms = enc.rle_results()
    total = 0
    for n, m in enumerate(metas):
        k = int(out_enc['count'][n])
        total += k
        assert segms[n] == _planes_segms(out_enc['mask_bits'][n], k, m[1][:2]), n
    return total


@pytest.mark.parametrize('batch', [1, 4])
@pytest.mark.parametrize('name', ['mm_gn_r50', 'ssd', 'bm_r50', 'vis', 'plusplus'])
def test_engine_rle_leaves_the_record_unchanged(name, batch):
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    sd, kw = _config_544(name)
    metas = _metas(name, batch)
    wc = {}
    engs = [SipMaskEngine(sd, (544, 544), batch=batch, max_ori_hw=(640, 640), min_mask_up=0.5, use_graph=True,
                          share_weights=wc, rle_bytes=b, **kw) for b in (0, 1 << 16)]
    for e in engs:
        e.set_image_meta(metas)
    imgs = torch.cat([synth.synthetic_image(544, 544, seed=30 + i) for i in range(batch)]).cuda()
    outs = [{k: v.clone() for k, v in e.forward(imgs).items()} for e in engs]
    total = _check_engine_pair(engs[0], engs[1], outs[0], outs[1], metas)
    assert total > 0
    # the raw pipelines replay their own graphs with the encoder in them
    raw = [im.cuda() for im in _raw_images([m[1][:2] for m in metas], seed=9)]
    pipeline = 'benchmark' if name == 'bm_r50' else 'mmdet'
    outs = [{k: v.clone() for k, v in e.forward_raw(raw if batch > 1 else raw[0], MEAN, pipeline).items()} for e in engs]
    _check_engine_pair(engs[0], engs[1], outs[0], outs[1], metas)


def _stream_refs(name, n_img, seed):
    _, _, rule, sizes = _config(name)
    rs = np.random.RandomState(seed)
    picks = [sizes[i] for i in rs.randint(0, len(sizes), n_img)]
    return rule, _raw_images(picks, seed=seed)


def _run_stream(name, masks, imgs, batch, in_flight, **kw):
    """Submits the images and reads every record right after its batch is dispatched (before the slot is reused)."""
    from sipmask_b200.serving import StreamRunner
    sd, ekw, rule, _ = _config(name)
    runner = StreamRunner(sd, in_flight=in_flight, batch=batch, max_src_hw=(1088, 1920), max_ori_hw=(1080, 1920),
                          min_mask_up=0.5, masks=masks, **rule, **ekw, **kw)
    recs = {}

    def collect():
        from sipmask_b200 import rle
        for k, images in enumerate(runner.slot_images):
            for j, m in enumerate(images):
                if m['ticket'] in recs:
                    continue
                r = runner.result(m['ticket'] if batch > 1 else k)
                rec = {key: (v.clone() if torch.is_tensor(v) else v) for key, v in r.items()}
                if masks == 'rle':
                    ib = runner.engines[k][m['pad_shape'][:2]].rle_img_bytes
                    rec['status'] = rle.read_region(runner.rle_regions[k].numpy()[j * ib:(j + 1) * ib], 100)[0]
                recs[m['ticket']] = rec
    for img in imgs:
        before = runner.dispatched
        runner.submit(img.pin_memory())
        if runner.dispatched != before:
            collect()
    runner.flush()
    torch.cuda.synchronize()
    collect()
    return runner, recs


def _compare_streams(bits_recs, rle_recs, tiny):
    from sipmask_b200 import rle
    assert sorted(bits_recs) == sorted(rle_recs)
    dets = 0
    for t in bits_recs:
        a, b = bits_recs[t], rle_recs[t]
        for k in ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'mask_scores', 'track_feats'):
            if k in a:
                assert torch.equal(a[k], b[k]), (t, k)
        assert 'mask_bits' not in b
        n = int(a['count'].reshape(-1)[0])
        dets += n
        ori = a['meta']['ori_shape'][:2]
        assert b['segms'] == rle.encode_planes(a['mask_bits'][:n].numpy(), ori), t
        assert all(s['size'] == [ori[0], ori[1]] for s in b['segms'])
        assert b['status'] == (_tiny_status(a['mask_bits'][:n].numpy(), ori) if tiny else 0), t
    assert dets > 0


# capacities so small that every image with a non-empty mask overflows: one run per mask, 4 string bytes per image
TINY = dict(rle_bytes=4, rle_runs=1)


def _tiny_status(bits, ori):
    """The status TINY capacities must give an image with these planes."""
    from sipmask_b200 import rle
    h, w = ori
    px = np.unpackbits(np.ascontiguousarray(bits[:, :h, :(w + 31) // 32]).view(np.uint8), axis=-1, bitorder='little')[..., :w]
    runs = [len(rle.counts(m)) for m in px]
    lens = [len(rle.encode(m)['counts']) for m in px]
    status = rle.RUNS_OVERFLOW if any(r > 1 for r in runs) else 0
    if sum(l for l, r in zip(lens, runs) if r <= 1) > rle.image_bytes(100, 4) - rle.header_bytes(100):
        status |= rle.BYTES_OVERFLOW
    return status


@pytest.mark.parametrize('tiny', [False, True])
def test_stream_runner_rle_batch1_six_in_flight(tiny):
    rule, imgs = _stream_refs('mm_gn_r50', 9, seed=21)
    _, bits_recs = _run_stream('mm_gn_r50', 'bits', imgs, 1, 6)
    runner, rle_recs = _run_stream('mm_gn_r50', 'rle', imgs, 1, 6, **(TINY if tiny else {}))
    assert len(runner.buckets) >= 2
    _compare_streams(bits_recs, rle_recs, tiny)


@pytest.mark.parametrize('tiny', [False, True])
def test_stream_runner_rle_batch32(tiny):
    rule, imgs = _stream_refs('ssd', 40, seed=22)
    _, bits_recs = _run_stream('ssd', 'bits', imgs, 32, 2)
    runner, rle_recs = _run_stream('ssd', 'rle', imgs, 32, 2, **(TINY if tiny else {}))
    assert runner.dispatched == 2
    _compare_streams(bits_recs, rle_recs, tiny)


@pytest.mark.parametrize('tiny', [False, True])
def test_pipelined_runner_rle_two_slots_one_graph(tiny):
    from sipmask_b200 import rle, synth
    from sipmask_b200.engine import SipMaskEngine
    from sipmask_b200.serving import PipelinedRunner
    sd, kw = _config_544('ssd')
    metas = _metas('ssd', 1)
    wc = {}
    runners = []
    for masks, ekw in (('bits', {}), ('rle', TINY if tiny else dict(rle_bytes=1 << 16))):
        eng = SipMaskEngine(sd, (544, 544), max_ori_hw=(640, 640), min_mask_up=0.5, use_graph=True, share_weights=wc,
                            **ekw, **kw)
        eng.set_image_meta(metas)
        runners.append(PipelinedRunner(eng, depth=2, masks=masks))
    assert runners[1].nslots == 2
    imgs = [synth.synthetic_image(544, 544, seed=50 + i).pin_memory() for i in range(6)]
    got = [[], []]

    def take(r, slot, g):
        res = {k: (v.clone() if torch.is_tensor(v) else v) for k, v in r.result(slot).items()}
        if r.rle:
            res['status'] = rle.read_region(r.rle_regions[slot].numpy(), 100)[0]
        g.append(res)
    for r, g in zip(runners, got):
        slots = []
        for img in imgs:
            if len(slots) == 2:                      # read the oldest slot before submit() reuses it
                take(r, slots.pop(0), g)
            slots.append(r.submit(img))
        r.drain()
        torch.cuda.synchronize()
        for slot in slots:
            take(r, slot, g)
    dets = 0
    ori = metas[0][1][:2]
    for a, b in zip(*got):
        for k in ('det', 'lab', 'cnt'):
            assert torch.equal(a[k], b[k]), k
        assert 'bits' not in b
        n = int(a['cnt'][0])
        dets += n
        assert b['segms'] == [rle.encode_planes(a['bits'][0, :n].numpy(), ori)]
        assert b['status'] == (_tiny_status(a['bits'][0, :n].numpy(), ori) if tiny else 0)
    assert dets > 0
    # the two slots of the one engine own different regions
    assert runners[1].rle_regions[0].data_ptr() != runners[1].rle_regions[1].data_ptr()
