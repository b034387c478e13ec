"""Detections drawn on the device (smb_render_dev, sipmask_b200.render, StreamRunner / VideoRunner render=True).

The kernel must reproduce the reference's show_result images exactly (tests/golden/ref_render.npz) and, with boxes, the
numpy restatement tests/render_ref.py; the runners' pictures must equal render_ref of the record they return over the
image that was submitted, and every other field must equal a runner without render."""
import os

import numpy as np
import pytest
import torch

import render_ref as RR
from test_gpu_stream import _config, _raw_images

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_render.npz')


def _record(cases, mx, cap_h, words, counts, seed=0):
    """Device record [N, mx, cap_h, words] of the cases' masks, with random bits everywhere outside each canvas and in
    every plane past the case's detections; det / labels / ids padded with random rows."""
    rs = np.random.RandomState(seed)
    N = len(cases)
    bits = rs.randint(-2 ** 31, 2 ** 31 - 1, (N, mx, cap_h, words), dtype=np.int64).astype(np.int32)
    det = rs.uniform(0, 1, (N, mx, 5)).astype(np.float32)
    labels = rs.randint(0, 80, (N, mx)).astype(np.int64)
    ids = rs.randint(-1, 40, (N, mx)).astype(np.int32)
    for n, c in enumerate(cases):
        k, h, w = c['masks'].shape
        planes = RR.pack_planes(c['masks'], words)                  # zero past w inside the words it owns
        junk = bits[n, :k, :h].view(np.uint32)
        keep = np.zeros((h, words * 32), bool)
        keep[:, :w] = True
        keep = np.packbits(keep, axis=-1, bitorder='little').view('<u4').reshape(h, words)
        bits[n, :k, :h] = ((junk & ~keep) | planes.view(np.uint32)).view(np.int32)
        det[n, :k], labels[n, :k], ids[n, :k] = c['det'], c['labels'], c['ids']
    cuda = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return cuda(bits), cuda(det), cuda(labels), cuda(np.array(counts, np.int32)), cuda(ids)


def _golden_cases():
    with np.load(GOLDEN) as z:
        g = {k: z[k] for k in z.files}
    cases = []
    for n in range(int(g['n_cases'])):
        cases.append({k[len('c%d_' % n):]: v for k, v in g.items() if k.startswith('c%d_' % n)})
    return g, cases


@pytest.mark.parametrize('boxes', [False, True])
def test_kernel_equals_reference_show_result(boxes):
    from sipmask_b200 import render
    g, cases = _golden_cases()
    thr = float(g['score_thr'])
    bits, det, labels, count, ids = _record(cases, 16, 40, 3, [len(c['det']) for c in cases])
    imgs = [torch.from_numpy(c['img']).cuda() for c in cases]
    render.render_images(imgs, det, labels, count, bits, num_classes=int(g['num_classes']), score_thr=thr, boxes=boxes)
    frames = [torch.from_numpy(c['img']).cuda() for c in cases]
    render.render_frames(frames, det, ids, count, bits, score_thr=thr, boxes=boxes)
    for n, c in enumerate(cases):
        got = imgs[n].cpu().numpy()
        if not boxes:
            assert torch.equal(imgs[n].cpu(), torch.from_numpy(c['mm_img'])), n
            want_v = c.get('vis_img', c['img'])
            assert torch.equal(frames[n].cpu(), torch.from_numpy(want_v)), n
        want = RR.render(c['img'], c['det'], len(c['det']), c['masks'], thr, render.image_palette(), labels=c['labels'],
                         boxes=boxes)
        assert np.array_equal(got, want), n
        want = RR.render(c['img'], c['det'], len(c['det']), c['masks'], thr, render.video_palette(), obj_ids=c['ids'],
                         boxes=boxes)
        assert np.array_equal(frames[n].cpu().numpy(), want), n


@pytest.mark.parametrize('video', [False, True])
def test_blends_on_all_pairs(video):
    """256 one-row images (pixel x = p in every channel), each with one full mask in colour c = its image index."""
    from sipmask_b200 import render
    N = 256
    imgs = torch.arange(256, dtype=torch.uint8).view(1, 256, 1).expand(N, 1, 256, 3).contiguous().cuda()
    bits = torch.full((N, 1, 1, 8), -1, dtype=torch.int32, device='cuda')
    det = torch.tensor([[[-9.0, -9.0, -8.0, -8.0, 1.0]]]).repeat(N, 1, 1).cuda()
    keys = torch.arange(N).view(N, 1).cuda()
    count = torch.ones(N, dtype=torch.int32, device='cuda')
    palette = np.repeat(np.arange(256, dtype=np.uint8)[:, None], 3, axis=1)
    if video:
        render.render_frames(imgs, det, keys.int(), count, bits, palette=palette)
    else:
        render.render_images(imgs, det, keys, count, bits, palette=palette)
    got = imgs.cpu().numpy()
    c = np.arange(256, dtype=np.uint8)[:, None, None]
    p = np.arange(256, dtype=np.uint8)[None, :, None]
    want = (RR.blend_frame if video else RR.blend_image)(np.broadcast_to(p, (256, 256, 3)), np.broadcast_to(c, (256, 256, 3)))
    assert np.array_equal(got[:, 0], want)


def _random_case(rs, h, w, k):
    masks = np.zeros((k, h, w), np.uint8)
    for d in range(k):
        y0, x0 = rs.randint(0, h), rs.randint(0, w)
        masks[d, y0:y0 + rs.randint(1, h + 1), x0:x0 + rs.randint(1, 600)] = 1
        masks[d] ^= (rs.rand(h, w) < 0.02).astype(np.uint8)
    det = np.zeros((k, 5), np.float32)
    det[:, 0], det[:, 2] = rs.uniform(-5, w + 5, k), rs.uniform(-5, w + 5, k)
    det[:, 1], det[:, 3] = rs.uniform(-5, h + 5, k), rs.uniform(-5, h + 5, k)
    det[:, 4] = rs.uniform(0, 1, k)
    det[::7, 4] = np.float32(0.3)
    return dict(img=rs.randint(0, 256, (h, w, 3)).astype(np.uint8), det=det, masks=masks,
                labels=rs.randint(0, 80, k).astype(np.int64), ids=rs.choice([-1, 0, 3, 7, 252, 253, 300], k).astype(np.int64))


@pytest.mark.parametrize('video', [False, True])
def test_one_launch_mixed_sizes_junk_and_counts(video):
    from sipmask_b200 import render
    rs = np.random.RandomState(7)
    sizes, counts = [(70, 2100), (1, 37), (33, 45), (33, 45)], [100, 1, -3, 150]
    cases = [_random_case(rs, h, w, 100) for h, w in sizes]
    bits, det, labels, count, ids = _record(cases, 100, 70, 66, counts, seed=1)
    imgs = [torch.from_numpy(c['img']).cuda() for c in cases]
    if video:
        render.render_frames(imgs, det, ids, count, bits)
    else:
        render.render_images(imgs, det, labels, count, bits)
    pal = render.video_palette() if video else render.image_palette()
    changed = 0
    for n, c in enumerate(cases):
        kw = dict(obj_ids=c['ids']) if video else dict(labels=c['labels'])
        want = RR.render(c['img'], c['det'], counts[n], c['masks'], 0.3, pal, **kw)
        assert np.array_equal(imgs[n].cpu().numpy(), want), n
        changed += int((want != c['img']).any())
    assert changed >= 2


def _check_picture(rec, img, thr, palette):
    cnt = int(rec['count'].reshape(-1)[0])
    h, w = img.shape[:2]
    masks = RR.unpack_planes(rec['mask_bits'].cpu().numpy(), h, w)
    want = RR.render(img.numpy(), rec['det_bboxes'].cpu().numpy(), cnt, masks, thr, palette,
                     labels=rec['det_labels'].cpu().numpy())
    assert np.array_equal(rec['render'].cpu().numpy(), want)
    return int((want != img.numpy()).any())


def _run(name, imgs, batch, in_flight, render, thr=0.3):
    """Every image through StreamRunner.step with a consumer that clones the device record on the current stream: no
    host wait between submissions, so staging slots are reused while earlier batches are still being drawn."""
    from sipmask_b200.serving import StreamRunner
    sd, ekw, rule, _ = _config(name)
    runner = StreamRunner(sd, in_flight=in_flight, batch=batch, max_src_hw=(1088, 1920), max_ori_hw=(1080, 1920),
                          min_mask_up=0.5, render=render, render_score_thr=thr, **rule, **ekw)
    recs = []

    def clone(rec):
        recs.append({k: v.clone() for k, v in rec.items()})
    for img in imgs:
        runner.step(img.pin_memory(), fn=clone)
    runner.flush(fn=clone)
    torch.cuda.synchronize()
    return runner, recs


# the synthetic SSD-style weights score below the default 0.3: that stream draws at a lower threshold
@pytest.mark.parametrize('name,batch,in_flight,n_img,thr', [('mm_gn_r50', 1, 2, 8, 0.3), ('ssd', 4, 2, 11, 0.1)])
def test_stream_runner_render(name, batch, in_flight, n_img, thr):
    from sipmask_b200 import render
    _, _, _, sizes = _config(name)
    rs = np.random.RandomState(3)
    imgs = _raw_images([sizes[i] for i in rs.randint(0, len(sizes), n_img)], seed=4)
    _, plain = _run(name, imgs, batch, in_flight, False)
    runner, drawn = _run(name, imgs, batch, in_flight, True, thr)
    assert len(plain) == len(drawn) == n_img
    pal = render.image_palette(81)
    changed = 0
    for img, a, b in zip(imgs, plain, drawn):
        assert set(b) == set(a) | {'render'}
        for k in a:
            assert torch.equal(a[k], b[k]), k
        assert tuple(b['render'].shape) == tuple(img.shape)
        changed += _check_picture(b, img, thr, pal)
    assert changed >= n_img // 2
    # result() carries the same picture as the device record
    k = (runner.dispatched - 1) % runner.n
    last = runner.slot_images[k][-1]
    res = runner.result(k if batch == 1 else last['ticket'])
    assert torch.equal(res['render'], drawn[-1]['render'].cpu())


def test_video_runner_render_several_lanes():
    from sipmask_b200 import render
    from sipmask_b200.cocoeval import segm_plane
    from sipmask_b200.serving import VideoRunner
    from test_gpu_video import _interleave, _read_before_reuse, _sd, _videos
    sd, kw, rule = _sd()
    videos = _videos()
    order = _interleave(videos)
    vr = VideoRunner(sd, lanes=4, batch=4, in_flight=2, max_src_hw=(1080, 1920), masks='rle', render=True,
                     render_score_thr=0.05, **rule, **kw)
    done, tickets = {}, []

    def read(t):
        r = vr.result(t)
        return dict(r, obj_ids=r['obj_ids'].clone(), det_bboxes=r['det_bboxes'].clone(), count=r['count'].clone(),
                    det_labels=r['det_labels'].clone(), render=r['render'].clone())
    for v, f in order:
        _read_before_reuse(vr, read, done, videos[v][1][f])
        tickets.append(vr.submit(videos[v][1][f], videos[v][0], f))
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    _read_before_reuse(vr, read, done)
    vr.flush()
    for t in tickets:
        if t not in done:
            done[t] = read(t)
    pal = render.video_palette()
    changed = 0
    for (v, f), t in zip(order, tickets):
        r, img = done[t], videos[v][1][f]
        h, w = img.shape[:2]
        cnt = int(r['count'].reshape(-1)[0])
        planes = np.zeros((len(r['det_bboxes']), h, (w + 31) // 32), np.uint32)
        for i, s in enumerate(r['segms'][:cnt]):
            planes[i] = segm_plane(s, h, w)
        ids = np.full(len(r['det_bboxes']), -1, np.int64)
        ids[:cnt] = r['obj_ids'].numpy()
        want = RR.render(img.numpy(), r['det_bboxes'].numpy(), cnt, RR.unpack_planes(planes.view(np.int32), h, w), 0.05,
                         pal, obj_ids=ids)
        assert np.array_equal(r['render'].numpy(), want), (v, f)
        changed += int((want != img.numpy()).any())
    assert changed >= len(tickets) // 2
