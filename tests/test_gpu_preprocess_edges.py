"""The raw-image preprocessing kernels at the edges of their size rules, against OpenCV and Pillow themselves:
smb_preprocess_u8_s2d(_dev) against cv2.resize(INTER_LINEAR), smb_preprocess_pil_u8_s2d_dev against
Image.resize(BILINEAR), each followed by BGR, minus the mean, fp16, in the stem's space-to-depth layout.

The shapes are the host sweeps of tests/test_preprocess_edges_host.py that fit a canvas, plus launches that mix the
layouts a served image can have: a row pitch above 3 * w, a source at an odd byte address, a resized size equal to the
canvas on one axis, filler rows, and PIL canvases resized horizontally first next to ones resized vertically first
(Pillow's order for images more than 100 times taller than wide whose height shrinks).  Every canvas starts as a
sentinel, so a cell the kernel never writes fails."""
import ctypes

import numpy as np
import pytest
import torch

from test_preprocess_edges_host import PIL_EDGES, cv2_sweep, pil_sweep

pytestmark = pytest.mark.gpu

MEAN = (102.9801, 115.9465, 122.7717)
SENTINEL = 7.0
BIG = (1408, 1408)          # canvas of the large cases
SMALL = (320, 320)          # canvas of the small ones


def _s2d(bgr_u8, H, W):
    """A resized BGR uint8 image -> minus the mean, fp16, zero-padded, in the stem's layout [H/2+3, W/2+4, 16]."""
    dh, dw = bgr_u8.shape[:2]
    p = np.zeros((H + 6, W + 8, 4), np.float16)
    p[3:3 + dh, 3:3 + dw, :3] = bgr_u8.astype(np.float32) - np.asarray(MEAN, np.float32)
    return p.reshape(H // 2 + 3, 2, W // 2 + 4, 2, 4).transpose(0, 2, 1, 3, 4).reshape(H // 2 + 3, W // 2 + 4, 16)


def _want(kind, img, dh, dw, H, W):
    if kind == 'pil':
        Image = pytest.importorskip('PIL.Image')
        rgb = np.asarray(Image.fromarray(img, 'RGB').resize((dw, dh), Image.BILINEAR))
        return _s2d(rgb[:, :, ::-1], H, W)
    cv2 = pytest.importorskip('cv2')
    return _s2d(cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR), H, W)


def _device_src(img, layout):
    """img on the GPU as a plain tensor, as a view with row pitch 3 * (w + 5) (the extra columns 255), or as a view
    starting at an odd byte address."""
    h, w = img.shape[:2]
    t = torch.from_numpy(img).cuda()
    if layout == 'pitch':
        buf = torch.full((h, w + 5, 3), 255, dtype=torch.uint8, device='cuda')
        buf[:, :w] = t
        v = buf[:, :w]
        assert v.stride(0) == 3 * (w + 5)
        return v
    if layout == 'odd':
        flat = torch.full((h * w * 3 + 1,), 255, dtype=torch.uint8, device='cuda')
        flat[1:] = t.flatten()
        v = flat[1:].view(h, w, 3)
        assert v.data_ptr() % 2 == 1
        return v
    return t


def _check_launch(kind, cases, hw):
    """One batched launch of `kind` ('pil' or 'cv2') over cases [(img or None, (dh, dw), layout)] in hw canvases; every
    canvas must equal the library's (a filler: zero)."""
    from sipmask_b200 import _lib as L, conv as C
    H, W = hw
    dev = torch.device('cuda', torch.cuda.current_device())
    kw = dict(order='RGB', max_downscale=C.PIL_MAX_DOWNSCALE) if kind == 'pil' else {}
    srcs = [None if img is None else _device_src(img, layout) for img, _, layout in cases]
    rows = (L.RawSrc * len(cases))(*[C.raw_src_row(s, (0, 0) if s is None else c[1], hw, MEAN, dev, **kw)
                                     for s, c in zip(srcs, cases)])
    rows_dev = torch.frombuffer(bytearray(bytes(rows)), dtype=torch.uint8).cuda()
    assert rows_dev.numel() == len(cases) * ctypes.sizeof(L.RawSrc)
    out = torch.full((len(cases), H // 2 + 3, W // 2 + 4, 16), SENTINEL, dtype=torch.float16, device='cuda')
    (C.preprocess_pil_rows if kind == 'pil' else C.preprocess_u8_rows)(rows_dev, out)
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    bad = []
    for n, (img, (dh, dw), layout) in enumerate(cases):
        want = np.zeros_like(got[n]) if img is None else _want(kind, img, dh, dw, H, W)
        if not np.array_equal(got[n], want):
            cells = int((got[n] != want).any(-1).sum())
            bad.append((n, None if img is None else img.shape[:2], (dh, dw), layout, cells))
    assert not bad, 'canvases differ (index, source, resized, layout, cells): %s' % bad


def _img(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, (h, w, 3), dtype=np.uint8)


def _sweep_launches(kind, sweep):
    """The sweep's pairs that fit a canvas, in launches of up to 32 small or 12 large canvases with a filler in each;
    every third source has a row pitch above 3 * w and every fifth an odd address."""
    pairs = [p for pairs in sweep.values() for p in pairs if p[1][0] <= BIG[0] and p[1][1] <= BIG[1]]
    small = [p for p in pairs if p[1][0] <= SMALL[0] and p[1][1] <= SMALL[1]]
    large = [p for p in pairs if p not in small]
    layouts = lambda i: 'pitch' if i % 3 == 1 else 'odd' if i % 5 == 2 else 'plain'  # noqa: E731
    n = 0
    for group, hw, per in ((small, SMALL, 31), (large, BIG, 11)):
        for i in range(0, len(group), per):
            cases = [(_img(h, w, 50 + n + j), (dh, dw), layouts(n + j))
                     for j, ((h, w), (dh, dw)) in enumerate(group[i:i + per])]
            cases.insert(len(cases) // 2, (None, (0, 0), 'plain'))
            _check_launch(kind, cases, hw)
            n += per
    return len(pairs)


def test_pil_kernel_sweep_equals_pillow():
    """Every pair of the host's Pillow sweep that fits a canvas: shrink bands up to 8x, one axis unchanged, upscales of
    1-pixel sources, wide and tall images, the benchmark rule around its switches and 200 random pairs."""
    pytest.importorskip('PIL.Image')
    assert _sweep_launches('pil', pil_sweep()) > 300


def test_pil_kernel_edges_equal_pillow():
    """One launch: exactly 8x on both axes (the most taps and the widest tile spans), 8x on one axis with an upscale on
    the other, one axis unchanged, the tall images Pillow resizes vertically first (2001x20, 1401x14, 1500x14, and
    10000x12 resized to the full canvas height) next to 2000x20 (h = 100 w: horizontally first), a resize to the full
    canvas height, a filler, pitched and odd-address sources."""
    pytest.importorskip('PIL.Image')
    import bm_transform_ref as P
    assert {dh for _, (dh, _) in PIL_EDGES} >= {BIG[0]} and max(dw for _, (_, dw) in PIL_EDGES) <= BIG[1]
    layouts = ['plain', 'pitch', 'pitch', 'odd', 'plain', 'odd', 'odd', 'pitch', 'plain', 'plain', 'pitch', 'odd', 'plain']
    cases = [(_img(h, w, 1 + i), hw, lay) for i, (((h, w), hw), lay) in enumerate(zip(PIL_EDGES, layouts))]
    cases.insert(10, (None, (0, 0), 'plain'))
    first = [P.pil_height_first(img.shape[0], img.shape[1], dh) for img, (dh, _), _ in cases if img is not None]
    assert sum(first) == 4 and not all(first)
    _check_launch('pil', cases, BIG)


def test_cv2_kernel_sweep_equals_opencv():
    """Every pair of the host's OpenCV sweep that fits a canvas (rescale_size at (1333, 800) and (544, 544) for extreme
    aspect ratios such as 2048x9, 9x2048 and 1x1, exact 2x / 4x shrinks, one axis unchanged, 1-pixel sources)."""
    pytest.importorskip('cv2')
    sweep = cv2_sweep()
    pairs = [p for _, pairs in sweep.items() for p in pairs]
    assert {((2048, 9), (1333, 6)), ((9, 2048), (6, 1333)), ((1, 1), (800, 800))} <= set(pairs)
    assert _sweep_launches('cv2', sweep) == len(pairs)


def test_cv2_kernel_edges_equal_opencv():
    """One batched launch with resizes to the full canvas height and width, pitched and odd-address sources and a filler,
    then 2048x9 through the single-image entry point from a pitched source."""
    cv2 = pytest.importorskip('cv2')
    from sipmask_b200 import conv as C
    H, W = BIG
    cases = [(_img(2048, 9, 21), (H, 6), 'pitch'),
             (_img(9, 700, 22), (5, W), 'odd'),
             (None, (0, 0), 'plain'),
             (_img(1, 1, 23), (H, W), 'plain'),
             (_img(960, 1280, 24), (480, 640), 'odd'),
             (_img(3, 5, 25), (3, 5), 'pitch')]                      # not resized: copied
    _check_launch('cv2', cases, (H, W))
    img = _img(2048, 9, 26)
    src = _device_src(img, 'pitch')
    out = torch.full((1, 1344 // 2 + 3, 32 // 2 + 4, 16), SENTINEL, dtype=torch.float16, device='cuda')
    C.preprocess_u8(src, (1333, 6), out, MEAN)
    torch.cuda.synchronize()
    want = _s2d(cv2.resize(img, (6, 1333), interpolation=cv2.INTER_LINEAR), 1344, 32)
    assert np.array_equal(out[0].cpu().numpy(), want)


def test_engine_forward_raw_equals_forward_on_pillow_tall_image():
    """2001x20, which Pillow resizes vertically first to 1300x13: the benchmark raw forward's stem input and every record
    field equal the same engine's forward of the fp32 image built from Pillow's output."""
    Image = pytest.importorskip('PIL.Image')
    import bm_transform_ref as P
    from test_gpu_stream import _check, _config, _raw_images
    from sipmask_b200 import conv as C
    from sipmask_b200.engine import SipMaskEngine
    from sipmask_b200.serving import bm_image_meta
    sd, kw, _, _ = _config('bm_r50')
    rgb = _raw_images([(2001, 20)], seed=12)[0].numpy()
    img_shape, pad, sf = bm_image_meta(2001, 20)
    (dh, dw), (H, W) = img_shape[:2], pad[:2]
    assert (dh, dw) == (1300, 13) and P.pil_height_first(2001, 20, dh)
    eng = SipMaskEngine(sd, (H, W), img_shape=img_shape, ori_shape=(2001, 20, 3), scale_factor=sf, use_graph=True, **kw)
    raw = {k: v[0].cpu().clone() for k, v in eng.forward_raw([torch.from_numpy(rgb).cuda()], pipeline='benchmark').items()}
    stem_raw = eng.img8.clone()
    r = np.asarray(Image.fromarray(rgb, 'RGB').resize((dw, dh), Image.BILINEAR))[:, :, ::-1]
    x = np.zeros((1, 3, H, W), np.float32)
    x[0, :, :dh, :dw] = (r.astype(np.float32) - np.asarray(MEAN, np.float32)).transpose(2, 0, 1)
    x = torch.from_numpy(x).cuda()
    ref = {k: v[0].cpu().clone() for k, v in eng.forward(x).items()}
    torch.cuda.synchronize()
    assert torch.equal(stem_raw, C.image_to_s2d16(x))
    _check(raw, ref, (2001, 20, 3))
