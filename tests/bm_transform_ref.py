"""TEST INFRASTRUCTURE ONLY - CPU restatement of SipMask-benchmark's test-time image transform, which the GPU tests compare
the device kernel (smb_preprocess_pil_u8_s2d_dev) and the raw serving path against.

Reference: SipMask-benchmark/fcos_core/data/transforms/build.py:17-36 (test: Resize(MIN_SIZE_TEST, MAX_SIZE_TEST) ->
ToTensor -> Normalize(PIXEL_MEAN, PIXEL_STD = 1, to_bgr255=True)), transforms.py:27-95, and to_image_list(size_divisible
= 32) in the model.  The image is a PIL RGB image; Resize is torchvision F.resize = PIL Image.resize(BILINEAR).
resize_pil_bilinear_u8 restates Pillow's libImaging/Resample.c for 8-bit images: separable, antialiased, 22-bit fixed
point, the first pass clipped to uint8.  The horizontal pass runs first, except where Pillow's Image.resize runs the
vertical one first: for an image more than 100 times taller than wide whose height shrinks.  PIN: tests/test_bm_raw_host.py compares it bit for bit with the
installed Pillow's Image.resize, and bm_preprocess with tensors the reference's own transforms produced
(tests/golden/ref_bm_transforms.npz).
"""
import numpy as np

MEAN_BGR = (102.9801, 115.9465, 122.7717)            # configs/sipmask/*.yaml via config/defaults.py: PIXEL_MEAN


def bm_resize_size(h, w, min_size=800, max_size=1333):
    """Resize.get_size (transforms.py:36-55) for an h x w image -> (oh, ow), in Python float arithmetic."""
    size = min_size
    if max_size is not None:
        mn, mx = float(min((w, h))), float(max((w, h)))
        if mx / mn * size > max_size:
            size = int(round(max_size * mn / mx))
    if (w <= h and w == size) or (h <= w and h == size):
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def _pil_bounds(n_in, n_out):
    """The tap bounds of Resample.c precompute_coeffs (bilinear, support 1): per output index the first tap and the number
    of taps [..., n_out], with the scale, support and centers they come from.  n_in may be an int64 array of shape [k, 1]:
    then the bounds of k axes n_in[i] -> n_out at once."""
    scale = np.asarray(n_in, np.float64) / float(n_out)
    fs = np.maximum(scale, 1.0)
    center = (np.arange(n_out, dtype=np.float64) + 0.5) * scale
    xmin = np.maximum(np.trunc(center - fs + 0.5).astype(np.int64), 0)
    cnt = np.minimum(np.trunc(center + fs + 0.5).astype(np.int64), n_in) - xmin
    return xmin, cnt, float(scale) if scale.ndim == 0 else scale, fs, center


def _pil_taps(n_in, n_out):
    """Resample.c precompute_coeffs + normalize_coeffs_8bpc (bilinear, support 1): per output index the first tap, the
    number of taps and the 22-bit fixed-point weights [n_out, ksize] (zero past the tap count)."""
    xmin, cnt, scale, fs, center = _pil_bounds(n_in, n_out)
    fs = float(fs)
    ss = 1.0 / fs
    ksize = int(np.ceil(fs)) * 2 + 1
    ws, ww = [], np.zeros(n_out)
    for x in range(ksize):                             # summed in tap order, as the C loop does
        t = np.abs(((x + xmin).astype(np.float64) - center + 0.5) * ss)
        w = np.where((x < cnt) & (t < 1.0), 1.0 - t, 0.0)
        ww = ww + w
        ws.append(w)
    k = np.stack(ws, 1)
    k = np.where(ww[:, None] != 0, k / np.where(ww == 0, 1.0, ww)[:, None], k)
    return xmin, cnt, np.trunc(0.5 + k * 4194304.0).astype(np.int64)


def _pil_pass(a, n_out, axis):
    """One 8-bit pass of Resample.c along `axis` of an int64 [h, w, c] array: clip8((2^21 + sum v * k) >> 22)."""
    xmin, _, kk = _pil_taps(a.shape[axis], n_out)
    acc = np.full(a.shape[:axis] + (n_out,) + a.shape[axis + 1:], 1 << 21, np.int64)
    for j in range(kk.shape[1]):
        idx = np.minimum(xmin + j, a.shape[axis] - 1)   # weights past the tap count are zero
        wj = kk[:, j].reshape((-1, 1, 1) if axis == 0 else (1, -1, 1))
        acc += np.take(a, idx, axis=axis) * wj
    return np.clip(acc >> 22, 0, 255)


def resize_pil_bilinear_u8(src, dh, dw):
    """uint8 [h,w,c] -> uint8 [dh,dw,c], bit-exact PIL Image.resize((dw, dh), Image.BILINEAR)."""
    sh, sw = src.shape[:2]
    if (sh, sw) == (dh, dw):
        return src.copy()
    a = src.astype(np.int64)
    # Pillow skips a pass whose axis keeps its size, and runs the vertical pass first for an image more than 100 times
    # taller than wide whose height shrinks (PIL/Image.py, Image.resize)
    for axis in ((0, 1) if pil_height_first(sh, sw, dh) else (1, 0)):
        if a.shape[axis] != (dh, dw)[axis]:
            a = _pil_pass(a, (dh, dw)[axis], axis)
    return a.astype(np.uint8)


def pil_height_first(h, w, dh):
    """Whether Image.resize runs the vertical pass of an h x w image resized to height dh first."""
    return h > 100 * w and dh < h


def bm_preprocess(rgb_u8, min_size=800, max_size=1333, mean=MEAN_BGR, size_divisor=32):
    """uint8 RGB [h,w,3] -> the benchmark test transform's fp32 NCHW [1,3,H,W] (BGR, mean-subtracted, zero-padded to a
    multiple of size_divisor) as a torch tensor."""
    import torch
    h, w = rgb_u8.shape[:2]
    oh, ow = bm_resize_size(h, w, min_size, max_size)
    r = resize_pil_bilinear_u8(rgb_u8, oh, ow)[:, :, ::-1].astype(np.float32) - np.asarray(mean, np.float32)
    H = (oh + size_divisor - 1) // size_divisor * size_divisor
    W = (ow + size_divisor - 1) // size_divisor * size_divisor
    out = np.zeros((H, W, 3), np.float32)
    out[:oh, :ow] = r
    return torch.from_numpy(np.ascontiguousarray(out.transpose(2, 0, 1))[None])
