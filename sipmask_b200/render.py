"""Detections drawn onto images on the device (csrc/render.cu): the picture of the reference's show_result.

  render_images <- SipMask-mmdetection/mmdet/apis/inference.py:119-184 (show_result; tools/test.py --show)
  render_frames <- SipMask-VIS/mmdet/models/detectors/base.py:90-192 (gen_colormask, show_result(is_video=True);
                   tools/test_video.py --show --save_path)

Both draw in place on the original uint8 HWC images (h x w = each image's ori_shape, channels in the order the images
came in: BGR for the reference's trees) from a device record: bit planes [N, max, cap_h, words], boxes and scores
[N, max, 5], count [N] and labels (images) or object ids (frames), so they work on the engine's and the runners'
records as well as on segm_raster's planes.

  images : the detections with fp32 score > score_thr, class-major (ascending label, detection order within a label, as
           np.vstack(bbox_result)); label l in image_palette()[l]; p <- (p + c) >> 1.
  frames : one entry per object id >= 0 at its first detection's position, drawn with its last detection (a dict keyed
           by id, as bbox2result_with_id), when that detection's score > score_thr; id i in video_palette()[i % 253]
           (the reference indexes past its 253 colours and raises); p <- uint8(c * 0.6 + p * 0.4) in float64.
  boxes  : after every mask, each drawn box's outline in (0, 255, 0): corners truncated toward zero, the border of the
           inclusive rectangle between them clipped to the image.  This is the pixel set OpenCV documents for
           cv2.rectangle(thickness=1, LINE_8); it is restated here, not checked against OpenCV itself.
The label text (cv2.putText) is not drawn.  A count <= 0, or no detection above the threshold, leaves the image as is.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from . import ops

DEFAULT_SCORE_THR = 0.3


def image_palette(num_classes=81):
    """[num_classes - 1, 3] uint8: label l's colour is the l-th np.random.randint(0, 256, (1, 3), dtype=np.uint8) after
    np.random.seed(42), as show_result draws one per label up to max(labels).  Each draw is independent of how many
    follow, so this one table equals the reference's for every image.  num_classes counts the background, as the
    head's does."""
    rs = np.random.RandomState(42)
    return np.concatenate([rs.randint(0, 256, (1, 3), dtype=np.uint8) for _ in range(int(num_classes) - 1)])


def video_palette():
    """[253, 3] uint8: gen_colormask()'s table, the VOC bit-reversal colours of 3 .. 255 (r, g, b in columns 0, 1, 2)."""
    cmap = np.zeros((256, 3), np.uint8)
    for i in range(256):
        r = g = b = 0
        c = i
        for j in range(8):
            r |= (c & 1) << (7 - j)
            g |= ((c >> 1) & 1) << (7 - j)
            b |= ((c >> 2) & 1) << (7 - j)
            c >>= 3
        cmap[i] = (r, g, b)
    return cmap[3:]


def device_palette(table, dev):
    return torch.from_numpy(np.ascontiguousarray(table, dtype=np.uint8)).to(dev)


def rows(images, dev):
    """Device smb_render_img_t rows for (src, dst, h, w) tuples (src / dst uint8 device tensors; dst may be src), copied
    on the current stream from pinned memory."""
    arr = (L.RenderImg * len(images))(*[L.RenderImg(s.data_ptr(), d.data_ptr(), int(h), int(w)) for s, d, h, w in images])
    host = torch.empty(ctypes.sizeof(arr), dtype=torch.uint8, pin_memory=True)
    ctypes.memmove(host.data_ptr(), ctypes.addressof(arr), ctypes.sizeof(arr))
    return host.to(dev, non_blocking=True)


def draw(images, det, count, mask_bits, rule, palette, score_thr=DEFAULT_SCORE_THR, boxes=True, labels=None, obj_ids=None):
    """One launch on the current stream: images = one (src, dst, h, w) per image of the record (see rows()); palette a
    device [rows, 3] uint8 table; rule _lib.RENDER_IMAGES (labels) or _lib.RENDER_VIDEO (obj_ids)."""
    n = len(images)
    if n == 0:
        return
    max_hw = (max(int(i[2]) for i in images), max(int(i[3]) for i in images))
    ops.render(rows(images, det.device), n, max_hw, mask_bits, det, count, palette, rule, score_thr, boxes,
               labels=labels, obj_ids=obj_ids)


def _checked(imgs, det, count, mask_bits, ids, ids_dtype, what):
    """Validated, batched views: (images as (img, img, h, w), det, count int32, mask_bits, ids)."""
    single = det.dim() == 2
    if single:
        det, mask_bits, ids = det[None], mask_bits[None], ids[None]
        imgs = [imgs]
        count = count.reshape(1)
    imgs = list(imgs)
    if det.dim() != 3 or det.shape[2] != 5 or det.dtype != torch.float32:
        raise ValueError('%s: det is an fp32 [N, max, 5] (or [max, 5]) tensor' % what)
    n, mx = det.shape[:2]
    if not 1 <= mx <= L.RENDER_MAX_NUM:
        raise ValueError('%s: %d detections per image, at most %d' % (what, mx, L.RENDER_MAX_NUM))
    if mask_bits.dim() != 4 or tuple(mask_bits.shape[:2]) != (n, mx) or mask_bits.dtype != torch.int32:
        raise ValueError('%s: mask_bits is an int32 [N, max, cap_h, words] record matching det' % what)
    if len(imgs) != n or count.numel() != n or tuple(ids.shape) != (n, mx):
        raise ValueError('%s: %d images, %d counts and ids %s for a record of %d images' % (what, len(imgs), count.numel(),
                                                                                          tuple(ids.shape), n))
    cap_h, words = mask_bits.shape[2:]
    for t in imgs + [det, count, mask_bits, ids]:
        if not t.is_cuda or t.device != det.device:
            raise ValueError('%s: every tensor must be on %s' % (what, det.device))
    for im in imgs:
        if im.dtype != torch.uint8 or im.dim() != 3 or im.shape[2] != 3 or not im.is_contiguous():
            raise ValueError('%s: images are contiguous uint8 [h, w, 3] tensors' % what)
        if im.shape[0] > cap_h or (im.shape[1] + 31) // 32 > words:
            raise ValueError('%s: a %dx%d image is larger than the record\'s %dx%d planes' % (what, im.shape[0], im.shape[1],
                                                                                           cap_h, 32 * words))
    images = [(im, im, im.shape[0], im.shape[1]) for im in imgs]
    return images, det.contiguous(), count.to(torch.int32).contiguous(), mask_bits.contiguous(), \
        ids.to(ids_dtype).contiguous()


def render_images(imgs, det, labels, count, mask_bits, num_classes=81, score_thr=DEFAULT_SCORE_THR, boxes=True,
                  palette=None):
    """Draw the detections of a device record onto its images in place, by SipMask-mmdetection's show_result.
    imgs: N contiguous uint8 [ori_h, ori_w, 3] CUDA tensors (a list, or a [N, h, w, 3] tensor); det [N, max, 5] fp32,
    labels [N, max], count [N], mask_bits [N, max, cap_h, words] int32, or one image's record without the N axis and
    one image.  palette: a [rows, 3] uint8 table in place of image_palette(num_classes).  One launch on the current
    stream; returns imgs."""
    images, det, count, bits, labels = _checked(imgs, det, count, mask_bits, labels, torch.int64, 'render_images')
    score_thr = score_threshold(score_thr, 'render_images: score_thr')
    pal = device_palette(image_palette(num_classes) if palette is None else palette, det.device)
    draw(images, det, count, bits, L.RENDER_IMAGES, pal, score_thr, boxes, labels=labels)
    return imgs


def render_frames(imgs, det, obj_ids, count, mask_bits, score_thr=DEFAULT_SCORE_THR, boxes=True, palette=None):
    """Draw the tracked detections of a device record onto its frames in place, by SipMask-VIS's show_result(is_video)
    (object id i coloured video_palette()[i % 253], or palette[i % rows]).  Arguments as render_images, with obj_ids
    [N, max] (an id < 0 is not drawn) in place of the labels.  Returns imgs."""
    images, det, count, bits, ids = _checked(imgs, det, count, mask_bits, obj_ids, torch.int32, 'render_frames')
    score_thr = score_threshold(score_thr, 'render_frames: score_thr')
    pal = device_palette(video_palette() if palette is None else palette, det.device)
    draw(images, det, count, bits, L.RENDER_VIDEO, pal, score_thr, boxes, obj_ids=ids)
    return imgs


def score_threshold(score_thr, what='score_thr'):
    """score_thr as the fp32 value the scores are compared with; ValueError unless it is a finite number."""
    try:
        v = np.float32(score_thr)
    except (TypeError, ValueError):
        raise ValueError('%s must be a number, got %r' % (what, score_thr))
    if not np.isfinite(v):
        raise ValueError('%s must be finite, got %r' % (what, score_thr))
    return float(v)
