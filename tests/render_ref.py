"""numpy restatement of the drawing rules of sipmask_b200.render (the reference's show_result for images and video
frames), written from the rules themselves: the golden fixture pins it to the reference, and the device kernel is
checked against it."""
import numpy as np

GREEN = np.array([0, 255, 0], np.uint8)


def _count(count, mx):
    return int(min(max(int(count), 0), mx))


def image_draws(det, labels, count, score_thr):
    """Detection indices drawn by the image rule, in draw order: score > score_thr in fp32, class-major, detection order
    within a label (np.vstack(bbox_result))."""
    n = _count(count, len(det))
    thr = np.float32(score_thr)
    sel = [i for i in range(n) if np.float32(det[i, 4]) > thr]
    return sorted(sel, key=lambda i: (int(labels[i]), i))


def frame_draws(det, obj_ids, count, score_thr):
    """(detection, object id) drawn by the video rule, in draw order: one entry per id >= 0 where the id first appears,
    holding the id's last detection (bbox2result_with_id's dict), kept when that detection's score > score_thr."""
    n = _count(count, len(det))
    entries = {}
    for i in range(n):
        oid = int(obj_ids[i])
        if oid >= 0:
            entries[oid] = i                  # a dict keeps the key's first position and takes the last value
    thr = np.float32(score_thr)
    return [(i, oid) for oid, i in entries.items() if np.float32(det[i, 4]) > thr]


def box_corners(box):
    """bbox[:4].astype(np.int32) -> (min x, max x, min y, max y)."""
    x0, y0, x1, y1 = np.asarray(box[:4], np.float32).astype(np.int32).tolist()
    return min(x0, x1), max(x0, x1), min(y0, y1), max(y0, y1)


def box_pixels(box, h, w):
    """The pixels cv2.rectangle(thickness=1, LINE_8) sets: the border of the inclusive rectangle, clipped to h x w."""
    xa, xb, ya, yb = box_corners(box)
    m = np.zeros((h, w), bool)
    ys = np.arange(h)[:, None]
    xs = np.arange(w)[None, :]
    inside = (ys >= ya) & (ys <= yb) & (xs >= xa) & (xs <= xb)
    edge = (ys == ya) | (ys == yb) | (xs == xa) | (xs == xb)
    m[inside & edge] = True
    return m


def blend_image(p, c):
    """uint8(p * 0.5 + c * 0.5)."""
    return ((p.astype(np.uint16) + c.astype(np.uint16)) >> 1).astype(np.uint8)


def blend_frame(p, c):
    """uint8(c * 0.6 + p * 0.4) in float64."""
    return (c.astype(np.uint8) * 0.6 + p.astype(np.uint8) * 0.4).astype(np.uint8)


def render(img, det, count, masks, score_thr, palette, labels=None, obj_ids=None, boxes=True):
    """The drawn copy of img [h, w, 3] uint8: masks [max, >= h, >= w] (dense, cropped here), labels -> the image rule,
    obj_ids -> the video rule, colours palette[key % len(palette)]."""
    out = np.array(img, np.uint8, copy=True)
    h, w = out.shape[:2]
    if obj_ids is None:
        draws = [(i, int(labels[i])) for i in image_draws(det, labels, count, score_thr)]
        blend = blend_image
    else:
        draws = frame_draws(det, obj_ids, count, score_thr)
        blend = blend_frame
    pal = np.asarray(palette, np.uint8)
    for i, key in draws:
        m = np.asarray(masks[i])[:h, :w].astype(bool)
        out[m] = blend(out[m], pal[key % len(pal)][None, :])
    if boxes:
        for i, _ in draws:
            out[box_pixels(det[i], h, w)] = GREEN
    return out


def unpack_planes(bits, h, w):
    """Bit planes [k, >= h, words] (int32, pixel x = bit x & 31 of word x >> 5) -> dense uint8 [k, h, w]."""
    b = np.ascontiguousarray(np.asarray(bits)[:, :h]).view(np.uint8)
    return np.unpackbits(b, axis=-1, bitorder='little')[..., :w]


def pack_planes(masks, words=None):
    """Dense [k, h, w] masks -> int32 bit planes [k, h, words] (words >= ceil(w / 32))."""
    masks = np.asarray(masks, np.uint8)
    k, h, w = masks.shape
    words = words or (w + 31) // 32
    px = np.zeros((k, h, 32 * words), np.uint8)
    px[..., :w] = masks
    return np.packbits(px, axis=-1, bitorder='little').view('<i4').reshape(k, h, words)
