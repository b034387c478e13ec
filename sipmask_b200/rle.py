"""COCO run-length encoding of binary masks (column-major counts + the compressed string), numpy only.

Replaces `pycocotools.mask.encode(np.array(im_mask[:, :, np.newaxis], order='F'))[0]`
(MM/mmdet/models/anchor_heads/sipmask_head.py:655-656); pycocotools is not vendored in the reference and is not
available in the build environment.  Output dict layout matches pycocotools: {'size': [h, w], 'counts': bytes}.
"""
import numpy as np


def counts(mask):
    """mask [H,W] {0,1} -> run lengths in column-major order, starting with the number of zeros."""
    flat = np.asarray(mask, dtype=np.uint8).T.reshape(-1)
    if flat.size == 0:
        return np.zeros((0,), np.int64)
    change = np.flatnonzero(flat[1:] != flat[:-1]) + 1
    bounds = np.concatenate([[0], change, [flat.size]])
    runs = np.diff(bounds)
    if flat[0] != 0:
        runs = np.concatenate([[0], runs])
    return runs.astype(np.int64)


def to_string(cnts):
    """pycocotools rleToString: 5 data bits per character (+ continuation bit), deltas against counts[i-2] for i > 2."""
    out = bytearray()
    for i, c in enumerate(cnts):
        x = int(c)
        if i > 2:
            x -= int(cnts[i - 2])
        more = True
        while more:
            ch = x & 0x1f
            x >>= 5
            more = (x != -1) if (ch & 0x10) else (x != 0)
            if more:
                ch |= 0x20
            out.append(ch + 48)
    return bytes(out)


def encode(mask):
    m = np.asarray(mask, dtype=np.uint8)
    return {'size': [int(m.shape[0]), int(m.shape[1])], 'counts': to_string(counts(m))}


# ---- the per-image regions the device encoder (smb_rle_encode_dev) writes: int32 header {status, n, off[max_num + 1]},
# then the n strings back to back (string i = bytes [off[i], off[i+1]) after the header)
RUNS_OVERFLOW, BYTES_OVERFLOW = 1, 2          # status bits: a mask had more runs than the encoder's capacity / the strings
                                              # did not fit the region


def header_bytes(max_num):
    return 4 * (int(max_num) + 3)


def image_bytes(max_num, rle_bytes):
    """Bytes of one image's region: the header + rle_bytes of strings, rounded up to 16."""
    return (header_bytes(max_num) + int(rle_bytes) + 15) // 16 * 16


def read_region(region, max_num):
    """One image's region (uint8 numpy array or CPU tensor) -> (status, n, [n strings] or None when status != 0)."""
    region = np.asarray(region, dtype=np.uint8)
    hb = header_bytes(max_num)
    hdr = region[:hb].view(np.int32)
    status, n = int(hdr[0]), min(max(int(hdr[1]), 0), int(max_num))
    if status != 0:
        return status, n, None
    off = hdr[2:3 + n].astype(np.int64)
    if off[0] != 0 or np.any(np.diff(off) < 0) or hb + off[-1] > region.size:
        raise ValueError('RLE region header is inconsistent: offsets %s for %d bytes' % (off.tolist(), region.size - hb))
    raw = region[hb:hb + off[-1]].tobytes()
    return 0, n, [raw[off[i]:off[i + 1]] for i in range(n)]


def encode_planes(bits, ori_hw):
    """Bit planes int32 [k, >= h, >= ceil(w / 32)] (pixel x = bit x & 31 of word x >> 5) -> the k RLE dicts of their
    h x w masks, on the host."""
    h, w = int(ori_hw[0]), int(ori_hw[1])
    b = np.ascontiguousarray(np.asarray(bits)[:, :h, :(w + 31) // 32]).astype('<i4', copy=False)
    px = np.unpackbits(b.view(np.uint8), axis=-1, bitorder='little')[..., :w]
    return [encode(m) for m in px]


def image_segms(region, max_num, ori_hw, planes):
    """One image's list of RLE dicts {'size': [h, w], 'counts': bytes} in detection order: from the region's strings, or,
    when its status reports an overflow, by encoding planes(n) (a callable returning the image's first n bit planes) on
    the host."""
    status, n, strings = read_region(region, max_num)
    if status != 0:
        return encode_planes(planes(n), ori_hw) if n else []
    size = [int(ori_hw[0]), int(ori_hw[1])]
    return [{'size': list(size), 'counts': s} for s in strings]
