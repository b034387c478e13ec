"""Host side of the device RLE strings: the character-count model the encoder kernel implements, the region layout the
pack kernel writes, and the COCO json of a record (sipmask_b200.coco) against the reference's own writers."""
import json
import os

import numpy as np
import pytest

from sipmask_b200 import coco, rle

HERE = os.path.dirname(os.path.abspath(__file__))


def _model(cnts):
    """What rle_encode_kernel computes per run: the pycocotools delta, its character count (the smallest n with
    -2^(5n-1) <= x < 2^(5n-1)), and each run's offset (exclusive scan of the counts)."""
    c = np.asarray(cnts, np.int64)
    x = c.copy()
    x[3:] -= c[1:-2]
    n = np.ones_like(x)
    while True:
        lim = np.int64(1) << (5 * n - 1)
        grow = (x >= lim) | (x < -lim)
        if not grow.any():
            break
        n += grow
    return x, n, np.concatenate([[0], np.cumsum(n)])


@pytest.mark.parametrize('seed', range(6))
def test_character_count_model_matches_to_string(seed):
    rs = np.random.RandomState(seed)
    cases = [[5], [0, 7], [2 ** 31 - 1], [0, 2 ** 31 - 1, 1, 2 ** 31 - 2], [15, 16, 0, 31, 32, 1023, 1024, 3, 2 ** 20]]
    cases.append(rs.randint(0, 2 ** (seed * 5 + 1), rs.randint(1, 400)).tolist())
    cases.append(rle.counts(rs.rand(37, 53) < 0.3).tolist())
    for cnts in cases:
        s = rle.to_string(cnts)
        x, n, off = _model(cnts)
        assert off[-1] == len(s), cnts
        for k in range(len(cnts)):
            # run k's characters are its delta alone, encoded as a one-count string
            assert s[off[k]:off[k + 1]] == rle.to_string([int(x[k])] if k < 3 else [0, 0, 0, int(x[k])])[-n[k]:], (cnts, k)


def _region(strings, max_num, rle_bytes, status=0):
    hb = rle.header_bytes(max_num)
    ib = rle.image_bytes(max_num, rle_bytes)
    r = np.zeros(ib, np.uint8)
    off = np.concatenate([[0], np.cumsum([len(s) for s in strings])]).astype(np.int32)
    hdr = np.concatenate([[status, len(strings)], off, np.full(max_num - len(strings), off[-1])]).astype(np.int32)
    r[:hb] = hdr.view(np.uint8)
    if status == 0:
        raw = b''.join(strings)
        r[hb:hb + len(raw)] = np.frombuffer(raw, np.uint8)
    return r


def test_region_layout_and_fallback():
    rs = np.random.RandomState(1)
    masks = (rs.rand(3, 21, 40) < 0.4).astype(np.uint8)
    want = [rle.encode(m) for m in masks]
    assert rle.header_bytes(100) == 412 and rle.image_bytes(100, 4) == 416 and rle.image_bytes(100, 5) == 432
    r = _region([w['counts'] for w in want], 100, 4096)
    assert rle.read_region(r, 100) == (0, 3, [w['counts'] for w in want])
    assert rle.image_segms(r, 100, (21, 40), None) == want
    planes = np.packbits(np.pad(masks, ((0, 0), (0, 3), (0, 24))), axis=-1, bitorder='little').view('<i4')
    for status in (rle.RUNS_OVERFLOW, rle.BYTES_OVERFLOW, rle.RUNS_OVERFLOW | rle.BYTES_OVERFLOW):
        r = _region([w['counts'] for w in want], 100, 16, status=status)
        assert rle.read_region(r, 100) == (status, 3, None)
        asked = []
        got = rle.image_segms(r, 100, (21, 40), lambda n: asked.append(n) or planes[:n])
        assert asked == [3] and got == want
    assert rle.image_segms(_region([], 100, 16, status=rle.BYTES_OVERFLOW), 100, (21, 40), None) == []


def _cases():
    with open(os.path.join(HERE, 'golden', 'ref_coco_json.json')) as f:
        return json.load(f)


@pytest.mark.parametrize('i', range(6))
def test_coco_json_equals_the_reference_writers(i):
    case = _cases()[i]
    r = case['rec']
    k = len(r['labels'])
    rec = dict(det_bboxes=np.asarray(r['det'], np.float32).reshape(k, 5), det_labels=np.asarray(r['labels'], np.int64),
               count=np.asarray([k], np.int32), segms=[{'size': list(r['size']), 'counts': s.encode()} for s in r['segms']])
    if 'mask_scores' in r:
        rec['mask_scores'] = np.asarray(r['mask_scores'], np.float32)
    # the record is padded past its count, as the engine's is
    rec['det_bboxes'] = np.concatenate([rec['det_bboxes'], np.full((3, 5), 7, np.float32)])
    rec['det_labels'] = np.concatenate([rec['det_labels'], np.full(3, 2, np.int64)])
    bm = case['kind'] == 'bm'
    if bm:
        rec['meta'] = dict(img_shape=tuple(r['img_shape']) + (3,), ori_shape=tuple(r['ori_shape']) + (3,))
    bbox_json, segm_json = coco.coco_json(rec, case['image_id'], case['cat_ids'], benchmark=bm)
    assert bbox_json == case['bbox_json']
    assert segm_json == case['segm_json']
    assert json.loads(json.dumps(segm_json)) == segm_json
