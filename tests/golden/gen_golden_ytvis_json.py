"""Generate tests/golden/ref_ytvis_json.json: the per-frame results and the YouTube-VIS result json the UNMODIFIED
SipMask-VIS reference writes for a few synthetic tracked videos, with the frames themselves.

    python tests/golden/gen_golden_ytvis_json.py        (needs the reference trees; run from the repository root)

Per frame: bbox2result_with_id (SipMask-VIS/mmdet/core/bbox/transforms.py:182-202) and the obj_segms dict the head builds
(models/anchor_heads/sipmask_head.py:648-665: one RLE per detection with an id >= 0, the last one winning), or the head's
early-return shape for a frame without detections (:608-611).  Per dataset: results2json_videoseg
(core/evaluation/coco_utils.py:205-246) with mmcv.dump bound to json.dump.  Imported through tests/golden/_ref_import.py;
pycocotools is absent: masks are encoded with sipmask_b200.rle.encode (pinned against the oracle by tests/test_head_api.py),
so both sides see the same strings.
"""
import collections
import collections.abc
import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
OUT = os.path.join(HERE, 'ref_ytvis_json.json')
NUM_CLASSES = 41
SIZE = (9, 13)


def _frame(rs, ids, labels=None):
    """One frame's record: k = len(ids) detections with the given object ids."""
    from sipmask_b200 import rle
    k = len(ids)
    x1 = rs.uniform(0, 60, k)
    y1 = rs.uniform(0, 40, k)
    det = np.stack([x1, y1, x1 + rs.uniform(1, 30, k), y1 + rs.uniform(1, 20, k), rs.uniform(0.03, 1, k)], 1)
    if labels is None:
        labels = rs.randint(0, NUM_CLASSES - 1, k)
    masks = (rs.rand(k, SIZE[0], SIZE[1]) < 0.3).astype(np.uint8)
    return dict(det=det.astype(np.float32).tolist(), labels=[int(l) for l in labels], ids=[int(i) for i in ids],
                segms=[rle.encode(m)['counts'].decode() for m in masks])


def _cases():
    rs = np.random.RandomState(5)
    f = lambda ids, labels=None: _frame(rs, ids, labels)                                            # noqa: E731
    return [
        ('two_videos', [[f([0, 1, 2]), f([0, 1, 2, 3]), f([1, 0, 3])],
                        [f([0, 1]), f([1, 0]), f([0, 2, 1]), f([2, 1, 0, 3])]]),
        ('one_frame_video', [[f([0, 1, 2, 3, 4])]]),
        ('duplicate_ids', [[f([0, 1, 2]), f([0, 1, 1, 2]), f([2, 2, 0])]]),
        ('negative_ids', [[f([0, 1]), f([-1, 1, 0, -1]), f([-1, -1])]]),
        ('empty_frame', [[f([0, 1]), f([]), f([1, 0])], [f([]), f([0])]]),
        ('absent_in_middle', [[f([0, 1]), f([1]), f([1, 2]), f([0, 2])]]),
        ('category_tie', [[f([0], [3]), f([0], [1]), f([0], [3]), f([0], [1]), f([0, 1], [7, 2])]]),
    ]


def main():
    sys.path.insert(0, ROOT)
    sys.path.insert(0, HERE)
    for n in ('Sequence', 'Mapping', 'Iterable'):     # python < 3.10 spellings used by the 2019 tree
        if not hasattr(collections, n):
            setattr(collections, n, getattr(collections.abc, n))
    import _ref_import
    _ref_import.install('/root/reference/SipMask-VIS')
    import mmcv
    mmcv.dump = lambda obj, path: json.dump(obj, open(path, 'w'))
    from mmdet.core.bbox.transforms import bbox2result_with_id
    from mmdet.core.evaluation.coco_utils import results2json_videoseg
    out = []
    for name, videos in _cases():
        img_ids, results, frames_out = [], [], []
        for vid, frames in enumerate(videos):
            for fid, fr in enumerate(frames):
                img_ids.append((vid, fid))
                det = torch.tensor(fr['det'], dtype=torch.float32).reshape(-1, 5)
                labels = torch.tensor(fr['labels'], dtype=torch.int64)
                ids = np.asarray(fr['ids'], np.int32)
                if det.shape[0] == 0:                # the head's early return: no ids, one empty list per class
                    segs = [[] for _ in range(NUM_CLASSES - 1)]
                else:
                    segs = {}
                    for i in range(det.shape[0]):
                        if ids[i] >= 0:
                            segs[ids[i]] = {'size': list(SIZE), 'counts': fr['segms'][i].encode()}
                dets = bbox2result_with_id(det, labels, ids)
                # the per-frame pair as the reference holds it, before results2json_videoseg decodes the strings in place
                frames_out.append(dict(
                    det=[[int(o), [float(v) for v in d['bbox']], int(d['label'])] for o, d in dets.items()],
                    seg=([[int(o), s['counts'].decode()] for o, s in segs.items()] if isinstance(segs, dict)
                         else len(segs))))
                results.append((dets, segs))

        class DS(object):
            pass
        ds = DS()
        ds.img_ids = img_ids
        DS.__len__ = lambda self: len(self.img_ids)
        with tempfile.TemporaryDirectory() as d:
            path = os.path.join(d, 'out.json')
            results2json_videoseg(ds, results, path)
            ref = json.load(open(path))
        out.append(dict(name=name, size=list(SIZE), videos=videos, frames=frames_out, json=ref))
    with open(OUT, 'w') as fh:
        json.dump(out, fh, indent=1)
    print('wrote %s (%d cases)' % (OUT, len(out)))


if __name__ == '__main__':
    main()
