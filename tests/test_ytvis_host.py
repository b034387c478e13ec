"""YouTube-VIS results on the host (sipmask_b200.ytvis): the per-frame pairs and the video json against the UNMODIFIED
SipMask-VIS writers (tests/golden/gen_golden_ytvis_json.py -> ref_ytvis_json.json), and VideoRunner's lane and
frame-order bookkeeping."""
import json
import os

import numpy as np
import pytest

from sipmask_b200 import ytvis


def _cases(golden_dir):
    return json.load(open(os.path.join(golden_dir, 'ref_ytvis_json.json')))


def _frames(case):
    """Per video, the frame pairs frame_result builds from the fixture's records."""
    out = []
    for frames in case['videos']:
        out.append([ytvis.frame_result(np.asarray(f['det'], np.float32).reshape(-1, 5), f['labels'], np.asarray(f['ids'], np.int32),
                                       [{'size': list(case['size']), 'counts': s.encode()} for s in f['segms']])
                    for f in frames])
    return out


def test_frame_results_equal_reference(golden_dir):
    for case in _cases(golden_dir):
        got = [fr for video in _frames(case) for fr in video]
        assert len(got) == len(case['frames']), case['name']
        for (det, seg), want in zip(got, case['frames']):
            # same ids in the same (dict) order, the last detection's box / label / mask for a duplicate id
            assert [[o, d['bbox'].tolist(), int(d['label'])] for o, d in det.items()] == want['det'], case['name']
            for o, d in det.items():
                assert d['bbox'].dtype == np.float32
            if isinstance(want['seg'], int):           # no detections: one empty list per class
                assert seg == [[] for _ in range(want['seg'])], case['name']
            else:
                assert [[o, s['counts'].decode()] for o, s in seg.items()] == want['seg'], case['name']


def test_video_json_equals_reference(golden_dir):
    for case in _cases(golden_dir):
        got = []
        for vid, frames in enumerate(_frames(case)):
            got += ytvis.video_json(vid + 1, frames)      # the reference's video_id is the dataset index + 1
        assert got == case['json'], case['name']
        assert json.loads(json.dumps(got)) == case['json']


def test_video_json_leaves_frames_unchanged(golden_dir):
    case = _cases(golden_dir)[0]
    frames = _frames(case)[0]
    before = [{o: dict(s) for o, s in seg.items()} for _, seg in frames]
    a = ytvis.video_json(1, frames)
    assert [{o: dict(s) for o, s in seg.items()} for _, seg in frames] == before
    assert ytvis.video_json(1, frames) == a


def test_book_lanes_and_frame_order():
    b = ytvis.VideoBook(2)
    assert b.commit('a', 0, 0) == (0, True)
    assert b.commit('b', 0, 1) == (1, True)
    assert b.commit('a', 1, 2) == (0, False)
    with pytest.raises(ValueError, match='end_video'):
        b.check('c', 0)
    with pytest.raises(ValueError, match='frame 0'):
        b.check('d', 3)
    with pytest.raises(ValueError, match='follows frame 1'):
        b.check('a', 3)
    with pytest.raises(ValueError, match='follows frame 1'):
        b.check('a', 1)
    b.end('b')
    with pytest.raises(ValueError, match='has ended'):
        b.check('b', 1)
    with pytest.raises(ValueError, match='not being served'):
        b.end('b')
    with pytest.raises(ValueError, match='not being served'):
        b.end('zz')
    assert b.check('c', 0) == (1, True)              # the freed lane
    b.end('a')
    assert b.commit('c', 0, 3) == (0, True)           # the lowest free lane
    assert b.videos['a']['frames'] == [0, 2] and b.videos['c']['frames'] == [3]


def test_book_check_changes_nothing():
    b = ytvis.VideoBook(1)
    b.check('a', 0)
    assert b.videos == {} and b.lanes == [None]
    b.commit('a', 0, 0)
    with pytest.raises(ValueError):
        b.commit('a', 2, 1)
    assert b.videos['a']['frames'] == [0]
