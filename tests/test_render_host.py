"""The drawing rules of sipmask_b200.render on the host: the numpy restatement (tests/render_ref.py) reproduces what the
reference's show_result functions drew and handed to imshow_det_bboxes (tests/golden/ref_render.npz), the colour tables
equal the reference's, and the runners reject what they cannot render before any device work."""
import os

import numpy as np
import pytest

import render_ref as RR

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_render.npz')


@pytest.fixture(scope='module')
def golden():
    with np.load(GOLDEN) as z:
        return {k: z[k] for k in z.files}


def _case(g, n):
    return {k[len('c%d_' % n):]: v for k, v in g.items() if k.startswith('c%d_' % n)}


def test_image_palette_equals_the_reference_draws(golden):
    from sipmask_b200 import render
    pal = render.image_palette(int(golden['num_classes']))
    assert pal.shape == (80, 3) and pal.dtype == np.uint8
    assert len(golden['mm_colors']) == 80                 # a case has label 79: the reference drew all 80 colours
    assert np.array_equal(pal, golden['mm_colors'])
    assert np.array_equal(render.image_palette(5), pal[:4])


def test_video_palette_equals_gen_colormask(golden):
    from sipmask_b200 import render
    pal = render.video_palette()
    assert pal.shape == (253, 3) and pal.dtype == np.uint8
    assert np.array_equal(pal, golden['vis_palette'])


def test_restatement_reproduces_image_rule(golden):
    from sipmask_b200 import render
    pal = render.image_palette(int(golden['num_classes']))
    thr = float(golden['score_thr'])
    drawn = 0
    for n in range(int(golden['n_cases'])):
        c = _case(golden, n)
        got = RR.render(c['img'], c['det'], len(c['det']), c['masks'], thr, pal, labels=c['labels'], boxes=False)
        assert np.array_equal(got, c['mm_img']), n
        drawn += int((got != c['img']).any())
        # the boxes imshow_det_bboxes draws: the handed boxes with score > its score_thr, corners as int32
        rec = c['mm_bboxes']
        want = sorted(RR.box_corners(b) for b in rec[rec[:, 4] > np.float32(c['mm_score_thr'])])
        mine = sorted(RR.box_corners(c['det'][i]) for i in RR.image_draws(c['det'], c['labels'], len(c['det']), thr))
        assert mine == want, n
    assert drawn >= 3


def test_restatement_reproduces_video_rule(golden):
    from sipmask_b200 import render
    pal = render.video_palette()
    thr = float(golden['score_thr'])
    for n in range(int(golden['n_cases'])):
        c = _case(golden, n)
        got = RR.render(c['img'], c['det'], len(c['det']), c['masks'], thr, pal, obj_ids=c['ids'], boxes=False)
        draws = RR.frame_draws(c['det'], c['ids'], len(c['det']), thr)
        if 'vis_img' not in c:                            # the reference returned early: no object id in the frame
            assert all(int(v) < 0 for v in c['ids']) and np.array_equal(got, c['img'])
            continue
        assert np.array_equal(got, c['vis_img']), n
        assert [RR.box_corners(c['det'][i]) for i, _ in draws] == [RR.box_corners(b) for b in c['vis_bboxes']], n
        assert [int(c['labels'][i]) for i, _ in draws] == c['vis_labels'].tolist(), n


def test_fixture_covers_the_edges(golden):
    thr = np.float32(golden['score_thr'])
    scores = np.concatenate([_case(golden, n)['det'][:, 4] for n in range(int(golden['n_cases']))])
    assert (scores == thr).any() and (scores == np.nextafter(thr, np.float32(1))).any()
    ids = np.concatenate([_case(golden, n)['ids'] for n in range(int(golden['n_cases']))])
    assert (ids == -1).any() and (ids == 252).any()
    c0 = _case(golden, 0)
    assert c0['img'].shape[1] % 32 and _case(golden, 2)['img'].shape[:2] == (1, 1)
    assert list(c0['labels']) != sorted(c0['labels'])


def test_blends_on_all_pairs():
    p, c = np.meshgrid(np.arange(256), np.arange(256))
    p, c = p.astype(np.uint8).ravel(), c.astype(np.uint8).ravel()
    # the reference's expressions: img * 0.5 + color * 0.5, and color * 0.6 + img * 0.4, float64 assigned to uint8
    assert np.array_equal(RR.blend_image(p, c), (p * 0.5 + c * 0.5).astype(np.uint8))
    assert np.array_equal(RR.blend_frame(p, c), (c * 0.6 + p * 0.4).astype(np.uint8))
    assert (c * 0.6 + p * 0.4).dtype == np.float64


def test_box_pixels_are_the_clipped_border():
    m = RR.box_pixels(np.array([-0.7, 1.9, 3.99, 4.2], np.float32), 6, 5)
    want = np.zeros((6, 5), bool)
    want[1, 0:4] = want[4, 0:4] = True
    want[1:5, 0] = want[1:5, 3] = True
    assert np.array_equal(m, want)
    # swapped corners give the same rectangle; a box around the image draws nothing inside it
    assert np.array_equal(RR.box_pixels(np.array([3.99, 4.2, -0.7, 1.9], np.float32), 6, 5), want)
    assert not RR.box_pixels(np.array([-3, -3, 9, 9], np.float32), 6, 5).any()


def test_runner_arguments_are_validated():
    from sipmask_b200.serving import StreamRunner
    with pytest.raises(ValueError, match='benchmark'):
        StreamRunner({}, render=True, benchmark=True)
    for bad in (float('nan'), float('inf'), 'high', None):
        with pytest.raises(ValueError, match='render_score_thr'):
            StreamRunner({}, render=True, render_score_thr=bad)


def test_render_functions_validate_threshold():
    from sipmask_b200 import render
    with pytest.raises(ValueError, match='score_thr'):
        render.score_threshold(float('nan'), 'score_thr')
    assert render.score_threshold(0.3) == float(np.float32(0.3))
