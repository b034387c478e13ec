"""Image pipeline (SURVEY.md 8f-3): the oracle's restatement of mmcv.imrescale / cv2.resize(INTER_LINEAR) / Normalize / Pad
against OpenCV itself (CPU, bit-exact), and the device kernel against the oracle (-m gpu, bit-exact)."""
import numpy as np
import pytest
import torch

from oracle import preprocess as P

cv2 = pytest.importorskip('cv2')

SHAPES = [(480, 640), (427, 640), (375, 500), (1080, 1920), (333, 500), (800, 1333), (64, 48), (7, 5),
          (2048, 9), (9, 2048), (1, 2048), (2048, 1), (1, 1)]                     # extreme aspect ratios


def _img(h, w, seed):
    return np.random.RandomState(seed).randint(0, 256, size=(h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize('h,w', SHAPES)
def test_oracle_resize_is_cv2_bit_exact(h, w):
    img = _img(h, w, h + w)
    nh, nw, sf = P.rescale_size(h, w, (1333, 800))
    assert max(nh, nw) <= 1333 and min(nh, nw) <= 800 and (max(nh, nw) == 1333 or min(nh, nw) == 800)
    want = cv2.resize(img, (nw, nh), interpolation=cv2.INTER_LINEAR)            # what mmcv.imrescale calls
    assert np.array_equal(P.resize_linear_u8(img, nh, nw), want)
    for (dh, dw) in [(33, 21), (h, w), (2 * h + 1, 3 * w - 2)]:
        assert np.array_equal(P.resize_linear_u8(img, dh, dw), cv2.resize(img, (dw, dh), interpolation=cv2.INTER_LINEAR))


def test_oracle_pipeline_matches_cv2_steps():
    img = _img(480, 640, 1)
    x, meta = P.preprocess(img)
    assert meta['img_shape'] == (800, 1067, 3) and meta['pad_shape'] == (800, 1088, 3) and abs(meta['scale_factor'] - 800 / 480) < 1e-12
    r = cv2.resize(img, (1067, 800), interpolation=cv2.INTER_LINEAR).astype(np.float32)
    r = cv2.subtract(r, np.array(P.MEAN_BGR, np.float64).reshape(1, -1))       # mmcv.imnormalize, std = 1
    assert np.array_equal(x[0, :, :800, :1067], r.transpose(2, 0, 1))
    assert (x[0, :, :, 1067:] == 0).all()


@pytest.mark.gpu
@pytest.mark.parametrize('h,w', [(480, 640), (375, 500), (800, 1333), (1080, 1920), (427, 640), (333, 500), (64, 48),
                                 (720, 1280)])
def test_device_preprocess_bit_exact(h, w):
    from sipmask_b200 import conv as C
    img = _img(h, w, 3 * h + w)
    x, meta = P.preprocess(img)
    nh, nw = meta['img_shape'][:2]
    H, W = meta['pad_shape'][:2]
    Hq, Wq = H // 2 + 3, W // 2 + 4
    out = torch.full((1, Hq, Wq, 16), 7.0, dtype=torch.float16, device='cuda')
    C.preprocess_u8(torch.from_numpy(img).cuda(), (nh, nw), out, P.MEAN_BGR)
    assert torch.equal(out, C.image_to_s2d16(torch.from_numpy(x).cuda()))      # the fp32 path of the engine
    # the oracle's image in the stem's space-to-depth layout, built on the host: zero-padded by 3 (to [H+6, W+8], 4
    # channels), q(Y, X, (dy*2+dx)*4 + c) = padded pixel (2Y+dy, 2X+dx, c)
    p = np.zeros((H + 6, W + 8, 4), np.float16)
    p[3:3 + H, 3:3 + W, :3] = x[0].transpose(1, 2, 0)
    want = p.reshape(Hq, 2, Wq, 2, 4).transpose(0, 2, 1, 3, 4).reshape(1, Hq, Wq, 16)
    assert np.array_equal(out.cpu().numpy(), want)


@pytest.mark.gpu
def test_engine_forward_raw_equals_forward_on_preprocessed():
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    img = _img(96, 144, 5)                                                      # -> 128 x 192 at scale (192, 128)
    x, meta = P.preprocess(img, scale=(192, 128))
    H, W = meta['pad_shape'][:2]
    sd = synth.detector_state_dict(depth=50, seed=1, cls_bias=-2.5)
    cfg = dict(nms_pre=200, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=30)
    eng = SipMaskEngine(sd, (H, W), test_cfg=cfg, img_shape=meta['img_shape'], use_graph=True)
    a = {k: v.clone() for k, v in eng.forward(torch.from_numpy(x).cuda()).items()}
    b = eng.forward_raw(torch.from_numpy(img).cuda())
    torch.cuda.synchronize()
    assert int(a['count'][0]) > 0
    for k in ('det_bboxes', 'det_labels', 'count', 'mask_bits'):
        assert torch.equal(a[k], b[k]), k
    b2 = eng.forward_raw(torch.from_numpy(img).cuda())                           # graph replay path
    torch.cuda.synchronize()
    assert torch.equal(a['mask_bits'], b2['mask_bits'])
