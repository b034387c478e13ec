"""Host checks of the config layer (sipmask_b200.config), the classwise AP table, CocoEvaluator.state() / merge() and the
byte transport of dist.gather_eval_state (gloo, world 2)."""
import os
import re
import socket

import numpy as np
import pytest
import torch

from sipmask_b200 import config as C

REF = os.environ.get('SIPMASK_REFERENCE', '/root/reference')
MM, VIS, BM = ('%s/%s/configs/sipmask' % (REF, t) for t in ('SipMask-mmdetection', 'SipMask-VIS', 'SipMask-benchmark'))
need_ref = pytest.mark.skipif(not os.path.isdir(MM), reason='the reference checkout is absent')

S = (8, 16, 32, 64, 128)


def _tc(score_thr, nms_pre=1000, max_per_img=100):
    return dict(nms_pre=nms_pre, score_thr=score_thr, max_per_img=max_per_img, nms=dict(type='nms', iou_thr=0.5))


def _mm(depth, stacked, gn, ssd, dcn=False, resc=False, thr=0.05):
    return dict(depth=depth, backbone_dcn=dcn, stacked_convs=stacked, gn=gn, ssd_flag=ssd, rescoring_flag=resc,
                num_classes=81, strides=S, test_cfg=_tc(thr), vis=False)


BIG = dict(resize=(1333, 800), keep_ratio=True)
SSD = dict(resize=(544, 544), keep_ratio=False)
VIS_KW = dict(depth=50, backbone_dcn=False, stacked_convs=3, gn=True, ssd_flag=False, rescoring_flag=False, num_classes=41,
              strides=S, test_cfg=_tc(0.03, 200, 10), vis=True)
BM_KW = dict(benchmark=True, stacked_convs=4, num_classes=81, strides=S,
             test_cfg=dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.6), max_per_img=100))

# config file -> (tree, engine_kwargs, runner_kwargs, batch_defaults)
EXPECTED = {
    MM + '/sipmask_r50_caffe_fpn_gn_1x.py': ('mmdet', _mm(50, 4, True, False), BIG, dict(batch=1, in_flight=6)),
    MM + '/sipmask_r50_caffe_fpn_gn_ms_2x.py': ('mmdet', _mm(50, 4, True, False), BIG, dict(batch=1, in_flight=6)),
    MM + '/sipmask_r101_caffe_fpn_gn_ms_4x.py': ('mmdet', _mm(101, 4, True, False), BIG, dict(batch=1, in_flight=6)),
    MM + '/sipmask_r50_caffe_fpn_ssd_6x.py': ('mmdet', _mm(50, 2, False, True, thr=0.1), SSD, dict(batch=32)),
    MM + '/sipmask_r50_caffe_fpn_ssd_gn_10x.py': ('mmdet', _mm(50, 2, True, True, thr=0.1), SSD, dict(batch=32)),
    MM + '/sipmask_r101_caffe_fpn_ssd_6x.py': ('mmdet', _mm(101, 2, False, True, thr=0.1), SSD, dict(batch=32)),
    MM + '/sipmask_r101_caffe_fpn_ssd_gn_10x.py': ('mmdet', _mm(101, 2, True, True, thr=0.1), SSD, dict(batch=32)),
    MM + '/sipmask++_r101_caffe_fpn_ssd_6x.py': ('mmdet', _mm(101, 2, False, True, True, True, 0.1), SSD, dict(batch=32)),
    MM + '/sipmask++_r101_caffe_fpn_ssd_gn_10x.py': ('mmdet', _mm(101, 2, True, True, True, True, 0.1), SSD,
                                                     dict(batch=32)),
    VIS + '/sipmask_r50_caffe_fpn_gn_1x.py': ('vis', VIS_KW, dict(resize=(640, 360), keep_ratio=True), {}),
    VIS + '/sipmask_r50_caffe_fpn_gn_ms_1x.py': ('vis', VIS_KW, dict(resize=(640, 360), keep_ratio=True), {}),
    BM + '/sipmask_R_50_FPN_1x.yaml': ('benchmark', dict(BM_KW, depth=50), dict(BIG, raw=True),
                                       dict(batch=1, in_flight=6)),
    BM + '/sipmask_R_101_FPN_ms_3x.yaml': ('benchmark', dict(BM_KW, depth=101), dict(BIG, raw=True),
                                           dict(batch=1, in_flight=6)),
}


@need_ref
def test_every_reference_config_maps():
    import glob
    files = sorted(glob.glob(MM + '/*.py') + glob.glob(VIS + '/*.py') + glob.glob(BM + '/*.yaml'))
    assert sorted(EXPECTED) == files
    for f, (t, ek, rk, bd) in EXPECTED.items():
        cfg = C.load_config(f)
        assert C.tree(cfg) == t, f
        assert C.engine_kwargs(cfg) == ek, f
        assert C.runner_kwargs(cfg) == rk, f
        assert C.batch_defaults(cfg) == bd, f


def _mutate(tmp_path, src, subs, name='cfg'):
    text = open(src).read()
    for old, new in subs:                             # the last occurrence: the test pipeline follows the train one
        assert old in text, (src, old)
        head, tail = text.rsplit(old, 1)
        text = head + new + tail
    path = tmp_path / (name + os.path.splitext(src)[1])
    path.write_text(text)
    return C.load_config(str(path))


@need_ref
@pytest.mark.parametrize('src,subs,key', [
    ('gn_1x', [('flip=False', 'flip=True')], 'MultiScaleFlipAug.flip'),
    ('gn_1x', [('img_scale=(1333, 800),\n        flip', 'img_scale=[(1333, 800), (1333, 640)],\n        flip')],
     'MultiScaleFlipAug.img_scale'),
    ('gn_1x', [('std=[1.0, 1.0, 1.0], to_rgb=False', 'std=[1.0, 1.0, 1.0], to_rgb=True')], 'Normalize.to_rgb'),
    ('gn_1x', [("dict(type='Pad', size_divisor=32)", "dict(type='Pad', size_divisor=64)")], 'Pad.size_divisor'),
    ('gn_1x', [("nms=dict(type='nms', iou_thr=0.5)", "nms=dict(type='matrix_nms', iou_thr=0.5)")], 'test_cfg.nms.type'),
    ('ssd_6x', [("nms=dict(type='nms', iou_thr=0.5)", "nms=dict(type='fast', iou_thr=0.5)")], 'test_cfg.nms.type'),
    ('pp', [("type='DCN', deformable_groups=1", "type='DCNv2', deformable_groups=1")], 'model.backbone.dcn.type'),
    ('vis', [('flip_ratio=0,\n        with_mask=False', 'flip_ratio=0.5,\n        with_mask=False')],
     'data.test.flip_ratio'),
    ('bm50', [('CENTER_SAMPLING_RADIUS: 1.5', 'CENTER_SAMPLING_RADIUS: 1.5\n    USE_DCN_IN_TOWER: True')],
     'USE_DCN_IN_TOWER'),
    ('bm50', [('SIZE_DIVISIBILITY: 32', 'SIZE_DIVISIBILITY: 64')], 'DATALOADER.SIZE_DIVISIBILITY'),
    # without strides SipMaskHead builds its default (4, 8, 16, 32, 64), not the engine's pyramid
    ('gn_1x', [('        strides=[8, 16, 32, 64, 128],\n', '')], 'model.bbox_head.strides'),
    ('bm50', [('USE_C5: False', 'USE_C5: True')], 'MODEL.RETINANET.USE_C5'),
    ('bm50', [('BACKBONE_OUT_CHANNELS: 256', 'BACKBONE_OUT_CHANNELS: 256\n    NUM_GROUPS: 32')],
     'MODEL.RESNETS.NUM_GROUPS'),
])
def test_unsupported_settings_raise_naming_the_key(tmp_path, src, subs, key):
    files = dict(gn_1x=MM + '/sipmask_r50_caffe_fpn_gn_1x.py', ssd_6x=MM + '/sipmask_r50_caffe_fpn_ssd_6x.py',
                 pp=MM + '/sipmask++_r101_caffe_fpn_ssd_6x.py', vis=VIS + '/sipmask_r50_caffe_fpn_gn_1x.py',
                 bm50=BM + '/sipmask_R_50_FPN_1x.yaml')
    cfg = _mutate(tmp_path, files[src], subs)
    with pytest.raises(ValueError, match=re.escape(key)):
        C.engine_kwargs(cfg)
        C.runner_kwargs(cfg)


def test_tree_and_unknown_files(tmp_path):
    p = tmp_path / 'x.py'
    p.write_text("data = dict(test=dict(type='VOCDataset'))\n")
    with pytest.raises(ValueError, match='data.test.type'):
        C.tree(C.load_config(str(p)))
    with pytest.raises(ValueError):
        C.load_config(str(tmp_path / 'x.json'))


# ------------------------------------------------------------------------------------------------ checkpoints
def _mm_cfg():
    return {'filename': 'synthetic.py', 'test_cfg': dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5),
                                                        max_per_img=100),
            'model': dict(type='SipMask', backbone=dict(type='ResNet', depth=50, style='caffe'),
                          neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1,
                                    add_extra_convs=True, extra_convs_on_inputs=False, num_outs=5,
                                    relu_before_extra_convs=True),
                          bbox_head=dict(type='SipMaskHead', num_classes=81, stacked_convs=2, norm_cfg=None,
                                         strides=[8, 16, 32, 64, 128])),
            'data': dict(test=dict(type='CocoDataset'))}


def test_load_checkpoint_formats():
    from sipmask_b200 import benchmark as B, synth
    cfg = _mm_cfg()
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False)
    for ck in (dict(state_dict=sd, meta=dict(CLASSES=('a', 'b'))), dict(state_dict={'module.' + k: v for k, v in sd.items()}),
               dict(sd)):
        got, classes = C.load_checkpoint(ck, cfg)
        assert sorted(got) == sorted(sd) and all(got[k] is sd[k] for k in sd)
        assert classes == (['a', 'b'] if 'meta' in ck else None)
    bad = dict(sd, **{'bbox_head.extra.weight': torch.zeros(1)})
    with pytest.raises(KeyError, match='bbox_head.extra.weight'):
        C.load_checkpoint(dict(state_dict=bad), cfg)
    gn4 = synth.detector_state_dict(50, stacked_convs=4, gn=True)          # a 4-conv GN detector for a 2-conv config
    with pytest.raises(KeyError):
        C.load_checkpoint(gn4, cfg)
    bm_cfg = {'filename': 'bm.yaml', 'bm': dict(C.BM_DEFAULTS, **{k: v[0] for k, v in C.BM_SHIPPED.items()}, **{
        'MODEL.BACKBONE.CONV_BODY': 'R-50-FPN-RETINANET', 'DATALOADER.SIZE_DIVISIBILITY': 32,
        'MODEL.SIPMASK.CENTERNESS_ON_REG': True, 'MODEL.SIPMASK.NORM_REG_TARGETS': True})}
    bm = B.synthetic_state_dict(depth=50)
    got, _ = C.load_checkpoint(dict(model={'module.' + k: v for k, v in bm.items()}, iteration=1), bm_cfg)
    assert sorted(got) == sorted(B.convert_state_dict(bm))
    with pytest.raises(KeyError):
        C.load_checkpoint(dict(model=dict(bm, **{'rpn.head.unknown.weight': torch.zeros(1)})), bm_cfg)


def test_load_checkpoint_from_file(tmp_path):
    from sipmask_b200 import synth
    sd = synth.detector_state_dict(50, stacked_convs=2, gn=False)
    torch.save(dict(state_dict=sd, meta=dict(CLASSES=['x'])), str(tmp_path / 'c.pth'))
    got, classes = C.load_checkpoint(str(tmp_path / 'c.pth'), _mm_cfg())
    assert classes == ['x'] and all(torch.equal(got[k], sd[k]) for k in sd)


# ------------------------------------------------------------------------------------------------ classwise
def test_classwise_table():
    from sipmask_b200 import cocoeval as E
    p = -np.ones((10, 101, 3, 4, 3))
    p[:, :, 0, 0, 2] = 0.5
    p[0, :50, 0, 0, 2] = -1                          # ignored
    p[:, :, 1, 0, 2] = np.linspace(0, 1, 101)[None]
    p[:, :, 1, 1:, :] = 7.0                           # other area ranges / maxDets do not count
    p[:, :, 1, 0, :2] = 9.0
    t = E.classwise_table(p, ['a', 'b', 'c'])
    assert [n for n, _ in t] == ['a', 'b', 'c']
    assert t[0][1] == 0.5 and t[1][1] == pytest.approx(0.5) and np.isnan(t[2][1])
    with pytest.raises(ValueError):
        E.classwise_table(p, ['a'])


# ------------------------------------------------------------------------------------------------ merge
def _gt():
    from sipmask_b200 import cocoeval as E
    ann = dict(images=[dict(id=i, height=20, width=30) for i in range(1, 9)],
               categories=[dict(id=c, name='c%d' % c, supercategory='s') for c in (3, 5)], annotations=[])
    return E.CocoGroundTruth(ann)


def _filled(gt, ids, seed, analyze):
    """A CPU evaluator holding fixed byte rows per image, as add_records leaves them."""
    from sipmask_b200 import cocoeval as E
    ev = E.CocoEvaluator(gt, gt.cat_ids, device='cpu', analyze=analyze)
    for i in ids:
        rng = np.random.default_rng(seed + i)
        for m in ev.metrics:
            ev.rows[m].append(torch.from_numpy(rng.integers(0, 256, 3 * E.OUT_DTYPE.itemsize, dtype=np.uint8)))
            ev.npig[m] += torch.from_numpy(rng.integers(0, 3, ev.npig[m].numel()).astype(np.int32))
            ev.n_results[m] += 3
            if analyze:
                ev.rows_c[m].append(torch.from_numpy(rng.integers(0, 256, 2 * E.OUT_DTYPE.itemsize, dtype=np.uint8)))
                ev.rows_so[m].append(torch.from_numpy(rng.integers(0, 256, E.OUT_DTYPE.itemsize, dtype=np.uint8)))
                ev.npig_ana[m] += 1
        ev.image_ids.append(i)
        ev._seen.add(i)
    return ev


def _records(t, w):
    b = t.contiguous().view(torch.uint8).numpy().tobytes()
    return sorted(b[n:n + w] for n in range(0, len(b), w))


@pytest.mark.parametrize('analyze', [False, True])
def test_merge_equals_one_evaluator(analyze):
    from sipmask_b200 import cocoeval as E
    gt = _gt()
    a, b = _filled(gt, [1, 3, 5, 7], 0, analyze), _filled(gt, [2, 4, 6], 0, analyze)
    a.status[0] = 2
    one = _filled(gt, [1, 2, 3, 4, 5, 6, 7], 0, analyze)          # another order of the same images
    one.status[0] = 2
    merged = E.CocoEvaluator(gt, gt.cat_ids, device='cpu', analyze=analyze)
    merged.merge([a.state(), b.state()])
    s1, s2 = merged.state(), one.state()
    assert list(s1) == merged.state_keys() and sorted(s1) == sorted(s2)
    assert s1['image_ids'].tolist() != s2['image_ids'].tolist()
    for k in s1:
        x, y = s1[k], s2[k]
        if k.startswith('rows') or k == 'image_ids':         # the same rows, in another order
            w = E.OUT_DTYPE.itemsize if k.startswith('rows') else 8
            assert _records(x, w) == _records(y, w), k
        else:
            assert x.dtype == y.dtype and torch.equal(x, y), k
    # an image evaluated on two ranks is refused, and nothing is merged
    with pytest.raises(ValueError, match='image id 3'):
        merged.merge([_filled(gt, [8, 3], 1, analyze).state()])
    assert merged.image_ids == [1, 3, 5, 7, 2, 4, 6]
    with pytest.raises(ValueError, match='twice'):
        E.CocoEvaluator(gt, gt.cat_ids, device='cpu', analyze=analyze).merge([a.state(), a.state()])
    other = E.CocoEvaluator(gt, gt.cat_ids, metrics=('bbox',), device='cpu')
    with pytest.raises(ValueError, match='settings'):
        other.merge([a.state()])


# ------------------------------------------------------------------------------------------------ gloo transport
def _free_port():
    s = socket.socket()
    s.bind(('127.0.0.1', 0))
    port = s.getsockname()[1]
    s.close()
    return port


class _FakeEvaluator:
    def __init__(self, rank):
        g = torch.Generator().manual_seed(rank)
        self.st = {'image_ids': torch.arange(rank, 7, 2, dtype=torch.int64), 'status': torch.tensor([rank], dtype=torch.int32),
                   'rows/bbox': torch.randint(0, 256, (40 * (3 + 5 * rank),), generator=g).to(torch.uint8),
                   'npig/bbox': torch.randint(0, 9, (13,), generator=g).to(torch.int32),
                   'n_results/bbox': torch.tensor([10 + rank], dtype=torch.int64)}

    def state_keys(self):
        return list(self.st)

    def state(self):
        return self.st


def _worker(rank, world, port, q):
    import torch.distributed as dist
    os.environ['MASTER_ADDR'] = '127.0.0.1'
    os.environ['MASTER_PORT'] = str(port)
    dist.init_process_group('gloo', rank=rank, world_size=world)
    from sipmask_b200 import dist as D
    got = D.gather_eval_state(_FakeEvaluator(rank))
    ok = len(got) == world
    for r in range(world):
        exp = _FakeEvaluator(r).state()
        ok = ok and list(got[r]) == list(exp) and all(got[r][k].dtype == exp[k].dtype and torch.equal(got[r][k], exp[k])
                                                        for k in exp)
    blobs = D.gather_bytes(b'rank%d' % rank * (rank + 1) if rank else b'', 'cpu')
    ok = ok and blobs == [b''] + [b'rank%d' % r * (r + 1) for r in range(1, world)]
    q.put((rank, bool(ok)))
    dist.barrier()
    dist.destroy_process_group()


def test_gather_eval_state_gloo_world2():
    import torch.multiprocessing as mp
    ctx = mp.get_context('spawn')
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = dict(q.get(timeout=120) for _ in procs)
    for p in procs:
        p.join(60)
    assert res == {0: True, 1: True}


def test_detector_keys_are_the_synthetic_dicts_keys():
    """load_checkpoint's key set (synth.detector_keys) names exactly what the synthetic detectors hold."""
    import itertools
    from sipmask_b200 import synth
    for depth, stacked, gn, resc, dcn, track in itertools.product((50, 101), (2, 3, 4), (True, False), (True, False),
                                                                  (True, False), (True, False)):
        sd = synth.backbone_state_dict(depth, stage_with_dcn=(False,) + (dcn,) * 3)
        sd.update(synth.neck_state_dict())
        sd.update(synth.head_state_dict(num_classes=41, stacked_convs=stacked, gn=gn, rescoring_flag=resc, track=track))
        keys = synth.detector_keys(depth, stacked, gn, resc, dcn, track)
        assert len(keys) == len(set(keys)) and set(keys) == set(sd), (depth, stacked, gn, resc, dcn, track)
