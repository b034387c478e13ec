"""GPU checks of config -> runner (sipmask_b200.config.from_config), tools/test.py and CocoEvaluator.merge, on a synthetic
COCO-format dataset written from a seed (PNG images of mixed sizes, polygon and RLE ground truth, mmcv-format
checkpoints): from_config's records equal the hand-configured runner's, tools/test.py's evaluate() equals
CocoEvalRunner's fed the same images, and two evaluators of disjoint halves, merged, equal one evaluator of all."""
import json
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SIZES = [(400, 600), (300, 450), (320, 480), (600, 400), (360, 240)]
NORM = "dict(mean=[102.9801, 115.9465, 122.7717], std=[1.0, 1.0, 1.0], to_rgb=False)"
MODEL = """
model = dict(type='SipMask',
    backbone=dict(type='ResNet', depth=50, num_stages=4, out_indices=(0, 1, 2, 3), frozen_stages=1,
                  norm_cfg=dict(type='BN', requires_grad=False), style='caffe'{dcn}),
    neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1, add_extra_convs=True,
              extra_convs_on_inputs=False, num_outs=5, relu_before_extra_convs=True),
    bbox_head=dict(type='SipMaskHead', num_classes={ncls}, in_channels=256, stacked_convs={stacked}, feat_channels=256,
                   strides=[8, 16, 32, 64, 128]{head}))
test_cfg = dict(nms_pre={nms_pre}, min_bbox_size=0, score_thr={thr}, nms=dict(type='nms', iou_thr=0.5), max_per_img={mpi})
img_norm_cfg = """ + NORM + "\n"
MM_DATA = """
test_pipeline = [dict(type='LoadImageFromFile'),
    dict(type='MultiScaleFlipAug', img_scale={scale}, flip=False,
         transforms=[dict(type='Resize', keep_ratio={keep}), dict(type='RandomFlip'), dict(type='Normalize', **img_norm_cfg),
                     dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                     dict(type='Collect', keys=['img'])])]
data = dict(test=dict(type='CocoDataset', ann_file='{ann}', img_prefix='{prefix}', pipeline=test_pipeline))
"""
VIS_DATA = """
data = dict(test=dict(type='YTVOSDataset', ann_file='{ann}', img_prefix='{prefix}', img_scale=(640, 360),
                      img_norm_cfg=img_norm_cfg, size_divisor=32, flip_ratio=0, with_mask=False, with_label=False,
                      test_mode=True))
"""
BM_YAML = """MODEL:
  RPN_ONLY: True
  RESNETS:
    BACKBONE_OUT_CHANNELS: 256
  RETINANET:
    USE_C5: False
  BACKBONE:
    CONV_BODY: "R-50-FPN-RETINANET"
  SIPMASK:
    NORM_REG_TARGETS: True
    CENTERNESS_ON_REG: True
INPUT:
  MIN_SIZE_TEST: 800
  MAX_SIZE_TEST: 1333
DATALOADER:
  SIZE_DIVISIBILITY: 32
"""
CFG = dict(nms_pre=1000, score_thr=0.05, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)


def _mask_rle(m):
    from sipmask_b200 import rle
    e = rle.encode(m)
    return {'size': e['size'], 'counts': e['counts'].decode()}


def _write_images(root, sizes, seed):
    import cv2
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_gpu_stream import _raw_images
    imgs = _raw_images(sizes, seed)
    names = []
    for n, img in enumerate(imgs):
        name = 'img_%03d.png' % n
        cv2.imwrite(os.path.join(root, name), img.numpy())
        names.append(name)
    return names


def _coco(tmp, n_img=40, n_cat=80, seed=0):
    """PNG images and an annotation json: boxes as polygons, compressed and uncompressed RLE, crowds."""
    from sipmask_b200 import rle
    rs = np.random.RandomState(seed)
    sizes = [SIZES[i] for i in rs.randint(0, len(SIZES), n_img)]
    img_dir = os.path.join(tmp, 'images')
    os.makedirs(img_dir, exist_ok=True)
    names = _write_images(img_dir, sizes, seed)
    ann = dict(images=[], categories=[dict(id=c + 1, name='cat%d' % (c + 1), supercategory='s%d' % (c % 3))
                                      for c in range(n_cat)], annotations=[])
    aid = 0
    for i, ((h, w), name) in enumerate(zip(sizes, names)):
        ann['images'].append(dict(id=100 + 3 * i, file_name=name, height=h, width=w))
        for _ in range(rs.randint(0, 6)):
            aid += 1
            x0, y0 = rs.randint(0, w - 40), rs.randint(0, h - 40)
            x1, y1 = x0 + rs.randint(20, min(200, w - x0) + 1), y0 + rs.randint(20, min(200, h - y0) + 1)
            m = np.zeros((h, w), bool)
            m[y0:y1, x0:x1] = True
            kind = aid % 3
            seg = ([[x0, y0, x0, y1, x1, y1, x1, y0]] if kind == 0 else _mask_rle(m) if kind == 1
                   else {'size': [h, w], 'counts': rle.counts(m).tolist()})
            ann['annotations'].append(dict(id=aid, image_id=100 + 3 * i, category_id=int(rs.randint(1, 6)),
                                           bbox=[float(x0), float(y0), float(x1 - x0), float(y1 - y0)],
                                           area=float(m.sum()), iscrowd=int(aid % 13 == 0), segmentation=seg))
    path = os.path.join(tmp, 'ann.json')
    with open(path, 'w') as f:
        json.dump(ann, f)
    return ann, path, img_dir


def _ytvis(tmp, seed=1):
    """Three PNG videos of mixed sizes and a YouTube-VIS annotation json."""
    rs = np.random.RandomState(seed)
    ann = dict(videos=[], categories=[dict(id=c) for c in range(1, 41)], annotations=[])
    root = os.path.join(tmp, 'frames')
    for v, ((h, w), nf) in enumerate((((360, 640), 4), ((480, 640), 3), ((400, 600), 3))):
        d = os.path.join(root, 'v%d' % v)
        os.makedirs(d)
        names = _write_images(d, [(h, w)] * nf, seed + v)
        ann['videos'].append(dict(id=v + 1, height=h, width=w, length=nf, file_names=['v%d/%s' % (v, n) for n in names]))
        m = np.zeros((h, w), bool)
        m[50:150, 60:200] = True
        ann['annotations'].append(dict(id=v + 1, video_id=v + 1, category_id=int(rs.randint(1, 41)), iscrowd=0,
                                       segmentations=[_mask_rle(m)] * nf, areas=[int(m.sum())] * nf))
    path = os.path.join(tmp, 'vis.json')
    with open(path, 'w') as f:
        json.dump(ann, f)
    return ann, path, root


def _tree(name, tmp, ann_path, prefix):
    """(config path, checkpoint path, state dict, hand-configured runner kwargs) of one tree."""
    from sipmask_b200 import benchmark as B, synth
    if name == 'bm':
        path = os.path.join(tmp, 'bm.yaml')
        with open(path, 'w') as f:
            f.write(BM_YAML)
        bm = B.synthetic_state_dict(depth=50, cls_bias=-2.5)
        ck = os.path.join(tmp, 'bm.pth')
        torch.save(dict(model={'module.' + k: v for k, v in bm.items()}), ck)
        return path, ck, B.convert_state_dict(bm), dict(benchmark=True, raw=True, depth=50, in_flight=6)
    if name == 'gn':
        sd = synth.detector_state_dict(50, stacked_convs=4, gn=True, cls_bias=-2.5)
        text = MODEL.format(dcn='', ncls=81, stacked=4, head='', nms_pre=1000, thr=0.05, mpi=100)
        text += MM_DATA.format(scale=(1333, 800), keep=True, ann=ann_path, prefix=prefix)
        hand = dict(in_flight=6, resize=(1333, 800), keep_ratio=True, depth=50, stacked_convs=4, gn=True, test_cfg=CFG)
    elif name == 'ssd':
        sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, rescoring_flag=True, backbone_dcn=True,
                                       cls_bias=-2.5)
        dcn = (", dcn=dict(type='DCN', deformable_groups=1, fallback_on_stride=False), "
               "stage_with_dcn=(False, True, True, True)")
        text = MODEL.format(dcn=dcn, ncls=81, stacked=2, head=', ssd_flag=True, norm_cfg=None, rescoring_flag=True',
                            nms_pre=1000, thr=0.1, mpi=100)
        text += MM_DATA.format(scale=(544, 544), keep=False, ann=ann_path, prefix=prefix)
        hand = dict(batch=32, in_flight=1, resize=(544, 544), keep_ratio=False, depth=50, stacked_convs=2, gn=False,
                    ssd_flag=True, backbone_dcn=True, rescoring_flag=True, test_cfg=dict(CFG, score_thr=0.1))
    else:
        sd = {}
        sd.update(synth.backbone_state_dict(50, 1))
        sd.update(synth.neck_state_dict(2))
        sd.update(synth.head_state_dict(3, num_classes=41, stacked_convs=3, gn=True, cls_bias=-2.5, track=True))
        text = MODEL.format(dcn='', ncls=41, stacked=3, head='', nms_pre=200, thr=0.03, mpi=10)
        text += VIS_DATA.format(ann=ann_path, prefix=prefix)
        hand = dict(resize=(640, 360), keep_ratio=True)          # VideoRunner's defaults are the VIS test settings
    path = os.path.join(tmp, name + '.py')
    with open(path, 'w') as f:
        f.write(text)
    ck = os.path.join(tmp, name + '.pth')
    torch.save(dict(state_dict={'module.' + k: v for k, v in sd.items()}, meta=dict(CLASSES=None)), ck)
    return path, ck, sd, hand


def _tool():
    import importlib.util
    spec = importlib.util.spec_from_file_location('smb_test_tool', os.path.join(ROOT, 'tools', 'test.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def _decode(path, rgb):
    import cv2
    from PIL import Image
    if rgb:
        return torch.from_numpy(np.asarray(Image.open(path).convert('RGB')).copy())
    return torch.from_numpy(cv2.imread(path, cv2.IMREAD_COLOR))


def _same_eval(a, b):
    skip = ('arrays', 'stats', 'analysis', 'classwise')
    assert {k: v for k, v in a.items() if k not in skip} == {k: v for k, v in b.items() if k not in skip}
    for m in b['arrays']:
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(a['arrays'][m][key], b['arrays'][m][key]), (m, key)
        assert np.array_equal(a['stats'][m], b['stats'][m])


def _coco_pass(runner, ann, img_dir, rgb, ids=True):
    """Every image of `ann` through the runner, one at a time (result after each submit); the records' host copies."""
    recs = []
    for im in ann['images']:
        img = _decode(os.path.join(img_dir, im['file_name']), rgb).pin_memory()
        t = runner.submit(img, im['id']) if ids else runner.submit(img)
        if runner.B > 1:
            runner.flush()
        r = runner.result(t)
        recs.append({k: (v.clone() if torch.is_tensor(v) else v) for k, v in r.items()})
    return recs


def _same_records(a, b):
    assert len(a) == len(b)
    for ra, rb in zip(a, b):
        for k in ('det_bboxes', 'det_labels', 'count', 'mask_scores'):
            if k in rb:
                assert torch.equal(ra[k], rb[k]), k
        assert ra['segms'] == rb['segms']


@pytest.fixture(scope='module')
def coco_data(tmp_path_factory):
    tmp = str(tmp_path_factory.mktemp('coco'))
    return (tmp,) + _coco(tmp)


def _with_detections(ann, recs, cat_ids, benchmark):
    """`ann` plus ground truth made of every other detection of a first pass (its RLE, or its box as a polygon; some
    crowds), so that the evaluation matches something."""
    from sipmask_b200 import coco
    out = dict(ann, annotations=list(ann['annotations']))
    aid = 10000
    for im, r in zip(ann['images'], recs):
        bj, sj = coco.coco_json(r, im['id'], cat_ids, benchmark=benchmark)
        for b, sg in list(zip(bj, sj))[::2]:
            aid += 1
            x, y, w, h = b['bbox']
            seg = sg['segmentation'] if aid % 3 else [[x, y, x, y + h, x + w, y + h, x + w, y]]
            out['annotations'].append(dict(id=aid, image_id=im['id'], category_id=b['category_id'], bbox=b['bbox'],
                                           area=float(w * h), iscrowd=int(aid % 11 == 0), segmentation=seg))
    return out


@pytest.mark.parametrize('name', ['gn', 'ssd', 'bm'])
def test_from_config_and_tool_equal_hand_configured_runner(coco_data, name):
    from sipmask_b200 import cocoeval, config as C
    from sipmask_b200.serving import CocoEvalRunner, StreamRunner
    tool = _tool()
    tmp, ann, _, img_dir = coco_data
    rgb = name == 'bm'
    cat_ids = [c['id'] for c in ann['categories']]
    hw = (max(im['height'] for im in ann['images']), max(im['width'] for im in ann['images']))
    common = dict(max_src_hw=hw, max_ori_hw=hw, masks='rle')
    ann_path = os.path.join(tmp, name + '_ann.json')
    cfg_path, ck, sd, hand = _tree(name, tmp, ann_path, img_dir)
    first = _coco_pass(StreamRunner(sd, render=not rgb, **common, **hand), ann, img_dir, rgb, ids=False)
    ann = _with_detections(ann, first, cat_ids, rgb)
    with open(ann_path, 'w') as f:
        json.dump(ann, f)
    gt = cocoeval.CocoGroundTruth(ann)
    ref_runner = CocoEvalRunner(sd, gt, cat_ids, **common, **hand)
    ref_recs = _coco_pass(ref_runner, ann, img_dir, rgb)
    _same_records(ref_recs, first)
    ref = ref_runner.evaluate()
    assert ref['bbox_mAP'] > 0.05 and ref['segm_mAP'] > 0.05, ref['bbox_mAP_copypaste']
    del ref_runner
    cfg = C.load_config(cfg_path)
    runner = C.from_config(cfg, ck, 'coco_eval', gt=gt, cat_ids=cat_ids, **common)
    assert runner.B == hand.get('batch', 1) and runner.n == hand['in_flight']
    _same_records(_coco_pass(runner, ann, img_dir, rgb), ref_recs)
    _same_eval(runner.evaluate(), ref)
    del runner
    assert sum(int(r['count'][0]) for r in ref_recs) > 0
    out = os.path.join(tmp, name + '_res')
    got = tool.main([cfg_path, ck, '--eval', 'bbox', 'segm', '--json-out', out, '--options', 'classwise=True']
                    + (['--ann', ann_path, '--img-prefix', img_dir] if name == 'bm'
                       else ['--out', out + '.pkl', '--show-dir', out + '_show']))
    _same_eval(got, ref)
    assert [n for n, _ in got['classwise']['bbox']] == ['cat%d' % c for c in cat_ids]
    from sipmask_b200 import coco
    bbox = [e for im, r in zip(ann['images'], ref_recs) for e in coco.coco_json(r, im['id'], cat_ids, benchmark=rgb)[0]]
    with open(out + '.bbox.json') as f:
        assert json.load(f) == json.loads(json.dumps(bbox))
    if name != 'bm':
        import pickle
        with open(out + '.pkl', 'rb') as f:
            res = pickle.load(f)
        assert len(res) == len(ann['images'])
        for (boxes, segs), r in zip(res, ref_recs):
            # bbox2result / get_seg_masks: per label, the detections of that label in record order
            k = int(r['count'][0])
            det, lab = r['det_bboxes'][:k].numpy(), r['det_labels'][:k].numpy().tolist()
            rows = [[j for j in range(k) if lab[j] == c] for c in range(80)]
            assert len(boxes) == 80 and all(b.dtype == np.float32 and np.array_equal(b, det[rw].reshape(-1, 5))
                                            for b, rw in zip(boxes, rows))
            masks = segs[0] if name == 'ssd' else segs
            assert masks == [[r['segms'][j] for j in rw] for rw in rows]
            if name == 'ssd':
                ms = r['mask_scores'][:k].numpy()
                assert all(np.array_equal(a, ms[rw]) for a, rw in zip(segs[1], rows))
        # --show-dir: the drawing of each image, as a render=True runner returns it
        import cv2
        for im, r in zip(ann['images'], first):
            drawn = cv2.imread(os.path.join(out + '_show', im['file_name']), cv2.IMREAD_COLOR)
            assert np.array_equal(drawn, r['render'].numpy()), im['file_name']


def test_vis_from_config_and_tool(tmp_path):
    from sipmask_b200 import config as C, ytviseval
    from sipmask_b200.serving import VideoEvalRunner
    tool = _tool()
    tmp = str(tmp_path)
    ann, ann_path, root = _ytvis(tmp)
    cfg_path, ck, sd, hand = _tree('vis', tmp, ann_path, root)

    def run(runner):
        frames = []
        for v in ann['videos']:
            for f, name in enumerate(v['file_names']):
                t = runner.submit(_decode(os.path.join(root, name), False).pin_memory(), v['id'], f)
                frames.append(runner.result(t)['frame'])
            runner.end_video(v['id'])
        res = runner.evaluate()
        return frames, res, [e for v in ann['videos'] for e in runner.video_json(v['id'])]

    hw = (480, 640)
    ref_frames, ref, ref_json = run(VideoEvalRunner(sd, ytviseval.YtvisGroundTruth(ann), max_src_hw=hw, **hand))
    got_frames, got, got_json = run(C.from_config(C.load_config(cfg_path), ck, 'video_eval',
                                                  gt=ytviseval.YtvisGroundTruth(ann), max_src_hw=hw))
    assert got_json == ref_json and len(got_frames) == len(ref_frames)
    for a, b in zip(got_frames, ref_frames):
        assert all(np.array_equal(x, y) for x, y in zip(a[0], b[0])) and a[1] == b[1]
    assert {k: v for k, v in got.items() if k not in ('arrays', 'stats')} == \
        {k: v for k, v in ref.items() if k not in ('arrays', 'stats')}
    out = os.path.join(tmp, 'vis_res')
    res = tool.main([cfg_path, ck, '--eval', 'segm', '--json-out', out])
    with open(out + '.json') as f:
        assert json.load(f) == json.loads(json.dumps(ref_json))
    assert {k: v for k, v in res.items() if k not in ('arrays', 'stats')} == \
           {k: v for k, v in ref.items() if k not in ('arrays', 'stats')}


def test_merged_halves_equal_one_evaluator():
    sys.path.insert(0, os.path.join(ROOT, 'tests'))
    from test_gpu_cocoeval import random_dataset
    from sipmask_b200 import cocoeval as E, dist as D
    gt, bbox, segm = random_dataset(7, n_img=12, big=True)
    for c in gt['categories']:
        c['supercategory'] = 's%d' % (c['id'] % 2)
    g = E.CocoGroundTruth(gt)

    def evaluator(ids):
        ev = E.CocoEvaluator(g, g.cat_ids, analyze=True)
        ids = ev._claim(ids)
        for m, res in (('bbox', bbox), ('segm', segm)):
            per = [(i, [r for r in res if r['image_id'] == i]) for i in ids]
            ev.add_results(per, m)
            ev.n_results[m] += sum(len(v) for _, v in per)
        ev.image_ids += ids
        ev._seen.update(ids)
        return ev

    ids = g.img_ids
    one = evaluator(ids).evaluate()
    halves = [evaluator(ids[0::2]), evaluator(ids[1::2])]
    merged = E.CocoEvaluator(g, g.cat_ids, analyze=True)
    merged.merge([D.gather_eval_state(h)[0] for h in halves])
    got = merged.evaluate()
    _same_eval(got, one)
    for m in ('bbox', 'segm'):
        assert np.array_equal(got['analysis'][m], one['analysis'][m]), m
