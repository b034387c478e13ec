"""Throughput of tools/test.py against the runner it drives, on a seeded synthetic COCO-format set.

Writes `--images` JPEG files of COCO-like sizes, an annotation json (one box polygon per image) and a synthetic
mmcv-format checkpoint into a temporary directory, then reports images/s of
  - tool   : tools/test.py CONFIG CHECKPOINT --eval bbox segm (checkpoint, build, host decode by its thread pool, run,
             evaluate), and
  - runner : CocoEvalRunner of the same settings fed the images already decoded and pinned (build, run, evaluate),
each after one untimed warm-up pass of the same command, with the card's name and power limit.  With --eval only, the
tool reads no record back (nothing consumes them); the difference is the host decode and the checkpoint load.

    python tools/time_test_tool.py --config ssd --images 512 --workers 8
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SIZES = [(480, 640), (427, 640), (640, 480), (375, 500), (640, 427), (333, 500)]
CONFIGS = {
    'ssd': dict(head=", stacked_convs=2, ssd_flag=True, norm_cfg=None", scale='(544, 544)', keep=False, thr=0.1,
                synth=dict(stacked_convs=2, gn=False)),
    'gn': dict(head=", stacked_convs=4", scale='(1333, 800)', keep=True, thr=0.05, synth=dict(stacked_convs=4, gn=True)),
}
TEXT = """model = dict(type='SipMask',
    backbone=dict(type='ResNet', depth=50, norm_cfg=dict(type='BN', requires_grad=False), style='caffe'),
    neck=dict(type='FPN', in_channels=[256, 512, 1024, 2048], out_channels=256, start_level=1, add_extra_convs=True,
              extra_convs_on_inputs=False, num_outs=5, relu_before_extra_convs=True),
    bbox_head=dict(type='SipMaskHead', num_classes=81, strides=[8, 16, 32, 64, 128]{head}))
test_cfg = dict(nms_pre=1000, min_bbox_size=0, score_thr={thr}, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
img_norm_cfg = dict(mean=[102.9801, 115.9465, 122.7717], std=[1.0, 1.0, 1.0], to_rgb=False)
test_pipeline = [dict(type='LoadImageFromFile'),
    dict(type='MultiScaleFlipAug', img_scale={scale}, flip=False,
         transforms=[dict(type='Resize', keep_ratio={keep}), dict(type='Normalize', **img_norm_cfg),
                     dict(type='Pad', size_divisor=32), dict(type='ImageToTensor', keys=['img']),
                     dict(type='Collect', keys=['img'])])]
data = dict(test=dict(type='CocoDataset', ann_file='{ann}', img_prefix='{prefix}', pipeline=test_pipeline))
"""


def dataset(tmp, n, seed=0):
    import cv2
    rs = np.random.RandomState(seed)
    ann = dict(images=[], categories=[dict(id=c + 1, name=str(c + 1)) for c in range(80)], annotations=[])
    img_dir = os.path.join(tmp, 'images')
    os.makedirs(img_dir)
    for i in range(n):
        h, w = SIZES[rs.randint(len(SIZES))]
        base = rs.randint(0, 256, (h // 16 + 2, w // 16 + 2, 3)).astype(np.uint8)
        img = cv2.resize(base, (w, h), interpolation=cv2.INTER_LINEAR)
        img = np.clip(img.astype(np.int16) + rs.randint(-20, 21, img.shape), 0, 255).astype(np.uint8)
        name = '%06d.jpg' % i
        cv2.imwrite(os.path.join(img_dir, name), img, [cv2.IMWRITE_JPEG_QUALITY, 90])
        ann['images'].append(dict(id=i + 1, file_name=name, height=h, width=w))
        x, y = rs.randint(0, w // 2), rs.randint(0, h // 2)
        ann['annotations'].append(dict(id=i + 1, image_id=i + 1, category_id=int(rs.randint(1, 81)), iscrowd=0,
                                       bbox=[x, y, 100, 80], area=8000.0,
                                       segmentation=[[x, y, x, y + 80, x + 100, y + 80, x + 100, y]]))
    path = os.path.join(tmp, 'ann.json')
    with open(path, 'w') as f:
        json.dump(ann, f)
    return ann, path, img_dir


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader', '-i', '0'],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = 'unknown'
    return name, limit


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--config', choices=sorted(CONFIGS), default='ssd')
    ap.add_argument('--images', type=int, default=512)
    ap.add_argument('--workers', type=int, default=8)
    args = ap.parse_args()
    assert torch.cuda.is_available(), 'time_test_tool.py needs a GPU'
    import cv2
    from sipmask_b200 import cocoeval, config as C, synth
    spec = importlib.util.spec_from_file_location('smb_test_tool', os.path.join(ROOT, 'tools', 'test.py'))
    tool = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(tool)
    c = CONFIGS[args.config]
    with tempfile.TemporaryDirectory() as tmp:
        ann, ann_path, img_dir = dataset(tmp, args.images)
        cfg_path = os.path.join(tmp, 'cfg.py')
        with open(cfg_path, 'w') as f:
            f.write(TEXT.format(head=c['head'], scale=c['scale'], keep=c['keep'], thr=c['thr'], ann=ann_path,
                                prefix=img_dir))
        ck = os.path.join(tmp, 'ck.pth')
        torch.save(dict(state_dict=synth.detector_state_dict(50, cls_bias=-2.5, **c['synth'])), ck)
        argv = [cfg_path, ck, '--eval', 'bbox', 'segm', '--workers', str(args.workers)]
        out = {}
        for _ in range(2):                                   # warm-up, then timed
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = tool.main(argv)
            torch.cuda.synchronize()
            out['tool_img_s'] = args.images / (time.perf_counter() - t0)
        cfg = C.load_config(cfg_path)
        ckpt = C.load_checkpoint(ck, cfg)
        imgs = [torch.from_numpy(cv2.imread(os.path.join(img_dir, im['file_name']))).pin_memory() for im in ann['images']]
        hw = (max(im['height'] for im in ann['images']), max(im['width'] for im in ann['images']))
        gt = cocoeval.CocoGroundTruth(ann)
        cat_ids = [cc['id'] for cc in ann['categories']]
        for _ in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            runner = C.from_config(cfg, ckpt, 'coco_eval', gt=gt, cat_ids=cat_ids, masks='rle', max_src_hw=hw,
                                   max_ori_hw=hw)
            for im, img in zip(ann['images'], imgs):
                runner.submit(img, im['id'])
            ref = runner.evaluate()
            torch.cuda.synchronize()
            out['runner_img_s'] = args.images / (time.perf_counter() - t0)
            del runner
        assert res['bbox_mAP_copypaste'] == ref['bbox_mAP_copypaste']
        name, limit = card()
        out.update(config=args.config, images=args.images, workers=args.workers, gpu=name, power_limit=limit,
                   cpus=os.cpu_count())
        print(json.dumps(out))


if __name__ == '__main__':
    main()
