"""Test a checkpoint from its reference config on the device: SipMask-mmdetection's tools/test.py (and dist_test.sh under
torchrun), SipMask-VIS's tools/test_video.py and SipMask-benchmark's test_net.py as one command.

    python tools/test.py CONFIG CHECKPOINT --ann ANN --img-prefix DIR [--eval bbox segm proposal]
        [--options classwise=True] [--out results.pkl] [--json-out PREFIX] [--show-dir DIR] [--launcher none|pytorch]
    torchrun --nproc_per_node 8 tools/test.py CONFIG CHECKPOINT --launcher pytorch --eval bbox segm

The config gives the engine and the test transform (sipmask_b200.config); images are read in the annotation file's
order and decoded on the host by a thread pool (cv2.imread, BGR, for mmdetection and SipMask-VIS configs; PIL
convert('RGB') for SipMask-benchmark ones), then resized, run, encoded and evaluated on the device.
  --out       the reference's per-image (bbox_results, segm_results): per class [k, 5] float32 arrays and RLE dicts,
              segm_results = (RLE lists, mask score arrays) for rescoring_flag configs; SipMask-VIS: the per-frame pairs
  --json-out  PREFIX.bbox.json and PREFIX.segm.json (results2json); SipMask-VIS: PREFIX.json (results2json_videoseg)
  --eval      prints MM's evaluate() dict (SipMask-VIS: 'segm', ytvos_eval's)
  --show-dir  each image drawn with its detections, under its file name (not for SipMask-benchmark configs)
Under --launcher pytorch rank r takes images r, r + world, ... (DistributedSampler without shuffling); each rank
evaluates its images on its own device and, once at the end, the evaluation state and the results are gathered
(sizes, then padded bytes) and rank 0 evaluates and writes in dataset order.  SipMask-VIS runs on one GPU, as
test_video.py does.
"""
import argparse
import collections
import json
import os
import pickle
import sys
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def parse_args(argv=None):
    p = argparse.ArgumentParser(description='Test (and evaluate) a SipMask checkpoint on the device')
    p.add_argument('config')
    p.add_argument('checkpoint')
    p.add_argument('--ann', help='annotation json (default: the config\'s data.test.ann_file)')
    p.add_argument('--img-prefix', help='image directory (default: the config\'s data.test.img_prefix)')
    p.add_argument('--eval', nargs='+', default=[], help="'bbox', 'segm', 'proposal' (SipMask-VIS: 'segm')")
    p.add_argument('--options', nargs='+', default=[], help='evaluate() arguments, KEY=VALUE: classwise=True')
    p.add_argument('--out', help='pickle of the per-image results')
    p.add_argument('--json-out', help='prefix of the result json files')
    p.add_argument('--show-dir', help='directory of the drawn images')
    p.add_argument('--launcher', choices=['none', 'pytorch'], default='none')
    p.add_argument('--workers', type=int, default=8, help='host decode threads')
    p.add_argument('--local_rank', '--local-rank', type=int, default=0)
    return p.parse_args(argv)


def _options(kvs):
    """MultipleKVAction's parsing (int, float, true / false); the one key evaluate() takes here is classwise."""
    out = {}
    for kv in kvs:
        if '=' not in kv:
            raise ValueError('--options %r: KEY=VALUE expected' % kv)
        key, val = kv.split('=', 1)
        if key != 'classwise':
            raise ValueError('--options %s: only classwise is supported' % key)
        if val.lower() not in ('true', 'false'):
            raise ValueError('--options classwise=%s: True or False' % val)
        out[key] = val.lower() == 'true'
    return out


def _decode(path, rgb):
    if rgb:
        from PIL import Image
        with Image.open(path) as im:
            arr = np.array(im.convert('RGB'))
    else:
        import cv2
        arr = cv2.imread(path, cv2.IMREAD_COLOR)
        if arr is None:
            raise FileNotFoundError('cannot read image %s' % path)
    return torch.from_numpy(np.ascontiguousarray(arr))


def _decoded(paths, rgb, workers):
    """The decoded images of `paths` in order, in pinned memory, decoded ahead by a pool of `workers` threads (a bounded
    window).  The pinning happens here, on the caller's thread: pinning allocates through CUDA, and a CUDA allocation
    from another thread while the runner captures an engine's CUDA graph (on its first forward) invalidates the capture."""
    with ThreadPoolExecutor(max_workers=max(1, workers)) as pool:
        window = collections.deque()
        it = iter(paths)
        for p in it:
            window.append(pool.submit(_decode, p, rgb))
            if len(window) >= 4 * max(1, workers):
                break
        for p in it:
            yield window.popleft().result().pin_memory()
            window.append(pool.submit(_decode, p, rgb))
        while window:
            yield window.popleft().result().pin_memory()


class _Reader:
    """Reads every image's record from the runner before its slot is reused: batch b runs in slot b % in_flight, and the
    next submit may dispatch into the slot of batch dispatched + 1 - in_flight.  fn=None: nothing consumes the records
    (evaluation only), so none is waited for or read."""

    def __init__(self, runner, fn):
        self.runner, self.fn, self.fifo, self.seen = runner, fn, collections.deque(), 0

    def before_submit(self):
        if self.fn is None:
            return
        self._register()
        r = self.runner
        while self.fifo and self.seen - len(self.fifo) <= r.dispatched + 1 - r.n:
            self._read(self.fifo.popleft())

    def drain(self):
        if self.fn is None:
            return
        self._register()
        while self.fifo:
            self._read(self.fifo.popleft())

    def _register(self):
        r = self.runner
        for b in range(self.seen, r.dispatched):
            self.fifo.append((b % r.n, [m['ticket'] for m in r.slot_images[b % r.n]]))
        self.seen = r.dispatched

    def _read(self, batch):
        from sipmask_b200.serving import VideoRunner
        r = self.runner
        slot, tickets = batch
        for t in tickets:           # StreamRunner.result takes the slot at batch 1, VideoRunner.result always the ticket
            self.fn(t, r.result(slot if r.B == 1 and not isinstance(r, VideoRunner) else t))


def _per_class(rec, ncls, rescoring):
    """One record as the reference's (bbox_results, segm_results) of one image."""
    k = int(rec['count'].reshape(-1)[0])
    det = rec['det_bboxes'][:k].numpy().astype(np.float32)
    labels = rec['det_labels'][:k].numpy()
    segms = rec['segms']
    bbox = [det[labels == i] for i in range(ncls)]
    segm = [[segms[j] for j in np.flatnonzero(labels == i)] for i in range(ncls)]
    if rescoring:
        ms = rec['mask_scores'][:k].numpy().astype(np.float32)
        return bbox, (segm, [ms[labels == i] for i in range(ncls)])
    return bbox, segm


def _dist_init(args):
    if args.launcher == 'none':
        return 0, 1
    import torch.distributed as dist
    local = int(os.environ.get('LOCAL_RANK', args.local_rank))
    torch.cuda.set_device(local)
    dist.init_process_group('nccl')
    return dist.get_rank(), dist.get_world_size()


def _gather_results(items, world, dev):
    """[(dataset index, payload)] of every rank, in dataset order, on rank 0 (None elsewhere)."""
    if world == 1:
        return [p for _, p in sorted(items, key=lambda x: x[0])]
    import torch.distributed as dist
    from sipmask_b200 import dist as D
    parts = D.gather_bytes(pickle.dumps(items, protocol=pickle.HIGHEST_PROTOCOL), dev)
    if dist.get_rank() != 0:
        return None
    return [p for _, p in sorted((x for b in parts for x in pickle.loads(b)), key=lambda x: x[0])]


def _print_eval(res):
    for k, v in res.items():
        if k not in ('stats', 'arrays', 'analysis', 'classwise'):
            print('%s: %s' % (k, v))
    for m, table in res.get('classwise', {}).items():
        print('\n%s per-category AP' % m)
        print('%-24s %s' % ('category', 'AP'))
        for name, ap in table:
            print('%-24s %.3f' % (name, ap))


def _run_coco(args, cfg, ckpt, t, rank, world, dev, opts):
    from sipmask_b200 import cocoeval, coco, config as C
    from sipmask_b200 import dist as D
    ek = C.engine_kwargs(cfg)
    bm = t == 'benchmark'
    if bm and args.out:
        raise ValueError('--out: SipMask-benchmark writes BoxList predictions; use --json-out for its results')
    with open(args.ann) as f:
        ann = json.load(f)
    images = ann['images']
    cat_ids = [int(c['id']) for c in ann['categories']]          # label i -> getCatIds()[i]
    if len(cat_ids) != ek['num_classes'] - 1:
        raise ValueError('%s has %d categories; the config\'s detector %d classes' % (args.ann, len(cat_ids),
                                                                                    ek['num_classes'] - 1))
    mine = list(range(rank, len(images), world))
    hw = (max(int(im['height']) for im in images), max(int(im['width']) for im in images))
    kw = dict(masks='rle', max_src_hw=hw, max_ori_hw=hw, device=dev, render=bool(args.show_dir))
    if args.eval:
        runner = C.from_config(cfg, ckpt, 'coco_eval', gt=cocoeval.CocoGroundTruth(ann), cat_ids=cat_ids,
                               metrics=list(args.eval), **kw)
    else:
        runner = C.from_config(cfg, ckpt, 'stream', **kw)
    index = {}                                  # ticket -> dataset index
    items = []

    def keep(ticket, rec):
        i = index.pop(ticket)
        im = images[i]
        payload = {}
        if args.json_out:
            payload['json'] = coco.coco_json(rec, int(im['id']), cat_ids, benchmark=bm)
        if args.out:
            payload['out'] = _per_class(rec, ek['num_classes'] - 1, ek.get('rescoring_flag', False))
        if args.show_dir:
            import cv2
            path = os.path.join(args.show_dir, im['file_name'])
            os.makedirs(os.path.dirname(path), exist_ok=True)
            cv2.imwrite(path, rec['render'].numpy())
        items.append((i, payload))

    reader = _Reader(runner, keep if args.json_out or args.out or args.show_dir else None)
    paths = [os.path.join(args.img_prefix, images[i]['file_name']) for i in mine]
    for i, img in zip(mine, _decoded(paths, bm, args.workers)):
        reader.before_submit()
        index[runner.i] = i
        if args.eval:
            runner.submit(img, int(images[i]['id']))
        else:
            runner.submit(img)
    if args.eval:
        runner.finish()
    else:
        runner.flush()
    reader.drain()
    res = None
    if args.eval:
        ev = runner.evaluator
        if world > 1:
            states = D.gather_eval_state(ev)
            if rank == 0:
                ev.merge([s for r, s in enumerate(states) if r != rank])
        if rank == 0:
            res = ev.evaluate(opts.get('classwise', False))
    if args.out or args.json_out:
        merged = _gather_results(items, world, dev)
        if rank == 0:
            if args.out:
                with open(args.out, 'wb') as f:
                    pickle.dump([p['out'] for p in merged], f)
            if args.json_out:
                for n, name in enumerate(('bbox', 'segm')):
                    with open('%s.%s.json' % (args.json_out, name), 'w') as f:
                        json.dump([e for p in merged for e in p['json'][n]], f)
    return res


def _run_vis(args, cfg, ckpt, world, dev):
    from sipmask_b200 import config as C, ytviseval
    if world != 1:
        raise ValueError('SipMask-VIS configs run on one GPU (test_video.py asserts gpus == 1)')
    if any(m != 'segm' for m in args.eval):
        raise ValueError("--eval %s: YouTube-VIS evaluates 'segm'" % ' '.join(args.eval))
    with open(args.ann) as f:
        ann = json.load(f)
    videos = ann['videos']
    hw = (max(int(v['height']) for v in videos), max(int(v['width']) for v in videos))
    kw = dict(max_src_hw=hw, max_ori_hw=hw, device=dev, render=bool(args.show_dir))
    if args.eval:
        runner = C.from_config(cfg, ckpt, 'video_eval', gt=ytviseval.YtvisGroundTruth(ann), **kw)
    else:
        runner = C.from_config(cfg, ckpt, 'video', **kw)
    where, frames = {}, {}

    def keep(ticket, rec):
        v, f = where.pop(ticket)
        frames[(v, f)] = rec['frame']
        if args.show_dir:
            import cv2
            path = os.path.join(args.show_dir, videos[v]['file_names'][f])
            os.makedirs(os.path.dirname(path), exist_ok=True)
            cv2.imwrite(path, rec['render'].numpy())

    reader = _Reader(runner, keep if args.out or args.show_dir else None)
    order = [(v, f) for v, vid in enumerate(videos) for f in range(len(vid['file_names']))]
    paths = [os.path.join(args.img_prefix, videos[v]['file_names'][f]) for v, f in order]
    for (v, f), img in zip(order, _decoded(paths, False, args.workers)):
        reader.before_submit()
        where[runner.i] = (v, f)
        runner.submit(img, videos[v]['id'], f)
        if f == len(videos[v]['file_names']) - 1:
            runner.end_video(videos[v]['id'])
    runner.flush()
    reader.drain()
    res = runner.evaluate() if args.eval else None
    results = [e for vid in videos for e in runner.video_json(vid['id'])]
    if args.out:
        with open(args.out, 'wb') as f:
            pickle.dump([frames[k] for k in order], f)
    if args.json_out:
        with open(args.json_out + '.json', 'w') as f:
            json.dump(results, f)
    return res


def main(argv=None):
    """Runs the command; returns the evaluate() dict on rank 0 with --eval (None otherwise)."""
    args = parse_args(argv)
    from sipmask_b200 import config as C
    opts = _options(args.options)
    cfg = C.load_config(args.config)
    t = C.tree(cfg)
    if t != 'benchmark':
        args.ann = args.ann or C._get(cfg, 'data.test.ann_file')
        args.img_prefix = args.img_prefix or C._get(cfg, 'data.test.img_prefix')
    elif not (args.ann and args.img_prefix):
        raise ValueError('SipMask-benchmark configs name their datasets through fcos_core\'s paths catalog: give --ann '
                         'and --img-prefix')
    if t == 'benchmark' and 'proposal' in args.eval:
        raise ValueError("--eval proposal: SipMask-benchmark's evaluation never evaluates box proposals of SipMask")
    if args.show_dir and t == 'benchmark':
        raise ValueError('--show-dir: SipMask-benchmark runners do not render')
    rank, world = _dist_init(args)
    dev = torch.device('cuda', torch.cuda.current_device())
    ckpt = C.load_checkpoint(args.checkpoint, cfg)
    if t == 'vis':
        res = _run_vis(args, cfg, ckpt, world, dev)
    else:
        res = _run_coco(args, cfg, ckpt, t, rank, world, dev, opts)
    if res is not None:
        _print_eval(res)
    if world > 1:
        import torch.distributed as dist
        dist.barrier()
        dist.destroy_process_group()
    return res


if __name__ == '__main__':
    main()
