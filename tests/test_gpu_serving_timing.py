"""The serving pipelines under adversarial stream timing (sipmask_b200.serving: EnginePool, PipelinedRunner,
StreamRunner, VideoRunner, CocoEvalRunner, VideoEvalRunner).

The slots of a pipeline are ordered only through events: the H2D stream, the D2H stream, one compute stream per slot,
the consumer's stream and the tracker stream.  On an idle GPU each stage is usually done long before the next one needs
it, so a missing wait goes unnoticed.  Here a bounded `torch.cuda._sleep` is enqueued at one seam of the pipeline at a
time (or at all of them), on the stream whose work a later stage must wait for:

  h2d            _Slots.upload, before the copy                     ev_in_ready (compute reads the new input)
  compute_start  _Slots.begin_compute, on the returned stream       ev_in_free (the next upload into the slot)
  compute_end    _Slots.publish, before the record (and before a    ev_out_ready (download, consumer, tracker); with
                 StreamRunner's drawing)                            render=True also ev_in_free
  d2h            _Slots.download, after its wait, before its copies ev_out_free (result(), the slot's next record)
  consumer       _Slots.hand_over, before work()                    ev_hold (the slot's next record)
  track          LaneTracker.associate, on the tracker stream       ev_assoc (the download), the slot's next record
  gt             CocoEvaluator.stage_gt, YtvisEvaluator.stage_frame, ev_in_ready of the batch that evaluates it
                 on the H2D stream
  eval           CocoEvaluator._match (each image's matches),       record_stream (the staged ground truth outlives its
                 YtvisEvaluator.overlap and .scatter                Python owner), ev_ovl (the scatter after the overlaps)

Every record must still equal, field by field (torch.equal), the record of the same image run serially (the same
runner configuration, one image at a time with a device synchronise after each).  The image sequences have a period
coprime to the slot count, so consecutive uses of a slot differ in content (and, for StreamRunner, in padded shape): a
stale input or output cannot have the right bytes.  Each record read from pinned memory is then overwritten with 0xFF
bytes, so a read that comes too early finds poison rather than an older copy of the right answer.

Positive control: after each sleep an event is recorded on the delayed stream; when the work that depends on it is
enqueued, that event must be found incomplete at least once per case and stage, or the case fails (its delay opened no
window).  The delay is calibrated on the device: about three forwards of the case, at least 5 ms (so a host hiccup does
not close a window) and capped so the file stays short."""
import time

import pytest
import torch

pytestmark = pytest.mark.gpu

MIN_MS, CAP_MS = 5.0, 40.0          # shortest and longest single delay: longer than a host hiccup, short enough for the file
CYCLES_PROBE = 10 ** 6

# stage -> the seams that enqueue work which must wait for the delayed work.  Slot stages keep one event per slot (the
# slot's latest delayed work) and a seam of slot k checks slot k's; the others keep their latest event.
WATCH = dict(h2d=('begin_compute',), gt=('begin_compute',), compute_start=('claim_input',),
             compute_end=('download', 'await_record', 'claim_input'), d2h=('wait', 'claim_output'),
             consumer=('claim_output',), track=('download',), eval=('scatter', 'stage_gt', 'stage_frame', 'claim_input'))
SLOT_STAGES = frozenset(('compute_start', 'compute_end', 'd2h', 'consumer'))


class _Late(object):
    """The copy list of slot k's download: iterating it (inside download's D2H stream context, after its wait) first
    enqueues the d2h delay."""

    def __init__(self, delays, k, copies):
        self.delays, self.k, self.copies = delays, k, list(copies)

    def __iter__(self):
        self.delays.delay('d2h', k=self.k)
        return iter(self.copies)


class Delays(object):
    """Bounded device sleeps at the pipeline's seams (see the module docstring), installed with monkeypatch, and the
    positive control of each delayed stage."""

    def __init__(self, monkeypatch, stages, cycles):
        from sipmask_b200 import cocoeval as CE, serving as S, tracker as T, ytviseval as YE
        self.stages, self.cycles = frozenset(stages), int(cycles)
        self.last = {s: {} for s in self.stages}        # stage -> {slot (or None): the event after its latest sleep}
        self.opened = {s: 0 for s in self.stages}       # dependent enqueues that found that delayed work still running
        self.slept = {s: 0 for s in self.stages}
        d = self
        slots = S._Slots
        orig = {n: getattr(slots, n) for n in ('claim_input', 'upload', 'begin_compute', 'claim_output', 'publish',
                                               'await_record', 'download', 'hand_over', 'wait')}
        render_batch, associate = S.StreamRunner._render_batch, T.LaneTracker.associate
        match, stage_gt = CE.CocoEvaluator._match, CE.CocoEvaluator.stage_gt
        overlap, scatter, stage_frame = YE.YtvisEvaluator.overlap, YE.YtvisEvaluator.scatter, YE.YtvisEvaluator.stage_frame

        def claim_input(self, k):
            d.watch('claim_input', k)
            return orig['claim_input'](self, k)

        def upload(self, dst, src):
            d.delay('h2d', self.h2d)
            return orig['upload'](self, dst, src)

        def begin_compute(self, k):
            d.watch('begin_compute', k)
            cs = orig['begin_compute'](self, k)
            d.delay('compute_start', cs, k)
            return cs

        def claim_output(self, k, cs):
            d.watch('claim_output', k)
            return orig['claim_output'](self, k, cs)

        def publish(self, k, cs):
            d.delay('compute_end', cs, k)
            return orig['publish'](self, k, cs)

        def await_record(self, k, stream):
            d.watch('await_record', k)
            return orig['await_record'](self, k, stream)

        def download(self, k, copies, after=None):
            d.watch('download', k)
            return orig['download'](self, k, _Late(d, k, copies), after)

        def hand_over(self, k, work):
            def late():
                d.delay('consumer', k=k)
                return work()
            return orig['hand_over'](self, k, late)

        def wait(self, k):
            d.watch('wait', k)
            return orig['wait'](self, k)

        def _render_batch(self, k, eng, images, dev):
            d.delay('compute_end', k=k)
            return render_batch(self, k, eng, images, dev)

        def assoc(self, *args, **kwargs):
            d.delay('track')
            return associate(self, *args, **kwargs)

        def coco_stage_gt(self, image_id, stream=None, masks=None):
            d.watch('stage_gt')
            d.delay('gt', stream)
            return stage_gt(self, image_id, stream, masks)

        def coco_match(self, *args, **kwargs):
            # add_records uploads its image rows from pageable memory, which waits for the slot's stream on the host;
            # the matches it enqueues after that read the staged ground truth, and are what the delay holds back
            d.delay('eval')
            return match(self, *args, **kwargs)

        def ytvis_stage_frame(self, video_id, frame_id, stream=None):
            d.watch('stage_frame')
            d.delay('gt', stream)
            return stage_frame(self, video_id, frame_id, stream)

        def ytvis_overlap(self, *args, **kwargs):
            d.delay('eval')
            return overlap(self, *args, **kwargs)

        def ytvis_scatter(self, *args, **kwargs):
            d.watch('scatter')
            d.delay('eval')
            return scatter(self, *args, **kwargs)
        for name, fn in (('claim_input', claim_input), ('upload', upload), ('begin_compute', begin_compute),
                         ('claim_output', claim_output), ('publish', publish), ('await_record', await_record),
                         ('download', download), ('hand_over', hand_over), ('wait', wait)):
            monkeypatch.setattr(slots, name, fn)
        monkeypatch.setattr(S.StreamRunner, '_render_batch', _render_batch)
        monkeypatch.setattr(T.LaneTracker, 'associate', assoc)
        monkeypatch.setattr(CE.CocoEvaluator, 'stage_gt', coco_stage_gt)
        monkeypatch.setattr(CE.CocoEvaluator, '_match', coco_match)
        monkeypatch.setattr(YE.YtvisEvaluator, 'stage_frame', ytvis_stage_frame)
        monkeypatch.setattr(YE.YtvisEvaluator, 'overlap', ytvis_overlap)
        monkeypatch.setattr(YE.YtvisEvaluator, 'scatter', ytvis_scatter)

    def delay(self, stage, stream=None, k=None):
        if stage not in self.stages:
            return None
        st = stream if stream is not None else torch.cuda.current_stream()
        with torch.cuda.stream(st):
            torch.cuda._sleep(self.cycles)
            ev = torch.cuda.Event()
            ev.record(st)
        self.last[stage][k if stage in SLOT_STAGES else None] = ev
        self.slept[stage] += 1
        return ev

    def watch(self, seam, k=None):
        """Dependent work of slot k (or of no slot) is about to be enqueued at `seam`: is the delayed work it depends on
        still running?"""
        for s in self.stages:
            if seam in WATCH[s]:
                ev = self.last[s].get(k if s in SLOT_STAGES else None)
                self.opened[s] += ev is not None and not ev.query()

    def check(self):
        """Every delayed stage slept, and its delay was still running when dependent work was enqueued."""
        print('delay %d cycles; sleeps %s; windows found open %s' % (self.cycles, self.slept, self.opened))
        for s in self.stages:
            assert self.slept[s] > 0, 'stage %s never slept' % s
            assert self.opened[s] > 0, 'the %s delay opened no window: the case would pass vacuously' % s


_SLEEP = {}


def _ms_per_cycle():
    if not _SLEEP:
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(CYCLES_PROBE)
        a.record()
        torch.cuda._sleep(CYCLES_PROBE)
        b.record()
        b.synchronize()
        _SLEEP['ms'] = a.elapsed_time(b) / CYCLES_PROBE
    return _SLEEP['ms']


def _calibrate(name, forward):
    """Cycles of a delay about three times one serial forward (forward() ends in a device synchronise), within
    [MIN_MS, CAP_MS]."""
    forward()
    ts = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        forward()
        ts.append((time.perf_counter() - t0) * 1e3)
    fwd = min(ts)
    per = _ms_per_cycle()
    ms = min(max(3 * fwd, MIN_MS), CAP_MS)
    cycles = int(ms / per)
    print('%s: serial forward %.2f ms, _sleep(%d) %.3f ms -> delay %d cycles (%.2f ms)'
          % (name, fwd, CYCLES_PROBE, per * CYCLES_PROBE, cycles, cycles * per))
    return cycles


def _poison(*ts):
    for t in ts:
        if torch.is_tensor(t) and t.numel():
            t.reshape(-1).view(torch.uint8).fill_(255)


def _poison_record(rec):
    """The consumer's clone source: overwritten on the consumer's stream once cloned, so the slot's next forward (which
    waits for the consumer) must rewrite it, and a consumer that read it too late would find poison."""
    _poison(*[v for v in rec.values() if torch.is_tensor(v)])


def _slot_order(recs, slots, key=None):
    """An order of the PERIOD images in which the images a slot takes in turn (positions i and i + n, for n in `slots`)
    always differ in detection count and mask bits, and in key(image) when given (e.g. the padded shape)."""
    import itertools
    cnt = [int(r['count'].reshape(-1)[0]) for r in recs]
    differ = [[cnt[a] != cnt[b] and not torch.equal(recs[a]['mask_bits'], recs[b]['mask_bits'])
               and (key is None or key(a) != key(b)) for b in range(PERIOD)] for a in range(PERIOD)]
    for p in itertools.permutations(range(PERIOD)):
        if all(differ[p[i]][p[(i + n) % PERIOD]] for n in slots for i in range(PERIOD)):
            return list(p)
    raise AssertionError('no order of the images gives every slot different counts in turn: %s' % cnt)


def _poisoned(t):
    return bool((t.reshape(-1).view(torch.uint8) == 255).all())


def _cpu(rec):
    return {k: (v.cpu().clone() if torch.is_tensor(v) else v) for k, v in rec.items()}


# ------------------------------------------------------------------------------------ EnginePool, PipelinedRunner
H, W = 128, 192
IMG_SHAPE = (H, W - 5, 3)
PERIOD = 7                                  # images per sequence: coprime to 2 and 3 slots
# a score threshold inside the images' score range and max_per_img above what they reach, so the detection count
# differs from image to image (at score_thr=0.4 every image here keeps max_per_img)
CFG = dict(nms_pre=200, score_thr=0.5, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)


@pytest.fixture(scope='module')
def small():
    from sipmask_b200 import synth
    from sipmask_b200.serving import make_engines
    from test_gpu_stream import _raw_images
    sd = synth.detector_state_dict(depth=50, seed=1, cls_bias=-2.5)
    serial = make_engines(sd, (H, W), in_flight=1, test_cfg=CFG, img_shape=IMG_SHAPE, use_graph=True)[0]
    fp32 = [synth.synthetic_image(H, W, seed=40 + s) for s in range(PERIOD)]
    raw = _raw_images([IMG_SHAPE[:2]] * PERIOD, seed=41)
    want = dict(fp32=[], raw=[])
    for x in fp32:
        serial.forward(x.cuda())
        torch.cuda.synchronize()
        want['fp32'].append(_cpu(serial._result()))
    for x in raw:
        serial.forward_raw(x.cuda())
        torch.cuda.synchronize()
        want['raw'].append(_cpu(serial._result()))
    order = {}
    for k, w in want.items():
        order[k] = _slot_order(w, (2, 3))                 # 2 and 3 slots
        print('%s inputs: detections per image %s, order %s' % (k, [int(r['count'][0]) for r in w], order[k]))
    x0 = fp32[0].cuda()
    cycles = _calibrate('128x192 engine', lambda: (serial.forward(x0), torch.cuda.synchronize()))
    ori = serial.image_metas[0][1][:2]
    return dict(sd=sd, inputs=dict(fp32=[x.pin_memory() for x in fp32], raw=[x.pin_memory() for x in raw]), want=want,
                order=order, cycles=cycles, ori=ori, cache={})


def _engines(small, n, rle):
    from sipmask_b200.serving import make_engines
    key = ('engines', n, rle)
    if key not in small['cache']:
        kw = dict(rle_bytes=1 << 16) if rle else {}
        small['cache'][key] = make_engines(small['sd'], (H, W), in_flight=n, test_cfg=CFG, img_shape=IMG_SHAPE,
                                           use_graph=True, **kw)
    return small['cache'][key]


def _same_engine_record(got, want, keys=('det_bboxes', 'det_labels', 'count', 'mask_bits', 'idxs_keep')):
    for k in keys:
        if k in got:
            assert torch.equal(got[k].cpu(), want[k]), k


@pytest.mark.parametrize('stages', [(), ('compute_end',), ('consumer',), ('compute_end', 'consumer')],
                         ids=['none', 'compute_end', 'consumer', 'all'])
def test_engine_pool_consumer_records(small, monkeypatch, stages):
    """EnginePool, 3 engines: each launch's input is written on the engine's stream right before it (7 images over 3
    engines), and the consumer copies the device record as bench's RecordLog.append does."""
    from sipmask_b200.dist import RecordLog
    from sipmask_b200.serving import EnginePool
    engs = _engines(small, 3, False)
    pool = small['cache'].get('pool')
    if pool is None:
        pool = small['cache']['pool'] = EnginePool(engs)
    torch.cuda.synchronize()
    d = Delays(monkeypatch, stages, small['cycles'])
    seq = [small['order']['fp32'][i % PERIOD] for i in range(3 * PERIOD)]
    dev_in = [x.cuda() for x in small['inputs']['fp32']]
    log = RecordLog(len(seq), engs[0].max_num, engs[0].dev)
    got = []

    def fn(rec):
        got.append({k: v.clone() for k, v in rec.items()})
        log.append(rec['det_bboxes'][0], rec['det_labels'][0], rec['count'][0:1])
        _poison_record(rec)
    for i in seq:
        k = pool.i % pool.n
        with torch.cuda.stream(pool.streams[k]):        # after the engine's previous forward, before its next
            engs[k].img.copy_(dev_in[i], non_blocking=True)
        pool.step(fn)
    pool.flush(fn)
    torch.cuda.synchronize()
    assert len(got) == len(seq)
    buf = log.buf.cpu()
    for j, i in enumerate(seq):
        w = small['want']['fp32'][i]
        _same_engine_record(got[j], w)
        n = int(w['count'][0])
        assert torch.equal(buf[j, :, :5], w['det_bboxes'][0])
        assert torch.equal(buf[j, :, 5], w['det_labels'][0].float())
        assert buf[j, :, 6].tolist() == [1.0] * n + [0.0] * (buf.shape[1] - n)
    if stages:
        d.check()


PIPE_STAGES = ('h2d', 'compute_start', 'compute_end', 'd2h', 'consumer')


def _pipe_stage_params():
    return [pytest.param(s, id=n) for s, n in [((), 'none')] + [((x,), x) for x in PIPE_STAGES] + [(PIPE_STAGES, 'all')]]


def _pipelined_params():
    out = []
    for cfg, name in (((3, 2, 'fp32', 'bits'), '3eng-fp32-bits'), ((3, 2, 'raw', 'rle'), '3eng-raw-rle'),
                      ((1, 2, 'fp32', 'rle'), '1eng-depth2-fp32-rle'), ((1, 2, 'raw', 'bits'), '1eng-depth2-raw-bits')):
        # one engine with raw input: forward_raw waits on the host for its previous source-row copy, which follows the
        # previous forward on the one compute stream, so the next upload into a slot is already ordered after the
        # slot's forward and a compute_start delay cannot open a window there
        stages = tuple(s for s in PIPE_STAGES if not (cfg[0] == 1 and cfg[2] == 'raw' and s == 'compute_start'))
        for st, sn in [((), 'none')] + [((x,), x) for x in stages] + [(stages, 'all')]:
            out.append(pytest.param(*(cfg + (st,)), id='%s-%s' % (name, sn)))
    return out


@pytest.mark.parametrize('n,depth,inp,masks,stages', _pipelined_params())
def test_pipelined_runner_records(small, monkeypatch, n, depth, inp, masks, stages):
    """PipelinedRunner: a pass handing every record to a consumer (the host never blocks, so the uploads into a slot
    race its previous forward), then a pass reading every result() right before its slot is reused."""
    from sipmask_b200 import rle as RL
    from sipmask_b200.serving import PipelinedRunner
    key = ('pipe', n, depth, inp, masks)
    runner = small['cache'].get(key)
    if runner is None:
        engs = _engines(small, n, masks == 'rle')
        runner = small['cache'][key] = PipelinedRunner(engs, depth=depth, masks=masks,
                                                       raw_hw=IMG_SHAPE[:2] if inp == 'raw' else None)
        for t in runner.in_dev:                        # no uninitialized input is ever read
            t.zero_()
    torch.cuda.synchronize()
    inputs, want, ori = small['inputs'][inp], small['want'][inp], small['ori']
    d = Delays(monkeypatch, stages, small['cycles'])
    seq = [small['order'][inp][i % PERIOD] for i in range(2 * PERIOD)]

    # pass 1: consumer records (the downloads of this pass are not read, so the consumer may poison what it cloned)
    got = []

    def fn(rec):
        got.append({k: v.clone() for k, v in rec.items()})
        _poison_record(rec)
    for i in seq:
        runner.step(inputs[i], fn)
    runner.flush(fn)
    torch.cuda.synchronize()
    assert len(got) == len(seq)
    for j, i in enumerate(seq):
        _same_engine_record(got[j], want[i])

    # pass 2: result() inside its validity window, pinned records poisoned after each read
    for k in range(runner.nslots):
        _poison(*runner.out_host[k].values())
        if runner.rle:
            _poison(runner.rle_regions[k])
    early = []

    def read(j, k):
        w = want[seq[j]]
        r = runner.result(k)
        for name, key in (('det', 'det_bboxes'), ('lab', 'det_labels'), ('cnt', 'count'), ('bits', 'mask_bits')):
            if name in r:
                assert torch.equal(r[name], w[key]), (j, name)
        cnt = int(w['count'][0])
        if runner.rle:
            assert 'bits' not in r
            assert r['segms'] == [RL.encode_planes(w['mask_bits'][0, :cnt].numpy(), ori)], j
            _poison(runner.rle_regions[k])
        _poison(*runner.out_host[k].values())
    slots = []
    for j, i in enumerate(seq):
        if j >= runner.nslots:
            read(j - runner.nslots, slots[j - runner.nslots])
        k = runner.submit(inputs[i])
        slots.append(k)
        if 'd2h' in stages:
            # direct control: while the sleep in front of this download's copies is still running, the pinned record
            # holds the poison.  Looked at only when the sleep is seen running both before and after the look, so a
            # slow host skips a look instead of failing it.
            ev = d.last['d2h'][k]
            if not ev.query():
                poisoned = all(_poisoned(t) for t in runner.out_host[k].values())
                if not ev.query():
                    early.append(poisoned)
    for j in range(len(seq) - runner.nslots, len(seq)):
        read(j, slots[j])
    torch.cuda.synchronize()
    if 'd2h' in stages:
        print('pinned records looked at before their download: %d of %d, poisoned: %s' % (len(early), len(seq), early))
        assert early and all(early), early
    if stages:
        d.check()


# ---------------------------------------------------------------------------------------- StreamRunner, VideoRunner
# padded shapes under the (640, 360) rule: A 384x640, B 384x480, C 640x384
SIZES_1 = [(360, 640), (540, 960), (480, 640), (360, 480), (720, 1280), (640, 360), (480, 640)]   # A A B B A C B
SIZES_4 = [(360, 640), (540, 960), (720, 1280), (360, 640), (480, 640), (360, 480), (640, 360)]   # A A A A B B C
REC_FIELDS = ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'track_feats', 'mask_bits', 'render')


@pytest.fixture(scope='module')
def vis():
    from sipmask_b200.serving import StreamRunner
    from test_gpu_stream import _raw_images
    from test_gpu_video import _sd
    sd, kw, rule = _sd()
    # the streams of images keep the detections above 0.27 (SipMask-VIS keeps 10 above 0.03, which every image here
    # reaches), so the detection count differs from image to image; the videos keep SipMask-VIS's setting
    skw = dict(kw, test_cfg=dict(kw['test_cfg'], score_thr=0.27, max_per_img=100))
    imgs = dict(b1=[x.pin_memory() for x in _raw_images(SIZES_1, seed=31)],
                b4=[x.pin_memory() for x in _raw_images(SIZES_4, seed=32)])
    serial = StreamRunner(sd, in_flight=1, batch=1, max_src_hw=(720, 1280), render=True, **rule, **skw)
    want = {}
    for name, seq in imgs.items():
        want[name] = []
        for x in seq:
            k = serial.submit(x)
            torch.cuda.synchronize()
            r = serial.result(k)
            want[name].append(dict(_cpu({f: r[f] for f in REC_FIELDS}), pad=r['meta']['pad_shape'][:2],
                                   ori=r['meta']['ori_shape'][:2]))
    # batch 1, 2 slots: the images a slot takes in turn differ in padded shape and count.  batch 4 keeps its order (a
    # full batch, then batches closed by a change of padded shape) with a different count for every image
    order = dict(b1=_slot_order(want['b1'], (2,), key=lambda i: want['b1'][i]['pad']), b4=list(range(PERIOD)))
    for name, w in want.items():
        counts = [int(r['count'].reshape(-1)[0]) for r in w]
        print('%s images: detections per image %s, padded shapes %s, order %s' % (name, counts, [r['pad'] for r in w],
                                                                                  order[name]))
    assert len(set(int(r['count'].reshape(-1)[0]) for r in want['b4'])) == PERIOD
    x0 = imgs['b1'][4]
    cycles = _calibrate('VIS stream 720x1280 image', lambda: (serial.result(serial.submit(x0)), torch.cuda.synchronize()))
    return dict(sd=sd, kw=kw, skw=skw, rule=rule, imgs=imgs, want=want, order=order, cycles=cycles, cache={})


def _same_stream_record(got, want, rle):
    for k in REC_FIELDS:
        if k == 'mask_bits' and rle:
            assert k not in got
            continue
        if k in got:
            a = got[k].cpu()
            assert torch.equal(a.reshape(want[k].shape) if k == 'count' else a, want[k]), k


STREAM_STAGES = PIPE_STAGES


@pytest.mark.parametrize('stages', _pipe_stage_params())
@pytest.mark.parametrize('batch,masks,render', [(1, 'bits', False), (4, 'bits', False), (1, 'rle', False),
                                                (1, 'bits', True)],
                         ids=['b1-bits', 'b4-bits', 'b1-rle', 'b1-render'])
def test_stream_runner_records(vis, monkeypatch, batch, masks, render, stages):
    """StreamRunner, 2 slots: 7 images whose consecutive uses of a slot differ in padded shape.  batch=4 dispatches a
    full batch, partial batches closed by a change of padded shape and a last one closed by flush()."""
    from sipmask_b200 import rle as RL
    from sipmask_b200.serving import StreamRunner
    from test_gpu_video import _read_before_reuse
    key = ('stream', batch, masks, render)
    runner = vis['cache'].get(key)
    if runner is None:
        runner = vis['cache'][key] = StreamRunner(vis['sd'], in_flight=2, batch=batch, max_src_hw=(720, 1280), masks=masks,
                                                  render=render, **vis['rule'], **vis['skw'])
        for t in runner.in_dev:
            t.zero_()
    name = 'b4' if batch > 1 else 'b1'
    imgs, want = vis['imgs'][name], vis['want'][name]
    seq = [vis['order'][name][i % PERIOD] for i in range(2 * PERIOD)]
    torch.cuda.synchronize()
    d = Delays(monkeypatch, stages, vis['cycles'])

    # pass 1: consumer records (the host never blocks; the downloads of this pass are not read, so the consumer may
    # poison what it cloned)
    got = []

    def fn(rec):
        got.append({k: v.clone() for k, v in rec.items()})
        _poison_record(rec)
    for i in seq:
        runner.step(imgs[i], fn)
    runner.flush(fn)
    torch.cuda.synchronize()
    assert len(got) == len(seq)
    for j, i in enumerate(seq):
        _same_stream_record(got[j], want[i], runner.rle)

    # pass 2: every result() before its slot is reused; pinned records poisoned after each read
    t0 = runner.i
    done = {t: None for t in range(t0)}           # earlier records: consumed above

    def read(t):
        k, j = runner._locate(t)
        m = runner.slot_images[k][j]
        r = runner.result(k if batch == 1 else t)
        w = want[seq[t - t0]]
        assert r['meta']['ori_shape'][:2] == w['ori']
        _same_stream_record(r, w, runner.rle)
        if runner.rle:
            cnt = int(w['count'].reshape(-1)[0])
            assert r['segms'] == RL.encode_planes(w['mask_bits'][:cnt].numpy(), w['ori']), t
            ib = runner.engines[k][m['pad_shape'][:2]].rle_img_bytes
            _poison(runner.rle_regions[k][j * ib:(j + 1) * ib])
        _poison(*[r[f] for f in REC_FIELDS if f in r])
        return True
    for i in seq:
        _read_before_reuse(runner, read, done, imgs[i])
        runner.submit(imgs[i])
    _read_before_reuse(runner, read, done)
    runner.flush()
    for t in range(t0, runner.i):
        if t not in done:
            done[t] = read(t)
    torch.cuda.synchronize()
    assert sum(t >= t0 for t in done) == len(seq)
    if stages:
        d.check()


# frames of test_gpu_video's three videos, at most two open at once (lanes=2): video 2 takes video 1's lane
VIDEO_ORDER = ([(v, f) for f in range(5) for v in (0, 1)] + [(2, 0), (0, 5)] + [(2, f) for f in range(1, 4)])


@pytest.fixture(scope='module')
def video(vis):
    from sipmask_b200.serving import VideoRunner
    from test_gpu_video import _host_path, _same_frame, _videos
    sd, kw, rule = vis['sd'], vis['kw'], vis['rule']
    videos = _videos()
    recs, js, frames, _ = _host_path(sd, kw, rule, videos, VIDEO_ORDER, 1, 'rle')
    for v, (vid, fr) in enumerate(videos):
        assert int(recs[(v, 0)]['count'].reshape(-1)[0]) > 0, vid      # a first frame resets its lane's state
    assert any((r['ids'] > 0).any() for r in recs.values())
    serial = VideoRunner(sd, lanes=2, in_flight=1, batch=1, max_src_hw=(1080, 1920), render=True, **rule, **kw)
    render = {}
    for v, f in VIDEO_ORDER:
        t = serial.submit(videos[v][1][f], videos[v][0], f)
        torch.cuda.synchronize()
        r = serial.result(t)
        assert r['obj_ids'].tolist() == recs[(v, f)]['ids'].tolist(), (v, f)
        assert _same_frame(r['frame'], frames[videos[v][0]][f]), (v, f)
        render[(v, f)] = r['render'].clone()
        if f == len(videos[v][1]) - 1:
            serial.end_video(videos[v][0])
    serial.flush()
    for vid, _ in videos:
        assert serial.video_json(vid) == js[vid]
    return dict(videos=videos, recs=recs, js=js, frames=frames, render=render, cache={})


VIDEO_STAGES = ('track', 'compute_end', 'd2h')


def _video_stage_params():
    return [pytest.param(s, id=n) for s, n in [((), 'none')] + [((x,), x) for x in VIDEO_STAGES] + [(VIDEO_STAGES, 'all')]]


@pytest.mark.parametrize('stages', _video_stage_params())
@pytest.mark.parametrize('batch,render', [(1, False), (2, False), (1, True)], ids=['b1', 'b2', 'b1-render'])
def test_video_runner_records(vis, video, monkeypatch, batch, render, stages):
    """VideoRunner, 2 lanes and 3 slots: records, object ids, per-frame pairs and the drawing equal the serial run and the
    host tracker's; every frame is read before its slot is reused."""
    from sipmask_b200.serving import VideoRunner
    from test_gpu_video import _read_before_reuse, _same_frame
    key = ('video', batch, render)
    vr = video['cache'].get(key)
    if vr is None:
        vr = video['cache'][key] = VideoRunner(vis['sd'], lanes=2, in_flight=3, batch=batch, max_src_hw=(1080, 1920),
                                               render=render, **vis['rule'], **vis['kw'])
        for t in vr.in_dev:
            t.zero_()
    videos, recs, frames = video['videos'], video['recs'], video['frames']
    torch.cuda.synchronize()
    d = Delays(monkeypatch, stages, vis['cycles'])
    done = {t: None for t in range(vr.i)}         # frames of earlier cases: read by them
    tickets = {}

    def read(t):
        r = vr.result(t)
        k, j = vr._locate(t)
        v, f = tickets[t]
        want = recs[(v, f)]
        cnt = int(want['count'].reshape(-1)[0])
        assert torch.equal(r['count'].reshape(-1), want['count'].reshape(-1)), (v, f)
        assert torch.equal(r['det_bboxes'][:cnt], want['det']) and torch.equal(r['det_labels'][:cnt], want['lab'])
        assert r['segms'] == want['segms'], (v, f)
        assert r['obj_ids'].tolist() == want['ids'].tolist(), (v, f)
        assert _same_frame(r['frame'], frames[videos[v][0]][f]), (v, f)
        if render:
            assert torch.equal(r['render'], video['render'][(v, f)]), (v, f)
        ib = vr.engines[k][vr.slot_images[k][j]['pad_shape'][:2]].rle_img_bytes
        _poison(vr.rle_regions[k][j * ib:(j + 1) * ib], vr.ids_host[k][j])
        _poison(*[r[n] for n in REC_FIELDS if n in r])
        return True
    for v, f in VIDEO_ORDER:
        img = videos[v][1][f]
        _read_before_reuse(vr, read, done, img)
        tickets[vr.i] = (v, f)
        vr.submit(img, videos[v][0], f)
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    _read_before_reuse(vr, read, done)
    vr.flush()
    for t in tickets:
        if t not in done:
            done[t] = read(t)
    for vid, _ in videos:
        assert vr.video_json(vid) == video['js'][vid], vid
    torch.cuda.synchronize()
    assert all(done[t] for t in tickets) and not vr.book.videos
    if stages:
        d.check()


# ------------------------------------------------------------------------------------ CocoEvalRunner, VideoEvalRunner
def _same_evaluation(got, want):
    """Every precision, recall and scores array and every stat of every metric, bit for bit."""
    import numpy as np
    assert sorted(got['arrays']) == sorted(want['arrays']) and sorted(got['stats']) == sorted(want['stats'])
    for m in want['arrays']:
        for key in ('precision', 'recall', 'scores'):
            assert np.array_equal(got['arrays'][m][key], want['arrays'][m][key]), (m, key)
    for m in want['stats']:
        assert np.array_equal(got['stats'][m], want['stats'][m]), m


def _cycles(name, fwd_ms):
    ms = min(max(3 * fwd_ms, MIN_MS), CAP_MS)
    cycles = int(ms / _ms_per_cycle())
    print('%s: serial image %.2f ms -> delay %d cycles (%.2f ms)' % (name, fwd_ms, cycles, cycles * _ms_per_cycle()))
    return cycles


@pytest.fixture(scope='module')
def coco():
    """test_gpu_cocoeval's seeded dataset (7 images, SipMask++ 544 runner, 2 slots) and its serial evaluation."""
    from sipmask_b200 import cocoeval as C
    from sipmask_b200.serving import CocoEvalRunner
    from test_gpu_cocoeval import _first_pass_gt, _runner_images, _runner_kw
    imgs = [x.pin_memory() for x in _runner_images(PERIOD, seed=21)]
    cat_ids = [1 + label % 12 for label in range(80)]
    gt = _first_pass_gt(imgs, cat_ids, seed=3)
    assert len(gt['annotations']) > 20
    sd, kw = _runner_kw(1, 'bits')
    serial = CocoEvalRunner(sd, C.CocoGroundTruth(gt), cat_ids, **dict(kw, in_flight=1))
    ts = []
    for n, x in enumerate(imgs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        serial.submit(x, 1000 + n)
        serial.finish()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) * 1e3)
    want = serial.evaluate()
    assert 0 < want['stats']['bbox'][0] < 1 and 0 < want['stats']['segm'][0] < 1, want['stats']
    return dict(sd=sd, kw=kw, gt=gt, cat_ids=cat_ids, imgs=imgs, want=want, cycles=_cycles('SipMask++ 544 image', min(ts)))


@pytest.mark.parametrize('stages', [(), ('gt',), ('eval',), ('gt', 'eval')], ids=['none', 'gt', 'eval', 'all'])
def test_coco_eval_runner_evaluation(coco, monkeypatch, stages):
    """CocoEvalRunner, 2 slots: the ground truth staged on the H2D stream and matched on the slot's stream, kept alive
    there by record_stream; box and mask AP equal the serial run's bit for bit."""
    from sipmask_b200 import cocoeval as C
    from sipmask_b200.serving import CocoEvalRunner
    runner = CocoEvalRunner(coco['sd'], C.CocoGroundTruth(coco['gt']), coco['cat_ids'], **coco['kw'])
    for t in runner.in_dev:
        t.zero_()
    torch.cuda.synchronize()
    d = Delays(monkeypatch, stages, coco['cycles'])
    for n, x in enumerate(coco['imgs']):
        runner.submit(x, 1000 + n)
    got = runner.evaluate()
    torch.cuda.synchronize()
    _same_evaluation(got, coco['want'])
    if stages:
        d.check()


@pytest.fixture(scope='module')
def ytvis(vis):
    """test_gpu_ytviseval's seeded ground truth of the three videos, and the serial evaluation with 2 lanes."""
    from sipmask_b200.serving import VideoEvalRunner
    from sipmask_b200.ytviseval import YtvisGroundTruth
    from test_gpu_video import _interleave
    from test_gpu_ytviseval import _first_pass, _gt_from_json, _vis_videos
    sd, kw, rule = vis['sd'], vis['kw'], vis['rule']
    videos = _vis_videos()
    js = _first_pass(sd, kw, rule, videos, _interleave(videos))
    ann = _gt_from_json(videos, js)
    serial = VideoEvalRunner(sd, YtvisGroundTruth(ann), lanes=2, eval_slots=2, batch=1, in_flight=1,
                             max_src_hw=(1080, 1920), masks='rle', **rule, **kw)
    for v, f in VIDEO_ORDER:
        serial.submit(videos[v][1][f], videos[v][0], f)
        torch.cuda.synchronize()
        if f == len(videos[v][1]) - 1:
            serial.end_video(videos[v][0])
    want = serial.evaluate()
    assert 0 < want['stats']['segm'][0] < 1, want['stats']
    return dict(ann=ann, videos=videos, want=want, json={vid: serial.video_json(vid) for vid, _ in videos})


@pytest.mark.parametrize('stages', [(), ('gt',), ('eval',), ('track',), ('gt', 'eval', 'track')],
                         ids=['none', 'gt', 'eval', 'track', 'all'])
@pytest.mark.parametrize('batch', [1, 2])
def test_video_eval_runner_evaluation(vis, ytvis, monkeypatch, batch, stages):
    """VideoEvalRunner, 2 lanes (2 accumulator slots: ended videos are matched mid-stream) and 3 slots: the overlaps on
    the slot's stream are ordered before their scatter on the tracker stream (ev_ovl); mask AP and every video's result
    json equal the serial run's."""
    from sipmask_b200.serving import VideoEvalRunner
    from sipmask_b200.ytviseval import YtvisGroundTruth
    videos = ytvis['videos']
    vr = VideoEvalRunner(vis['sd'], YtvisGroundTruth(ytvis['ann']), lanes=2, eval_slots=2, batch=batch, in_flight=3,
                         max_src_hw=(1080, 1920), masks='rle', **vis['rule'], **vis['kw'])
    for t in vr.in_dev:
        t.zero_()
    torch.cuda.synchronize()
    d = Delays(monkeypatch, stages, vis['cycles'])
    for v, f in VIDEO_ORDER:
        vr.submit(videos[v][1][f], videos[v][0], f)
        if f == len(videos[v][1]) - 1:
            vr.end_video(videos[v][0])
    got = vr.evaluate()
    torch.cuda.synchronize()
    _same_evaluation(got, ytvis['want'])
    for vid, _ in videos:
        assert vr.video_json(vid) == ytvis['json'][vid], vid
    if stages:
        d.check()
