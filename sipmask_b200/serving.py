"""Pipelined host <-> device serving loop around SipMaskEngine.

The reference moves data synchronously: `scatter` uploads the image (MM/mmdet/apis/inference.py:83) and every detection's
mask is copied back one by one (`masks[i].cpu().numpy()`, sipmask_head.py:645-657).  Here the upload of image i+1 and
the download of result i-1 run on their own streams (the GPU has independent H2D / D2H copy engines) while the
CUDA-graph replay of image i runs on a compute stream; device staging buffers decouple the three.
Per image: one 12.9 MB H2D (fp32 NCHW 800x1344) and one 13.4 MB D2H (fixed-shape record + bit-packed masks).

Images in flight.  One 800x1344 image is ~75 short convolution launches, most of them latency-bound chains that leave
SMs idle (layer3/4 have 33 / 9 M-tiles for 132 SMs).  `make_engines(..., in_flight=n)` builds n engines that share ONE
copy of the packed weights but own their activations and CUDA graph; `EnginePool` / `PipelinedRunner` replay them
round-robin on n streams with the persistent conv grids capped (64 CTAs), so the images fill each other's bubbles.
Every forward is still one image (imgs_per_gpu == 1, base.py:118-119); only the throughput changes.
"""
import contextlib
import gc

import numpy as np
import torch

from . import _lib as L
from . import conv as C
from . import render as R
from ._lib import TRACK_CAPACITY, SmbError
from .engine import SipMaskEngine

# grid cap / planner min_tiles per number of images in flight
_TUNING = {1: dict(max_ctas=None, head_max_ctas=None, min_tiles=48)}


def _tuning(n):
    if n in _TUNING:
        return dict(_TUNING[n])
    cap = 48 if n >= 6 else 64
    return dict(max_ctas=cap, head_max_ctas=cap, min_tiles=16)


def _masks_mode(masks):
    """True for masks='rle' (COCO RLE strings encoded on the device), False for masks='bits' (bit planes)."""
    if masks not in ('bits', 'rle'):
        raise ValueError("masks is 'bits' or 'rle', got %r" % (masks,))
    return masks == 'rle'


# string bytes per image of a masks='rle' runner's regions unless rle_bytes is given
DEFAULT_RLE_BYTES = 1 << 16


@contextlib.contextmanager
def _min_tiles(n):
    """Engines built inside the block plan their convolutions with the planner's min_tiles set to n."""
    prev = C.set_min_tiles(n)
    try:
        yield
    finally:
        C.set_min_tiles(prev)


def make_engines(state_dict, img_hw, in_flight=1, **kw):
    """n engines for n images in flight (weights shared, activations private)."""
    tune = _tuning(in_flight)
    min_tiles = kw.pop('min_tiles', tune.pop('min_tiles'))
    for k, v in tune.items():
        kw.setdefault(k, v)
    engs = []
    with _min_tiles(min_tiles):
        for i in range(in_flight):
            engs.append(SipMaskEngine(state_dict, img_hw, share_weights=engs[0] if engs else None, **kw))
    return engs


def _image_segms(region, eng, j, ori, planes):
    """Image j's list of RLE dicts from the pinned region eng's encoder wrote a slot's strings into; an image whose
    strings overflowed the encoder's capacities is encoded on the host from planes[j] (the forward's device bit planes)."""
    from . import rle as R
    ib = eng.rle_img_bytes
    return R.image_segms(region.numpy()[j * ib:(j + 1) * ib], eng.max_num, ori, lambda n: planes[j, :n].cpu().numpy())


def _record(o):
    """The record of a slot's buffers (device or host), under the engine's record names."""
    rec = dict(det_bboxes=o['det'], det_labels=o['lab'], count=o['cnt'])
    for name, key in (('idx', 'idxs_keep'), ('bits', 'mask_bits'), ('trk', 'track_feats'), ('msc', 'mask_scores'),
                      ('render', 'render')):
        if name in o:
            rec[key] = o[name]
    return rec


def _queue_step(pending, n, ks, fn, consume):
    """Queue the slots just launched (ks) in pending; with fn, hand the OLDEST to consume(slot, fn) while all n slots are
    in flight, so the consumer (e.g. the all-gather) never stalls the slots behind it.  Without fn nothing is queued."""
    pending += ks
    if fn is None:
        pending.clear()
    while len(pending) >= n:
        consume(pending.pop(0), fn)


def _queue_flush(pending, fn, consume):
    """Hand every queued slot to consume(slot, fn), oldest first (fn=None: drop them)."""
    while pending:
        k = pending.pop(0)
        if fn is not None:
            consume(k, fn)


class _Slots(object):
    """The streams and events of n staging slots, and the order of the work on them.  Slot k has an input (what
    the H2D stream uploads and compute reads) and an output (the record compute writes, the D2H stream downloads and a
    consumer reads on its own stream).  Five events per slot decide when each may be overwritten:
      ev_in_ready   the uploads into slot k are done: its compute waits for them;
      ev_in_free    compute consumed slot k's input: the next upload into slot k waits for it;
      ev_out_ready  compute wrote slot k's record: its download and its consumer wait for it;
      ev_out_free   slot k's download is done: the slot's next record and result() wait for it;
      ev_hold       slot k's last consumer is done with the record (None before the first): the next record waits for it.
    copies=False: no H2D / D2H streams (the inputs are in the engines, the records are read where compute wrote them).
    streams=False: every slot computes on the current stream."""

    def __init__(self, dev, n, streams=True, copies=True):
        self.dev, self.n = dev, n
        self.h2d = torch.cuda.Stream(device=dev) if copies else None
        self.d2h = torch.cuda.Stream(device=dev) if copies else None
        self.streams = [torch.cuda.Stream(device=dev) for _ in range(n)] if streams else None
        self.ev_in_ready, self.ev_in_free, self.ev_out_ready, self.ev_out_free = ([torch.cuda.Event() for _ in range(n)]
                                                                                  for _ in range(4))
        self.ev_hold = [None] * n

    def warm_up(self, engs, fwd):
        """fwd(engine) twice per engine on its slot's stream (warm-up + graph capture), then wait for them."""
        cur = torch.cuda.current_stream(self.dev)
        for st, eng in zip(self.streams or [cur], engs):
            if self.streams:
                st.wait_stream(cur)
            with torch.cuda.stream(st):
                fwd(eng)
                fwd(eng)
        for st in self.streams or [cur]:
            st.synchronize()

    def mark_free(self):
        """Every slot's input and output may be overwritten once the current stream's work so far is done."""
        cur = torch.cuda.current_stream(self.dev)
        for e in self.ev_in_free + self.ev_out_free:
            e.record(cur)

    def claim_input(self, k):
        """The uploads that follow wait until compute consumed slot k's previous input."""
        self.h2d.wait_event(self.ev_in_free[k])

    def upload(self, dst, src):
        with torch.cuda.stream(self.h2d):
            dst.copy_(src, non_blocking=True)

    def begin_compute(self, k):
        """What the H2D stream uploaded so far is slot k's input: returns the slot's compute stream, made to wait for it."""
        self.ev_in_ready[k].record(self.h2d)
        cs = self.streams[k] if self.streams else torch.cuda.current_stream(self.dev)
        cs.wait_event(self.ev_in_ready[k])
        return cs

    def input_free(self, k, cs):
        """Slot k's input is consumed once cs's work so far is done."""
        self.ev_in_free[k].record(cs)

    def claim_output(self, k, cs):
        """cs's next work, which writes slot k's record, waits until the slot's previous record is downloaded and
        released by its consumer."""
        if self.d2h is not None:
            cs.wait_event(self.ev_out_free[k])
        if self.ev_hold[k] is not None:
            cs.wait_event(self.ev_hold[k])

    def publish(self, k, cs):
        """Slot k's record is complete once cs's work so far is done."""
        self.ev_out_ready[k].record(cs)

    def await_record(self, k, stream):
        """stream waits until slot k's record is published."""
        stream.wait_event(self.ev_out_ready[k])

    def download(self, k, copies, after=None):
        """The (host, device) copies on the D2H stream once slot k's record is published, or once the event `after` (of
        work that waited for the record) is; the slot's output is free when they are done."""
        with torch.cuda.stream(self.d2h):
            self.d2h.wait_event(self.ev_out_ready[k] if after is None else after)
            for dst, src in copies:
                dst.copy_(src, non_blocking=True)
            self.ev_out_free[k].record(self.d2h)

    def hold(self, k, stream):
        """Slot k's next record waits until stream's work so far is done."""
        if self.ev_hold[k] is None:
            self.ev_hold[k] = torch.cuda.Event()
        self.ev_hold[k].record(stream)

    def hand_over(self, k, work):
        """work() on the CURRENT stream once slot k's record is published; the slot's next record waits for what work
        enqueued.  Returns work's result."""
        cur = torch.cuda.current_stream(self.dev)
        self.await_record(k, cur)
        r = work()
        self.hold(k, cur)
        return r

    def join(self, *streams):
        """Make the current stream wait for `streams`, by default for the downloads (and so for every record in flight),
        or for the compute streams when there are none."""
        cur = torch.cuda.current_stream(self.dev)
        for s in streams or ([self.d2h] if self.d2h is not None else self.streams):
            cur.wait_stream(s)

    def wait(self, k):
        """Block the host until slot k's download has finished."""
        self.ev_out_free[k].synchronize()


class EnginePool(object):
    """Round-robin replay of n resident engines on n streams (inputs already in each engine's `img`).  Each engine's
    outputs are its slot's record."""

    def __init__(self, engines):
        self.engs = list(engines)
        self.n = len(self.engs)
        dev = self.engs[0].dev
        self.dev = dev
        self.slots = _Slots(dev, self.n, copies=False)
        self.i = 0
        self.pending = []
        self.slots.warm_up(self.engs, lambda eng: eng.forward(None))
        for k in range(self.n):
            self.slots.hold(k, torch.cuda.current_stream(dev))

    @property
    def streams(self):
        return self.slots.streams

    def launch(self):
        """Enqueue one image on the next engine; returns its index.  Does not block the host."""
        k = self.i % self.n
        st = self.streams[k]
        self.slots.claim_output(k, st)
        with torch.cuda.stream(st):
            self.engs[k].forward(None)
        self.slots.publish(k, st)
        self.i += 1
        return k

    def consume(self, k, fn):
        """Run fn(engine_k_outputs) on the CURRENT stream once image k is done; engine k is not replayed again before fn's
        work has finished (used for the all-gather of the detection record)."""
        return self.slots.hand_over(k, lambda: fn(self.engs[k]._result()))

    def step(self, fn=None):
        """One image: launch it, and (if fn is given) hand the OLDEST image in flight to fn on the current stream, so the
        consumer (e.g. the all-gather) never stalls the images behind it."""
        _queue_step(self.pending, self.n, [self.launch()], fn, self.consume)

    def flush(self, fn=None):
        """Consume what is still in flight and make the current stream wait for all of it."""
        _queue_flush(self.pending, fn, self.consume)
        self.join()

    def join(self):
        """Make the current stream wait for everything in flight."""
        self.slots.join()


class PipelinedRunner(object):
    """raw_hw=(h, w): the host hands over the decoder's uint8 BGR HWC image (h*w*3 bytes H2D instead of 4*3*H*W) and the
    step starts with the fused resize / normalise / pad kernel (engine.forward_raw, SURVEY 8f-3).

    masks='rle' (engines built with rle_bytes > 0): every slot owns a pinned region the engine's encoder writes the COCO RLE
    strings into during the forward (set_rle_dest before each replay, so slots that share one engine and graph still own
    their region); the bit planes are not downloaded.  result() then carries 'segms' (per image of the forward, the list of
    RLE dicts) in place of 'bits'.  The bit planes stay in the slot's device record, from which an image whose strings
    overflowed the encoder's capacities is encoded on the host."""

    def __init__(self, engines, depth=2, raw_hw=None, masks='bits'):
        self.engs = list(engines) if isinstance(engines, (list, tuple)) else [engines]
        self.n = len(self.engs)
        self.eng = engine = self.engs[0]
        self.rle = _masks_mode(masks)
        if self.rle and not all(e.rle_bytes for e in self.engs):
            raise ValueError("masks='rle' needs engines built with rle_bytes > 0")
        # one staging slot per engine when several images are in flight, `depth` slots for a single engine
        self.nslots = self.n if self.n > 1 else depth
        ns = self.nslots
        dev = engine.dev
        self.dev = dev
        # several engines: each slot computes on its engine's stream; one engine: every slot on the current stream
        self.slots = _Slots(dev, ns, streams=self.n > 1)
        self.raw = raw_hw is not None
        if self.raw:
            assert engine.N == 1, 'raw uint8 input: one image per forward'
            self.in_dev = [torch.empty((int(raw_hw[0]), int(raw_hw[1]), 3), dtype=torch.uint8, device=dev) for _ in range(ns)]
        else:
            self.in_dev = [torch.empty_like(engine.img) for _ in range(ns)]
        self.out_dev = [dict(det=torch.empty_like(engine.det), lab=torch.empty_like(engine.labels),
                             cnt=torch.empty_like(engine.count), bits=torch.empty_like(engine.mask_bits)) for _ in range(ns)]
        if engine.vis:                            # SipMask-VIS: the 512-d tracking features travel with the record
            for o in self.out_dev:
                o['trk'] = torch.empty_like(engine.det_track)
        if engine.rescoring:                      # SipMask++: the mask scores travel with the record
            for o in self.out_dev:
                o['msc'] = torch.empty_like(engine.mask_scores)
        # rle: the planes stay on the device (the overflow fallback's copy), the strings arrive in the slot's region
        self.out_host = [{k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in o.items()
                          if not (self.rle and k == 'bits')} for o in self.out_dev]
        if self.rle:
            self.rle_regions = [torch.zeros(engine.N * engine.rle_img_bytes, dtype=torch.uint8).pin_memory() for _ in range(ns)]
            self.slot_oris = [None] * ns
        self.i = 0
        self.pending = []
        self.h2d_bytes = self.in_dev[0].numel() * self.in_dev[0].element_size()
        # fixed-size downloads per forward (rle: plus the strings and headers the encoder writes, which vary per image)
        self.d2h_bytes = sum(v.numel() * v.element_size() for v in self.out_host[0].values())
        self.slots.warm_up(self.engs, lambda eng: self._fwd(eng, 0))
        self.slots.mark_free()

    def _fwd(self, eng, k):
        if self.raw:
            eng.forward_raw(self.in_dev[k])
        else:
            eng.forward(None)

    def submit(self, host_img):
        """host_img: pinned fp32 NCHW tensor (or pinned uint8 HWC BGR image in raw mode).  Enqueues upload -> graph replay -> download; returns the slot index.
        Nothing here blocks the host."""
        k = self.i % self.nslots
        eng = self.engs[k % self.n]
        sl = self.slots
        sl.claim_input(k)
        sl.upload(self.in_dev[k], host_img)
        o = self.out_dev[k]
        cs = sl.begin_compute(k)
        with torch.cuda.stream(cs):
            if self.rle:
                eng.set_rle_dest(self.rle_regions[k])      # this slot's strings go to this slot's region
                self.slot_oris[k] = [m[1][:2] for m in eng.image_metas]
            if self.raw:
                eng.forward_raw(self.in_dev[k])            # preprocess kernel reads the staged uint8 image, then the graph
                sl.input_free(k, cs)
            else:
                eng.img.copy_(self.in_dev[k], non_blocking=True)
                sl.input_free(k, cs)
                eng.forward(None)
            sl.claim_output(k, cs)
            o['det'].copy_(eng.det, non_blocking=True)
            o['lab'].copy_(eng.labels, non_blocking=True)
            o['cnt'].copy_(eng.count, non_blocking=True)
            o['bits'].copy_(eng.mask_bits, non_blocking=True)
            if 'trk' in o:
                o['trk'].copy_(eng.det_track, non_blocking=True)
            if 'msc' in o:
                o['msc'].copy_(eng.mask_scores, non_blocking=True)
            sl.publish(k, cs)
        sl.download(k, [(h, o[name]) for name, h in self.out_host[k].items()])
        self.i += 1
        return k

    def consume(self, slot, fn):
        """Run fn(slot's device record) on the CURRENT stream once it is ready; the slot is not overwritten before fn's
        work has finished (used for the all-gather of the detection record)."""
        rec = _record(self.out_dev[slot])
        return self.slots.hand_over(slot, lambda: fn(rec))

    def step(self, host_img, fn=None):
        """submit() + hand the OLDEST slot in flight to fn (see EnginePool.step).  Returns the submitted slot."""
        k = self.submit(host_img)
        _queue_step(self.pending, self.nslots, [k], fn, self.consume)
        return k

    def flush(self, fn=None):
        _queue_flush(self.pending, fn, self.consume)
        self.join()

    def result(self, slot):
        """Blocks until the slot's download finished; returns pinned host tensors (valid until the slot is reused).
        masks='rle': a dict of them with 'segms' (one list of RLE dicts per image of the forward) in place of 'bits'."""
        self.slots.wait(slot)
        if not self.rle:
            return self.out_host[slot]
        eng = self.engs[slot % self.n]
        rec = dict(self.out_host[slot])
        rec['segms'] = [_image_segms(self.rle_regions[slot], eng, i, ori, self.out_dev[slot]['bits'])
                        for i, ori in enumerate(self.slot_oris[slot])]
        return rec

    def join(self):
        """Make the current stream wait for the downloads (and so for every image in flight)."""
        self.slots.join()

    def drain(self):
        self.slots.d2h.synchronize()
        self.slots.h2d.synchronize()


def rescale_size(h, w, scale=(1333, 800)):
    """mmcv.imrescale's size rule (keep ratio): (new_h, new_w, scale_factor) with scale_factor = min(long / max(h, w),
    short / min(h, w)) and new = int(old * scale_factor + 0.5)."""
    max_long, max_short = max(scale), min(scale)
    sf = min(max_long / max(h, w), max_short / min(h, w))
    return int(h * float(sf) + 0.5), int(w * float(sf) + 0.5), sf


def image_meta(h, w, resize=(1333, 800), keep_ratio=True, size_divisor=32):
    """(img_shape, pad_shape, scale_factor) of an h x w image under the test pipeline's Resize + Pad (mmdet
    datasets/transforms.py): keep_ratio rescales by one factor (a python float), otherwise each axis goes to
    resize = (new_w, new_h) and scale_factor = float32 [w_scale, h_scale, w_scale, h_scale]."""
    if keep_ratio:
        nh, nw, sf = rescale_size(h, w, resize)
    else:
        nw, nh = int(resize[0]), int(resize[1])
        sf = np.array([nw / w, nh / h, nw / w, nh / h], dtype=np.float32)
    return (nh, nw, 3), (_pad(nh, size_divisor), _pad(nw, size_divisor), 3), sf


def _pad(v, size_divisor):
    """v rounded up to a multiple of size_divisor (the Pad transform)."""
    return (int(v) + size_divisor - 1) // size_divisor * size_divisor


def largest_pad_shapes(resize=(1333, 800), keep_ratio=True, size_divisor=32):
    """The padded shapes no other image exceeds under the rule: (short, long) and (long, short) for keep_ratio,
    the one fixed shape otherwise."""
    if not keep_ratio:
        return [(_pad(resize[1], size_divisor), _pad(resize[0], size_divisor))]
    s, l = _pad(min(resize), size_divisor), _pad(max(resize), size_divisor)
    return [(s, l), (l, s)] if s != l else [(s, l)]


def bm_resize_size(h, w, min_size=800, max_size=1333):
    """SipMask-benchmark's test size rule (fcos_core/data/transforms/transforms.py:36-55, Resize.get_size) for an h x w
    image -> (oh, ow), in Python float arithmetic: the short side becomes min_size unless the long side would exceed
    max_size, in which case the short side becomes int(round(max_size * short / long)); an image whose short side already
    has that size is not resized; otherwise long = int(size * long / short).  The long side is not bounded: extreme
    aspect ratios (1 x 2048) keep their size."""
    size = min_size
    if max_size is not None:
        mn, mx = float(min((w, h))), float(max((w, h)))
        if mx / mn * size > max_size:
            size = int(round(max_size * mn / mx))
    if (w <= h and w == size) or (h <= w and h == size):
        return h, w
    if w < h:
        return int(size * h / w), size
    return size, int(size * w / h)


def bm_image_meta(h, w, min_size=800, max_size=1333, size_divisor=32):
    """(img_shape, pad_shape, scale_factor) of an h x w image under SipMask-benchmark's test transform (bm_resize_size,
    then to_image_list(size_divisible=32)).  The benchmark post-processing reads only img_shape and ori_shape
    (postproc.image_geometry(benchmark=True)); scale_factor = min(oh / h, ow / w) is the ratio its mask resize uses."""
    nh, nw = bm_resize_size(h, w, min_size, max_size)
    return (nh, nw, 3), (_pad(nh, size_divisor), _pad(nw, size_divisor), 3), min(nh / h, nw / w)


class StreamRunner(object):
    """Serves a stream of images of ANY size.  Every image runs the network on the canvas of its own padded shape (one
    engine per padded shape, a "bucket", built and captured on first use); only the post-processing geometry
    (img_shape, ori_shape, scale_factor) changes per image, written into the engine's geometry rows before its graph is
    replayed (SipMaskEngine.set_image_meta).

    in_flight slots, each with its own stream and ONE arena (device memory sized for the largest padded shape the resize
    rule produces) from which every bucket engine of the slot carves its activations: a second bucket costs its graph
    and bookkeeping, not another activation set.  Packed weights are shared by all engines.

    submit(img): a uint8 BGR HWC image of any size up to max_src_hw (raw mode; the resize runs on the GPU).  For
    SipMask-benchmark checkpoints (benchmark=True) either a uint8 RGB HWC image as PIL decodes it (raw=True: the
    benchmark's own test transform, PIL bilinear resize under bm_resize_size with min(resize) / max(resize) as min / max
    size, runs on the GPU), or a preprocessed fp32 NCHW image padded to a multiple of 32 together with its meta =
    (img_shape, ori_shape, scale_factor).  result(slot) returns the record with mask_bits cropped to the image's
    [max, ori_h, ceil(ori_w / 32)].  raw=True rejects, before anything is enqueued, images whose padded shape falls
    outside the arena's shapes (800x1344 / 1344x800 for the default rule: aspect ratios beyond about 24:1) and resizes
    that shrink more than conv.PIL_MAX_DOWNSCALE times on an axis.

    batch=B > 1 (raw images only): every forward runs B images of ONE padded shape through batch-B bucket engines (the
    throughput mode of the 544x544 configs).  Each image is uploaded into its slot's staging as soon as it is submitted;
    the open batch is dispatched when it holds B images, when the next image has a different padded shape, or on flush().
    Dispatch = geometry rows + source rows + one graph replay + one download of the real images' records.  A partial
    batch is completed with filler images (all-zero canvases with the last real image's geometry) that are computed but
    never returned.  submit() returns a ticket (the image's index in the stream) and result(ticket) that image's record.
    The mask record of a batch-B engine holds B * max * max_ori_h * ceil(max_ori_w / 32) words and is cleared every
    forward: set max_ori_hw to the largest original size expected, not the 2048 x 2048 default.

    masks='rle': the engines encode every detection's COCO RLE string on the device (rle_bytes string bytes per image,
    default DEFAULT_RLE_BYTES) into a pinned region each slot owns, shared by the slot's bucket engines; the bit planes are
    neither copied nor downloaded.  result() returns 'segms' (the image's list of RLE dicts {'size': [ori_h, ori_w],
    'counts': bytes}) in place of mask_bits; an image whose strings overflowed the encoder's capacities is encoded on the
    host from the bucket engine's planes, which stay valid until the slot is reused.  consume() hands fn the device record
    without mask_bits.

    render=True: every image is also drawn with its detections on the device (render.render_images: the masks blended in
    their labels' colours and the boxes of the detections with score > render_score_thr, as SipMask-mmdetection's
    show_result draws them) and result() / consume() carry 'render', the uint8 [ori_h, ori_w, 3] picture in the image's
    channel order.  The drawing reads the source image from the slot's input staging and writes the slot's render
    buffer, right after the record copies: so the slot's input is released after it (once the slot's output is claimed)
    instead of right after the forward.  Each slot holds a device and a pinned host render buffer of
    batch * max_src_hw[0] * max_src_hw[1] * 3 bytes.  benchmark=True runners do not render."""

    bm_raw = False
    _render_rule = L.RENDER_IMAGES                   # render=True: the rule render.draw applies                                    # benchmark=True, raw=True: raw RGB images, PIL resize on the GPU

    def __init__(self, state_dict, in_flight=1, resize=(1333, 800), keep_ratio=True, max_src_hw=(2048, 2048),
                 max_ori_hw=None, min_mask_up=0.5, mean=(102.9801, 115.9465, 122.7717), device='cuda', batch=1,
                 raw=False, masks='bits', render=False, render_score_thr=R.DEFAULT_SCORE_THR, **engine_kw):
        self.rle = _masks_mode(masks)
        self.render = bool(render)
        if self.render:
            if engine_kw.get('benchmark', False):
                raise ValueError('render=True: benchmark=True runners do not render')
            self.render_thr = R.score_threshold(render_score_thr, 'render_score_thr')
        if self.rle:
            engine_kw.setdefault('rle_bytes', DEFAULT_RLE_BYTES)
            if int(engine_kw['rle_bytes']) <= 0:
                raise ValueError("masks='rle' needs rle_bytes > 0")
        self.sd, self.n, self.B = state_dict, int(in_flight), int(batch)
        self.resize, self.keep_ratio, self.mean = tuple(resize), keep_ratio, mean
        self.max_src_hw = tuple(int(v) for v in max_src_hw)
        self.max_ori_hw = tuple(int(v) for v in (max_ori_hw or max_src_hw))
        self.min_mask_up = float(min_mask_up)
        self.benchmark = bool(engine_kw.get('benchmark', False))
        if self.B < 1:
            raise ValueError('batch must be at least 1, got %d' % self.B)
        self.bm_raw = bool(raw)
        if self.bm_raw and not self.benchmark:
            raise ValueError('raw=True selects raw RGB images for benchmark=True runners; other runners always take raw '
                             'BGR images')
        if self.benchmark and self.B > 1 and not self.bm_raw:
            raise ValueError('benchmark=True runners take one preprocessed image per forward (batch=1); raw=True batches '
                             'raw images')
        if self.bm_raw and not keep_ratio:
            raise ValueError('SipMask-benchmark resizes keep the aspect ratio: keep_ratio=False is not supported')
        self.dev = torch.device(device)
        if self.dev.index is None:
            self.dev = torch.device('cuda', torch.cuda.current_device())
        self.kw = dict(engine_kw, max_ori_hw=self.max_ori_hw, min_mask_up=self.min_mask_up, use_graph=True)
        self.tune = _tuning(self.n)
        for k in ('max_ctas', 'head_max_ctas'):
            self.kw.setdefault(k, self.tune[k])
        self._wcache = {}
        self.engines = [{} for _ in range(self.n)]            # slot -> {padded (H, W): engine}
        self.build_seconds = {}                               # padded (H, W) -> [build + capture seconds per slot]
        # arena: what an engine of the largest padded shape carves (measured by building it once without an arena)
        need = 0
        for hw in largest_pad_shapes(self.resize, self.keep_ratio):
            need = max(need, self._new_engine(hw, None).arena_bytes)
        gc.collect()                                          # the measuring engines' launch closures hold cycles
        torch.cuda.synchronize(self.dev)
        self.arena_bytes = need
        self.arenas = [torch.empty(need, dtype=torch.uint8, device=self.dev) for _ in range(self.n)]
        self.slots = _Slots(self.dev, self.n)
        if self.benchmark and not self.bm_raw:
            ph, pw = max(largest_pad_shapes(self.resize, self.keep_ratio), key=lambda s: s[0] * s[1])
            self.src_elems = 3 * max(ph, pw) ** 2
            self.in_dev = [torch.empty(self.src_elems, dtype=torch.float32, device=self.dev) for _ in range(self.n)]
        else:
            # B source images per slot, image j at [j * src_elems, (j + 1) * src_elems)
            self.src_elems = self.max_src_hw[0] * self.max_src_hw[1] * 3
            self.in_dev = [torch.empty(self.B * self.src_elems, dtype=torch.uint8, device=self.dev) for _ in range(self.n)]
        self.out_dev, self.out_host = [], []
        self.rle_regions = [None] * self.n                # masks='rle': per slot, the pinned region of its batch's strings
        if self.render:
            table = (R.image_palette(self.kw.get('num_classes', 81)) if self._render_rule == L.RENDER_IMAGES
                     else R.video_palette())
            self.render_palette = R.device_palette(table, self.dev)
        self._init_queue()
        self.slots.mark_free()

    def _init_queue(self):
        """Host bookkeeping of the batches: tickets, the open batch, what each slot holds."""
        self.i = 0                                    # next ticket
        self.dispatched = 0                           # batches dispatched so far; batch b runs in slot b % in_flight
        self._open = None                             # dict(slot, pad, images) of the batch being filled
        self.slot_images = [[] for _ in range(self.n)]    # per slot: the image dicts of the batch it holds, in order
        self.meta = [None] * self.n                   # per slot: its batch's last image dict (its only one at batch 1)
        self.pending = []

    def _new_engine(self, hw, arena):
        H, W = hw
        cap = self.max_ori_hw
        ori = (min(H, cap[0]), min(W, cap[1]), 3)
        kw = {k: v for k, v in self.kw.items() if k != 'min_tiles'}
        with _min_tiles(self.kw.get('min_tiles', self.tune['min_tiles'])):
            return SipMaskEngine(self.sd, (H, W), batch=self.B, img_shape=(H, W, 3), ori_shape=ori, scale_factor=1.0,
                                 share_weights=self._wcache, arena=arena, device=self.dev, **kw)

    def _engine(self, k, hw):
        """The slot's engine for padded shape hw, built in the slot's arena and captured on first use."""
        eng = self.engines[k].get(hw)
        if eng is None:
            import time
            torch.cuda.synchronize(self.dev)
            t0 = time.perf_counter()
            eng = self._new_engine(hw, self.arenas[k])
            with torch.cuda.stream(self.slots.streams[k]):
                if self.benchmark and not self.bm_raw:
                    eng.forward(None)                  # warm-up + capture
                else:
                    eng.forward_raw([torch.zeros((32, 32, 3), dtype=torch.uint8, device=self.dev)] * self.B, self.mean,
                                    self._pipeline)
            torch.cuda.synchronize(self.dev)
            self.build_seconds.setdefault(hw, []).append(time.perf_counter() - t0)
            self.engines[k][hw] = eng
        return eng

    @property
    def _pipeline(self):
        return 'benchmark' if self.bm_raw else 'mmdet'

    @property
    def buckets(self):
        return sorted(set(hw for d in self.engines for hw in d))

    def check(self, src_hw=None, meta=None):
        """Host-side validation of one image: (img_shape, pad_shape, scale_factor, ori_shape).  Raises ValueError (or the
        mask kernel's SmbError for a mask shrink beyond 4x) before anything is enqueued."""
        from .postproc import fused_mask_tile, image_geometry
        if meta is None:
            h, w = int(src_hw[0]), int(src_hw[1])
            if not (0 < h <= self.max_src_hw[0] and 0 < w <= self.max_src_hw[1]):
                raise ValueError('image %dx%d exceeds max_src_hw %dx%d' % (h, w, self.max_src_hw[0], self.max_src_hw[1]))
            if self.bm_raw:
                img_shape, pad, sf = self._bm_meta(h, w)
            else:
                img_shape, pad, sf = image_meta(h, w, self.resize, self.keep_ratio)
            ori = (h, w, 3)
        else:
            img_shape, ori, sf = meta
            pad = tuple(src_hw) + (3,)
            if pad[0] % 32 or pad[1] % 32 or pad[0] < img_shape[0] or pad[1] < img_shape[1]:
                raise ValueError('padded input %dx%d does not hold the %dx%d image in multiples of 32'
                                 % (pad[0], pad[1], img_shape[0], img_shape[1]))
            if pad[0] * pad[1] > max(a * b for a, b in largest_pad_shapes(self.resize, self.keep_ratio)):
                raise ValueError('padded input %dx%d is larger than the resize rule produces' % pad[:2])
        if not (0 < ori[0] <= self.max_ori_hw[0] and 0 < ori[1] <= self.max_ori_hw[1]):
            raise ValueError('ori_shape %dx%d exceeds max_ori_hw %dx%d' % (ori[0], ori[1], self.max_ori_hw[0],
                                                                            self.max_ori_hw[1]))
        g = image_geometry((pad[0] // 2, pad[1] // 2), img_shape, ori, sf, ssd_flag=self.kw.get('ssd_flag', False),
                           benchmark=self.benchmark, legacy_interp=self.kw.get('legacy_interp', False))
        fused_mask_tile(g.ry, g.rx, sizes=(pad[0] // 2, pad[1] // 2, g.full_h, g.full_w))
        r = float(np.float32(1.0 / self.min_mask_up))
        if g.ry > r or g.rx > r:
            raise ValueError('mask resize step (%g, %g) of the %dx%d image is steeper than min_mask_up=%g allows'
                             % (g.ry, g.rx, ori[0], ori[1], self.min_mask_up))
        return tuple(img_shape), tuple(pad), sf, tuple(ori)

    def _bm_meta(self, h, w):
        """bm_image_meta of an h x w raw RGB image, or ValueError if the runner cannot serve it."""
        img_shape, pad, sf = bm_image_meta(h, w, min(self.resize), max(self.resize))
        if not any(pad[0] <= a and pad[1] <= b for a, b in largest_pad_shapes(self.resize, True)):
            raise ValueError('image %dx%d: the SipMask-benchmark size rule (short side %d, long side at most %d, aspect kept, '
                             'padded to 32) gives %dx%d, outside the padded shapes %s the runner serves'
                             % (h, w, min(self.resize), max(self.resize), pad[0], pad[1],
                                ' / '.join('%dx%d' % s for s in largest_pad_shapes(self.resize, True))))
        f = C.PIL_MAX_DOWNSCALE
        if not (0 < img_shape[0] and 0 < img_shape[1]) or h > f * img_shape[0] or w > f * img_shape[1]:
            raise ValueError('image %dx%d resized to %dx%d by the SipMask-benchmark size rule shrinks more than %dx on an '
                             'axis' % (h, w, img_shape[0], img_shape[1], f))
        return img_shape, pad, sf

    def _out(self, k, eng, oris):
        """Slot k's device / pinned host record for the images of a batch with these ori_shapes: per image a dict of
        views, and per field the number of elements the images use (a prefix of the slot's flat buffers)."""
        mx = eng.max_num
        spec = dict(det=((mx, 5), torch.float32), lab=((mx,), torch.long), cnt=((1,), torch.int32), idx=((mx,), torch.long))
        if not self.rle:
            spec['bits'] = (None, torch.int32)
        if eng.vis:
            spec['trk'] = ((mx, 512), torch.float32)
        if eng.rescoring:
            spec['msc'] = ((mx,), torch.float32)
        if self.render:
            spec['render'] = (None, torch.uint8)
        if k >= len(self.out_dev):
            self.out_dev += [None] * (k + 1 - len(self.out_dev))
            self.out_host += [None] * (k + 1 - len(self.out_host))
        if self.out_dev[k] is None:
            cap = dict(bits=mx * self.max_ori_hw[0] * ((self.max_ori_hw[1] + 31) // 32), render=self.src_elems)
            self.out_dev[k] = {n: torch.empty(self.B * cap.get(n, int(np.prod(s or ()))), dtype=d, device=self.dev)
                               for n, (s, d) in spec.items()}
            self.out_host[k] = {n: torch.empty(v.numel(), dtype=v.dtype).pin_memory() for n, v in self.out_dev[k].items()}
        used = {n: 0 for n in spec}
        dev, host = [], []
        for oh, ow in oris:
            shape = dict((n, s) for n, (s, d) in spec.items())
            if 'bits' in shape:
                shape['bits'] = (mx, oh, (ow + 31) // 32)
            if 'render' in shape:
                shape['render'] = (oh, ow, 3)
            dev.append({})
            host.append({})
            for n, sh in shape.items():
                o, ne = used[n], int(np.prod(sh))
                dev[-1][n] = self.out_dev[k][n][o:o + ne].view(sh)
                host[-1][n] = self.out_host[k][n][o:o + ne].view(sh)
                used[n] = o + ne
        return dev, host, used

    def submit(self, img, meta=None):
        """img: uint8 BGR HWC host image (pinned for an asynchronous upload; RGB for benchmark=True, raw=True), or with
        meta = (img_shape, ori_shape, scale_factor) an fp32 NCHW [1, 3, H, W] preprocessed image (benchmark=True without
        raw).  Validates, uploads the image into the open batch's staging and dispatches the batch when it is due (see the
        class docstring).  Returns the slot (batch=1) or the image's ticket (batch > 1)."""
        if (self.benchmark and not self.bm_raw) != (meta is not None):
            raise ValueError('benchmark=True runners take preprocessed fp32 images with their meta (raw=True: raw uint8 '
                             'RGB images); others raw uint8 images')
        if meta is None:
            if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
                raise ValueError('raw input is a uint8 HWC %s image' % ('RGB' if self.bm_raw else 'BGR'))
            img_shape, pad, sf, ori = self.check(img.shape[:2])
        else:
            if img.dtype != torch.float32 or img.dim() != 4 or img.shape[:2] != (1, 3):
                raise ValueError('preprocessed input is an fp32 [1, 3, H, W] image')
            img_shape, pad, sf, ori = self.check(img.shape[2:], meta)
        if self._open is not None and self._open['pad'] != pad[:2]:
            self._dispatch()                          # a new padded shape closes the open batch before it is staged
        if self._open is None:
            self._open = dict(slot=self.dispatched % self.n, pad=pad[:2], images=[])
            self._begin(self._open['slot'], pad[:2])
        ob = self._open
        m = dict(ticket=self.i, img_shape=img_shape, pad_shape=pad, scale_factor=sf, ori_shape=ori)
        m['src'] = self._stage(ob['slot'], len(ob['images']), img)
        ob['images'].append(m)
        self.i += 1
        if len(ob['images']) == self.B:
            self._dispatch()
        return ob['slot'] if self.B == 1 else m['ticket']

    def _begin(self, k, hw):
        """A batch opens in slot k: its engine exists, and the uploads wait until the slot's previous batch consumed its
        input."""
        self._engine(k, hw)
        self.slots.claim_input(k)

    def _stage(self, k, j, img):
        """Upload image j of slot k's open batch into its staging on the H2D stream; returns the device view."""
        src = self.in_dev[k][j * self.src_elems:j * self.src_elems + img.numel()].view(img.shape)
        self.slots.upload(src, img)
        return src

    def _dispatch(self):
        """Close the open batch: run it in its slot and enqueue the download of its real images' records."""
        ob, self._open = self._open, None
        k, images = ob['slot'], ob['images']
        self._launch(k, ob['pad'], images)
        for m in images:
            m.pop('src', None)
        self.slot_images[k] = images
        self.meta[k] = images[-1]
        self.dispatched += 1
        return k

    def _launch(self, k, pad, images):
        eng = self._engine(k, pad)
        sl = self.slots
        nr = len(images)
        metas = [(m['img_shape'], m['ori_shape'], m['scale_factor']) for m in images]
        cs = sl.begin_compute(k)
        with torch.cuda.stream(cs):
            eng.set_image_meta(metas + [metas[-1]] * (self.B - nr))      # fillers: the last real image's geometry
            if self.rle:
                if self.rle_regions[k] is None:
                    self.rle_regions[k] = torch.zeros(self.B * eng.rle_img_bytes, dtype=torch.uint8).pin_memory()
                eng.set_rle_dest(self.rle_regions[k])
            if self.benchmark and not self.bm_raw:
                eng.img.copy_(images[0]['src'], non_blocking=True)
                eng.forward(None)
            else:
                eng.forward_raw([m['src'] for m in images] + [None] * (self.B - nr), self.mean, self._pipeline)
            if not self.render:
                sl.input_free(k, cs)
            sl.claim_output(k, cs)
            dev, host, used = self._out(k, eng, [m['ori_shape'][:2] for m in images])
            flat = self.out_dev[k]
            mx = eng.max_num
            flat['det'][:used['det']].view(nr, mx, 5).copy_(eng.det[:nr])
            flat['lab'][:used['lab']].view(nr, mx).copy_(eng.labels[:nr])
            flat['cnt'][:nr].copy_(eng.count[:nr])
            flat['idx'][:used['idx']].view(nr, mx).copy_(eng.idx[:nr])
            if 'trk' in flat:
                flat['trk'][:used['trk']].view(nr, mx, 512).copy_(eng.det_track[:nr])
            if 'msc' in flat:
                flat['msc'][:used['msc']].view(nr, mx).copy_(eng.mask_scores[:nr])
            for j, (m, o) in enumerate(zip(images, dev)):
                if 'bits' in o:
                    oh, wq = o['bits'].shape[1:]
                    o['bits'].copy_(eng.mask_bits[j, :, :oh, :wq])
            if self.render:
                # the source images are still in the slot's input staging and the render buffer is claimed output: the
                # input is released only once this has read it
                self._render_batch(k, eng, images, dev)
                sl.input_free(k, cs)
            sl.publish(k, cs)
            self._after_forward(k, eng, images)
        for m, o, h in zip(images, dev, host):
            m['dev'], m['host'] = o, h
        self._download(k, used, images)

    def _render_batch(self, k, eng, images, dev):
        """render=True, on slot k's stream after the record copies: draw each real image of the batch from its staged
        source into its render buffer, from the bucket engine's record."""
        nr = len(images)
        R.draw([(m['src'], o['render'], m['ori_shape'][0], m['ori_shape'][1]) for m, o in zip(images, dev)],
               eng.det[:nr], eng.count[:nr], eng.mask_bits[:nr], L.RENDER_IMAGES, self.render_palette, self.render_thr,
               labels=eng.labels[:nr])

    def _after_forward(self, k, eng, images):
        """Work on slot k's stream right after the batch's forward and record copies, while the bucket engine still holds
        the batch's full record (mask_bits included, also with masks='rle'); the slot's next forward is ordered after it
        and the download does not wait for it.  Nothing here; CocoEvalRunner evaluates the batch."""

    def _download(self, k, used, images):
        """Enqueue the download of slot k's record (the first used[name] elements of every field) once its batch is done."""
        self.slots.download(k, [(self.out_host[k][name][:n], self.out_dev[k][name][:n]) for name, n in used.items()])

    def consume(self, slot, fn):
        """Run fn(record on the device) on the CURRENT stream for every image of the slot's batch, in submission order,
        once the batch is done; the slot is not overwritten before fn's work has finished.  Returns fn's result (batch=1)
        or the list of them."""
        rs = self.slots.hand_over(slot, lambda: [fn(_record(m['dev'])) for m in self.slot_images[slot]])
        return rs[0] if self.B == 1 else rs

    def step(self, img, fn=None, meta=None):
        """submit() + hand the images of the OLDEST batch in flight to fn once in_flight batches are dispatched (see
        EnginePool.step).  Returns what submit() returned."""
        before = self.dispatched
        r = self.submit(img, meta)
        _queue_step(self.pending, self.n, [b % self.n for b in range(before, self.dispatched)], fn, self.consume)
        return r

    def flush(self, fn=None):
        """Dispatch the open batch, hand every batch still pending to fn, and make the current stream wait for the
        downloads."""
        if self._open is not None:
            self.pending.append(self._dispatch())
        _queue_flush(self.pending, fn, self.consume)
        self._join()

    def _join(self):
        self.slots.join()

    def _locate(self, ticket):
        if self._open is not None and any(m['ticket'] == ticket for m in self._open['images']):
            raise ValueError('ticket %d is in the open batch: flush() dispatches it' % ticket)
        for k, images in enumerate(self.slot_images):
            for j, m in enumerate(images):
                if m['ticket'] == ticket:
                    return k, j
        raise ValueError('ticket %d is not held by any slot (never submitted, or its slot was reused)' % ticket)

    def result(self, key):
        """key: the slot submit() returned (batch=1) or the image's ticket (batch > 1).  Blocks until the download
        finished; returns the pinned host record (det_bboxes, det_labels, count, idxs_keep, mask_bits [max, ori_h,
        ceil(ori_w / 32)], track_feats / mask_scores when enabled) and the image's meta.  Valid until the slot is reused.
        masks='rle': segms (the image's RLE dicts, in detection order) in place of mask_bits."""
        k, j = (key, 0) if self.B == 1 else self._locate(key)
        self.slots.wait(k)
        m = self.slot_images[k][j]
        rec = _record(m['host'])
        if self.rle:
            eng = self.engines[k][m['pad_shape'][:2]]
            rec['segms'] = _image_segms(self.rle_regions[k], eng, j, m['ori_shape'][:2], eng.mask_bits)
        rec['meta'] = dict(img_shape=m['img_shape'], pad_shape=m['pad_shape'], ori_shape=m['ori_shape'],
                           scale_factor=m['scale_factor'])
        return rec


# SipMask-VIS test configuration (SipMask-VIS/configs/sipmask/sipmask_r50_caffe_fpn_gn_1x.py)
VIS_ENGINE_KW = dict(vis=True, stacked_convs=3, num_classes=41,
                     test_cfg=dict(nms_pre=200, score_thr=0.03, nms=dict(type='nms', iou_thr=0.5), max_per_img=10))


class VideoRunner(StreamRunner):
    """Serves videos from a SipMask-VIS checkpoint: StreamRunner's frames (any size, batches, resize on the GPU) plus the
    tracker association on the device after every batch, and YouTube-VIS results (tools/test_video.py ->
    results2json_videoseg).

    submit(frame, video_id, frame_id) -> ticket.  A new video starts at frame 0 and takes the lowest free lane of the
    device tracker (tracker.LaneTracker, one tracker state per lane); every later frame must follow the previous one.
    end_video(video_id) frees the lane; its tracker state stays, so that, as in the reference's single tracker, the next
    video on the lane carries it over when its first frame has no detections.  With lanes=1 and the videos submitted in
    dataset order the runner therefore reproduces test_video.py's sequential state.  A new video that takes over a lane
    whose previous video still has frames in the open batch dispatches that batch first, so each lane belongs to one
    video per launch.  Otherwise frames of any videos share batches as in StreamRunner.

    Streams.  Once a batch's record is in the slot's device buffers (ev_out_ready), one tracker stream, shared by all
    slots, associates the batch's frames (one smb_track_assoc_dev launch) and writes their object ids; batches are
    dispatched in submission order, so this stream runs every video's frames in order whatever slot they ran in.  The
    slot's download waits for the association, so the slot is not reused before the association has read its record.
    The tracking features stay on the device: the download is the record without them, the ids and the lanes' status.

    result(ticket) -> the frame's record (without track_feats) plus obj_ids [count] int32, segms (masks='rle') or
    mask_bits ('bits'), and frame, the reference's per-frame pair (ytvis.frame_result).  Valid until the next batch opens
    in the frame's slot.
    An association that overflowed max_objects on the frame's lane raises SmbError naming the video.
    video_json(video_id) -> the video's results2json_videoseg entries (ytvis.video_json), once the video has ended and
    its frames are dispatched.  The runner keeps every frame's pair until then (before a slot takes a new batch, the
    frames it holds are read into their videos) and forgets the video afterwards, so its video_id may be served again.
    For a video whose lane overflowed max_objects, video_json forgets the video and raises SmbError.

    render=True (render_score_thr as StreamRunner's): result() also carries 'render', the frame drawn as SipMask-VIS's
    show_result(is_video=True) draws it (render.render_frames), coloured by the object ids of the association.  The
    source frames are copied into the slot's render buffer before the slot's input is released, and the bucket engine's
    planes into a device buffer of the slot (also with masks='rle'; it is not downloaded); the drawing runs on the tracker
    stream after the association, from the slot's buffers only, before the download that waits for the association."""

    _render_rule = L.RENDER_VIDEO

    def __init__(self, state_dict, lanes=8, batch=1, in_flight=6, resize=(640, 360), keep_ratio=True,
                 max_src_hw=(1920, 1920), max_ori_hw=None, masks='rle', max_objects=4096, match_coeff=(1.0, 2.0, 10.0),
                 **engine_kw):
        from .tracker import LaneTracker
        from .ytvis import VideoBook
        for k, v in VIS_ENGINE_KW.items():
            engine_kw.setdefault(k, v)
        if not engine_kw['vis']:
            raise ValueError('VideoRunner serves SipMask-VIS checkpoints: vis=False is not supported')
        super(VideoRunner, self).__init__(state_dict, in_flight=in_flight, resize=resize, keep_ratio=keep_ratio,
                                          max_src_hw=max_src_hw, max_ori_hw=max_ori_hw, batch=batch, masks=masks, **engine_kw)
        self.num_classes = int(engine_kw['num_classes'])
        self.tracker = LaneTracker(lanes, max_objects, match_coeff, self.dev, max_rows=self.B, depth=2 * self.n + 2)
        self.book = VideoBook(lanes)
        self.s_trk = torch.cuda.Stream(device=self.dev)
        self.s_trk.wait_stream(torch.cuda.current_stream(self.dev))        # the lanes' initial state
        self.ev_assoc = [torch.cuda.Event() for _ in range(self.n)]
        self.ids_dev, self.ids_host = [None] * self.n, [None] * self.n
        self.planes_dev = [None] * self.n           # render=True: per slot, its batch's bit planes for the drawing
        self.status_dev = [torch.zeros(self.tracker.lanes, dtype=torch.int32, device=self.dev) for _ in range(self.n)]
        self.status_host = [torch.zeros(self.tracker.lanes, dtype=torch.int32).pin_memory() for _ in range(self.n)]
        self.rows = {}                      # ticket -> (lane, is_first, video_id, frame_id)
        self.frames = {}                    # video_id -> {frame_id: the frame's (det, seg) pair}
        self.overflowed = set()             # videos with an association beyond max_objects
        self._unread = set()                # dispatched tickets whose pair is not in self.frames yet

    def submit(self, img, video_id, frame_id):
        """img: uint8 BGR HWC host frame of video_id (pinned for an asynchronous upload).  Raises ValueError before
        anything is enqueued for a frame out of order, a new video when every lane is busy, or an image the runner cannot
        serve.  Returns the frame's ticket."""
        lane, first = self.book.check(video_id, frame_id)
        if img.dtype != torch.uint8 or img.dim() != 3 or img.shape[2] != 3:
            raise ValueError('raw input is a uint8 HWC BGR image')
        self.check(img.shape[:2])
        if first and self._open is not None and any(self.rows[m['ticket']][0] == lane for m in self._open['images']):
            self._dispatch()                                # the lane's previous video still has frames in the open batch
        t = self.i
        self.rows[t] = (lane, first, video_id, int(frame_id))
        try:
            super(VideoRunner, self).submit(img)
        except Exception:
            del self.rows[t]
            raise
        self.book.commit(video_id, frame_id, t)
        return t

    def step(self, *args, **kwargs):
        raise TypeError('VideoRunner: use submit(frame, video_id, frame_id) and result(ticket)')

    def end_video(self, video_id):
        """The video has no more frames: its lane is free for the next new video (the lane's state stays)."""
        self.book.end(video_id)

    def _begin(self, k, hw):
        # a batch opens in slot k: read the frames the slot still holds first (an RLE overflow falls back to the bucket
        # engine's planes, and building a new padded-shape engine runs a warm-up forward in the slot's arena); from here on
        # the slot no longer holds them
        self._read_slot(k)
        for m in self.slot_images[k]:
            del self.rows[m['ticket']]
        self.slot_images[k] = []
        super(VideoRunner, self)._begin(k, hw)

    def _launch(self, k, pad, images):
        super(VideoRunner, self)._launch(k, pad, images)
        self._unread.update(m['ticket'] for m in images)

    def _render_batch(self, k, eng, images, dev):
        # the slot's next forward rewrites the bucket engine's planes without waiting for the tracker stream: the drawing
        # after the association reads the slot's own copies of the sources and planes
        if self.planes_dev[k] is None:
            self.planes_dev[k] = torch.empty_like(eng.mask_bits)
        nr = len(images)
        self.planes_dev[k][:nr].copy_(eng.mask_bits[:nr])
        for m, o in zip(images, dev):
            o['render'].copy_(m['src'])

    def _download(self, k, used, images):
        nr = len(images)
        mx = used['lab'] // nr
        if self.ids_dev[k] is None:
            self.ids_dev[k] = torch.empty((self.B, mx), dtype=torch.int32, device=self.dev)
            self.ids_host[k] = torch.empty((self.B, mx), dtype=torch.int32).pin_memory()
        flat, st, trk = self.out_dev[k], self.s_trk, self.tracker
        with torch.cuda.stream(st):
            self.slots.await_record(k, st)
            trk.associate([self.rows[m['ticket']][:2] for m in images], flat['det'][:nr * mx * 5].view(nr, mx, 5),
                          flat['lab'][:nr * mx].view(nr, mx), flat['cnt'][:nr], flat['trk'][:nr * mx * 512].view(nr, mx, 512),
                          ids=self.ids_dev[k][:nr])
            self.status_dev[k].copy_(trk.status)            # this launch's status bits, then clear them for the next
            trk.status.zero_()
            self._after_associate(k, images)
            if self.render:
                R.draw([(m['dev']['render'], m['dev']['render']) + tuple(m['ori_shape'][:2]) for m in images],
                       flat['det'][:nr * mx * 5].view(nr, mx, 5), flat['cnt'][:nr], self.planes_dev[k][:nr],
                       L.RENDER_VIDEO, self.render_palette, self.render_thr, obj_ids=self.ids_dev[k][:nr])
            self.ev_assoc[k].record(st)
        # the tracking features stay on the device
        copies = [(self.out_host[k][name][:n], flat[name][:n]) for name, n in used.items() if name != 'trk']
        self.slots.download(k, copies + [(self.ids_host[k][:nr], self.ids_dev[k][:nr]),
                                         (self.status_host[k], self.status_dev[k])], after=self.ev_assoc[k])

    def _after_associate(self, k, images):
        """Work on the tracker stream right after slot k's batch is associated (its object ids are in ids_dev[k]); the
        slot's download waits for it.  Nothing here; VideoEvalRunner accumulates the batch's overlaps by object id."""

    def _read(self, k, j):
        """Frame j of slot k's batch (downloaded): its record with obj_ids, segms / mask_bits and frame; records the
        frame's pair for its video."""
        from . import rle as R
        from .ytvis import frame_result
        m = self.slot_images[k][j]
        rec = StreamRunner.result(self, k if self.B == 1 else m['ticket'])
        rec.pop('track_feats', None)
        lane, _, video_id, frame_id = self.rows[m['ticket']]
        cnt = int(rec['count'].reshape(-1)[0])
        rec['obj_ids'] = self.ids_host[k][j, :cnt]
        segms = rec['segms'] if self.rle else R.encode_planes(rec['mask_bits'][:cnt].numpy(), m['ori_shape'][:2])
        rec['frame'] = frame_result(rec['det_bboxes'][:cnt].numpy(), rec['det_labels'][:cnt].numpy(),
                                    rec['obj_ids'].numpy(), segms, self.num_classes)
        if int(self.status_host[k][lane]) & TRACK_CAPACITY:
            self.overflowed.add(video_id)
        if m['ticket'] in self._unread:
            self._unread.discard(m['ticket'])
            self.frames.setdefault(video_id, {})[frame_id] = rec['frame']
        return rec, video_id

    def _read_slot(self, k):
        for j, m in enumerate(self.slot_images[k]):
            if m['ticket'] in self._unread:
                self._read(k, j)

    def result(self, ticket):
        k, j = self._locate(ticket)
        rec, video_id = self._read(k, j)
        if video_id in self.overflowed:
            self._raise_overflow(video_id)
        return rec

    def _raise_overflow(self, video_id):
        raise SmbError('video %r: more than max_objects=%d tracked objects on its lane' % (video_id, self.tracker.capacity))

    def video_json(self, video_id):
        """The video's YouTube-VIS result entries (results2json_videoseg), with video_id as given to submit."""
        from .ytvis import video_json
        v = self.book.videos.get(video_id)
        if v is None or not v['ended']:
            raise ValueError('video %r has not ended: end_video() first' % (video_id,))
        if self._open is not None and any(m['ticket'] in v['frames'] for m in self._open['images']):
            raise ValueError('video %r has frames in the open batch: flush() dispatches them' % (video_id,))
        for k in range(self.n):
            self._read_slot(k)
        got = self.frames.pop(video_id, {})            # the runner forgets the video, also when it overflowed
        del self.book.videos[video_id]
        if video_id in self.overflowed:
            self.overflowed.discard(video_id)
            self._raise_overflow(video_id)
        return video_json(video_id, [got[f] for f in range(len(v['frames']))])


class CocoEvalRunner(StreamRunner):
    """StreamRunner plus COCO box and mask AP (pycocotools COCOeval, as CocoDataset.evaluate runs it) from the stream.

    submit(img, image_id[, meta]) checks the image against the ground truth (known id, not submitted before, ori_shape
    equal to the annotation's height x width) before anything is enqueued, then packs the image's ground truth (a
    malformed segmentation raises here) and uploads it from pinned memory on the H2D stream with the image; its planes are
    rasterized on the device.  Right after each batch's forward, on the
    slot's stream, the batch's real images are evaluated from the bucket engine's record (cocoeval.CocoEvaluator
    .add_records: the result json's values, IoU and matching on the device).  flush() dispatches the open batch;
    evaluate() accumulates and summarizes every image submitted so far and returns MM's evaluate() dict plus the raw
    stats and arrays.  result(ticket) still returns each record, so the result json can be written as well.
      gt      : cocoeval.CocoGroundTruth; cat_ids: COCO category id per 0-based label (as coco.coco_json takes it)
      metrics : 'bbox', 'segm' and / or 'proposal' (MM's class-agnostic AR@100 / 300 / 1000 of the boxes and box scores,
                matched on the slot's stream like the others; not on SipMask-benchmark checkpoints)
      params  : cocoeval.CocoParams or CocoParams2 for 'bbox' / 'segm' (None: COCOeval's default Params), e.g. a
                cat_ids subset
      proposal_nums: the maxDets of 'proposal' (a record holds at most max_per_img detections, as the bbox json does)
      analyze : also run coco_error_analysis.py's matches after every batch; evaluate() then returns its arrays under
                'analysis' (cocoeval.CocoEvaluator)
    Every other argument is StreamRunner's; SipMask-VIS (vis=True) is not supported."""

    def __init__(self, state_dict, gt, cat_ids, metrics=('bbox', 'segm'), params=None, analyze=False,
                 proposal_nums=(100, 300, 1000), **kw):
        from .cocoeval import CocoEvaluator, CocoParams, check_metrics
        check_metrics(metrics)                            # names raise before the engines are built
        if kw.get('vis'):
            raise ValueError('CocoEvalRunner: YouTube-VIS evaluation (vis=True) is not supported')
        if params is not None and not isinstance(params, CocoParams):
            raise ValueError('CocoEvalRunner: params must be a cocoeval.CocoParams')
        if analyze:
            gt.supercategory_index()                      # raises before the engines are built
        super(CocoEvalRunner, self).__init__(state_dict, **kw)
        self.evaluator = CocoEvaluator(gt, cat_ids, metrics=metrics, benchmark=self.benchmark, device=self.dev,
                                       params=params, analyze=analyze, proposal_nums=proposal_nums)
        torch.cuda.current_stream(self.dev).synchronize()   # the evaluator's zeroed state, before the slots use it
        self._eval_rows = {}                # ticket -> (image id, its staged ground truth) until its batch is evaluated
        self._submitted = set()

    def submit(self, img, image_id, meta=None):
        """img / meta as StreamRunner.submit; image_id: the image's COCO id.  Returns what StreamRunner.submit returns."""
        image_id = int(image_id)
        ori = tuple(meta[1][:2]) if meta is not None else tuple(img.shape[:2])
        if image_id in self._submitted:
            raise ValueError('image id %d is evaluated twice' % image_id)
        self.evaluator.check_image(image_id, ori)
        t = self.i
        self._eval_rows[t] = (image_id, self.evaluator.stage_gt(image_id, self.slots.h2d))
        try:
            r = super(CocoEvalRunner, self).submit(img, meta)
        except Exception:
            self._eval_rows.pop(t, None)
            raise
        self._submitted.add(image_id)
        return r

    def step(self, *args, **kwargs):
        raise TypeError('CocoEvalRunner: use submit(img, image_id), flush() and evaluate()')

    def _after_forward(self, k, eng, images):
        rec = dict(det_bboxes=eng.det, det_labels=eng.labels, count=eng.count, mask_bits=eng.mask_bits)
        if eng.rescoring:
            rec['mask_scores'] = eng.mask_scores
        ids, gts = zip(*[self._eval_rows.pop(m['ticket']) for m in images])
        self.evaluator.add_records(rec, eng.geom, list(ids), [m['ori_shape'] for m in images], gts=list(gts))

    def finish(self):
        """Dispatch the open batch and make the current stream wait for every slot's evaluation: the evaluator then holds
        every image submitted (its state() can be gathered across ranks)."""
        self.flush()
        self.slots.join(*self.slots.streams)

    def evaluate(self, classwise=False):
        """finish() and return CocoEvaluator.evaluate(classwise)'s dict."""
        self.finish()
        return self.evaluator.evaluate(classwise)


class VideoEvalRunner(VideoRunner):
    """VideoRunner plus YouTube-VIS mask AP (YTVOSeval, as SipMask-VIS's ytvos_eval runs it) from the stream.

    submit(frame, video_id, frame_id) takes the video's YouTube-VIS id and checks the frame against the ground truth
    (known video, its height x width, a frame inside its length, a video not evaluated before) before anything is
    enqueued; it then packs the frame's ground truth and uploads it on the H2D stream with the frame (the planes are
    rasterized on the device, with the frame's overlaps).
      - Right after each batch's forward, on the slot's stream: every detection's pixel count and its intersections with
        the frame's ground-truth objects (ytviseval kernel a), from the bucket engine's planes.
      - Right after the association, on the tracker stream: the last detection of each object id is added into its
        video's accumulators (kernel b).  Each video being evaluated holds one of `eval_slots` accumulator slots (default
        2 x lanes) from its frame 0 until its sequence match; when none is free, the ended videos are matched first.
      - Once a video has ended and its frames are read, its result json (VideoRunner.video_json) gives every object's
        score and category, and one launch on the tracker stream matches it (kernel c).
    end_video(video_id) raises ValueError unless the video got exactly its annotated number of frames.  evaluate()
    dispatches the open batch, matches every ended video and returns YtvisEvaluator.evaluate()'s dict; every video
    submitted must have ended.  video_json(video_id) returns what VideoRunner returns, also for a video already matched
    (the runner keeps the entries of matched videos until they are asked for).
      gt        : ytviseval.YtvisGroundTruth
      cat_ids   : the category ids the results carry (default 1 .. num_classes - 1, label + 1 as video_json writes)
      max_gts   : ground-truth objects per video the accumulators hold
    A video whose lane overflowed max_objects raises SmbError from video_json and evaluate(), as in VideoRunner.  Every
    other argument is VideoRunner's."""

    def __init__(self, state_dict, gt, cat_ids=None, eval_slots=None, max_gts=64, **kw):
        from .ytviseval import YtvisEvaluator
        super(VideoEvalRunner, self).__init__(state_dict, **kw)
        slots = int(eval_slots) if eval_slots is not None else 2 * self.tracker.lanes
        if slots < self.tracker.lanes:
            raise ValueError('eval_slots=%d: at least one accumulator slot per lane (%d)' % (slots, self.tracker.lanes))
        cats = range(1, self.num_classes) if cat_ids is None else cat_ids
        with torch.cuda.stream(self.s_trk):
            self.evaluator = YtvisEvaluator(gt, cats, slots=slots, objects=self.tracker.capacity, max_gts=max_gts,
                                            device=self.dev)
        self.s_trk.synchronize()            # the evaluator's zeroed state, before the slots use it
        self._free = list(range(slots))     # accumulator slots not held by a video
        self._vslot = {}                    # video id -> its accumulator slot until its sequence match
        self._staged = {}                   # ticket -> its frame's staged ground truth until the batch's overlaps
        self._ovl = [None] * self.n         # per slot: its batch's overlaps, until the association adds them up
        self.ev_ovl = [torch.cuda.Event() for _ in range(self.n)]
        self._json = {}                     # matched video -> its result entries, until video_json asks for them

    def submit(self, img, video_id, frame_id):
        frame_id = int(frame_id)
        if img.dim() != 3:
            raise ValueError('raw input is a uint8 HWC BGR image')
        self.evaluator.check_frame(video_id, frame_id, tuple(img.shape[:2]))
        _, first = self.book.check(video_id, frame_id)
        if first:
            slot = self._acquire()
            self._vslot[video_id] = slot
            with torch.cuda.stream(self.s_trk):     # after the previous holder's sequence match
                self.evaluator.begin_video(video_id, slot)
        t = self.i
        try:
            staged = self._staged[t] = self.evaluator.stage_frame(video_id, frame_id, self.slots.h2d)
            super(VideoEvalRunner, self).submit(img, video_id, frame_id)
        except Exception:
            self._staged.pop(t, None)
            if first:
                self.evaluator.abort_video(video_id)
                self._free.append(self._vslot.pop(video_id))
            raise
        self.evaluator.commit_frame(staged)
        return t

    def _acquire(self):
        if not self._free:
            ended = [v for v in self._vslot if self.book.videos[v]['ended']]
            if ended and self._open is not None:
                self._dispatch()
            for v in ended:
                self._finish(v)
        if not self._free:
            raise ValueError('all %d accumulator slots hold videos that have not ended' % self.evaluator.slots)
        return self._free.pop(0)

    def end_video(self, video_id):
        v = self.book.videos.get(video_id)
        if v is not None and not v['ended'] and video_id in self._vslot:
            n = self.evaluator.gt.videos[video_id]['length']
            if len(v['frames']) != n:
                raise ValueError('video %r ends after %d frames, the annotation has %d' % (video_id, len(v['frames']), n))
        super(VideoEvalRunner, self).end_video(video_id)

    def _after_forward(self, k, eng, images):
        nr, mx = len(images), eng.max_num
        cap_h, words = eng.mask_bits.shape[2:]
        plane = cap_h * words
        base = eng.mask_bits.data_ptr()
        staged = [self._staged.pop(m['ticket']) for m in images]
        self._ovl[k] = self.evaluator.overlap(staged, [base + 4 * j * mx * plane for j in range(nr)], plane, words, mx,
                                              count=eng.count)
        self.ev_ovl[k].record(torch.cuda.current_stream(self.dev))

    def _after_associate(self, k, images):
        ovl, self._ovl[k] = self._ovl[k], None
        self.s_trk.wait_event(self.ev_ovl[k])
        nr = len(images)
        self.evaluator.scatter(ovl, self.ids_dev[k][:nr], count=self.out_dev[k]['cnt'][:nr])

    def _finish(self, video_id):
        """Read the ended video's result entries and enqueue its sequence match on the tracker stream."""
        for k in range(self.n):
            self._read_slot(k)
        fr = self.frames.get(video_id, {})
        obj_ids = list(dict.fromkeys(oid for f in sorted(fr) for oid in fr[f][0]))     # video_json's entry order
        try:
            entries = VideoRunner.video_json(self, video_id)
        except SmbError:
            self.evaluator.abort_video(video_id)
            self._free.append(self._vslot.pop(video_id))
            raise
        slot = self._vslot.pop(video_id)
        self._json[video_id] = entries
        try:
            with torch.cuda.stream(self.s_trk):
                self.evaluator.end_video(video_id, entries, obj_ids)
        except ValueError:
            self.evaluator.abort_video(video_id)
            raise
        finally:
            self._free.append(slot)

    def video_json(self, video_id):
        if video_id not in self._json:
            if video_id not in self._vslot:
                return super(VideoEvalRunner, self).video_json(video_id)
            self._finish(video_id)
        return self._json.pop(video_id)

    def evaluate(self):
        """Dispatch the open batch, match every ended video, wait for the slot and tracker streams and return
        YtvisEvaluator.evaluate()'s dict."""
        self.flush()
        open_videos = [v for v in self._vslot if not self.book.videos[v]['ended']]
        if open_videos:
            raise ValueError('video %r has not ended: end_video() first' % (open_videos[0],))
        for v in list(self._vslot):
            self._finish(v)
        self.slots.join(*self.slots.streams, self.s_trk)
        return self.evaluator.evaluate()
