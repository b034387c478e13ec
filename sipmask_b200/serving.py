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
import torch

from . import conv as C
from .engine import SipMaskEngine

# grid cap / planner min_tiles per number of images in flight
_TUNING = {1: dict(max_ctas=None, head_max_ctas=None, min_tiles=48)}


def _tuning(n):
    if n in _TUNING:
        return dict(_TUNING[n])
    cap = 48 if n >= 6 else 64
    return dict(max_ctas=cap, head_max_ctas=cap, min_tiles=16)


def make_engines(state_dict, img_hw, in_flight=1, **kw):
    """n engines for n images in flight (weights shared, activations private)."""
    tune = _tuning(in_flight)
    prev = C.set_min_tiles(kw.pop('min_tiles', tune.pop('min_tiles')))
    for k, v in tune.items():
        kw.setdefault(k, v)
    try:
        engs = []
        for i in range(in_flight):
            engs.append(SipMaskEngine(state_dict, img_hw, share_weights=engs[0] if engs else None, **kw))
    finally:
        C.set_min_tiles(prev)
    return engs


class EnginePool(object):
    """Round-robin replay of n resident engines on n streams (inputs already in each engine's `img`)."""

    def __init__(self, engines):
        self.engs = list(engines)
        self.n = len(self.engs)
        dev = self.engs[0].dev
        self.dev = dev
        self.streams = [torch.cuda.Stream(device=dev) for _ in self.engs]
        self.ev_done = [torch.cuda.Event() for _ in self.engs]
        self.ev_consumed = [torch.cuda.Event() for _ in self.engs]
        self.i = 0
        self.pending = []
        cur = torch.cuda.current_stream(dev)
        for st, eng in zip(self.streams, self.engs):
            st.wait_stream(cur)
            with torch.cuda.stream(st):
                eng.forward(None)                  # warm-up + graph capture on the engine's own stream
                eng.forward(None)
        for st in self.streams:
            st.synchronize()
        for e in self.ev_consumed:
            e.record(cur)

    def launch(self):
        """Enqueue one image on the next engine; returns its index.  Does not block the host."""
        k = self.i % self.n
        st = self.streams[k]
        st.wait_event(self.ev_consumed[k])
        with torch.cuda.stream(st):
            self.engs[k].forward(None)
        self.ev_done[k].record(st)
        self.i += 1
        return k

    def consume(self, k, fn):
        """Run fn(engine_k_outputs) on the CURRENT stream once image k is done; engine k is not replayed again before fn's
        work has finished (used for the all-gather of the detection record)."""
        cur = torch.cuda.current_stream(self.dev)
        cur.wait_event(self.ev_done[k])
        eng = self.engs[k]
        r = fn(eng._result())
        self.ev_consumed[k].record(cur)
        return r

    def step(self, fn=None):
        """One image: launch it, and (if fn is given) hand the OLDEST image in flight to fn on the current stream, so the
        consumer (e.g. the all-gather) never stalls the images behind it."""
        self.pending.append(self.launch())
        if fn is not None and len(self.pending) >= self.n:
            self.consume(self.pending.pop(0), fn)

    def flush(self, fn=None):
        """Consume what is still in flight and make the current stream wait for all of it."""
        while self.pending:
            k = self.pending.pop(0)
            if fn is not None:
                self.consume(k, fn)
        self.join()

    def join(self):
        """Make the current stream wait for everything in flight."""
        cur = torch.cuda.current_stream(self.dev)
        for st in self.streams:
            cur.wait_stream(st)


class PipelinedRunner(object):
    """raw_hw=(h, w): the host hands over the decoder's uint8 BGR HWC image (h*w*3 bytes H2D instead of 4*3*H*W) and the
    step starts with the fused resize / normalise / pad kernel (engine.forward_raw, SURVEY 8f-3)."""

    def __init__(self, engines, depth=2, raw_hw=None):
        self.engs = list(engines) if isinstance(engines, (list, tuple)) else [engines]
        self.n = len(self.engs)
        self.eng = engine = self.engs[0]
        # one staging slot per engine when several images are in flight, `depth` slots for a single engine
        self.nslots = self.n if self.n > 1 else depth
        ns = self.nslots
        dev = engine.dev
        self.dev = dev
        self.s_h2d = torch.cuda.Stream(device=dev)
        self.s_d2h = torch.cuda.Stream(device=dev)
        self.s_comp = [torch.cuda.Stream(device=dev) for _ in self.engs] if self.n > 1 else [None]
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
        self.out_host = [{k: torch.empty(v.shape, dtype=v.dtype).pin_memory() for k, v in o.items()} for o in self.out_dev]
        self.ev_in_ready = [torch.cuda.Event() for _ in range(ns)]      # H2D of slot finished
        self.ev_in_free = [torch.cuda.Event() for _ in range(ns)]       # compute consumed the slot's input
        self.ev_out_ready = [torch.cuda.Event() for _ in range(ns)]     # compute wrote the slot's output
        self.ev_out_free = [torch.cuda.Event() for _ in range(ns)]      # D2H of slot finished
        self.ev_hold = [None] * ns                                      # optional: a consumer still reads out_dev[slot]
        self.i = 0
        self.pending = []
        self.h2d_bytes = self.in_dev[0].numel() * self.in_dev[0].element_size()
        self.d2h_bytes = sum(v.numel() * v.element_size() for v in self.out_dev[0].values())
        cur = torch.cuda.current_stream(dev)
        if self.n > 1:
            for st, eng in zip(self.s_comp, self.engs):
                st.wait_stream(cur)
                with torch.cuda.stream(st):
                    self._fwd(eng, 0)              # warm-up + graph capture on the engine's own stream
                    self._fwd(eng, 0)
            for st in self.s_comp:
                st.synchronize()
        else:
            self._fwd(engine, 0)
            self._fwd(engine, 0)
            cur.synchronize()
        for e in self.ev_in_free + self.ev_out_free:
            e.record(cur)

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
        cur = torch.cuda.current_stream(self.dev)
        cs = self.s_comp[k % self.n] or cur
        with torch.cuda.stream(self.s_h2d):
            self.s_h2d.wait_event(self.ev_in_free[k])
            self.in_dev[k].copy_(host_img, non_blocking=True)
            self.ev_in_ready[k].record(self.s_h2d)
        with torch.cuda.stream(cs):
            cs.wait_event(self.ev_in_ready[k])
            if self.raw:
                eng.forward_raw(self.in_dev[k])            # preprocess kernel reads the staged uint8 image, then the graph
                self.ev_in_free[k].record(cs)
            else:
                eng.img.copy_(self.in_dev[k], non_blocking=True)
                self.ev_in_free[k].record(cs)
                eng.forward(None)
            cs.wait_event(self.ev_out_free[k])
            if self.ev_hold[k] is not None:
                cs.wait_event(self.ev_hold[k])
            o = self.out_dev[k]
            o['det'].copy_(eng.det, non_blocking=True)
            o['lab'].copy_(eng.labels, non_blocking=True)
            o['cnt'].copy_(eng.count, non_blocking=True)
            o['bits'].copy_(eng.mask_bits, non_blocking=True)
            if 'trk' in o:
                o['trk'].copy_(eng.det_track, non_blocking=True)
            self.ev_out_ready[k].record(cs)
        with torch.cuda.stream(self.s_d2h):
            self.s_d2h.wait_event(self.ev_out_ready[k])
            for name in o:
                self.out_host[k][name].copy_(o[name], non_blocking=True)
            self.ev_out_free[k].record(self.s_d2h)
        self.i += 1
        return k

    def consume(self, slot, fn):
        """Run fn(slot's device record) on the CURRENT stream once it is ready; the slot is not overwritten before fn's
        work has finished (used for the all-gather of the detection record)."""
        cur = torch.cuda.current_stream(self.dev)
        cur.wait_event(self.ev_out_ready[slot])
        o = self.out_dev[slot]
        rec = dict(det_bboxes=o['det'], det_labels=o['lab'], count=o['cnt'], mask_bits=o['bits'])
        if 'trk' in o:
            rec['track_feats'] = o['trk']
        r = fn(rec)
        if self.ev_hold[slot] is None:
            self.ev_hold[slot] = torch.cuda.Event()
        self.ev_hold[slot].record(cur)
        return r

    def step(self, host_img, fn=None):
        """submit() + hand the OLDEST slot in flight to fn (see EnginePool.step).  Returns the submitted slot."""
        k = self.submit(host_img)
        self.pending.append(k)
        if fn is not None and len(self.pending) >= self.nslots:
            self.consume(self.pending.pop(0), fn)
        elif fn is None:
            self.pending.clear()
        return k

    def flush(self, fn=None):
        while self.pending:
            k = self.pending.pop(0)
            if fn is not None:
                self.consume(k, fn)
        self.join()

    def result(self, slot):
        """Blocks until the slot's download finished; returns pinned host tensors (valid until the slot is reused)."""
        self.ev_out_free[slot].synchronize()
        return self.out_host[slot]

    def join(self):
        """Make the current stream wait for the downloads (and so for every image in flight)."""
        torch.cuda.current_stream(self.dev).wait_stream(self.s_d2h)

    def drain(self):
        self.s_d2h.synchronize()
        self.s_h2d.synchronize()
