"""SipMask-VIS tracker association on gathered detection records (SURVEY 8f-2).

Replaces the stateful tail of `SipMaskHead.get_bboxes` in SipMask-VIS (VIS/mmdet/models/anchor_heads/sipmask_head.py:612-667,
`compute_comp_scores` :544-562, `bbox_overlaps` core/bbox/geometry.py:4-63).  The association is inherently sequential in
frame order and tiny (<= max_per_img = 10 detections x a few dozen tracked objects), so it is a vectorised HOST step on the
records the GPUs produced: boxes / labels from the fixed-shape detection record, 512-d box-centre features gathered on the
device (`smb_gather_track_feats`) and shipped with the record.  Frames of a clip may be sharded over GPUs; after the
end-of-run all-gather every rank (or rank 0) runs this in frame order.

    comp = log_softmax([0 | feats . prev_feats^T]) + 1.0 * log(score) + 2.0 * [0 | IoU(+1)] + 10 * [1 | label equal]
    argmax == 0 -> new object id (appended); otherwise the detection claims object argmax-1 if its comp score beats the best
    claim so far (earlier claimants keep the id they were given - reference behaviour), and the object's stored feature / box
    are replaced by the claimant's (the stored label is not).
"""
import numpy as np


def bbox_overlaps(b1, b2):
    lt = np.maximum(b1[:, None, :2], b2[None, :, :2])
    rb = np.minimum(b1[:, None, 2:4], b2[None, :, 2:4])
    wh = np.clip(rb - lt + np.float32(1), 0, None)
    overlap = wh[:, :, 0] * wh[:, :, 1]
    a1 = (b1[:, 2] - b1[:, 0] + np.float32(1)) * (b1[:, 3] - b1[:, 1] + np.float32(1))
    a2 = (b2[:, 2] - b2[:, 0] + np.float32(1)) * (b2[:, 3] - b2[:, 1] + np.float32(1))
    return overlap / (a1[:, None] + a2[None, :] - overlap)


def log_softmax(x):
    m = x.max(axis=1, keepdims=True)
    z = x - m
    return z - np.log(np.exp(z).sum(axis=1, keepdims=True))


class Tracker(object):
    """native=True (default when the library is present): the per-frame step runs in C (`smb_track_step`, ~2 us instead of
    ~150 us of numpy calls - at 8 GPUs the python version was the bottleneck of a clip); the numpy implementation below is the
    same algorithm and is what `native=False` runs."""

    def __init__(self, match_coeff=(1.0, 2.0, 10.0), native=True, capacity=4096, feat_dim=512):
        self.match_coeff = tuple(np.float32(c) for c in match_coeff)
        self.prev_roi_feats = self.prev_bboxes = self.prev_det_labels = None
        self.native = native
        self.capacity, self.feat_dim = capacity, feat_dim
        if native:
            import ctypes
            from . import _lib as L
            self._L, self._ct = L, ctypes
            self._coef = np.asarray(self.match_coeff, np.float32)
            self._pd = np.zeros((capacity, 5), np.float32)
            self._pl = np.zeros((capacity,), np.int64)
            self._pf = np.zeros((capacity, feat_dim), np.float32)
            self._np = -1                                   # -1: no state yet (first frame of a video)
            self._fn = L.lib().smb_track_step
            self._state_ptrs = [ctypes.c_void_p(a.ctypes.data) for a in (self._pd, self._pl, self._pf, self._coef)]

    def reset(self):
        self.prev_roi_feats = self.prev_bboxes = self.prev_det_labels = None
        if self.native:
            self._np = -1

    @property
    def num_objects(self):
        return max(self._np, 0) if self.native else (0 if self.prev_bboxes is None else self.prev_bboxes.shape[0])

    def _step_native(self, det, lab, feats, is_first):
        ct, n = self._ct, det.shape[0]
        if n == 0:
            return np.zeros((0,), np.int32)
        assert feats.shape[1] == self.feat_dim
        det, lab, feats = np.ascontiguousarray(det), np.ascontiguousarray(lab), np.ascontiguousarray(feats)
        if is_first or self._np < 0:
            assert n <= self.capacity
            self._pd[:n], self._pl[:n], self._pf[:n] = det, lab, feats
            self._np = n
            return np.arange(n, dtype=np.int32)
        ids = np.empty((n,), np.int32)
        vp = ct.c_void_p
        r = self._fn(vp(det.ctypes.data), vp(lab.ctypes.data), vp(feats.ctypes.data), n, self.feat_dim, self._state_ptrs[0],
                     self._state_ptrs[1], self._state_ptrs[2], self._np, self.capacity, self._state_ptrs[3], vp(ids.ctypes.data))
        self._L.check(r if r < 0 else 0, 'smb_track_step')
        self._np = r
        return ids

    def step(self, det_bboxes, det_labels, det_roi_feats, is_first):
        """det_bboxes [n,5] f32 (x1,y1,x2,y2,score), det_labels [n] int, det_roi_feats [n,512] f32 -> det_obj_ids [n] int32."""
        det = np.asarray(det_bboxes, np.float32)
        lab = np.asarray(det_labels, np.int64)
        feats = np.asarray(det_roi_feats, np.float32)
        if self.native:
            return self._step_native(det, lab, feats, is_first)
        n = det.shape[0]
        if n == 0:
            return np.zeros((0,), np.int32)
        if is_first or self.prev_bboxes is None:
            self.prev_bboxes, self.prev_roi_feats, self.prev_det_labels = det.copy(), feats.copy(), lab.copy()
            return np.arange(n, dtype=np.int32)
        prod = feats @ self.prev_roi_feats.T
        score = np.concatenate([np.zeros((n, 1), np.float32), prod], 1)
        ll = log_softmax(score)
        delta = np.concatenate([np.ones((n, 1), np.float32), (self.prev_det_labels[None, :] == lab[:, None]).astype(np.float32)], 1)
        iou = np.concatenate([np.zeros((n, 1), np.float32), bbox_overlaps(det[:, :4], self.prev_bboxes[:, :4])], 1)
        c0, c1, c2 = self.match_coeff
        comp = ll + c0 * np.log(det[:, 4:5]) + c1 * iou + c2 * delta
        match_ids = comp.argmax(axis=1)
        ids = -np.ones(n, np.int32)
        best = -100.0 * np.ones(self.prev_bboxes.shape[0])
        for i, mid in enumerate(match_ids):
            if mid == 0:
                ids[i] = self.prev_roi_feats.shape[0]
                self.prev_roi_feats = np.concatenate([self.prev_roi_feats, feats[i:i + 1]], 0)
                self.prev_bboxes = np.concatenate([self.prev_bboxes, det[i:i + 1]], 0)
                self.prev_det_labels = np.concatenate([self.prev_det_labels, lab[i:i + 1]], 0)
            else:
                obj = int(mid) - 1
                if comp[i, mid] > best[obj]:
                    ids[i] = obj
                    best[obj] = comp[i, mid]
                    self.prev_roi_feats[obj] = feats[i]
                    self.prev_bboxes[obj] = det[i]
        return ids


class LaneTracker(object):
    """The association on the DEVICE (smb_track_assoc_dev): `lanes` videos, each with its tracker state in device memory
    (boxes [lanes, capacity, 5], labels [lanes, capacity], features [lanes, capacity, 512], n_obj [lanes] (-1: no state
    yet), status [lanes]).  associate() enqueues one launch for a batch of frame records on the current stream; the frame
    rows go through pinned staging (a ring of `depth` buffers, each reused only after the event of its last launch) and one
    stream-ordered H2D copy, as the engine's geometry rows do.  Nothing here waits for the device except that reuse."""

    def __init__(self, lanes, capacity=4096, match_coeff=(1.0, 2.0, 10.0), device='cuda', max_rows=64, depth=16):
        import torch
        self.lanes, self.capacity, self.max_rows = int(lanes), int(capacity), int(max_rows)
        if self.lanes < 1 or self.capacity < 1 or self.max_rows < 1:
            raise ValueError('LaneTracker: lanes, capacity and max_rows must be positive')
        self.match_coeff = tuple(float(np.float32(c)) for c in match_coeff)
        self.dev = torch.device(device)
        if self.dev.index is None:
            self.dev = torch.device('cuda', torch.cuda.current_device())
        L, C = self.lanes, self.capacity
        self.boxes = torch.zeros((L, C, 5), dtype=torch.float32, device=self.dev)
        self.labels = torch.zeros((L, C), dtype=torch.int64, device=self.dev)
        self.feats = torch.zeros((L, C, 512), dtype=torch.float32, device=self.dev)
        self.n_obj = torch.full((L,), -1, dtype=torch.int32, device=self.dev)
        self.status = torch.zeros((L,), dtype=torch.int32, device=self.dev)
        self.state = dict(boxes=self.boxes, labels=self.labels, feats=self.feats, n_obj=self.n_obj, status=self.status)
        self._host = [torch.empty((self.max_rows, 2), dtype=torch.int32).pin_memory() for _ in range(depth)]
        self._rows = [torch.empty((self.max_rows, 2), dtype=torch.int32, device=self.dev) for _ in range(depth)]
        self._ev = [None] * depth
        self._i = 0
        self._ws = {}                                  # max_num -> workspace

    def associate(self, rows, det, labels, count, track_feats, ids=None):
        """rows: one (lane, is_first) per frame of the batch (lane < 0: a filler, skipped); det [N, max, 5], labels
        [N, max] int64, count int32 [N], track_feats [N, max, 512] on the device.  Enqueues the association on the current
        stream and returns ids int32 [N, max] (written when it runs)."""
        import torch
        from . import ops
        n = len(rows)
        if n > self.max_rows:
            raise ValueError('LaneTracker: %d frame rows, max_rows is %d' % (n, self.max_rows))
        for lane, _ in rows:
            if int(lane) >= self.lanes:
                raise ValueError('LaneTracker: lane %d of %d' % (int(lane), self.lanes))
        s = self._i % len(self._host)
        self._i += 1
        if self._ev[s] is not None:
            self._ev[s].synchronize()                  # the launch that last read this staging has run
        host, dev = self._host[s], self._rows[s]
        h = host.numpy()
        for r, (lane, first) in enumerate(rows):
            h[r, 0], h[r, 1] = int(lane), int(bool(first))
        dev[:n].copy_(host[:n], non_blocking=True)
        mx = det.shape[1]
        ws = self._ws.get(mx)
        if ws is None:
            ws = self._ws[mx] = torch.empty(ops.track_assoc_workspace_bytes(self.lanes, mx, self.capacity),
                                            dtype=torch.uint8, device=self.dev)
        ids = ops.track_assoc(dev[:n], det, labels, count, track_feats, self.state, self.match_coeff, ids=ids, workspace=ws)
        if self._ev[s] is None:
            self._ev[s] = torch.cuda.Event()
        self._ev[s].record(torch.cuda.current_stream(self.dev))
        return ids
