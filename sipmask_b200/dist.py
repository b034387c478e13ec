"""The one collective of the path: an all-gather of the fixed-shape detection record (SURVEY.md §8e).

The reference gathers *pickled python results* with two NCCL all_gathers (sizes, then padded payload;
MM/mmdet/apis/test.py:117-147).  Here every rank contributes one [max_per_img, 7] fp32 record
(x1, y1, x2, y2, score, label, valid) per image, so a single `all_gather_into_tensor` suffices and the shape is static
(CUDA-graph friendly).  Images are sharded one per GPU; there is no other communication on the path.
"""
import torch
import torch.distributed as dist


def pack_record(det_bboxes, det_labels, count):
    """det_bboxes [max,5] f32, det_labels [max] i64, count int32 tensor [1] (device) -> [max,7] f32."""
    max_num = det_bboxes.shape[0]
    valid = (torch.arange(max_num, device=det_bboxes.device) < count.to(torch.long)).to(det_bboxes.dtype)
    return torch.cat([det_bboxes, det_labels.to(det_bboxes.dtype).unsqueeze(1), valid.unsqueeze(1)], 1)


def gather_records(record, out=None):
    """record [max,7] -> [world, max,7] on every rank (one collective)."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return record.unsqueeze(0)
    if out is None:
        out = record.new_empty((world,) + tuple(record.shape))
    if dist.get_backend() == 'nccl':
        dist.all_gather_into_tensor(out, record.contiguous())
    else:                                             # gloo (CPU tests)
        parts = [torch.empty_like(record) for _ in range(world)]
        dist.all_gather(parts, record.contiguous())
        out.copy_(torch.stack(parts, 0))
    return out


def unpack_records(gathered):
    """[world,max,7] -> list over ranks of (det_bboxes [k,5], det_labels [k] int64) in rank (= image) order."""
    res = []
    for r in range(gathered.shape[0]):
        rec = gathered[r]
        k = int(rec[:, 6].sum().item())
        res.append((rec[:k, :5].clone(), rec[:k, 5].to(torch.long)))
    return res


class RecordLog(object):
    """Detection records of a whole run, gathered ONCE at the end (north_star: "a single NCCL all-gather of detections at
    the end only").  `append` writes one image's [max,7] record into the next row of a device buffer on the caller's stream
    (no communication); `gather` is the single collective: [cap,max,7] per rank -> [world,cap,max,7] on every rank.
    Per-image gathering (`gather_records` after every image) put a latency-bound 2.8 KB collective on the critical path of
    every step (r1: scaling efficiency 0.96 already at 2 GPUs)."""

    def __init__(self, capacity, max_num, device, feat_dim=0):
        """feat_dim > 0 (SipMask-VIS): every record row also carries the detection's tracking feature, [max, 7 + feat_dim]
        (SURVEY 8e: "+ [10,512] track features = 20 KB")."""
        self.buf = torch.zeros((capacity, max_num, 7 + feat_dim), dtype=torch.float32, device=device)
        self.cap, self.n = capacity, 0
        self._ar = torch.arange(max_num, device=device).view(max_num, 1)

    def append(self, det_bboxes, det_labels, count, feats=None):
        row = self.buf[self.n % self.cap]
        row[:, :5].copy_(det_bboxes, non_blocking=True)
        row[:, 5:6].copy_(det_labels.view(-1, 1), non_blocking=True)
        row[:, 6:7].copy_(self._ar < count.view(1, 1), non_blocking=True)
        if feats is not None:
            row[:, 7:].copy_(feats, non_blocking=True)
        self.n += 1

    def reset(self):
        self.n = 0

    def gather(self, out=None):
        """-> [world, cap, max, 7]; rows >= number of appended images are stale / zero."""
        world = dist.get_world_size() if dist.is_initialized() else 1
        if world == 1:
            return self.buf.unsqueeze(0)
        if out is None:
            out = self.buf.new_empty((world,) + tuple(self.buf.shape))
        if dist.get_backend() == 'nccl':
            dist.all_gather_into_tensor(out, self.buf)
        else:
            parts = [torch.empty_like(self.buf) for _ in range(world)]
            dist.all_gather(parts, self.buf)
            out.copy_(torch.stack(parts, 0))
        return out


def gather_rle(counts, n_counts):
    """Instance masks across ranks (apis/test.py:117-147 gathers the complete result incl. segm RLEs): the fixed-capacity
    run-length tensors of ops.mask_rle_counts - counts [max,cap] int32, n_counts [max] int32 - all-gathered as they are
    (two collectives of static shape).  Returns ([world,max,cap], [world,max])."""
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return counts.unsqueeze(0), n_counts.unsqueeze(0)
    oc = counts.new_empty((world,) + tuple(counts.shape))
    on = n_counts.new_empty((world,) + tuple(n_counts.shape))
    if dist.get_backend() == 'nccl':
        dist.all_gather_into_tensor(oc, counts.contiguous())
        dist.all_gather_into_tensor(on, n_counts.contiguous())
    else:
        pc = [torch.empty_like(counts) for _ in range(world)]
        pn = [torch.empty_like(n_counts) for _ in range(world)]
        dist.all_gather(pc, counts.contiguous())
        dist.all_gather(pn, n_counts.contiguous())
        oc.copy_(torch.stack(pc, 0))
        on.copy_(torch.stack(pn, 0))
    return oc, on


def track_gathered(gathered, n_frames, tracker, first_frames=(0,)):
    """SipMask-VIS association on the gathered records (SURVEY 8e/8f-2): frames were sharded round-robin over ranks (frame
    f = step * world + rank), `gathered` is RecordLog.gather() with feat_dim = 512, [world, cap, max, 519] (host or device).
    Runs `tracker` (sipmask_b200.tracker.Tracker) sequentially in frame order and returns the list of det_obj_ids."""
    g = gathered.cpu().numpy() if hasattr(gathered, 'cpu') else gathered
    world = g.shape[0]
    ids = []
    for f in range(n_frames):
        rec = g[f % world, f // world]
        k = int(rec[:, 6].sum())
        ids.append(tracker.step(rec[:k, :5], rec[:k, 5].astype('int64'), rec[:k, 7:], f in first_frames))
    return ids


def gather_parts(parts):
    """Variable-size byte buffers of every rank, in two collectives: an all-gather of the sizes (one int64 per part),
    then one of the parts concatenated and padded to the largest rank's total (apis/test.py's collect_results_gpu does
    the same with one pickled buffer).  parts: a list of 1-D uint8 tensors on this rank's device (the same number on
    every rank).  Returns, per rank in rank order, its list of parts (views of the gathered buffer)."""
    dev = parts[0].device if parts else torch.device('cpu')
    sizes = torch.tensor([p.numel() for p in parts], dtype=torch.int64, device=dev)
    world = dist.get_world_size() if dist.is_initialized() else 1
    if world == 1:
        return [list(parts)]
    all_sizes = [torch.empty_like(sizes) for _ in range(world)]
    dist.all_gather(all_sizes, sizes)
    totals = [int(s.sum()) for s in all_sizes]
    buf = torch.zeros(max(totals + [1]), dtype=torch.uint8, device=dev)
    if parts:
        flat = torch.cat(parts)
        buf[:flat.numel()].copy_(flat)
    bufs = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(bufs, buf)
    out = []
    for b, s in zip(bufs, all_sizes):
        offs = [0] + torch.cumsum(s, 0).tolist()
        out.append([b[offs[i]:offs[i + 1]] for i in range(len(parts))])
    return out


def gather_bytes(data, device):
    """Every rank's `data` (bytes) through gather_parts (staged on `device`: NCCL moves device memory).  Returns the list
    of bytes in rank order."""
    t = torch.frombuffer(bytearray(data), dtype=torch.uint8) if len(data) else torch.zeros(0, dtype=torch.uint8)
    return [p[0].cpu().numpy().tobytes() for p in gather_parts([t.to(device)])]


def gather_eval_state(evaluator):
    """Every rank's cocoeval.CocoEvaluator.state(), in rank order, on every rank: the state's tensors as bytes through
    gather_parts (one all-gather of the sizes, one of the padded bytes), read back with the local state's dtypes.  Call
    it once, after the last image; rank 0 then merges the others' states (CocoEvaluator.merge) and evaluates."""
    local = evaluator.state()
    keys = evaluator.state_keys()
    parts = [local[k].contiguous().view(-1).view(torch.uint8) for k in keys]
    return [{k: p.clone().view(local[k].dtype) for k, p in zip(keys, ps)} for ps in gather_parts(parts)]
