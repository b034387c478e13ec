"""YouTube-VIS mask AP on the device: YTVOSeval (the youtubevos pycocotools fork, iouType 'segm', default Params) as
SipMask-VIS's ytvos_eval runs it (SipMask-VIS/mmdet/core/evaluation/coco_utils.py:11-33) after tools/test_video.py.

The evaluation unit is a video.  The sequence IoU of a result entry d and a ground-truth object g (ytvoseval's iou_seq)
sums, over the frames, |d & g| where both are present and |d| or |g| where one is ("present" = not None; an empty mask
is present with area 0), and divides once.  Every term is an integer pixel count, so with
    U = sum |d| (frames d is present) + sum |g| (frames g is present) - sum |d & g| (frames both are)
the IoU needs three int64 sums per (entry, ground truth), accumulated frame by frame as batches finish:
  a. smb_ytvis_overlap_dev : per frame, each detection's pixel count and its intersection with every ground truth present
  b. smb_ytvis_scatter_dev : the last detection of each object id added into its video's accumulators (a pool of slots,
                             one per video being evaluated)
  c. smb_ytvis_match_dev   : once the video's result entries are final (score = mean of the frame scores, category =
                             majority vote), the IoU, the ranks and evaluateVid's greedy matching
then COCOeval's accumulate (cocoeval.accumulate, the same kernel) and summarize with YTVIS's area ranges
(0-128^2-256^2-1e5^2, still labelled small / medium / large).  avg_area, the area the ranges test, is the mean of the
non-zero frame areas: maskUtils.area of each frame's RLE for a result, the annotation's own `areas` for a ground truth.

Restated only: the youtubevos pycocotools is neither vendored in the reference (an empty submodule) nor installed where
this was written, so the semantics are those of its published ytvoseval.py / ytvos.py as read, not pinned by running it.
"""
import ctypes

import numpy as np
import torch

from . import _lib as L
from .cocoeval import (AREA_RNG_LBL, IOU_THRS, MAX_DETS, OUT_DTYPE, DET_CAP, MAX_CATS, accumulate, mm_results,
                       plane_stats, segm_plane, summarize)

FRAME_DTYPE = np.dtype([('det', '<u8'), ('det_stride', '<i8'), ('det_pitch', '<i4'), ('n_det', '<i4'), ('h', '<i4'),
                        ('w', '<i4'), ('gt_pitch', '<i4'), ('n_gt', '<i4'), ('g0', '<i4'), ('slot', '<i4')])
GTF_DTYPE = np.dtype([('plane', '<u8'), ('g', '<i4'), ('ext', '<i4', (4,)), ('pad', '<i4')])
VGT_DTYPE = np.dtype([('avg_area', '<f8'), ('sum_area', '<i8'), ('id', '<i8'), ('crowd', '<i4'), ('g', '<i4')])
ENT_DTYPE = np.dtype([('score', '<f8'), ('obj', '<i4'), ('cat', '<i4')])
assert (FRAME_DTYPE.itemsize, GTF_DTYPE.itemsize, VGT_DTYPE.itemsize, ENT_DTYPE.itemsize) == (48, 32, 32, 16)

# YTVOSeval Params (iouType 'segm'): COCO's thresholds and maxDets, its own area ranges
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 128 ** 2], [128 ** 2, 256 ** 2], [256 ** 2, 1e5 ** 2]]
OBJECTS, GTS, RANGE = 1, 2, 4        # status bits (SMB_YTVIS_*)


def _ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _pinned_to(arr, dev):
    """Upload a numpy array's bytes from pinned memory on the current stream (no host wait)."""
    b = np.ascontiguousarray(arr).view(np.uint8).reshape(-1)
    if b.size == 0:
        b = np.zeros(16, np.uint8)
    return torch.from_numpy(b).pin_memory().to(dev, non_blocking=True)


def avg_area(areas):
    """ytvoseval _toMask: the mean of the areas that are neither None nor 0, or 0 when none is."""
    vals = [a for a in areas if a]
    return 0 if len(vals) == 0 else np.array(vals).mean()


# ---------------------------------------------------------------------------------------------------- ground truth
class YtvisGroundTruth:
    """A loaded YouTube-VIS annotation json, indexed as ytvos.YTVOS and YTVOSeval._prepare see it.
      videos  : video id -> dict(h, w, length)
      cat_ids : sorted category ids; vid_ids: sorted video ids
    Per video, its annotations of those categories in annotation-file order: id, cat, iscrowd, segmentations (one per
    frame, None where absent: polygons, uncompressed or compressed RLE) and avg_area of its `areas`."""

    def __init__(self, ann_dict):
        try:
            self.videos = {int(v['id']): dict(h=int(v['height']), w=int(v['width']), length=int(v['length']))
                           for v in ann_dict['videos']}
            self.cat_ids = sorted(int(c['id']) for c in ann_dict['categories'])
            anns = ann_dict['annotations']
        except (KeyError, TypeError, ValueError) as e:
            raise ValueError('YtvisGroundTruth: malformed videos / categories: %r' % (e,))
        if len(set(self.cat_ids)) != len(self.cat_ids) or not 0 < len(self.cat_ids) <= MAX_CATS:
            raise ValueError('YtvisGroundTruth: need 1..%d distinct category ids' % MAX_CATS)
        self.vid_ids = sorted(self.videos)
        self.cat_index = {c: i for i, c in enumerate(self.cat_ids)}
        self.anns = {v: [] for v in self.vid_ids}
        for a in anns:
            try:
                vid, cat = int(a['video_id']), int(a['category_id'])
                segs, areas = list(a['segmentations']), list(a['areas'])
                row = dict(id=int(a['id']), cat=cat, iscrowd=int(bool(a.get('iscrowd', 0))), segmentations=segs,
                           areas=areas)
            except (KeyError, TypeError, ValueError) as e:
                raise ValueError('YtvisGroundTruth: malformed annotation %r: %r' % (a.get('id') if isinstance(a, dict) else a, e))
            if vid not in self.videos or cat not in self.cat_index:
                continue                                       # getAnnIds(vidIds=p.vidIds, catIds=p.catIds)
            n = self.videos[vid]['length']
            if len(segs) != n or len(areas) != n:
                raise ValueError('YtvisGroundTruth: annotation %d has %d segmentations and %d areas for a video of %d '
                                 'frames' % (row['id'], len(segs), len(areas), n))
            row['avg_area'] = avg_area(areas)
            self.anns[vid].append(row)

    def check_frame(self, video_id, frame_id, hw, max_gts=None):
        """Raises ValueError unless video_id is a ground-truth video with an h x w canvas and frame_id one of its frames
        (and, with max_gts, it has at most max_gts objects)."""
        v = self.videos.get(video_id) if isinstance(video_id, (int, np.integer)) else None
        if v is None:
            raise ValueError('video id %r is not in the ground truth' % (video_id,))
        if tuple(int(s) for s in hw[:2]) != (v['h'], v['w']):
            raise ValueError('video %d: frame of %dx%d, the annotation has %dx%d' % (video_id, hw[0], hw[1], v['h'], v['w']))
        if not 0 <= int(frame_id) < v['length']:
            raise ValueError('video %d has %d frames, got frame %d' % (video_id, v['length'], int(frame_id)))
        if max_gts is not None and len(self.anns[video_id]) > max_gts:
            raise ValueError('video %d has %d ground-truth objects, max_gts is %d' % (video_id, len(self.anns[video_id]),
                                                                                       max_gts))

    def frame(self, video_id, frame_id):
        """The ground-truth objects present in one frame: (rows GTF_DTYPE without plane pointers, planes [n, h, pitch]
        uint32, pixel counts [n] int64)."""
        v = self.videos[video_id]
        h, w = v['h'], v['w']
        pitch = (w + 31) // 32
        present = [(g, a) for g, a in enumerate(self.anns[video_id]) if a['segmentations'][frame_id] is not None]
        rows = np.zeros(len(present), GTF_DTYPE)
        planes = np.zeros((len(present), h, pitch), np.uint32)
        areas = np.zeros(len(present), np.int64)
        for r, (g, a) in enumerate(present):
            planes[r] = segm_plane(a['segmentations'][frame_id], h, w, 'annotation %d frame %d' % (a['id'], frame_id))
            areas[r], rows[r]['ext'] = plane_stats(planes[r], w)
            rows[r]['g'] = g
        return rows, planes, areas

    def packed_frame(self, video_id, frame_id):
        """frame()'s rows with the segmentations packed for the device rasterizer instead of rasterized: (rows GTF_DTYPE
        without plane pointers and extents, segm_raster.SegmPack with row r's segmentation in plane r).  Raises what
        frame() raises, from the numbers alone."""
        from .segm_raster import SegmPack
        v = self.videos[video_id]
        present = [(g, a) for g, a in enumerate(self.anns[video_id]) if a['segmentations'][frame_id] is not None]
        rows = np.zeros(len(present), GTF_DTYPE)
        pack = SegmPack()
        for r, (g, a) in enumerate(present):
            pack.add(a['segmentations'][frame_id], v['h'], v['w'], r, 'annotation %d frame %d' % (a['id'], frame_id))
            rows[r]['g'] = g
        return rows, pack

    def video(self, video_id):
        """The video's ground truth for its sequence match: (rows VGT_DTYPE without sum_area, grouped by category
        index with annotation order inside, per-category offsets [K+1])."""
        anns = self.anns[video_id]
        order = sorted(range(len(anns)), key=lambda g: self.cat_index[anns[g]['cat']])      # stable
        rows = np.zeros(len(anns), VGT_DTYPE)
        cnt = np.zeros(len(self.cat_ids) + 1, np.int32)
        for r, g in enumerate(order):
            a = anns[g]
            rows[r]['avg_area'] = a['avg_area']
            rows[r]['id'] = a['id']
            rows[r]['crowd'] = a['iscrowd']
            rows[r]['g'] = g
            cnt[self.cat_index[a['cat']] + 1] += 1
        return rows, np.cumsum(cnt).astype(np.int32)


# ---------------------------------------------------------------------------------------------------- evaluator
class YtvisEvaluator:
    """Device state of one YouTube-VIS evaluation: a pool of `slots` accumulator slots (one per video being evaluated;
    objects x max_gts int64 intersections, objects int64 areas and int32 non-zero frame counts, max_gts int64 ground-truth
    pixel sums each), the evaluated
    entries' matched / ignored rows and npig per (category, area range).
      gt       : YtvisGroundTruth
      cat_ids  : the category ids result entries may carry (default the ground truth's); any other raises ValueError.
                 Entries of a category in cat_ids without ground-truth category are not evaluated, as in _prepare.
    A video is evaluated by begin_video (its slot, zeroed on the current stream), stage_frame / overlap / scatter per
    frame batch, and end_video with its result entries; evaluate() accumulates every ended video."""

    def __init__(self, gt, cat_ids=None, slots=8, objects=1024, max_gts=64, device=None):
        self.gt = gt
        self.dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
        self.cat_ids = set(int(c) for c in (gt.cat_ids if cat_ids is None else cat_ids))
        self.K = len(gt.cat_ids)
        self.slots, self.objects, self.max_gts = int(slots), int(objects), int(max_gts)
        if self.slots < 1 or self.objects < 1 or self.max_gts < 1:
            raise ValueError('YtvisEvaluator: slots, objects and max_gts must be positive')
        S, O, G = self.slots, self.objects, self.max_gts
        with torch.cuda.device(self.dev):
            self.acc_inter = torch.zeros((S, O, G), dtype=torch.int64, device=self.dev)
            self.acc_area = torch.zeros((S, O), dtype=torch.int64, device=self.dev)
            self.acc_nz = torch.zeros((S, O), dtype=torch.int32, device=self.dev)
            self.gt_area = torch.zeros((S, G), dtype=torch.int64, device=self.dev)     # per ground truth: sum of its frames' pixels
            self.raster_status = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self.status = torch.zeros(1, dtype=torch.int32, device=self.dev)
            self.npig = torch.zeros(self.K * 4, dtype=torch.int32, device=self.dev)
        self.rows = []
        self.n_results = 0
        self.video_ids = []                  # ended videos, in end order
        self._vids = {}                      # video id -> dict(slot, frames) while being evaluated
        self._iou_thr = np.ascontiguousarray(IOU_THRS, dtype=np.float64)
        self._area_rng = np.ascontiguousarray(np.array(AREA_RNG, dtype=np.float64).reshape(-1))

    # ---- checks
    def check_frame(self, video_id, frame_id, hw):
        """Raises ValueError unless frame frame_id of an h x w image can be evaluated next for video_id."""
        self.gt.check_frame(video_id, frame_id, hw, self.max_gts)
        if int(frame_id) == 0 and (video_id in self._vids or video_id in self.video_ids):
            raise ValueError('video %d is evaluated twice' % video_id)

    # ---- per video / frame
    def begin_video(self, video_id, slot):
        """Video video_id accumulates into `slot` (zeroed on the current stream)."""
        if not 0 <= slot < self.slots:
            raise ValueError('accumulator slot %d of %d' % (slot, self.slots))
        self.acc_inter[slot].zero_()
        self.acc_area[slot].zero_()
        self.acc_nz[slot].zero_()
        self.gt_area[slot].zero_()
        self._vids[video_id] = dict(slot=int(slot), frames=0)

    def abort_video(self, video_id):
        self._vids.pop(video_id, None)

    def stage_frame(self, video_id, frame_id, stream=None):
        """Pack what describes one frame's ground-truth masks (polygon vertices, run lengths) and upload it from pinned
        memory on `stream` (default: the current stream); its planes are reserved on the device and rasterized there by
        overlap().  commit_frame() then counts the frame."""
        from . import segm_raster as SR
        rows, pack = self.gt.packed_frame(video_id, int(frame_id))
        v = self.gt.videos[video_id]
        pitch = (v['w'] + 31) // 32
        words = v['h'] * pitch
        stream = stream or torch.cuda.current_stream(self.dev)
        with torch.cuda.device(self.dev), torch.cuda.stream(stream):
            st, _ = SR.staged(pack, self.dev)
            planes = torch.empty(max(len(rows) * words, 1), dtype=torch.int32, device=self.dev)
        if len(rows):
            rows['plane'] = np.uint64(planes.data_ptr()) + np.arange(len(rows), dtype=np.uint64) * np.uint64(words * 4)
        return dict(video_id=video_id, rows=rows, planes=planes, raster=st, stream=stream, h=v['h'], w=v['w'], pitch=pitch)

    def commit_frame(self, staged):
        self._vids[staged['video_id']]['frames'] += 1

    def overlap(self, staged, dets, det_stride, det_pitch, max_num, count=None, n_det=None):
        """Kernel a on the current stream for a batch of frames: staged[n] = frame n's stage_frame, dets[n] = the
        device address of its first detection plane (det_stride / det_pitch words); count: int32 device tensor [N], or
        n_det: host numbers.  The frames' ground truth is rasterized first, on the same stream.  Returns dict(frames, inter,
        area, max_num, ...) of device tensors for scatter()."""
        from . import segm_raster as SR
        N = len(staged)
        cur = torch.cuda.current_stream(self.dev)
        fr = np.zeros(N, FRAME_DTYPE)
        g0 = 0
        for n, s in enumerate(staged):
            fr[n]['det'] = int(dets[n])
            fr[n]['det_stride'] = det_stride
            fr[n]['det_pitch'] = det_pitch
            fr[n]['n_det'] = 0 if n_det is None else n_det[n]
            fr[n]['h'], fr[n]['w'], fr[n]['gt_pitch'] = s['h'], s['w'], s['pitch']
            fr[n]['n_gt'], fr[n]['g0'] = len(s['rows']), g0
            fr[n]['slot'] = self._vids[s['video_id']]['slot']
            g0 += len(s['rows'])
            if s['stream'] != cur:                   # uploaded on another stream: keep it until this stream is done
                s['planes'].record_stream(cur)
                s['raster']['items'].record_stream(cur)
        gts = np.concatenate([s['rows'] for s in staged]) if N else np.zeros(0, GTF_DTYPE)
        # where scatter() adds each ground truth's pixel count: its slot's row of gt_area (columns the overlap kernel
        # reports as out of range are left out)
        slots = np.repeat([self._vids[s['video_id']]['slot'] for s in staged], [len(s['rows']) for s in staged])
        ok = (gts['g'] >= 0) & (gts['g'] < self.max_gts)
        cells = (slots.astype(np.int64) * self.max_gts + gts['g'])[ok]
        with torch.cuda.device(self.dev):
            frames = _pinned_to(fr, self.dev)
            gts_dev = _pinned_to(gts, self.dev)
            gt_area = torch.zeros(max(len(gts), 1), dtype=torch.int32, device=self.dev)
            gt_sel = _pinned_to(np.concatenate([cells, np.nonzero(ok)[0].astype(np.int64)]), self.dev)
            g0, rows32 = 0, gts_dev.view(torch.int32)    # smb_ytvis_gt_frame_t: ext is int32 3..6 of 8
            for s in staged:
                n = len(s['rows'])
                if n:
                    SR.raster(s['raster'], s['planes'], n, s['h'] * s['pitch'], s['pitch'], self.raster_status,
                              area=gt_area[g0:], area_stride=1, ext=rows32[g0 * 8 + 3:], ext_stride=8)
                g0 += n
            inter = torch.empty(max(N, 1) * max_num * self.max_gts, dtype=torch.int32, device=self.dev)
            area = torch.empty(max(N, 1) * max_num, dtype=torch.int32, device=self.dev)
            L.check(L.lib().smb_ytvis_overlap_dev(L.ptr(frames), N, L.ptr(count), max_num, L.ptr(gts_dev), len(gts),
                                                  self.max_gts, L.ptr(inter), L.ptr(area), L.ptr(self.status),
                                                  L.stream_ptr()), 'smb_ytvis_overlap_dev')
        return dict(frames=frames, inter=inter, area=area, max_num=max_num, n=N, gts=gts_dev, gt_area=gt_area, gt_sel=gt_sel,
                    n_sel=len(cells))

    def scatter(self, ovl, ids, count=None):
        """Kernel b on the current stream: ovl from overlap(), ids int32 device tensor [N, max_num] of object ids, count
        as for overlap().  The frames' ground-truth pixel counts are added into their videos' sums as well."""
        cur = torch.cuda.current_stream(self.dev)
        for key in ('frames', 'inter', 'area', 'gt_area', 'gt_sel'):
            ovl[key].record_stream(cur)
        with torch.cuda.device(self.dev):
            if ovl['n_sel']:
                sel = ovl['gt_sel'].view(torch.int64)
                k = ovl['n_sel']
                self.gt_area.view(-1).index_add_(0, sel[:k], ovl['gt_area'][sel[k:2 * k]].to(torch.int64))
            L.check(L.lib().smb_ytvis_scatter_dev(L.ptr(ovl['frames']), ovl['n'], L.ptr(count), L.ptr(ids), ovl['max_num'],
                                                  L.ptr(ovl['inter']), L.ptr(ovl['area']), self.max_gts,
                                                  L.ptr(self.acc_inter), L.ptr(self.acc_area), L.ptr(self.acc_nz),
                                                  self.slots, self.objects, L.ptr(self.status), L.stream_ptr()),
                    'smb_ytvis_scatter_dev')

    def end_video(self, video_id, entries, obj_ids):
        """Kernel c on the current stream, once every frame of the video is scattered: entries = its result json
        entries (results2json_videoseg), obj_ids = each entry's object id (its accumulator row).  Validates before
        anything is enqueued; returns the video's slot, free for the next video once this stream has passed here."""
        st = self._vids.get(video_id)
        if st is None:
            raise ValueError('video %r is not being evaluated' % (video_id,))
        v = self.gt.videos[video_id]
        if st['frames'] != v['length']:
            raise ValueError('video %d ended after %d frames, the annotation has %d' % (video_id, st['frames'], v['length']))
        if len(obj_ids) != len(entries):
            raise ValueError('video %d: %d entries and %d object ids' % (video_id, len(entries), len(obj_ids)))
        if len(entries) > DET_CAP:
            raise ValueError('video %d: %d result entries (at most %d)' % (video_id, len(entries), DET_CAP))
        if len(self.gt.anns[video_id]) > self.max_gts:
            raise ValueError('video %d has %d ground-truth objects, max_gts is %d' % (video_id, len(self.gt.anns[video_id]),
                                                                                       self.max_gts))
        ents = np.zeros(len(entries), ENT_DTYPE)
        for e, (r, o) in enumerate(zip(entries, obj_ids)):
            try:
                cat = int(r['category_id'])
                ents[e]['score'] = float(r['score'])
            except (KeyError, TypeError, ValueError) as err:
                raise ValueError('video %d: malformed result entry %r: %r' % (video_id, r, err))
            if cat not in self.cat_ids:
                raise ValueError('video %d: category %d is not among the evaluated categories' % (video_id, cat))
            ents[e]['cat'] = self.gt.cat_index.get(cat, -1)
            ents[e]['obj'] = int(o)
        gts, off = self.gt.video(video_id)
        lib = L.lib()
        with torch.cuda.device(self.dev):
            ents_dev, gts_dev, off_dev = _pinned_to(ents, self.dev), _pinned_to(gts, self.dev), _pinned_to(off, self.dev)
            if len(gts):                             # smb_ytvis_gt_t: sum_area is int64 1 of 4, from the slot's sums
                rows64 = gts_dev.view(torch.int64)[:len(gts) * 4].view(len(gts), 4)
                g = _pinned_to(gts['g'].astype(np.int64), self.dev).view(torch.int64)[:len(gts)]
                rows64[:, 1] = self.gt_area[st['slot']][g]
            ws_bytes = lib.smb_ytvis_match_workspace_bytes(len(gts))
            ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
            out = torch.empty(max(len(ents), 1) * OUT_DTYPE.itemsize, dtype=torch.uint8, device=self.dev)
            L.check(lib.smb_ytvis_match_dev(L.ptr(ents_dev), len(ents), L.ptr(gts_dev), len(gts), L.ptr(off_dev), self.K,
                                            st['slot'], L.ptr(self.acc_inter), L.ptr(self.acc_area), L.ptr(self.acc_nz),
                                            self.slots, self.objects, self.max_gts, ctypes.c_int64(video_id),
                                            _ptr(self._iou_thr), _ptr(self._area_rng), L.ptr(out),
                                            ctypes.c_int64(len(ents)), L.ptr(self.npig), L.ptr(self.status), L.ptr(ws),
                                            ctypes.c_size_t(ws_bytes), L.stream_ptr()), 'smb_ytvis_match_dev')
        if len(ents):
            self.rows.append(out)
        self.n_results += len(ents)
        del self._vids[video_id]
        self.video_ids.append(video_id)
        return st['slot']

    # ---- accumulate + summarize
    def evaluate(self):
        """Accumulate and summarize every ended video.  Returns {'segm_mAP', 'segm_mAP_50', 'segm_mAP_75', 'segm_mAP_s',
        'segm_mAP_m', 'segm_mAP_l', 'segm_mAP_copypaste'} plus 'stats' and 'arrays' ({'segm': {'precision', 'recall',
        'scores'}}) with YTVOSeval's eval arrays."""
        with torch.cuda.device(self.dev):
            status = int(self.status.item())
            if status & OBJECTS:
                raise L.SmbError('YouTube-VIS evaluation: an object id reached the accumulators\' capacity of %d objects'
                                 % self.objects)
            if status & GTS:
                raise L.SmbError('YouTube-VIS evaluation: a ground-truth column reached max_gts=%d' % self.max_gts)
            if status:
                raise L.SmbError('YouTube-VIS evaluation status %d' % status)
            from .segm_raster import check_status
            check_status(self.raster_status)
            if self.n_results == 0:
                raise ValueError('segm: the results of the evaluated videos are empty')
            p, r, s = accumulate(self.rows, self.npig, self.K, self.dev)
        stats = summarize(p, r, AREA_RNG_LBL, MAX_DETS)
        out = mm_results('segm', stats)
        out['stats'] = {'segm': stats}
        out['arrays'] = {'segm': dict(precision=p, recall=r, scores=s)}
        return out


def evaluate_json(gt, results, cat_ids=None, vid_ids=None, chunk=16, device=None):
    """YTVOSeval of a result list in the results2json_videoseg format (the reference's output, or VideoRunner.video_json
    over all videos) against `gt` on the device: the same kernels, with each present frame's RLE string parsed to run
    lengths on the host and rasterized on the device, and each entry its own accumulator row.  vid_ids: the evaluated videos (p.vidIds; default every ground-truth video).  A
    result whose video is not in the ground truth, whose segmentations do not cover the video's frames or whose
    category is not in cat_ids raises ValueError; results of other ground-truth videos are not evaluated."""
    vids = gt.vid_ids if vid_ids is None else sorted(set(int(v) for v in vid_ids))
    for v in vids:
        if v not in gt.videos:
            raise ValueError('video id %r is not in the ground truth' % (v,))
    per = {v: [] for v in vids}
    cats = set(int(c) for c in (gt.cat_ids if cat_ids is None else cat_ids))
    for r in results:
        if not isinstance(r, dict) or 'video_id' not in r or not isinstance(r.get('segmentations'), list):
            raise ValueError('malformed result entry %r' % (r,))
        v = int(r['video_id'])
        if v not in gt.videos:                       # loadRes: 'Results do not correspond to current coco set'
            raise ValueError('results: video %r is not in the ground truth' % (r['video_id'],))
        if len(r['segmentations']) != gt.videos[v]['length']:
            raise ValueError('results: an entry of video %d has %d segmentations for %d frames'
                             % (v, len(r['segmentations']), gt.videos[v]['length']))
        if int(r.get('category_id', -1)) not in cats:
            raise ValueError('results: category %r of video %d is not among the evaluated categories'
                             % (r.get('category_id'), v))
        if v in per:
            per[v].append(r)
    if len(results) == 0:
        raise ValueError('segm: the results are empty')
    objects = max([1] + [len(e) for e in per.values()])
    max_gts = max([1] + [len(gt.anns[v]) for v in vids])
    from . import segm_raster as SR
    ev = YtvisEvaluator(gt, cat_ids, slots=1, objects=objects, max_gts=max_gts, device=device)
    dev = ev.dev
    with torch.cuda.device(dev):
        for v in vids:
            ents = per[v]
            info = gt.videos[v]
            h, w, n_f = info['h'], info['w'], info['length']
            pitch = (w + 31) // 32
            ev.check_frame(v, 0, (h, w))
            ev.begin_video(v, 0)
            max_num = max(1, len(ents))
            for f0 in range(0, n_f, chunk):
                fs = list(range(f0, min(f0 + chunk, n_f)))
                staged, pack, n_det = [], SR.SegmPack(), []
                ids = np.full((len(fs), max_num), -1, np.int32)
                for n, f in enumerate(fs):
                    s = ev.stage_frame(v, f)
                    staged.append(s)
                    present = [e for e, r in enumerate(ents) if r['segmentations'][f] is not None]
                    for j, e in enumerate(present):
                        seg = ents[e]['segmentations'][f]
                        if not isinstance(seg, dict):
                            raise ValueError('results: video %d frame %d: segmentation must be an RLE dict' % (v, f))
                        pack.add(seg, h, w, sum(n_det) + j, 'result of video %d frame %d' % (v, f))
                    ids[n, :len(present)] = present
                    n_det.append(len(present))
                stride = h * pitch
                P = sum(n_det)
                pl = torch.empty(max(P * stride, 1), dtype=torch.int32, device=dev)
                if P:
                    SR.raster(SR.staged(pack, dev)[0], pl, P, stride, pitch, ev.raster_status)
                base, offs = pl.data_ptr(), np.concatenate([[0], np.cumsum(n_det)[:-1]]).astype(np.int64)
                ovl = ev.overlap(staged, [base + 4 * stride * int(o) for o in offs], stride, pitch, max_num, n_det=n_det)
                ev.scatter(ovl, torch.from_numpy(ids).to(dev))
                for s in staged:
                    ev.commit_frame(s)
            ev.end_video(v, ents, list(range(len(ents))))
    return ev.evaluate()
