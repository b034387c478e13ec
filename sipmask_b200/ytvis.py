"""YouTube-VIS results of tracked video frames, exactly as SipMask-VIS writes them (host only), and the lane and
frame-order bookkeeping of serving.VideoRunner.

Per frame, the reference's test output is the pair (bbox2result_with_id, obj_segms) (SipMask-VIS/mmdet/core/bbox/
transforms.py:182-202, models/anchor_heads/sipmask_head.py:604-611,648-665): {obj_id: {'bbox': [5] float32, 'label'}} and
{obj_id: rle} over the detections with an id >= 0, the last detection winning for a duplicate id; a frame without
detections gives ({}, one empty list per class).  Per video, results2json_videoseg (core/evaluation/coco_utils.py:205-246)
writes one entry per object id, in order of first appearance: the mean of its float32 scores, the majority vote of its
labels (+1; a tie goes to the smaller label) and one RLE per frame, None where the object is absent.
"""
import numpy as np


def frame_result(det, labels, obj_ids, segms, num_classes=41):
    """One frame's (det, seg) pair.  det [k, 5] float32, labels [k], obj_ids [k], segms the k RLE dicts of the frame's
    detections in detection order; num_classes counts the background, as the head's does."""
    det = np.array(det, np.float32).reshape(-1, 5)             # copies: the record's buffers are reused
    labels = np.array(labels, np.int64).reshape(-1)
    obj_ids = np.asarray(obj_ids).reshape(-1)
    k = det.shape[0]
    if not (labels.shape[0] == obj_ids.shape[0] == len(segms) == k):
        raise ValueError('frame_result: %d boxes, %d labels, %d ids and %d segms' % (k, labels.shape[0], obj_ids.shape[0],
                                                                                    len(segms)))
    if k == 0:
        return {}, [[] for _ in range(num_classes - 1)]
    dets, segs = {}, {}
    for i in range(k):
        oid = int(obj_ids[i])
        if oid >= 0:
            dets[oid] = {'bbox': det[i], 'label': labels[i]}
            segs[oid] = segms[i]
    return dets, segs


def video_json(video_id, frames):
    """The results2json_videoseg entries of one video: frames = its (det, seg) pairs in frame order (frame id = index)."""
    objs = {}
    for frame_id, (det, seg) in enumerate(frames):
        for oid in det:
            o = objs.setdefault(oid, {'scores': [], 'cats': [], 'segms': {}})
            o['scores'].append(det[oid]['bbox'][4])
            o['cats'].append(det[oid]['label'])
            s = seg[oid]
            counts = s['counts']
            o['segms'][frame_id] = {'size': list(s['size']), 'counts': counts.decode() if isinstance(counts, bytes) else counts}
    out = []
    for o in objs.values():
        out.append({'video_id': video_id,
                    'score': np.array(o['scores']).mean().item(),
                    'category_id': np.bincount(np.array(o['cats'])).argmax().item() + 1,
                    'segmentations': [o['segms'].get(f) for f in range(len(frames))]})
    return out


class VideoBook(object):
    """Which video holds which lane, and the frame order of every video.  A new video starts at frame 0 and takes the
    lowest free lane; each later frame must follow the previous one; end_video frees the lane (its tracker state stays,
    as the reference's single tracker keeps it across videos).  check() validates without changing anything."""

    def __init__(self, lanes):
        self.lanes = [None] * int(lanes)              # lane -> the video holding it
        self.videos = {}                              # video_id -> dict(lane, frames: [ticket per frame], ended)

    def check(self, video_id, frame_id):
        """(lane, is_first) of the next frame, or ValueError."""
        frame_id = int(frame_id)
        v = self.videos.get(video_id)
        if v is None:
            if frame_id != 0:
                raise ValueError('video %r: a new video starts at frame 0, got frame %d' % (video_id, frame_id))
            free = [l for l, h in enumerate(self.lanes) if h is None]
            if not free:
                raise ValueError('video %r: all %d lanes hold videos; end_video() frees one' % (video_id, len(self.lanes)))
            return free[0], True
        if v['ended']:
            raise ValueError('video %r has ended' % (video_id,))
        if frame_id != len(v['frames']):
            raise ValueError('video %r: frame %d follows frame %d, got frame %d' % (video_id, len(v['frames']),
                                                                                    len(v['frames']) - 1, frame_id))
        return v['lane'], False

    def commit(self, video_id, frame_id, ticket):
        lane, first = self.check(video_id, frame_id)
        if first:
            self.videos[video_id] = dict(lane=lane, frames=[], ended=False)
            self.lanes[lane] = video_id
        self.videos[video_id]['frames'].append(ticket)
        return lane, first

    def end(self, video_id):
        v = self.videos.get(video_id)
        if v is None or v['ended']:
            raise ValueError('video %r is not being served' % (video_id,))
        v['ended'] = True
        self.lanes[v['lane']] = None
