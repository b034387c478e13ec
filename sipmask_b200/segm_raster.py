"""Segmentations for the device rasterizer (csrc/segm_raster.cu): the host packs what describes the masks (polygon
vertices, run lengths) and validates it from those numbers alone; the device makes the bit planes.

SegmPack.add() accepts what cocoeval.segm_plane accepts and raises what it raises, with the same messages: polygons
(frPyObjects: a first element of exactly 4 numbers makes every element an frBbox box), an uncompressed RLE, or a
compressed one (its string parsed to counts by the library's rleFrString).  No pixel is touched here.
"""
import numpy as np
import torch

from . import _lib as L
from . import ops
from .cocoeval import _check_size, string_to_counts

ITEM_DTYPE = np.dtype([('kind', '<i4'), ('plane', '<i4'), ('off', '<i8'), ('n', '<i8'), ('h', '<i4'), ('w', '<i4')])
assert ITEM_DTYPE.itemsize == 32
POLYGON, RUNS = 0, 1
# rleFrPoly casts 5 * coordinate + .5 to int and subtracts two such values in int: the device does the same arithmetic, so
# the scaled coordinates stay well inside int32 (on the host the cast of anything larger is undefined anyway)
COORD_LIMIT = float(2 ** 29) / 5


class SegmPack:
    """Items, a float64 vertex pool and a uint32 count pool for one smb_segm_raster_dev launch."""

    def __init__(self):
        self.items, self.xy, self.counts = [], [], []
        self.n_xy = self.n_counts = 0
        self.max_hw = self.max_w = 0

    def _item(self, kind, plane, off, n, h, w):
        self.items.append((kind, plane, off, n, h, w))
        self.max_hw, self.max_w = max(self.max_hw, h * w), max(self.max_w, w)

    def _runs(self, cnts, plane, h, w, what):
        cnts = np.ascontiguousarray(np.asarray(cnts, dtype=np.int64))
        if cnts.ndim != 1 or (cnts.size and (cnts.min() < 0 or cnts.max() > 0xffffffff)):
            raise ValueError('%s: run lengths must be a list of non-negative integers' % what)
        if int(cnts.sum()) != h * w:
            raise ValueError('%s: smb_coco_rle_to_bits: the runs do not cover the %d x %d canvas' % (what, h, w))
        self._item(RUNS, plane, self.n_counts, cnts.size, h, w)
        self.counts.append(cnts.astype(np.uint32))
        self.n_counts += cnts.size

    def add(self, segm, h, w, plane, what='segmentation'):
        """One segmentation of an h x w canvas, OR-ed into plane `plane` of the launch."""
        h, w = int(h), int(w)
        if h < 0 or w < 0 or h * w >= 2 ** 31:
            raise ValueError('%s: a canvas of %d x %d pixels is not supported' % (what, h, w))
        if isinstance(segm, list):
            if len(segm) == 0 or not isinstance(segm[0], (list, tuple)):
                raise ValueError('%s: a polygon list needs lists of coordinates' % what)
            n0 = len(segm[0])
            if n0 == 4:                                           # frBbox: [x, y, x, y+h, x+w, y+h, x+w, y]
                polys = []
                for bb in segm:
                    if len(bb) != 4:
                        raise ValueError('%s: boxes must have 4 numbers' % what)
                    x, y, bw, bh = [float(v) for v in bb]
                    xe, ye = x + bw, y + bh
                    polys.append([x, y, x, ye, xe, ye, xe, y])
            elif n0 > 4:
                polys = [[float(v) for v in p] for p in segm]
            else:
                raise ValueError('%s: input type is not supported (a polygon of %d numbers)' % (what, n0))
            for p in polys:
                xy = np.asarray(p, dtype=np.float64)[:len(p) // 2 * 2]
                if not (np.abs(xy) < COORD_LIMIT).all():
                    raise ValueError('%s: polygon coordinates must be finite and below %g in magnitude' % (what, COORD_LIMIT))
                self._item(POLYGON, plane, self.n_xy, xy.size // 2, h, w)
                self.xy.append(xy)
                self.n_xy += xy.size // 2
            return
        if not isinstance(segm, dict) or 'counts' not in segm or 'size' not in segm:
            raise ValueError('%s: not a polygon list or an RLE dict' % what)
        _check_size(segm, h, w, what)
        counts = segm['counts']
        if isinstance(counts, list):
            self._runs(counts, plane, h, w, what)
        elif isinstance(counts, (str, bytes)):
            self._runs(string_to_counts(counts), plane, h, w, what)
        else:
            raise ValueError('%s: counts must be a list or a string' % what)

    def arrays(self):
        """(items ITEM_DTYPE [n], vertices float64 [2 * n_xy], counts uint32 [n_counts])."""
        items = np.array(self.items, dtype=ITEM_DTYPE) if self.items else np.zeros(0, ITEM_DTYPE)
        xy = np.concatenate(self.xy) if self.xy else np.zeros(0, np.float64)
        counts = np.concatenate(self.counts) if self.counts else np.zeros(0, np.uint32)
        return items, xy, counts


def upload(arrays, dev):
    """The arrays' bytes in one pinned buffer, copied to `dev` on the current stream without a host wait.  Returns one
    uint8 device view per array (16-byte aligned; an empty array gets a view of 16 bytes)."""
    parts = [np.ascontiguousarray(a).view(np.uint8).reshape(-1) for a in arrays]
    sizes = [max((p.size + 15) // 16 * 16, 16) for p in parts]
    host = torch.empty(sum(sizes), dtype=torch.uint8).pin_memory()
    view, offs, o = host.numpy(), [], 0
    for p, s in zip(parts, sizes):
        view[o:o + p.size] = p
        offs.append(o)
        o += s
    buf = host.to(dev, non_blocking=True)
    return [buf[o:o + s] for o, s in zip(offs, sizes)]


def staged(pack, dev, extra=()):
    """Upload a pack (and `extra` arrays with it) on the current stream: (dict for raster(), extra's device views)."""
    items, xy, counts = pack.arrays()
    views = upload([items, xy, counts] + list(extra), dev)
    st = dict(items=views[0], n_items=len(items), xy=views[1], n_xy=pack.n_xy, counts=views[2], n_counts=pack.n_counts,
              max_hw=pack.max_hw, max_w=pack.max_w)
    return st, views[3:]


def raster(st, planes, n_planes, plane_stride, pitch, status, area=None, area_stride=1, ext=None, ext_stride=4):
    """Rasterize a staged pack into `planes` on the current stream (ops.segm_raster with the pack's sizes)."""
    ops.segm_raster(st['items'], st['n_items'], st['xy'], st['n_xy'], st['counts'], st['n_counts'], st['max_hw'],
                    st['max_w'], planes, n_planes, plane_stride, pitch, status, area=area, area_stride=area_stride,
                    ext=ext, ext_stride=ext_stride)


def rasterize(segms, h, w, device=None):
    """Bit planes [len(segms), h, ceil(w / 32)] int32 and their stats [len(segms), 5] int32 ({pixel count, row0, row1,
    word0, word1}) on the device, one plane per segmentation (what segm_plane + plane_stats give on the host)."""
    dev = torch.device(device) if device is not None else torch.device('cuda', torch.cuda.current_device())
    pack = SegmPack()
    for p, s in enumerate(segms):
        pack.add(s, h, w, p)
    pitch = (int(w) + 31) // 32
    n = len(segms)
    with torch.cuda.device(dev):
        st, _ = staged(pack, dev)
        planes = torch.empty((n, int(h), pitch), dtype=torch.int32, device=dev)
        stats = torch.zeros((n, 5), dtype=torch.int32, device=dev)
        status = torch.zeros(1, dtype=torch.int32, device=dev)
        raster(st, planes, n, int(h) * pitch, pitch, status, area=stats, area_stride=5, ext=stats[:, 1:], ext_stride=5)
        check_status(status)
    return planes, stats


def check_status(status):
    s = int(status.item())
    if s:
        raise L.SmbError('segmentation rasterizer: an item\'s pool range, plane index or canvas is outside its launch '
                         '(status %d)' % s)
