"""Times the two mask ABI calls (dense pos_masks, fused bit-packed) at the BASELINE config-A sizes for one kernel family:
N = 100 detections with 32-512 px boxes on a 400 x 672 x 32 fp16 prototype map, L2 flushed between launches, CUDA
events, median of 12.  Prints one JSON line.

usage: python tools/time_masks.py [tensor|scalar]      (default: tensor)"""
import json
import os
import statistics
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sipmask_b200 import ops  # noqa: E402

family = sys.argv[1] if len(sys.argv) > 1 else 'tensor'
assert family in ('tensor', 'scalar'), 'family must be tensor or scalar'
ops.set_mask_tensor_dot(family == 'tensor')
dev = 'cuda'
H, W, IMG_W, N = 800, 1344, 1333, 100
Hm, Wm = H // 2, W // 2
g = torch.Generator().manual_seed(0)
protos = torch.relu(torch.randn(Hm, Wm, 32, generator=g)).half().to(dev)
cofs = torch.randn(N, 128, generator=g).to(dev)
cx, cy = torch.rand(N, generator=g) * IMG_W, torch.rand(N, generator=g) * H
bw, bh = torch.rand(N, generator=g) * 480 + 32, torch.rand(N, generator=g) * 480 + 32
boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1).clamp(min=0).to(dev)
pos = torch.empty((N, Hm, Wm), dtype=torch.float32, device=dev)
bits = torch.empty((N, H, (IMG_W + 31) // 32), dtype=torch.int32, device=dev)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def time_kernel(fn, reps=14):
    ts = []
    for i in range(reps):
        flush.fill_(i)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts[2:])


dense = time_kernel(lambda: ops.mask_assemble(protos, cofs, boxes, 0.5, layout='hwc', out=pos))
fused = time_kernel(lambda: ops.mask_assemble_pack(protos, cofs, boxes, 0.5, (H, IMG_W), 0.4, layout='hwc', out=bits))
dense_bytes = Hm * Wm * 64 + N * 528 + N * Hm * Wm * 4
fused_bytes = Hm * Wm * 64 + N * 528 + bits.numel() * 4
print(json.dumps(dict(family=family,
                      dense_ms=dense, dense_gbs=dense_bytes / dense / 1e6, fused_ms=fused, fused_gbs=fused_bytes / fused / 1e6,
                      checksum=[int(bits.ne(0).sum()), float(pos.sum())])))
