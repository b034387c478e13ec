"""Times SipMask++ mask rescoring on the GPU and prints one JSON line.

1. Rescoring alone at config 4's shape: 32 images x 100 valid detections, 272 x 272 cropped masks.  Times `mask_dense`
   (smb_mask_assemble, fp16 HWC prototypes -> fp16 masks, once per image as the engine issues it), the tensor-core chain
   (ops.mask_rescore_f16) and the fp32 CUDA-core chain (ops.mask_rescore) on the same masks: CUDA events after warm-up,
   median of 20 launches.  GFLOP/s from the algorithmic FLOPs (ops.rescore_flops_per_row), bytes from the shapes.
2. The engine at config 4 (R50, 544 x 544, batch 32, stacked_convs=2, gn=False, ssd_flag=True, backbone_dcn=True) with
   rescoring_flag off and on, alternated 3 x each: images/s over timed graph replays.

usage: python tools/time_rescore.py [--steps 20]"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from sipmask_b200 import ops, synth  # noqa: E402
from sipmask_b200.engine import SipMaskEngine  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument('--steps', type=int, default=20)
args = ap.parse_args()
assert torch.cuda.is_available(), 'time_rescore.py measures on the GPU'
dev = 'cuda'
gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                     capture_output=True, text=True).stdout.strip()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)


def median_ms(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return statistics.median(ts)


# ---------------------------------------------------------------------------------------------- 1. rescoring alone
N_IMG, ROWS, HM, WM = 32, 100, 272, 272
R = N_IMG * ROWS
g = torch.Generator().manual_seed(0)
sd = synth.head_state_dict(3, stacked_convs=2, gn=False, rescoring_flag=True, prefix='')
cw = [sd['convs_scoring.%d.conv.weight' % i] for i in range(6)]
cb = [sd['convs_scoring.%d.conv.bias' % i] for i in range(6)]
w1, b1 = sd['mask_scoring.weight'], sd['mask_scoring.bias']
wt = ops.RescoreWeights(cw, cb, w1, b1, dev)
protos = torch.relu(torch.randn(N_IMG, HM, WM, 32, generator=g)).half().to(dev)
cofs = (torch.randn(N_IMG, ROWS, 128, generator=g) * 0.3).to(dev)
cx, cy = torch.rand(N_IMG, ROWS, generator=g) * 2 * WM, torch.rand(N_IMG, ROWS, generator=g) * 2 * HM
bw, bh = torch.rand(N_IMG, ROWS, generator=g) * 300 + 32, torch.rand(N_IMG, ROWS, generator=g) * 300 + 32
boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], -1).clamp(0, 2 * HM).to(dev)   # image space
pos16 = torch.empty((N_IMG, ROWS, HM, WM), dtype=torch.float16, device=dev)
labels = torch.randint(0, 80, (N_IMG, ROWS), generator=g).to(dev)
det = torch.rand(N_IMG, ROWS, 5, generator=g).to(dev)
count = torch.full((N_IMG,), ROWS, dtype=torch.int32, device=dev)
ws = torch.empty(ops.mask_rescore_f16_workspace_bytes(R, HM, WM), dtype=torch.uint8, device=dev)
scores = torch.empty((N_IMG, ROWS), dtype=torch.float32, device=dev)


def dense():
    for n in range(N_IMG):
        ops.mask_assemble(protos[n], cofs[n], boxes[n], 0.5, layout='hwc', out=pos16[n])


t_dense = median_ms(dense)
t_f16 = median_ms(lambda: ops.mask_rescore_f16(pos16, count, wt, labels, det, workspace=ws, out=scores))
pos32 = pos16.view(R, HM, WM).float()
cwd, cbd, w1d, b1d = [w.to(dev) for w in cw], [b.to(dev) for b in cb], w1.to(dev), b1.to(dev)
old = {}


def fp32_chain():
    old['s'] = ops.mask_rescore(pos32, cwd, cbd, w1d, b1d, labels.view(R), det.view(R, 5))


t_f32 = median_ms(fp32_chain)
want, got = old['s'].double().cpu(), scores.view(R).double().cpu()
err = (got - want).abs()
bound = 1e-2 * want.abs() + 2e-3 * want.abs().max()

flops = R * ops.rescore_flops_per_row(HM, WM)
hs = [HM]
for _ in range(6):
    hs.append((hs[-1] - 3) // 2 + 1)
ch = ops.RESCORE_CHANNELS
act = [R * hs[l] * hs[l] * ch[l] for l in range(7)]           # elements of each layer's output (layer 0 = the masks)
# tensor-core chain: masks read once, layers 2-5 written and read back in fp16 (layer 1 and 6 stay on chip)
f16_bytes = 2 * act[0] + sum(2 * 2 * act[l] for l in range(2, 6)) + R * (5 * 4 + 8 + 4)
# fp32 chain: masks read in fp32, every layer written and read back in fp32
f32_bytes = 4 * act[0] + sum(2 * 4 * act[l] for l in range(1, 7)) + R * (5 * 4 + 8 + 4)
dense_bytes = N_IMG * HM * WM * 32 * 2 + R * (128 + 4) * 4 + 2 * act[0]
alone = dict(shape=[N_IMG, ROWS, HM, WM], mflop_per_row=ops.rescore_flops_per_row(HM, WM) / 1e6,
             mask_dense_ms=t_dense, mask_dense_gbs=dense_bytes / t_dense / 1e6,
             f16_chain_ms=t_f16, f16_chain_tflops=flops / t_f16 / 1e9, f16_chain_gb=f16_bytes / 1e9,
             f16_chain_gbs=f16_bytes / t_f16 / 1e6,
             fp32_chain_ms=t_f32, fp32_chain_tflops=flops / t_f32 / 1e9, fp32_chain_gb=f32_bytes / 1e9,
             speedup=t_f32 / t_f16, max_err_over_max=float(err.max() / want.abs().max()),
             within_bound=bool((err <= bound).all()), nonzero_scores=int((want != 0).sum()))
# per-kernel split of the tensor-core chain, in a profiled run of its own (not part of the timings above)
from torch.profiler import ProfilerActivity, profile  # noqa: E402
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for _ in range(5):
        ops.mask_rescore_f16(pos16, count, wt, labels, det, workspace=ws, out=scores)
    torch.cuda.synchronize()
alone['f16_kernels_ms'] = {e.key.replace('void smb::', '').split('(')[0]: e.device_time_total / 5 / 1e3
                           for e in prof.key_averages() if 'rescore_' in e.key}
del pos32, old, ws, pos16
torch.cuda.empty_cache()

# ------------------------------------------------------------------------------------------ 2. the engine, config 4
EH = EW = 544
BATCH = 32
cfg = dict(nms_pre=1000, score_thr=0.1, nms=dict(type='nms', iou_thr=0.5), max_per_img=100)
sd = synth.detector_state_dict(50, stacked_convs=2, gn=False, rescoring_flag=True, backbone_dcn=True, seed=1, cls_bias=-2.5)
kw = dict(batch=BATCH, depth=50, stacked_convs=2, gn=False, ssd_flag=True, backbone_dcn=True, test_cfg=cfg, use_graph=True)
img = synth.synthetic_image(EH, EW, batch=BATCH, seed=0).to(dev)
off = SipMaskEngine(sd, (EH, EW), **kw)
on = SipMaskEngine(sd, (EH, EW), rescoring_flag=True, share_weights=off, **kw)
for e in (off, on):
    e.forward(img)
    e.forward(None)
torch.cuda.synchronize()


def ips(e):
    for _ in range(3):
        e.forward(None)
    e0.record()
    for _ in range(args.steps):
        e.forward(None)
    e1.record()
    torch.cuda.synchronize()
    return BATCH * args.steps / (e0.elapsed_time(e1) / 1e3)


runs = dict(off=[], on=[])
for _ in range(3):
    runs['off'].append(ips(off))
    runs['on'].append(ips(on))
same = all(torch.equal(off._result()[k], on._result()[k]) for k in ('det_bboxes', 'det_labels', 'count', 'idxs_keep', 'mask_bits'))
engine = dict(workload='R50 544x544 bs32 stacked_convs=2 gn=False ssd_flag backbone_dcn', steps=args.steps,
              images_per_s_off=runs['off'], images_per_s_on=runs['on'],
              median_off=statistics.median(runs['off']), median_on=statistics.median(runs['on']),
              mean_count=float(on.count.float().mean()), record_bit_identical=same,
              rescore_gflop_per_forward_full=on.rescore_flops / 1e9, conv_gflop_per_forward=on.conv_flops / 1e9)
print(json.dumps(dict(gpu=gpu, rescore_alone=alone, engine=engine)))
