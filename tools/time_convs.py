"""Warm, back-to-back timing (CUDA events) of every convolution plan of the bench workload: shape, us, TFLOP/s, and each
plan against its floor: HBM bytes (input, weights, output and residual once each) at 3.35 TB/s and its FLOPs at the
989 TFLOP/s dense fp16 tensor peak (H100 SXM data sheet), the larger of the two being the bound (B = HBM, T = tensor)."""
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sipmask_b200 import synth  # noqa: E402
from sipmask_b200 import conv  # noqa: E402
from sipmask_b200.engine import SipMaskEngine  # noqa: E402

HBM_BPS, TENSOR_FLOPS = 3.35e12, 989e12


def _nbytes(ts):
    return sum(t.numel() * t.element_size() for t in ts if isinstance(t, torch.Tensor))


def plan_bytes(plan):
    """Algorithmic HBM bytes of one launch: every operand tensor the plan was built on, read or written once."""
    k = plan._keep
    if isinstance(plan, conv.StemPlan):                  # (image, weight, bias, out)
        return _nbytes(k)
    if isinstance(plan, conv.ConvPlanMulti):             # (inputs, weight, outputs, bias, gn_stats, levels)
        return _nbytes(k[0]) + _nbytes(k[1:2]) + _nbytes(k[2]) + _nbytes(k[3:4])
    return _nbytes(k[:5])                                # (input, weight, output, bias, residual, gn_stats)


sd = synth.detector_state_dict(50, seed=1, cls_bias=bench.CLS_BIAS)
eng = SipMaskEngine(sd, (bench.H, bench.W), test_cfg=bench.TEST_CFG, img_shape=(bench.H, bench.IMG_W, 3), use_graph=False)
eng.forward(synth.synthetic_image(bench.H, bench.W, seed=0).cuda())
torch.cuda.synchronize()
print('pairs above score_thr: %d of %d candidates x %d classes' % (int((eng.cand_scores[0] > 0.05).sum()), eng.ncand, eng.ncls))
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device='cuda')
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
tot_w = tot_c = tot_floor = 0.0
print('%-44s %8s %5s %6s %3s %8s %8s %8s %7s %7s %7s %2s %6s' % ('conv', 'M', 'N', 'K', 'k', 'warm_us', 'cold_us', 'TF/s(w)',
                                                              'MB', 'hbm_us', 'mma_us', 'b', 'fl/w'))
REPS = 20
for plan, m in zip(eng.conv_plans, eng.conv_meta):
    for _ in range(3):
        plan.run()
    torch.cuda.synchronize()
    # warm: REPS back-to-back launches replayed from a CUDA graph (no Python / driver launch cost in the number)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            plan.run()
    g.replay()
    torch.cuda.synchronize()
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    warm = e0.elapsed_time(e1) / REPS * 1e3
    cold = []
    for i in range(3):
        flush.fill_(i)
        e0.record()
        plan.run()
        e1.record()
        torch.cuda.synchronize()
        cold.append(e0.elapsed_time(e1) * 1e3)
    cold = sorted(cold)[1]
    nb = plan_bytes(plan)
    hbm_us, mma_us = nb / HBM_BPS * 1e6, m['flops'] / TENSOR_FLOPS * 1e6
    floor = max(hbm_us, mma_us)
    tot_w += warm
    tot_c += cold
    tot_floor += floor
    print('%-44s %8d %5d %6d %3d %8.1f %8.1f %8.1f %7.1f %7.1f %7.1f %2s %6.2f %s%s' % (
        m['name'][-44:], m['M'], m['N'], m['K'], m['k'], warm, cold, m['flops'] / warm / 1e6, nb / 1e6, hbm_us, mma_us,
        'B' if hbm_us >= mma_us else 'T', floor / warm, 'R' if m['res'] else '', 'G' if m['gn'] else ''))
print('sum warm(graph) %.1f us, sum cold %.1f us, sum of floors %.1f us, %.1f GFLOP' % (tot_w, tot_c, tot_floor,
                                                                                   eng.conv_flops / 1e9))
