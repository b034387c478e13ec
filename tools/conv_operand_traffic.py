"""Is a convolution bound by L2->SM operand traffic or by the SM?  Two measurements on the workload-A engine:

1. Per conv: the modelled L2->SM operand bytes per tile and per launch (one A box of the 128-pixel patch per tap and
   64-channel block, plus the weight box), the warm time (CUDA graph of 20 launches, as tools/time_convs.py) and the operand
   GB/s that time implies.  Beside it, for 3x3 stride-1 convs, the bytes a halo-staged A operand would move: one
   {64 ch, 16, 18} box of a 16 x 8 patch with its halo per 64-channel block, plus the nine weight boxes.
2. Contention sweep: the multi-level tower conv and fpn_convs.0 with the persistent grid capped at 16 / 33 / 66 / 132 CTAs.
   A CTA runs one tile per wave (waves = ceil(units / CTAs); all tiles of these convs have the same K), so time / waves is
   the time one tile takes while that many CTAs stream operands at once.  If operand traffic set the pace, it would grow
   with the number of CTAs while the operand GB/s flattens."""
import math
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sipmask_b200 import conv as C  # noqa: E402
from sipmask_b200 import synth  # noqa: E402
from sipmask_b200.engine import SipMaskEngine  # noqa: E402

REPS = 20
MIN_TILES = 48          # planner default (smb_conv_set_min_tiles)
A_BOX = 128 * 64 * 2    # A box: 128 pixels x 64 channels fp16
HALO_BOX = 18 * 16 * 64 * 2


def choose_patch(H, W):
    """conv_wgmma.cu choose_patch: the BH x BW = 128 patch with the fewest tiles."""
    best = None
    for bh, bw in ((1, 128), (2, 64), (4, 32), (8, 16), (16, 8)):
        t = math.ceil(H / bh) * math.ceil(W / bw)
        if best is None or t < best[0]:
            best = (t, bh, bw)
    return best[1], best[2]


def n_tile(tiles_m, cout):
    cmax = (cout + 63) // 64 * 64
    for c in (256, 128, 64):
        if c <= cmax and tiles_m * math.ceil(cout / c) >= MIN_TILES:
            return c
    return 64


def model(levels, nimg, cin, cout, k, halo=False):
    """levels: output (H, W) per level -> (work units, operand bytes per unit) of one launch."""
    if halo:
        tiles_m = nimg * sum(math.ceil(h / 16) * math.ceil(w / 8) for h, w in levels)
    else:
        tiles_m = nimg * sum(math.ceil(h / bh) * math.ceil(w / bw) for (h, w), (bh, bw) in
                             zip(levels, [choose_patch(h, w) for h, w in levels]))
    nt = n_tile(tiles_m, cout)
    cb = cin // 64
    per_unit = cb * HALO_BOX + 9 * cb * nt * 128 if halo else k * k * cb * (A_BOX + nt * 128)
    return tiles_m * math.ceil(cout / nt), per_unit


def warm_us(plan):
    for _ in range(3):
        plan.run()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(REPS):
            plan.run()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS * 1e3


def main():
    sd = synth.detector_state_dict(50, seed=1, cls_bias=bench.CLS_BIAS)
    eng = SipMaskEngine(sd, (bench.H, bench.W), test_cfg=bench.TEST_CFG, img_shape=(bench.H, bench.IMG_W, 3), use_graph=False)
    eng.forward(synth.synthetic_image(bench.H, bench.W, seed=0).cuda())
    torch.cuda.synchronize()

    print('== per conv (warm, CUDA graph of %d launches); operand KB per work unit and MB per launch, halo = 3x3/1 model' % REPS)
    print('%-36s %3s %5s %5s %6s %8s %9s %8s %8s %8s %7s' % ('conv', 'k', 'Cin', 'Cout', 'units', 'KB/unit', 'KB/u halo',
                                                             'MB', 'MB halo', 'warm_us', 'GB/s'))
    tot = {}
    for plan, m in zip(eng.conv_plans, eng.conv_meta):
        outs = plan.out if isinstance(plan.out, list) else [plan.out]
        levels = [(o.shape[1], o.shape[2]) for o in outs]
        nimg, cout = outs[0].shape[0], m['N']
        t = warm_us(plan)
        if m['name'] == 'stem':
            print('%-36s %3d %5s %5d %6s %8s %9s %8s %8s %8.1f' % (m['name'], m['k'], '-', cout, '-', '-', '-', '-', '-', t))
            continue
        k = m['k']
        cin = m['K'] // (k * k)
        units, per_unit = model(levels, nimg, cin, cout, k)
        is_3x3s1 = k == 3 and m['stride'] == 1
        hu, hpu = model(levels, nimg, cin, cout, k, halo=True) if is_3x3s1 else (units, per_unit)
        a = tot.setdefault('3x3 stride 1' if is_3x3s1 else 'other', [0.0, 0.0, 0.0])
        a[0] += t; a[1] += units * per_unit / 1e6; a[2] += hu * hpu / 1e6
        print('%-36s %3d %5d %5d %6d %8.0f %9.0f %8.1f %8.1f %8.1f %7.0f' % (
            m['name'][-36:], k, cin, cout, units, per_unit / 1024, hpu / 1024, units * per_unit / 1e6, hu * hpu / 1e6, t,
            units * per_unit / t / 1e3))
    for key, (t, a, b) in sorted(tot.items()):
        print('sum %-13s warm %7.1f us, operand MB per forward %7.1f (halo model %7.1f)' % (key, t, a, b))

    print('\n== contention sweep: grid capped by set_max_ctas; us/wave = time one tile takes with that many CTAs')
    g = torch.Generator().manual_seed(0)
    lv = [(o.shape[1], o.shape[2]) for o in eng.fpn_outs]
    w = torch.randn(256, 256, 3, 3, generator=g) / 48.0
    wk, _ = C.pack_weight(w, device='cuda')
    bias = torch.randn(256, generator=g).cuda()
    xs = [(torch.randn(1, h, w_, 256, generator=g) * 0.5).half().cuda() for h, w_ in lv]
    outs = [torch.empty(1, h, w_, 256, dtype=torch.float16, device='cuda') for h, w_ in lv]
    stats = [torch.zeros(1, 32, 2, dtype=torch.int64, device='cuda') for _ in lv]
    cases = [('tower (5 levels)', lv, lambda: C.ConvPlanMulti(xs, wk, outs, 3, gn_stats=stats)),
             ('fpn_convs.0', lv[:1], lambda: C.ConvPlan(xs[0], wk, outs[0], 3, 1, bias=bias))]
    print('%-18s %5s %6s %6s %9s %9s %8s' % ('conv', 'CTAs', 'units', 'waves', 'us', 'us/wave', 'GB/s'))
    for name, levels, mk in cases:
        units, per_unit = model(levels, 1, 256, 256, 3)
        for cap in (16, 33, 66, 132):
            t = warm_us(mk().set_max_ctas(cap))
            waves = math.ceil(units / min(cap, units))
            print('%-18s %5d %6d %6d %9.1f %9.2f %8.0f' % (name, min(cap, units), units, waves, t, t / waves,
                                                          units * per_unit / t / 1e3))

    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip()
    print('\ncard (name, power limit, SM clock now, max SM clock): %s' % q)


if __name__ == '__main__':
    main()
