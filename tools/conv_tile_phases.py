"""Where a convolution tile's time goes, per plan of the bench workload: mainloop, epilogue, time blocked waiting for
epilogue slots, and the warp-9 copy engine's waits.

Compiles conv_wgmma.cu with -DSMB_CONV_PHASES (clock64 stamps, see the kernel) into a temporary library linked with the
other objects of the in-tree build, so run build() first; `--lib` takes such a library built beforehand instead, and
`--build-only` just builds one.  Each plan runs once warm, then once stamped at its own grid and once with the grid capped
at 16 CTAs (`--caps`).  Per plan and grid: mean µs per recorded tile of a consumer warpgroup from mainloop start to the last
`wgmma_wait<0>` (main), from there to the end of its epilogue (epi), the part of epi blocked in `epi_full` waits (blk), the
MMA-idle fraction epi / (main + epi), chunks per tile, and warp 9's µs per tile blocked in `wait_group.read` and on
`epi_ready`.  GroupNorm plans also report the part of epi spent in the statistics' shuffle reductions (gn_shfl) and in
handing the tile's statistics over (gn_hand: the statistics barriers, or the wait for the previous tile's flush).
Each link of the chunk chain is reported per tile, summed over its chunks: from the slot being ready to the results in
registers (cmp: ldmatrix, arithmetic and gn_shfl), stmatrix (stsm), the proxy fence (fence), the slot arrival (arr), and
the staging of the tile's bias before its first chunk (bias); and on warp 9's side per tile, the store steps' issue and
commit time outside the epi_ready waits (w9st) and the fills' issue time (w9fill).
`--src` times another version of conv_wgmma.cu (e.g. a parent commit's, with the same stamps).  Cycles are converted with the ratio of globaltimer to clock64 over all CTAs of the launch (sm_mhz)."""
import argparse
import ctypes
import glob
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PHASE_TILE = 11                                                # kPhaseTile of the kernel's timing build
sys.path.insert(0, ROOT)
from sipmask_b200 import build as B  # noqa: E402
from sipmask_b200 import _lib  # noqa: E402


def build_timing_lib(out, src=None):
    objdir = os.path.join(ROOT, 'sipmask_b200', 'lib', 'obj')
    objs = [o for o in sorted(glob.glob(os.path.join(objdir, '*.o'))) if os.path.basename(o) != 'conv_wgmma.o']
    if not objs:
        raise SystemExit('no objects under %s: run build() first' % objdir)
    tmp = tempfile.mkdtemp(prefix='conv_phases_')
    obj = os.path.join(tmp, 'conv_wgmma_phases.o')
    subprocess.check_call([B.NVCC] + [f for f in B.FLAGS if f not in ('-Xptxas', '-v')] +
                          ['-DSMB_CONV_PHASES', '-I', B.CSRC, '-c', src or os.path.join(B.CSRC, 'conv_wgmma.cu'), '-o', obj])
    subprocess.check_call([B.NVCC, '-shared', '-o', out, obj] + objs + ['-gencode', 'arch=compute_90a,code=sm_90a'])
    return out


def stamp(plan, buf, words, torch):
    buf.zero_()
    _lib.lib().smb_conv_phase_buffer(ctypes.c_void_p(buf.data_ptr()), 1)
    plan.run()
    torch.cuda.synchronize()
    _lib.lib().smb_conv_phase_buffer(None, 1)
    r = buf.view(-1, words).cpu().numpy().astype('int64')
    ctas = r[r[:, 1] != 0]
    ns_per_cyc = (ctas[:, 2] - ctas[:, 0]).sum() / (ctas[:, 3] - ctas[:, 1]).sum()
    tiles = ctas[:, 16:].reshape(len(ctas), -1, PHASE_TILE)    # [cta, sample * 2 + wg, PHASE_TILE]
    k = ns_per_cyc
    have = tiles[:, :, 0] != 0
    main = ((tiles[:, :, 1] - tiles[:, :, 0]) * k)[have] / 1e3
    epi = ((tiles[:, :, 2] - tiles[:, :, 1]) * k)[have] / 1e3
    blk = (tiles[:, :, 3] * k)[have] / 1e3
    shfl = (tiles[:, :, 4] * k)[have] / 1e3
    hand = (tiles[:, :, 5] * k)[have] / 1e3
    links = [float(((tiles[:, :, i] * k)[have] / 1e3).mean()) for i in (6, 7, 8, 9, 10)]
    ntiles = ctas[:, 8].sum()                                 # all tiles; the first kPhaseSamples per CTA are recorded
    stores = ctas[:, 6].sum()
    return dict(ctas=int(len(ctas)), tiles=int(ntiles), sm_mhz=float(1e3 / ns_per_cyc), main_us=float(main.mean()), epi_us=float(epi.mean()),
                blocked_us=float(blk.mean()), gn_shfl_us=float(shfl.mean()), gn_hand_us=float(hand.mean()), idle=float(epi.mean() / (main.mean() + epi.mean())),
                chunks=float(stores / ntiles) if stores else 0.0,
                w9_read_us=float((ctas[:, 4] * ns_per_cyc).sum() / 1e3 / ntiles),
                w9_ready_us=float((ctas[:, 5] * ns_per_cyc).sum() / 1e3 / ntiles),
                cmp_us=links[0], stsm_us=links[1], fence_us=links[2], arrive_us=links[3], bias_us=links[4],
                w9_store_us=float(((ctas[:, 9] - ctas[:, 5]) * ns_per_cyc).sum() / 1e3 / ntiles),
                w9_fill_us=float((ctas[:, 10] * ns_per_cyc).sum() / 1e3 / ntiles))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--lib', help='a timing library built beforehand (--build-only)')
    ap.add_argument('--build-only', metavar='OUT', help='build the timing library to OUT and exit')
    ap.add_argument('--caps', default='16', help='grid caps after the plan\'s own grid, comma-separated')
    ap.add_argument('--json', help='write the per-plan numbers to this file')
    ap.add_argument('--src', help='time this conv_wgmma.cu instead of the tree\'s')
    ap.add_argument('--only', help='time only the plans whose name contains one of these comma-separated strings '
                                   '(`gn`: the plans with GroupNorm statistics)')
    args = ap.parse_args()
    if args.build_only:
        print(build_timing_lib(args.build_only, args.src))
        return
    lib = args.lib or build_timing_lib(os.path.join(tempfile.mkdtemp(prefix='conv_phases_'), 'libsipmask_b200.so'),
                                       args.src)
    _lib.LIB_PATH = lib
    import torch
    import bench
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    words = _lib.lib().smb_conv_phase_buffer(None, 1)
    sd = synth.detector_state_dict(50, seed=1, cls_bias=bench.CLS_BIAS)
    eng = SipMaskEngine(sd, (bench.H, bench.W), test_cfg=bench.TEST_CFG, img_shape=(bench.H, bench.IMG_W, 3), use_graph=False)
    eng.forward(synth.synthetic_image(bench.H, bench.W, seed=0).cuda())
    torch.cuda.synchronize()
    buf = torch.zeros(1024 * words, dtype=torch.int64, device='cuda')
    caps = [int(c) for c in args.caps.split(',') if c]
    out = []
    only = [o for o in (args.only or '').split(',') if o]
    print('%-40s %5s %5s %5s | %4s %5s %8s %8s %8s %8s %8s %6s %8s %8s %6s | %7s %7s %7s %7s %7s %7s %7s' % (
        'conv', 'Cout', 'K', 'chunk', 'ctas', 'tiles', 'main_us', 'epi_us', 'blk_us', 'gnshf_us', 'gnhnd_us', 'idle',
        'w9rd_us', 'w9rdy_us', 'MHz', 'bias', 'cmp', 'stsm', 'fence', 'arr', 'w9st', 'w9fill'))
    for plan, m in zip(eng.conv_plans, eng.conv_meta):
        if only and not any(o in m['name'] or (o == 'gn' and m['gn']) for o in only):
            continue
        name = m['name'] + (' GN %dx%d' % (m['k'], m['k']) if m['gn'] else '')
        plan.run()
        torch.cuda.synchronize()
        rows = [stamp(plan, buf, words, torch)]
        for c in caps:
            plan.set_max_ctas(c)
            rows.append(stamp(plan, buf, words, torch))
        for r in rows:
            print('%-40s %5d %5d %5.1f | %4d %5d %8.2f %8.2f %8.2f %8.2f %8.2f %6.3f %8.2f %8.2f %6.0f | %7.2f %7.2f %7.2f %7.2f '
                  '%7.2f %7.2f %7.2f' % (
                      name[-40:], m['N'], m['K'], r['chunks'], r['ctas'], r['tiles'], r['main_us'], r['epi_us'],
                      r['blocked_us'], r['gn_shfl_us'], r['gn_hand_us'], r['idle'], r['w9_read_us'], r['w9_ready_us'],
                      r['sm_mhz'], r['bias_us'], r['cmp_us'], r['stsm_us'], r['fence_us'], r['arrive_us'], r['w9_store_us'],
                      r['w9_fill_us']))
        out.append(dict(name=name, Cout=m['N'], K=m['K'], flops=m['flops'], grids=rows))
    print('card: %s' % torch.cuda.get_device_name(0))
    if args.json:
        with open(args.json, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
