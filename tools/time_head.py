"""Graph-replay time of the head section (first fork .. last join) for several persistent-grid caps (head_max_ctas)."""
import os
import sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from sipmask_b200 import synth  # noqa: E402
from sipmask_b200.engine import SipMaskEngine  # noqa: E402

sd = synth.detector_state_dict(50, seed=1, cls_bias=bench.CLS_BIAS)
img = synth.synthetic_image(bench.H, bench.W, seed=0).cuda()
for cap in (74, 0, 100):
    eng = SipMaskEngine(sd, (bench.H, bench.W), test_cfg=bench.TEST_CFG, img_shape=(bench.H, bench.IMG_W, 3), use_graph=False,
                        head_max_ctas=cap)
    eng.forward(img)
    torch.cuda.synchronize()
    names = eng.op_names
    first = names.index('fork', names.index('memset'))
    last = len(names) - 1 - names[::-1].index('join')
    sub = list(range(first, last + 1))
    full_ops, full_tags, full_names = eng.ops, eng.op_tags, eng.op_names
    eng.ops = [full_ops[i] for i in sub]
    eng.op_tags = [full_tags[i] for i in sub]
    eng.op_names = [full_names[i] for i in sub]
    eng._run_ops()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(5):
            eng._run_ops()
    g.replay()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(4):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    print('head_max_ctas=%s: head section %.1f us (%d ops)' % (cap, e0.elapsed_time(e1) / 20 * 1e3, len(sub)))
    del eng, g
