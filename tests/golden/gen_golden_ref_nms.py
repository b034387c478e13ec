"""Generate tests/golden/ref_nms_cpu.npz: the keep lists of the reference's own nms_cpu.cpp (compiled into oracle/_ref by
oracle/build.py::build_ref_nms) on the seeded inputs of tests/test_oracle_golden.py::test_nms_matches_reference_cpp.

    python tests/golden/gen_golden_ref_nms.py
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, 'oracle', '_ref'))
sys.path.insert(0, os.path.dirname(HERE))

import sipmask_ref_nms_cpu as ref  # noqa: E402
import test_oracle_golden as T  # noqa: E402


def main():
    g = {}
    for n, thr, dets in T.nms_reference_cases():
        g['keep_%d_%g' % (n, thr)] = ref.nms(torch.from_numpy(dets), thr).numpy().astype(np.int64)
    np.savez_compressed(os.path.join(HERE, 'ref_nms_cpu.npz'), **g)


if __name__ == '__main__':
    main()
