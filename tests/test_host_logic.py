"""Host-side logic that needs no GPU: resize specification, mask resize factors, bench workloads and thread detection."""
import math
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def test_resize_spec_follows_torch_interpolate_sizes():
    import torch
    import torch.nn.functional as F
    from sipmask_b200 import ops
    for H, W, up in [(48, 62, 2.0), (48, 62, 2.0 / 1.6667), (50, 64, (2 / 1.3, 2 / 1.7)), (60, 41, 2.0 / 3.1), (400, 672, 2.0)]:
        x = torch.zeros(1, 1, H, W)
        sf = tuple(float(u) for u in up) if isinstance(up, tuple) else float(up)
        want = F.interpolate(x, scale_factor=sf, mode='bilinear', align_corners=False).shape[2:]
        fh, fw, ry, rx = ops.resize_spec(H, W, up)
        assert (fh, fw) == tuple(want)
        uh, uw = (up if isinstance(up, tuple) else (up, up))
        assert ry == float(np.float32(1.0 / uh)) and rx == float(np.float32(1.0 / uw))
        assert ops.resize_spec(H, W, up, legacy_interp=True) == (fh, fw, 0.0, 0.0)


def test_mask_up_factors_match_oracle():
    from oracle import postproc as P
    from sipmask_b200 import postproc as Q
    for sf, ssd in [(1.0, False), (1.6667, False), (np.float32(1.25), False), (np.array([1.7, 1.3, 1.7, 1.3], np.float32), True),
                    (np.ones(4, np.float32), True)]:
        assert P.mask_up_factors(sf, ssd) == Q.mask_up_factors(sf, ssd)
    assert Q.mask_up_factors(np.array([1.7, 1.3, 1.7, 1.3], np.float32), True) == (float(np.float32(2) / np.float32(1.3)),
                                                                                   float(np.float32(2) / np.float32(1.7)))


def test_bench_workloads_and_threads():
    import bench
    assert set(bench.WORKLOADS) == {'A', 'A101', 'B', 'C'}
    for k, wl in bench.WORKLOADS.items():
        assert wl['H'] % 32 == 0 and wl['W'] % 32 == 0 and wl['img_w'] <= wl['W']
        cfg = bench.test_cfg(wl)
        assert cfg['max_per_img'] in (10, 100) and cfg['nms']['iou_thr'] == 0.5
    n, info = bench.host_threads()
    assert 1 <= n <= info['affinity'] and (info['cgroup_quota'] is None or n <= math.floor(info['cgroup_quota'] + 1e-6) or n == 1)
    sd = bench.state_dict_for(bench.WORKLOADS['C'])
    assert 'bbox_head.sipmask_track.weight' in sd and sd['bbox_head.fcos_cls.weight'].shape[0] == 40


def test_record_log_single_process():
    import torch
    from sipmask_b200 import dist as D
    log = D.RecordLog(3, 5, 'cpu', feat_dim=4)
    for i in range(4):                                   # ring: the 4th append overwrites row 0
        log.append(torch.full((5, 5), float(i)), torch.arange(5), torch.tensor([2], dtype=torch.int32), torch.full((5, 4), float(i)))
    g = log.gather()
    assert g.shape == (1, 3, 5, 11)
    assert g[0, 0, 0, 0] == 3 and g[0, 1, 0, 0] == 1 and g[0, :, :, 6].sum() == 6 and g[0, 0, 0, 7] == 3


def test_crop_cell_index_needs_no_division():
    """The tensor-core mask kernels pick the CropSplit cell with `(w - x1) >= roi_w` instead of the reference's
    `(int)((w - x1) / roi_w)` (crop_split_cuda_kernel.cu:50-51).  The two agree for every float32 pair with a >= 0, b > 0:
    IEEE division rounds to nearest, so the truncated quotient is >= 1 exactly when a >= b and >= 2 exactly when a >= 2b
    (`crop_idx` in mask_assemble.cu).  Checked on random pairs and on the neighbours of b and 2b, where it could break."""
    rng = np.random.RandomState(0)
    b = np.concatenate([rng.uniform(0.05, 700.0, 200000), 2.0 ** rng.randint(-4, 10, 1000), rng.uniform(0.05, 1.0, 50000)]).astype(np.float32)
    cands = [rng.uniform(0.0, 3.0, b.size).astype(np.float32) * b]
    for k in (1.0, 2.0):
        t = (np.float32(k) * b).astype(np.float32)
        cands += [t, np.nextafter(t, np.float32(0)), np.nextafter(t, np.float32(1e9)),
                  np.nextafter(np.nextafter(t, np.float32(0)), np.float32(0))]
    for a in cands:
        a = a.astype(np.float32)
        q = (a / b).astype(np.float32)                       # IEEE float32 division, round to nearest even
        idx = q.astype(np.int32)                             # truncation, as the C cast
        fast = (a >= b).astype(np.int32) + (a >= (b + b)).astype(np.int32)
        low = idx <= 2
        assert (np.minimum(idx, 2)[low] == fast[low]).all()
        assert ((idx >= 1) == (a >= b)).all() and ((idx >= 2) == (a >= b + b)).all()


def test_fp16_hi_lo_coefficient_split_keeps_fp32_logits():
    """The tensor-core mask kernels feed the fp32 coefficients as fp16 hi + fp16 lo (load_b_frag in mask_assemble.cu):
    hi = fp16(c), lo = fp16(c - hi): 22 mantissa bits for |c| >= 0.125; below that lo is an fp16 subnormal and the error is
    absolute, <= 2^-25 per coefficient.  A numpy model of that split with fp32 accumulation stays within
    2^-21 * sum|p c| + 2^-24 * sum|p| of the float64 dot product - the same order as the sequential fp32 fmaf of the scalar
    kernels - including tiny coefficients and coefficients clamped at the fp16 range."""
    rng = np.random.RandomState(1)
    p = np.maximum(rng.randn(4096, 32), 0).astype(np.float16)                  # prototypes: fp16 storage
    for scale in (1.0, 1e-3, 40.0, 3e4):
        c = (rng.randn(4096, 32) * scale).astype(np.float32)
        cc = np.clip(c, -65000.0, 65000.0)
        hi = cc.astype(np.float16)
        lo = (cc - hi.astype(np.float32)).astype(np.float16)
        assert np.isfinite(hi.astype(np.float32)).all()
        exact = (p.astype(np.float64) * cc.astype(np.float64)).sum(1)
        acc = np.zeros(4096, np.float32)
        for k in range(32):                                                    # fp32 accumulation of exact fp16 x fp16 products
            acc = acc + p[:, k].astype(np.float32) * hi[:, k].astype(np.float32)
            acc = acc + p[:, k].astype(np.float32) * lo[:, k].astype(np.float32)
        bound = (np.abs(p.astype(np.float64) * cc.astype(np.float64))).sum(1) * 2.0 ** -21 + \
            np.abs(p.astype(np.float64)).sum(1) * 2.0 ** -24 + 1e-9
        assert (np.abs(acc.astype(np.float64) - exact) <= bound).all(), scale
        seq = np.zeros(4096, np.float32)
        for k in range(32):                                                    # the scalar kernels' arithmetic
            seq = seq + p[:, k].astype(np.float32) * cc[:, k]
        assert (np.abs(seq.astype(np.float64) - exact) <= bound).all(), scale



def test_groupnorm_apply_multi_rejects_unsupported_channels():
    """The multi-level GroupNorm apply covers C in {256, 512, 1024, 2048}; any other C is refused before a launch (the
    argument checks run first, so the placeholder pointers are never dereferenced)."""
    import ctypes
    from sipmask_b200 import _lib
    lib = _lib.lib()
    ptrs = (ctypes.c_void_p * 1)(16)
    hw = (ctypes.c_int * 1)(4)
    for C in (128, 768, 4096):
        rc = lib.smb_groupnorm_relu_apply_multi(1, ptrs, ptrs, hw, hw, 1, C, C, ctypes.c_void_p(16), ctypes.c_void_p(16),
                                                ctypes.c_float(1e-5), 1, None)
        assert rc == -1, C
        assert b'unsupported' in lib.smb_last_error()
