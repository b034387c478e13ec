"""Seeded inputs shared by tests/golden/gen_golden_ref_train_ops.py and the GPU tests of the training-side operators
(tests/test_gpu_deform_conv_grad.py, tests/test_gpu_sigmoid_focal_loss.py)."""
import numpy as np
import torch

# (B, C, H, W, dg): kernel-level DeformConv backward cases
COL2IM_CASES = [(2, 64, 9, 11, 1), (1, 256, 13, 21, 4),
                # four 8-channel vectors per lane; 120 vectors (lanes with 4 and with 3); one vector per group; more
                # groups than lanes; three images; maps where every sample lies near a border
                (1, 1024, 5, 6, 1), (1, 960, 6, 5, 4), (2, 64, 7, 9, 8), (1, 512, 5, 7, 64), (3, 128, 4, 5, 2),
                (2, 64, 1, 1, 1), (1, 128, 1, 4, 2), (1, 64, 4, 1, 1), (3, 256, 2, 2, 4)]
# (C, gamma, alpha): sigmoid focal loss cases
FOCAL_CASES = [(c, g, a) for c in (80, 40, 1) for g in (2.0, 1.5, 0.0) for a in (0.25, 0.5)]
SAMPLE = 4096                      # sampled elements per col2im output


def sample_index(n, seed):
    """the fixed sample of flat output indices whose reference values are stored"""
    return np.sort(np.random.RandomState(seed).choice(n, size=min(SAMPLE, n), replace=False)).astype(np.int64)


def col2im_inputs(B, C, H, W, dg):
    """x [B,C,H,W] fp16-representable, offset [B,dg*18,H,W], grad_col [C*9, B, H, W] (the reference's column layout).
    Sampling points: row r < 7 of the h components (every tap) lands exactly on -1, -0.5, 0, H-1, H-0.5, H, 2 (integer
    positions and the borders of (-1, H)); the same for the w components along columns; pixels at +-40 px; the last
    row rounded to integers.  Maps of fewer than 3 rows or columns sample near the borders instead (below)."""
    g = torch.Generator().manual_seed(B * 1000 + C + H)
    x = torch.randn(B, C, H, W, generator=g).half().float()
    off = torch.randn(B, dg * 18, H, W, generator=g) * 2.5
    hs = [-1.0, -0.5, 0.0, H - 1.0, H - 0.5, float(H), 2.0]
    ws = [-1.0, -0.5, 0.0, W - 1.0, W - 0.5, float(W), 2.0]
    for gi in range(dg):
        for tap in range(9):
            i, j = tap // 3, tap % 3
            ch, cw = gi * 18 + 2 * tap, gi * 18 + 2 * tap + 1
            for r, t in enumerate(hs[:H]):
                off[:, ch, r, :] = t - (r - 1 + i)
            for c, t in enumerate(ws[:W]):
                off[:, cw, :, c] = t - (c - 1 + j)
    off[:, :, -1, :] = torch.round(off[:, :, -1, :])
    off[:, 0::2, H // 2, W // 2] = 40.0
    off[:, 1::2, H // 2, W // 2 - 1] = -40.0
    gcol = torch.randn(C * 9, B, H, W, generator=g)
    if min(H, W) < 3:
        # one or two rows or columns: the pinned positions above would all fall outside.  Instead every sampling point
        # lies within 0.25 px of the map's extent (-1, H) x (-1, W), most of them inside, on a 2^-8 grid (exact in fp32,
        # and the borders and integer positions themselves occur)
        ch = torch.arange(dg * 18) % 18
        tap, d = ch // 2, ch % 2
        lim = torch.where(d == 0, float(H), float(W)).view(1, -1, 1, 1)
        base = torch.where((d == 0).view(-1, 1, 1), (tap // 3).view(-1, 1, 1) + torch.arange(H).view(1, H, 1),
                           (tap % 3).view(-1, 1, 1) + torch.arange(W).view(1, 1, W)).float() - 1.0
        pos = torch.round((torch.rand(B, dg * 18, H, W, generator=g) * (lim + 1.5) - 1.25) * 256) / 256
        off = pos - base
    return x, off, gcol


def focal_inputs(C):
    """logits [N, C] with 0, +-1e-3, +-15, +-88, +-100 in every row's first columns and N(0, 4^2) elsewhere; targets
    cover -1, 0 and every class, then random; d_loss random."""
    N = C + 42
    g = torch.Generator().manual_seed(C)
    logits = torch.randn(N, C, generator=g) * 4.0
    special = torch.tensor([0.0, 1e-3, -1e-3, 15.0, -15.0, 88.0, -88.0, 100.0, -100.0])
    for n in range(N):
        k = (n % special.numel())
        vals = torch.roll(special, k)[:C]
        logits[n, :vals.numel()] = vals
    targets = torch.cat([torch.tensor([-1, 0]), torch.arange(1, C + 1),
                         torch.randint(-1, C + 1, (N - C - 2,), generator=g)]).long()
    d_loss = torch.rand(N, C, generator=g) * 2.0 - 0.5
    return logits.contiguous(), targets, d_loss.contiguous()


def focal_key(C, gamma, alpha):
    return 'focal_%d_%g_%g' % (C, gamma, alpha)
