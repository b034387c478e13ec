"""The convolution's GroupNorm statistics, recomputed on the host bit for bit (run with -m gpu).

A GroupNorm plan sums, per (image, group), the pre-activation values and their squares in 64-bit fixed point.  The
documented order: each consumer warp owns 16 rows of a 128-pixel tile; lane l holds rows l / 4 and l / 4 + 8 and
channels 2 (l % 4), + 1 of every 8-channel block, and sums them in fp32 (the square term as fma(f0, f0, f1 * f1)); per
group (one block, or two blocks added in order for 16-channel groups) the 32 lanes' values are summed over the pairing
tree with offsets 16, 8, 4, 2, 1; the warp's sum is rounded to an integer at 2^20 (sum) and 2^16 (sum of squares); the
integers are summed over warps and tiles.  Here the pre-activation values come from an fp32-output plan of the same
convolution without ReLU, and the statistics of both epilogues (fp16 through shared memory, fp32 from registers) must
equal the host's at any number of CTAs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.float16).cuda()


def _patch(H, W):
    """choose_patch: the BH x BW = 128 patch with the fewest tiles, the first (widest) on ties."""
    best = None
    for bh, bw in ((1, 128), (2, 64), (4, 32), (8, 16), (16, 8)):
        t = -(-H // bh) * -(-W // bw)
        if best is None or t < best[0]:
            best = (t, bh, bw)
    return best[1], best[2]


def _fma32(a, b, c):
    """fp32 fma(a, b, c), correctly rounded: the exact product in float64, TwoSum, then round-to-odd before float32."""
    p = a.astype(np.float64) * b.astype(np.float64)           # exact: 24 x 24 bits
    c = c.astype(np.float64)
    s = p + c
    bb = s - p
    e = (p - (s - bb)) + (c - bb)                              # s + e == p + c exactly
    bits = s.view(np.int64)
    fix = (e != 0) & ((bits & 1) == 0)                         # inexact and even: step to the odd neighbour toward e
    s = np.where(fix, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def host_gn_stats(y, gn_group):
    """Fixed-point {sum * 2^20, sum of squares * 2^16} per (image, group) of y [N, H, W, C] float32, in the kernel's order."""
    N, H, W, C = y.shape
    BH, BW = _patch(H, W)
    ty, tx = -(-H // BH), -(-W // BW)
    t = np.zeros((N, ty * BH, tx * BW, C), np.float32)
    t[:, :H, :W] = y
    v = np.zeros((N, ty * BH, tx * BW), bool)
    v[:, :H, :W] = True
    # [N, ty, BH, tx, BW, ...] -> tile rows r = by * BW + bx; r = 16 w + 8 i + rg (warp w, row half i, lane row rg)
    t = t.reshape(N, ty, BH, tx, BW, C).transpose(0, 1, 3, 2, 4, 5).reshape(N, ty, tx, 8, 2, 8, C // 8, 4, 2)
    v = v.reshape(N, ty, BH, tx, BW).transpose(0, 1, 3, 2, 4).reshape(N, ty, tx, 8, 2, 8, 1, 1)
    f0, f1 = t[..., 0], t[..., 1]                               # [N, ty, tx, w, i, rg, block, cq]
    zero = np.float32(0)
    a, q2 = f0 + f1, _fma32(f0, f0, f1 * f1)
    out = []
    for term, scale in ((a, 2.0 ** 20), (q2, 2.0 ** 16)):
        s = np.where(v[:, :, :, :, 0], zero + term[:, :, :, :, 0], zero)
        s = np.where(v[:, :, :, :, 1], s + term[:, :, :, :, 1], s)   # [N, ty, tx, w, rg, block, cq]
        if gn_group == 16:
            s = s[..., 0::2, :] + s[..., 1::2, :]
        x = s.transpose(0, 1, 2, 3, 5, 4, 6).reshape(N, ty, tx, 8, -1, 32)   # lanes: l = 4 rg + cq
        lanes = np.arange(32)
        for o in (16, 8, 4, 2, 1):
            x = x + x[..., lanes ^ o]
        fixed = np.rint(x[..., 0].astype(np.float64) * scale).astype(np.int64)   # exact: a power-of-two scale
        out.append(fixed.sum(axis=(1, 2, 3)))                  # [N, groups]
    return np.stack(out, axis=-1)


def _operands(seed, N, sizes, cin, cout):
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(seed)
    xs = [_nhwc(torch.randn(N, cin, h, w, generator=g)) for h, w in sizes]
    wk, _ = conv.pack_weight(torch.randn(cout, cin, 3, 3, generator=g) / (9 * cin) ** 0.5, device='cuda')
    bias = torch.randn(cout, generator=g).cuda()
    return xs, wk, bias


def _run(xs, wk, bias, cout, dtype, relu, ctas, multi):
    from sipmask_b200 import conv
    N = xs[0].shape[0]
    outs = [torch.full((N, x.shape[1], x.shape[2], cout), float('nan'), dtype=dtype, device='cuda') for x in xs]
    st = [torch.zeros((N, 32, 2), dtype=torch.int64, device='cuda') for _ in xs]   # Cout / 32 channels per group
    if multi:
        plan = conv.ConvPlanMulti(xs, wk, outs, 3, relu=relu, bias=bias, gn_stats=st)
    else:
        plan = conv.ConvPlan(xs[0], wk, outs[0], 3, 1, relu=relu, bias=bias, gn_stats=st[0])
    plan.set_max_ctas(ctas)
    plan.run()
    torch.cuda.synchronize()
    return outs, st


def _check(sizes, cout, ctas, multi, seed):
    xs, wk, bias = _operands(seed, 2, sizes, 64, cout)
    y32, st32 = _run(xs, wk, bias, cout, torch.float32, False, ctas, multi)    # register epilogue, pre-activation out
    _, st16 = _run(xs, wk, bias, cout, torch.float16, True, ctas, multi)       # shared-memory epilogue, ReLU
    for l in range(len(sizes)):
        want = host_gn_stats(y32[l].cpu().numpy(), cout // 32)
        assert np.array_equal(st32[l].cpu().numpy(), want), ('fp32 plan', l)
        assert np.array_equal(st16[l].cpu().numpy(), want), ('fp16 plan', l)


# 30 x 50: 16 x 8 patches, ragged in x and y (2 x 7 tiles per image, 28 M-tiles); Cout 256 = 8-channel groups over two
# N = 128 tiles, 512 = 16-channel groups over two N = 256 tiles; 1 and 7 CTAs run many tiles each, 132 one
@pytest.mark.parametrize('cout', [256, 512])
@pytest.mark.parametrize('ctas', [1, 7, 132])
def test_gn_stats_match_host(cout, ctas):
    _check([(30, 50)], cout, ctas, False, seed=cout + ctas)


@pytest.mark.parametrize('ctas', [1, 7, 132])
def test_gn_stats_multi_level_match_host(ctas):
    _check([(25, 42), (13, 21), (7, 11), (4, 6), (2, 3)], 256, ctas, True, seed=41 + ctas)
