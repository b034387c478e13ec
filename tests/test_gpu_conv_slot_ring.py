"""The shared-memory epilogue's slot ring at every N tile (run with -m gpu).

Each consumer warpgroup owns a ring of three slots, and warp 9 walks the same chunk sequence three chunks ahead, storing
each chunk and refilling its slot.  A warpgroup's half tile is 8 / 4 / 2 chunks at N = 256 / 128 / 64, so the ring wraps
within and across tiles at different points.  Whatever N, the number of CTAs (and so how many tiles one ring carries), a
residual prefetched into the slots or the clipping of the last chunk, the fp16 output must equal the fp32
(register-epilogue) output rounded, and the integer GroupNorm statistics must be equal."""
import pytest
import torch

from test_gpu_conv_epilogue import _nhwc, _pair

pytestmark = pytest.mark.gpu


def _operands(seed, N, H, W, cin, cout, k, res):
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(seed)
    x = _nhwc(torch.randn(N, cin, H, W, generator=g))
    wk, _ = conv.pack_weight(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5, device='cuda')
    bias = torch.randn(cout, generator=g).cuda()
    r = _nhwc(torch.randn(N, cout, H, W, generator=g)) if res else None
    return x, wk, bias, r


# Cout 256 / 128 / 64 -> N tile 256 / 128 / 64 (8 / 4 / 2 chunks per warpgroup); 70 x 100 gives 63 M-tiles of 8 x 16,
# ragged in x and y
@pytest.mark.parametrize('cout', [256, 128, 64])
@pytest.mark.parametrize('k,cin', [(1, 64), (3, 64)])
@pytest.mark.parametrize('res', [False, True])
@pytest.mark.parametrize('ctas', [1, 3, 7])
def test_slot_ring_wraps_across_tiles(cout, k, cin, res, ctas):
    """More tiles than CTAs, so every ring wraps across tiles; the same bits as the uncapped grid."""
    x, wk, bias, r = _operands(cout + 10 * k + ctas, 1, 70, 100, cin, cout, k, res)
    gn = cout == 256
    o16, o32, s16, s32 = _pair(x, wk, k, 1, 70, 100, cout, bias=bias, residual=r, relu=True, gn=gn, max_ctas=ctas)
    assert torch.equal(o16, o32.half())
    full16, _, fs16, _ = _pair(x, wk, k, 1, 70, 100, cout, bias=bias, residual=r, relu=True, gn=gn)
    assert torch.equal(o16, full16)
    if gn:
        assert torch.equal(s16, s32) and torch.equal(s16, fs16)


# Cout 208 (N = 256: 7 chunks, the last one half clipped), 80 (N = 128: 3 chunks), 48 (N = 64: 2 chunks); 78 M-tiles
@pytest.mark.parametrize('cout', [208, 80, 48])
@pytest.mark.parametrize('res', [False, True])
def test_slot_ring_clipped_chunks(cout, res):
    x, wk, bias, r = _operands(cout, 2, 50, 84, 128, cout, 3, res)
    for ctas in (3, None):
        o16, o32, _, _ = _pair(x, wk, 3, 1, 50, 84, cout, bias=bias, residual=r, relu=False, alpha=0.75, max_ctas=ctas)
        assert torch.equal(o16, o32.half()), ctas


@pytest.mark.parametrize('ctas', [3, None])
def test_slot_ring_multi_level_with_gn_stats(ctas):
    """A 5-level N = 256 launch with statistics, tiles of several levels in one CTA's ring."""
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(29)
    sizes = [(50, 84), (25, 42), (13, 21), (7, 11), (4, 6)]
    N = 2
    xs = [_nhwc(torch.randn(N, 256, h, w, generator=g)) for h, w in sizes]
    wk, _ = conv.pack_weight(torch.randn(256, 256, 3, 3, generator=g) / 48.0, device='cuda')
    bias = torch.randn(256, generator=g).cuda()
    got = []
    for dt in (torch.float16, torch.float32):
        outs = [torch.full((N, h, w, 256), float('nan'), dtype=dt, device='cuda') for h, w in sizes]
        st = [torch.zeros((N, 32, 2), dtype=torch.int64, device='cuda') for _ in sizes]
        plan = conv.ConvPlanMulti(xs, wk, outs, 3, relu=True, bias=bias, gn_stats=st)
        if ctas:
            plan.set_max_ctas(ctas)
        plan.run()
        torch.cuda.synchronize()
        got.append((outs, st))
    for l in range(len(sizes)):
        assert torch.equal(got[0][0][l], got[1][0][l].half()), l
        assert torch.equal(got[0][1][l], got[1][1][l]), l


@pytest.mark.parametrize('cout,res', [(256, False), (256, True), (128, True)])
def test_slot_ring_into_channel_slice(cout, res):
    """Output into a channel slice of a wider buffer at N = 256 / 128: the other channels stay as they were."""
    from sipmask_b200 import conv
    x, wk, bias, r = _operands(cout + res, 1, 70, 100, 128, cout, 3, res)
    big = torch.full((1, 70, 100, cout + 128), 7.0, dtype=torch.float16, device='cuda')
    view = big[..., 64:64 + cout]
    conv.ConvPlan(x, wk, view, 3, 1, relu=True, bias=bias, residual=r).set_max_ctas(3).run()
    ref = torch.empty((1, 70, 100, cout), dtype=torch.float32, device='cuda')
    conv.ConvPlan(x, wk, ref, 3, 1, relu=True, bias=bias, residual=r).run()
    torch.cuda.synchronize()
    assert torch.equal(view, ref.half())
    assert (big[..., :64] == 7).all() and (big[..., 64 + cout:] == 7).all()
