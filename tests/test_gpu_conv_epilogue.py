"""The convolution's two epilogues compute the same bits (run with -m gpu).

fp16-output plans with no residual or a same-shape one store through shared memory and TMA; fp32-output plans store
from registers.  Both apply acc + bias, x alpha, + residual, GroupNorm statistics, ReLU to the same fp32 values, so the
fp16 output must equal the fp32 output rounded with .half(), and the integer GroupNorm statistics must be equal."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _nhwc(x):
    return x.permute(0, 2, 3, 1).contiguous().to(torch.float16).cuda()


def _pair(x, wk, k, stride, Ho, Wo, cout, bias=None, residual=None, relu=False, alpha=1.0, gn=False, max_ctas=None):
    """Runs the same convolution into an fp16 and an fp32 output, twice each; returns (out16, out32, stats16, stats32)."""
    from sipmask_b200 import conv
    res = []
    for dt in (torch.float16, torch.float32):
        out = torch.full((x.shape[0], Ho, Wo, cout), float('nan'), dtype=dt, device='cuda')
        st = torch.zeros((x.shape[0], 32, 2), dtype=torch.int64, device='cuda') if gn else None
        plan = conv.ConvPlan(x, wk, out, k, stride, relu=relu, bias=bias, residual=residual, gn_stats=st, alpha=alpha)
        if max_ctas:
            plan.set_max_ctas(max_ctas)
        plan.run()
        torch.cuda.synchronize()
        first, st_first = out.clone(), st.clone() if gn else None
        if gn:
            st.zero_()
        plan.run()
        torch.cuda.synchronize()
        assert torch.equal(out, first), 'second run differs (%s)' % dt
        if gn:
            assert torch.equal(st, st_first), 'second run statistics differ (%s)' % dt
        res.append((out, st))
    return res[0][0], res[1][0], res[0][1], res[1][1]


# (N, H, W, cin, cout, k, stride): N tiles 64 / 128 / 256, Cout 2048 (8 N-tiles), Cout 48 (a half-clipped 32-channel
# chunk), patches 1x128 (3 x 128), 8x16 (20 x 13, ragged in x and y) and 16x8 (30 x 7), batch 2, stride 2
SHAPES = [
    (1, 25, 42, 64, 64, 1, 1),
    (2, 25, 42, 512, 128, 1, 1),
    (1, 200, 336, 64, 256, 1, 1),       # layer1 conv3: 525 M-tiles, one k-block
    (2, 13, 21, 256, 2048, 1, 1),
    (1, 13, 21, 256, 48, 3, 1),
    (1, 3, 128, 256, 256, 3, 1),
    (2, 20, 13, 256, 256, 3, 1),
    (1, 30, 7, 128, 256, 1, 1),
    (2, 25, 42, 256, 512, 1, 2),
]


@pytest.mark.parametrize('N,H,W,cin,cout,k,stride', SHAPES)
@pytest.mark.parametrize('res,relu,alpha', [(False, False, 1.0), (True, True, 1.0), (True, False, 0.75),
                                            (False, True, 1.25)])
def test_fp16_epilogue_equals_fp32_epilogue(N, H, W, cin, cout, k, stride, res, relu, alpha):
    g = torch.Generator().manual_seed(H * 131 + W * 7 + cin + cout + k + stride)
    from sipmask_b200 import conv
    x = _nhwc(torch.randn(N, cin, H, W, generator=g))
    w = torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5
    wk, _ = conv.pack_weight(w, device='cuda')
    bias = torch.randn(cout, generator=g).cuda()
    Ho, Wo = (H + 2 * (k // 2) - k) // stride + 1, (W + 2 * (k // 2) - k) // stride + 1
    r = _nhwc(torch.randn(N, cout, Ho, Wo, generator=g)) if res else None
    gn = cout in (256, 512)
    o16, o32, s16, s32 = _pair(x, wk, k, stride, Ho, Wo, cout, bias=bias, residual=r, relu=relu, alpha=alpha, gn=gn)
    assert torch.equal(o16, o32.half())
    if gn:
        assert torch.equal(s16, s32)


@pytest.mark.parametrize('res', [False, True])
def test_fp16_epilogue_slot_ring_wraps_across_tiles(res):
    """Seven CTAs over many tiles: every CTA's slot ring wraps many times within and across tiles."""
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(3)
    N, H, W, cin, cout = 1, 50, 84, 128, 256
    x = _nhwc(torch.randn(N, cin, H, W, generator=g))
    wk, _ = conv.pack_weight(torch.randn(cout, cin, 3, 3, generator=g) / 34.0, device='cuda')
    bias = torch.randn(cout, generator=g).cuda()
    r = _nhwc(torch.randn(N, cout, H, W, generator=g)) if res else None
    o16, o32, s16, s32 = _pair(x, wk, 3, 1, H, W, cout, bias=bias, residual=r, relu=True, gn=True, max_ctas=7)
    assert torch.equal(o16, o32.half()) and torch.equal(s16, s32)
    full16, _, fs16, _ = _pair(x, wk, 3, 1, H, W, cout, bias=bias, residual=r, relu=True, gn=True)
    assert torch.equal(o16, full16) and torch.equal(s16, fs16)


def test_fp16_epilogue_multi_level_with_gn_stats():
    """A 5-level launch: per-level output maps, GroupNorm statistics, fp16 == fp32 rounded."""
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(17)
    sizes = [(25, 42), (13, 21), (7, 11), (4, 6), (2, 3)]
    N = 2
    xs = [_nhwc(torch.randn(N, 256, h, w, generator=g)) for h, w in sizes]
    wk, _ = conv.pack_weight(torch.randn(256, 256, 3, 3, generator=g) / 48.0, device='cuda')
    bias = torch.randn(256, generator=g).cuda()
    got = []
    for dt in (torch.float16, torch.float32):
        outs = [torch.full((N, h, w, 256), float('nan'), dtype=dt, device='cuda') for h, w in sizes]
        st = [torch.zeros((N, 32, 2), dtype=torch.int64, device='cuda') for _ in sizes]
        conv.ConvPlanMulti(xs, wk, outs, 3, relu=True, bias=bias, gn_stats=st).run()
        torch.cuda.synchronize()
        got.append((outs, st))
    for l in range(len(sizes)):
        assert torch.equal(got[0][0][l], got[1][0][l].half()), l
        assert torch.equal(got[0][1][l], got[1][1][l]), l


def test_fp16_epilogue_into_channel_slice():
    """An fp16 output at a pitch wider than Cout (a channel slice of a wider buffer) leaves the other channels alone."""
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(23)
    x = _nhwc(torch.randn(1, 128, 20, 13, generator=g))
    wk, _ = conv.pack_weight(torch.randn(64, 128, 3, 3, generator=g) / 34.0, device='cuda')
    big = torch.full((1, 20, 13, 192), 7.0, dtype=torch.float16, device='cuda')
    view = big[..., 64:128]
    conv.ConvPlan(x, wk, view, 3, 1, relu=True).run()
    ref = torch.empty((1, 20, 13, 64), dtype=torch.float32, device='cuda')
    conv.ConvPlan(x, wk, ref, 3, 1, relu=True).run()
    torch.cuda.synchronize()
    assert torch.equal(view, ref.half())
    assert (big[..., :64] == 7).all() and (big[..., 128:] == 7).all()


@pytest.mark.parametrize('H,W', [(64, 96), (224, 352)])
def test_stem_fp16_epilogue_is_deterministic(H, W):
    """The stem (N = 64, K = 256, 2100 tiles at 800 x 1344) stores through shared memory: same bits on every run, and
    within the per-element convolution bound of the float64 value of its operands."""
    from sipmask_b200 import conv
    g = torch.Generator().manual_seed(H + W)
    img = torch.randn(2, 3, H, W, generator=g).cuda()
    w = torch.randn(64, 3, 7, 7, generator=g) * 0.1
    bn = (torch.rand(64, generator=g) + 0.5, torch.randn(64, generator=g) * 0.1, torch.randn(64, generator=g) * 0.1,
          torch.rand(64, generator=g) + 0.5)
    wk, bias = conv.pack_stem_weight_s2d(w, bn, device='cuda')
    q = conv.image_to_s2d16(img)
    out = torch.full((2, H // 2, W // 2, 64), float('nan'), dtype=torch.float16, device='cuda')
    plan = conv.StemPlan(q, wk, bias, out, 2, H, W)
    plan.run()
    torch.cuda.synchronize()
    first = out.clone()
    plan.run()
    torch.cuda.synchronize()
    assert torch.equal(out, first)
    # element by element: a 4x4 valid convolution over the space-to-depth input, weights viewed as [64, 4, 4, 16]
    from oracle import numerics as NU
    y, m = NU.conv_reference(q, wk, 4, 1, bias=bias, pad=0, out_hw=out.shape[1:3])
    NU.check_conv(out, y, m, 256, relu=True, what='stem %dx%d' % (H, W))
