"""The convolution at the edges of its planner (run with -m gpu).

Every case first asserts, through ConvPlan.info(), the planner path it was written for (output patch, N tile, epilogue)
and that oracle/numerics.py's conv_patch names the same patch as the plan, then checks the output element by element
against the float64 value of its own fp16 operands (NU.conv_reference + NU.check_conv) and the GroupNorm statistics
with NU.check_gn_stats where the plan produces them.  Epilogue paths that apply to the same convolution are compared
bit for bit with the shared-memory / TMA epilogue.

Inputs of the small stride-2 cases lie inside larger buffers whose other memory holds a large finite fp16 sentinel: a
tap that reads outside the image instead of taking the TMA zero fill picks up the sentinel (or the next image) and
breaks the bound, deterministically and inside memory the test owns.

Run with -s to print the (patch, N tile, epilogue) of every case."""
import pytest
import torch

from oracle import numerics as NU

pytestmark = pytest.mark.gpu

SENTINEL = 1024.0
PATCHES = [(1, 128), (2, 64), (4, 32), (8, 16), (16, 8)]
# per patch: an exact map (whole tiles) and a ragged one (partial tiles along x, and along y where BH > 1)
PATCH_MAPS = {(1, 128): [(2, 256), (3, 200)], (2, 64): [(4, 192), (5, 150)], (4, 32): [(8, 96), (10, 70)],
              (8, 16): [(16, 48), (19, 35)], (16, 8): [(32, 24), (45, 21)]}


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _randn(g, *shape, scale=1.0):
    return (torch.randn(*shape, generator=g) * scale).to(torch.float16).cuda()


def _weight(g, cout, cin, k):
    from sipmask_b200 import conv
    wk, _ = conv.pack_weight(torch.randn(cout, cin, k, k, generator=g) / (cin * k * k) ** 0.5, device='cuda')
    return wk


def _exact_operands(g, x_shape, cout, k):
    """Integer inputs in [-3, 3], weights and bias on a 1/64 grid (|w| <= 1/2, |b| <= 2): every partial sum is exact in
    fp32, so every fp16 output is the correctly rounded value.  The misrounded-fraction check is a statistic, meaningless
    on the few hundred outputs of a 1 x 1 map; here it is exactly 0, and the per-element bound decides.  A tap that
    reads the sentinel adds 1024 x w to an output."""
    from sipmask_b200 import conv
    x = torch.randint(-3, 4, x_shape, generator=g).to(torch.float16).cuda()
    w = torch.randint(-32, 33, (cout, x_shape[3], k, k), generator=g).float() / 64
    wk, _ = conv.pack_weight(w, device='cuda')
    bias = (torch.randint(-128, 129, (cout,), generator=g).float() / 64).cuda()
    return x, wk, bias


def _out_hw(H, W, k, stride):
    p = k // 2
    return (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1


def _path(info, out, residual_upsample=False):
    """The epilogue a launch of this plan takes, from what the plan reports."""
    if out.dtype == torch.float32:
        return 'register fp32'
    if residual_upsample:
        return 'register fp16 upsampled residual'
    return 'tma fp16' if info['epi_tma'] else 'register fp16'


def _plan(x, wk, out, k, stride=1, min_tiles=None, **kw):
    from sipmask_b200 import conv
    prev = conv.set_min_tiles(min_tiles) if min_tiles is not None else None
    try:
        return conv.ConvPlan(x, wk, out, k, stride, **kw)
    finally:
        if prev is not None:
            conv.set_min_tiles(prev)


def _assert_patches(info, outs, what):
    """Per level: the plan's output size, its patch == NU.conv_patch, and the tile counts of that patch."""
    assert info['num_levels'] == len(outs), what
    tiles = 0
    for l, (lv, o) in enumerate(zip(info['levels'], outs)):
        Ho, Wo = o.shape[1], o.shape[2]
        assert (lv['H_out'], lv['W_out']) == (Ho, Wo), (what, l, lv)
        assert (lv['BH'], lv['BW']) == NU.conv_patch(Ho, Wo), (what, l, lv)
        assert (lv['tiles_y'], lv['tiles_x']) == (-(-Ho // lv['BH']), -(-Wo // lv['BW'])), (what, l, lv)
        tiles += o.shape[0] * lv['tiles_x'] * lv['tiles_y']
    assert info['tiles_m'] == tiles, what


def _report(what, info, path):
    pats = ','.join('%dx%d' % (lv['BH'], lv['BW']) for lv in info['levels'])
    print('conv edge case %-48s patch %-14s n_tile %3d x%d  %s' % (what, pats, info['n_tile'], info['n_tiles_n'], path))


def _run(plan):
    plan.run()
    torch.cuda.synchronize()


def _check(out, x, wk, k, stride=1, bias=None, alpha=1.0, residual=None, residual_upsample=False, relu=False, stats=None,
           what='conv'):
    y, m = NU.conv_reference(x, wk, k, stride, bias=bias, alpha=alpha, residual=residual,
                             residual_upsample=residual_upsample)
    patch = NU.conv_patch(out.shape[1], out.shape[2])
    NU.check_conv(out, y, m, wk.shape[1], relu=relu, what=what, patch=patch)
    if stats is not None:
        NU.check_gn_stats(stats, y, m, wk.shape[1], what=what)


def _stats(N):
    return torch.zeros((N, 32, 2), dtype=torch.int64, device='cuda')


# --------------------------------------------------------------------------------------------- patches x kernel size
@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('k', [1, 3])
@pytest.mark.parametrize('exact', [True, False])
@pytest.mark.parametrize('patch', PATCHES)
def test_every_patch(patch, exact, k, N):
    """Each of the planner's five 128-pixel patches, on a map of whole tiles and on a ragged one, stride 1, with bias,
    ReLU and GroupNorm statistics (fp16 output: the shared-memory / TMA epilogue)."""
    H, W = PATCH_MAPS[patch][0 if exact else 1]
    g = _gen(H * 1000 + W * 10 + k + N)
    cin, cout = 64, 256
    x = _randn(g, N, H, W, cin)
    wk = _weight(g, cout, cin, k)
    bias = torch.randn(cout, generator=g).cuda()
    out = torch.full((N, H, W, cout), float('nan'), dtype=torch.float16, device='cuda')
    st = _stats(N)
    plan = _plan(x, wk, out, k, relu=True, bias=bias, gn_stats=st)
    info = plan.info()
    what = '%dx%d %s map %dx%d, %dx%d conv, N=%d' % (patch + ('exact' if exact else 'ragged', H, W, k, k, N))
    _assert_patches(info, [out], what)
    assert (info['levels'][0]['BH'], info['levels'][0]['BW']) == patch, what
    assert (H % patch[0] == 0 and W % patch[1] == 0) == exact and (exact or W % patch[1] != 0), what
    assert info['epi_tma'] == 1, what
    _report(what, info, _path(info, out))
    _run(plan)
    _check(out, x, wk, k, bias=bias, relu=True, stats=st, what=what)


# ------------------------------------------------------------------------------------------------------------ N tiles
def _expected_n_tile(cout, min_tiles, tiles_m):
    """The planner's rule: the largest of 256 / 128 / 64 not above Cout rounded up to 64 that still gives min_tiles
    tiles, else 64."""
    cmax = -(-cout // 64) * 64
    for c in (256, 128, 64):
        if c <= cmax and tiles_m * -(-cout // c) >= min_tiles:
            return c
    return 64


@pytest.mark.parametrize('dtype', [torch.float16, torch.float32])
@pytest.mark.parametrize('min_tiles', [1, 1 << 30])
@pytest.mark.parametrize('cout', [16, 48, 80, 128, 208, 256, 336, 512])
def test_every_n_tile(cout, min_tiles, dtype):
    """N tiles 256 / 128 / 64 (min_tiles 1 takes the widest tile Cout allows, 1 << 30 the narrowest), with Cout values
    that leave the last N tile partly or mostly empty; fp16 (shared-memory epilogue) and fp32 (register) outputs, bias,
    alpha != 1, GroupNorm statistics where Cout has 32 groups of 8 or 16 channels."""
    N, H, W, cin, k = 2, 13, 21, 128, 3
    g = _gen(cout * 7 + min_tiles % 1000)
    x = _randn(g, N, H, W, cin)
    wk = _weight(g, cout, cin, k)
    bias = torch.randn(cout, generator=g).cuda()
    gn = cout in (256, 512)
    st = _stats(N) if gn else None
    out = torch.full((N, H, W, cout), float('nan'), dtype=dtype, device='cuda')
    plan = _plan(x, wk, out, k, min_tiles=min_tiles, bias=bias, gn_stats=st, alpha=0.625)
    info = plan.info()
    what = 'Cout %d, min_tiles %d, %s' % (cout, min_tiles, str(dtype)[6:])
    _assert_patches(info, [out], what)
    want = _expected_n_tile(cout, min_tiles, info['tiles_m'])
    assert want == (min(256, -(-cout // 64) * 64) if min_tiles == 1 else 64)
    assert info['n_tile'] == want and info['n_tiles_n'] == -(-cout // want), (what, info)
    assert info['stages'] == {256: 4, 128: 6, 64: 8}[want], (what, info)
    assert info['epi_tma'] == int(dtype == torch.float16), (what, info)
    assert 1 <= info['grid'] <= info['tiles_m'] * info['n_tiles_n'] and info['smem_bytes'] <= 227 * 1024, (what, info)
    _report(what, info, _path(info, out))
    _run(plan)
    _check(out, x, wk, k, bias=bias, alpha=0.625, stats=st, what=what)


# ---------------------------------------------------------------------------------------------------------- epilogues
@pytest.mark.parametrize('min_tiles', [None, 1])
@pytest.mark.parametrize('N,H,W,k', [(2, 13, 21, 3), (3, 3, 200, 1)])
def test_epilogue_paths_same_bits(N, H, W, k, min_tiles):
    """One convolution with bias, a same-shape residual, ReLU, alpha != 1 and GroupNorm statistics through every epilogue
    that can run it: shared memory / TMA (fp16, 16-byte aligned operands); registers with fp16 output, reached through an
    output pitch of Cout + 4 and through a residual 8 bytes off 16-byte alignment; registers with fp32 output.  All
    within the bound, all the same bits (fp32 rounded to fp16), the same statistics.  min_tiles=1: N tile 256."""
    cin, cout, alpha = 128, 256, 0.75
    g = _gen(N * 100 + H + W + k)
    x = _randn(g, N, H, W, cin)
    wk = _weight(g, cout, cin, k)
    bias = torch.randn(cout, generator=g).cuda()
    res = _randn(g, N, H, W, cout)
    n = res.numel()
    res_off = torch.full((n + 16,), SENTINEL, dtype=torch.float16, device='cuda')
    res8 = res_off[4:4 + n].view(res.shape)              # 8 bytes past a 16-byte boundary
    res8.copy_(res)
    assert res8.data_ptr() % 16 == 8
    wide = torch.full((N, H, W, cout + 4), SENTINEL, dtype=torch.float16, device='cuda')
    cases = [('tma fp16', torch.full((N, H, W, cout), float('nan'), dtype=torch.float16, device='cuda'), res, 1),
             ('register fp16, out pitch Cout + 4', wide[..., :cout], res, 0),
             ('register fp16, residual 8 bytes off', torch.full((N, H, W, cout), float('nan'), dtype=torch.float16,
                                                                 device='cuda'), res8, 1),
             ('register fp32', torch.full((N, H, W, cout), float('nan'), dtype=torch.float32, device='cuda'), res, 0)]
    got = []
    for name, out, r, epi in cases:
        out.fill_(float('nan'))
        st = _stats(N)
        plan = _plan(x, wk, out, k, min_tiles=min_tiles, relu=True, bias=bias, residual=r, gn_stats=st, alpha=alpha)
        info = plan.info()
        what = '%s, %dx%d conv on %dx%dx%d, min_tiles %s' % (name, k, k, N, H, W, min_tiles)
        _assert_patches(info, [out], what)
        assert info['epi_tma'] == epi, (what, info)
        assert min_tiles != 1 or info['n_tile'] == 256, (what, info)
        _report(what, info, name)
        _run(plan)
        _check(out, x, wk, k, bias=bias, alpha=alpha, residual=r, relu=True, stats=st, what=what)
        got.append((name, out, st))
    assert (wide[..., cout:] == SENTINEL).all(), 'the pitch-(Cout + 4) output wrote past Cout'
    ref, ref_st = got[0][1], got[0][2]
    for name, out, st in got[1:]:
        o = out.half() if out.dtype == torch.float32 else out
        assert torch.equal(o, ref), '%s differs from the shared-memory epilogue' % name
        assert torch.equal(st, ref_st), '%s: GroupNorm statistics differ from the shared-memory epilogue' % name


@pytest.mark.parametrize('min_tiles', [None, 1])
@pytest.mark.parametrize('H,W,rh,rw', [(26, 42, 13, 21), (25, 41, 13, 21), (3, 200, 2, 100), (7, 5, 3, 3)])
def test_upsampled_residual_epilogue(H, W, rh, rw, min_tiles):
    """The nearest-upsampled residual (FPN lateral) always stores from registers: within the bound, and the same bits as
    the shared-memory epilogue given the upsampled residual as a same-shape tensor (the epilogue's own fp32 index rule),
    fp16 and fp32 outputs, with GroupNorm statistics.  min_tiles=1: N tile 256."""
    N, cin, cout, alpha = 2, 128, 256, 1.25
    g = _gen(H * W + rh + rw)
    x = _randn(g, N, H, W, cin)
    wk = _weight(g, cout, cin, 1)
    bias = torch.randn(cout, generator=g).cuda()
    coarse = _randn(g, N, rh, rw, cout)

    def src(n_out, n_in):
        f = torch.tensor(float(n_in), dtype=torch.float32) / torch.tensor(float(n_out), dtype=torch.float32)
        return torch.floor(torch.arange(n_out, dtype=torch.float32) * f).long().clamp(max=n_in - 1).cuda()
    full = coarse[:, src(H, rh)][:, :, src(W, rw)].contiguous()
    got = []
    for dt, r, up in ((torch.float16, coarse, True), (torch.float32, coarse, True), (torch.float16, full, False)):
        out = torch.full((N, H, W, cout), float('nan'), dtype=dt, device='cuda')
        st = _stats(N)
        plan = _plan(x, wk, out, 1, min_tiles=min_tiles, relu=True, bias=bias, residual=r, residual_upsample=up,
                     gn_stats=st, alpha=alpha)
        info = plan.info()
        what = '%s residual %dx%d -> %dx%d, %s, min_tiles %s' % ('upsampled' if up else 'same-shape', rh, rw, H, W,
                                                                 str(dt)[6:], min_tiles)
        _assert_patches(info, [out], what)
        assert min_tiles != 1 or info['n_tile'] == 256, (what, info)
        assert info['epi_tma'] == int(dt == torch.float16 and not up), (what, info)
        _report(what, info, _path(info, out, residual_upsample=up))
        _run(plan)
        _check(out, x, wk, 1, bias=bias, alpha=alpha, residual=r, residual_upsample=up, relu=True, stats=st, what=what)
        got.append((out, st))
    (u16, s16), (u32, s32), (t16, ts) = got
    assert torch.equal(u16, t16), 'upsampled residual (registers) differs from the same-shape residual (shared memory)'
    assert torch.equal(u32.half(), t16) and torch.equal(s16, ts) and torch.equal(s32, ts)


# ----------------------------------------------------------------------------------------------- input channel slices
@pytest.mark.parametrize('off', [0, 64])
@pytest.mark.parametrize('k,stride', [(1, 1), (3, 1), (1, 2), (3, 2)])
def test_input_channel_slice(k, stride, off):
    """x is the channel slice [..., off:off + Cin] of a wider buffer (in_pitch = Cin + 64) whose other channels hold the
    sentinel: within the bound, and the same bits as the same input made contiguous."""
    N, H, W, cin, cout = 2, 11, 19, 128, 64
    g = _gen(k * 10 + stride + off)
    wide = torch.full((N, H, W, cin + 64), SENTINEL, dtype=torch.float16, device='cuda')
    x = wide[..., off:off + cin]
    x.copy_(_randn(g, N, H, W, cin))
    assert x.stride(2) == cin + 64
    wk = _weight(g, cout, cin, k)
    bias = torch.randn(cout, generator=g).cuda()
    Ho, Wo = _out_hw(H, W, k, stride)
    outs = []
    for inp in (x, x.contiguous()):
        out = torch.full((N, Ho, Wo, cout), float('nan'), dtype=torch.float16, device='cuda')
        plan = _plan(inp, wk, out, k, stride, bias=bias, relu=True)
        info = plan.info()
        what = 'Cin %d at channel %d of %d, %dx%d/%d' % (cin, off, cin + 64, k, k, stride)
        _assert_patches(info, [out], what)
        if inp is x:
            _report(what, info, _path(info, out))
        _run(plan)
        outs.append(out)
    _check(outs[0], x, wk, k, stride, bias=bias, relu=True, what=what)
    assert torch.equal(outs[0], outs[1]), what


# ----------------------------------------------------------------------------------------------- stride 2, tiny maps
@pytest.mark.parametrize('N', [1, 3])
@pytest.mark.parametrize('W', [1, 2, 3])
@pytest.mark.parametrize('H', [1, 2, 3])
@pytest.mark.parametrize('k', [3, 1])
def test_stride2_tiny_map(k, H, W, N):
    """Stride-2 convolutions of 1..3-row and 1..3-column maps (FPN P6 / P7 on small canvases).  The input lies inside a
    sentinel-filled buffer, with more sentinel memory after it than any tap could reach: every tap outside the image must
    read the zero fill (padding), not the next image or the memory after the tensor."""
    cin, cout = 128, 64
    g = _gen(k * 100 + H * 10 + W + N)
    n = N * H * W * cin
    lead = 64                                            # 128 bytes of sentinel before the image
    buf = torch.full((lead + n + (2 * H + 4) * (2 * W + 4) * cin,), SENTINEL, dtype=torch.float16, device='cuda')
    x = buf[lead:lead + n].view(N, H, W, cin)
    x0, wk, bias = _exact_operands(g, (N, H, W, cin), cout, k)
    x.copy_(x0)
    Ho, Wo = _out_hw(H, W, k, 2)
    out = torch.full((N, Ho, Wo, cout), float('nan'), dtype=torch.float16, device='cuda')
    plan = _plan(x, wk, out, k, 2, bias=bias)
    info = plan.info()
    what = '%dx%d/2 on %dx%dx%d' % (k, k, N, H, W)
    _assert_patches(info, [out], what)
    _report(what, info, _path(info, out))
    _run(plan)
    assert (buf[:lead] == SENTINEL).all() and (buf[lead + n:] == SENTINEL).all()
    _check(out, x, wk, k, 2, bias=bias, what=what)


# -------------------------------------------------------------------------------------------------------- multi-level
@pytest.mark.parametrize('k,dtype', [(3, torch.float16), (1, torch.float16), (3, torch.float32)])
def test_multi_level_with_a_1x1_level(k, dtype):
    """One launch over four levels down to a 1 x 1 map, three images: per level within the bound (GroupNorm statistics
    for fp16 outputs) and the same bits as one single-level plan per level.  Exact operands (_exact_operands): the 1 x 1
    level has only N x Cout outputs."""
    from sipmask_b200 import conv
    N, cin, cout = 3, 128, 256
    sizes = [(7, 11), (4, 6), (2, 3), (1, 1)]
    xs, wk, bias = zip(*[_exact_operands(_gen(k * 7 + l), (N, h, w, cin), cout, k) for l, (h, w) in enumerate(sizes)])
    xs, wk, bias = list(xs), wk[0], bias[0]
    gn = dtype == torch.float16
    outs = [torch.full((N, h, w, cout), float('nan'), dtype=dtype, device='cuda') for h, w in sizes]
    sts = [_stats(N) for _ in sizes] if gn else None
    plan = conv.ConvPlanMulti(xs, wk, outs, k, relu=True, bias=bias, gn_stats=sts)
    info = plan.info()
    what = 'multi-level %dx%d, %s, levels %s' % (k, k, str(dtype)[6:], sizes)
    _assert_patches(info, outs, what)
    assert info['epi_tma'] == int(gn), (what, info)
    _report(what, info, _path(info, outs[0]))
    _run(plan)
    for l in range(len(sizes)):
        _check(outs[l], xs[l], wk, k, bias=bias, relu=True, stats=sts[l] if gn else None, what='%s level %d' % (what, l))
        o = torch.full_like(outs[l], float('nan'))
        st = _stats(N) if gn else None
        _run(conv.ConvPlan(xs[l], wk, o, k, relu=True, bias=bias, gn_stats=st))
        assert torch.equal(o, outs[l]), (what, l)
        if gn:
            assert torch.equal(st, sts[l]), (what, l)


# ------------------------------------------------------------------------------------------------ host-side rejection
def test_misaligned_residual_is_rejected_on_the_host():
    """A residual that is only 2-byte aligned cannot be read as __half2 pairs: smb_conv_run refuses it without a launch."""
    from sipmask_b200 import _lib
    N, H, W, cin, cout = 1, 5, 7, 64, 64
    g = _gen(1)
    x = _randn(g, N, H, W, cin)
    wk = _weight(g, cout, cin, 1)
    n = N * H * W * cout
    buf = torch.zeros((n + 8,), dtype=torch.float16, device='cuda')
    res = buf[1:1 + n].view(N, H, W, cout)
    assert res.data_ptr() % 4 == 2
    out = torch.full((N, H, W, cout), float('nan'), dtype=torch.float16, device='cuda')
    plan = _plan(x, wk, out, 1, residual=res)
    with pytest.raises(_lib.SmbError, match='4-byte aligned'):
        plan.run()
    torch.cuda.synchronize()
    assert torch.isnan(out.float()).all(), 'the rejected launch wrote its output'


# ------------------------------------------------------------------------------------- engines on short canvases
def _oracle_feats(sd, img):
    from oracle import model as M
    net = M.SipMaskDetector(50)
    net.load_state_dict(sd, strict=True)
    net.eval()
    with torch.no_grad():
        return net.extract_feat(img)


@pytest.mark.parametrize('canvas,img_shape', [((64, 1344), (60, 1333, 3)), ((32, 64), (32, 61, 3))])
def test_engine_on_short_canvas(canvas, img_shape):
    """Engines whose FPN P6 / P7 convolutions see 1-row (and 1-column) maps: every layer within its bound (the layer
    audit), and P3-P7 against the fp32 CPU oracle as in the full-size parity test."""
    from sipmask_b200 import synth
    from sipmask_b200.engine import SipMaskEngine
    from test_gpu_layer_audit import audit
    H, W = canvas
    sd = synth.detector_state_dict(50, 4, gn=True, seed=1, cls_bias=-2.5)
    img = synth.synthetic_image(H, W, seed=0)
    eng = SipMaskEngine(sd, canvas, img_shape=img_shape, use_graph=False)
    p6, p7 = eng.fpn_outs[3], eng.fpn_outs[4]
    assert min(p6.shape[1], p7.shape[1]) == 1 or min(p6.shape[2], p7.shape[2]) == 1, (p6.shape, p7.shape)
    eng.img.copy_(img)
    lines = []
    audit(eng, log=lines.append)
    print('\n'.join(lines))
    feats = _oracle_feats(sd, img)
    for l, (p, r) in enumerate(zip(eng.fpn_outs, feats)):
        a, b = p.float().cpu().permute(0, 3, 1, 2).double().flatten(), r.double().flatten()
        e = ((a - b).norm() / (b.norm() + 1e-12)).item()
        assert e < 1e-2, 'canvas %s: FPN level %d rel err %g' % (canvas, l, e)
