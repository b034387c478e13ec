"""The fine-tuning operators of csrc/train_ops.cu at their edges (run with -m gpu; -s prints each case's configuration).

  * smb_deform_weight_grad on fp16 operands given directly (teacher forcing): every split configuration (one split, one
    pixel block per split, a short last split, P below / at / just past one 64-pixel block, many splits), ragged M and N
    tiles down to Cout = K = 8.  Integer operands make dW exact, so it must be the float64 value bit for bit; random
    operands are held to a per-element bound.  The operands lie inside NaN-filled buffers and dW is followed by NaN
    sentinel words, so a read past a tensor map or a write past dW shows.
  * the grad_col GEMM of the backward (a 1x1 plan, K = Cout, N = 9 Cin, fp32 output) at the planner's N tiles;
  * smb_deform_col2im: grad_offset independent of grad_input and of the offset's pitch, grad_input of grad_offset;
  * smb_deform_grad_scale against a restatement of its scale rule, at the clamps, with non-finite inputs and with the
    maximum in the first, the last and the last block's elements;
  * the module at fp16 inputs, im2col_step, zero and out-of-map gradients, a non-contiguous grad_output.
"""
import ctypes

import pytest
import torch

import train_ops_inputs as T
from oracle import numerics as NU

pytestmark = pytest.mark.gpu

NAN = float('nan')


def _cdiv(a, b):
    return -(-a // b)


def _gen(seed):
    return torch.Generator().manual_seed(seed)


# -------------------------------------------------------------------------------------------- weight gradient (wgmma)
WG_TILE, WG_KB, WG_TARGET_CTAS = 128, 64, 264


def wgrad_split(cout, kc, P):
    """The kernel's split rule (wgrad_split in csrc/train_ops.cu) -> (pixel blocks, blocks per split, splits)."""
    tiles = _cdiv(cout, WG_TILE) * _cdiv(kc, WG_TILE)
    kb_total = _cdiv(P, WG_KB)
    want = max(1, min(_cdiv(WG_TARGET_CTAS, tiles), kb_total))
    kps = _cdiv(kb_total, want)
    return kb_total, kps, _cdiv(kb_total, kps)


def _splits_from_workspace(cout, kc, P):
    from sipmask_b200 import _lib as L
    n = int(L.lib().smb_deform_weight_grad_workspace_bytes(cout, kc, ctypes.c_longlong(P)))
    assert n % (cout * kc * 4) == 0
    return n // (cout * kc * 4)


# (Cout, K, P, what the case is for)
WGRAD_CASES = [
    (1024, 9216, 300, 'one split (576 tiles)'),
    (128, 576, 1280, 'one pixel block per split'),
    (128, 576, 6800, 'last split shorter'),
    (8, 8, 40, 'P < 64, Cout = K = 8'),
    (64, 72, 64, 'P = 64, upper warpgroup box out of bounds'),
    (72, 72, 65, 'P = 65, last split one pixel'),
    (192, 1728, 33600, 'large P, many splits'),
    (1024, 72, 1000, 'ragged N inside a box'),
    (8, 9216, 200, 'Cout 8, wide K'),
    (64, 1728, 500, 'Cout 64'),
    (72, 576, 3000, 'ragged M inside a box'),
    (192, 8, 129, 'K = 8, ragged M'),
    (128, 9216, 4096, 'whole tiles, several blocks per split'),
]


def _nan_embedded(t, lead, tail):
    """t as a contiguous view at element `lead` of a NaN-filled buffer with `tail` NaN elements after it."""
    buf = torch.full((lead + t.numel() + tail,), NAN, dtype=t.dtype, device=t.device)
    v = buf[lead:lead + t.numel()].view(t.shape)
    v.copy_(t)
    assert v.data_ptr() % 16 == 0
    return v


def _wgrad_direct(g16, col, scale):
    """smb_deform_weight_grad through the C entry point, with 4 NaN words before dW, 64 after it and 64 after the
    workspace; asserts that every sentinel word is unchanged afterwards.  -> dW [Cout, K]."""
    from sipmask_b200 import _lib as L
    P, cout = g16.shape
    kc = col.shape[1]
    n = cout * kc
    out = torch.full((4 + n + 64,), NAN, dtype=torch.float32, device='cuda')
    wsb = int(L.lib().smb_deform_weight_grad_workspace_bytes(cout, kc, ctypes.c_longlong(P)))
    ws = torch.full((wsb // 4 + 64,), NAN, dtype=torch.float32, device='cuda')
    before = (out[:4].clone(), out[4 + n:].clone(), ws[wsb // 4:].clone())
    dw = out[4:4 + n].view(cout, kc)
    L.check(L.lib().smb_deform_weight_grad(L.ptr(g16), L.ptr(col), ctypes.c_longlong(P), cout, kc, L.ptr(scale),
                                           L.ptr(dw), L.ptr(ws), ctypes.c_size_t(wsb), L.stream_ptr()),
            'smb_deform_weight_grad')
    torch.cuda.synchronize()
    after = (out[:4], out[4 + n:], ws[wsb // 4:])
    for a, b in zip(before, after):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32)), 'smb_deform_weight_grad wrote past dW / workspace'
    return dw.clone()


@pytest.mark.parametrize('mode', ['exact s=1', 'exact s=2^8', 'random'])
@pytest.mark.parametrize('cout,kc,P,what', WGRAD_CASES)
def test_weight_grad(cout, kc, P, what, mode):
    from sipmask_b200 import conv
    kb_total, kps, splits = wgrad_split(cout, kc, P)
    assert _splits_from_workspace(cout, kc, P) == splits, what
    last = kb_total - (splits - 1) * kps
    tiles = _cdiv(cout, WG_TILE) * _cdiv(kc, WG_TILE)
    # the configuration each case was written for
    assert {'one split (576 tiles)': splits == 1 and tiles >= WG_TARGET_CTAS,
            'one pixel block per split': kps == 1 and splits == kb_total > 1,
            'last split shorter': 0 < last < kps,
            'P < 64, Cout = K = 8': P < 64 and kb_total == 1,
            'P = 64, upper warpgroup box out of bounds': P == 64 and kb_total == 1 and cout <= 64,
            'P = 65, last split one pixel': kb_total == 2 and splits == 2,
            'large P, many splits': splits >= 8 and kps >= 32,
            'ragged N inside a box': kc % 64 != 0,
            'Cout 8, wide K': cout == 8 and kc == 9216,
            'Cout 64': cout == 64,
            'ragged M inside a box': cout % 64 != 0,
            'K = 8, ragged M': kc == 8 and cout % 128 != 0,
            'whole tiles, several blocks per split': kps > 1 and cout % 128 == 0 and kc % 128 == 0}[what], what
    print('wgrad %-42s Cout %4d K %4d P %5d: %2d M x %2d N tiles, %3d blocks, %2d per split, %2d splits (last %d)  %s' % (
        what, cout, kc, P, _cdiv(cout, WG_TILE), _cdiv(kc, WG_TILE), kb_total, kps, splits, last, mode))
    g = _gen(cout * 7 + kc * 3 + P)
    if mode.startswith('exact'):
        # integers in [-4, 4]: every product is an integer <= 16 and every partial sum <= 16 P < 2^20, exact in fp32
        # however the tensor cores and the split reduction order it; 1/s is a power of two
        g16 = torch.randint(-4, 5, (P, cout), generator=g).half().cuda()
        col = torch.randint(-4, 5, (P, kc), generator=g).half().cuda()
        s = 1.0 if mode == 'exact s=1' else 2.0 ** 8
    else:
        g16 = (torch.randn(P, cout, generator=g) * 2.0 ** 12).half().cuda()
        col = torch.randn(P, kc, generator=g).half().cuda()
        s = 2.0 ** 4
    scale = torch.tensor([s, 1.0 / s], dtype=torch.float32, device='cuda')
    tail = WG_KB * max(cout, kc) + 64                     # more than one pixel block past the end
    gv = _nan_embedded(g16, 8, tail)
    cv = _nan_embedded(col, 8, tail)
    dw = _wgrad_direct(gv, cv, scale)
    g64, c64 = g16.double(), col.double()
    want = (g64.t() @ c64) / s
    if mode.startswith('exact'):
        assert torch.equal(dw.double(), want), (what, (dw.double() - want).abs().max().item())
    else:
        m = (g64.abs().t() @ c64.abs()) / s
        bound = 2.0 ** -23 * want.abs() + (NU.gamma_k(WG_KB * kps) + (splits - 1) * 2.0 ** -24) * m
        NU.check_bound(dw.view(1, 1, cout, kc), want.view(1, 1, cout, kc), bound.view(1, 1, cout, kc),
                       what='wgrad %s' % what, fp16=False)
        assert torch.equal(conv.deform_weight_grad(gv, cv, scale), dw), 'two runs differ: %s' % what


# ---------------------------------------------------------------------------------------- grad_col GEMM (1x1, fp32)
def _expected_n_tile(n, min_tiles, tiles_m):
    """The planner's N tile: the largest of 256 / 128 / 64 not above N rounded up to 64 that still gives min_tiles
    tiles, else 64."""
    cmax = _cdiv(n, 64) * 64
    for c in (256, 128, 64):
        if c <= cmax and tiles_m * _cdiv(n, c) >= min_tiles:
            return c
    return 64


@pytest.mark.parametrize('cout,cin', [(64, 64), (64, 256), (64, 1024), (128, 192), (1024, 64), (1024, 1024)])
def test_grad_col_gemm(cout, cin):
    """grad_col = g16 . W as the backward runs it: ConvPlan(g16 [N,H,W,Cout], W^T [9 Cin, Cout], fp32 out, 1x1)."""
    from sipmask_b200 import conv
    N, H, W = 2, 13, 21
    g = _gen(cout + cin)
    w = torch.randn(cout, cin, 3, 3, generator=g) / (3 * cin ** 0.5)
    wt = conv.pack_weight(w, device='cuda')[0].t().contiguous()                   # [9 Cin, Cout] K-major, as backward
    g16 = (torch.randn(N, H, W, cout, generator=g) * 2.0 ** 12).half().cuda()
    out = torch.full((N, H, W, 9 * cin), NAN, dtype=torch.float32, device='cuda')
    min_tiles = conv.set_min_tiles(1)
    conv.set_min_tiles(min_tiles)
    plan = conv.ConvPlan(g16, wt, out, 1, 1)
    info = plan.info()
    n = 9 * cin
    want_tile = _expected_n_tile(n, min_tiles, info['tiles_m'])
    what = 'grad_col K %d N %d on %dx%dx%d' % (cout, n, N, H, W)
    assert info['num_levels'] == 1 and info['levels'][0]['H_out'] == H and info['levels'][0]['W_out'] == W, what
    assert info['n_tile'] == want_tile and info['n_tiles_n'] == _cdiv(n, want_tile), (what, info)
    assert info['epi_tma'] == 0, (what, info)                                 # fp32 output: the register epilogue
    print('%-40s n_tile %3d x%-3d tiles_m %d  register fp32' % (what, info['n_tile'], info['n_tiles_n'], info['tiles_m']))
    plan.run()
    torch.cuda.synchronize()
    y, m = NU.conv_reference(g16, wt, 1)
    NU.check_conv(out, y, m, cout, what=what)


# -------------------------------------------------------------------------------------------------------- col2im
def _col2im_operands(B, C, H, W, dg):
    x, off, gcol = T.col2im_inputs(B, C, H, W, dg)
    gcl = gcol.view(C, 9, B, H, W).permute(2, 3, 4, 1, 0).reshape(B, H, W, 9 * C).contiguous().cuda()
    return x.permute(0, 2, 3, 1).contiguous().half().cuda(), off.permute(0, 2, 3, 1).contiguous().cuda(), gcl


@pytest.mark.parametrize('B,C,H,W,dg', T.COL2IM_CASES)
def test_col2im_outputs_independent(B, C, H, W, dg):
    """grad_offset (fixed-order sums): the same bits with and without grad_input, over two runs and with the offsets a
    channel slice of a wider tensor.  grad_input (float atomics): the same with and without grad_offset, up to the
    order of the atomic additions."""
    from sipmask_b200 import conv
    xh, off, gcl = _col2im_operands(B, C, H, W, dg)
    one = torch.ones(2, device='cuda')
    vecs = C // 8
    print('col2im B %d C %4d dg %2d map %2dx%-2d: %d-%d vectors per lane, %d groups per lane' % (
        B, C, dg, H, W, vecs // 32, _cdiv(vecs, 32), _cdiv(dg, 32)))
    gin, goff = conv.deform_col2im(gcl, xh, off, dg, one)
    _, goff2 = conv.deform_col2im(gcl, xh, off, dg, one, grad_input=False)
    gin2, none = conv.deform_col2im(gcl, xh, off, dg, one, grad_offset=False)
    _, goff3 = conv.deform_col2im(gcl, xh, off, dg, one)
    wide = torch.full((B, H, W, dg * 18 + 24), NAN, dtype=torch.float32, device='cuda')
    offs = wide[..., 8:8 + dg * 18]
    offs.copy_(off)
    assert offs.stride(2) == dg * 18 + 24
    gin4, goff4 = conv.deform_col2im(gcl, xh, offs, dg, one)
    torch.cuda.synchronize()
    assert none is None and torch.isfinite(goff).all() and torch.isfinite(gin).all()
    for name, o in (('without grad_input', goff2), ('second run', goff3), ('offset pitch %d' % offs.stride(2), goff4)):
        assert torch.equal(o.view(torch.int32), goff.view(torch.int32)), 'grad_offset differs: %s' % name
    # bilinear weights are non-negative: grad_input of |grad_col| is the sum of the magnitudes of every atomic addend
    mag, _ = conv.deform_col2im(gcl.abs(), xh, off, dg, one, grad_offset=False)
    bound = 2.0 ** -16 * mag.double()
    for name, o in (('without grad_offset', gin2), ('offset pitch', gin4)):
        assert ((o.double() - gin.double()).abs() <= bound).all(), 'grad_input differs: %s' % name


# ------------------------------------------------------------------------------------------------ gradient scaling
def scale_from_amax_bits(bits):
    """{s, 1/s} of smb_deform_grad_scale for amax |grad_out| given as fp32 bits (scale_from_amax_bits in train_ops.cu)."""
    k = 0
    if bits != 0 and bits < 0x7f800000:
        e = (bits >> 23) - 127
        k = min(max(14 - e, -126), 126)
    return k


def _amax_bits(g):
    return int((g.view(torch.int32) & 0x7fffffff).max().item())


def _scale_case(name, shape):
    """-> (grad_out [N,C,H,W] fp32 on the device, the exponent k the case was written for, or None)."""
    r = torch.randn(shape, generator=_gen(sum(map(ord, name))))
    n = r.numel()

    def put(t, i, v):
        t = t.clone().view(-1)
        t[i] = v
        return t.view(shape)
    cases = {
        'zeros': lambda: (torch.zeros(shape), 0),
        'amax 2^14': lambda: (put(r.clamp(-8, 8), n // 3, 2.0 ** 14), 0),
        'amax 2^15 - 2^-9': lambda: (put(r.clamp(-8, 8), 5, -(2.0 ** 15 - 2.0 ** -9)), 0),
        'amax 70000 (s < 1)': lambda: (put(r, n - 2, 70000.0), -2),
        'amax FLT_MAX': lambda: (put(r, 7, 3.4028234663852886e38), -113),
        'amax 2^-117 (clamp at 126)': lambda: (put(r.clamp(-3.9, 3.9) * 2.0 ** -119, 1, 2.0 ** -117), 126),
        'subnormal amax': lambda: (r.clamp(-1, 1) * 1e-40, 126),
        'negative only': lambda: (-(r.abs().clamp(2.0, 3.9)) * 2.0 ** -20, 33),
        '+inf': lambda: (put(r, n // 2, float('inf')), 0),
        'NaN': lambda: (put(r, n - 1, NAN), 0),
        'amax first element': lambda: (put(r.clamp(-3.9, 3.9), 0, 100.0), 8),
        'amax last element': lambda: (put(r.clamp(-3.9, 3.9), n - 1, -100.0), 8),
        'amax in the last block': lambda: (put(r.clamp(-3.9, 3.9), LAST_BLOCK_ELEM, 100.0), 8),
        'C 8 HW 1': lambda: (r * 1e-3, None),
        'one block': lambda: (r * 1e-3, None),
        'capped grid, amax last': lambda: (put(r.clamp(-3.9, 3.9), n - 1, 300.0), 6),
    }
    t, k = cases[name]()
    return t.float().contiguous().cuda(), k


LAST_BLOCK_ELEM = 99 * 256 + 17                 # read by block 99 in its first pass when the grid has 100 blocks


SCALE_CASES = [('zeros', (1, 64, 5, 7)), ('amax 2^14', (2, 64, 9, 11)), ('amax 2^15 - 2^-9', (2, 64, 9, 11)),
               ('amax 70000 (s < 1)', (2, 64, 9, 11)), ('amax FLT_MAX', (1, 128, 13, 21)),
               ('amax 2^-117 (clamp at 126)', (1, 256, 13, 21)), ('subnormal amax', (1, 256, 13, 21)),
               ('negative only', (2, 64, 9, 11)), ('+inf', (1, 64, 9, 11)), ('NaN', (1, 64, 9, 11)),
               ('amax first element', (1, 64, 40, 80)), ('amax last element', (1, 64, 40, 80)),
               ('amax in the last block', (1, 64, 40, 80)), ('C 8 HW 1', (1, 8, 1, 1)), ('one block', (2, 16, 4, 4)),
               ('capped grid, amax last', (2, 256, 100, 84))]


def _same_half_bits(a, b):
    na, nb = torch.isnan(a), torch.isnan(b)
    assert torch.equal(na, nb)
    z = torch.zeros((), dtype=a.dtype, device=a.device)
    return torch.equal(torch.where(na, z, a).view(torch.int16), torch.where(nb, z, b).view(torch.int16))


@pytest.mark.parametrize('name,shape', SCALE_CASES)
def test_grad_scale(name, shape):
    from sipmask_b200 import conv
    g, k_case = _scale_case(name, shape)
    N, C, H, W = shape
    bits = _amax_bits(g)
    k = scale_from_amax_bits(bits)
    blocks = _cdiv(g.numel() // 8, 256)
    # the configuration each case was written for
    if k_case is not None:
        assert k == k_case, (name, k)
    if name == 'subnormal amax':
        assert 0 < bits < 0x00800000
    if name == 'amax 2^-117 (clamp at 126)':
        assert 14 - ((bits >> 23) - 127) > 126
    if name in ('+inf', 'NaN'):
        assert bits >= 0x7f800000
    if name == 'negative only':
        assert (g < 0).all()
    if name == 'amax in the last block':
        assert blocks == 100 and g.view(-1)[LAST_BLOCK_ELEM].item() == 100.0
    if name == 'one block':
        assert blocks == 1
    if name.startswith('capped grid'):
        props = torch.cuda.get_device_properties(0)
        assert blocks > props.multi_processor_count * (props.max_threads_per_multi_processor // 256)
    print('grad scale %-28s %dx%dx%dx%d: %5d blocks wanted, amax bits %08x, s = 2^%d' % (name, N, C, H, W, blocks, bits, k))
    out, scale = conv.deform_grad_scale(g)
    torch.cuda.synchronize()
    assert scale.cpu().tolist() == [2.0 ** k, 2.0 ** -k], (name, scale.cpu().tolist(), k)
    want = (g * torch.tensor(2.0 ** k, dtype=torch.float32, device='cuda')).half().permute(0, 2, 3, 1).contiguous()
    assert out.shape == (N, H, W, C) and out.dtype == torch.float16
    assert _same_half_bits(out, want), name
    if name == 'zeros':
        assert not out.float().any()


# --------------------------------------------------------------------------------------------------- module level
def _module_inputs(B, C, Cout, H, W, dg, seed=0):
    g = _gen(seed + C + H)
    x = torch.randn(B, C, H, W, generator=g).half().float()
    off = torch.round(torch.randn(B, dg * 18, H, W, generator=g) * 2.0 * 1024) / 1024
    w = (torch.randn(Cout, C, 3, 3, generator=g) / (3 * C ** 0.5)).half().float()
    gy = torch.randn(B, Cout, H, W, generator=g) * 1e-3
    return x.cuda(), off.cuda(), w.cuda(), gy.cuda()


def _rel(a, b):
    a, b = a.double(), b.double()
    return ((a - b).norm() / b.norm()).item()


def _grads(x, off, w, gy, dg, im2col_step=64):
    from sipmask_b200 import ops
    xr, offr, wr = x.clone().requires_grad_(True), off.clone().requires_grad_(True), w.clone().requires_grad_(True)
    ops.deform_conv(xr, offr, wr, 1, 1, 1, 1, dg, im2col_step).backward(gy)
    return xr.grad, offr.grad, wr.grad


def _ref64(x, off, w, gy, dg):
    from oracle import ops as O
    x64, off64, w64 = [t.double().requires_grad_(True) for t in (x, off, w)]
    with torch.device('cuda'):
        O.deform_conv(x64, off64, w64, padding=1, deformable_groups=dg).backward(gy.double())
    return x64.grad, off64.grad, w64.grad


def test_fp16_inputs_give_fp16_gradients():
    """fp16 x and offsets: grad_input and grad_offset come back in fp16 (the reference returns the input's dtype), dW in
    fp32, all within the module bound of test_gpu_deform_conv_grad.py plus the fp16 rounding of the output."""
    x, off, w, gy = _module_inputs(2, 128, 64, 13, 21, 2)
    xh, offh = x.half(), off.half()                     # the float64 reference sees the same fp16 values
    got = _grads(xh, offh, w, gy, 2)
    want = _ref64(xh.float(), offh.float(), w, gy, 2)
    print('fp16 inputs 2x128x13x21 -> Cout 64, dg 2: grad dtypes %s' % [str(t.dtype)[6:] for t in got])
    assert [t.dtype for t in got] == [torch.float16, torch.float16, torch.float32]
    for name, a, b in zip(('grad_input', 'grad_offset', 'grad_weight'), got, want):
        assert torch.isfinite(a).all(), name
        assert _rel(a, b) <= 3e-3 + 2.0 ** -11, (name, _rel(a, b))


def test_im2col_step():
    """The backward does not depend on im2col_step (the reference splits the batch into steps; here one pass covers it):
    im2col_step 1, 2 and 4 at B = 4 give the same dW and grad_offset bits; 3 does not divide the batch and raises the
    reference's assertion."""
    from sipmask_b200 import ops
    x, off, w, gy = _module_inputs(4, 64, 64, 9, 11, 1)
    print('im2col_step 1, 2, 4 and 3 at B = 4, 64 -> 64 channels, 9x11')
    ref = _grads(x, off, w, gy, 1, 4)
    for step in (1, 2):
        got = _grads(x, off, w, gy, 1, step)
        assert torch.equal(got[2], ref[2]) and torch.equal(got[1], ref[1]), step
    with pytest.raises(AssertionError, match='im2col step must divide batchsize'):
        ops.deform_conv(x, off, w, 1, 1, 1, 1, 1, 3)


def test_zero_grad_out_gives_zero_gradients():
    x, off, w, gy = _module_inputs(2, 256, 128, 13, 21, 4)
    print('zero grad_out, 2x256x13x21 -> 128, dg 4')
    for name, t in zip(('grad_input', 'grad_offset', 'grad_weight'), _grads(x, off, w, torch.zeros_like(gy), 4)):
        assert not torch.isnan(t).any() and not t.any(), name


def test_samples_outside_the_map_give_zero_gradients():
    """Offsets of +-1000 put every sampling point outside (-1, H) x (-1, W): the columns, the output and all three
    gradients are exactly zero."""
    x, off, w, gy = _module_inputs(2, 256, 128, 13, 21, 4)
    sign = torch.where(torch.randn(off.shape, generator=_gen(3)) > 0, 1.0, -1.0).cuda()
    far = sign * 1000.0
    print('offsets +-1000, 2x256x13x21 -> 128, dg 4')
    from sipmask_b200 import ops
    assert not ops.deform_conv(x, far, w, 1, 1, 1, 1, 4).any()
    for name, t in zip(('grad_input', 'grad_offset', 'grad_weight'), _grads(x, far, w, gy, 4)):
        assert not torch.isnan(t).any() and not t.any(), name


def test_non_contiguous_grad_output():
    """A grad_output in channels-last memory, and the gradient of a loss over y[:, :, 1:] (zero first row), against
    float64."""
    from sipmask_b200 import ops
    x, off, w, _ = _module_inputs(2, 128, 128, 13, 21, 4)
    g = _gen(5)
    gy_cl = (torch.randn(2, 13, 21, 128, generator=g) * 1e-3).cuda().permute(0, 3, 1, 2)
    seen = []
    xr, offr, wr = x.clone().requires_grad_(True), off.clone().requires_grad_(True), w.clone().requires_grad_(True)
    y = ops.deform_conv(xr, offr, wr, 1, 1, 1, 1, 4)
    y.register_hook(lambda t: seen.append(t.is_contiguous()))
    y.backward(gy_cl)
    assert seen == [False]
    print('channels-last grad_output and a loss over y[:, :, 1:], 2x128x13x21 -> 128, dg 4')
    want = _ref64(x, off, w, gy_cl.contiguous(), 4)
    for name, a, b in zip(('grad_input', 'grad_offset', 'grad_weight'), (xr.grad, offr.grad, wr.grad), want):
        assert _rel(a, b) <= 3e-3, (name, _rel(a, b))
    gy_row = (torch.randn(2, 128, 13, 21, generator=g) * 1e-3).cuda()
    xr, offr, wr = x.clone().requires_grad_(True), off.clone().requires_grad_(True), w.clone().requires_grad_(True)
    (ops.deform_conv(xr, offr, wr, 1, 1, 1, 1, 4)[:, :, 1:] * gy_row[:, :, 1:]).sum().backward()
    gy_full = gy_row.clone()
    gy_full[:, :, 0] = 0
    want = _ref64(x, off, w, gy_full, 4)
    for name, a, b in zip(('grad_input', 'grad_offset', 'grad_weight'), (xr.grad, offr.grad, wr.grad), want):
        assert _rel(a, b) <= 3e-3, (name, _rel(a, b))


def test_one_pixel_maps_through_the_function():
    """deform_conv itself (no padding by a module) on 1 x 1 maps of two images.  A permuted 1 x 1 offset tensor counts as
    contiguous with stride(2) == 1, so its pixel pitch has to come from the image stride: the second image must sample
    with its own offsets in the forward and in both gradient kernels."""
    x, off, w, gy = _module_inputs(2, 64, 64, 1, 1, 1, seed=7)
    off = off * 0.25                                    # most sampling points inside (-1, 1) x (-1, 1)
    print('deform_conv on 2 x 64 x 1 x 1 maps, dg 1: offset pixel pitch from the image stride')
    from oracle import ops as O
    from sipmask_b200 import ops
    with torch.device('cuda'):
        y64 = O.deform_conv(x.double(), off.double(), w.double(), padding=1)
    y = ops.deform_conv(x, off, w, 1, 1, 1, 1, 1)
    assert y[1].abs().max() > 0
    assert _rel(y, y64) <= 3e-3, _rel(y, y64)
    names = ('grad_input', 'grad_offset', 'grad_weight')
    got, want = _grads(x, off, w, gy, 1), _ref64(x, off, w, gy, 1)
    for name, a, b in zip(names, got, want):
        assert _rel(a, b) <= 3e-3, (name, _rel(a, b))
    for name, a, b in zip(names[:2], got[:2], want[:2]):            # the second image on its own
        assert b[1].abs().max() > 0 and _rel(a[1], b[1]) <= 3e-3, (name, _rel(a[1], b[1]))
