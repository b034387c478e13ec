"""The per-element checker of the layer audit (oracle/numerics.py) accepts a correct kernel and rejects small defects.

A correct kernel is emulated on the CPU: fp16 operands multiplied exactly and accumulated in fp32, the fp32 epilogue
(bias, alpha, residual, ReLU) and one rounding to fp16.  Each planted defect touches one 128-pixel tile (or one GroupNorm
partial) of a layer at an engine-like shape, and must be rejected with a message that names the element and its tile."""
import re

import pytest
import torch
import torch.nn.functional as F

from oracle import numerics as NU


def _operands(N, H, W, cin, cout, k, seed, res_hw=None, cout_pad=None):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, H, W, cin, generator=g).half()
    w = (torch.randn(cout, k * k * cin, generator=g) / (k * k * cin) ** 0.5)
    if cout_pad:
        w = torch.cat([w, torch.zeros(cout_pad - cout, w.shape[1])])
        cout = cout_pad
    bias = torch.randn(cout, generator=g) * 0.5
    res = torch.randn(N, res_hw[0], res_hw[1], cout, generator=g).half() if res_hw else None
    return x, w.half(), bias, res


def _emulate(x16, w16, k, stride=1, bias=None, alpha=1.0, residual=None, relu=False, out_dtype=torch.float16,
             drop_k=None, shift_tap=None, parity=0):
    """fp32-accumulating convolution of the fp16 operands -> (out, pre-activation fp32).  Defect knobs: drop_k = K column
    left out of the sum, shift_tap = (tap, dx) reads that tap one pixel off, parity = 1 samples the odd input positions."""
    x = x16.float()
    N, H, W, Cin = x.shape
    p = k // 2
    Ho, Wo = (H + 2 * p - k) // stride + 1, (W + 2 * p - k) // stride + 1
    xp = F.pad(x, (0, 0, p + 1, p + 1, p + 1, p + 1))          # one spare pixel on every side for the defects
    taps = []
    for r in range(k):
        for s in range(k):
            dx = shift_tap[1] if shift_tap is not None and shift_tap[0] == r * k + s else 0
            y0, x0 = 1 + r + parity, 1 + s + parity + dx
            taps.append(xp[:, y0:y0 + (Ho - 1) * stride + 1:stride, x0:x0 + (Wo - 1) * stride + 1:stride, :])
    col = torch.cat(taps, 3).reshape(-1, k * k * Cin)
    w = w16.float().t().clone()
    if drop_k is not None:
        w[drop_k] = 0
    acc = (col @ w).view(N, Ho, Wo, -1)
    if bias is not None:
        acc = acc + bias.float()
    if alpha != 1.0:
        acc = acc * alpha
    if residual is not None:
        acc = acc + residual.float()
    out = acc.clamp(min=0) if relu else acc
    return out.to(out_dtype), acc


def _tile(Ho, Wo, ty, tx, nb):
    bh, bw = NU.conv_patch(Ho, Wo)
    return (slice(None), slice(ty * bh, (ty + 1) * bh), slice(tx * bw, (tx + 1) * bw), slice(64 * nb, 64 * nb + 64))


def _check(out, x, w, k, stride=1, bias=None, alpha=1.0, residual=None, relu=False, what='conv'):
    y, m = NU.conv_reference(x, w, k, stride, bias=bias, alpha=alpha, residual=residual)
    return NU.check_conv(out, y, m, w.shape[1], relu=relu, what=what)


CASES = [   # N, H, W, cin, cout, k, stride, residual, relu, alpha, out dtype, cout_pad
    (2, 13, 21, 64, 128, 3, 1, False, False, 1.0, torch.float16, None),      # ragged 16 x 8 patches, 3x3
    (2, 25, 42, 128, 128, 1, 1, True, True, 1.0, torch.float16, None),       # 1x1 + residual + ReLU
    (2, 26, 42, 64, 128, 3, 2, False, True, 1.0, torch.float16, None),       # stride 2
    (1, 7, 11, 64, 24, 3, 1, False, False, 1.3, torch.float32, 32),           # fp32 head, alpha, Cout padded
    (1, 1, 2, 64, 64, 3, 1, False, False, 1.0, torch.float16, None),          # a 1 x 2 pyramid level
]


@pytest.mark.parametrize('N,H,W,cin,cout,k,stride,res,relu,alpha,dt,cpad', CASES)
def test_checker_accepts_emulated_kernel(N, H, W, cin, cout, k, stride, res, relu, alpha, dt, cpad):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    x, w, b, r = _operands(N, H, W, cin, cout, k, H * W + cin, (Ho, Wo) if res else None, cpad)
    out, _ = _emulate(x, w, k, stride, b, alpha, r, relu, dt)
    st = _check(out, x, w, k, stride, b, alpha, r, relu)
    assert st['ratio'] < 0.5, st
    if dt == torch.float16:
        assert st['misrounded'] <= NU.max_misrounded(w.shape[1]), st


def _rejects(out, *args, **kw):
    with pytest.raises(NU.BoundError) as e:
        _check(out, *args, **kw)
    msg = str(e.value)
    assert re.search(r'image \d+, y \d+, x \d+, channel \d+ \(tile \d+,\d+ of \d+x\d+ pixels, N block \d+\)', msg), msg
    return msg


def _plant(good, bad, sl):
    out = good.clone()
    out[sl] = bad[sl]
    return out


def test_rejects_one_dropped_k_channel_in_one_tile():
    x, w, b, _ = _operands(2, 13, 21, 64, 128, 3, 1)
    good, _ = _emulate(x, w, 3, bias=b)
    sl = _tile(13, 21, 0, 1, 1)
    bad, _ = _emulate(x, w, 3, bias=b, drop_k=4 * 64 + 17)           # centre tap, channel 17
    msg = _rejects(_plant(good, bad, sl), x, w, 3, bias=b)
    assert 'tile 0,1' in msg and 'N block 1' in msg, msg


def test_rejects_one_tap_shifted_by_a_pixel():
    x, w, b, _ = _operands(2, 13, 21, 64, 128, 3, 2)
    good, _ = _emulate(x, w, 3, bias=b)
    bad, _ = _emulate(x, w, 3, bias=b, shift_tap=(5, 1))
    msg = _rejects(_plant(good, bad, _tile(13, 21, 0, 2, 0)), x, w, 3, bias=b)
    assert 'tile 0,2' in msg, msg


def test_rejects_missing_bias_on_one_8_channel_block():
    x, w, b, _ = _operands(2, 25, 42, 128, 128, 1, 3)
    good, _ = _emulate(x, w, 1, bias=b, relu=True)
    b2 = b.clone()
    b2[72:80] = 0
    bad, _ = _emulate(x, w, 1, bias=b2, relu=True)
    msg = _rejects(_plant(good, bad, _tile(25, 42, 3, 0, 1)), x, w, 1, bias=b, relu=True)
    assert 'N block 1' in msg, msg


def test_rejects_residual_taken_from_the_other_image():
    x, w, b, r = _operands(2, 25, 42, 128, 128, 1, 4, res_hw=(25, 42))
    good, _ = _emulate(x, w, 1, bias=b, residual=r, relu=True)
    bad, _ = _emulate(x, w, 1, bias=b, residual=r.flip(0), relu=True)
    sl = (slice(1, 2),) + _tile(25, 42, 2, 0, 0)[1:]
    msg = _rejects(_plant(good, bad, sl), x, w, 1, bias=b, residual=r, relu=True)
    assert 'image 1' in msg, msg


def test_rejects_stale_last_row_of_a_ragged_tile():
    x, w, b, _ = _operands(2, 13, 21, 64, 128, 3, 5)
    good, _ = _emulate(x, w, 3, bias=b)
    x_prev, _, _, _ = _operands(2, 13, 21, 64, 128, 3, 6)          # the previous forward's image
    stale, _ = _emulate(x_prev, w, 3, bias=b)
    bh, bw = NU.conv_patch(13, 21)
    assert 13 % bh and 21 % bw                                        # the last tile is ragged in both directions
    sl = (slice(None), slice(12, 13), slice(2 * bw, 21), slice(0, 128))
    msg = _rejects(_plant(good, stale, sl), x, w, 3, bias=b)
    assert 'y 12' in msg and 'tile 0,2' in msg, msg
    # a row the kernel never wrote at all (NaN-filled before the run)
    unwritten = good.clone()
    unwritten[sl] = float('nan')
    assert 'y 12' in _rejects(unwritten, x, w, 3, bias=b)


def test_rejects_swapped_stride2_parity():
    x, w, b, _ = _operands(2, 26, 42, 64, 128, 3, 7)
    good, _ = _emulate(x, w, 3, 2, bias=b, relu=True)
    bad, _ = _emulate(x, w, 3, 2, bias=b, relu=True, parity=1)
    Ho, Wo = good.shape[1], good.shape[2]
    msg = _rejects(_plant(good, bad, _tile(Ho, Wo, 0, 1, 1)), x, w, 3, 2, bias=b, relu=True)
    assert 'tile 0,1' in msg and 'N block 1' in msg, msg


def _gn_partials(pre):
    """The epilogue's fixed-point GroupNorm partials of an fp32 pre-activation [N, H, W, C] with 8- or 16-channel groups:
    [N, 32, n_partials, 2] int64, one per (tile, consumer warp = 16 patch rows), summed over the warp's valid pixels."""
    N, H, W, C = pre.shape
    bh, bw = NU.conv_patch(H, W)
    ys, xs = torch.meshgrid(torch.arange(H), torch.arange(W), indexing='ij')
    tiles_x = -(-W // bw)
    key = ((ys // bh) * tiles_x + xs // bw) * 8 + ((ys % bh) * bw + xs % bw) // 16
    nk = int(key.max()) + 1
    f = pre.double().reshape(N, H * W, 32, C // 32)
    part = torch.zeros(N, 32, nk, 2, dtype=torch.int64)
    for kk in range(nk):
        sel = (key.reshape(-1) == kk)
        if sel.any():
            fs = f[:, sel]
            part[:, :, kk, 0] = torch.round(fs.sum((1, 3)).float().double() * NU.GN_SUM_SCALE).long()
            part[:, :, kk, 1] = torch.round((fs * fs).sum((1, 3)).float().double() * NU.GN_SQ_SCALE).long()
    return part


def test_gn_statistics_accept_emulation_and_reject_one_missing_partial():
    x, w, b, _ = _operands(2, 13, 21, 256, 256, 3, 8)
    out, pre = _emulate(x, w, 3, bias=b)
    y, m = NU.conv_reference(x, w, 3, bias=b)
    part = _gn_partials(pre)
    stats = part.sum(2)
    assert NU.check_gn_stats(stats, y, m, w.shape[1]) < 0.5
    n, grp = 1, 9
    kk = int(torch.argmax(part[n, grp, :, 1]))                       # drop one partial (sum and sum of squares)
    bad = stats.clone()
    bad[n, grp] -= part[n, grp, kk]
    with pytest.raises(NU.BoundError, match='image 1, group 9'):
        NU.check_gn_stats(bad, y, m, w.shape[1])


def test_fp16_rounding_helpers():
    v = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 3 * 2 ** -11, 2.0 ** -20, 65504.0, -3.0 - 2 ** -10 - 2 ** -30],
                     dtype=torch.float64)
    assert NU.fp16_spacing(v).tolist() == [2 ** -10, 2 ** -10, 2 ** -10, 2 ** -24, 32.0, 2 ** -9]
    # ties to even, one rounding: -3 - 2^-10 - 2^-30 is just past the midpoint -> rounds away from -3
    assert NU.round_to_fp16(v).tolist() == [1.0, 1.0, 1.0 + 4 * 2 ** -11, 2.0 ** -20, 65504.0, -3.0 - 2 ** -9]
    assert NU.round_to_fp16(v).tolist() == v.numpy().astype('float16').astype('float64').tolist()


def _rescore_emulation(seed=0, H=127, W=131, n_img=2, max_rows=3, count=(2, 1)):
    """The fp16-storage / fp32-accumulate rescoring chain on the CPU, its layers 2-5 in 0xFF-filled buffers."""
    g = torch.Generator().manual_seed(seed)
    ch = (1, 16, 16, 16, 32, 64, 128)
    cw = [(torch.randn(ch[i + 1], 9 * ch[i], generator=g) * (2.0 / (9 * ch[i])) ** 0.5).half() for i in range(6)]
    cb = [torch.randn(ch[i + 1], generator=g) * 0.05 for i in range(6)]
    sw = (torch.randn(80, 128, generator=g) / 128 ** 0.5).half()
    sb = torch.randn(80, generator=g) * 0.1
    pos = torch.rand(n_img, max_rows, H, W, generator=g).half()
    labels = torch.randint(0, 80, (n_img, max_rows), generator=g)
    det = torch.rand(n_img, max_rows, 5, generator=g)
    cnt = torch.tensor(count, dtype=torch.int32)
    R = n_img * max_rows
    x = pos.reshape(R, H, W, 1)
    acts = []
    for i in range(6):
        out, pre = _emulate_valid_s2(x, cw[i], cb[i])
        if i == 0:
            out = pre.clamp(min=0).half()           # layer 1: fp32 FMAs, ReLU, fp16
        acts.append(out)
        x = out
    layers = []
    for l in range(2, 6):
        a = torch.full(acts[l - 1].shape, -1, dtype=torch.int16).view(torch.float16)
        for n in range(n_img):
            a[n * max_rows:n * max_rows + int(cnt[n])] = acts[l - 1][n * max_rows:n * max_rows + int(cnt[n])]
        layers.append(a)
    h6 = acts[5].float()                            # conv 6, ReLU, fp16
    s = (h6 * sw.float()[labels.view(-1)].view(R, 1, 1, 128)).sum(-1) + sb[labels.view(-1)].view(R, 1, 1)
    scores = s.clamp(min=0).amax((1, 2)) * det.view(R, 5)[:, 4]
    live = torch.tensor([r % max_rows < int(cnt[r // max_rows]) for r in range(R)])
    scores = torch.where(live, scores, torch.zeros_like(scores)).view(n_img, max_rows)
    return pos, cnt, cw, cb, sw, sb, labels, det, layers, scores


def _emulate_valid_s2(x16, w16, b):
    """3x3 stride-2 valid convolution of fp16 NHWC, fp32 accumulation, + bias, ReLU -> (fp16, fp32 pre-activation)."""
    N, H, W, C = x16.shape
    Ho, Wo = (H - 3) // 2 + 1, (W - 3) // 2 + 1
    x = x16.float()
    taps = [x[:, r:r + 2 * (Ho - 1) + 1:2, s:s + 2 * (Wo - 1) + 1:2, :] for r in range(3) for s in range(3)]
    pre = (torch.cat(taps, 3).reshape(-1, 9 * C) @ w16.float().t()).view(N, Ho, Wo, -1) + b.float()
    return pre.clamp(min=0).half(), pre


def test_rescore_checker_accepts_emulation_and_rejects_defects():
    args = _rescore_emulation()
    res = NU.check_rescore_chain(*args)
    assert all(v < 1.0 for v in res.values()), res
    pos, cnt, cw, cb, sw, sb, labels, det, layers, scores = args
    bad = [t.clone() for t in layers]                       # one layer-3 value of a live row off by a few ulps
    bad[1][1, 5, 7, 3] = bad[1][1, 5, 7, 3] * 1.01 + 0.01
    with pytest.raises(NU.BoundError, match='layer 3'):
        NU.check_rescore_chain(pos, cnt, cw, cb, sw, sb, labels, det, bad, scores)
    bad = [t.clone() for t in layers]                       # a live row of layer 4 left unwritten
    bad[2][3, 0, 0, 0] = torch.tensor(-1, dtype=torch.int16).view(torch.float16)
    with pytest.raises(NU.BoundError, match='layer 4: live row 3'):
        NU.check_rescore_chain(pos, cnt, cw, cb, sw, sb, labels, det, bad, scores)
    bad = [t.clone() for t in layers]                       # a row past the count written
    bad[0][2] = 0
    with pytest.raises(NU.BoundError, match='row 2 past the count'):
        NU.check_rescore_chain(pos, cnt, cw, cb, sw, sb, labels, det, bad, scores)
    s2 = scores.clone()
    s2[0, 1] *= 1.05                                        # a score 5 % off
    with pytest.raises(NU.BoundError, match='score'):
        NU.check_rescore_chain(pos, cnt, cw, cb, sw, sb, labels, det, layers, s2)
