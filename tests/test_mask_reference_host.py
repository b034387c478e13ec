"""The float64 mask reference of oracle/numerics.py on the CPU: its crop geometry equals the C oracle's CropSplit at every
pixel, its values hold the oracle's fp32 masks within their bounds, its decided bits equal F.interpolate(...) > thr, and
check_mask_bits rejects planes built from deliberately wrong variants of the same computation (so the bound is not
vacuous)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import numerics as NU  # noqa: E402

THR = 0.4


def _case(H, W, N, seed, cof_scale=1.0):
    g = torch.Generator().manual_seed(seed)
    protos = torch.relu(torch.randn(32, H, W, generator=g))
    cofs = torch.randn(N, 128, generator=g) * cof_scale
    cx, cy = torch.rand(N, generator=g) * W * 2, torch.rand(N, generator=g) * H * 2
    bw, bh = torch.rand(N, generator=g) * W * 1.4 + 0.3, torch.rand(N, generator=g) * H * 1.4 + 0.3
    boxes = torch.stack([cx - bw / 2, cy - bh / 2, cx + bw / 2, cy + bh / 2], 1)
    boxes[0] = torch.tensor([0.0, 0.0, 2.0 * W, 2.0 * H])                 # whole image
    boxes[1] = torch.tensor([16.0, 8.0, 48.0, 24.0])                      # integer roi edges
    boxes[2] = torch.tensor([30.2, 14.6, 30.9, 15.3])                     # below one prototype pixel
    boxes[3] = torch.tensor([-7.0, -3.0, 21.0, 2.0 * H + 9.0])            # negative, hangs over the map
    boxes[4] = torch.tensor([20.0, 10.0, 12.0, 30.0])                     # x2 < x1: empty
    return protos, cofs, boxes


def _oracle():
    from oracle import cbind
    return cbind


@pytest.mark.parametrize('H,W,N', [(37, 53, 12), (9, 70, 7), (40, 64, 9)])
def test_crop_geometry_equals_oracle_crop_split(H, W, N):
    cbind = _oracle()
    _, _, boxes = _case(H, W, N, H + W)
    for scale in (0.5, np.array([0.6, 0.45, 0.6, 0.45], np.float32)):
        rois, _, _ = NU.crop_rois(boxes.numpy(), scale)
        data = np.broadcast_to(np.arange(1, 5, dtype=np.float32).reshape(4, 1, 1, 1), (4, H, W, N))
        want = cbind.crop_split(data, rois).transpose(2, 0, 1)            # cell + 1 inside the roi, 0 outside
        geo, _ = NU.crop_geometry(boxes.numpy(), scale, H, W)
        got = np.zeros((N, H, W), np.float32)
        for n, ((y0, y1, x0, x1), ih, iw) in enumerate(geo):
            got[n, y0:y1, x0:x1] = np.clip(2 * ih[:, None] + iw[None, :], 0, 3) + 1
        np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize('H,W,N,cof_scale', [(37, 53, 12, 1.0), (48, 62, 9, 40.0), (9, 70, 7, 1e-3)])
def test_values_bound_the_oracle_and_bits_equal_torch_interpolate(H, W, N, cof_scale):
    """The oracle's sequential fp32 masks lie within the scalar family's bounds; the reference's decided bits equal
    F.interpolate(oracle masks, align_corners=False) > thr for both coordinate rules and several factors."""
    cbind = _oracle()
    protos, cofs, boxes = _case(H, W, N, 3 * H + N, cof_scale)
    pos = cbind.mask_assemble(protos.numpy(), cofs.numpy(), (boxes * 0.5).numpy())
    vals = NU.mask_values(protos, cofs, boxes, 0.5, 'scalar')
    assert NU.check_mask_values(torch.from_numpy(pos), vals, 'oracle') <= 1.0
    assert sum(int(d.v.size) for d in vals) > 0
    for up in (2.0, 2.0 / 1.6667, (2 / 1.3, 2 / 1.7), 2.0 / 3.1, 2.5):
        sf = tuple(float(u) for u in up) if isinstance(up, tuple) else float(up)
        uh, uw = (up if isinstance(up, tuple) else (up, up))
        for legacy in (False, True):
            want = F.interpolate(torch.from_numpy(pos).unsqueeze(0), scale_factor=sf, mode='bilinear', align_corners=False,
                                 recompute_scale_factor=True if legacy else None).squeeze(0) > THR
            fh, fw = want.shape[1:]
            r = (0.0, 0.0) if legacy else (1.0 / uh, 1.0 / uw)
            for oh, ow in ((fh, fw), (fh - 3, fw - 5), (fh + 4, fw + 33)):
                ref = NU.resize_reference(vals, H, W, (fh, fw), r, (oh, ow), THR, proto_bytes=128)
                words = (ow + 31) // 32
                canvas = np.zeros((N, oh, words * 32), bool)
                canvas[:, :min(oh, fh), :min(ow, fw)] = want[:, :min(oh, fh), :min(ow, fw)].numpy()
                bits = np.packbits(canvas, axis=-1, bitorder='little').view(np.int32).reshape(N, oh, words)
                st = NU.check_mask_bits(bits, ref, N, what='interpolate up=%r legacy=%d' % (up, legacy))
                assert st['ambiguous'] < NU.MASK_AMBIGUOUS_CAP


def _honest(H=40, W=100, N=6, up=2.0 / 1.6667, out_pad=(0, -3)):
    protos, cofs, boxes = _case(H, W, N, 11, 40.0)                        # steep logits: many sharp mask edges
    boxes[1] = torch.tensor([0.0, 0.0, 2.0 * W, 2.0 * H])
    vals = NU.mask_values(protos, cofs, boxes, 0.5, 'scalar')
    fh, fw = int(np.floor(H * up)), int(np.floor(W * up))
    out_hw = (fh + out_pad[0], fw + out_pad[1])
    ref = NU.resize_reference(vals, H, W, (fh, fw), (1.0 / up, 1.0 / up), out_hw, THR, proto_bytes=128)
    words = (out_hw[1] + 31) // 32
    return protos, cofs, boxes, vals, ref, (H, W, (fh, fw), up, out_hw, words)


def test_reference_planes_pass():
    _, _, _, _, ref, (H, W, full, up, out_hw, words) = _honest()
    N = len(ref.dets)
    bits = NU.reference_bits(ref, N + 2, out_hw[0], words)
    st = NU.check_mask_bits(bits, ref, N)
    assert st['pixels'] == N * out_hw[0] * min(out_hw[1], full[1]) and st['margin'] > 1.0


def _wrong_resize(vals, shape, monkeypatch, tamper_x=None, r=None):
    """Planes of the reference computed with a tampered source index (x axis) or another step."""
    H, W, full, up, out_hw, words = shape
    orig = NU.src_index

    def patched(rr, n_out, n_in):
        forms = orig(rr, n_out, n_in)
        if tamper_x is not None and n_in == W:
            forms = [tamper_x(*f) for f in forms]
        return forms
    monkeypatch.setattr(NU, 'src_index', patched)
    try:
        ref = NU.resize_reference(vals, H, W, full, r or (1.0 / up, 1.0 / up), out_hw, THR, proto_bytes=128)
    finally:
        monkeypatch.setattr(NU, 'src_index', orig)
    return NU.reference_bits(ref, len(vals), out_hw[0], words)


def test_check_rejects_a_source_column_shifted_at_a_tile_seam(monkeypatch):
    _, _, _, vals, ref, shape = _honest()

    def shift(i0, i1, lam):                      # output pixels reading source column 64 (an 8x64 dense tile seam) read 65
        i0, i1 = i0.copy(), i1.copy()
        sel = i0 == 64
        i0[sel] += 1
        i1[sel] = np.minimum(i1[sel] + 1, shape[1] - 1)
        return i0, i1, lam
    bits = _wrong_resize(vals, shape, monkeypatch, tamper_x=shift)
    with pytest.raises(NU.BoundError, match='dense tile'):
        NU.check_mask_bits(bits, ref, len(vals))


def test_check_rejects_the_other_interpolation_rule(monkeypatch):
    _, _, _, vals, ref, shape = _honest()
    H, W, full, up, out_hw, words = shape
    legacy = (float(np.float32(H) / np.float32(full[0])), float(np.float32(W) / np.float32(full[1])))
    assert legacy != ref.r_yx
    bits = _wrong_resize(vals, shape, monkeypatch, r=legacy)
    with pytest.raises(NU.BoundError):
        NU.check_mask_bits(bits, ref, len(vals))


def test_check_rejects_a_cell_off_by_one_on_one_row():
    protos, cofs, boxes, vals, ref, shape = _honest()
    H, W, full, up, out_hw, words = shape
    d = vals[1]                                                          # the whole-image detection
    y0, y1, x0, x1 = d.win
    row = (y1 - y0) // 4                                                 # a row of the upper cells
    C = cofs.double().numpy()[1].reshape(4, 32)
    cell = d.cell[row] ^ 1                                               # idx_w off by one
    z = (C[cell] * protos.double().numpy()[:, y0 + row, x0:x1].T).sum(1)
    wrong = [NU.MaskVals(v.win, v.v.copy(), v.b, v.inside, v.cell, v.roi) for v in vals]
    wrong[1].v[row] = 1.0 / (1.0 + np.exp(-z))
    bad = NU.resize_reference(wrong, H, W, full, (1.0 / up, 1.0 / up), out_hw, THR, proto_bytes=128)
    bits = NU.reference_bits(bad, len(vals), out_hw[0], words)
    with pytest.raises(NU.BoundError, match='detection 1'):
        NU.check_mask_bits(bits, ref, len(vals))


def test_check_rejects_a_bit_past_out_w_and_a_plane_at_the_count():
    _, _, _, vals, ref, shape = _honest()
    H, W, full, up, out_hw, words = shape
    N = len(vals)
    assert out_hw[1] % 32 != 0
    bits = NU.reference_bits(ref, N + 1, out_hw[0], words)
    NU.check_mask_bits(bits, ref, N)
    past = bits.copy().view(np.uint32)
    past[2, 5, words - 1] |= np.uint32(1) << np.uint32(out_hw[1] % 32)
    with pytest.raises(NU.BoundError, match='outside'):
        NU.check_mask_bits(past.view(np.int32), ref, N)
    extra = bits.copy()
    extra[N, 0, 0] = 1
    with pytest.raises(NU.BoundError, match='past the count'):
        NU.check_mask_bits(extra, ref, N)
    with pytest.raises(NU.BoundError, match='past the count'):
        NU.check_mask_bits(bits, ref, N - 1)                             # plane N - 1 is a live mask, not zero


def test_check_rejects_a_wrong_value_and_a_value_outside_the_crop():
    protos, cofs, boxes, vals, _, _ = _honest()
    cbind = _oracle()
    pos = cbind.mask_assemble(protos.numpy(), cofs.numpy(), (boxes * 0.5).numpy())
    assert NU.check_mask_values(torch.from_numpy(pos), vals) <= 1.0
    assert NU.check_mask_values(torch.from_numpy(pos).half(), vals) <= 1.0
    y0, y1, x0, x1 = vals[0].win
    i, j = np.unravel_index(int(np.argmax(vals[0].b)), vals[0].b.shape)   # the loosest pixel: still caught
    bad = pos.copy()
    bad[0, y0 + i, x0 + j] += np.float32(vals[0].b[i, j] * 1.5)
    with pytest.raises(NU.BoundError, match='detection 0'):
        NU.check_mask_values(torch.from_numpy(bad), vals)
    y0, y1, x0, x1 = vals[2].win                                         # the sub-pixel roi: zeros all around it
    out = pos.copy()
    out[2, y1, x0] = 1e-30
    with pytest.raises(NU.BoundError, match='outside the crop'):
        NU.check_mask_values(torch.from_numpy(out), vals)
