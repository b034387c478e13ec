"""Host-side checks of the fused mask loss: the argument checks raise before anything is launched, the target rule
(at least 3 of each 2 x 2 block, pad / crop with zeros) is what the installed torch's interpolate + gt(0.5) computes on
{0, 1} masks, and the float64 reference agrees with the composition's formula on the CPU (no GPU needed)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import mask_loss_inputs as MI


@pytest.fixture
def no_launch(monkeypatch):
    from sipmask_b200 import _lib

    def fail():
        raise AssertionError('the library was called')
    monkeypatch.setattr(_lib, 'lib', fail)


def _args(B=2, M=3, H=8, W=40, G=2):
    return dict(feat_masks=torch.zeros(B, 32, H, W), cofs=torch.zeros(M, 128), boxes=torch.zeros(M, 4),
                img_offsets=torch.tensor([0, 1, M][:B + 1], dtype=torch.int32),
                targets=torch.zeros(G, H, (W + 31) // 32, dtype=torch.int32), gt_rows=torch.zeros(M, dtype=torch.int64),
                weights=torch.zeros(M))


def test_mask_loss_rejects_before_launch(no_launch):
    from sipmask_b200 import ops, _lib
    bad = [('feat_masks', torch.zeros(2, 32, 8, 40, dtype=torch.float16), 'feat_masks'),
           ('feat_masks', torch.zeros(2, 16, 8, 40), 'feat_masks'),
           ('cofs', torch.zeros(3, 96), 'cofs'),
           ('cofs', torch.zeros(3, 128, dtype=torch.float64), 'cofs'),
           ('boxes', torch.zeros(2, 4), 'boxes'),
           ('weights', torch.zeros(3, dtype=torch.float64), 'weights'),
           ('gt_rows', torch.zeros(3), 'gt_rows'),
           ('img_offsets', torch.zeros(2, dtype=torch.int32), 'img_offsets'),
           ('targets', torch.zeros(2, 8, 1, dtype=torch.int32), 'targets'),
           ('targets', torch.zeros(2, 8, 2, dtype=torch.uint8), 'targets'),
           ('cofs', torch.zeros(128, 3).t(), 'contiguous|CUDA')]
    for name, t, msg in bad:
        a = _args()
        a[name] = t
        with pytest.raises(_lib.SmbError, match=msg):
            ops.sipmask_mask_loss(**a)
    with pytest.raises(_lib.SmbError, match='CUDA'):
        ops.sipmask_mask_loss(**_args())
    with pytest.raises(_lib.SmbError, match='CUDA'):
        ops.sipmask_mask_targets([torch.zeros(2, 16, 16)], (8, 8))
    with pytest.raises(_lib.SmbError, match='bad mask size'):
        ops.sipmask_mask_targets([torch.zeros(2, 16, 16)], (0, 8))


@pytest.mark.parametrize('hf,wf,H,W', [(16, 20, 8, 10), (17, 21, 8, 10), (9, 13, 8, 10), (30, 31, 8, 10), (3, 5, 4, 4)])
def test_target_rule_matches_installed_torch(hf, wf, H, W):
    rs = np.random.RandomState(hf * 100 + wf)
    m = (rs.rand(5, hf, wf) < 0.55).astype(np.float32)
    gm = F.interpolate(torch.from_numpy(m).unsqueeze(0), scale_factor=0.5, mode='bilinear', align_corners=False)[0]
    new = gm.new_zeros(5, H, W)
    h, w = min(H, gm.shape[1]), min(W, gm.shape[2])
    new[:, :h, :w] = gm[:, :h, :w]
    want = new.gt(0.5).numpy()
    ho, wo = hf // 2, wf // 2
    cnt = m[:, 0:2 * ho:2, 0:2 * wo:2] + m[:, 1:2 * ho:2, 0:2 * wo:2] + m[:, 0:2 * ho:2, 1:2 * wo:2] + m[:, 1:2 * ho:2, 1:2 * wo:2]
    rule = np.zeros((5, H, W), dtype=bool)
    rule[:, :min(H, ho), :min(W, wo)] = (cnt >= 3)[:, :H, :W]
    assert (rule == want).all()


def test_pack_bits_layout():
    p = np.zeros((1, 2, 40), dtype=bool)
    p[0, 0, 0] = p[0, 0, 31] = p[0, 1, 33] = True
    w = MI.pack_bits(p).numpy().view(np.uint32)
    assert w.shape == (1, 2, 2)
    assert w[0, 0, 0] == (1 | (1 << 31)) and w[0, 0, 1] == 0 and w[0, 1, 0] == 0 and w[0, 1, 1] == 2


def test_reference64_matches_composition_formula_on_cpu():
    """The float64 reference (used by the GPU tests) against a dense restatement of the reference block on the CPU in
    float64: CropSplit's cell selection by the same geometry, BCE with the -100 clamp, the per-instance normalisation."""
    inp = MI.clustered_inputs(2, 20, 36, 7, seed=1)
    loss, dX, dC = MI.reference64(inp)
    feat = inp['feat'].double().requires_grad_(True)
    cofs = inp['cofs'].double().requires_grad_(True)
    offs = inp['offsets'].tolist()
    tot = []
    for b in range(2):
        n0, n1 = offs[b], offs[b + 1]
        X = feat[b].permute(1, 2, 0)
        P = torch.sigmoid(torch.stack([X @ cofs[n0:n1, 32 * q:32 * q + 32].t() for q in range(4)]))   # [4, H, W, M]
        cl = MI.cells(inp['boxes'][n0:n1], 20, 36).permute(1, 2, 0)                               # [H, W, M]
        pred = torch.gather(P, 0, cl.clamp(min=0).unsqueeze(0)).squeeze(0) * (cl >= 0)
        gt = inp['planes'].double().index_select(0, inp['rows'][n0:n1]).permute(1, 2, 0) * (cl >= 0)
        pre = F.binary_cross_entropy(pred, gt, reduction='none').sum(dim=(0, 1))
        bx = inp['boxes'][n0:n1].double()
        pre = pre / (bx[:, 2] - bx[:, 0]) / (bx[:, 3] - bx[:, 1]) / (n1 - n0)
        tot.append((pre * inp['weights'][n0:n1].double()).sum())
    tot = torch.stack(tot)
    tot.sum().backward()
    assert torch.allclose(loss, tot.detach(), rtol=1e-12)
    assert torch.allclose(dX, feat.grad, rtol=1e-9, atol=1e-15) and torch.allclose(dC, cofs.grad, rtol=1e-9, atol=1e-15)
