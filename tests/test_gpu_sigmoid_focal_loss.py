"""ops.sigmoid_focal_loss / SigmoidFocalLoss against the reference's own kernels: SigmoidFocalLossForward / Backward
(MM/mmdet/ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-100) were run on the seeded inputs of
tests/train_ops_inputs.py by tests/golden/gen_golden_ref_train_ops.py; the loss and the gradient must be the same bits."""
import ctypes
import os

import numpy as np
import pytest
import torch

import train_ops_inputs as T

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'ref_train_ops.npz')


@pytest.fixture(scope='module')
def gold():
    return np.load(GOLDEN)


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize('C,gamma,alpha', T.FOCAL_CASES)
def test_forward_backward_bit_equal_to_reference_kernel(gold, C, gamma, alpha):
    from sipmask_b200 import ops
    logits, targets, d_loss = [t.cuda() for t in T.focal_inputs(C)]
    x = logits.clone().requires_grad_(True)
    loss = ops.sigmoid_focal_loss(x, targets, gamma, alpha)
    loss.backward(d_loss)
    key = T.focal_key(C, gamma, alpha)
    np.testing.assert_array_equal(_bits(loss.detach().cpu().numpy()), _bits(gold[key + '_loss']))
    np.testing.assert_array_equal(_bits(x.grad.cpu().numpy()), _bits(gold[key + '_grad']))
    # every target kind occurs: ignored (-1), background (0) and each class
    assert set(targets.tolist()) >= set(range(-1, C + 1))


FOCAL_GRID = 4096 * 512                    # threads of the largest focal-loss grid; beyond that the kernels stride


@pytest.mark.parametrize('C,gamma,alpha', [(80, 2.0, 0.25), (80, 1.5, 0.5), (1, 2.0, 0.25), (1, 0.0, 0.5)])
def test_past_one_grid(gold, C, gamma, alpha):
    """The fixture's rows tiled to more than two grids' worth of elements (two 1333 x 800 images at 80 classes give about
    3.6 M), with a partial last stride.  Every element depends only on its logit, target and class, so the loss and the
    gradient must be the fixture's bits tiled the same way."""
    from sipmask_b200 import ops
    logits, targets, d_loss = T.focal_inputs(C)
    N = logits.shape[0]
    reps = 2 * FOCAL_GRID // (N * C) + 1
    n = reps * N * C
    assert n > 2 * FOCAL_GRID and n % FOCAL_GRID != 0
    print('focal loss C %d: %d rows x %d = %d elements, %d grid strides, last one %d elements' % (
        C, N, reps, n, -(-n // FOCAL_GRID), n % FOCAL_GRID))
    x = logits.repeat(reps, 1).cuda().requires_grad_(True)
    loss = ops.sigmoid_focal_loss(x, targets.repeat(reps).cuda(), gamma, alpha)
    loss.backward(d_loss.repeat(reps, 1).cuda())
    key = T.focal_key(C, gamma, alpha)
    np.testing.assert_array_equal(_bits(loss.detach().cpu().numpy()), np.tile(_bits(gold[key + '_loss']), (reps, 1)))
    np.testing.assert_array_equal(_bits(x.grad.cpu().numpy()), np.tile(_bits(gold[key + '_grad']), (reps, 1)))


def test_module_returns_the_sum():
    from sipmask_b200 import ops
    logits, targets, _ = [t.cuda() for t in T.focal_inputs(40)]
    m = ops.SigmoidFocalLoss(2.0, 0.25)
    assert repr(m) == 'SigmoidFocalLoss(gamma=2.0, alpha=0.25)'
    assert torch.equal(m(logits, targets), ops.sigmoid_focal_loss(logits, targets, 2.0, 0.25).sum())


def test_empty_batch_launches_nothing(monkeypatch):
    from sipmask_b200 import ops, _lib
    lib = _lib.lib()
    # the entry points themselves accept N = 0 without pointers and return before any launch
    assert lib.smb_sigmoid_focal_loss_forward(None, None, 0, 80, ctypes.c_float(2), ctypes.c_float(0.25), None, None) == 0
    assert lib.smb_sigmoid_focal_loss_backward(None, None, None, 0, 80, ctypes.c_float(2), ctypes.c_float(0.25), None,
                                                None) == 0
    called = []
    monkeypatch.setattr(_lib, 'lib', lambda: called.append(1) or lib)
    x = torch.zeros((0, 80), device='cuda', requires_grad=True)
    loss = ops.sigmoid_focal_loss(x, torch.zeros(0, dtype=torch.int64, device='cuda'))
    loss.sum().backward()
    assert loss.shape == (0, 80) and x.grad.shape == (0, 80)
    assert not called


def test_other_dtypes_raise():
    from sipmask_b200 import ops, _lib
    t = torch.ones(4, dtype=torch.int64, device='cuda')
    for dt in (torch.float16, torch.float64):
        with pytest.raises(_lib.SmbError):
            ops.sigmoid_focal_loss(torch.zeros(4, 80, dtype=dt, device='cuda'), t)
    with pytest.raises(_lib.SmbError):
        ops.sigmoid_focal_loss(torch.zeros(4, 80, device='cuda'), t.int())
