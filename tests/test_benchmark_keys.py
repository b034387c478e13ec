"""convert_state_dict accepts exactly the key set of one detector: extra blocks are an error, not silently ignored."""
import pytest
import torch


def test_extra_backbone_block_is_rejected():
    from sipmask_b200 import benchmark as B
    bm = B.synthetic_state_dict(depth=101)
    bm['backbone.body.layer3.30.conv1.weight'] = torch.zeros(256, 1024, 1, 1)
    with pytest.raises(KeyError, match='layer3.30'):
        B.convert_state_dict(bm)


def test_synthetic_dict_has_bm_shapes():
    from sipmask_b200 import benchmark as B
    bm = B.synthetic_state_dict(depth=50)
    assert all(bm['rpn.head.scales.%d.scale' % i].shape == (1,) for i in range(5))      # layers/scale.py:8
    assert not any(k.endswith('num_batches_tracked') for k in bm)                        # FrozenBatchNorm2d buffers
