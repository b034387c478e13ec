"""sipmask_b200 - H100-native (sm_90a) implementation of SipMask's per-image inference hot path.

Public surface (mirrors the reference's operator / registry API, SURVEY.md §8b):
    sipmask_b200.ops        CropSplit, crop_split, nms, multiclass_nms_idx, fast_nms, mask_assemble, ...
    sipmask_b200.head       SipMaskHead, FCOSHead (drop-in nn.Modules, reference state_dict keys)
    sipmask_b200.engine     SipMaskEngine (whole image -> detections + bit-packed masks, CUDA-graph replay)
    sipmask_b200.registry   register() / register_ops() hooks for an installed mmdet
The compute lives in sipmask_b200/lib/libsipmask_b200.so (C ABI: include/sipmask_b200.h); there is no CPU path.
"""
__version__ = '0.1.0'
