"""ctypes loader for libsipmask_b200.so (the C ABI declared in include/sipmask_b200.h).

There is NO fallback: if the library is missing or the device is not sm_90 every op raises.
"""
import ctypes
import os

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, 'lib', 'libsipmask_b200.so')

F32, F16 = 0, 1


class SmbError(RuntimeError):
    pass


class Level(ctypes.Structure):
    _fields_ = [('cls', ctypes.c_void_p), ('ctr', ctypes.c_void_p), ('box', ctypes.c_void_p),
                ('cls_pitch', ctypes.c_int), ('ctr_pitch', ctypes.c_int), ('box_pitch', ctypes.c_int),
                ('h', ctypes.c_int), ('w', ctypes.c_int), ('stride', ctypes.c_int),
                ('box_scale', ctypes.c_float), ('box_mul', ctypes.c_float)]


class ConvDesc(ctypes.Structure):
    _fields_ = [(n, ctypes.c_int) for n in (
        'N', 'H', 'W', 'Cin', 'Cout', 'kh', 'kw', 'stride', 'pad', 'relu', 'has_bias', 'has_residual',
        'residual_upsample', 'res_h', 'res_w', 'out_dtype', 'gn_stats', 'in_pitch', 'out_pitch')]


class ConvLevel(ctypes.Structure):
    _fields_ = [('inp', ctypes.c_void_p), ('out', ctypes.c_void_p), ('residual', ctypes.c_void_p),
                ('gn_stats', ctypes.c_void_p), ('H', ctypes.c_int), ('W', ctypes.c_int), ('res_h', ctypes.c_int),
                ('res_w', ctypes.c_int)]


CONV_MAX_LEVELS = 5                  # SMB_CONV_MAX_LEVELS


class ConvPlanInfo(ctypes.Structure):
    """smb_conv_plan_info_t: what the planner chose for a convolution plan (include/sipmask_b200.h)."""
    _fields_ = [(n, ctypes.c_int) for n in ('num_levels', 'tiles_m', 'n_tile', 'n_tiles_n', 'stages', 'epi_tma', 'grid',
                                            'smem_bytes')] + \
        [(n, ctypes.c_int * CONV_MAX_LEVELS) for n in ('H_out', 'W_out', 'BH', 'BW', 'tiles_x', 'tiles_y')]


class ImgGeom(ctypes.Structure):
    """smb_img_geom_t: one image's post-processing geometry (include/sipmask_b200.h)."""
    _fields_ = [('img_h', ctypes.c_int), ('img_w', ctypes.c_int), ('scale', ctypes.c_float * 4),
                ('roi_scale', ctypes.c_float * 4), ('full_h', ctypes.c_int), ('full_w', ctypes.c_int),
                ('ry', ctypes.c_float), ('rx', ctypes.c_float), ('out_h', ctypes.c_int), ('out_w', ctypes.c_int),
                ('track_sx', ctypes.c_float), ('track_sy', ctypes.c_float)]


class RawSrc(ctypes.Structure):
    """smb_raw_src_t: one image of a batched preprocessing launch (include/sipmask_b200.h)."""
    _fields_ = [('src', ctypes.c_void_p), ('src_h', ctypes.c_int), ('src_w', ctypes.c_int), ('src_pitch_bytes', ctypes.c_int),
                ('dst_h', ctypes.c_int), ('dst_w', ctypes.c_int), ('mean', ctypes.c_float * 3)]


class TrackFrame(ctypes.Structure):
    """smb_track_frame_t: one frame row of a device tracker association (include/sipmask_b200.h)."""
    _fields_ = [('lane', ctypes.c_int32), ('is_first', ctypes.c_int32)]


class RenderImg(ctypes.Structure):
    """smb_render_img_t: one image of a render launch (include/sipmask_b200.h)."""
    _fields_ = [('src', ctypes.c_void_p), ('dst', ctypes.c_void_p), ('h', ctypes.c_int32), ('w', ctypes.c_int32)]


RENDER_IMAGES, RENDER_VIDEO, RENDER_MAX_NUM = 0, 1, 1024    # SMB_RENDER_IMAGES / SMB_RENDER_VIDEO / SMB_RENDER_MAX_NUM

TRACK_CAPACITY = 1                   # SMB_TRACK_CAPACITY: a lane had more tracked objects than its capacity


class RescoreWeights(ctypes.Structure):
    _fields_ = [('conv_w', ctypes.c_void_p * 6), ('conv_b', ctypes.c_void_p * 6), ('score_w', ctypes.c_void_p),
                ('score_b', ctypes.c_void_p), ('num_classes', ctypes.c_int)]


_lib = None

# every symbol include/sipmask_b200.h declares (checked by tests/test_abi.py)
SYMBOLS = [
    'smb_last_error', 'smb_version', 'smb_check_device', 'smb_mask_assemble', 'smb_mask_upsample2_threshold', 'smb_mask_upsample2_threshold_pack', 'smb_mask_resize_threshold', 'smb_mask_resize_threshold_pack', 'smb_mask_assemble_pack', 'smb_mask_set_tensor_dot',
    'smb_crop_split_forward', 'smb_crop_split_backward', 'smb_crop_split_gt', 'smb_mask_rle_counts', 'smb_rle_to_string', 'smb_conv3x3s2_relu_f32', 'smb_mask_rescore', 'smb_mask_rescore_f16_workspace_bytes', 'smb_mask_rescore_f16', 'smb_nms', 'smb_decode_workspace_bytes', 'smb_decode_topk',
    'smb_multiclass_nms_workspace_bytes', 'smb_multiclass_nms', 'smb_soft_nms', 'smb_multiclass_soft_nms_workspace_bytes',
    'smb_multiclass_soft_nms', 'smb_pair_decode_slots', 'smb_pair_decode_workspace_bytes',
    'smb_pair_decode_topk', 'smb_ml_nms_workspace_bytes', 'smb_ml_nms_topk', 'smb_fast_nms_workspace_bytes', 'smb_fast_nms',
    'smb_gather_rows_f32', 'smb_gather_det_inputs', 'smb_gather_track_feats', 'smb_track_step', 'smb_conv_plan_create', 'smb_conv_plan_create_multi', 'smb_conv_plan_destroy', 'smb_conv_plan_set_max_ctas', 'smb_conv_set_min_tiles',
    'smb_conv_run', 'smb_conv_plan_info',
    'smb_groupnorm_relu_apply', 'smb_groupnorm_stats', 'smb_deform_im2col', 'smb_offset_conv1x1', 'smb_groupnorm_relu_apply_multi', 'smb_offset_conv1x1_multi', 'smb_offset_conv1x1_relu_multi', 'smb_deform_im2col_multi', 'smb_maxpool3x3s2',
    'smb_upsample_bilinear', 'smb_stem_plan_create_s2d', 'smb_image_to_s2d16', 'smb_preprocess_u8_s2d',
    'smb_mask_assemble_dev', 'smb_mask_assemble_pack_dev', 'smb_decode_topk_dev', 'smb_pair_decode_topk_dev',
    'smb_gather_track_feats_dev', 'smb_preprocess_u8_s2d_dev', 'smb_preprocess_pil_u8_s2d_dev',
    'smb_rle_encode_workspace_bytes', 'smb_rle_encode_dev', 'smb_host_device_pointer',
    'smb_track_assoc_workspace_bytes', 'smb_track_assoc_dev',
    'smb_coco_poly_counts', 'smb_coco_poly_to_bits', 'smb_coco_rle_to_bits', 'smb_coco_rle_from_string',
    'smb_coco_plane_stats', 'smb_coco_det_from_record_dev', 'smb_coco_match_workspace_bytes', 'smb_coco_match_dev',
    'smb_coco_accumulate_dev', 'smb_coco_params_check', 'smb_coco_match_params_workspace_bytes',
    'smb_coco_match_params_dev', 'smb_coco_accumulate_params_dev', 'smb_coco_analysis_workspace_bytes',
    'smb_coco_analysis_match_dev', 'smb_coco_params2_check', 'smb_coco_match_params2_workspace_bytes',
    'smb_coco_match_params2_dev', 'smb_coco_accumulate_params2_dev',
    'smb_ytvis_overlap_dev', 'smb_ytvis_scatter_dev', 'smb_ytvis_match_workspace_bytes', 'smb_ytvis_match_dev',
    'smb_segm_raster_workspace_bytes', 'smb_segm_raster_dev', 'smb_render_dev',
    'smb_deform_grad_scale_workspace_bytes', 'smb_deform_grad_scale', 'smb_deform_col2im',
    'smb_deform_weight_grad_workspace_bytes', 'smb_deform_weight_grad', 'smb_sigmoid_focal_loss_forward',
    'smb_sigmoid_focal_loss_backward', 'smb_mask_targets', 'smb_mask_loss_workspace_bytes', 'smb_mask_loss',
]


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise SmbError('%s not found: run `python -c "import __graft_entry__ as g; g.build()"` '
                           '(there is no CPU / PyTorch fallback)' % LIB_PATH)
        L = ctypes.CDLL(LIB_PATH)
        L.smb_last_error.restype = ctypes.c_char_p
        for n in ('smb_decode_workspace_bytes', 'smb_multiclass_nms_workspace_bytes', 'smb_fast_nms_workspace_bytes',
                  'smb_multiclass_soft_nms_workspace_bytes',
                  'smb_mask_rescore_f16_workspace_bytes', 'smb_pair_decode_workspace_bytes', 'smb_ml_nms_workspace_bytes',
                  'smb_rle_encode_workspace_bytes', 'smb_track_assoc_workspace_bytes', 'smb_coco_match_workspace_bytes',
                  'smb_ytvis_match_workspace_bytes', 'smb_segm_raster_workspace_bytes',
                  'smb_coco_match_params_workspace_bytes', 'smb_coco_analysis_workspace_bytes',
                  'smb_coco_match_params2_workspace_bytes', 'smb_deform_grad_scale_workspace_bytes',
                  'smb_deform_weight_grad_workspace_bytes', 'smb_mask_loss_workspace_bytes'):
            getattr(L, n).restype = ctypes.c_size_t
        L.smb_conv_plan_destroy.restype = None
        _lib = L
    return _lib


def check(rc, what=''):
    if rc != 0:
        raise SmbError('%s failed (%d): %s' % (what, rc, lib().smb_last_error().decode()))


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)


def stream_ptr():
    """The CURRENT device's current stream.  Callers run under `device_guard` / `torch.cuda.device(tensor.device)`, so this
    is the stream of the device that owns the tensors (not of whatever device happened to be current)."""
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def _find_device(objs):
    import torch
    for o in objs:
        if isinstance(o, torch.Tensor):
            if o.is_cuda:
                return o.device
        elif isinstance(o, (list, tuple)):
            d = _find_device(o)
            if d is not None:
                return d
    return None


def device_guard(fn):
    """Run `fn` with the CUDA device of its first CUDA tensor argument made current, so that the stream passed to the C ABI,
    the per-device kernel attributes and every launch belong to the tensors' device (multi-GPU processes, head.cuda(1))."""
    import functools

    @functools.wraps(fn)
    def wrapper(*args, **kwargs):
        import torch
        dev = _find_device(args) or _find_device(tuple(kwargs.values()))
        if dev is None or dev.index is None or dev.index == torch.cuda.current_device():
            return fn(*args, **kwargs)
        with torch.cuda.device(dev):
            return fn(*args, **kwargs)
    return wrapper


def f4(vals):
    return (ctypes.c_float * 4)(*[float(v) for v in vals])
