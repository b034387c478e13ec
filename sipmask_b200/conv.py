"""Host side of the wgmma convolution engine: weight packing (BN folding, K-major fp16) and plan objects.

Reference modules replaced: nn.Conv2d (+ eval BatchNorm2d, bias, residual add, ReLU) in
MM/mmdet/models/backbones/resnet.py:203-239, MM/mmdet/models/necks/fpn.py:138-178,
MM/mmdet/ops/conv_module.py:124-132, MM/mmdet/models/anchor_heads/sipmask_head.py:241-287.
Activations are NHWC fp16 torch tensors; all compute happens in libsipmask_b200.so.
"""
import ctypes

import torch

from . import _lib as L


def pack_weight(w, bn=None, eps=1e-5, cout_pad=None, device=None):
    """[Cout,Cin,kh,kw] fp32 (+ eval BN (gamma,beta,mean,var)) -> ([Cout_pad, kh*kw*Cin] fp16 K-major, bias fp32|None).

    K index = (r*kw + s)*Cin + ci, matching the tap order of the TMA producer.  Frozen BN
    (resnet.py:514-521) folds to w *= gamma/sqrt(var+eps), bias = beta - mean*gamma/sqrt(var+eps)."""
    w = w.detach().float()
    cout, cin, kh, kw = w.shape
    bias = None
    if bn is not None:
        gamma, beta, mean, var = [t.detach().float() for t in bn]
        s = gamma / torch.sqrt(var + eps)
        w = w * s.view(-1, 1, 1, 1)
        bias = beta - mean * s
    wk = w.permute(0, 2, 3, 1).reshape(cout, kh * kw * cin)
    cp = cout_pad or ((cout + 15) // 16 * 16)
    if cp != cout:
        wk = torch.cat([wk, wk.new_zeros(cp - cout, wk.shape[1])], 0)
        if bias is not None:
            bias = torch.cat([bias, bias.new_zeros(cp - cout)])
    wk = wk.to(torch.float16).contiguous()
    if device is not None:
        wk = wk.to(device)
        bias = bias.to(device) if bias is not None else None
    return wk, bias


def pack_stem_weight_s2d(w, bn, eps=1e-5, device=None):
    """7x7 stem [64,3,7,7] -> [64, 4*64] for the space-to-depth stem: K = a*64 + b*16 + (dy*2+dx)*4 + c holds filter tap
    (r, s) = (2a+dy, 2b+dx), channel c (taps with r == 7 or s == 7 and c == 3 are zero)."""
    gamma, beta, mean, var = [t.detach().float() for t in bn]
    s = gamma / torch.sqrt(var + eps)
    w = w.detach().float() * s.view(-1, 1, 1, 1)
    w8 = w.new_zeros(64, 4, 8, 8)                        # [co, c(3->4), r(7->8), s(7->8)]
    w8[:, :3, :7, :7] = w
    # [co, c, a, dy, b, dx] -> [co, a, b, dy, dx, c]
    wk = w8.view(64, 4, 4, 2, 4, 2).permute(0, 2, 4, 3, 5, 1).reshape(64, 256).to(torch.float16).contiguous()
    bias = (beta - mean * s).contiguous()
    if device is not None:
        wk, bias = wk.to(device), bias.to(device)
    return wk, bias


def set_min_tiles(n):
    """Planner knob for plans created afterwards (smb_conv_set_min_tiles); returns the previous value."""
    return int(L.lib().smb_conv_set_min_tiles(int(n)))


class ConvPlan(object):
    """One convolution bound to fixed input / weight / output buffers (TMA descriptors are baked at creation)."""

    def __init__(self, x, weight, out, k, stride=1, relu=False, bias=None, residual=None, residual_upsample=False,
                 gn_stats=None, cin=None, alpha=1.0):
        assert x.is_cuda and x.dtype == torch.float16 and x.dim() == 4 and x.stride(3) == 1
        N, H, W, _ = x.shape
        cin = cin if cin is not None else x.shape[3]
        in_pitch = x.stride(2)
        assert x.stride(1) == W * in_pitch and x.stride(0) == H * W * in_pitch
        cout = weight.shape[0]
        assert weight.shape[1] == k * k * cin and weight.dtype == torch.float16 and weight.is_contiguous()
        assert out.stride(3) == 1
        out_pitch = out.stride(2)
        d = L.ConvDesc()
        d.N, d.H, d.W, d.Cin, d.Cout = N, H, W, cin, cout
        d.kh = d.kw = k
        d.stride = stride
        d.pad = k // 2
        d.relu = int(relu)
        d.has_bias = int(bias is not None)
        d.has_residual = int(residual is not None)
        d.residual_upsample = int(residual_upsample)
        if residual is not None:
            d.res_h, d.res_w = residual.shape[1], residual.shape[2]
            assert residual.dtype == torch.float16 and residual.is_contiguous() and residual.shape[3] == cout
        d.out_dtype = L.F32 if out.dtype == torch.float32 else L.F16
        d.gn_stats = int(gn_stats is not None)
        d.in_pitch = in_pitch
        d.out_pitch = out_pitch
        self._keep = (x, weight, out, bias, residual, gn_stats)
        self.desc = d                                  # what the kernel is told (read by the layer audit)
        self.bias, self.residual, self.gn_stats, self.alpha = bias, residual, gn_stats, float(alpha)
        self.handle = ctypes.c_void_p()
        self.dev = x.device
        with torch.cuda.device(self.dev):
            L.check(L.lib().smb_conv_plan_create(ctypes.byref(d), L.ptr(x), L.ptr(weight), L.ptr(out),
                                                 ctypes.byref(self.handle)), 'smb_conv_plan_create')
        self.out = out

    def set_max_ctas(self, n):
        L.check(L.lib().smb_conv_plan_set_max_ctas(self.handle, int(n)), 'smb_conv_plan_set_max_ctas')
        return self

    def info(self):
        """What the planner chose (smb_conv_plan_info): dict with num_levels, tiles_m, n_tile, n_tiles_n, stages, epi_tma
        (as decided at creation), grid, smem_bytes, and per level a list of dicts H_out, W_out, BH, BW, tiles_x, tiles_y."""
        i = L.ConvPlanInfo()
        L.check(L.lib().smb_conv_plan_info(self.handle, ctypes.byref(i)), 'smb_conv_plan_info')
        keys = ('H_out', 'W_out', 'BH', 'BW', 'tiles_x', 'tiles_y')
        res = {n: int(getattr(i, n)) for n in ('num_levels', 'tiles_m', 'n_tile', 'n_tiles_n', 'stages', 'epi_tma', 'grid',
                                               'smem_bytes')}
        res['levels'] = [{k: int(getattr(i, k)[l]) for k in keys} for l in range(i.num_levels)]
        return res

    def run(self, stream=None):
        if self.dev.index != torch.cuda.current_device():        # launch on the plan's device and ITS current stream
            with torch.cuda.device(self.dev):
                return self.run(stream)
        L.check(L.lib().smb_conv_run(self.handle, L.ptr(self.bias), L.ptr(self.residual), L.ptr(self.gn_stats),
                                     ctypes.c_float(self.alpha), stream if stream is not None else L.stream_ptr()),
                'smb_conv_run')
        return self.out

    def __del__(self):
        try:
            if self.handle:
                L.lib().smb_conv_plan_destroy(self.handle)
                self.handle = None
        except Exception:
            pass


class ConvPlanMulti(ConvPlan):
    """One stride-1 convolution with shared weights over several feature-pyramid levels = ONE launch
    (the reference loops over levels in python, sipmask_head.py:250-271)."""

    def __init__(self, xs, weight, outs, k, relu=False, bias=None, gn_stats=None, alpha=1.0):
        nl = len(xs)
        N = xs[0].shape[0]
        cin = xs[0].shape[3]
        in_pitch = xs[0].stride(2)
        out_pitch = outs[0].stride(2)
        cout = weight.shape[0]
        assert weight.shape[1] == k * k * cin and weight.dtype == torch.float16 and weight.is_contiguous()
        lv = (L.ConvLevel * nl)()
        for i, (x, o) in enumerate(zip(xs, outs)):
            assert x.is_cuda and x.dtype == torch.float16 and x.stride(3) == 1 and x.stride(2) == in_pitch
            assert x.shape[0] == N and x.stride(1) == x.shape[2] * in_pitch and x.stride(0) == x.shape[1] * x.shape[2] * in_pitch
            assert o.stride(3) == 1 and o.stride(2) == out_pitch and o.dtype == outs[0].dtype
            st = gn_stats[i] if gn_stats is not None else None
            lv[i] = L.ConvLevel(x.data_ptr(), o.data_ptr(), 0, st.data_ptr() if st is not None else 0, x.shape[1], x.shape[2], 0, 0)
        d = L.ConvDesc()
        d.N, d.H, d.W, d.Cin, d.Cout = N, 0, 0, cin, cout
        d.kh = d.kw = k
        d.stride = 1
        d.pad = k // 2
        d.relu = int(relu)
        d.has_bias = int(bias is not None)
        d.has_residual = 0
        d.out_dtype = L.F32 if outs[0].dtype == torch.float32 else L.F16
        d.gn_stats = int(gn_stats is not None)
        d.in_pitch = in_pitch
        d.out_pitch = out_pitch
        self._keep = (xs, weight, outs, bias, gn_stats, lv)
        self.desc, self.levels = d, lv                 # descriptor and level table the kernel is told (read by the layer audit)
        self.bias, self.residual, self.gn_stats, self.alpha = bias, None, None, float(alpha)
        self.handle = ctypes.c_void_p()
        self.dev = xs[0].device
        with torch.cuda.device(self.dev):
            L.check(L.lib().smb_conv_plan_create_multi(ctypes.byref(d), nl, lv, L.ptr(weight), ctypes.byref(self.handle)),
                    'smb_conv_plan_create_multi')
        self.out = outs


class StemPlan(ConvPlan):
    """7x7/2 stem + folded BN + ReLU (resnet.py:448-460) on the space-to-depth image [N,H/2+3,W/2+4,16]
    (image_to_s2d16 / preprocess_u8) with weights [64,256] (pack_stem_weight_s2d)."""

    def __init__(self, img8, weight, bias, out, N, H, W):
        self._keep = (img8, weight, bias, out)
        self.bias, self.residual, self.gn_stats, self.alpha = bias, None, None, 1.0
        self.handle = ctypes.c_void_p()
        self.dev = img8.device
        assert tuple(img8.shape) == (N, H // 2 + 3, W // 2 + 4, 16) and img8.is_contiguous()
        assert tuple(weight.shape) == (64, 256)
        with torch.cuda.device(self.dev):
            L.check(L.lib().smb_stem_plan_create_s2d(N, H, W, L.ptr(img8), L.ptr(weight), L.ptr(out),
                                                     ctypes.byref(self.handle)), 'smb_stem_plan_create_s2d')
        self.out = out


# ------------------------------------------------------------------------------------- small wrappers
@L.device_guard
def image_to_s2d16(img, out=None):
    """img [N,3,H,W] fp32 -> the stem's space-to-depth input [N, H/2+3, W/2+4, 16] fp16 (smb_image_to_s2d16)."""
    N, _, H, W = img.shape
    if out is None:
        out = torch.empty((N, H // 2 + 3, W // 2 + 4, 16), dtype=torch.float16, device=img.device)
    L.check(L.lib().smb_image_to_s2d16(L.ptr(img.contiguous()), L.ptr(out), N, H, W, L.stream_ptr()), 'smb_image_to_s2d16')
    return out


@L.device_guard
def preprocess_u8(src, resized_hw, out, mean):
    """uint8 BGR HWC CUDA image -> resized (cv2 INTER_LINEAR, bit-exact) - mean -> zero-padded fp16 stem input in the
    space-to-depth layout `out` [1, H/2+3, W/2+4, 16] (smb_preprocess_u8_s2d)."""
    assert src.is_cuda and src.dtype == torch.uint8 and src.dim() == 3 and src.shape[2] == 3 and src.stride(2) == 1 \
        and src.stride(1) == 3
    assert out.dtype == torch.float16 and out.is_contiguous() and out.shape[0] == 1 and out.shape[3] == 16
    m = (ctypes.c_float * 3)(*[float(v) for v in mean])
    H, W = 2 * (out.shape[1] - 3), 2 * (out.shape[2] - 4)
    L.check(L.lib().smb_preprocess_u8_s2d(L.ptr(src), int(src.shape[0]), int(src.shape[1]), int(src.stride(0)),
                                          int(resized_hw[0]), int(resized_hw[1]), m, L.ptr(out), H, W, L.stream_ptr()),
            'smb_preprocess_u8_s2d')
    return out


@L.device_guard
def preprocess_u8_rows(rows, out):
    """preprocess_u8 for a batch in one launch: canvas n of `out` [N, H/2+3, W/2+4, 16] from the smb_raw_src_t row n of
    `rows` (a device tensor of N rows, read when the kernel runs; smb_preprocess_u8_s2d_dev).  The rows are not checked on
    the device: write only rows that SipMaskEngine.forward_raw / raw_src_row validated."""
    assert out.dtype == torch.float16 and out.is_contiguous() and out.dim() == 4 and out.shape[3] == 16
    assert rows.is_cuda and rows.dtype == torch.uint8 and rows.numel() == out.shape[0] * ctypes.sizeof(L.RawSrc)
    H, W = 2 * (out.shape[1] - 3), 2 * (out.shape[2] - 4)
    L.check(L.lib().smb_preprocess_u8_s2d_dev(L.ptr(rows), int(out.shape[0]), L.ptr(out), H, W, L.stream_ptr()),
            'smb_preprocess_u8_s2d_dev')
    return out


@L.device_guard
def preprocess_pil_rows(rows, out):
    """SipMask-benchmark's test transform for a batch in one launch: canvas n of `out` [N, H/2+3, W/2+4, 16] from the
    smb_raw_src_t row n of `rows` (a device tensor of N rows; src is an RGB image, mean in BGR order), PIL bilinear resize
    bit-exact, BGR, mean-subtracted, zero-padded (smb_preprocess_pil_u8_s2d_dev).  The rows are not checked on the
    device: write only rows that raw_src_row validated with max_downscale=PIL_MAX_DOWNSCALE."""
    assert out.dtype == torch.float16 and out.is_contiguous() and out.dim() == 4 and out.shape[3] == 16
    assert rows.is_cuda and rows.dtype == torch.uint8 and rows.numel() == out.shape[0] * ctypes.sizeof(L.RawSrc)
    H, W = 2 * (out.shape[1] - 3), 2 * (out.shape[2] - 4)
    L.check(L.lib().smb_preprocess_pil_u8_s2d_dev(L.ptr(rows), int(out.shape[0]), L.ptr(out), H, W, L.stream_ptr()),
            'smb_preprocess_pil_u8_s2d_dev')
    return out


# the steepest downscale per axis smb_preprocess_pil_u8_s2d_dev supports (its filter has at most 17 taps)
PIL_MAX_DOWNSCALE = 8


def raw_src_row(src, resized_hw, canvas_hw, mean, device, order='BGR', max_downscale=None):
    """The smb_raw_src_t row of one uint8 HWC image (channel `order`: BGR for the cv2 pipeline, RGB for the PIL one) on
    `device` resized to resized_hw inside a canvas_hw canvas, or a filler row (all-zero canvas, nothing read) for
    src=None.  max_downscale: the steepest shrink per axis the kernel supports (None: no limit).  Raises ValueError for
    anything the kernel could not read safely."""
    r = L.RawSrc()
    r.mean[:] = [float(v) for v in mean]
    if src is None:
        return r
    if not isinstance(src, torch.Tensor) or src.dtype != torch.uint8 or src.dim() != 3 or src.shape[2] != 3:
        raise ValueError('raw input is a uint8 HWC %s image' % order)
    h, w = int(src.shape[0]), int(src.shape[1])
    if src.stride(2) != 1 or src.stride(1) != 3 or not 3 * w <= src.stride(0) < 2 ** 31:
        raise ValueError('raw input must have HWC strides (row pitch, 3, 1), got %s' % (tuple(src.stride()),))
    if src.device != device:
        raise ValueError('raw input is on %s, the engine on %s' % (src.device, device))
    dh, dw = int(resized_hw[0]), int(resized_hw[1])
    if h <= 0 or w <= 0 or not (0 < dh <= canvas_hw[0] and 0 < dw <= canvas_hw[1]):
        raise ValueError('image %dx%d resized to %dx%d does not fit the %dx%d canvas' % (h, w, dh, dw, canvas_hw[0],
                                                                                        canvas_hw[1]))
    if max_downscale is not None and (h > max_downscale * dh or w > max_downscale * dw):
        raise ValueError('image %dx%d resized to %dx%d shrinks more than %gx on an axis' % (h, w, dh, dw, max_downscale))
    r.src, r.src_h, r.src_w, r.src_pitch_bytes, r.dst_h, r.dst_w = src.data_ptr(), h, w, int(src.stride(0)), dh, dw
    return r


@L.device_guard
def maxpool3x3s2(x, out=None):
    N, H, W, C = x.shape
    Ho, Wo = (H - 1) // 2 + 1, (W - 1) // 2 + 1
    if out is None:
        out = torch.empty((N, Ho, Wo, C), dtype=torch.float16, device=x.device)
    L.check(L.lib().smb_maxpool3x3s2(L.ptr(x), L.ptr(out), N, H, W, C, L.stream_ptr()), 'smb_maxpool3x3s2')
    return out


@L.device_guard
def groupnorm_stats(x, stats=None):
    N, H, W, C = x.shape
    if stats is None:
        stats = torch.empty((N, 32, 2), dtype=torch.int64, device=x.device)
    L.check(L.lib().smb_groupnorm_stats(L.ptr(x), N, H * W, C, x.stride(2), L.ptr(stats), L.stream_ptr()),
            'smb_groupnorm_stats')
    return stats


@L.device_guard
def groupnorm_relu_apply(x, stats, gamma, beta, eps=1e-5, relu=True):
    N, H, W, C = x.shape
    L.check(L.lib().smb_groupnorm_relu_apply(L.ptr(x), N, H * W, C, x.stride(2), L.ptr(stats), L.ptr(gamma), L.ptr(beta),
                                             ctypes.c_float(eps), int(relu), L.stream_ptr()), 'smb_groupnorm_relu_apply')
    return x


@L.device_guard
def offset_conv1x1(bbox, scale, weight, out=None):
    """bbox [N,H,W,>=4] fp32 channel-last (pitch = stride(2)); weight [n_off,4] fp32 -> [N,H,W,n_off] fp32."""
    N, H, W, _ = bbox.shape
    n_off = weight.shape[0]
    if out is None:
        out = torch.empty((N, H, W, n_off), dtype=torch.float32, device=bbox.device)
    L.check(L.lib().smb_offset_conv1x1(L.ptr(bbox), bbox.stride(2), ctypes.c_float(scale), L.ptr(weight), n_off, L.ptr(out),
                                       ctypes.c_longlong(N * H * W), L.stream_ptr()), 'smb_offset_conv1x1')
    return out


def _pixel_pitch(t):
    """Elements between neighbouring pixels of an [N, H, W, C] view whose pixels are evenly spaced (a channel slice of a
    wider tensor included).  The stride of a size-1 dimension is arbitrary (a permuted 1 x 1 map counts as contiguous
    with stride(2) == 1), so the pitch comes from the innermost dimension longer than 1."""
    N, H, W, C = t.shape
    p = t.stride(2) if W > 1 else t.stride(1) if H > 1 else t.stride(0) if N > 1 else C
    assert (C == 1 or t.stride(3) == 1) and (H == 1 or t.stride(1) == W * p) and (N == 1 or t.stride(0) == H * W * p)
    return p


@L.device_guard
def deform_im2col(x, offset, dg, out=None):
    """x [N,H,W,C] fp16, offset [N,H,W,dg*18] fp32 -> col [N,H,W,9*C] fp16."""
    N, H, W, C = x.shape
    assert x.is_contiguous()
    if out is None:
        out = torch.empty((N, H, W, 9 * C), dtype=torch.float16, device=x.device)
    L.check(L.lib().smb_deform_im2col(L.ptr(x), L.ptr(offset), _pixel_pitch(offset), L.ptr(out), N, H, W, C, int(dg),
                                      L.stream_ptr()), 'smb_deform_im2col')
    return out


@L.device_guard
def deform_grad_scale(grad_out):
    """grad_out [N,C,H,W] fp32 contiguous -> (s * grad_out as [N,H,W,C] fp16, device {s, 1/s} fp32) with s a power of two
    chosen on the device from amax |grad_out| (smb_deform_grad_scale)."""
    N, C, H, W = grad_out.shape
    out = torch.empty((N, H, W, C), dtype=torch.float16, device=grad_out.device)
    scale = torch.empty(2, dtype=torch.float32, device=grad_out.device)
    ws = torch.empty(int(L.lib().smb_deform_grad_scale_workspace_bytes()), dtype=torch.uint8, device=grad_out.device)
    L.check(L.lib().smb_deform_grad_scale(L.ptr(grad_out), N, C, H, W, L.ptr(out), L.ptr(scale), L.ptr(ws),
                                          ctypes.c_size_t(ws.numel()), L.stream_ptr()), 'smb_deform_grad_scale')
    return out, scale


@L.device_guard
def deform_col2im(grad_col, x, offset, dg, scale, grad_input=True, grad_offset=True):
    """grad_col [N,H,W,9C] fp32 (s * the column gradient), x [N,H,W,C] fp16, offset [N,H,W,dg*18] fp32, scale {s, 1/s}
    -> (grad_input [N,H,W,C] fp32 | None, grad_offset [N,H,W,dg*18] fp32 | None) (smb_deform_col2im)."""
    N, H, W, C = x.shape
    assert x.is_contiguous() and grad_col.is_contiguous()
    gin = torch.zeros((N, H, W, C), dtype=torch.float32, device=x.device) if grad_input else None
    goff = torch.empty((N, H, W, dg * 18), dtype=torch.float32, device=x.device) if grad_offset else None
    L.check(L.lib().smb_deform_col2im(L.ptr(grad_col), L.ptr(x), L.ptr(offset), _pixel_pitch(offset), L.ptr(scale), L.ptr(gin),
                                      L.ptr(goff), N, H, W, C, int(dg), L.stream_ptr()), 'smb_deform_col2im')
    return gin, goff


@L.device_guard
def deform_weight_grad(grad_f16, col, scale):
    """grad_f16 [N,H,W,Cout] fp16, col [N,H,W,K] fp16 -> dW [Cout, K] fp32 = sum over pixels / s (smb_deform_weight_grad)."""
    cout, k = grad_f16.shape[-1], col.shape[-1]
    P = grad_f16.numel() // cout
    assert grad_f16.is_contiguous() and col.is_contiguous() and col.numel() == P * k
    dw = torch.empty((cout, k), dtype=torch.float32, device=col.device)
    ws = torch.empty(max(int(L.lib().smb_deform_weight_grad_workspace_bytes(cout, k, ctypes.c_longlong(P))), 16),
                     dtype=torch.uint8, device=col.device)
    L.check(L.lib().smb_deform_weight_grad(L.ptr(grad_f16), L.ptr(col), ctypes.c_longlong(P), cout, k, L.ptr(scale),
                                           L.ptr(dw), L.ptr(ws), ctypes.c_size_t(ws.numel()), L.stream_ptr()),
            'smb_deform_weight_grad')
    return dw


@L.device_guard
def upsample_bilinear(x, factor, out=None, out_choff=0, relu=False):
    N, H, W, C = x.shape
    if out is None:
        out = torch.empty((N, H * factor, W * factor, C), dtype=torch.float16, device=x.device)
    assert out.shape[0] == N and out.stride(3) == 1 and out.stride(1) == out.shape[2] * out.stride(2)
    L.check(L.lib().smb_upsample_bilinear(L.ptr(x), x.stride(2), L.ptr(out), out.stride(2), int(out_choff), N, H, W,
                                          out.shape[1], out.shape[2], C, int(factor), int(relu), L.stream_ptr()),
            'smb_upsample_bilinear')
    return out


# ------------------------------------------------------------------------------------- multi-level wrappers
def _parr(ts):
    return (ctypes.c_void_p * len(ts))(*[t.data_ptr() for t in ts])


def _iarr(vals):
    return (ctypes.c_int * len(vals))(*[int(v) for v in vals])


@L.device_guard
def groupnorm_relu_apply_multi(xs, stats, gamma, beta, eps=1e-5, relu=True):
    N, _, _, C = xs[0].shape
    L.check(L.lib().smb_groupnorm_relu_apply_multi(len(xs), _parr(xs), _parr(stats), _iarr([x.shape[1] for x in xs]),
                                                   _iarr([x.shape[2] for x in xs]), N, C, xs[0].stride(2), L.ptr(gamma),
                                                   L.ptr(beta), ctypes.c_float(eps), int(relu), L.stream_ptr()),
            'smb_groupnorm_relu_apply_multi')
    return xs


@L.device_guard
def offset_conv1x1_multi(bboxes, scales, weight, offs, relu=False):
    """relu=True: offsets from relu(scale * bbox) (smb_offset_conv1x1_relu_multi)."""
    N = bboxes[0].shape[0]
    sc = (ctypes.c_float * len(scales))(*[float(v) for v in scales])
    fn = L.lib().smb_offset_conv1x1_relu_multi if relu else L.lib().smb_offset_conv1x1_multi
    L.check(fn(len(bboxes), _parr(bboxes), bboxes[0].stride(2), sc, L.ptr(weight), weight.shape[0], _parr(offs),
               _iarr([b.shape[1] for b in bboxes]), _iarr([b.shape[2] for b in bboxes]), N, L.stream_ptr()),
            'smb_offset_conv1x1_multi')
    return offs


@L.device_guard
def deform_im2col_multi(xs, offs, dg, cols):
    N, _, _, C = xs[0].shape
    L.check(L.lib().smb_deform_im2col_multi(len(xs), _parr(xs), _parr(offs), offs[0].stride(2), _parr(cols),
                                            _iarr([x.shape[1] for x in xs]), _iarr([x.shape[2] for x in xs]), N, C, int(dg),
                                            L.stream_ptr()), 'smb_deform_im2col_multi')
    return cols
