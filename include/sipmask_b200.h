/*
 * sipmask_b200 - C ABI of the H100-native (sm_90a) SipMask inference hot path.
 *
 * Drop-in boundary (SURVEY.md §8b).  Every entry point replaces one native
 * (pybind) entry point or one python/ATen call sequence of the reference
 * (JialeCao001/SipMask @ bc63fa9, paths relative to SipMask-mmdetection/mmdet/).
 *
 * Conventions
 *   - extern "C", plain pointers + sizes, no torch types.
 *   - all pointers are DEVICE pointers unless named host_*; the caller owns every
 *     buffer including workspaces (query with *_workspace_bytes); the library never
 *     allocates or frees device memory and never synchronises the device.
 *   - every launch goes to the caller's `stream` (the reference's CropSplit launches on
 *     the legacy default stream, ops/crop/src/crop_split_cuda_kernel.cu:77 - fixed here).
 *   - return 0 on success, a negative SMB_E* code otherwise; smb_last_error() gives a
 *     thread-local message.  (The reference only printf()s CUDA launch errors,
 *     crop_split_cuda_kernel.cu:81-85.)
 *   - dtype codes: SMB_F32 = 0, SMB_F16 = 1.
 */
#ifndef SIPMASK_B200_H_
#define SIPMASK_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct CUstream_st* smb_stream_t; /* == cudaStream_t */

#define SMB_OK 0
#define SMB_EINVAL (-1)   /* bad argument / unsupported shape */
#define SMB_ECUDA (-2)    /* CUDA runtime / driver error      */
#define SMB_EWORKSPACE (-3) /* workspace too small            */
#define SMB_EARCH (-4)    /* device is not sm_90              */

#define SMB_F32 0
#define SMB_F16 1

const char* smb_last_error(void);
int smb_version(void);
/* 0 if the current device can run the sm_90a kernels, SMB_EARCH otherwise. */
int smb_check_device(void);

/* ------------------------------------------------------------------ per-image post-processing geometry
 * Everything the post-processing reads per image, one row per image.  The *_dev entry points below read it from a DEVICE
 * pointer when the kernel runs, so a captured CUDA graph can serve images of different sizes through the same network
 * shape: the host rewrites the rows between replays.  The host-argument entry points build the same row from their
 * arguments and pass it by value to the same kernels.
 *   img_h, img_w       : the resized image (decode clamps boxes to [0, img_w-1] x [0, img_h-1])
 *   scale[4]           : decode divides the clamped boxes by these (scale_factor per coordinate; 1 = no rescale)
 *   roi_scale[4]       : rois = boxes * roi_scale (scale_factor / 2 for MM, 0.5 for BM)
 *   full_h, full_w     : the mask's interpolated size; ry, rx: source step per output pixel (> 0)
 *   out_h, out_w       : the ori_shape canvas the masks are pasted into
 *   track_sx, track_sy : SipMask-VIS: the track-feature lookup multiplies the boxes by these */
typedef struct {
  int img_h, img_w;
  float scale[4];
  float roi_scale[4];
  int full_h, full_w;
  float ry, rx;
  int out_h, out_w;
  float track_sx, track_sy;
} smb_img_geom_t;

/* ------------------------------------------------------------------ mask assembly
 * Replaces sipmask_head.py:615-627: 4x (protos @ cof_k^T) -> sigmoid -> stack ->
 * CropSplit(ops/crop/src/crop_split_cuda_kernel.cu:19-59) -> permute, as ONE kernel
 * that evaluates only the selected sub-region's dot product for in-box pixels.
 *   protos : [32,H,W] (layout_hwc=0, the reference's `feat_mask`) or [H,W,32] (layout_hwc=1)
 *   cofs   : [N,128] fp32, per detection (00|01|10|11 blocks of 32, sipmask_head.py:616-619)
 *   boxes  : [N,4] fp32 image-space boxes; rois = boxes * box_scale (sipmask_head.py:623,
 *            box_scale = scale_factor / 2), per-coordinate box_scale[4]
 *   out    : [N,H,W] (fp32 or fp16) = the reference's pos_masks.permute(2,0,1)
 */
int smb_mask_assemble(const void* protos, int protos_dtype, int layout_hwc,
                      const float* cofs, const float* boxes, const float* host_box_scale4,
                      void* out, int out_dtype, int H, int W, int N, smb_stream_t stream);
/* The same with the roi scale read from the device row `geom` (roi_scale only). */
int smb_mask_assemble_dev(const void* protos, int protos_dtype, int layout_hwc, const float* cofs, const float* boxes,
                          const smb_img_geom_t* geom, void* out, int out_dtype, int H, int W, int N, smb_stream_t stream);

/* Bilinear resize (align_corners=False) + `> thr` of pos_masks (sipmask_head.py:630-633), pasted top-left into
 * [N,out_h,out_w] and truncated (sipmask_head.py:648-654).  The reference interpolates by 2/scale_factor (per axis
 * scale_factor[3:1:-1] on the SSD path): the caller passes the interpolated size (full_h, full_w) =
 * (floor(H * 2/sf_h), floor(W * 2/sf_w)) and the source step per output pixel (ry, rx): src = (dst + 0.5) * r - 0.5 with
 * r = 1 / (2/sf) (what F.interpolate(scale_factor=...) does in PyTorch >= 1.6), or r <= 0 for in/out
 * (recompute_scale_factor=True, the behaviour of PyTorch <= 1.5, the version range the reference README pins).
 *   pos : [N,H,W] fp32/fp16      out_u8 : [N,out_h,out_w] uint8 {0,1}; pixels beyond (full_h, full_w) are 0. */
int smb_mask_resize_threshold(const void* pos, int pos_dtype, uint8_t* out_u8, int N, int H, int W, int full_h,
                              int full_w, float ry, float rx, int out_h, int out_w, float thr, smb_stream_t stream);
/* Bit-packed variant: out_bits [N,out_h,ceil(out_w/32)] uint32, pixel x = bit (x & 31) of word (x >> 5). */
int smb_mask_resize_threshold_pack(const void* pos, int pos_dtype, uint32_t* out_bits, int N, int H, int W,
                                   int full_h, int full_w, float ry, float rx, int out_h, int out_w, float thr,
                                   smb_stream_t stream);
/* scale_factor == 1 shorthands: full size = (2H, 2W). */
int smb_mask_upsample2_threshold(const void* pos, int pos_dtype, uint8_t* out_u8, int N, int H, int W,
                                 int out_h, int out_w, float thr, smb_stream_t stream);
int smb_mask_upsample2_threshold_pack(const void* pos, int pos_dtype, uint32_t* out_bits, int N, int H, int W,
                                      int out_h, int out_w, float thr, smb_stream_t stream);

/* SipMask++ mask rescoring (sipmask_head.py:200-219,635-643; SURVEY.md 8a-10).
 * smb_conv3x3s2_relu_f32: one ConvModule of `convs_scoring`: NCHW fp32 conv3x3, stride 2, padding 0, + bias, ReLU;
 *   in [N,Cin,H,W] -> out [N,Cout,(H-3)/2+1,(W-3)/2+1], weight [Cout,Cin,3,3].
 * smb_mask_rescore: relu(mask_scoring 1x1) -> global max-pool -> the detection's own class -> times det[:,4]:
 *   feat [N,C,h,w], weight1x1 [num_classes,C], labels int64 [N], det [N,5], n_valid device int (or NULL) -> scores [N]. */
int smb_conv3x3s2_relu_f32(const float* in, const float* weight, const float* bias, float* out, int N, int Cin, int H,
                           int W, int Cout, smb_stream_t stream);
int smb_mask_rescore(const float* feat, int N, int C, int h, int w, const float* weight1x1, const float* bias1x1,
                     int num_classes, const int64_t* labels, const float* det, const int* n_valid, float* scores,
                     smb_stream_t stream);

/* The same rescoring on tensor cores, for a batch of images (the engine's path): fp16 masks, weights and activations,
 * fp32 accumulation (mma.sync.m16n8k16), layers 1+2 fused so that layer 1 never reaches memory.
 *   pos_masks : [n_img*max_rows, H, W] fp16 cropped stride-2 masks, row r = img*max_rows + j
 *   count     : device int [n_img]; rows j >= clamp(count[img], 0, max_rows) do no work and score exactly 0
 *   labels    : int64 [n_img*max_rows] (0-based; a label outside [0, num_classes) scores 0), det [n_img*max_rows, 5]
 *   scores    : fp32 [n_img*max_rows] = det[:,4] * max_p relu(mask_scoring(conv6(...(conv1(mask)))))[label]
 *   weights   : HOST struct of device pointers.  conv_w[i]: fp16 [Cout_i, 9*Cin_i] with K = (r*3 + s)*Cin_i + ci (the
 *               convolution engine's packing, conv.pack_weight), (Cin, Cout) = (1,16) (16,16) (16,16) (16,32) (32,64)
 *               (64,128); conv_b[i]: fp32 [Cout_i]; score_w: fp16 [>= num_classes, 128] (mask_scoring 1x1, row = class);
 *               score_b: fp32 [num_classes].
 * H, W >= 127 (127 -> 63 -> 31 -> 15 -> 7 -> 3 -> 1).  SMB_EINVAL without a launch for null pointers, smaller masks or a
 * workspace smaller than smb_mask_rescore_f16_workspace_bytes(n_img*max_rows, H, W) (which is 0 for invalid shapes). */
typedef struct {
  const void* conv_w[6];
  const float* conv_b[6];
  const void* score_w;
  const float* score_b;
  int num_classes;
} smb_rescore_weights_t;
size_t smb_mask_rescore_f16_workspace_bytes(int R, int H, int W);
int smb_mask_rescore_f16(const void* pos_masks, int n_img, int max_rows, int H, int W, const int* count,
                         const smb_rescore_weights_t* host_weights, const int64_t* labels, const float* det, float* scores,
                         void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* COCO RLE of bit-packed masks on the device (replaces the per-detection `masks[i].cpu().numpy()` + pycocotools
 * `mask_util.encode(order='F')` tail, sipmask_head.py:645-657; SURVEY.md 8f-1).
 *   mask_bits : [N, mask_h, words] uint32 (pixel x = bit x&31 of word x>>5), cropped to the top-left H x W (= ori_shape),
 *               any width
 *   n_valid   : device int (number of valid detections, may be NULL = N)
 *   counts    : [N, cap] uint32 run lengths in COLUMN-major order, starting with the zeros run
 *   n_counts  : [N] int32: number of runs, 0 for det >= *n_valid, or -(boundaries+1) if cap was too small */
int smb_mask_rle_counts(const uint32_t* mask_bits, int N, int mask_h, int words, int H, int W, const int* n_valid,
                        uint32_t* counts, int cap, int* n_counts, smb_stream_t stream);
/* HOST helper (plain C, no CUDA): pycocotools' rleToString of `n` run lengths; returns the length written, -1 if cap is
 * too small.  counts is a host pointer. */
int smb_rle_to_string(const uint32_t* host_counts, int n, char* host_out, int cap);

/* The pycocotools strings of a whole batch of engine records, encoded on the device (two launches, graph-capturable):
 *   mask_bits : [N, max_num, cap_h, words] uint32 (the engine's record), count: device int [N] (clamped to [0, max_num]),
 *   geom      : device rows [N]; image n's canvas is (out_h, out_w) of its row (clamped to cap_h x 32*words)
 *   dst       : DEVICE word holding the address (as the device sees it, see smb_host_device_pointer) of an arena of
 *               N * img_bytes bytes, read when the kernel runs (0: nothing is written).  Image n's region starts at
 *               n * img_bytes: int32 header {status, n, off[max_num + 1]} (4 * (max_num + 3) bytes), then the strings of
 *               its n detections back to back, string i = bytes [off[i], off[i+1]) after the header.
 *   status    : 0, or SMB_RLE_RUNS_OVERFLOW (a mask has more than run_cap runs) | SMB_RLE_BYTES_OVERFLOW (the strings exceed
 *               img_bytes - header).  With a non-zero status the strings are not written; nothing is ever written outside
 *               the image's region.
 * Every pointer is read when the kernels run, so the rows, counts and destination may change between graph replays.
 * max_num <= 1024, img_bytes a multiple of 16, workspace >= smb_rle_encode_workspace_bytes(N, max_num, run_cap). */
#define SMB_RLE_RUNS_OVERFLOW 1
#define SMB_RLE_BYTES_OVERFLOW 2
size_t smb_rle_encode_workspace_bytes(int N, int max_num, int run_cap);
int smb_rle_encode_dev(const uint32_t* mask_bits, int N, int max_num, int cap_h, int words, const int* count,
                       const smb_img_geom_t* geom, int run_cap, const uint64_t* dst, int img_bytes, void* workspace,
                       size_t workspace_bytes, smb_stream_t stream);
/* The device address of page-locked host memory (cudaHostGetDevicePointer), for the dst word above. */
int smb_host_device_pointer(void* host_ptr, void** dev_ptr_out);

/* Fully fused mask path (sipmask_head.py:609-633,648-654): prototypes -> selected sub-region dot product -> sigmoid ->
 * crop -> bilinear resize to (full_h, full_w) -> `> thr` -> bit-pack into [N,out_h,ceil(out_w/32)] (a memset node zero-fills
 * the planes, one kernel writes the words that intersect a box).  pos_masks is never written to memory.
 * Same arguments as smb_mask_assemble; resize / output as smb_mask_resize_threshold_pack.  Shrinking by more than 4x
 * (scale_factor > 8) returns SMB_EINVAL. */
int smb_mask_assemble_pack(const void* protos, int protos_dtype, int layout_hwc, const float* cofs, const float* boxes,
                           const float* host_box_scale4, uint32_t* out_bits, int H, int W, int N, int full_h, int full_w,
                           float ry, float rx, int out_h, int out_w, float thr, smb_stream_t stream);
/* The same with roi scale, resize and canvas read from the device row `geom` when the kernel runs.  out_bits is
 * [N, cap_h, ceil(cap_w/32)]: it is zero-filled, then bits are written inside [min(out_h, full_h), min(out_w, full_w)] only;
 * geom->out_h <= cap_h and geom->out_w <= cap_w are the caller's to guarantee.  The tile is sized for (max_ry, max_rx),
 * the steepest source step the row may hold (geom->ry <= max_ry, geom->rx <= max_rx, both > 0); a row beyond them writes
 * nothing.  The bits do not depend on the tile. */
int smb_mask_assemble_pack_dev(const void* protos, int protos_dtype, int layout_hwc, const float* cofs, const float* boxes,
                               const smb_img_geom_t* geom, float max_ry, float max_rx, uint32_t* out_bits, int H, int W, int N,
                               int cap_h, int cap_w, float thr, smb_stream_t stream);

/* fp16 prototypes run the tensor-core variants of smb_mask_assemble / smb_mask_assemble_pack (mma.sync dot products with
 * the fp32 coefficients split into fp16 hi + lo; same crop geometry, mask values within ~1e-6 of the scalar kernels).
 * on = 1 / 0 selects them / the scalar-fmaf kernels for later calls, on < 0 only queries; returns the previous setting
 * (initial value: 1).  fp32 prototypes always run the scalar kernels. */
int smb_mask_set_tensor_dot(int on);

/* ------------------------------------------------------------------ CropSplit (operator API)
 * Replaces crop_split_cuda.crop_split_cuda_forward(data, rois, out, H, W, c, n)
 * (ops/crop/src/crop_split_cuda.cpp:14-36).  data [c*c,H,W,N], rois [N,4], out [H,W,N]; c == 2.
 */
int smb_crop_split_forward(const void* data, const void* rois, void* out, int dtype,
                           int H, int W, int c, int N, smb_stream_t stream);

/* Training-side companions (SURVEY 8f-4).  smb_crop_split_backward replaces crop_split_cuda_backward
 * (ops/crop/src/crop_split_cuda_kernel.cu:90-163): top_grad [H,W,N] -> bottom_grad [c*c,H,W,N], every element written
 * (the reference zero-initialises and atomically adds).  smb_crop_split_gt replaces crop_split_gt_cuda_forward AND
 * _backward (ops/crop/src/crop_split_gt_cuda_kernel.cu:19-49,76-104): out[h,w,n] = data[h,w,n] inside roi n, else 0. */
int smb_crop_split_backward(const void* top_grad, const void* rois, void* bottom_grad, int dtype, int H, int W, int c, int N,
                            smb_stream_t stream);
int smb_crop_split_gt(const void* data, const void* rois, void* out, int dtype, int H, int W, int N, smb_stream_t stream);

/* ------------------------------------------------------------------ NMS (operator API)
 * Replaces nms_cuda.nms(dets, thr) (ops/nms/src/nms_kernel.cu:71-138) without the D2H bitmask copy
 * and host sweep.  dets [n,5] fp32; keep_out [n] int64 receives ORIGINAL indices ascending;
 * n_keep_out device int32.  cmp_ge: 0 = suppress IoU > thr (CUDA ref), 1 = IoU >= thr (CPU ref).
 * n <= 8192.
 */
int smb_nms(const float* dets, int n, float iou_thr, int cmp_ge, int plus_one,
            int64_t* keep_out, int* n_keep_out, smb_stream_t stream);

/* ------------------------------------------------------------------ decode + per-level top-k
 * Replaces sipmask_head.py:556-592 (sigmoid, max_c(score*ctr) top-k per level, distance2bbox
 * core/bbox/transforms.py:202-223, concat, /scale_factor, no bg column).
 * Level l has hw[l] locations on a w[l]-wide grid with stride[l]; its tensors are channel-last:
 *   cls[l] : [hw,C] fp32 logits with row pitch cls_pitch (elements);  ctr[l] : [hw] pitch ctr_pitch
 *   box[l] : [hw,4] fp32 distances (already x stride) with row pitch box_pitch
 * Outputs (n_total = sum_l min(hw[l], nms_pre) when nms_pre > 0):
 *   cand_boxes [n_total,4], cand_scores [n_total,C] (sigmoid), cand_ctr [n_total] (sigmoid),
 *   cand_loc [n_total] int32 = level-concatenated location index (for gathering coefficients).
 */
typedef struct {
  const float* cls; const float* ctr; const float* box;
  int cls_pitch, ctr_pitch, box_pitch;
  int h, w, stride;
  float box_scale, box_mul; /* distance = (box * box_scale) * box_mul : (1,1) for the reference's bbox_preds,
                               (Scale_l, stride_l) when `box` is the raw fcos_reg output (sipmask_head.py:261,268) */
} smb_level_t;

size_t smb_decode_workspace_bytes(int num_levels, const smb_level_t* host_levels, int nms_pre);
int smb_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre,
                    int img_h, int img_w, const float* host_scale4 /* scale_factor per coordinate (boxes are divided by it), or NULL */,
                    float* cand_boxes, float* cand_scores, float* cand_ctr, int* cand_loc,
                    void* workspace, size_t workspace_bytes, smb_stream_t stream);
/* The same with img_h / img_w / scale read from the device row `geom`. */
int smb_decode_topk_dev(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre,
                        const smb_img_geom_t* geom, float* cand_boxes, float* cand_scores, float* cand_ctr, int* cand_loc,
                        void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ multi-class NMS
 * Replaces core/post_processing/bbox_nms.py:79-146 (python loop over classes, one nms_cuda +
 * D2H + host sweep per class) with two launches and no host sync.
 *   boxes [n,4], scores [n,C] (raw sigmoid, no bg column), ctr [n] (score factor)
 *   det_out [max_num,5] (x1,y1,x2,y2,score*ctr), label_out [max_num] int64 (0-based),
 *   idx_out [max_num] int64 (row of boxes), count_out device int32.
 * Order: class-major / ascending row when total <= max_num, else descending score
 * (ties: class-major order) - bbox_nms.py:135-140.   n <= 4096, max_num <= 1024.
 */
size_t smb_multiclass_nms_workspace_bytes(int n, int num_classes);
int smb_multiclass_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                       float score_thr, float iou_thr, int max_num, int cmp_ge,
                       float* det_out, int64_t* label_out, int64_t* idx_out, int* count_out,
                       void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ soft-NMS
 * ops/nms/src/nms_cpu.cpp:70-209 (soft_nms_cpu_kernel) bit for bit in float32, one list per CTA held in shared memory.
 * method: SMB_SOFT_NMS_LINEAR (weight 1 - IoU above iou_thr) or SMB_SOFT_NMS_GAUSSIAN (weight expf(-IoU^2 / sigma), the
 * C library's expf of an FMA host); a decayed score below min_score removes the element.
 *   smb_soft_nms: dets [n,5] -> dets_out [n,5] (the kept rows in selection order, decayed scores), inds_out [n] int64
 *   (positions in dets), count_out device int32 = the number kept.
 *   smb_multiclass_soft_nms: smb_multiclass_nms with soft-NMS per class (bbox_nms.py:79-146 with nms.type = soft_nms):
 *   class lists in ascending row order, kept rows in selection order, decayed score*ctr in det_out; the top max_num by
 *   decayed score when more are kept (ties: class-major order).
 * n <= 5120 candidates (SMB_EINVAL without a launch above it or for another method), max_num <= 1024.  Graph-capturable:
 * stream-ordered, no allocation, no synchronisation. */
#define SMB_SOFT_NMS_LINEAR 1
#define SMB_SOFT_NMS_GAUSSIAN 2
int smb_soft_nms(const float* dets, int n, float iou_thr, int method, float sigma, float min_score, float* dets_out,
                 int64_t* inds_out, int* count_out, smb_stream_t stream);
size_t smb_multiclass_soft_nms_workspace_bytes(int n, int num_classes);
int smb_multiclass_soft_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                            float score_thr, float iou_thr, int max_num, int method, float sigma, float min_score,
                            float* det_out, int64_t* label_out, int64_t* idx_out, int* count_out,
                            void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ fast NMS (SSD / VIS path)
 * Replaces SipMaskHead.fast_nms (sipmask_head.py:868-910): per-class descending sort, top_k,
 * IoU without +1 (:912-959), triu, column max, `iou_max <= thr && score > score_thr`, global
 * descending sort, first max_num.   scores [n,C] sigmoid, ctr [n]; n <= 4096, top_k <= 256.
 */
size_t smb_fast_nms_workspace_bytes(int n, int num_classes, int top_k);
int smb_fast_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                 float score_thr, float iou_thr, int top_k, int max_num,
                 float* det_out, int64_t* label_out, int64_t* idx_out, int* count_out,
                 void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ SipMask-benchmark post-processing
 * (SipMask-benchmark/fcos_core/modeling/rpn/sipmask/inference.py:90-190, csrc/cuda/ml_nms.cu).
 * smb_pair_decode_topk: candidates are (location, class) pairs with sigmoid(cls) > score_thr.  Per level, when more than
 *   nms_pre pass, the nms_pre with the largest sigmoid(cls) * sigmoid(ctr) are kept (ties -> lower pair index loc*C + c).
 *   Output order: level by level, ascending pair index inside a level.  Sigmoids are 1 / (1 + exp(-x)) with exp in
 *   double rounded to float and IEEE float add / divide.  box = location -/+ relu(box * box_scale) * box_mul, clipped to
 *   [0, img_w-1] x [0, img_h-1]; score = sqrt(sigmoid(cls) * sigmoid(ctr)); label = class (0-based); loc =
 *   level-concatenated location.  *n_cand (device) = number of candidates; slots past it hold zeros and label / loc -1.
 *   n_slots >= smb_pair_decode_slots(...) = sum_l min(h_l * w_l * C, nms_pre).  The workspace holds one key per pair.
 *   1 <= nms_pre <= 5120, C <= 1024, h*w*C < 2^31 per level.
 * smb_ml_nms_topk: label-aware NMS over n = min(*n_dev, cap) candidates (cap <= 5120): descending score, ties by ascending
 *   index, suppress when IoU (+1 areas) > iou_thr within a label.  Survivors in ascending candidate order; when more than
 *   max_per_img (> 0) survive, keep scores >= the max_per_img-th largest (ties can keep more).  The first out_cap kept rows
 *   go to det_out [out_cap,5] (box, score), label_out / idx_out int64 [out_cap] (candidate row); *count_out =
 *   min(kept, out_cap), *kept_total_out = kept.  Rows past the count: zeros, label / idx -1. */
int smb_pair_decode_slots(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre);
size_t smb_pair_decode_workspace_bytes(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre);
int smb_pair_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, float score_thr, int nms_pre,
                         int img_h, int img_w, float* cand_boxes, float* cand_scores, int* cand_labels, int* cand_loc,
                         int* n_cand, int n_slots, void* workspace, size_t workspace_bytes, smb_stream_t stream);
/* The same with img_h / img_w read from the device row `geom`. */
int smb_pair_decode_topk_dev(int num_levels, const smb_level_t* host_levels, int num_classes, float score_thr, int nms_pre,
                             const smb_img_geom_t* geom, float* cand_boxes, float* cand_scores, int* cand_labels,
                             int* cand_loc, int* n_cand, int n_slots, void* workspace, size_t workspace_bytes,
                             smb_stream_t stream);
size_t smb_ml_nms_workspace_bytes(int cap);
int smb_ml_nms_topk(const float* boxes, const float* scores, const int* labels, const int* n_dev, int cap, float iou_thr,
                    int max_per_img, int out_cap, float* det_out, int64_t* label_out, int64_t* idx_out, int* count_out,
                    int* kept_total_out, void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* The gather between NMS and mask assembly (mlvl_cofs[idxs_keep], det_bboxes[:, :4]; sipmask_head.py:612,623) in one launch:
 * det_cofs[i,:] = cof_src[cand_loc[idx[i]],:] (row pitch cof_pitch floats), det_boxes[i,:] = det[i,:4] for i < *count,
 * zeros after; loc_out (may be NULL) receives the level-concatenated location of each kept detection (-1 after count).
 * cof_src is either one image's level-concatenated [tot, pitch] buffer (num_levels = 0) or a batched level-major buffer
 * [level][n_img][hw_l][pitch] with host_level_hw[l] = h_l * w_l, of which image `img` is gathered. */
int smb_gather_det_inputs(const float* cof_src, int cof_pitch, const int* cand_loc, const int64_t* idx, const float* det,
                          const int* count_dev, int max_rows, int row_elems, float* det_cofs, float* det_boxes,
                          int64_t* loc_out, int num_levels, const int* host_level_hw, int n_img, int img, smb_stream_t stream);

/* SipMask-VIS `extract_box_feature_center_single` (SipMask-VIS/mmdet/models/anchor_heads/sipmask_head.py:609-613,768-781):
 * out[i,:] = track[floor((y1+y2)*sy/2/stride), floor((x1+x2)*sx/2/stride), :] for i < *count, zeros after.
 * track [h,w,C] fp32 channel-last (the `sipmask_track` output), det [max_rows,5], (sx, sy) = scale_factor when the
 * detections were rescaled (res_det_bboxes = det * scale_factor), feat_stride = 8. */
int smb_gather_track_feats(const float* track, int h, int w, int C, const float* det, const int* count_dev, int max_rows,
                           float scale_x, float scale_y, float feat_stride, float* out, smb_stream_t stream);
/* The same with (scale_x, scale_y) = (geom->track_sx, geom->track_sy) read from the device row. */
int smb_gather_track_feats_dev(const float* track, int h, int w, int C, const float* det, const int* count_dev, int max_rows,
                               const smb_img_geom_t* geom, float feat_stride, float* out, smb_stream_t stream);

/* HOST helper (plain C++, no CUDA): one frame of the SipMask-VIS tracker association (SipMask-VIS/mmdet/models/anchor_heads/
 * sipmask_head.py:544-562,612-667) on host arrays.  State = the tracked objects' boxes [capacity,5], labels [capacity],
 * features [capacity,feat_dim], of which the first n_prev are valid; updated in place.  host_ids_out [n] receives the object
 * ids (-1: lost the claim).  Returns the new number of tracked objects, or a negative SMB_E* code. */
int smb_track_step(const float* host_det, const int64_t* host_labels, const float* host_feats, int n, int feat_dim,
                   float* host_prev_det, int64_t* host_prev_labels, float* host_prev_feats, int n_prev, int capacity,
                   const float* host_match_coeff3, int32_t* host_ids_out);

/* The same association on the DEVICE for every frame of a batch, one launch (graph-capturable).  Each video runs on a lane
 * whose tracker state is caller-owned device memory:
 *   state_boxes [lanes, capacity, 5] f32, state_labels [lanes, capacity] i64, state_feats [lanes, capacity, 512] f32,
 *   n_obj [lanes] i32 (the number of tracked objects; -1: no state yet), status [lanes] i32 (bits are OR-ed in).
 * Frame r of the batch is frames[r] (device rows); its record is det [N, max_num, 5], labels [N, max_num],
 * count [N] (clamped to [0, max_num]), track_feats [N, max_num, 512]; ids [N, max_num] receives its object ids.
 * The rows of one lane are associated in batch order, each exactly as smb_track_step associates a frame:
 *   - count 0: ids -1, state unchanged (even with is_first: the reference returns before the tracker);
 *   - is_first, or n_obj < 0: the state becomes the frame's detections, ids 0..n-1;
 *   - otherwise the comp matrix against the n_obj tracked objects, first maximum per row, appends and best claims.
 * An object appended beyond capacity is not stored: its detection gets id -1 and status[lane] |= SMB_TRACK_CAPACITY.
 * Rows whose lane is outside [0, lanes) (lane < 0: a filler) touch no state and get ids -1.  ids past a row's count are -1.
 * Every pointer is read when the kernel runs; n_obj is clamped to [-1, capacity].  Feature arrays 16-byte aligned,
 * max_num <= 1024, workspace >= smb_track_assoc_workspace_bytes(lanes, max_num, capacity). */
#define SMB_TRACK_FEAT_DIM 512
#define SMB_TRACK_CAPACITY 1
typedef struct {
  int32_t lane;      /* the video's lane, < 0: filler row */
  int32_t is_first;  /* non-zero: the video's first frame (the reference's img_meta['is_first']) */
} smb_track_frame_t;
size_t smb_track_assoc_workspace_bytes(int lanes, int max_num, int capacity);
int smb_track_assoc_dev(const smb_track_frame_t* frames, int N, const float* det, const int64_t* labels, const int* count,
                        const float* track_feats, int max_num, float* state_boxes, int64_t* state_labels, float* state_feats,
                        int* n_obj, int* status, int lanes, int capacity, const float* host_match_coeff3, int32_t* ids,
                        void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ COCO box / mask AP (pycocotools 2.0 COCOeval)
 * bbox and segm evaluation with the default parameters: 10 IoU thresholds, 101 recall thresholds, 4 area ranges,
 * maxDets 1 / 10 / 100.  Masks are bit planes in the image's h x w canvas (pixel x = bit x&31 of word x>>5).
 *
 * Detection row, as the result json carries it: xywh box, score[0] = bbox score, score[1] = segm score, area_box = w * h
 * (loadRes), the plane's word offset in the detection planes, its pixel count (maskUtils.area), the category index
 * (-1: none) and ext = {row0, row1, word0, word1} (half-open) of its set bits. */
typedef struct {
  double box[4];
  double score[2];
  double area_box;
  int64_t plane;
  int32_t area_mask;
  int32_t cat;
  int32_t ext[4];
  int32_t order;   /* the detection's position in the result json (ties of equal scores keep this order) */
  int32_t pad;
} smb_coco_det_t;
/* Ground-truth row: bbox, the annotation's own area, plane offset, annotation id, iscrowd, pixel count, extents. */
typedef struct {
  double box[4];
  double area;
  int64_t plane;
  int64_t id;
  int32_t crowd;
  int32_t area_mask;
  int32_t ext[4];
} smb_coco_gt_t;
/* One image of a match launch: canvas, row pitches (words) of its detection and ground-truth planes, number of detection
 * rows (the record path writes it), image id, and its first output row. */
typedef struct {
  int32_t h, w;
  int32_t det_pitch, gt_pitch;
  int32_t n_det, pad;
  int64_t image_id;
  int64_t out_off;
} smb_coco_img_t;
/* Per detection and metric: score, image, matched / ignored bits (bit t*4 + a), category index (K: not evaluated) and its
 * rank by score inside its (image, category) (-1: not evaluated). */
typedef struct {
  double score;
  int64_t image_id;
  uint64_t matched;
  uint64_t ignored;
  int32_t cat;
  int32_t rank;
} smb_coco_out_t;
#define SMB_COCO_T 10
#define SMB_COCO_R 101
#define SMB_COCO_A 4
#define SMB_COCO_MAX_DET 100
#define SMB_COCO_DET_CAP 4096
#define SMB_COCO_MAX_CATS 2048
#define SMB_COCO_LABEL_RANGE 1   /* status: a record label outside [0, num_labels) */
#define SMB_COCO_CAPACITY 2      /* status: an output row outside [0, n_out) */
#define SMB_COCO_ANALYSIS_RANGE 4 /* status: an annotation position or a supercategory index outside its table */

/* HOST helpers (plain C++, no CUDA), pycocotools maskApi.c restated:
 *   smb_coco_poly_counts     : rleFrPoly's run lengths of one polygon of k vertices (*host_n = their number; written
 *                              when it is <= cap)
 *   smb_coco_poly_to_bits    : the same polygon OR-ed into a bit plane (merge of several polygons = union)
 *   smb_coco_rle_to_bits     : column-major run lengths (zeros first) OR-ed into a bit plane; SMB_EINVAL unless they
 *                              cover h * w pixels exactly
 *   smb_coco_rle_from_string : rleFrString of a compressed counts string (*host_n = the number of counts, at most len;
 *                              written when it is <= cap; SMB_EINVAL on a malformed string)
 *   smb_coco_plane_stats     : {pixel count, row0, row1, word0, word1} of an h x w plane */
int smb_coco_poly_counts(const double* host_xy, int k, int h, int w, uint32_t* host_counts, int cap, int* host_n);
int smb_coco_poly_to_bits(const double* host_xy, int k, int h, int w, uint32_t* host_plane, int pitch);
int smb_coco_rle_to_bits(const uint32_t* host_counts, int n, int h, int w, uint32_t* host_plane, int pitch);
int smb_coco_rle_from_string(const char* host_s, int len, uint32_t* host_counts, int cap, int* host_n);
int smb_coco_plane_stats(const uint32_t* host_plane, int h, int w, int pitch, int32_t* host_stats5);

/* Detection rows [N, max_num] of a batch of engine records, identical to what coco.coco_json writes: MM boxes
 * (x2 - x1) + 1 in float64, BM boxes resized by the float32 ratio out / img of the geometry row with TO_REMOVE = 1 in
 * float32; segm score = mask_scores (MM only, may be NULL); category = label_cat[label] (a label outside [0, num_labels)
 * gives -1 and sets SMB_COCO_LABEL_RANGE in *status).  The planes are mask_bits' [cap_h, words] planes cropped to the
 * geometry row's (out_h, out_w).  imgs[n].n_det = clamp(count[n], 0, max_num). */
int smb_coco_det_from_record_dev(const float* det, const int64_t* labels, const int* count, const float* mask_scores,
                                 const uint32_t* mask_bits, int N, int max_num, int cap_h, int words,
                                 const smb_img_geom_t* geom, const int32_t* label_cat, int num_labels, int benchmark,
                                 smb_coco_det_t* rows, smb_coco_img_t* imgs, int* status, smb_stream_t stream);
/* computeIoU + evaluateImg (maxDet 100) of every (image, category) with a ground truth or a detection, one CTA per image:
 *   dets [n_img, det_cap] (image b's rows b*det_cap + [0, n_det)), gts: rows of image b's category k are
 *   [gt_cat_off[b*(K+1)+k], gt_cat_off[b*(K+1)+k+1]) in annotation order; metric 0 = bbox, 1 = segm.
 *   host_iou_thr[10], host_area_rng[4][2] (float64, as COCOeval's Params hold them).
 *   out: row imgs[b].out_off + j for detection j of image b (every row [0, n_det) of the image is written);
 *   npig [K, 4]: non-ignored ground truths are added (int atomics).
 * det_cap <= SMB_COCO_DET_CAP, K <= SMB_COCO_MAX_CATS, workspace >= smb_coco_match_workspace_bytes(n_gt). */
size_t smb_coco_match_workspace_bytes(int n_gt);
int smb_coco_match_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                       const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt,
                       const uint32_t* gt_planes, int64_t gt_plane_words, const int32_t* gt_cat_off, int K, int metric,
                       const double* host_iou_thr, const double* host_area_rng, smb_coco_out_t* out, int64_t n_out,
                       int* npig, int* status, void* workspace, size_t workspace_bytes, smb_stream_t stream);
/* accumulate: rows sorted by (category, score descending, image id, rank), category k's rows [cat_off[k], cat_off[k+1]);
 * rec_thr[101] device float64; precision / scores [10, 101, K, 4, 3], recall [10, K, 4, 3] float64 (pycocotools layout),
 * -1 where a (category, area range) has no non-ignored ground truth. */
int smb_coco_accumulate_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K, const int* npig,
                            const double* rec_thr, const int* host_max_dets3, double* precision, double* recall,
                            double* scores, smb_stream_t stream);

/* COCOeval with user-given Params (p.iouThrs, p.recThrs, p.areaRng as float64 data, in any order; p.maxDets ascending, as
 * COCOeval.evaluate() sorts them).
 * Limits: 1 <= T, 1 <= A, T * A <= SMB_COCO_MAX_TA (the matched / ignored bits of a row are one uint64 each);
 * 1 <= M <= SMB_COCO_MAX_M with every maxDet in [1, SMB_COCO_MAX_DET], in ascending order; 1 <= R <= SMB_COCO_R; no NaN.  A launch with
 * Params outside them returns SMB_EINVAL.  The default Params make these entry points compute what the two above do.
 * useCats = 0 and maxDets above SMB_COCO_MAX_DET go through smb_coco_params2_t below. */
#define SMB_COCO_MAX_TA 64
#define SMB_COCO_MAX_M 3
typedef struct {
  int32_t T, A, M, R;
  int32_t max_dets[SMB_COCO_MAX_M];
  int32_t pad;
  double iou_thr[SMB_COCO_MAX_TA];
  double area_rng[SMB_COCO_MAX_TA][2];
  double rec_thr[SMB_COCO_R];
} smb_coco_params_t;
/* SMB_OK when *host_params is within the limits, else SMB_EINVAL with the limit in smb_last_error(). */
int smb_coco_params_check(const smb_coco_params_t* host_params);
/* smb_coco_match_dev with Params: matched / ignored bit t*A + a, the first maxDets[M-1] detections of each (image,
 * category) ranked, npig [K, A]; workspace >= smb_coco_match_params_workspace_bytes(n_gt, host_params). */
size_t smb_coco_match_params_workspace_bytes(int n_gt, const smb_coco_params_t* host_params);
int smb_coco_match_params_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                              const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt,
                              const uint32_t* gt_planes, int64_t gt_plane_words, const int32_t* gt_cat_off, int K,
                              int metric, const smb_coco_params_t* host_params, smb_coco_out_t* out, int64_t n_out,
                              int* npig, int* status, void* workspace, size_t workspace_bytes, smb_stream_t stream);
/* smb_coco_accumulate_dev with Params: npig [K, A]; precision / scores [T, R, K, A, M], recall [T, K, A, M].  As in
 * pycocotools, the recall thresholds after the first one the detections do not reach keep precision and score 0. */
int smb_coco_accumulate_params_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K,
                                   const int* npig, const smb_coco_params_t* host_params, double* precision,
                                   double* recall, double* scores, smb_stream_t stream);

/* COCOeval Params with p.useCats and maxDets up to SMB_COCO_MAX_DET2 (the *_params2_* entry points).  The fields are
 * smb_coco_params_t's, with use_cats in place of its padding:
 *   use_cats 1: one group per (image, category), as the entry points above;
 *   use_cats 0: one pooled group per image (computeIoU / evaluateImg over the concatenation of the image's rows of every
 *               category), rows written with category index 0 and npig [1, A], so accumulate runs with K = 1.
 * The K categories of a launch are p.catIds: the host packs an image's ground truth category-major (category index,
 * then annotation order) and gives a detection the index of its category (-1: not evaluated).  In a pooled group,
 * detections rank by score descending, then category index, then json order, which is np.argsort(-score,
 * kind='mergesort') over pycocotools' concatenation; ground truths keep the packed order.
 * Limits: those of smb_coco_params_t, except every maxDet in [1, SMB_COCO_MAX_DET2]; use_cats 0 or 1.  The shared memory
 * of a match launch grows with det_cap and maxDets[M-1] (about 122 KB at 4096 rows and 1000). */
#define SMB_COCO_MAX_DET2 1000
typedef struct {
  int32_t T, A, M, R;
  int32_t max_dets[SMB_COCO_MAX_M];
  int32_t use_cats;
  double iou_thr[SMB_COCO_MAX_TA];
  double area_rng[SMB_COCO_MAX_TA][2];
  double rec_thr[SMB_COCO_R];
} smb_coco_params2_t;
int smb_coco_params2_check(const smb_coco_params2_t* host_params);
/* workspace >= smb_coco_match_params2_workspace_bytes(n_gt, host_params): [n_gt, maxDets[M-1]] IoUs, [n_gt, T*A] bytes. */
size_t smb_coco_match_params2_workspace_bytes(int n_gt, const smb_coco_params2_t* host_params);
int smb_coco_match_params2_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                               const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt,
                               const uint32_t* gt_planes, int64_t gt_plane_words, const int32_t* gt_cat_off, int K,
                               int metric, const smb_coco_params2_t* host_params, smb_coco_out_t* out, int64_t n_out,
                               int* npig, int* status, void* workspace, size_t workspace_bytes, smb_stream_t stream);
/* smb_coco_accumulate_params_dev with these Params (K = 1 for use_cats 0). */
int smb_coco_accumulate_params2_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K,
                                    const int* npig, const smb_coco_params2_t* host_params, double* precision,
                                    double* recall, double* scores, smb_stream_t stream);

/* coco_error_analysis.py's per-category evaluations with relabelled ground truth (iouThrs [.1], maxDets [100], the four
 * area ranges host_area_rng[4][2]), for every (image, category) with detections: category k's detections against the
 * image's ground truths in annotation order, where an annotation of another category counts as a crowd annotation of k
 * when it is in k's supercategory (Sim, bit a of the row) or always (Oth, bit 4 + a).
 *   gt_pos [n_gt]: position of each ground-truth row in its image's annotation order (a permutation of [0, G_img));
 *   sup [K]: supercategory index of each category, in [0, n_sup).
 * Rows as smb_coco_match_dev writes them; no npig (the plain evaluation's applies).  A position or supercategory index
 * out of range sets SMB_COCO_ANALYSIS_RANGE.  workspace >= smb_coco_analysis_workspace_bytes(n_gt). */
size_t smb_coco_analysis_workspace_bytes(int n_gt);
int smb_coco_analysis_match_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                                const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt,
                                const uint32_t* gt_planes, int64_t gt_plane_words, const int32_t* gt_cat_off,
                                const int32_t* gt_pos, const int32_t* sup, int n_sup, int K, int metric,
                                const double* host_area_rng, smb_coco_out_t* out, int64_t n_out, int* status,
                                void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ YouTube-VIS mask AP (YTVOSeval, iouType 'segm')
 * The sequence IoU of a result entry d and a ground-truth object g over a video is sum_f I_f / U with
 *   U = sum A_d (frames where d is present) + sum A_g (frames where g is present) - sum I (frames where both are),
 * all integer pixel counts, so it is accumulated frame by frame in int64 and divided once in float64.
 *
 * One frame row of an overlap / scatter launch: its detection planes (absolute device pointer of detection 0, words from
 * one detection plane to the next, words per row), its number of detections when no count array is given, its h x w
 * canvas, the row pitch of its ground-truth planes, its ground-truth rows [g0, g0 + n_gt) and its accumulator slot
 * (< 0: the row accumulates nothing). */
typedef struct {
  const uint32_t* det;
  int64_t det_stride;
  int32_t det_pitch;
  int32_t n_det;
  int32_t h, w;
  int32_t gt_pitch;
  int32_t n_gt, g0;
  int32_t slot;
} smb_ytvis_frame_t;
/* A ground-truth object present in a frame: its plane (absolute device pointer, h x gt_pitch words), its index in the
 * video's ground truth (the accumulator column) and ext = {row0, row1, word0, word1} (half-open) of its set bits. */
typedef struct {
  const uint32_t* plane;
  int32_t g;
  int32_t ext[4];
  int32_t pad;
} smb_ytvis_gt_frame_t;
/* A ground-truth object of a video at its sequence match: avg_area (mean of its non-zero annotation areas), the sum of
 * its pixel counts over the frames it is present in, its annotation id, iscrowd and accumulator column. */
typedef struct {
  double avg_area;
  int64_t sum_area;
  int64_t id;
  int32_t crowd;
  int32_t g;
} smb_ytvis_gt_t;
/* A result entry of a video, in json order: its score, object id (accumulator row) and category index (-1: none). */
typedef struct {
  double score;
  int32_t obj;
  int32_t cat;
} smb_ytvis_entry_t;
#define SMB_YTVIS_OBJECTS 1   /* status: an object id at or beyond the accumulators' object capacity */
#define SMB_YTVIS_GTS 2       /* status: a ground-truth column at or beyond g_max */
#define SMB_YTVIS_RANGE 4     /* status: a slot, ground-truth row or output row outside its buffer */

/* Per-frame overlaps, one CTA per (frame row, detection): area[n, j] = pixel count of detection j (j < count[n], or < frames[n].n_det
 * when count is NULL, clamped to max_num) over the h x w canvas, inter[n, j, g] = |detection j AND ground truth g| for
 * every ground truth g present in the frame; every other entry of inter [N, max_num, g_max] and area [N, max_num] is 0. */
int smb_ytvis_overlap_dev(const smb_ytvis_frame_t* frames, int N, const int* count, int max_num,
                          const smb_ytvis_gt_frame_t* gts, int n_gts, int g_max, int32_t* inter, int32_t* area, int* status,
                          smb_stream_t stream);
/* Adds every frame row's overlaps into its slot's accumulators, keyed by object id: for each object id >= 0 among the
 * row's detections (count / n_det as above, ids [N, max_num]) only its LAST detection counts (a frame's result keeps the
 * last detection of a duplicate id).  acc_inter [slots, objects, g_max] += inter, acc_area [slots, objects] += area,
 * acc_nz [slots, objects] += (area > 0); int64 / int32 atomics. */
int smb_ytvis_scatter_dev(const smb_ytvis_frame_t* frames, int N, const int* count, const int32_t* ids, int max_num,
                          const int32_t* inter, const int32_t* area, int g_max, int64_t* acc_inter, int64_t* acc_area,
                          int32_t* acc_nz, int slots, int objects, int* status, smb_stream_t stream);
/* evaluateVid of one video (slot's accumulators) for every category, one CTA: the sequence IoU, ranks by score
 * (descending, stable over json order, the first SMB_COCO_MAX_DET kept), evaluateImg's greedy matching for the 10 x 4
 * (threshold, area range) pairs with avg_area as the area.  gts of category k are [gt_cat_off[k], gt_cat_off[k + 1])
 * in annotation order; out row e (< n_out) receives entry e with image_id = video_id (smb_coco_accumulate_dev's input);
 * npig [K, 4] is added to.  n_ent <= SMB_COCO_DET_CAP, workspace >= smb_ytvis_match_workspace_bytes(n_gt). */
size_t smb_ytvis_match_workspace_bytes(int n_gt);
int smb_ytvis_match_dev(const smb_ytvis_entry_t* ents, int n_ent, const smb_ytvis_gt_t* gts, int n_gt,
                        const int32_t* gt_cat_off, int K, int slot, const int64_t* acc_inter, const int64_t* acc_area,
                        const int32_t* acc_nz, int slots, int objects, int g_max, int64_t video_id,
                        const double* host_iou_thr, const double* host_area_rng, smb_coco_out_t* out, int64_t n_out,
                        int* npig, int* status, void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* ------------------------------------------------------------------ segmentations to bit planes on the device
 * What pycocotools' rleFrPoly / rleFrBbox / rleFrString followed by rleDecode compute, as the bit planes the evaluators
 * read (row-major [h, pitch] uint32, pixel x = bit x&31 of word x>>5, bits past w zero), without a sort: a column-major
 * mask is the parity of the number of run boundaries at or before each pixel, so every boundary toggles one bit of a
 * column-major scratch bitmap and a prefix XOR fills it.
 *
 * One item: a polygon (kind 0: n vertices, float64 x,y pairs from vertex `off` of the vertex pool; an frBbox box is its
 * four-vertex polygon) or column-major run lengths (kind 1: n uint32 counts from `off` of the count pool, zeros first),
 * in an h x w canvas, OR-ed into plane `plane` of the launch.  Items of one plane are adjacent (annToRLE's merge of an
 * annotation's polygons).  The caller guarantees 5 * |coordinate| < 2^29 and that run lengths sum to h * w. */
typedef struct {
  int32_t kind;
  int32_t plane;
  int64_t off, n;
  int32_t h, w;
} smb_segm_item_t;
#define SMB_SEGM_RANGE 1   /* status: an item's pool range, plane index or canvas is outside what the launch owns */

/* Zeroes planes [n_planes, plane_stride_words] and rasterizes the items into them on `stream` (memsets and three
 * launches, no allocation or synchronisation; graph-capturable).  n_xy: vertices in xy_pool; max_hw / max_w: the largest
 * h * w (< 2^31) and w of any item, which size the workspace (>= smb_segm_raster_workspace_bytes).  area / ext (either may
 * be NULL): plane p's pixel count goes to area[p * area_stride] and its {row0, row1, word0, word1} (half-open, zeros for
 * an empty plane) to ext[p * ext_stride ...], strides in int32 units, so both can land inside the caller's rows.  An item
 * that fails a bound writes nothing and sets SMB_SEGM_RANGE in *status. */
size_t smb_segm_raster_workspace_bytes(int n_items, int64_t max_hw, int max_w);
int smb_segm_raster_dev(const smb_segm_item_t* items, int n_items, const double* xy_pool, int64_t n_xy,
                        const uint32_t* count_pool, int64_t n_counts, int64_t max_hw, int max_w, uint32_t* planes,
                        int n_planes, int64_t plane_stride_words, int pitch, int32_t* area, int64_t area_stride,
                        int32_t* ext, int64_t ext_stride, int* status, void* workspace, size_t workspace_bytes,
                        smb_stream_t stream);

/* ------------------------------------------------------------------ detections drawn onto images on the device
 * The picture of the reference's show_result, for a batch of uint8 HWC 3-channel images in one launch:
 *   rule SMB_RENDER_IMAGES : SipMask-mmdetection/mmdet/apis/inference.py:119-184 (show_result).  Drawn: the detections
 *                            with score > score_thr (fp32), class-major (ascending label, detection order within a label),
 *                            colour palette[label % palette_rows], blend p <- (p + c) >> 1 (= uint8(p * 0.5 + c * 0.5)).
 *   rule SMB_RENDER_VIDEO  : SipMask-VIS/mmdet/models/detectors/base.py:90-192 (gen_colormask, show_result(is_video)).
 *                            Drawn: one entry per object id >= 0, at the position of the id's first detection and with
 *                            its last detection's score, box and mask (bbox2result_with_id's dict), when that score >
 *                            score_thr; colour palette[obj_id % palette_rows], blend p <- uint8(c * 0.6 + p * 0.4) in
 *                            float64 (each product and the sum rounded on its own).
 * Masks are blended in draw order, every channel c of a set pixel with the colour's byte c.  boxes != 0: then every
 * drawn box's outline in (0, 255, 0): corners truncated toward zero, the border of the inclusive rectangle [min x, max x]
 * x [min y, max y] clipped to the image (what cv2.rectangle(thickness=1) sets).  The label text is not drawn.
 *   imgs      : device rows [N]; image n is read from src and written to dst (src == dst: in place), h x w pixels
 *               (its ori_shape) of 3 bytes, rows 3 * w bytes apart.  A row with h or w <= 0, a null pointer, h > max_h
 *               or w > max_w is left untouched.  An image with nothing to draw is copied (src != dst) or left as it is.
 *   mask_bits : the engine's record [N, max_num, cap_h, words] (pixel x = bit x&31 of word x>>5); only the planes of
 *               image n's first count[n] (clamped to [0, max_num]) detections, rows < min(h, cap_h) and bits < w are read
 *   det       : [N, max_num, 5] fp32 boxes + score; labels [N, max_num] int64 (images), obj_ids [N, max_num] int32 (videos;
 *               the other may be NULL); palette [palette_rows, 3] uint8 device table.
 * max_num <= SMB_RENDER_MAX_NUM; max_w is bounded by the shared memory a CTA may use (about 70,000 pixels on sm_90). */
typedef struct {
  const uint8_t* src;
  uint8_t* dst;
  int32_t h, w;
} smb_render_img_t;
#define SMB_RENDER_IMAGES 0
#define SMB_RENDER_VIDEO 1
#define SMB_RENDER_MAX_NUM 1024
int smb_render_dev(const smb_render_img_t* imgs, int N, int max_h, int max_w, const uint32_t* mask_bits, int max_num,
                   int cap_h, int words, const float* det, const int64_t* labels, const int* count, const int32_t* obj_ids,
                   const uint8_t* palette, int palette_rows, int rule, float score_thr, int boxes, smb_stream_t stream);

/* gather rows: dst[i,:] = src[idx[i],:] for i < *count (device count), zero otherwise. */
int smb_gather_rows_f32(const float* src, int src_pitch, const int64_t* idx, const int* count_dev,
                        int max_rows, int row_elems, float* dst, smb_stream_t stream);

/* ------------------------------------------------------------------ convolution engine (wgmma)
 * Replaces every nn.Conv2d (+ folded eval BatchNorm, bias, residual add, ReLU) on the path
 * (models/backbones/resnet.py:203-239, models/necks/fpn.py:138-178, ops/conv_module.py:124-132,
 * anchor_heads/sipmask_head.py:241-287) with one implicit-GEMM kernel:
 *   D[pixels, Cout] = sum_{taps, Cin} A[pixel + tap, Cin] * Wt[Cout, tap, Cin]
 * A is the NHWC fp16 activation read through TMA tensor maps (one 2D-patch box per tap; zero
 * fill outside the image gives the padding), W is [Cout, taps*Cin] fp16 K-major, the fp32
 * accumulators live in registers (two warpgroups of wgmma.m64nNk16, M=128), the epilogue applies
 * scale/bias (folded BN), residual, ReLU, optional GroupNorm statistics, and writes NHWC.
 */
typedef struct smb_conv_plan smb_conv_plan_t;

typedef struct {
  int N, H, W, Cin;          /* input  NHWC (Cin % 64 == 0; the 3-channel stem uses smb_stem_plan_create_s2d) */
  int Cout;                  /* multiple of 16, <= 256 per N-tile (larger Cout is tiled) */
  int kh, kw, stride, pad;   /* 1x1/3x3 stride 1|2, pad = k/2 ; 7x7/2 stem uses the dedicated plan */
  int relu;                  /* apply ReLU in the epilogue */
  int has_bias;              /* per-channel fp32 bias (folded BN shift / conv bias) */
  int has_residual;          /* add an NHWC fp16 tensor of the output shape before ReLU */
  int residual_upsample;     /* residual is the coarser FPN level: nearest-neighbour gather (fpn.py:149-152) */
  int res_h, res_w;          /* residual spatial size when residual_upsample */
  int out_dtype;             /* SMB_F16 or SMB_F32 */
  int gn_stats;              /* accumulate per-(image,group) {sum*2^20, sumsq*2^16} as int64 fixed point into stats[N*32*2]
                                (integer atomics: bit-reproducible run to run) */
  int in_pitch, out_pitch;   /* channel pitch (elements) of input / output rows; 0 = dense */
} smb_conv_desc_t;

int smb_conv_plan_create(const smb_conv_desc_t* desc, const void* in, const void* weight, void* out,
                         smb_conv_plan_t** plan_out);

/* One launch over several feature-pyramid levels that share the weights (the FCOS towers / heads are applied to
 * P3..P7 in a python loop in the reference, sipmask_head.py:250-271).  desc->H/W are ignored; stride must be 1.
 * Per-level residual / gn_stats pointers are baked into the plan (pass NULLs to smb_conv_run). */
typedef struct {
  const void* in; void* out;
  const void* residual; void* gn_stats;
  int H, W, res_h, res_w;
} smb_conv_level_t;
int smb_conv_plan_create_multi(const smb_conv_desc_t* desc, int num_levels, const smb_conv_level_t* levels,
                               const void* weight, smb_conv_plan_t** plan_out);
void smb_conv_plan_destroy(smb_conv_plan_t* plan);
/* Cap the persistent grid of a plan (multiple of its cluster size), so that independent convolutions launched on
 * different streams share the GPU instead of running one after the other with half-empty last waves. */
int smb_conv_plan_set_max_ctas(smb_conv_plan_t* plan, int max_ctas);
/* Planner knob for plans created AFTER the call: the N tile is the largest of {256,128,64} that still yields at least
 * `min_tiles` output tiles (default 48; <= 0 restores the default).  Small values favour fat tiles (fewer bytes through
 * L2 -> SM per FLOP), large values favour occupancy of a single stream.  Returns the previous value. */
int smb_conv_set_min_tiles(int min_tiles);
/* out = relu?( (acc + bias) * alpha + residual ); alpha carries the per-level `Scale` of fcos_reg
 * (sipmask_head.py:261, ops/scale.py:12-15).  The residual must be 4-byte aligned (SMB_EINVAL without a launch). */
int smb_conv_run(const smb_conv_plan_t* plan, const float* bias, const void* residual, void* gn_stats,
                 float alpha, smb_stream_t stream);
/* What the planner chose for a plan, so that tests can state which kernel path a shape reaches.  Per level: the
 * BH x BW = 128-pixel output patch and the tile counts; per plan: the N tile (256 / 128 / 64) and the number of N tiles,
 * the operand ring's stages, whether fp16 outputs go through the shared-memory / TMA epilogue (as decided at creation:
 * a same-shape residual that is not 16-byte aligned still takes the register epilogue at run time), the persistent grid
 * and the dynamic shared memory of a launch. */
#define SMB_CONV_MAX_LEVELS 5
typedef struct {
  int num_levels, tiles_m;
  int n_tile, n_tiles_n, stages, epi_tma, grid, smem_bytes;
  int H_out[SMB_CONV_MAX_LEVELS], W_out[SMB_CONV_MAX_LEVELS];
  int BH[SMB_CONV_MAX_LEVELS], BW[SMB_CONV_MAX_LEVELS], tiles_x[SMB_CONV_MAX_LEVELS], tiles_y[SMB_CONV_MAX_LEVELS];
} smb_conv_plan_info_t;
int smb_conv_plan_info(const smb_conv_plan_t* plan, smb_conv_plan_info_t* info);

/* ------------------------------------------------------------------ elementwise / gather kernels (NHWC fp16) */
/* GroupNorm(32 groups, eps) + ReLU applied in place from precomputed per-(image,group) sum/sumsq
 * (ops/norm.py:43-49 + conv_module.py:124-132).  x [N*HW, C] fp16. */
int smb_groupnorm_relu_apply(void* x, int n_img, int hw, int C, int pitch, const void* stats /* int64 [n_img*32*2] */,
                             const float* gamma, const float* beta, float eps, int relu, smb_stream_t stream);
/* stats for a tensor that did not come out of smb_conv_run (e.g. DCN output computed elsewhere). */
int smb_groupnorm_stats(const void* x, int n_img, int hw, int C, int pitch, void* stats /* int64 */, smb_stream_t stream);

/* Deformable im2col (ops/dcn/src/deform_conv_cuda_kernel.cu:85-115,191-243), channel-last:
 *   x [H,W,C] fp16, offset [H,W,dg*18] fp32 (per dg: 2*(i*3+j)=dh, +1=dw) with pitch off_pitch >= dg*18
 *   -> col [H*W, 9*C] fp16, K index = tap*C + c (3x3, stride 1, pad 1, dil 1). */
int smb_deform_im2col(const void* x, const float* offset, int off_pitch, void* col,
                      int n_img, int H, int W, int C, int deformable_groups, smb_stream_t stream);

/* FeatureAlign.conv_offset (sipmask_head.py:30-33,50): off[pix,o] = sum_k W[o,k] * (bbox[pix,k] * scale), fp32. */
int smb_offset_conv1x1(const float* bbox, int bbox_pitch, float scale, const float* weight, int n_off, float* off,
                       long long npix, smb_stream_t stream);

/* Multi-level (batched over feature-pyramid levels, shared parameters) variants of the three kernels above:
 * one launch instead of one per level.  Pointer arrays are HOST arrays of device pointers.
 * smb_groupnorm_relu_apply_multi supports C in {256, 512, 1024, 2048} (SMB_EINVAL otherwise). */
int smb_groupnorm_relu_apply_multi(int num_levels, void* const* xs, const void* const* stats, const int* Hs, const int* Ws,
                                   int n_img, int C, int pitch, const float* gamma, const float* beta, float eps, int relu,
                                   smb_stream_t stream);
int smb_offset_conv1x1_multi(int num_levels, const float* const* bboxes, int bbox_pitch, const float* scales,
                             const float* weight, int n_off, float* const* offs, const int* Hs, const int* Ws, int n_img,
                             smb_stream_t stream);
/* The same offsets from relu(scale * bbox) (SipMask-benchmark FeatureAlign input with NORM_REG_TARGETS,
 * SipMask-benchmark/fcos_core/modeling/rpn/sipmask/sipmask.py:161-171). */
int smb_offset_conv1x1_relu_multi(int num_levels, const float* const* bboxes, int bbox_pitch, const float* scales,
                                  const float* weight, int n_off, float* const* offs, const int* Hs, const int* Ws, int n_img,
                                  smb_stream_t stream);
int smb_deform_im2col_multi(int num_levels, const void* const* xs, const float* const* offs, int off_pitch,
                            void* const* cols, const int* Hs, const int* Ws, int n_img, int C, int deformable_groups,
                            smb_stream_t stream);

/* MaxPool2d(3, 2, 1) (backbones/resnet.py:460), NHWC fp16. */
int smb_maxpool3x3s2(const void* x, void* y, int N, int H, int W, int C, smb_stream_t stream);

/* Bilinear upsample by an integer factor, align_corners=False (sipmask_head.py:279,285), NHWC fp16,
 * writing into a channel slice of a wider tensor (out_pitch, out_choff) so torch.cat is free.  y is [N, out_h, out_w]
 * pixels: normally out_h = H*factor, out_w = W*factor; otherwise the upsampled image is cropped or its last row / column
 * repeated, and nothing is written outside y.  factor 1 (a channel-slice copy) needs out_h = H, out_w = W. */
int smb_upsample_bilinear(const void* x, int in_pitch, void* y, int out_pitch, int out_choff,
                          int N, int H, int W, int out_h, int out_w, int C, int factor, int relu, smb_stream_t stream);

/* Stem 7x7/2 conv (3->64) + folded BN + ReLU (backbones/resnet.py:448-460) in space-to-depth form (K = 256): the
 * zero-padded image (pixel (y,x) at (y+3, x+3)) is stored as [N, H/2+3, W/2+4, 16] fp16 with element
 * (Y, X, (dy*2+dx)*4 + c) = padded pixel (2Y+dy, 2X+dx) channel c (c == 3: zero), the weights as [64, 4*64] with
 * K = a*64 + b*16 + (dy*2+dx)*4 + c for filter tap (r, s) = (2a+dy, 2b+dx). */
int smb_stem_plan_create_s2d(int N, int H, int W, const void* img_s2d16, const void* weight256, void* out,
                             smb_conv_plan_t** plan_out);
/* Image preparation: NCHW fp32 -> the stem's space-to-depth input above (H, W even). */
int smb_image_to_s2d16(const float* img_nchw_f32, void* out_s2d16, int N, int H, int W, smb_stream_t stream);

/* Test-time image pipeline on the device (SURVEY.md 8f-3; transforms.py:97-110 Resize(keep_ratio), :335-363 Normalize
 * (std = 1, to_rgb = False), :274-300 Pad(32); mmcv.imrescale -> cv2.resize(INTER_LINEAR) restated bit-exactly):
 *   src       : uint8 BGR HWC [src_h, src_w, 3] device image, row pitch in bytes
 *   dst_h/w   : resized size (mmcv rule: int(h * s + 0.5), s = min(max_long / max(h, w), max_short / min(h, w)))
 *   out_s2d16 : the stem's space-to-depth input [H/2+3, W/2+4, 16] fp16 of the padded H x W image (H, W even, padded
 *               size >= dst); everything outside the resized image is zero (= zero padding AFTER mean subtraction, as in
 *               the reference) */
int smb_preprocess_u8_s2d(const uint8_t* src, int src_h, int src_w, int src_pitch_bytes, int dst_h, int dst_w,
                          const float* host_mean3, void* out_s2d16, int H, int W, smb_stream_t stream);

/* One image of a batched preprocessing launch, read from DEVICE memory when the kernel runs (so a captured CUDA graph
 * serves new images and sizes: the host rewrites the rows between replays).
 *   src              : absolute device pointer of the image's uint8 BGR HWC pixels, row pitch src_pitch_bytes (>= 3 * src_w)
 *   dst_h, dst_w     : the resized size (the image's img_shape), <= the canvas H x W
 *   mean[3]          : subtracted per channel (kept in the row, so a captured graph never holds a stale mean)
 * A filler row (dst_h == 0 or dst_w == 0) writes an all-zero canvas and reads nothing (src may be null): a partial batch
 * fills its remaining images with such rows.  The rows are not validated on the device; the caller validates them. */
typedef struct {
  const uint8_t* src;
  int src_h, src_w, src_pitch_bytes;
  int dst_h, dst_w;
  float mean[3];
} smb_raw_src_t;

/* smb_preprocess_u8_s2d for a batch: out_s2d16 [N, H/2+3, W/2+4, 16] fp16, canvas n from rows[n] (device pointer to N
 * rows), one launch over all N canvases.  Same kernel as smb_preprocess_u8_s2d (which passes its one row by value), so
 * every canvas is bit-identical to the single-image entry point.  Reads sum(src bytes), writes N*(H/2+3)*(W/2+4)*32 bytes. */
int smb_preprocess_u8_s2d_dev(const smb_raw_src_t* rows, int N, void* out_s2d16, int H, int W, smb_stream_t stream);

/* SipMask-benchmark's test transform for a batch (SipMask-benchmark/fcos_core/data/transforms/build.py:17-36,
 * transforms.py:27-95: PIL Image.resize(BILINEAR) -> to_tensor -> to_bgr255 -> normalize(std = 1) -> pad), restated
 * bit-exactly (Pillow's separable antialiased 22-bit fixed-point filter, horizontal pass clipped to uint8 first):
 *   rows[n].src   : RGB HWC uint8, as PIL decodes it (the other fields as for smb_preprocess_u8_s2d_dev)
 *   rows[n].mean  : in output (BGR) order; output channel c = float(src[2 - c]) - mean[c], rounded once to fp16
 * Same [N, H/2+3, W/2+4, 16] canvas, halo / padding zeros and filler rows as smb_preprocess_u8_s2d_dev.  A downscale of
 * more than 8x on either axis is not supported (the caller rejects it).  Reads sum(src bytes), writes
 * N*(H/2+3)*(W/2+4)*32 bytes. */
int smb_preprocess_pil_u8_s2d_dev(const smb_raw_src_t* rows, int N, void* out_s2d16, int H, int W, smb_stream_t stream);

/* ------------------------------------------------------------------ training-side operators (train_ops.cu)
 * DeformConv backward, 3x3 / stride 1 / pad 1 / dilation 1 / groups 1, channel-last like smb_deform_im2col.  Replaces
 * deform_conv_backward_input_cuda and deform_conv_backward_parameters_cuda (ops/dcn/src/deform_conv_cuda.cpp:262-470).
 *
 * smb_deform_grad_scale: grad_out [N, C, H, W] fp32 (NCHW, as autograd passes it) -> out_f16 [N, H, W, C] = s * grad_out,
 * with s = 2^k chosen on the device so that amax |grad_out| lands in [2^14, 2^15) (s = 1 when amax is 0 or not finite),
 * no host synchronisation.  scale (device, 2 floats) receives {s, 1 / s}.  C % 8 == 0.  One cooperative launch;
 * workspace: smb_deform_grad_scale_workspace_bytes(). */
size_t smb_deform_grad_scale_workspace_bytes(void);
int smb_deform_grad_scale(const float* grad_out, int n_img, int C, int H, int W, void* out_f16, float* scale,
                          void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* smb_deform_col2im: deformable_col2im_coord and deformable_col2im (ops/dcn/src/deform_conv_cuda_kernel.cu:337-465) in one
 * pass over grad_col [N, H, W, 9 * C] fp32 (column k = tap * C + c, holding s * the column gradient):
 *   grad_offset [N, H, W, dg * 18] fp32 (channel g * 18 + 2 * tap + {0: h, 1: w}), every element written, each a
 *     fixed-order sum over the group's C / dg channels of get_coordinate_weight (kernel.cu:145-188) x grad_col / s;
 *   grad_input [N, H, W, C] fp32, ACCUMULATED (zero it first) with float atomics: get_gradient_weight (kernel.cu:117-143)
 *     x grad_col / s.
 * Either output may be null (not both).  x [N, H, W, C] fp16, offset [N, H, W, >= dg * 18] fp32 with pitch off_pitch,
 * scale = smb_deform_grad_scale's {s, 1 / s}.  C % 8 == 0, C <= 1024, (C / dg) % 8 == 0. */
int smb_deform_col2im(const float* grad_col, const void* x, const float* offset, int off_pitch, const float* scale,
                      float* grad_input, float* grad_offset, int n_img, int H, int W, int C, int deformable_groups,
                      smb_stream_t stream);

/* smb_deform_weight_grad: grad_weight [Cout, K] fp32 = sum_p grad_f16[p, co] * col[p, k] / s over P pixels, the
 * columns' GEMM of deform_conv_backward_parameters_cuda (deform_conv_cuda.cpp:376-470; col recomputed by
 * smb_deform_im2col, K = 9 * C).  grad_f16 [P, Cout] fp16 (smb_deform_grad_scale's output), col [P, K] fp16.  wgmma with
 * MN-major operands, split over pixels; the splits are summed in a fixed order, so the result is the same bits on every
 * run.  Cout % 8 == 0, K % 8 == 0, 16-byte aligned pointers; workspace: smb_deform_weight_grad_workspace_bytes. */
size_t smb_deform_weight_grad_workspace_bytes(int Cout, int K, long long P);
int smb_deform_weight_grad(const void* grad_f16, const void* col, long long P, int Cout, int K, const float* scale,
                           float* grad_weight, void* workspace, size_t workspace_bytes, smb_stream_t stream);

/* Sigmoid focal loss (ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-100, SigmoidFocalLoss_forward_cuda /
 * _backward_cuda): logits [N, C] fp32, targets [N] int64 (1-based class, 0 = background, < 0 ignored), d_losses [N, C]
 * fp32 -> losses / d_logits [N, C] fp32, every element written.  The reference's expressions operation by operation,
 * so the results are the reference kernel's bits.  N = 0 launches nothing. */
int smb_sigmoid_focal_loss_forward(const float* logits, const int64_t* targets, int N, int num_classes, float gamma,
                                   float alpha, float* losses, smb_stream_t stream);
int smb_sigmoid_focal_loss_backward(const float* logits, const int64_t* targets, const float* d_losses, int N,
                                    int num_classes, float gamma, float alpha, float* d_logits, smb_stream_t stream);

/* ------------------------------------------------------------------ SipMask mask loss (mask_loss.cu)
 * The mask-loss block of SipMaskHead.loss (models/anchor_heads/sipmask_head.py:437-463), fused: no [H, W, M] tensor is
 * stored.
 *
 * smb_mask_targets: gt mask planes -> bits [G, H, ceil(W / 32)] uint32 (bit x % 32 of word x / 32 is pixel x), equal to
 * F.interpolate(scale_factor=0.5, bilinear, align_corners=False) -> zero pad / crop to H x W -> gt(0.5) on {0, 1} masks
 * (any non-zero byte counts as 1).  src: uint8 planes; planes [G, 3] int64 (device) = {byte offset of the plane in src,
 * Hf, Wf}.  One launch; G = 0 launches nothing. */
int smb_mask_targets(const void* src, const long long* planes, int G, int H, int W, uint32_t* bits, smb_stream_t stream);

/* smb_mask_loss: feat [B, 32, H, W] fp32 NCHW, cofs [M, 128] fp32, boxes [M, 4] fp32 (mask coordinates), img_offsets
 * [B + 1] int32 (instances of image b are img_offsets[b] .. img_offsets[b + 1] - 1), targets from smb_mask_targets with G
 * planes, gt_rows [M] int32 (a row outside [0, G) reads as an empty mask), weights [M] fp32; all on the device.
 *   g == NULL (forward): loss [B] fp32, loss[b] = sum over b's instances n and the pixels inside n's box of
 *     BCE(sigmoid(z), t) * w_n / (bw_n * bh_n * M_b) (torch's CUDA sigmoid and binary_cross_entropy, logs clamped at
 *     -100; CropSplit's cell geometry).
 *   g [B] (backward): d_feat [B, 32, H, W] (every element written) and / or d_cofs [M, 128] (every element written) for
 *     the upstream gradient g of loss; either may be NULL, not both.
 * Every sum has a fixed order (the same bits on every run); no host synchronisation.  M = 0, images without instances
 * and boxes outside the map give 0.  workspace: smb_mask_loss_workspace_bytes(B, M, H, W). */
size_t smb_mask_loss_workspace_bytes(int B, int M, int H, int W);
int smb_mask_loss(const float* feat, const float* cofs, const float* boxes, const int* img_offsets, const uint32_t* targets,
                  int G, const int* gt_rows, const float* weights, const float* g, int B, int M, int H, int W, float* loss,
                  float* d_feat, float* d_cofs, void* workspace, size_t workspace_bytes, smb_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* SIPMASK_B200_H_ */
