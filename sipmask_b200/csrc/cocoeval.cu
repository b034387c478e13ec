// COCO box and mask AP (pycocotools 2.0 COCOeval, iouType 'bbox' / 'segm', default parameters) on the device, plus the
// host rasterizer of the ground truth (pycocotools maskApi.c rleFrPoly / rleFrString restated).
//
//   smb_coco_det_from_record_dev : engine record -> detection rows as the result json carries them (coco.coco_json)
//   smb_coco_match_dev           : computeIoU + evaluateImg for every (image, category) of a batch of images
//   smb_coco_accumulate_dev      : accumulate's precision / recall / scores arrays from the globally sorted rows
//   smb_coco_*_params_dev        : the same two with user-given Params (thresholds, area ranges, maxDets, recall
//                                  thresholds as data); the default Params give what the two above give
//   smb_coco_*_params2_dev       : the same with useCats 0 (one pooled group per image) and maxDets up to 1000
//   smb_coco_analysis_match_dev  : coco_error_analysis.py's Sim / Oth evaluations (relabelled ground truth) of a batch
//
// Every float64 operation whose result is compared with pycocotools is an explicit _rn intrinsic, so nvcc cannot
// contract it into an FMA (x86-64 pycocotools has none).
#include <math.h>
#include <limits.h>
#include <algorithm>
#include <vector>

#include "coco_match.cuh"
#include "cta.cuh"

namespace {

using smb_match::kT;
using smb_match::kA;
using smb_match::kMaxDet;
using smb_match::MatchParams;
constexpr int kR = SMB_COCO_R;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// ------------------------------------------------------------------------------------------------ 2a: record -> rows
__global__ void __launch_bounds__(kThreads) det_from_record_kernel(
    const float* __restrict__ det, const int64_t* __restrict__ labels, const int* __restrict__ count,
    const float* __restrict__ mask_scores, const uint32_t* __restrict__ mask_bits, int max_num, int cap_h, int words,
    const smb_img_geom_t* __restrict__ geom, const int32_t* __restrict__ label_cat, int num_labels, int benchmark,
    smb_coco_det_t* __restrict__ rows, smb_coco_img_t* __restrict__ imgs, int* __restrict__ status) {
  const int n = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lid = tid & 31;
  const int cnt = min(max(count[n], 0), max_num);
  const smb_img_geom_t g = geom[n];
  const int oh = min(max(g.out_h, 0), cap_h), ow = min(max(g.out_w, 0), words * 32);
  const int ow_words = (ow + 31) >> 5;
  const uint32_t last_mask = (ow & 31) ? ((1u << (ow & 31)) - 1u) : 0xffffffffu;
  if (tid == 0) imgs[n].n_det = cnt;
  for (int j = warp; j < max_num; j += kWarps) {
    smb_coco_det_t r;
    const size_t rj = (size_t)n * max_num + j;
    const int64_t plane = (int64_t)rj * cap_h * words;
    // ---- area and extents by popcount over the ori_shape canvas (maskUtils.area)
    int area = 0, r0 = INT_MAX, r1 = -1, w0 = INT_MAX, w1 = -1;
    if (j < cnt) {
      const uint32_t* p = mask_bits + plane;
      for (int y = 0; y < oh; ++y) {
        for (int x = lid; x < ow_words; x += 32) {
          uint32_t v = p[(size_t)y * words + x];
          if (x == ow_words - 1) v &= last_mask;
          if (v) { area += __popc(v); r0 = min(r0, y); r1 = max(r1, y); w0 = min(w0, x); w1 = max(w1, x); }
        }
      }
      for (int o = 16; o > 0; o >>= 1) {
        area += __shfl_xor_sync(0xffffffffu, area, o);
        r0 = min(r0, __shfl_xor_sync(0xffffffffu, r0, o));
        r1 = max(r1, __shfl_xor_sync(0xffffffffu, r1, o));
        w0 = min(w0, __shfl_xor_sync(0xffffffffu, w0, o));
        w1 = max(w1, __shfl_xor_sync(0xffffffffu, w1, o));
      }
    }
    if (lid != 0) continue;
    if (j >= cnt) {
      memset(&r, 0, sizeof(r));
      r.cat = -1;
      rows[rj] = r;
      continue;
    }
    const float* d = det + rj * 5;
    if (benchmark) {
      // BoxList.resize to the ori_shape canvas: float32 boxes times the float32 ratio (torch scalar arithmetic), then
      // TO_REMOVE = 1 in float32 (coco_eval.py prepare_for_coco_detection)
      const float rw = __double2float_rn(__ddiv_rn((double)g.out_w, (double)g.img_w));
      const float rh = __double2float_rn(__ddiv_rn((double)g.out_h, (double)g.img_h));
      const float x1 = __fmul_rn(d[0], rw), y1 = __fmul_rn(d[1], rh), x2 = __fmul_rn(d[2], rw), y2 = __fmul_rn(d[3], rh);
      r.box[0] = x1;
      r.box[1] = y1;
      r.box[2] = __fadd_rn(__fsub_rn(x2, x1), 1.0f);
      r.box[3] = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
    } else {
      // MM xyxy2xywh on python floats of the float32 boxes: (x2 - x1) + 1 in float64
      r.box[0] = d[0];
      r.box[1] = d[1];
      r.box[2] = __dadd_rn(__dsub_rn((double)d[2], (double)d[0]), 1.0);
      r.box[3] = __dadd_rn(__dsub_rn((double)d[3], (double)d[1]), 1.0);
    }
    r.score[0] = d[4];
    r.score[1] = (!benchmark && mask_scores) ? (double)mask_scores[rj] : (double)d[4];
    r.area_box = __dmul_rn(r.box[2], r.box[3]);              // loadRes: bb[2] * bb[3]
    r.plane = plane;
    r.area_mask = area;
    if (area > 0) {
      r.ext[0] = r0; r.ext[1] = r1 + 1; r.ext[2] = w0; r.ext[3] = w1 + 1;
    } else {
      r.ext[0] = r.ext[1] = r.ext[2] = r.ext[3] = 0;
    }
    const int64_t lab = labels[rj];
    // json order: MM writes label-major (ascending labels), record order inside a label; BM record order
    r.order = benchmark ? j : (int)min(max(lab, (int64_t)0), (int64_t)num_labels) * max_num + j;
    r.pad = 0;
    if (lab < 0 || lab >= num_labels) {
      r.cat = -1;
      atomicOr(status, SMB_COCO_LABEL_RANGE);
    } else {
      r.cat = label_cat[lab];
    }
    rows[rj] = r;
  }
}

// ------------------------------------------------------------------------------------------------ 2b + 2c: IoU, matching
__device__ __forceinline__ double box_iou(const double* d, const double* g, int crowd) {
  // maskApi.c bbIou, operation by operation
  const double da = __dmul_rn(d[2], d[3]), ga = __dmul_rn(g[2], g[3]);
  const double w = __dsub_rn(fmin(__dadd_rn(d[2], d[0]), __dadd_rn(g[2], g[0])), fmax(d[0], g[0]));
  if (w <= 0) return 0.0;
  const double h = __dsub_rn(fmin(__dadd_rn(d[3], d[1]), __dadd_rn(g[3], g[1])), fmax(d[1], g[1]));
  if (h <= 0) return 0.0;
  const double i = __dmul_rn(w, h);
  const double u = crowd ? da : __dsub_rn(__dadd_rn(da, ga), i);
  return __ddiv_rn(i, u);
}

// computeIoU's [D, G] matrix of the sorted detections (rows s_sorted[d] of drow) against ground truths gt_of(g) = {row in
// gts (-1: none, IoU 0), iscrowd}: bbIou for metric 0, rleIou of the bit planes for metric 1 (one warp per pair).
template <typename GtOf>
__device__ __forceinline__ void iou_matrix(int metric, int D, int G, const smb_coco_det_t* __restrict__ drow,
                                           const int* s_sorted, const smb_coco_gt_t* __restrict__ gts, GtOf gt_of, int H,
                                           int dpitch, int gpitch, const uint32_t* __restrict__ det_planes,
                                           int64_t det_plane_words, const uint32_t* __restrict__ gt_planes,
                                           int64_t gt_plane_words, double* __restrict__ ious) {
  const int tid = threadIdx.x, warp = tid >> 5, lid = tid & 31;
  if (metric == 0) {
    for (int p = tid; p < D * G; p += kThreads) {
      const int d = p / G, g = p - d * G;
      const int2 gc = gt_of(g);
      ious[p] = gc.x < 0 ? 0.0 : box_iou(drow[s_sorted[d]].box, gts[gc.x].box, gc.y);
    }
  } else {
    for (int p = warp; p < D * G; p += kWarps) {
      const int d = p / G, g = p - d * G;
      const int2 gc = gt_of(g);
      const smb_coco_det_t& dr = drow[s_sorted[d]];
      const smb_coco_gt_t& gr = gts[max(gc.x, 0)];
      const int y0 = max(max(dr.ext[0], gr.ext[0]), 0), y1 = min(min(dr.ext[1], gr.ext[1]), H);
      const int x0 = max(max(dr.ext[2], gr.ext[2]), 0), x1 = min(min(min(dr.ext[3], gr.ext[3]), dpitch), gpitch);
      const int nx = x1 - x0;
      int inter = 0;
      const bool dok = dr.plane >= 0 && dr.plane + (int64_t)H * dpitch <= det_plane_words;
      const bool gok = gc.x >= 0 && gr.plane >= 0 && gr.plane + (int64_t)H * gpitch <= gt_plane_words;
      if (dok && gok && nx > 0 && y1 > y0) {
        const uint32_t* pd = det_planes + dr.plane;
        const uint32_t* pg = gt_planes + gr.plane;
        for (int e = lid; e < (y1 - y0) * nx; e += 32) {
          const int y = y0 + e / nx, x = x0 + e % nx;
          inter += __popc(pd[(size_t)y * dpitch + x] & pg[(size_t)y * gpitch + x]);
        }
      }
      for (int o = 16; o > 0; o >>= 1) inter += __shfl_xor_sync(0xffffffffu, inter, o);
      if (lid == 0) {
        double v = 0.0;                            // rleIou: i == 0 -> 0
        if (inter > 0) {
          const long long u = gc.y ? (long long)dr.area_mask : (long long)dr.area_mask + gr.area_mask - inter;
          v = __ddiv_rn((double)inter, (double)u);
        }
        ious[p] = v;
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) match_kernel(
    const smb_coco_img_t* __restrict__ imgs, const smb_coco_det_t* __restrict__ dets, int det_cap,
    const uint32_t* __restrict__ det_planes, int64_t det_plane_words, const smb_coco_gt_t* __restrict__ gts, int n_gt,
    const uint32_t* __restrict__ gt_planes, int64_t gt_plane_words, const int32_t* __restrict__ gt_cat_off, int K,
    int metric, MatchParams P, smb_coco_out_t* __restrict__ out, int64_t n_out, int* __restrict__ npig,
    double* __restrict__ iou_ws, uint8_t* __restrict__ gtm_ws, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_m = (uint64_t*)smem;                 // [kMaxDet] matched bits (t * P.A + a) of the sorted detections
  uint64_t* s_ig = s_m + kMaxDet;                  // [kMaxDet] ignore bits
  int* s_sorted = (int*)(s_ig + kMaxDet);          // [kMaxDet] detection row of rank r
  int* s_start = s_sorted + kMaxDet;               // [K + 1] per category: first entry of s_list
  int* s_list = s_start + K + 1;                   // [det_cap] detections grouped by category, record order inside
  const int b = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lid = tid & 31;
  const smb_coco_img_t im = imgs[b];
  const int nd = min(max(im.n_det, 0), det_cap);
  const smb_coco_det_t* drow = dets + (size_t)b * det_cap;
  const int32_t* goff = gt_cat_off + (size_t)b * (K + 1);
  const int H = max(im.h, 0), gpitch = max(im.gt_pitch, 0), dpitch = max(im.det_pitch, 0);
  auto out_row = [&](int j) -> smb_coco_out_t* {
    const int64_t o = im.out_off + j;
    return (o >= 0 && o < n_out) ? out + o : nullptr;
  };
  // every row of the image starts excluded (cat = K sorts after every category); its category's pass overwrites it
  for (int j = tid; j < det_cap; j += kThreads) {
    smb_coco_out_t* o = out_row(j);
    if (o) { o->score = 0; o->image_id = im.image_id; o->matched = 0; o->ignored = 0; o->cat = K; o->rank = -1; }
  }
  // counting sort of the detections by category, stable (thread 0: at most det_cap steps)
  if (tid == 0) {
    for (int k = 0; k <= K; ++k) s_start[k] = 0;
    for (int j = 0; j < nd; ++j) {
      const int c = drow[j].cat;
      if (c >= 0 && c < K) s_start[c + 1]++;
    }
    for (int k = 0; k < K; ++k) s_start[k + 1] += s_start[k];
    for (int j = 0; j < nd; ++j) {
      const int c = drow[j].cat;
      if (c >= 0 && c < K) s_list[s_start[c]++] = j;
    }
    for (int k = K; k > 0; --k) s_start[k] = s_start[k - 1];
    s_start[0] = 0;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    const int l0 = s_start[k], n = s_start[k + 1] - l0;
    const int g0 = min(max(goff[k], 0), n_gt), g1 = min(max(goff[k + 1], g0), n_gt), G = g1 - g0;
    if (n == 0 && G == 0) continue;                // evaluateImg returns None
    const int D = min(n, P.max_det);
    // ---- rank inside (image, category): score descending, stable over the json order
    for (int i = tid; i < n; i += kThreads) {
      const int j = s_list[l0 + i];
      const double s = drow[j].score[metric];
      const int oj = drow[j].order;
      int r = 0;
      for (int q = 0; q < n; ++q) {
        const int jq = s_list[l0 + q];
        const double sq = drow[jq].score[metric];
        const int oq = drow[jq].order;
        r += (sq > s) || (sq == s && (oq < oj || (oq == oj && jq < j)));
      }
      if (r < P.max_det) s_sorted[r] = j;          // computeIoU keeps the first maxDets[-1]
    }
    for (int i = tid; i < D; i += kThreads) { s_m[i] = 0; s_ig[i] = 0; }
    __syncthreads();
    // ---- IoU [D, G] (ground truths in annotation order)
    double* ious = iou_ws + (size_t)kMaxDet * g0;
    iou_matrix(metric, D, G, drow, s_sorted, gts, [&](int g) { return make_int2(g0 + g, gts[g0 + g].crowd); }, H, dpitch,
               gpitch, det_planes, det_plane_words, gt_planes, gt_plane_words, ious);
    __syncthreads();
    // ---- evaluateImg's greedy matching, one thread per (threshold, area range)
    smb_match::greedy_match(
        tid, D, G, ious, gtm_ws + (size_t)P.T * P.A * g0, P,
        [&](int g) {
          const smb_coco_gt_t& gr = gts[g0 + g];
          return smb_match::MatchGt{gr.area, gr.id, gr.crowd};
        },
        [&](int d) {
          const smb_coco_det_t& dr = drow[s_sorted[d]];
          return metric == 0 ? dr.area_box : (double)dr.area_mask;
        },
        npig + k * P.A, s_m, s_ig);
    __syncthreads();
    for (int r = tid; r < D; r += kThreads) {
      const int j = s_sorted[r];
      smb_coco_out_t* o = out_row(j);
      if (o) {
        o->score = drow[j].score[metric];
        o->matched = s_m[r];
        o->ignored = s_ig[r];
        o->cat = k;
        o->rank = r;
      } else {
        atomicOr(status, SMB_COCO_CAPACITY);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ 2b' + 2c': Params2
// match_kernel for smb_coco_params2_t: useCats 0 (one pooled group per image) or 1, and up to SMB_COCO_MAX_DET2 ranked
// detections per group.  The image's detections are ranked at once by a bitonic sort of their indices in shared memory,
// with the keys staged there too: (group, score descending, category index, json order, row), a total order, so the sort
// needs no stability.  group = category index with useCats 1, 0 with useCats 0; rows of no evaluated category sort last.
// A group is then a run of the sorted indices, found by binary search, and its first min(n, maxDet) entries are its
// ranked detections, as computeIoU keeps them.  IoU, the greedy loop and the output rows are match_kernel's.
// Dynamic shared memory: s_m / s_ig [max_det] uint64, then per padded row (n_pad = det_cap rounded up to a power of two)
// score double, tie uint64 = (category index << 32 | order), group int, sorted index int, then s_start [groups + 1].
constexpr int kMaxDet2 = SMB_COCO_MAX_DET2;

__host__ __device__ inline int pad_pow2(int n) {
  int p = 1;
  while (p < n) p <<= 1;
  return p;
}

inline size_t match2_smem_bytes(int det_cap, int K, int max_det, int use_cats) {
  const size_t n_pad = (size_t)pad_pow2(det_cap);
  return 2 * (size_t)max_det * sizeof(uint64_t) + n_pad * (sizeof(double) + sizeof(uint64_t) + 2 * sizeof(int)) +
         (size_t)((use_cats ? K : 1) + 1) * sizeof(int);
}

__global__ void __launch_bounds__(kThreads) match2_kernel(
    const smb_coco_img_t* __restrict__ imgs, const smb_coco_det_t* __restrict__ dets, int det_cap,
    const uint32_t* __restrict__ det_planes, int64_t det_plane_words, const smb_coco_gt_t* __restrict__ gts, int n_gt,
    const uint32_t* __restrict__ gt_planes, int64_t gt_plane_words, const int32_t* __restrict__ gt_cat_off, int K,
    int metric, int use_cats, MatchParams P, smb_coco_out_t* __restrict__ out, int64_t n_out, int* __restrict__ npig,
    double* __restrict__ iou_ws, uint8_t* __restrict__ gtm_ws, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int n_pad = pad_pow2(det_cap), n_grp = use_cats ? K : 1;
  uint64_t* s_m = (uint64_t*)smem;                 // [max_det] matched bits of the ranked detections of a group
  uint64_t* s_ig = s_m + P.max_det;                // [max_det] ignore bits
  double* s_score = (double*)(s_ig + P.max_det);   // [n_pad] per row
  uint64_t* s_tie = (uint64_t*)(s_score + n_pad);  // [n_pad] per row
  int* s_grp = (int*)(s_tie + n_pad);              // [n_pad] per row (INT_MAX: not evaluated)
  int* s_idx = s_grp + n_pad;                      // [n_pad] rows in rank order (-1: padding)
  int* s_start = s_idx + n_pad;                    // [n_grp + 1] first sorted position of each group
  const int b = blockIdx.x, tid = threadIdx.x;
  const smb_coco_img_t im = imgs[b];
  const int nd = min(max(im.n_det, 0), det_cap);
  const smb_coco_det_t* drow = dets + (size_t)b * det_cap;
  const int32_t* goff = gt_cat_off + (size_t)b * (K + 1);
  const int H = max(im.h, 0), gpitch = max(im.gt_pitch, 0), dpitch = max(im.det_pitch, 0);
  auto out_row = [&](int j) -> smb_coco_out_t* {
    const int64_t o = im.out_off + j;
    return (o >= 0 && o < n_out) ? out + o : nullptr;
  };
  for (int j = tid; j < det_cap; j += kThreads) {
    smb_coco_out_t* o = out_row(j);
    if (o) { o->score = 0; o->image_id = im.image_id; o->matched = 0; o->ignored = 0; o->cat = n_grp; o->rank = -1; }
  }
  for (int j = tid; j < n_pad; j += kThreads) {
    s_idx[j] = j < nd ? j : -1;
    if (j < nd) {
      const int c = drow[j].cat;
      const bool ok = c >= 0 && c < K;
      s_grp[j] = ok ? (use_cats ? c : 0) : INT_MAX;
      s_score[j] = drow[j].score[metric];
      s_tie[j] = ((uint64_t)(uint32_t)c << 32) | (uint32_t)drow[j].order;
    }
  }
  auto before = [&](int x, int y) -> bool {        // x ranks before y; padding (-1) after everything
    if (y < 0) return x >= 0;
    if (x < 0) return false;
    if (s_grp[x] != s_grp[y]) return s_grp[x] < s_grp[y];
    if (s_score[x] != s_score[y]) return s_score[x] > s_score[y];
    if (s_tie[x] != s_tie[y]) return s_tie[x] < s_tie[y];
    return x < y;
  };
  smb::cta_bitonic_sort(s_idx, n_pad, before);    // synchronises before it reads the rows staged above
  // group g's sorted positions are [s_start[g], s_start[g + 1]): the first position whose group is >= g
  for (int g = tid; g <= n_grp; g += kThreads) {
    int lo = 0, hi = nd;
    while (lo < hi) {
      const int mid = (lo + hi) >> 1;
      if (s_grp[s_idx[mid]] < g) lo = mid + 1; else hi = mid;
    }
    s_start[g] = lo;
  }
  __syncthreads();
  for (int k = 0; k < n_grp; ++k) {
    const int l0 = s_start[k], n = s_start[k + 1] - l0;
    const int c0 = use_cats ? k : 0, c1 = use_cats ? k + 1 : K;
    const int g0 = min(max(goff[c0], 0), n_gt), g1 = min(max(goff[c1], g0), n_gt), G = g1 - g0;
    if (n == 0 && G == 0) continue;                // evaluateImg returns None
    const int D = min(n, P.max_det);
    const int* ranked = s_idx + l0;
    for (int i = tid; i < D; i += kThreads) { s_m[i] = 0; s_ig[i] = 0; }
    double* ious = iou_ws + (size_t)P.max_det * g0;
    iou_matrix(metric, D, G, drow, ranked, gts, [&](int g) { return make_int2(g0 + g, gts[g0 + g].crowd); }, H, dpitch,
               gpitch, det_planes, det_plane_words, gt_planes, gt_plane_words, ious);
    __syncthreads();
    smb_match::greedy_match(
        tid, D, G, ious, gtm_ws + (size_t)P.T * P.A * g0, P,
        [&](int g) {
          const smb_coco_gt_t& gr = gts[g0 + g];
          return smb_match::MatchGt{gr.area, gr.id, gr.crowd};
        },
        [&](int d) {
          const smb_coco_det_t& dr = drow[ranked[d]];
          return metric == 0 ? dr.area_box : (double)dr.area_mask;
        },
        npig + k * P.A, s_m, s_ig);
    __syncthreads();
    for (int r = tid; r < D; r += kThreads) {
      const int j = ranked[r];
      smb_coco_out_t* o = out_row(j);
      if (o) {
        o->score = drow[j].score[metric];
        o->matched = s_m[r];
        o->ignored = s_ig[r];
        o->cat = k;
        o->rank = r;
      } else {
        atomicOr(status, SMB_COCO_CAPACITY);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ 2e: error analysis
// coco_error_analysis.py evaluates category k's detections alone against a ground truth in which the annotations of
// other categories become crowd (ignored) annotations of k: those of k's supercategory (Sim, variant 0) or all of them
// (Oth, variant 1); iouThrs [.1], maxDets [100].  Its rows are one CTA per image, per category with detections there:
// rank as match_kernel, one IoU matrix against every ground truth of the image (a relabelled one is crowd, IoU =
// inter / area_d), and the greedy loop once per (variant v, area range a) over the image's annotations in file order,
// filtered to the variant's set; bit v * A + a of the row.  npig is the plain evaluation's (only k's own ground truths
// count), so none is written here.
//   gt_pos [n_gt]: position of ground-truth row r in its image's annotation order; sup [K]: supercategory index
//   pos_ws : [n_gt] rows by annotation position (base + p), then [n_gt] their category
__global__ void __launch_bounds__(kThreads) analysis_match_kernel(
    const smb_coco_img_t* __restrict__ imgs, const smb_coco_det_t* __restrict__ dets, int det_cap,
    const uint32_t* __restrict__ det_planes, int64_t det_plane_words, const smb_coco_gt_t* __restrict__ gts, int n_gt,
    const uint32_t* __restrict__ gt_planes, int64_t gt_plane_words, const int32_t* __restrict__ gt_cat_off,
    const int32_t* __restrict__ gt_pos, const int32_t* __restrict__ sup, int n_sup, int K, int metric, MatchParams P,
    smb_coco_out_t* __restrict__ out, int64_t n_out, double* __restrict__ iou_ws, uint8_t* __restrict__ gtm_ws,
    int32_t* __restrict__ pos_ws, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_m = (uint64_t*)smem;                 // [kMaxDet] matched bits (v * P.A + a) of the sorted detections
  uint64_t* s_ig = s_m + kMaxDet;                  // [kMaxDet] ignore bits
  int* s_sorted = (int*)(s_ig + kMaxDet);          // [kMaxDet] detection row of rank r
  int* s_start = s_sorted + kMaxDet;               // [K + 1] per category: first entry of s_list
  int* s_list = s_start + K + 1;                   // [det_cap] detections grouped by category, record order inside
  const int b = blockIdx.x, tid = threadIdx.x;
  const smb_coco_img_t im = imgs[b];
  const int nd = min(max(im.n_det, 0), det_cap);
  const smb_coco_det_t* drow = dets + (size_t)b * det_cap;
  const int32_t* goff = gt_cat_off + (size_t)b * (K + 1);
  const int H = max(im.h, 0), gpitch = max(im.gt_pitch, 0), dpitch = max(im.det_pitch, 0);
  const int base = min(max(goff[0], 0), n_gt), Gi = min(max(goff[K], base), n_gt) - base;
  int32_t* pos_row = pos_ws + base;
  int32_t* pos_cat = pos_ws + n_gt + base;
  auto out_row = [&](int j) -> smb_coco_out_t* {
    const int64_t o = im.out_off + j;
    return (o >= 0 && o < n_out) ? out + o : nullptr;
  };
  for (int j = tid; j < det_cap; j += kThreads) {
    smb_coco_out_t* o = out_row(j);
    if (o) { o->score = 0; o->image_id = im.image_id; o->matched = 0; o->ignored = 0; o->cat = K; o->rank = -1; }
  }
  for (int p = tid; p < Gi; p += kThreads) pos_row[p] = -1;
  if (tid == 0) {
    for (int k = 0; k <= K; ++k) s_start[k] = 0;
    for (int j = 0; j < nd; ++j) {
      const int c = drow[j].cat;
      if (c >= 0 && c < K) s_start[c + 1]++;
    }
    for (int k = 0; k < K; ++k) s_start[k + 1] += s_start[k];
    for (int j = 0; j < nd; ++j) {
      const int c = drow[j].cat;
      if (c >= 0 && c < K) s_list[s_start[c]++] = j;
    }
    for (int k = K; k > 0; --k) s_start[k] = s_start[k - 1];
    s_start[0] = 0;
  }
  __syncthreads();
  // ---- the image's ground truths in annotation order: row and category of position p
  for (int k = 0; k < K; ++k) {
    const int g0 = min(max(goff[k], base), base + Gi), g1 = min(max(goff[k + 1], g0), base + Gi);
    for (int r = g0 + tid; r < g1; r += kThreads) {
      const int p = gt_pos[r];
      if (p < 0 || p >= Gi) { atomicOr(status, SMB_COCO_ANALYSIS_RANGE); continue; }
      pos_row[p] = r;
      pos_cat[p] = k;
    }
  }
  for (int k = tid; k < K; k += kThreads)
    if (sup[k] < 0 || sup[k] >= n_sup) atomicOr(status, SMB_COCO_ANALYSIS_RANGE);
  __syncthreads();
  for (int p = tid; p < Gi; p += kThreads)
    if (pos_row[p] < 0) atomicOr(status, SMB_COCO_ANALYSIS_RANGE);  // a position no row holds (or two rows share)
  for (int k = 0; k < K; ++k) {
    const int l0 = s_start[k], n = s_start[k + 1] - l0;
    if (n == 0) continue;                          // no rows; npig comes from the plain evaluation
    const int D = min(n, P.max_det);
    for (int i = tid; i < n; i += kThreads) {
      const int j = s_list[l0 + i];
      const double s = drow[j].score[metric];
      const int oj = drow[j].order;
      int r = 0;
      for (int q = 0; q < n; ++q) {
        const int jq = s_list[l0 + q];
        const double sq = drow[jq].score[metric];
        const int oq = drow[jq].order;
        r += (sq > s) || (sq == s && (oq < oj || (oq == oj && jq < j)));
      }
      if (r < P.max_det) s_sorted[r] = j;
    }
    for (int i = tid; i < D; i += kThreads) { s_m[i] = 0; s_ig[i] = 0; }
    __syncthreads();
    double* ious = iou_ws + (size_t)kMaxDet * base;
    iou_matrix(metric, D, Gi, drow, s_sorted, gts,
               [&](int g) {
                 const int r = pos_row[g];
                 return make_int2(r, r < 0 ? 1 : (pos_cat[g] == k ? gts[r].crowd : 1));
               },
               H, dpitch, gpitch, det_planes, det_plane_words, gt_planes, gt_plane_words, ious);
    __syncthreads();
    const int sup_k = sup[k];
    const int v = tid / P.A;
    smb_match::greedy_match(
        tid, D, Gi, ious, gtm_ws + (size_t)P.T * P.A * base, P,
        [&](int g) {
          const int r = pos_row[g];
          if (r < 0) return smb_match::MatchGt{0.0, 0, 1, 1};
          const int c = pos_cat[g];
          const smb_coco_gt_t& gr = gts[r];
          const bool own = c == k;
          const bool in_set = own || v == 1 || sup[c] == sup_k;
          return smb_match::MatchGt{gr.area, gr.id, own ? gr.crowd : 1, in_set ? 0 : 1};
        },
        [&](int d) {
          const smb_coco_det_t& dr = drow[s_sorted[d]];
          return metric == 0 ? dr.area_box : (double)dr.area_mask;
        },
        nullptr, s_m, s_ig);
    __syncthreads();
    for (int r = tid; r < D; r += kThreads) {
      const int j = s_sorted[r];
      smb_coco_out_t* o = out_row(j);
      if (o) {
        o->score = drow[j].score[metric];
        o->matched = s_m[r];
        o->ignored = s_ig[r];
        o->cat = k;
        o->rank = r;
      } else {
        atomicOr(status, SMB_COCO_CAPACITY);
      }
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ 2d: accumulate
// What accumulate reads of the Params: A area ranges, M maxDets, R recall thresholds (rec_thr, unless the launch passes
// them as a device array).
struct AccParams {
  int A, M, R;
  int max_dets[SMB_COCO_MAX_M];
  double rec_thr[kR];
};

// grid (K, A * M, T)
__global__ void __launch_bounds__(kThreads) accumulate_kernel(
    const smb_coco_out_t* __restrict__ rows, const int32_t* __restrict__ cat_off, int64_t n_rows, int K,
    const int* __restrict__ npig_in, const double* __restrict__ rec_thr_dev, AccParams P, double* __restrict__ precision,
    double* __restrict__ recall, double* __restrict__ scores) {
  __shared__ int s_wi[kWarps];
  __shared__ double s_wd[kWarps];
  __shared__ double s_q[kR], s_ss[kR];
  const int A = P.A, M = P.M, R = P.R;
  const int k = blockIdx.x, a = blockIdx.y / M, mi = blockIdx.y % M, t = blockIdx.z, tid = threadIdx.x;
  const int max_det = P.max_dets[mi];
  auto rec_thr = [&](int r) { return rec_thr_dev ? rec_thr_dev[r] : P.rec_thr[r]; };
  const int64_t s0 = min(max((int64_t)cat_off[k], (int64_t)0), n_rows);
  const int64_t s1 = min(max((int64_t)cat_off[k + 1], s0), n_rows);
  const uint64_t bit = 1ull << (t * A + a);
  const int npig = npig_in[k * A + a];
  auto p_idx = [&](int r) { return ((((size_t)t * R + r) * K + k) * A + a) * M + mi; };
  const size_t r_idx = (((size_t)t * K + k) * A + a) * M + mi;
  if (npig <= 0) {                                 // no ground truth to recall: every entry stays -1
    for (int r = tid; r < R; r += kThreads) { precision[p_idx(r)] = -1.0; scores[p_idx(r)] = -1.0; }
    if (tid == 0) recall[r_idx] = -1.0;
    return;
  }
  for (int r = tid; r < R; r += kThreads) { s_q[r] = 0.0; s_ss[r] = 0.0; }
  // ---- totals: included detections (rank < maxDet), tp, fp
  int nd = 0, tp_tot = 0, fp_tot = 0;
  for (int64_t base = s0; base < s1; base += kThreads) {
    const int64_t e = base + tid;
    int inc = 0, tpf = 0, fpf = 0;
    if (e < s1) {
      const smb_coco_out_t& o = rows[e];
      inc = o.rank >= 0 && o.rank < max_det;
      const bool ig = o.ignored & bit, m = o.matched & bit;
      tpf = inc && m && !ig;
      fpf = inc && !m && !ig;
    }
    int tot;
    smb::cta_inclusive_scan<kThreads>(inc, smb::Sum(), s_wi, &tot); nd += tot;
    smb::cta_inclusive_scan<kThreads>(tpf, smb::Sum(), s_wi, &tot); tp_tot += tot;
    smb::cta_inclusive_scan<kThreads>(fpf, smb::Sum(), s_wi, &tot); fp_tot += tot;
  }
  const double dn = (double)npig;
  if (tid == 0) recall[r_idx] = nd ? __ddiv_rn((double)tp_tot, dn) : 0.0;
  // ---- right to left: cumulative counts from the suffix sums, the precision envelope as a suffix maximum, and for
  // every recall threshold the first detection whose recall reaches it (searchsorted 'left')
  int c_inc = 0, c_tp = 0, c_fp = 0;               // counts strictly after the current chunk
  double c_max = -1.0;
  for (int64_t base = 0; base < s1 - s0; base += kThreads) {
    const int64_t e = s1 - 1 - (base + tid);
    int inc = 0, tpf = 0, fpf = 0;
    double score = 0.0;
    if (e >= s0) {
      const smb_coco_out_t& o = rows[e];
      inc = o.rank >= 0 && o.rank < max_det;
      const bool ig = o.ignored & bit, m = o.matched & bit;
      tpf = inc && m && !ig;
      fpf = inc && !m && !ig;
      score = o.score;
    }
    int ti, tt, tf;
    const int si = smb::cta_inclusive_scan<kThreads>(inc, smb::Sum(), s_wi, &ti) + c_inc;
    const int st = smb::cta_inclusive_scan<kThreads>(tpf, smb::Sum(), s_wi, &tt) + c_tp;
    const int sf = smb::cta_inclusive_scan<kThreads>(fpf, smb::Sum(), s_wi, &tf) + c_fp;
    const int tp = tp_tot - (st - tpf), fp = fp_tot - (sf - fpf);   // cumulative counts up to and including e
    double pr = -1.0;
    if (inc) pr = __ddiv_rn((double)tp, __dadd_rn((double)(fp + tp), 2.220446049250313e-16));   // + np.spacing(1)
    double tm;
    double env = smb::cta_inclusive_scan<kThreads>(pr, smb::Max(), s_wd, &tm);
    env = env > c_max ? env : c_max;
    if (inc) {
      const bool first = (nd - si) == 0;
      const double rc = __ddiv_rn((double)tp, dn);
      const double rc_prev = first ? -INFINITY : __ddiv_rn((double)(tp - tpf), dn);
      if (rc > rc_prev) {
        for (int r = 0; r < R; ++r) {
          const double x = rec_thr(r);
          if (rc_prev < x && x <= rc) { s_q[r] = env; s_ss[r] = score; }
        }
      }
    }
    c_inc += ti; c_tp += tt; c_fp += tf;
    c_max = c_max > tm ? c_max : tm;
  }
  __syncthreads();
  // searchsorted past the last detection raises IndexError in pycocotools, which leaves that recall threshold and every
  // later one at 0 (with ascending thresholds they are exactly the ones no detection reaches)
  if (tid == 0) {
    const double rc_last = nd ? __ddiv_rn((double)tp_tot, dn) : -INFINITY;
    int r0 = 0;
    while (r0 < R && rec_thr(r0) <= rc_last) ++r0;
    for (int r = r0; r < R; ++r) { s_q[r] = 0.0; s_ss[r] = 0.0; }
  }
  __syncthreads();
  for (int r = tid; r < R; r += kThreads) { precision[p_idx(r)] = s_q[r]; scores[p_idx(r)] = s_ss[r]; }
}

// ------------------------------------------------------------------------------------------------ host rasterizer
// pycocotools maskApi.c rleFrPoly: the run lengths of one polygon (k vertices) in an h x w canvas.
std::vector<uint32_t> poly_counts(const double* xy, int k, int h, int w) {
  const double scale = 5;
  std::vector<int> x(k + 1), y(k + 1);
  for (int j = 0; j < k; ++j) x[j] = (int)(scale * xy[j * 2 + 0] + .5);
  for (int j = 0; j < k; ++j) y[j] = (int)(scale * xy[j * 2 + 1] + .5);
  if (k > 0) { x[k] = x[0]; y[k] = y[0]; }
  std::vector<int> u, v;
  for (int j = 0; j < k; ++j) {
    int xs = x[j], xe = x[j + 1], ys = y[j], ye = y[j + 1];
    const int dx = abs(xe - xs), dy = abs(ys - ye);
    const bool flip = (dx >= dy && xs > xe) || (dx < dy && ys > ye);
    if (flip) { std::swap(xs, xe); std::swap(ys, ye); }
    if (dx == 0 && dy == 0) {                      // s = 0/0 = NaN: pycocotools stores (int)NaN, INT_MIN on x86-64
      u.push_back(xs);
      v.push_back(INT_MIN);
      continue;
    }
    const double s = dx >= dy ? (double)(ye - ys) / dx : (double)(xe - xs) / dy;
    if (dx >= dy) {
      for (int d = 0; d <= dx; ++d) {
        const int t = flip ? dx - d : d;
        u.push_back(t + xs);
        v.push_back((int)(ys + s * t + .5));
      }
    } else {
      for (int d = 0; d <= dy; ++d) {
        const int t = flip ? dy - d : d;
        v.push_back(t + ys);
        u.push_back((int)(xs + s * t + .5));
      }
    }
  }
  std::vector<uint32_t> a;
  for (size_t j = 1; j < u.size(); ++j) {
    if (u[j] == u[j - 1]) continue;
    double xd = (double)(u[j] < u[j - 1] ? u[j] : u[j] - 1);
    xd = (xd + .5) / scale - .5;
    if (floor(xd) != xd || xd < 0 || xd > (double)(w - 1)) continue;
    double yd = (double)(v[j] < v[j - 1] ? v[j] : v[j - 1]);
    yd = (yd + .5) / scale - .5;
    if (yd < 0) yd = 0; else if (yd > h) yd = h;
    yd = ceil(yd);
    a.push_back((uint32_t)((int)xd * h + (int)yd));
  }
  a.push_back((uint32_t)h * (uint32_t)w);
  std::sort(a.begin(), a.end());
  uint32_t p = 0;
  for (auto& e : a) { const uint32_t t = e; e -= p; p = t; }
  std::vector<uint32_t> b;
  size_t j = 0;
  b.push_back(a[j++]);
  while (j < a.size()) {
    if (a[j] > 0) {
      b.push_back(a[j++]);
    } else {
      ++j;
      if (j < a.size()) b.back() += a[j++];
    }
  }
  return b;
}

// OR the mask of column-major run lengths into a bit plane; -1 if the runs do not cover exactly h * w pixels.
int or_runs(const uint32_t* cnts, int n, int h, int w, uint32_t* plane, int pitch) {
  uint64_t pos = 0;
  const uint64_t total = (uint64_t)h * w;
  for (int i = 0; i < n; ++i) {
    const uint64_t end = pos + cnts[i];
    if (end > total) return -1;
    if (i & 1) {
      for (uint64_t q = pos; q < end; ++q) {
        const int x = (int)(q / h), y = (int)(q % h);
        plane[(size_t)y * pitch + (x >> 5)] |= 1u << (x & 31);
      }
    }
    pos = end;
  }
  return pos == total ? 0 : -1;
}

}  // namespace

extern "C" int smb_coco_poly_counts(const double* host_xy, int k, int h, int w, uint32_t* host_counts, int cap, int* host_n) {
  SMB_CHECK_ARG(k >= 0 && h >= 0 && w >= 0 && (k == 0 || host_xy) && host_n, "smb_coco_poly_counts: bad arguments");
  const std::vector<uint32_t> c = poly_counts(host_xy, k, h, w);
  *host_n = (int)c.size();
  if ((int)c.size() <= cap && host_counts) memcpy(host_counts, c.data(), c.size() * sizeof(uint32_t));
  return SMB_OK;
}

extern "C" int smb_coco_poly_to_bits(const double* host_xy, int k, int h, int w, uint32_t* host_plane, int pitch) {
  SMB_CHECK_ARG(k >= 0 && h >= 0 && w >= 0 && (k == 0 || host_xy) && host_plane && pitch >= (w + 31) / 32,
                "smb_coco_poly_to_bits: bad arguments");
  const std::vector<uint32_t> c = poly_counts(host_xy, k, h, w);
  return or_runs(c.data(), (int)c.size(), h, w, host_plane, pitch) == 0 ? SMB_OK : SMB_EINVAL;
}

extern "C" int smb_coco_rle_to_bits(const uint32_t* host_counts, int n, int h, int w, uint32_t* host_plane, int pitch) {
  SMB_CHECK_ARG(n >= 0 && h >= 0 && w >= 0 && (n == 0 || host_counts) && host_plane && pitch >= (w + 31) / 32,
                "smb_coco_rle_to_bits: bad arguments");
  SMB_CHECK_ARG(or_runs(host_counts, n, h, w, host_plane, pitch) == 0,
                "smb_coco_rle_to_bits: the runs do not cover the %d x %d canvas", h, w);
  return SMB_OK;
}

extern "C" int smb_coco_rle_from_string(const char* host_s, int len, uint32_t* host_counts, int cap, int* host_n) {
  SMB_CHECK_ARG(len >= 0 && (len == 0 || host_s) && host_n, "smb_coco_rle_from_string: bad arguments");
  // maskApi.c rleFrString: 5 bits per character, continuation bit 0x20, sign bit 0x10 on the last, deltas from m > 2
  int m = 0, p = 0;
  std::vector<uint32_t> cnts;
  while (p < len) {
    long long x = 0;
    int k = 0, more = 1;
    while (more) {
      SMB_CHECK_ARG(p < len && k < 7, "smb_coco_rle_from_string: truncated or overlong value at byte %d", p);
      const int c = host_s[p] - 48;
      SMB_CHECK_ARG(c >= 0 && c < 64, "smb_coco_rle_from_string: byte %d is not an RLE character", p);
      x |= (long long)(c & 0x1f) << (5 * k);
      more = c & 0x20;
      ++p;
      ++k;
      if (!more && (c & 0x10)) x |= -1LL << (5 * k);
    }
    if (m > 2) x += (long long)cnts[m - 2];
    SMB_CHECK_ARG(x >= 0 && x <= 0xffffffffLL, "smb_coco_rle_from_string: count %lld out of range", x);
    cnts.push_back((uint32_t)x);
    ++m;
  }
  *host_n = m;
  if (m <= cap && host_counts && m) memcpy(host_counts, cnts.data(), m * sizeof(uint32_t));
  return SMB_OK;
}

extern "C" int smb_coco_plane_stats(const uint32_t* host_plane, int h, int w, int pitch, int32_t* host_stats5) {
  SMB_CHECK_ARG(host_plane && host_stats5 && h >= 0 && w >= 0 && pitch >= (w + 31) / 32, "smb_coco_plane_stats: bad arguments");
  const int words = (w + 31) / 32;
  const uint32_t last = (w & 31) ? ((1u << (w & 31)) - 1u) : 0xffffffffu;
  int area = 0, r0 = INT_MAX, r1 = -1, w0 = INT_MAX, w1 = -1;
  for (int y = 0; y < h; ++y)
    for (int x = 0; x < words; ++x) {
      uint32_t v = host_plane[(size_t)y * pitch + x];
      if (x == words - 1) v &= last;
      if (v) {
        area += __builtin_popcount(v);
        r0 = std::min(r0, y); r1 = std::max(r1, y); w0 = std::min(w0, x); w1 = std::max(w1, x);
      }
    }
  host_stats5[0] = area;
  if (area) { host_stats5[1] = r0; host_stats5[2] = r1 + 1; host_stats5[3] = w0; host_stats5[4] = w1 + 1; }
  else host_stats5[1] = host_stats5[2] = host_stats5[3] = host_stats5[4] = 0;
  return SMB_OK;
}

// ------------------------------------------------------------------------------------------------ device entry points
namespace {

int launch_match(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap, const uint32_t* det_planes,
                 int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt, const uint32_t* gt_planes,
                 int64_t gt_plane_words, const int32_t* gt_cat_off, int K, int metric, const MatchParams& P,
                 smb_coco_out_t* out, int64_t n_out, int* npig, int* status, void* workspace, smb_stream_t stream) {
  double* iou_ws = (double*)workspace;
  uint8_t* gtm_ws = (uint8_t*)workspace + smb::align_up((size_t)n_gt * kMaxDet * sizeof(double), 256);
  const size_t smem = 2 * kMaxDet * sizeof(uint64_t) + (size_t)(kMaxDet + K + 1 + det_cap) * sizeof(int);
  match_kernel<<<n_img, kThreads, smem, (cudaStream_t)stream>>>(imgs, dets, det_cap, det_planes, det_plane_words, gts, n_gt,
                                                               gt_planes, gt_plane_words, gt_cat_off, K, metric, P, out, n_out,
                                                               npig, iou_ws, gtm_ws, status);
  SMB_LAUNCH_OK("match_kernel");
  return SMB_OK;
}

}  // namespace

extern "C" int smb_coco_det_from_record_dev(const float* det, const int64_t* labels, const int* count, const float* mask_scores,
                                            const uint32_t* mask_bits, int N, int max_num, int cap_h, int words,
                                            const smb_img_geom_t* geom, const int32_t* label_cat, int num_labels,
                                            int benchmark, smb_coco_det_t* rows, smb_coco_img_t* imgs, int* status,
                                            smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && max_num >= 1 && cap_h >= 0 && words >= 0 && num_labels >= 0,
                "smb_coco_det_from_record_dev: bad sizes (N %d, max_num %d, cap_h %d, words %d)", N, max_num, cap_h, words);
  if (N == 0) return SMB_OK;
  SMB_CHECK_ARG(det && labels && count && mask_bits && geom && (label_cat || num_labels == 0) && rows && imgs && status,
                "smb_coco_det_from_record_dev: null pointer");
  det_from_record_kernel<<<N, kThreads, 0, (cudaStream_t)stream>>>(det, labels, count, mask_scores, mask_bits, max_num, cap_h,
                                                                   words, geom, label_cat, num_labels, benchmark, rows, imgs,
                                                                   status);
  SMB_LAUNCH_OK("det_from_record_kernel");
  return SMB_OK;
}

extern "C" size_t smb_coco_match_workspace_bytes(int n_gt) { return smb_match::match_workspace_bytes(n_gt); }

extern "C" int smb_coco_match_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                                  const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts, int n_gt,
                                  const uint32_t* gt_planes, int64_t gt_plane_words, const int32_t* gt_cat_off, int K,
                                  int metric, const double* host_iou_thr, const double* host_area_rng,
                                  smb_coco_out_t* out, int64_t n_out, int* npig, int* status, void* workspace,
                                  size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n_img >= 0 && det_cap >= 1 && det_cap <= SMB_COCO_DET_CAP && K >= 1 && K <= SMB_COCO_MAX_CATS && n_gt >= 0 &&
                    (metric == 0 || metric == 1) && n_out >= 0 && det_plane_words >= 0 && gt_plane_words >= 0,
                "smb_coco_match_dev: bad sizes (n_img %d, det_cap %d, K %d, n_gt %d, metric %d)", n_img, det_cap, K, n_gt,
                metric);
  SMB_CHECK_ARG(host_iou_thr && host_area_rng, "smb_coco_match_dev: null thresholds");
  if (n_img == 0) return SMB_OK;
  SMB_CHECK_ARG(imgs && dets && gt_cat_off && out && npig && status && (gts || n_gt == 0) && workspace,
                "smb_coco_match_dev: null pointer");
  SMB_CHECK_ARG(metric == 0 || (det_planes && (gt_planes || n_gt == 0)), "smb_coco_match_dev: segm needs the planes");
  SMB_CHECK_ARG(workspace_bytes >= smb_coco_match_workspace_bytes(n_gt), "smb_coco_match_dev: workspace of %zu bytes, %zu needed",
                workspace_bytes, smb_coco_match_workspace_bytes(n_gt));
  return launch_match(imgs, n_img, dets, det_cap, det_planes, det_plane_words, gts, n_gt, gt_planes, gt_plane_words,
                      gt_cat_off, K, metric, smb_match::default_params(host_iou_thr, host_area_rng), out, n_out, npig, status,
                      workspace, stream);
}

extern "C" int smb_coco_accumulate_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K,
                                       const int* npig, const double* rec_thr, const int* host_max_dets3, double* precision,
                                       double* recall, double* scores, smb_stream_t stream) {
  SMB_CHECK_ARG(n_rows >= 0 && K >= 1 && K <= SMB_COCO_MAX_CATS, "smb_coco_accumulate_dev: bad sizes (n_rows %lld, K %d)",
                (long long)n_rows, K);
  SMB_CHECK_ARG(cat_off && npig && rec_thr && host_max_dets3 && precision && recall && scores && (rows || n_rows == 0),
                "smb_coco_accumulate_dev: null pointer");
  AccParams P;
  P.A = kA;
  P.M = 3;
  P.R = kR;
  for (int m = 0; m < 3; ++m) P.max_dets[m] = host_max_dets3[m];
  accumulate_kernel<<<dim3(K, kA * 3, kT), kThreads, 0, (cudaStream_t)stream>>>(rows, cat_off, n_rows, K, npig, rec_thr, P,
                                                                               precision, recall, scores);
  SMB_LAUNCH_OK("accumulate_kernel");
  return SMB_OK;
}

extern "C" size_t smb_coco_analysis_workspace_bytes(int n_gt) {
  if (n_gt < 0) return 0;
  return smb_match::match_workspace_bytes(n_gt, 2 * kA) + smb::align_up((size_t)n_gt * 2 * sizeof(int32_t), 256);
}

extern "C" int smb_coco_analysis_match_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                                           const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts,
                                           int n_gt, const uint32_t* gt_planes, int64_t gt_plane_words,
                                           const int32_t* gt_cat_off, const int32_t* gt_pos, const int32_t* sup,
                                           int n_sup, int K, int metric, const double* host_area_rng,
                                           smb_coco_out_t* out, int64_t n_out, int* status, void* workspace,
                                           size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n_img >= 0 && det_cap >= 1 && det_cap <= SMB_COCO_DET_CAP && K >= 1 && K <= SMB_COCO_MAX_CATS && n_gt >= 0 &&
                    n_sup >= 1 && (metric == 0 || metric == 1) && n_out >= 0 && det_plane_words >= 0 && gt_plane_words >= 0,
                "smb_coco_analysis_match_dev: bad sizes (n_img %d, det_cap %d, K %d, n_gt %d, n_sup %d, metric %d)", n_img,
                det_cap, K, n_gt, n_sup, metric);
  SMB_CHECK_ARG(host_area_rng, "smb_coco_analysis_match_dev: null area ranges");
  if (n_img == 0) return SMB_OK;
  SMB_CHECK_ARG(imgs && dets && gt_cat_off && sup && out && status && ((gts && gt_pos) || n_gt == 0) && workspace,
                "smb_coco_analysis_match_dev: null pointer");
  SMB_CHECK_ARG(metric == 0 || (det_planes && (gt_planes || n_gt == 0)), "smb_coco_analysis_match_dev: segm needs the planes");
  SMB_CHECK_ARG(workspace_bytes >= smb_coco_analysis_workspace_bytes(n_gt),
                "smb_coco_analysis_match_dev: workspace of %zu bytes, %zu needed", workspace_bytes,
                smb_coco_analysis_workspace_bytes(n_gt));
  MatchParams P;                                   // variants Sim / Oth as two "thresholds" of .1; maxDets [100]
  P.T = 2;
  P.A = kA;
  P.max_det = kMaxDet;
  P.iou_thr[0] = P.iou_thr[1] = 0.1;
  for (int a = 0; a < kA; ++a) { P.area_rng[a][0] = host_area_rng[2 * a]; P.area_rng[a][1] = host_area_rng[2 * a + 1]; }
  const size_t match_ws = smb_match::match_workspace_bytes(n_gt, 2 * kA);
  double* iou_ws = (double*)workspace;
  uint8_t* gtm_ws = (uint8_t*)workspace + smb::align_up((size_t)n_gt * kMaxDet * sizeof(double), 256);
  int32_t* pos_ws = (int32_t*)((uint8_t*)workspace + match_ws);
  const size_t smem = 2 * kMaxDet * sizeof(uint64_t) + (size_t)(kMaxDet + K + 1 + det_cap) * sizeof(int);
  analysis_match_kernel<<<n_img, kThreads, smem, (cudaStream_t)stream>>>(
      imgs, dets, det_cap, det_planes, det_plane_words, gts, n_gt, gt_planes, gt_plane_words, gt_cat_off, gt_pos, sup, n_sup,
      K, metric, P, out, n_out, iou_ws, gtm_ws, pos_ws, status);
  SMB_LAUNCH_OK("analysis_match_kernel");
  return SMB_OK;
}

extern "C" int smb_coco_params_check(const smb_coco_params_t* p) {
  SMB_CHECK_ARG(p, "smb_coco_params_check: null Params");
  SMB_CHECK_ARG(p->T >= 1 && p->A >= 1 && p->T * p->A <= SMB_COCO_MAX_TA,
                "Params: %d IoU thresholds x %d area ranges; 1 <= T, 1 <= A and T * A <= %d (one uint64 of bits per row)",
                p->T, p->A, SMB_COCO_MAX_TA);
  SMB_CHECK_ARG(p->M >= 1 && p->M <= SMB_COCO_MAX_M, "Params: %d maxDets; 1 to %d", p->M, SMB_COCO_MAX_M);
  for (int m = 0; m < p->M; ++m) {
    SMB_CHECK_ARG(p->max_dets[m] >= 1 && p->max_dets[m] <= SMB_COCO_MAX_DET, "Params: maxDet %d outside [1, %d]",
                  p->max_dets[m], SMB_COCO_MAX_DET);
    // COCOeval.evaluate() sorts maxDets before anything reads them; the last one is the number of detections kept
    SMB_CHECK_ARG(m == 0 || p->max_dets[m] >= p->max_dets[m - 1], "Params: maxDets must be ascending (%d after %d)",
                  p->max_dets[m], p->max_dets[m - 1]);
  }
  SMB_CHECK_ARG(p->R >= 1 && p->R <= SMB_COCO_R, "Params: %d recall thresholds; 1 to %d", p->R, SMB_COCO_R);
  for (int t = 0; t < p->T; ++t) SMB_CHECK_ARG(!isnan(p->iou_thr[t]), "Params: IoU threshold %d is NaN", t);
  for (int a = 0; a < p->A; ++a)
    SMB_CHECK_ARG(!isnan(p->area_rng[a][0]) && !isnan(p->area_rng[a][1]), "Params: area range %d has a NaN", a);
  for (int r = 0; r < p->R; ++r) SMB_CHECK_ARG(!isnan(p->rec_thr[r]), "Params: recall threshold %d is NaN", r);
  return SMB_OK;
}

extern "C" size_t smb_coco_match_params_workspace_bytes(int n_gt, const smb_coco_params_t* p) {
  if (!p || smb_coco_params_check(p) != SMB_OK) return 0;
  return smb_match::match_workspace_bytes(n_gt, p->T * p->A);
}

extern "C" int smb_coco_match_params_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                                         const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts,
                                         int n_gt, const uint32_t* gt_planes, int64_t gt_plane_words,
                                         const int32_t* gt_cat_off, int K, int metric, const smb_coco_params_t* p,
                                         smb_coco_out_t* out, int64_t n_out, int* npig, int* status, void* workspace,
                                         size_t workspace_bytes, smb_stream_t stream) {
  const int rc = smb_coco_params_check(p);
  if (rc != SMB_OK) return rc;
  SMB_CHECK_ARG(n_img >= 0 && det_cap >= 1 && det_cap <= SMB_COCO_DET_CAP && K >= 1 && K <= SMB_COCO_MAX_CATS && n_gt >= 0 &&
                    (metric == 0 || metric == 1) && n_out >= 0 && det_plane_words >= 0 && gt_plane_words >= 0,
                "smb_coco_match_params_dev: bad sizes (n_img %d, det_cap %d, K %d, n_gt %d, metric %d)", n_img, det_cap, K,
                n_gt, metric);
  if (n_img == 0) return SMB_OK;
  SMB_CHECK_ARG(imgs && dets && gt_cat_off && out && npig && status && (gts || n_gt == 0) && workspace,
                "smb_coco_match_params_dev: null pointer");
  SMB_CHECK_ARG(metric == 0 || (det_planes && (gt_planes || n_gt == 0)), "smb_coco_match_params_dev: segm needs the planes");
  const size_t need = smb_match::match_workspace_bytes(n_gt, p->T * p->A);
  SMB_CHECK_ARG(workspace_bytes >= need, "smb_coco_match_params_dev: workspace of %zu bytes, %zu needed", workspace_bytes,
                need);
  MatchParams P;
  P.T = p->T;
  P.A = p->A;
  P.max_det = p->max_dets[p->M - 1];
  for (int t = 0; t < p->T; ++t) P.iou_thr[t] = p->iou_thr[t];
  for (int a = 0; a < p->A; ++a) { P.area_rng[a][0] = p->area_rng[a][0]; P.area_rng[a][1] = p->area_rng[a][1]; }
  return launch_match(imgs, n_img, dets, det_cap, det_planes, det_plane_words, gts, n_gt, gt_planes, gt_plane_words,
                      gt_cat_off, K, metric, P, out, n_out, npig, status, workspace, stream);
}

extern "C" int smb_coco_accumulate_params_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K,
                                              const int* npig, const smb_coco_params_t* p, double* precision,
                                              double* recall, double* scores, smb_stream_t stream) {
  const int rc = smb_coco_params_check(p);
  if (rc != SMB_OK) return rc;
  SMB_CHECK_ARG(n_rows >= 0 && K >= 1 && K <= SMB_COCO_MAX_CATS,
                "smb_coco_accumulate_params_dev: bad sizes (n_rows %lld, K %d)", (long long)n_rows, K);
  SMB_CHECK_ARG(cat_off && npig && precision && recall && scores && (rows || n_rows == 0),
                "smb_coco_accumulate_params_dev: null pointer");
  AccParams P;
  P.A = p->A;
  P.M = p->M;
  P.R = p->R;
  for (int m = 0; m < p->M; ++m) P.max_dets[m] = p->max_dets[m];
  for (int r = 0; r < p->R; ++r) P.rec_thr[r] = p->rec_thr[r];
  accumulate_kernel<<<dim3(K, p->A * p->M, p->T), kThreads, 0, (cudaStream_t)stream>>>(rows, cat_off, n_rows, K, npig,
                                                                                      nullptr, P, precision, recall, scores);
  SMB_LAUNCH_OK("accumulate_kernel");
  return SMB_OK;
}

extern "C" int smb_coco_params2_check(const smb_coco_params2_t* p) {
  SMB_CHECK_ARG(p, "smb_coco_params2_check: null Params");
  SMB_CHECK_ARG(p->use_cats == 0 || p->use_cats == 1, "Params: useCats %d; 0 or 1", p->use_cats);
  SMB_CHECK_ARG(p->T >= 1 && p->A >= 1 && p->T * p->A <= SMB_COCO_MAX_TA,
                "Params: %d IoU thresholds x %d area ranges; 1 <= T, 1 <= A and T * A <= %d (one uint64 of bits per row)",
                p->T, p->A, SMB_COCO_MAX_TA);
  SMB_CHECK_ARG(p->M >= 1 && p->M <= SMB_COCO_MAX_M, "Params: %d maxDets; 1 to %d", p->M, SMB_COCO_MAX_M);
  for (int m = 0; m < p->M; ++m) {
    SMB_CHECK_ARG(p->max_dets[m] >= 1 && p->max_dets[m] <= SMB_COCO_MAX_DET2, "Params: maxDet %d outside [1, %d]",
                  p->max_dets[m], SMB_COCO_MAX_DET2);
    SMB_CHECK_ARG(m == 0 || p->max_dets[m] >= p->max_dets[m - 1], "Params: maxDets must be ascending (%d after %d)",
                  p->max_dets[m], p->max_dets[m - 1]);
  }
  SMB_CHECK_ARG(p->R >= 1 && p->R <= SMB_COCO_R, "Params: %d recall thresholds; 1 to %d", p->R, SMB_COCO_R);
  for (int t = 0; t < p->T; ++t) SMB_CHECK_ARG(!isnan(p->iou_thr[t]), "Params: IoU threshold %d is NaN", t);
  for (int a = 0; a < p->A; ++a)
    SMB_CHECK_ARG(!isnan(p->area_rng[a][0]) && !isnan(p->area_rng[a][1]), "Params: area range %d has a NaN", a);
  for (int r = 0; r < p->R; ++r) SMB_CHECK_ARG(!isnan(p->rec_thr[r]), "Params: recall threshold %d is NaN", r);
  return SMB_OK;
}

extern "C" size_t smb_coco_match_params2_workspace_bytes(int n_gt, const smb_coco_params2_t* p) {
  if (!p || smb_coco_params2_check(p) != SMB_OK) return 0;
  return smb_match::match_workspace_bytes(n_gt, p->T * p->A, p->max_dets[p->M - 1]);
}

extern "C" int smb_coco_match_params2_dev(const smb_coco_img_t* imgs, int n_img, const smb_coco_det_t* dets, int det_cap,
                                          const uint32_t* det_planes, int64_t det_plane_words, const smb_coco_gt_t* gts,
                                          int n_gt, const uint32_t* gt_planes, int64_t gt_plane_words,
                                          const int32_t* gt_cat_off, int K, int metric, const smb_coco_params2_t* p,
                                          smb_coco_out_t* out, int64_t n_out, int* npig, int* status, void* workspace,
                                          size_t workspace_bytes, smb_stream_t stream) {
  const int rc = smb_coco_params2_check(p);
  if (rc != SMB_OK) return rc;
  SMB_CHECK_ARG(n_img >= 0 && det_cap >= 1 && det_cap <= SMB_COCO_DET_CAP && K >= 1 && K <= SMB_COCO_MAX_CATS && n_gt >= 0 &&
                    (metric == 0 || metric == 1) && n_out >= 0 && det_plane_words >= 0 && gt_plane_words >= 0,
                "smb_coco_match_params2_dev: bad sizes (n_img %d, det_cap %d, K %d, n_gt %d, metric %d)", n_img, det_cap, K,
                n_gt, metric);
  if (n_img == 0) return SMB_OK;
  SMB_CHECK_ARG(imgs && dets && gt_cat_off && out && npig && status && (gts || n_gt == 0) && workspace,
                "smb_coco_match_params2_dev: null pointer");
  SMB_CHECK_ARG(metric == 0 || (det_planes && (gt_planes || n_gt == 0)), "smb_coco_match_params2_dev: segm needs the planes");
  const int max_det = p->max_dets[p->M - 1];
  const size_t need = smb_match::match_workspace_bytes(n_gt, p->T * p->A, max_det);
  SMB_CHECK_ARG(workspace_bytes >= need, "smb_coco_match_params2_dev: workspace of %zu bytes, %zu needed", workspace_bytes,
                need);
  MatchParams P;
  P.T = p->T;
  P.A = p->A;
  P.max_det = max_det;
  for (int t = 0; t < p->T; ++t) P.iou_thr[t] = p->iou_thr[t];
  for (int a = 0; a < p->A; ++a) { P.area_rng[a][0] = p->area_rng[a][0]; P.area_rng[a][1] = p->area_rng[a][1]; }
  double* iou_ws = (double*)workspace;
  uint8_t* gtm_ws = (uint8_t*)workspace + smb::align_up((size_t)n_gt * max_det * sizeof(double), 256);
  const size_t smem = match2_smem_bytes(det_cap, K, max_det, p->use_cats);
  if (smem > 48 * 1024)
    SMB_CUDA_OK(cudaFuncSetAttribute(match2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  match2_kernel<<<n_img, kThreads, smem, (cudaStream_t)stream>>>(imgs, dets, det_cap, det_planes, det_plane_words, gts, n_gt,
                                                                gt_planes, gt_plane_words, gt_cat_off, K, metric, p->use_cats,
                                                                P, out, n_out, npig, iou_ws, gtm_ws, status);
  SMB_LAUNCH_OK("match2_kernel");
  return SMB_OK;
}

extern "C" int smb_coco_accumulate_params2_dev(const smb_coco_out_t* rows, int64_t n_rows, const int32_t* cat_off, int K,
                                               const int* npig, const smb_coco_params2_t* p, double* precision,
                                               double* recall, double* scores, smb_stream_t stream) {
  const int rc = smb_coco_params2_check(p);
  if (rc != SMB_OK) return rc;
  SMB_CHECK_ARG(n_rows >= 0 && K >= 1 && K <= SMB_COCO_MAX_CATS,
                "smb_coco_accumulate_params2_dev: bad sizes (n_rows %lld, K %d)", (long long)n_rows, K);
  SMB_CHECK_ARG(cat_off && npig && precision && recall && scores && (rows || n_rows == 0),
                "smb_coco_accumulate_params2_dev: null pointer");
  AccParams P;
  P.A = p->A;
  P.M = p->M;
  P.R = p->R;
  for (int m = 0; m < p->M; ++m) P.max_dets[m] = p->max_dets[m];
  for (int r = 0; r < p->R; ++r) P.rec_thr[r] = p->rec_thr[r];
  accumulate_kernel<<<dim3(K, p->A * p->M, p->T), kThreads, 0, (cudaStream_t)stream>>>(rows, cat_off, n_rows, K, npig,
                                                                                      nullptr, P, precision, recall, scores);
  SMB_LAUNCH_OK("accumulate_kernel");
  return SMB_OK;
}
