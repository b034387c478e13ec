// YouTube-VIS mask AP (the youtubevos pycocotools fork's YTVOSeval, iouType 'segm', default parameters) on the device.
//
//   smb_ytvis_overlap_dev : per frame, each detection's pixel count and its intersection with every ground truth present
//   smb_ytvis_scatter_dev : per frame, the last detection of every object id added into its video's int64 accumulators
//   smb_ytvis_match_dev   : at the end of a video, the sequence IoU from the accumulators and evaluateVid's matching
//
// The sequence IoU sum_f |d_f & g_f| / (sum |d_f| + sum |g_f| - sum |d_f & g_f|) (frames where the object is present)
// is a quotient of integer sums, so the frames are accumulated exactly as they finish and divided once in float64 with
// an explicit _rn intrinsic.  accumulate is COCOeval's (smb_coco_accumulate_dev).
#include <limits.h>

#include "coco_match.cuh"

namespace {

using smb_match::kA;
using smb_match::kMaxDet;
using smb_match::kT;
using smb_match::MatchParams;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

// ------------------------------------------------------------------------------------------------ a: per-frame overlaps
// One CTA per (frame row n, detection j): its threads stride over the plane's words, then over each ground truth's
// overlapping extent, so a frame's planes are read by max_num CTAs at once.
__device__ __forceinline__ void block_reduce5(int v[5], int (*s_red)[5]) {
  const int lid = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int o = 16; o > 0; o >>= 1) {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    v[1] = min(v[1], __shfl_xor_sync(0xffffffffu, v[1], o));
    v[2] = max(v[2], __shfl_xor_sync(0xffffffffu, v[2], o));
    v[3] = min(v[3], __shfl_xor_sync(0xffffffffu, v[3], o));
    v[4] = max(v[4], __shfl_xor_sync(0xffffffffu, v[4], o));
  }
  if (lid == 0)
    for (int i = 0; i < 5; ++i) s_red[warp][i] = v[i];
  __syncthreads();
  for (int w = 0; w < kWarps; ++w) {
    if (w == 0) {
      for (int i = 0; i < 5; ++i) v[i] = s_red[0][i];
    } else {
      v[0] += s_red[w][0];
      v[1] = min(v[1], s_red[w][1]); v[2] = max(v[2], s_red[w][2]);
      v[3] = min(v[3], s_red[w][3]); v[4] = max(v[4], s_red[w][4]);
    }
  }
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) overlap_kernel(const smb_ytvis_frame_t* __restrict__ frames, const int* __restrict__ count,
                                                           int max_num, const smb_ytvis_gt_frame_t* __restrict__ gts, int n_gts,
                                                           int g_max, int32_t* __restrict__ inter, int32_t* __restrict__ area,
                                                           int* __restrict__ status) {
  __shared__ int s_red[kWarps][5];
  const int n = blockIdx.x, j = blockIdx.y, tid = threadIdx.x;
  const smb_ytvis_frame_t f = frames[n];
  const int cnt = min(max(count ? count[n] : f.n_det, 0), max_num);
  const int h = max(f.h, 0), dp = max(f.det_pitch, 0), gp = max(f.gt_pitch, 0);
  const int ow = min(max(f.w, 0), dp * 32);
  const int ow_words = (ow + 31) >> 5;
  const uint32_t last_mask = (ow & 31) ? ((1u << (ow & 31)) - 1u) : 0xffffffffu;
  const int g0 = min(max(f.g0, 0), n_gts);
  const int g1 = min(max(f.n_gt, 0), n_gts - g0) + g0;
  if (j == 0 && tid == 0 && (f.g0 < 0 || f.n_gt < 0 || (int64_t)f.g0 + f.n_gt > n_gts)) atomicOr(status, SMB_YTVIS_RANGE);
  int32_t* in_row = inter + ((size_t)n * max_num + j) * g_max;
  for (int g = tid; g < g_max; g += kThreads) in_row[g] = 0;
  if (j >= cnt) {
    if (tid == 0) area[(size_t)n * max_num + j] = 0;
    return;
  }
  // ---- pixel count and extents over the canvas (maskUtils.area)
  const uint32_t* p = f.det + (int64_t)j * f.det_stride;
  int v[5] = {0, INT_MAX, -1, INT_MAX, -1};      // area, row0, row1, word0, word1
  for (int e = tid; e < h * ow_words; e += kThreads) {
    const int y = e / ow_words, x = e - y * ow_words;
    uint32_t u = p[(size_t)y * dp + x];
    if (x == ow_words - 1) u &= last_mask;
    if (u) { v[0] += __popc(u); v[1] = min(v[1], y); v[2] = max(v[2], y); v[3] = min(v[3], x); v[4] = max(v[4], x); }
  }
  block_reduce5(v, s_red);
  if (tid == 0) area[(size_t)n * max_num + j] = v[0];
  if (v[0] == 0) return;
  // ---- intersections: AND + popcount over the rows and words where both extents overlap
  for (int gi = g0; gi < g1; ++gi) {
    const smb_ytvis_gt_frame_t gr = gts[gi];
    if (gr.g < 0 || gr.g >= g_max) {
      if (tid == 0) atomicOr(status, SMB_YTVIS_GTS);
      continue;
    }
    const int y0 = max(max(v[1], gr.ext[0]), 0), y1 = min(min(v[2] + 1, gr.ext[1]), h);
    const int x0 = max(max(v[3], gr.ext[2]), 0), x1 = min(min(min(v[4] + 1, gr.ext[3]), ow_words), gp);
    const int nx = x1 - x0;
    int c[5] = {0, 0, 0, 0, 0};
    if (nx > 0 && y1 > y0) {
      for (int e = tid; e < (y1 - y0) * nx; e += kThreads) {
        const int y = y0 + e / nx, x = x0 + e % nx;
        uint32_t u = p[(size_t)y * dp + x] & gr.plane[(size_t)y * gp + x];
        if (x == ow_words - 1) u &= last_mask;
        c[0] += __popc(u);
      }
    }
    block_reduce5(c, s_red);
    if (tid == 0) in_row[gr.g] = c[0];
  }
}

// ------------------------------------------------------------------------------------------------ b: scatter by object id
__global__ void __launch_bounds__(128) scatter_kernel(const smb_ytvis_frame_t* __restrict__ frames, const int* __restrict__ count,
                                                      const int32_t* __restrict__ ids, int max_num, const int32_t* __restrict__ inter,
                                                      const int32_t* __restrict__ area, int g_max, int64_t* __restrict__ acc_inter,
                                                      int64_t* __restrict__ acc_area, int32_t* __restrict__ acc_nz, int slots,
                                                      int objects, int* __restrict__ status) {
  const int n = blockIdx.x;
  const smb_ytvis_frame_t f = frames[n];
  if (f.slot < 0) return;
  if (f.slot >= slots) {
    if (threadIdx.x == 0) atomicOr(status, SMB_YTVIS_RANGE);
    return;
  }
  const int cnt = min(max(count ? count[n] : f.n_det, 0), max_num);
  const int32_t* id_row = ids + (size_t)n * max_num;
  for (int j = threadIdx.x; j < cnt; j += blockDim.x) {
    const int id = id_row[j];
    if (id < 0) continue;                          // no object (a lost claim, or an append beyond the tracker's capacity)
    bool last = true;
    for (int q = j + 1; q < cnt && last; ++q) last = id_row[q] != id;
    if (!last) continue;
    if (id >= objects) {
      atomicOr(status, SMB_YTVIS_OBJECTS);
      continue;
    }
    const size_t o = (size_t)f.slot * objects + id;
    const int a = area[(size_t)n * max_num + j];
    if (a) {
      atomicAdd((unsigned long long*)&acc_area[o], (unsigned long long)a);
      atomicAdd(&acc_nz[o], 1);
    }
    const int32_t* in = inter + ((size_t)n * max_num + j) * g_max;
    for (int g = 0; g < g_max; ++g)
      if (in[g]) atomicAdd((unsigned long long*)&acc_inter[o * g_max + g], (unsigned long long)in[g]);
  }
}

// ------------------------------------------------------------------------------------------------ c: sequence match
__global__ void __launch_bounds__(kThreads) seq_match_kernel(
    const smb_ytvis_entry_t* __restrict__ ents, int n_ent, const smb_ytvis_gt_t* __restrict__ gts, int n_gt,
    const int32_t* __restrict__ gt_cat_off, int K, int slot, const int64_t* __restrict__ acc_inter,
    const int64_t* __restrict__ acc_area, const int32_t* __restrict__ acc_nz, int slots, int objects, int g_max,
    int64_t video_id, MatchParams P, smb_coco_out_t* __restrict__ out, int64_t n_out, int* __restrict__ npig,
    double* __restrict__ iou_ws, uint8_t* __restrict__ gtm_ws, int* __restrict__ status) {
  extern __shared__ __align__(16) unsigned char smem[];
  uint64_t* s_m = (uint64_t*)smem;                 // [kMaxDet] matched bits (t * kA + a) of the sorted entries
  uint64_t* s_ig = s_m + kMaxDet;                  // [kMaxDet] ignore bits
  double* s_area = (double*)(s_ig + kMaxDet);      // [kMaxDet] avg_area of the sorted entries
  int* s_sorted = (int*)(s_area + kMaxDet);        // [kMaxDet] entry of rank r
  int* s_start = s_sorted + kMaxDet;               // [K + 1] per category: first entry of s_list
  int* s_list = s_start + K + 1;                   // [n_ent] entries grouped by category, json order inside
  const int tid = threadIdx.x;
  const bool slot_ok = slot >= 0 && slot < slots;
  if (tid == 0 && !slot_ok) atomicOr(status, SMB_YTVIS_RANGE);
  auto obj_row = [&](int e) -> int64_t {           // the entry's accumulator row, -1 when out of range
    const int obj = ents[e].obj;
    return (slot_ok && obj >= 0 && obj < objects) ? (int64_t)slot * objects + obj : -1;
  };
  for (int e = tid; e < n_ent; e += kThreads) {
    if (e < n_out) {
      smb_coco_out_t& o = out[e];
      o.score = 0; o.image_id = video_id; o.matched = 0; o.ignored = 0; o.cat = K; o.rank = -1;
    } else {
      atomicOr(status, SMB_YTVIS_RANGE);
    }
    if (obj_row(e) < 0) atomicOr(status, SMB_YTVIS_OBJECTS);
  }
  if (tid == 0) {
    for (int k = 0; k <= K; ++k) s_start[k] = 0;
    for (int e = 0; e < n_ent; ++e) {
      const int c = ents[e].cat;
      if (c >= 0 && c < K) s_start[c + 1]++;
    }
    for (int k = 0; k < K; ++k) s_start[k + 1] += s_start[k];
    for (int e = 0; e < n_ent; ++e) {
      const int c = ents[e].cat;
      if (c >= 0 && c < K) s_list[s_start[c]++] = e;
    }
    for (int k = K; k > 0; --k) s_start[k] = s_start[k - 1];
    s_start[0] = 0;
  }
  __syncthreads();
  for (int k = 0; k < K; ++k) {
    const int l0 = s_start[k], n = s_start[k + 1] - l0;
    const int g0 = min(max(gt_cat_off[k], 0), n_gt), g1 = min(max(gt_cat_off[k + 1], g0), n_gt), G = g1 - g0;
    if (n == 0 && G == 0) continue;                // evaluateVid returns None
    const int D = min(n, kMaxDet);
    // ---- rank inside (video, category): score descending, stable over the json order
    for (int i = tid; i < n; i += kThreads) {
      const int e = s_list[l0 + i];
      const double s = ents[e].score;
      int r = 0;
      for (int q = 0; q < n; ++q) {
        const int eq = s_list[l0 + q];
        const double sq = ents[eq].score;
        r += (sq > s) || (sq == s && eq < e);
      }
      if (r < kMaxDet) s_sorted[r] = e;            // computeIoU keeps the first maxDets[-1]
    }
    for (int i = tid; i < D; i += kThreads) { s_m[i] = 0; s_ig[i] = 0; }
    __syncthreads();
    // ---- avg_area (mean of the non-zero frame areas) and the sequence IoU [D, G]
    for (int d = tid; d < D; d += kThreads) {
      const int64_t o = obj_row(s_sorted[d]);
      const int nz = o >= 0 ? acc_nz[o] : 0;
      s_area[d] = nz > 0 ? __ddiv_rn((double)acc_area[o], (double)nz) : 0.0;
    }
    double* ious = iou_ws + (size_t)kMaxDet * g0;
    for (int p = tid; p < D * G; p += kThreads) {
      const int d = p / G, g = p - d * G;
      const int64_t o = obj_row(s_sorted[d]);
      const smb_ytvis_gt_t& gr = gts[g0 + g];
      double v = 0.0;
      if (gr.g < 0 || gr.g >= g_max) {
        atomicOr(status, SMB_YTVIS_GTS);
      } else {
        const int64_t i = o >= 0 ? acc_inter[o * g_max + gr.g] : 0;
        const int64_t u = (o >= 0 ? acc_area[o] : 0) + gr.sum_area - i;
        if (u > 0) v = __ddiv_rn((double)i, (double)u);   // iou_seq: i / u, 0 when u == 0
      }
      ious[p] = v;
    }
    __syncthreads();
    // ---- evaluateVid: evaluateImg's greedy matching on the sequence IoUs, avg_area as the area
    smb_match::greedy_match(
        tid, D, G, ious, gtm_ws + (size_t)kT * kA * g0, P,
        [&](int g) {
          const smb_ytvis_gt_t& gr = gts[g0 + g];
          return smb_match::MatchGt{gr.avg_area, gr.id, gr.crowd};
        },
        [&](int d) { return s_area[d]; }, npig + k * kA, s_m, s_ig);
    __syncthreads();
    for (int r = tid; r < D; r += kThreads) {
      const int e = s_sorted[r];
      if (e < n_out) {
        smb_coco_out_t& o = out[e];
        o.score = ents[e].score;
        o.matched = s_m[r];
        o.ignored = s_ig[r];
        o.cat = k;
        o.rank = r;
      }
    }
    __syncthreads();
  }
}

}  // namespace

extern "C" int smb_ytvis_overlap_dev(const smb_ytvis_frame_t* frames, int N, const int* count, int max_num,
                                     const smb_ytvis_gt_frame_t* gts, int n_gts, int g_max, int32_t* inter, int32_t* area,
                                     int* status, smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && max_num >= 1 && max_num <= SMB_COCO_DET_CAP && n_gts >= 0 && g_max >= 1,
                "smb_ytvis_overlap_dev: bad sizes (N %d, max_num %d, n_gts %d, g_max %d)", N, max_num, n_gts, g_max);
  if (N == 0) return SMB_OK;
  SMB_CHECK_ARG(frames && inter && area && status && (gts || n_gts == 0), "smb_ytvis_overlap_dev: null pointer");
  overlap_kernel<<<dim3(N, max_num), kThreads, 0, (cudaStream_t)stream>>>(frames, count, max_num, gts, n_gts, g_max, inter, area, status);
  SMB_LAUNCH_OK("overlap_kernel");
  return SMB_OK;
}

extern "C" int smb_ytvis_scatter_dev(const smb_ytvis_frame_t* frames, int N, const int* count, const int32_t* ids, int max_num,
                                     const int32_t* inter, const int32_t* area, int g_max, int64_t* acc_inter,
                                     int64_t* acc_area, int32_t* acc_nz, int slots, int objects, int* status,
                                     smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && max_num >= 1 && max_num <= SMB_COCO_DET_CAP && g_max >= 1 && slots >= 1 && objects >= 1,
                "smb_ytvis_scatter_dev: bad sizes (N %d, max_num %d, g_max %d, slots %d, objects %d)", N, max_num, g_max,
                slots, objects);
  if (N == 0) return SMB_OK;
  SMB_CHECK_ARG(frames && ids && inter && area && acc_inter && acc_area && acc_nz && status,
                "smb_ytvis_scatter_dev: null pointer");
  scatter_kernel<<<N, 128, 0, (cudaStream_t)stream>>>(frames, count, ids, max_num, inter, area, g_max, acc_inter, acc_area,
                                                      acc_nz, slots, objects, status);
  SMB_LAUNCH_OK("scatter_kernel");
  return SMB_OK;
}

extern "C" size_t smb_ytvis_match_workspace_bytes(int n_gt) { return smb_match::match_workspace_bytes(n_gt); }

extern "C" int smb_ytvis_match_dev(const smb_ytvis_entry_t* ents, int n_ent, const smb_ytvis_gt_t* gts, int n_gt,
                                   const int32_t* gt_cat_off, int K, int slot, const int64_t* acc_inter,
                                   const int64_t* acc_area, const int32_t* acc_nz, int slots, int objects, int g_max,
                                   int64_t video_id, const double* host_iou_thr, const double* host_area_rng,
                                   smb_coco_out_t* out, int64_t n_out, int* npig, int* status, void* workspace,
                                   size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n_ent >= 0 && n_ent <= SMB_COCO_DET_CAP && n_gt >= 0 && K >= 1 && K <= SMB_COCO_MAX_CATS && slots >= 1 &&
                    objects >= 1 && g_max >= 1 && n_out >= 0,
                "smb_ytvis_match_dev: bad sizes (n_ent %d, n_gt %d, K %d, slots %d, objects %d, g_max %d)", n_ent, n_gt, K,
                slots, objects, g_max);
  SMB_CHECK_ARG(host_iou_thr && host_area_rng, "smb_ytvis_match_dev: null thresholds");
  SMB_CHECK_ARG(gt_cat_off && npig && status && acc_inter && acc_area && acc_nz && workspace && (ents || n_ent == 0) &&
                    (gts || n_gt == 0) && (out || n_out == 0),
                "smb_ytvis_match_dev: null pointer");
  SMB_CHECK_ARG(workspace_bytes >= smb_match::match_workspace_bytes(n_gt),
                "smb_ytvis_match_dev: workspace of %zu bytes, %zu needed", workspace_bytes,
                smb_match::match_workspace_bytes(n_gt));
  const MatchParams P = smb_match::default_params(host_iou_thr, host_area_rng);
  double* iou_ws = (double*)workspace;
  uint8_t* gtm_ws = (uint8_t*)workspace + smb::align_up((size_t)n_gt * kMaxDet * sizeof(double), 256);
  const size_t smem = 3 * kMaxDet * 8 + (size_t)(kMaxDet + K + 1 + n_ent) * sizeof(int);
  if (smem > 48 * 1024)
    SMB_CUDA_OK(cudaFuncSetAttribute(seq_match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  seq_match_kernel<<<1, kThreads, smem, (cudaStream_t)stream>>>(ents, n_ent, gts, n_gt, gt_cat_off, K, slot, acc_inter,
                                                               acc_area, acc_nz, slots, objects, g_max, video_id, P, out,
                                                               n_out, npig, iou_ws, gtm_ws, status);
  SMB_LAUNCH_OK("seq_match_kernel");
  return SMB_OK;
}
