// COCOeval.evaluateImg's greedy matching of one (image, category), shared by COCO's per-image match (cocoeval.cu) and
// YTVOSeval's per-video match (ytviseval.cu), whose evaluateVid runs the same loop on sequence IoUs.
#pragma once
#include "common.cuh"

namespace smb_match {

constexpr int kT = SMB_COCO_T, kA = SMB_COCO_A, kMaxDet = SMB_COCO_MAX_DET, kMaxTA = SMB_COCO_MAX_TA;

// What the loop reads of COCOeval's Params: T IoU thresholds and A area ranges (T * A <= kMaxTA, any order), and
// maxDets[-1], the detections kept per (image, category).
struct MatchParams {
  int T, A, max_det;
  double iou_thr[kMaxTA];
  double area_rng[kMaxTA][2];
};

// The default Params' thresholds and ranges as COCOeval holds them (host_iou_thr[kT], host_area_rng[kA][2]).
inline MatchParams default_params(const double* host_iou_thr, const double* host_area_rng) {
  MatchParams P;
  P.T = kT;
  P.A = kA;
  P.max_det = kMaxDet;
  for (int t = 0; t < kT; ++t) P.iou_thr[t] = host_iou_thr[t];
  for (int a = 0; a < kA; ++a) { P.area_rng[a][0] = host_area_rng[2 * a]; P.area_rng[a][1] = host_area_rng[2 * a + 1]; }
  return P;
}

// What the loop reads of a ground truth: the area its range test uses, its annotation id (a match to id 0 does not count,
// as pycocotools tests dtm != 0), iscrowd, and skip: not part of this thread's ground-truth set (the error analysis runs
// one set per thread over the same IoU matrix; every other caller leaves it 0).
struct MatchGt {
  double area;
  int64_t id;
  int crowd;
  int skip;
};

// One thread per (threshold t, area range a), tid = t * P.A + a < P.T * P.A; the other threads return at once.
//   ious    : [D, G] of the D score-sorted detections (at most P.max_det) and the G ground truths in annotation order
//   gtm     : P.T * P.A * G bytes of workspace
//   gt_at(g): MatchGt of ground truth g; det_area(d): the area of sorted detection d
//   npig_k  : [P.A] non-ignored ground truths of the category, added with integer atomics by the t == 0 threads (NULL:
//             not counted)
//   s_m/s_ig: [D] matched / ignored bits (t * P.A + a) of the sorted detections, zeroed by the caller
template <typename GtAt, typename DetArea>
__device__ __forceinline__ void greedy_match(int tid, int D, int G, const double* __restrict__ ious, uint8_t* __restrict__ gtm_ws,
                                             const MatchParams& P, GtAt gt_at, DetArea det_area, int* npig_k, uint64_t* s_m,
                                             uint64_t* s_ig) {
  if (tid >= P.T * P.A) return;
  const int t = tid / P.A, a = tid - t * P.A;
  const double lo = P.area_rng[a][0], hi = P.area_rng[a][1];
  uint8_t* gtm = gtm_ws + (size_t)tid * G;
  for (int g = 0; g < G; ++g) gtm[g] = 0;
  auto gt_ig = [&](int g) {                        // 2: skipped, never equal to a pass
    const MatchGt gr = gt_at(g);
    return gr.skip ? 2 : (int)(gr.crowd || gr.area < lo || gr.area > hi);
  };
  if (t == 0 && npig_k) {
    int np = 0;
    for (int g = 0; g < G; ++g) np += gt_ig(g) == 0;
    if (np) atomicAdd(npig_k + a, np);
  }
  const double thr = P.iou_thr[t] < 1.0 - 1e-10 ? P.iou_thr[t] : 1.0 - 1e-10;
  const uint64_t bit = 1ull << tid;
  for (int d = 0; d < D; ++d) {
    double iou = thr;
    int m = -1, mig = 0;
    // ground truths stably reordered: not ignored first
    for (int pass = 0; pass < 2 && !(pass == 1 && m > -1 && mig == 0); ++pass) {
      for (int g = 0; g < G; ++g) {
        const int ig = gt_ig(g);
        if (ig != pass) continue;
        if (gtm[g] && !gt_at(g).crowd) continue;
        if (m > -1 && mig == 0 && ig == 1) break;
        const double v = ious[(size_t)d * G + g];
        if (v < iou) continue;
        iou = v;
        m = g;
        mig = ig;
      }
    }
    const double area = det_area(d);
    bool matched = false, ignored = false;
    if (m > -1) {
      gtm[m] = 1;
      matched = gt_at(m).id != 0;
      ignored = mig;
    }
    if (!matched && (area < lo || area > hi)) ignored = true;
    if (matched) atomicOr((unsigned long long*)&s_m[d], (unsigned long long)bit);
    if (ignored) atomicOr((unsigned long long*)&s_ig[d], (unsigned long long)bit);
  }
}

// Workspace of one match launch over n_gt ground truths: [n_gt, max_det] IoUs and [n_gt, ta] gtm bytes, ta = T * A.
inline size_t match_workspace_bytes(int n_gt, int ta = kT * kA, int max_det = kMaxDet) {
  if (n_gt < 0 || ta < 0 || max_det < 0) return 0;
  return smb::align_up((size_t)n_gt * max_det * sizeof(double), 256) + smb::align_up((size_t)n_gt * ta, 256) + 256;
}

}  // namespace smb_match
