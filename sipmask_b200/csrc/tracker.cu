// SipMask-VIS tracker association step - HOST code (plain C++, no CUDA), part of the C ABI like smb_rle_to_string.
//
// Replaces the per-frame tail of SipMaskHead.get_bboxes in SipMask-VIS
// (SipMask-VIS/mmdet/models/anchor_heads/sipmask_head.py:612-667, compute_comp_scores :544-562, bbox_overlaps
// core/bbox/geometry.py:4-63).  The association is sequential in frame order and tiny (<= 10 detections x a few dozen tracked
// objects); in python/numpy it costs ~150 us of host time per frame, which caps a clip sharded over several GPUs at a few
// thousand frames/s.  Here it is ~2 us per frame.
//
//   comp[i][0]   = logsoftmax_i[0] + c0*log(score_i)            + c2            (dummy column: IoU 0, label match 1)
//   comp[i][j+1] = logsoftmax_i[j+1] + c0*log(score_i) + c1*IoU(det_i, prev_j) + c2*[label_i == prev_label_j]
//   argmax == 0 -> new object (appended, visible to the NEXT frame only; the comp matrix of this frame keeps its width);
//   else the detection claims object argmax-1 when its comp beats the best claim so far, and overwrites the object's stored
//   feature / box (not its label); earlier claimants keep their id (reference behaviour).
#include <math.h>
#include <stdint.h>
#include <string.h>

#include <vector>

#include "common.cuh"

// 512-term dot product; the host compiler emits an AVX2 + FMA clone next to the baseline one and picks at load time
// (function multi-versioning), so the library still runs on any x86-64 host.
#if defined(__x86_64__) && defined(__GNUC__) && !defined(__CUDA_ARCH__)
__attribute__((target_clones("avx2,fma", "default")))
#endif
static float dot_f32(const float* __restrict__ a, const float* __restrict__ b, int n) {
  float a8[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int k = 0;
  for (; k + 8 <= n; k += 8)
    for (int e = 0; e < 8; ++e) a8[e] += a[k + e] * b[k + e];
  float acc = ((a8[0] + a8[1]) + (a8[2] + a8[3])) + ((a8[4] + a8[5]) + (a8[6] + a8[7]));
  for (; k < n; ++k) acc += a[k] * b[k];
  return acc;
}

extern "C" int smb_track_step(const float* host_det, const int64_t* host_labels, const float* host_feats, int n, int feat_dim,
                              float* host_prev_det, int64_t* host_prev_labels, float* host_prev_feats, int n_prev, int capacity,
                              const float* host_match_coeff3, int32_t* host_ids_out) {
  SMB_CHECK_ARG(n >= 0 && feat_dim > 0 && n_prev >= 0 && capacity >= n_prev, "smb_track_step: bad sizes");
  SMB_CHECK_ARG(n == 0 || (host_det && host_labels && host_feats && host_ids_out), "smb_track_step: null input");
  SMB_CHECK_ARG(host_prev_det && host_prev_labels && host_prev_feats && host_match_coeff3, "smb_track_step: null state");
  if (n == 0) return n_prev;
  const float c0 = host_match_coeff3[0], c1 = host_match_coeff3[1], c2 = host_match_coeff3[2];
  const int m = n_prev;                       // width of this frame's comparison (objects appended now are not candidates)
  std::vector<float> comp((size_t)n * (m + 1));
  std::vector<double> best(m > 0 ? m : 1, -100.0);
  int np = n_prev;
  // comp matrix first (the reference computes it before any state update)
  for (int i = 0; i < n; ++i) {
    const float* d = host_det + (size_t)i * 5;
    const float* f = host_feats + (size_t)i * feat_dim;
    float* row = comp.data() + (size_t)i * (m + 1);
    row[0] = 0.f;
    float mx = 0.f;
    for (int j = 0; j < m; ++j) {
      const float* pf = host_prev_feats + (size_t)j * feat_dim;
      const float acc = dot_f32(f, pf, feat_dim);       // eight independent partial sums (vectorisable)
      row[j + 1] = acc;
      mx = acc > mx ? acc : mx;
    }
    float se = 0.f;
    for (int j = 0; j <= m; ++j) se += expf(row[j] - mx);
    const float lse = logf(se);
    const float ls = c0 * logf(d[4]);
    const float area_d = (d[2] - d[0] + 1.f) * (d[3] - d[1] + 1.f);
    for (int j = 0; j <= m; ++j) {
      float v = (row[j] - mx) - lse + ls;
      if (j == 0) {
        v += c2;
      } else {
        const float* pd = host_prev_det + (size_t)(j - 1) * 5;
        const float w = fminf(d[2], pd[2]) - fmaxf(d[0], pd[0]) + 1.f, h = fminf(d[3], pd[3]) - fmaxf(d[1], pd[1]) + 1.f;
        const float ov = (w > 0.f ? w : 0.f) * (h > 0.f ? h : 0.f);
        const float area_p = (pd[2] - pd[0] + 1.f) * (pd[3] - pd[1] + 1.f);
        v += c1 * (ov / (area_d + area_p - ov));
        if (host_prev_labels[j - 1] == host_labels[i]) v += c2;
      }
      row[j] = v;
    }
  }
  for (int i = 0; i < n; ++i) {
    const float* row = comp.data() + (size_t)i * (m + 1);
    int arg = 0;
    for (int j = 1; j <= m; ++j)
      if (row[j] > row[arg]) arg = j;             // first maximum, like torch.max / numpy.argmax
    if (arg == 0) {
      if (np >= capacity) { smb::set_error("smb_track_step: more than %d tracked objects", capacity); return SMB_EINVAL; }
      host_ids_out[i] = np;
      memcpy(host_prev_feats + (size_t)np * feat_dim, host_feats + (size_t)i * feat_dim, sizeof(float) * feat_dim);
      memcpy(host_prev_det + (size_t)np * 5, host_det + (size_t)i * 5, sizeof(float) * 5);
      host_prev_labels[np] = host_labels[i];
      ++np;
    } else {
      const int obj = arg - 1;
      host_ids_out[i] = -1;
      if ((double)row[arg] > best[obj]) {
        host_ids_out[i] = obj;
        best[obj] = (double)row[arg];
        memcpy(host_prev_feats + (size_t)obj * feat_dim, host_feats + (size_t)i * feat_dim, sizeof(float) * feat_dim);
        memcpy(host_prev_det + (size_t)obj * 5, host_det + (size_t)i * 5, sizeof(float) * 5);
      }
    }
  }
  return np;
}
