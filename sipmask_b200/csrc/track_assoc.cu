// SipMask-VIS tracker association on the DEVICE: every frame of a dispatched batch in one launch, each video on a lane
// whose tracker state lives in device memory (the host step is smb_track_step in tracker.cu; same algorithm, same
// formula, see the comment at the top of that file).
//
// One CTA per lane.  The CTA scans the batch's frame rows and associates the rows of its lane in batch order, so several
// frames of one video in one launch see each other's state updates.  Per row:
//   1. warps compute the n x m 512-term dot products (detection features . tracked features), float4 loads and a shuffle
//      reduction, into the lane's workspace;
//   2. one warp per detection turns its row into the comp row (log-softmax with the dummy column, log score, IoU with the
//      +1 convention, label match) and takes the first maximum;
//   3. one thread runs the claim loop in detection order (appends, best claim so far starting at -100), which decides the
//      final writer of every object before
//   4. the warps copy the winners' boxes / features (and the appended objects' labels) into the state.
// fp32 throughout, accurate expf / logf, and the IoU and comp terms with explicitly rounded products (__fmul_rn), so the
// compiler cannot contract them into FMAs: apart from the dot products and the exp-sum, every value is the one the host
// step computes.
#include "common.cuh"

namespace {

constexpr int kFeat = SMB_TRACK_FEAT_DIM;
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxNum = 1024;

struct Coef {
  float c0, c1, c2;
};

__device__ __forceinline__ float warp_sum(float v) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
  for (int o = 16; o > 0; o >>= 1) {
    const float w = __shfl_xor_sync(0xffffffffu, v, o);
    v = w > v ? w : v;
  }
  return v;
}

// copy one detection (box, features, optionally label) into state slot dst: one warp
__device__ __forceinline__ void copy_object(const float* box, const float* feat, const int64_t* label, float* sbox,
                                            float* sfeat, int64_t* slab, int dst, bool with_label, int lid) {
  const float4* f = reinterpret_cast<const float4*>(feat);
  float4* o = reinterpret_cast<float4*>(sfeat + (size_t)dst * kFeat);
  for (int q = lid; q < kFeat / 4; q += 32) o[q] = f[q];
  if (lid < 5) sbox[(size_t)dst * 5 + lid] = box[lid];
  if (lid == 0 && with_label) slab[dst] = *label;
}

__global__ void __launch_bounds__(kThreads) track_assoc_kernel(
    const smb_track_frame_t* __restrict__ frames, int N, const float* __restrict__ det, const int64_t* __restrict__ labels,
    const int* __restrict__ count, const float* __restrict__ feats, int max_num, float* __restrict__ sbox_all,
    int64_t* __restrict__ slab_all, float* __restrict__ sfeat_all, int* __restrict__ n_obj, int* __restrict__ status,
    int lanes, int cap, Coef c, int32_t* __restrict__ ids, float* __restrict__ ws) {
  extern __shared__ int smem[];
  int* s_arg = smem;                                  // [max_num] argmax of each comp row
  float* s_val = reinterpret_cast<float*>(smem + max_num);   // [max_num] comp value at the argmax
  int* s_dst = smem + 2 * max_num;                    // [max_num] state slot detection i writes, -1: none
  int* s_cobj = smem + 3 * max_num;                   // [max_num] claim loop: objects claimed in this row
  int* s_cwr = smem + 4 * max_num;                    //           and their current (best) claimant
  __shared__ int s_nobj, s_status;

  const int lane = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lid = tid & 31;
  float* sbox = sbox_all + (size_t)lane * cap * 5;
  int64_t* slab = slab_all + (size_t)lane * cap;
  float* sfeat = sfeat_all + (size_t)lane * cap * kFeat;
  float* dots = ws + (size_t)lane * max_num * (cap + 1);
  if (tid == 0) {
    const int v = n_obj[lane];
    s_nobj = v < -1 ? -1 : (v > cap ? cap : v);       // -1: no state yet
    s_status = 0;
  }
  bool touched = false;

  for (int r = 0; r < N; ++r) {
    const smb_track_frame_t fr = frames[r];
    int32_t* id_row = ids + (size_t)r * max_num;
    if (fr.lane < 0 || fr.lane >= lanes) {            // filler row (or a lane outside the state): ids only
      if (lane == 0)
        for (int i = tid; i < max_num; i += kThreads) id_row[i] = -1;
      continue;
    }
    if (fr.lane != lane) continue;
    touched = true;
    const int cnt = count[r];
    const int n = cnt < 0 ? 0 : (cnt > max_num ? max_num : cnt);
    for (int i = n + tid; i < max_num; i += kThreads) id_row[i] = -1;
    if (n == 0) continue;                             // the reference returns before the tracker: state unchanged
    const float* d_det = det + (size_t)r * max_num * 5;
    const int64_t* d_lab = labels + (size_t)r * max_num;
    const float* d_feat = feats + (size_t)r * max_num * kFeat;
    __syncthreads();                                  // the previous row's state writes and s_nobj are visible
    const int m = s_nobj;
    const bool first = fr.is_first != 0 || m < 0;
    __syncthreads();                                  // every thread has read s_nobj before thread 0 changes it

    if (!first) {
      // 1. dot products, one warp per (detection, object) pair
      const int pairs = n * m;
      for (int p = warp; p < pairs; p += kWarps) {
        const int i = p / m, j = p - i * m;
        const float4* a = reinterpret_cast<const float4*>(d_feat + (size_t)i * kFeat);
        const float4* b = reinterpret_cast<const float4*>(sfeat + (size_t)j * kFeat);
        float acc = 0.f;
#pragma unroll
        for (int q = 0; q < kFeat / 128; ++q) {
          const float4 x = __ldg(a + lid + 32 * q), y = b[lid + 32 * q];
          acc = fmaf(x.x, y.x, acc);
          acc = fmaf(x.y, y.y, acc);
          acc = fmaf(x.z, y.z, acc);
          acc = fmaf(x.w, y.w, acc);
        }
        acc = warp_sum(acc);
        if (lid == 0) dots[(size_t)i * (m + 1) + j + 1] = acc;
      }
      __syncthreads();
      // 2. comp row and its first maximum, one warp per detection
      for (int i = warp; i < n; i += kWarps) {
        const float* row = dots + (size_t)i * (m + 1);
        float mx = 0.f;                               // the dummy column's score
        for (int j = 1 + lid; j <= m; j += 32) mx = row[j] > mx ? row[j] : mx;
        mx = warp_max(mx);
        float se = 0.f;
        for (int j = lid; j <= m; j += 32) se += expf((j == 0 ? 0.f : row[j]) - mx);
        se = warp_sum(se);
        const float lse = logf(se);
        const float* d = d_det + (size_t)i * 5;
        const float ls = __fmul_rn(c.c0, logf(d[4]));
        const float area_d = __fmul_rn(d[2] - d[0] + 1.f, d[3] - d[1] + 1.f);
        const int64_t lab = d_lab[i];
        float bv = 0.f;
        int bj = -1;
        for (int j = lid; j <= m; j += 32) {
          float v = ((j == 0 ? 0.f : row[j]) - mx) - lse + ls;
          if (j == 0) {
            v += c.c2;
          } else {
            const float* pd = sbox + (size_t)(j - 1) * 5;
            const float w = fminf(d[2], pd[2]) - fmaxf(d[0], pd[0]) + 1.f, h = fminf(d[3], pd[3]) - fmaxf(d[1], pd[1]) + 1.f;
            const float ov = __fmul_rn(w > 0.f ? w : 0.f, h > 0.f ? h : 0.f);
            const float area_p = __fmul_rn(pd[2] - pd[0] + 1.f, pd[3] - pd[1] + 1.f);
            v += __fmul_rn(c.c1, ov / (area_d + area_p - ov));
            if (slab[j - 1] == lab) v += c.c2;
          }
          if (bj < 0 || v > bv) { bv = v; bj = j; }    // this lane's first maximum (its j increase)
        }
        for (int o = 16; o > 0; o >>= 1) {            // the first maximum of the row: larger value, then smaller index
          const float ov = __shfl_xor_sync(0xffffffffu, bv, o);
          const int oj = __shfl_xor_sync(0xffffffffu, bj, o);
          if (oj >= 0 && (bj < 0 || ov > bv || (ov == bv && oj < bj))) { bv = ov; bj = oj; }
        }
        if (lid == 0) { s_arg[i] = bj; s_val[i] = bv; }
      }
      __syncthreads();
    }
    // 3. ids and the final writer of every state slot (sequential, as the reference's loop)
    if (tid == 0) {
      int np = first ? 0 : m, nclaims = 0;
      for (int i = 0; i < n; ++i) {
        int id = -1, dst = -1;
        if (first || s_arg[i] == 0) {                 // new object, visible from the next row on
          if (np < cap) {
            id = dst = np++;
          } else {
            s_status |= SMB_TRACK_CAPACITY;
          }
        } else {
          const int obj = s_arg[i] - 1;
          int k = 0;
          while (k < nclaims && s_cobj[k] != obj) ++k;
          const float best = k < nclaims ? s_val[s_cwr[k]] : -100.f;
          if (s_val[i] > best) {
            id = dst = obj;
            if (k < nclaims) s_dst[s_cwr[k]] = -1;     // the earlier claimant keeps its id, not the object's state
            else s_cobj[nclaims++] = obj;
            s_cwr[k] = i;
          }
        }
        s_dst[i] = dst;
        id_row[i] = id;
      }
      s_nobj = np;
    }
    __syncthreads();
    // 4. state copies; slots >= the old width are appended objects, which also take the label
    const int lab_from = first ? 0 : m;
    for (int i = warp; i < n; i += kWarps) {
      const int dst = s_dst[i];
      if (dst >= 0)
        copy_object(d_det + (size_t)i * 5, d_feat + (size_t)i * kFeat, d_lab + i, sbox, sfeat, slab, dst, dst >= lab_from, lid);
    }
  }
  __syncthreads();
  if (tid == 0 && touched) {
    n_obj[lane] = s_nobj;
    if (s_status) status[lane] |= s_status;
  }
}

}  // namespace

extern "C" size_t smb_track_assoc_workspace_bytes(int lanes, int max_num, int capacity) {
  if (lanes < 1 || max_num < 1 || capacity < 1) return 0;
  return smb::align_up((size_t)lanes * max_num * ((size_t)capacity + 1) * sizeof(float), 256);
}

extern "C" int smb_track_assoc_dev(const smb_track_frame_t* frames, int N, const float* det, const int64_t* labels,
                                   const int* count, const float* track_feats, int max_num, float* state_boxes,
                                   int64_t* state_labels, float* state_feats, int* n_obj, int* status, int lanes, int capacity,
                                   const float* host_match_coeff3, int32_t* ids, void* workspace, size_t workspace_bytes,
                                   smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && lanes >= 1 && capacity >= 1 && max_num >= 1 && max_num <= kMaxNum,
                "smb_track_assoc_dev: bad sizes (N %d, lanes %d, capacity %d, max_num %d)", N, lanes, capacity, max_num);
  SMB_CHECK_ARG(host_match_coeff3, "smb_track_assoc_dev: null match coefficients");
  if (N == 0) return SMB_OK;
  SMB_CHECK_ARG(frames && det && labels && count && track_feats && state_boxes && state_labels && state_feats && n_obj && status &&
                    ids && workspace,
                "smb_track_assoc_dev: null pointer");
  SMB_CHECK_ARG(((uintptr_t)track_feats & 15) == 0 && ((uintptr_t)state_feats & 15) == 0,
                "smb_track_assoc_dev: feature arrays must be 16-byte aligned");
  SMB_CHECK_ARG(workspace_bytes >= smb_track_assoc_workspace_bytes(lanes, max_num, capacity),
                "smb_track_assoc_dev: workspace of %zu bytes, %zu needed", workspace_bytes,
                smb_track_assoc_workspace_bytes(lanes, max_num, capacity));
  const Coef c{host_match_coeff3[0], host_match_coeff3[1], host_match_coeff3[2]};
  const size_t smem = (size_t)5 * max_num * sizeof(int);
  track_assoc_kernel<<<lanes, kThreads, smem, (cudaStream_t)stream>>>(frames, N, det, labels, count, track_feats, max_num,
                                                                      state_boxes, state_labels, state_feats, n_obj, status,
                                                                      lanes, capacity, c, ids, (float*)workspace);
  SMB_LAUNCH_OK("track_assoc_kernel");
  return SMB_OK;
}
