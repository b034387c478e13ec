// Device-side detection post-processing for sm_90a: per-level top-k + box decode, single-class NMS,
// batched multi-class NMS, fast NMS.  No host synchronisation, no D2H copies.
//
// Reference (SipMask-mmdetection/mmdet/):
//   models/anchor_heads/sipmask_head.py:556-605      per-level sigmoid/top-k/decode, NMS dispatch
//   core/bbox/transforms.py:202-223                  distance2bbox
//   core/post_processing/bbox_nms.py:79-146          multiclass_nms_idx (python loop over 80 classes)
//   ops/nms/src/nms_kernel.cu:14-22,24-68,71-138     devIoU(+1), bitmask kernel, D2H + host sweep
//   models/anchor_heads/sipmask_head.py:868-959      fast_nms / jaccard (no +1)
// These paths are integer/compare work on a few thousand boxes: latency-bound, not bandwidth-bound.
// One CTA per class keeps the sorted boxes and the suppression state in shared memory.
#include "common.cuh"
#include "cta.cuh"

namespace smb {

constexpr int NT = 1024;          // threads per CTA for all kernels in this file
constexpr int MAXN = 5120;        // max candidates per class list held in shared memory (>= 5 levels x nms_pre = 1000)
constexpr int MAXP = 8192;        // power of two >= MAXN: the bitonic sorts of up to MAXN keys pad to this many
static_assert(MAXP >= MAXN && (MAXP & (MAXP - 1)) == 0, "MAXP must be the padded sort length of MAXN keys");
constexpr int NMS1 = 8192;        // max boxes of the single-list operator smb_nms

// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float iou_ref(const float4 a, const float4 b, const float one) {
  // ops/nms/src/nms_kernel.cu:14-22 with separate IEEE roundings (no FMA contraction).
  const float left = fmaxf(a.x, b.x), right = fminf(a.z, b.z);
  const float top = fmaxf(a.y, b.y), bottom = fminf(a.w, b.w);
  const float width = fmaxf(__fadd_rn(__fsub_rn(right, left), one), 0.f);
  const float height = fmaxf(__fadd_rn(__fsub_rn(bottom, top), one), 0.f);
  const float interS = __fmul_rn(width, height);
  const float Sa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), one), __fadd_rn(__fsub_rn(a.w, a.y), one));
  const float Sb = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), one), __fadd_rn(__fsub_rn(b.w, b.y), one));
  return __fdiv_rn(interS, __fsub_rn(__fadd_rn(Sa, Sb), interS));
}

__device__ __forceinline__ float jaccard_ref(const float4 a, const float4 b) {
  // sipmask_head.py:912-959 (no +1; clamp(max_xy - min_xy, min=0))
  const float iw = fmaxf(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), 0.f);
  const float ih = fmaxf(__fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)), 0.f);
  const float inter = __fmul_rn(iw, ih);
  const float area_a = __fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y));
  const float area_b = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
  return __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, area_b), inter));
}

// descending-score / ascending-position composite: smaller key == earlier in the sorted order
__device__ __forceinline__ unsigned long long desc_key(float score, unsigned pos) {
  unsigned b = __float_as_uint(score);
  b = (b & 0x80000000u) ? ~b : (b | 0x80000000u);   // total order on floats
  return ((unsigned long long)(~b) << 32) | pos;
}
__device__ __forceinline__ float key_score(unsigned long long k) {
  unsigned b = ~(unsigned)(k >> 32);
  b = (b & 0x80000000u) ? (b & 0x7fffffffu) : ~b;
  return __uint_as_float(b);
}

// Greedy NMS sweep over `m` boxes already sorted by descending score in shared memory.
// On return bit r of rem[] is set iff sorted row r is suppressed.  `plus_one`/`cmp_ge` select the
// reference comparator (nms_kernel.cu:61 `>` vs nms_cpu.cpp:56 `>=`).
__device__ void greedy_sweep_n(const float4* sb, int m, float thr, int cmp_ge, float one,
                               unsigned long long* rem, int rem_words, unsigned long long* diag,
                               unsigned long long* s_keep);

// ---------------------------------------------------------------------------------------------
// Single-class NMS operator: dets [n,5]; keep ascending original indices.
// ---------------------------------------------------------------------------------------------
struct NmsSmem {
  unsigned long long keys[NMS1];
  float4 sb[NMS1];
  unsigned long long rem[NMS1 / 64];
  unsigned long long diag[64];
  unsigned long long keepbits;
  int warp[32];
  unsigned char kept[NMS1];
};

__global__ void __launch_bounds__(NT) nms_single_kernel(const float* __restrict__ dets, int n, float thr, int cmp_ge,
                                                        float one, long long* __restrict__ keep_out,
                                                        int* __restrict__ n_keep_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  NmsSmem& S = *reinterpret_cast<NmsSmem*>(smem_raw);
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += NT)
    S.keys[i] = (i < n) ? desc_key(dets[i * 5 + 4], (unsigned)i) : ~0ull;
  cta_bitonic_sort(S.keys, P, Less());
  for (int r = threadIdx.x; r < n; r += NT) {
    const int i = (int)(S.keys[r] & 0xffffffffu);
    S.sb[r] = make_float4(dets[i * 5], dets[i * 5 + 1], dets[i * 5 + 2], dets[i * 5 + 3]);
  }
  __syncthreads();
  greedy_sweep_n(S.sb, n, thr, cmp_ge, one, S.rem, NMS1 / 64, S.diag, &S.keepbits);
  for (int i = threadIdx.x; i < n; i += NT) S.kept[i] = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < n; r += NT)
    if (!((S.rem[r >> 6] >> (r & 63)) & 1ull)) S.kept[(int)(S.keys[r] & 0xffffffffu)] = 1;
  __syncthreads();
  int running = 0;
  for (int base = 0; base < n; base += NT) {
    const int i = base + threadIdx.x;
    const int f = (i < n) ? S.kept[i] : 0;
    int tot;
    const int ex = cta_exclusive_scan<NT>(f, Sum(), 0, S.warp, &tot);
    if (f) keep_out[running + ex] = i;
    running += tot;
  }
  if (threadIdx.x == 0) *n_keep_out = running;
}

__device__ void greedy_sweep_n(const float4* sb, int m, float thr, int cmp_ge, float one,
                               unsigned long long* rem, int rem_words, unsigned long long* diag,
                               unsigned long long* s_keep) {
  // On return bit r of rem[] is set iff sorted row r is suppressed.
  const int nblk = (m + 63) >> 6;
  for (int i = threadIdx.x; i < rem_words; i += blockDim.x) rem[i] = 0ull;
  __syncthreads();
  for (int b = 0; b < nblk; ++b) {
    const int base = b << 6;
    if (threadIdx.x < 64) diag[threadIdx.x] = 0ull;
    __syncthreads();
    {
      const int r = threadIdx.x >> 4, c0 = (threadIdx.x & 15) << 2;
      if (base + r < m) {
        const float4 a = sb[base + r];
        unsigned long long bits = 0ull;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const int c = c0 + q;
          if (c > r && base + c < m) {
            const float v = iou_ref(a, sb[base + c], one);
            if (cmp_ge ? (v >= thr) : (v > thr)) bits |= 1ull << c;
          }
        }
        if (bits) atomicOr(&diag[r], bits);
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cur = rem[b], keep = 0ull;
      const int lim = min(64, m - base);
      for (int t = 0; t < lim; ++t) {
        if (!((cur >> t) & 1ull)) { keep |= 1ull << t; cur |= diag[t]; }
      }
      rem[b] = cur;
      *s_keep = keep;
    }
    __syncthreads();
    const unsigned long long keep = *s_keep;
    for (int j = base + 64 + threadIdx.x; j < m; j += blockDim.x) {
      if ((rem[j >> 6] >> (j & 63)) & 1ull) continue;
      const float4 bj = sb[j];
      unsigned long long kk = keep;
      while (kk) {
        const int t = __ffsll((long long)kk) - 1;
        kk &= kk - 1;
        const float v = iou_ref(sb[base + t], bj, one);
        if (cmp_ge ? (v >= thr) : (v > thr)) { atomicOr(&rem[j >> 6], 1ull << (j & 63)); break; }
      }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------
// Multi-class NMS, stage 1: one CTA per class.
//   ws_idx  [C][n] int   : kept candidate rows (ascending) of class c
//   ws_score[C][n] float : their score*ctr
//   ws_count[C]          : number kept
// ---------------------------------------------------------------------------------------------
// Multi-class NMS, stage 1a: one CTA per class - candidate compaction (raw score > thr), score *= ctr, stable
// descending sort.  Writes, per class c (row pitch n):
//   w_cidx[c][pos]   candidate row (ascending)          w_cscore[c][pos]  score*ctr
//   w_keys[c][r]     sorted composite keys (low 32 bits = pos)    w_sbox[c][r]  boxes in sorted order
//   w_m[c]           number of candidates
struct McPrepSmem {
  unsigned long long keys[MAXP];
  int cidx[MAXN];
  float cscore[MAXN];
  int warp[32];
};

__global__ void __launch_bounds__(NT) mc_prepare_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                        const float* __restrict__ ctr, int n, int C, float score_thr,
                                                        int* __restrict__ w_cidx, float* __restrict__ w_cscore,
                                                        unsigned long long* __restrict__ w_keys, float4* __restrict__ w_sbox,
                                                        int* __restrict__ w_m) {
  pdl_wait();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  McPrepSmem& S = *reinterpret_cast<McPrepSmem*>(smem_raw);
  const int c = blockIdx.x;
  int m = 0;
  for (int base = 0; base < n; base += NT) {
    const int i = base + threadIdx.x;
    float s = 0.f;
    int f = 0;
    if (i < n) { s = scores[(size_t)i * C + c]; f = s > score_thr; }       // bbox_nms.py:111
    int tot;
    const int ex = cta_exclusive_scan<NT>(f, Sum(), 0, S.warp, &tot);
    if (f) { S.cidx[m + ex] = i; S.cscore[m + ex] = __fmul_rn(s, ctr[i]); }  // bbox_nms.py:122
    m += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) w_m[c] = m;
  if (m == 0) return;
  int P = 1;
  while (P < m) P <<= 1;
  for (int i = threadIdx.x; i < P; i += NT) S.keys[i] = (i < m) ? desc_key(S.cscore[i], (unsigned)i) : ~0ull;
  cta_bitonic_sort(S.keys, P, Less());
  for (int r = threadIdx.x; r < m; r += NT) {
    const unsigned long long k = S.keys[r];
    const int pos = (int)(k & 0xffffffffu);
    w_keys[(size_t)c * n + r] = k;
    w_sbox[(size_t)c * n + r] = *reinterpret_cast<const float4*>(boxes + (size_t)S.cidx[pos] * 4);
    w_cidx[(size_t)c * n + r] = S.cidx[r];          // by position (r < m covers all positions)
    w_cscore[(size_t)c * n + r] = S.cscore[r];
  }
}

// Stage 1b: suppression bit-matrix, spread over the whole GPU.  Work item = one 64x64 tile (class c, row block rb,
// column block cb >= rb); bit t of mask[c][rb*64 + r][cb] is set iff IoU(sorted r, sorted cb*64+t) exceeds the
// threshold and the column comes later in the sorted order (ops/nms/src/nms_kernel.cu:24-68, all classes at once).
__global__ void __launch_bounds__(64) mc_mask_kernel(const float4* __restrict__ w_sbox, const int* __restrict__ w_m, int n, int C,
                                                     int nbmax, float iou_thr, int cmp_ge,
                                                     unsigned long long* __restrict__ mask) {
  pdl_wait();
  __shared__ int s_pref[1025];
  __shared__ float4 s_col[64];
  __shared__ int s_tile[3];
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int c = 0; c < C; ++c) {
      s_pref[c] = acc;
      const int nb = (w_m[c] + 63) >> 6;
      acc += nb * (nb + 1) / 2;
    }
    s_pref[C] = acc;
  }
  __syncthreads();
  const int total = s_pref[C];
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    if (threadIdx.x == 0) {
      int c = 0;
      while (s_pref[c + 1] <= t) ++c;
      int u = t - s_pref[c];
      const int nb = (w_m[c] + 63) >> 6;
      int rb = 0;
      while (u >= nb - rb) { u -= nb - rb; ++rb; }
      s_tile[0] = c; s_tile[1] = rb; s_tile[2] = rb + u;
    }
    __syncthreads();
    const int c = s_tile[0], rb = s_tile[1], cb = s_tile[2];
    const int m = w_m[c];
    const float4* sb = w_sbox + (size_t)c * n;
    const int col = cb * 64 + threadIdx.x;
    s_col[threadIdx.x] = (col < m) ? sb[col] : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    const int row = rb * 64 + threadIdx.x;
    if (row < m) {
      const float4 a = sb[row];
      unsigned long long bits = 0ull;
      const int lim = min(64, m - cb * 64);
      const int start = (rb == cb) ? threadIdx.x + 1 : 0;
      for (int q = start; q < lim; ++q) {
        const float v = iou_ref(a, s_col[q], 1.0f);
        if (cmp_ge ? (v >= iou_thr) : (v > iou_thr)) bits |= 1ull << q;
      }
      mask[((size_t)c * n + row) * nbmax + cb] = bits;
    }
    __syncthreads();
  }
}

// Stage 1c: one CTA per class - sequential sweep over the bit-matrix (the reference does this on the host after a
// D2H copy, nms_kernel.cu:105-131), then kept rows in ascending candidate order (nms_kernel.cu:135-138).
struct McSweepSmem {
  unsigned long long rem[MAXN / 64];
  unsigned long long diag[64];
  unsigned long long keepbits;
  int warp[32];
  unsigned char kept[MAXN];
};

__global__ void __launch_bounds__(NT) mc_sweep_kernel(const unsigned long long* __restrict__ mask,
                                                      const unsigned long long* __restrict__ w_keys,
                                                      const int* __restrict__ w_cidx, const float* __restrict__ w_cscore,
                                                      const int* __restrict__ w_m, int n, int nbmax, int* __restrict__ ws_idx,
                                                      float* __restrict__ ws_score, int* __restrict__ ws_count) {
  pdl_wait();
  __shared__ McSweepSmem S;
  const int c = blockIdx.x;
  const int m = w_m[c];
  if (m == 0) {
    if (threadIdx.x == 0) ws_count[c] = 0;
    return;
  }
  const int nb = (m + 63) >> 6;
  const unsigned long long* mk = mask + (size_t)c * n * nbmax;
  for (int i = threadIdx.x; i < MAXN / 64; i += NT) S.rem[i] = 0ull;
  __syncthreads();
  for (int b = 0; b < nb; ++b) {
    const int base = b << 6;
    if (threadIdx.x < 64) S.diag[threadIdx.x] = (base + threadIdx.x < m) ? mk[(size_t)(base + threadIdx.x) * nbmax + b] : 0ull;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cur = S.rem[b], keep = 0ull;
      const int lim = min(64, m - base);
      for (int t = 0; t < lim; ++t)
        if (!((cur >> t) & 1ull)) { keep |= 1ull << t; cur |= S.diag[t]; }
      S.rem[b] = cur;
      S.keepbits = keep;
    }
    __syncthreads();
    // OR the rows of the kept boxes into the later column words: thread = (column word j, row slice)
    const unsigned long long keep = S.keepbits;
    const int nlater = nb - (b + 1);
    if (nlater > 0) {
      const int j = b + 1 + (threadIdx.x % nlater);
      const int slice = threadIdx.x / nlater, nslices = NT / nlater;
      if (slice < nslices) {
        unsigned long long acc = 0ull;
        for (int t = slice; t < 64; t += nslices)
          if ((keep >> t) & 1ull) acc |= mk[(size_t)(base + t) * nbmax + j];
        if (acc) atomicOr(&S.rem[j], acc);
      }
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < m; i += NT) S.kept[i] = 0;
  __syncthreads();
  for (int r = threadIdx.x; r < m; r += NT)
    if (!((S.rem[r >> 6] >> (r & 63)) & 1ull)) S.kept[(int)(w_keys[(size_t)c * n + r] & 0xffffffffu)] = 1;
  __syncthreads();
  int running = 0;
  for (int base = 0; base < m; base += NT) {
    const int p = base + threadIdx.x;
    const int f = (p < m) ? S.kept[p] : 0;
    int tot;
    const int ex = cta_exclusive_scan<NT>(f, Sum(), 0, S.warp, &tot);
    if (f) {
      ws_idx[(size_t)c * n + running + ex] = w_cidx[(size_t)c * n + p];
      ws_score[(size_t)c * n + running + ex] = w_cscore[(size_t)c * n + p];
    }
    running += tot;
  }
  if (threadIdx.x == 0) ws_count[c] = running;
}

// ---------------------------------------------------------------------------------------------
// Stage 2 (single CTA): concatenate class lists (class-major), keep the top `max_num` by score
// when there are more (bbox_nms.py:135-140), emit dets / labels / rows.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(NT) finalize_kernel(const float* __restrict__ boxes, int n, int C, int max_num,
                                                      int always_sort, const int* __restrict__ ws_idx,
                                                      const float* __restrict__ ws_score,
                                                      const int* __restrict__ ws_count, int list_pitch,
                                                      unsigned long long* __restrict__ gkey,
                                                      int* __restrict__ gval, float* __restrict__ det_out,
                                                      long long* __restrict__ label_out,
                                                      long long* __restrict__ idx_out, int* __restrict__ count_out) {
  pdl_wait();
  __shared__ int s_off[1025];
  __shared__ int s_warp[32];
  __shared__ unsigned long long s_sel[1024];
  __shared__ SelectSmem s_select;
  // class offsets
  {
    const int v = (threadIdx.x < C) ? ws_count[threadIdx.x] : 0;
    int tot;
    const int ex = cta_exclusive_scan<NT>(v, Sum(), 0, s_warp, &tot);
    if (threadIdx.x < C) s_off[threadIdx.x] = ex;
    if (threadIdx.x == 0) s_off[C] = tot;
  }
  __syncthreads();
  const int K = s_off[C];
  // zero-fill outputs beyond the count so the fixed-shape record is deterministic
  const int kout = min(K, max_num);
  for (int i = threadIdx.x; i < max_num; i += NT) {
    if (i >= kout) {
      for (int q = 0; q < 5; ++q) det_out[i * 5 + q] = 0.f;
      label_out[i] = -1;
      idx_out[i] = -1;
    }
  }
  if (threadIdx.x == 0) *count_out = kout;
  if (K == 0) return;
  if (K <= max_num && !always_sort) {
    for (int c = 0; c < C; ++c) {
      const int cnt = s_off[c + 1] - s_off[c];
      for (int k = threadIdx.x; k < cnt; k += NT) {
        const int g = s_off[c] + k;
        const int row = ws_idx[(size_t)c * list_pitch + k];
        const float4 b = *reinterpret_cast<const float4*>(boxes + (size_t)row * 4);
        det_out[g * 5 + 0] = b.x; det_out[g * 5 + 1] = b.y; det_out[g * 5 + 2] = b.z; det_out[g * 5 + 3] = b.w;
        det_out[g * 5 + 4] = ws_score[(size_t)c * list_pitch + k];
        label_out[g] = c;
        idx_out[g] = row;
      }
    }
    return;
  }
  // compact composite keys: ascending key == descending score, ties by class-major position
  for (int c = 0; c < C; ++c) {
    const int cnt = s_off[c + 1] - s_off[c];
    for (int k = threadIdx.x; k < cnt; k += NT) {
      const int g = s_off[c] + k;
      gkey[g] = desc_key(ws_score[(size_t)c * list_pitch + k], (unsigned)g);
      gval[g] = (c << 16) | ws_idx[(size_t)c * list_pitch + k];
    }
  }
  // the kout smallest keys in order (keys are unique); the select synchronises before it reads gkey
  cta_smallest_sorted<NT>(K, kout, [&](int g) { return gkey[g]; }, s_sel, 1024, s_select);
  for (int r = threadIdx.x; r < kout; r += NT) {
    const unsigned long long k = s_sel[r];
    const int g = (int)(k & 0xffffffffu);
    const int v = gval[g];
    const int row = v & 0xffff, c = v >> 16;
    const float4 b = *reinterpret_cast<const float4*>(boxes + (size_t)row * 4);
    det_out[r * 5 + 0] = b.x; det_out[r * 5 + 1] = b.y; det_out[r * 5 + 2] = b.z; det_out[r * 5 + 3] = b.w;
    det_out[r * 5 + 4] = key_score(k);
    label_out[r] = c;
    idx_out[r] = row;
  }
}

// ---------------------------------------------------------------------------------------------
// fast_nms stage 1: one CTA per class (sipmask_head.py:868-891).
// ---------------------------------------------------------------------------------------------
struct FastSmem {
  unsigned long long keys[MAXP];
  float4 sb[256];
  float sscore[256];
  unsigned char kept[256];
  int warp[32];
};

__global__ void __launch_bounds__(NT) fast_nms_class_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                            const float* __restrict__ ctr, int n, int C, float score_thr,
                                                            float iou_thr, int top_k, int* __restrict__ ws_idx,
                                                            float* __restrict__ ws_score, int* __restrict__ ws_count) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  FastSmem& S = *reinterpret_cast<FastSmem*>(smem_raw);
  const int c = blockIdx.x;
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += NT)
    S.keys[i] = (i < n) ? desc_key(__fmul_rn(scores[(size_t)i * C + c], ctr[i]), (unsigned)i) : ~0ull;
  cta_bitonic_sort(S.keys, P, Less());
  const int m = min(n, top_k);
  for (int r = threadIdx.x; r < m; r += NT) {
    const unsigned long long k = S.keys[r];
    S.sb[r] = *reinterpret_cast<const float4*>(boxes + (size_t)(k & 0xffffffffu) * 4);
    S.sscore[r] = key_score(k);
  }
  __syncthreads();
  // column max of the strictly-upper-triangular IoU matrix; torch.max propagates NaN
  for (int j = threadIdx.x; j < m; j += NT) {
    float mx = 0.f;      // triu_ leaves zeros on/below the diagonal, so the max is >= 0
    bool nan = false;
    const float4 bj = S.sb[j];
    for (int i = 0; i < j; ++i) {
      const float v = jaccard_ref(S.sb[i], bj);
      if (v != v) nan = true;
      mx = fmaxf(mx, v);
    }
    const bool keep = !nan && (mx <= iou_thr) && (S.sscore[j] > score_thr);
    S.kept[j] = keep ? 1 : 0;
  }
  __syncthreads();
  int running = 0;
  for (int base = 0; base < m; base += NT) {
    const int p = base + threadIdx.x;
    const int f = (p < m) ? S.kept[p] : 0;
    int tot;
    const int ex = cta_exclusive_scan<NT>(f, Sum(), 0, S.warp, &tot);
    if (f) {
      ws_idx[(size_t)c * top_k + running + ex] = (int)(S.keys[p] & 0xffffffffu);
      ws_score[(size_t)c * top_k + running + ex] = S.sscore[p];
    }
    running += tot;
  }
  if (threadIdx.x == 0) ws_count[c] = running;
}

// ---------------------------------------------------------------------------------------------
// decode + per-level top-k
// ---------------------------------------------------------------------------------------------
constexpr int MAXLVL = 8;
struct Levels {
  smb_level_t lv[MAXLVL];
  int loc_off[MAXLVL + 1];    // level-concatenated location offsets
  int cand_off[MAXLVL + 1];   // candidate offsets
  int num;
};

// s[loc] = max_c(sigmoid(cls)*sigmoid(ctr)) = sigmoid(max_c cls) * sigmoid(ctr)   (sipmask_head.py:572)
__global__ void level_score_kernel(Levels L, int C, float* __restrict__ s) {
  pdl_wait();
  const int total = L.loc_off[L.num];
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int loc = blockIdx.x * warps_per_block + (threadIdx.x >> 5); loc < total; loc += gridDim.x * warps_per_block) {
    int l = 0;
    while (loc >= L.loc_off[l + 1]) ++l;
    const int i = loc - L.loc_off[l];
    const float* row = L.lv[l].cls + (size_t)i * L.lv[l].cls_pitch;
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, row[c]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) {
      const float ct = L.lv[l].ctr[(size_t)i * L.lv[l].ctr_pitch];
      s[loc] = __fmul_rn(sigmoidf_(mx), sigmoidf_(ct));
    }
  }
}

// one CTA per level: selected location indices (descending score, ties -> lower index)
__global__ void __launch_bounds__(NT) level_topk_kernel(Levels L, int nms_pre, const float* __restrict__ s,
                                                        int* __restrict__ sel) {
  pdl_wait();
  __shared__ unsigned long long s_sel[1024];
  __shared__ SelectSmem s_select;
  const int l = blockIdx.x;
  const int hw = L.loc_off[l + 1] - L.loc_off[l];
  const float* sl = s + L.loc_off[l];
  int* out = sel + L.cand_off[l];
  if (nms_pre <= 0 || hw <= nms_pre) {
    for (int i = threadIdx.x; i < hw; i += NT) out[i] = i;
    return;
  }
  cta_smallest_sorted<NT>(hw, nms_pre, [&](int i) { return desc_key(sl[i], (unsigned)i); }, s_sel, 1024, s_select);
  for (int r = threadIdx.x; r < nms_pre; r += NT) out[r] = (int)(s_sel[r] & 0xffffffffu);
}

// one warp per candidate: box decode + sigmoid scores
__global__ void gather_decode_kernel(Levels L, int C, GeomArg ga, const int* __restrict__ sel, float* __restrict__ cand_boxes,
                                     float* __restrict__ cand_scores, float* __restrict__ cand_ctr,
                                     int* __restrict__ cand_loc) {
  pdl_wait();
  const smb_img_geom_t g = load_geom(ga);
  const int total = L.cand_off[L.num];
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int q = blockIdx.x * warps_per_block + (threadIdx.x >> 5); q < total; q += gridDim.x * warps_per_block) {
    int l = 0;
    while (q >= L.cand_off[l + 1]) ++l;
    const int i = sel[q];
    const smb_level_t& lv = L.lv[l];
    const float* row = lv.cls + (size_t)i * lv.cls_pitch;
    for (int c = lane; c < C; c += 32) cand_scores[(size_t)q * C + c] = sigmoidf_(row[c]);
    if (lane == 0) {
      const int y = i / lv.w, x = i - y * lv.w;
      const float px = (float)(x * lv.stride + lv.stride / 2), py = (float)(y * lv.stride + lv.stride / 2);
      const float* d = lv.box + (size_t)i * lv.box_pitch;
      const float d0 = __fmul_rn(__fmul_rn(d[0], lv.box_scale), lv.box_mul), d1 = __fmul_rn(__fmul_rn(d[1], lv.box_scale), lv.box_mul);
      const float d2 = __fmul_rn(__fmul_rn(d[2], lv.box_scale), lv.box_mul), d3 = __fmul_rn(__fmul_rn(d[3], lv.box_scale), lv.box_mul);
      float x1 = __fsub_rn(px, d0), y1 = __fsub_rn(py, d1);
      float x2 = __fadd_rn(px, d2), y2 = __fadd_rn(py, d3);
      const float mw = (float)(g.img_w - 1), mh = (float)(g.img_h - 1);
      x1 = fminf(fmaxf(x1, 0.f), mw); y1 = fminf(fmaxf(y1, 0.f), mh);
      x2 = fminf(fmaxf(x2, 0.f), mw); y2 = fminf(fmaxf(y2, 0.f), mh);
      // mlvl_bboxes /= scale_factor (sipmask_head.py:587-588): true division (by 1 when there is no rescale: exact)
      x1 = __fdiv_rn(x1, g.scale[0]); y1 = __fdiv_rn(y1, g.scale[1]); x2 = __fdiv_rn(x2, g.scale[2]); y2 = __fdiv_rn(y2, g.scale[3]);
      *reinterpret_cast<float4*>(cand_boxes + (size_t)q * 4) = make_float4(x1, y1, x2, y2);
      cand_ctr[q] = sigmoidf_(lv.ctr[(size_t)i * lv.ctr_pitch]);
      cand_loc[q] = L.loc_off[l] + i;
    }
  }
}

__global__ void gather_rows_kernel(const float* __restrict__ src, int src_pitch, const long long* __restrict__ idx,
                                   const int* __restrict__ count, int max_rows, int row_elems, float* __restrict__ dst) {
  pdl_wait();
  const int total = max_rows * row_elems;
  const int cnt = *count;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int r = t / row_elems, e = t - r * row_elems;
    dst[t] = (r < cnt) ? src[(size_t)idx[r] * src_pitch + e] : 0.f;
  }
}

// det_cofs[i,:] = cof_src[cand_loc[idx[i]], :], det_boxes[i,:] = det[i,:4] for i < *count, zeros after: the gather between
// NMS and mask assembly (mlvl_cofs[idxs_keep], det_bboxes[:, :4], sipmask_head.py:612,623) as ONE launch.
// Row table of a level-major, image-inside-level buffer [level][image][hw_l][pitch]: row(loc) of image `img` =
// loc_off[l] * n_img + img * hw_l + (loc - loc_off[l]); num == 0: plain [tot][pitch] (row = loc).
struct LocMap {
  int num, n_img, img;
  int loc_off[MAXLVL + 1];
};
__device__ __forceinline__ long long loc_row(const LocMap& m, int loc) {
  if (m.num == 0) return loc;
  int l = 0;
#pragma unroll
  for (int i = 1; i < MAXLVL; ++i)
    if (i < m.num && loc >= m.loc_off[i]) l = i;
  const int hw = m.loc_off[l + 1] - m.loc_off[l];
  return (long long)m.loc_off[l] * m.n_img + (long long)m.img * hw + (loc - m.loc_off[l]);
}

__global__ void gather_det_inputs_kernel(const float* __restrict__ cof_src, int cof_pitch, const int* __restrict__ cand_loc,
                                         const long long* __restrict__ idx, const float* __restrict__ det,
                                         const int* __restrict__ count, int max_rows, int row_elems,
                                         float* __restrict__ det_cofs, float* __restrict__ det_boxes,
                                         long long* __restrict__ loc_out, LocMap lm) {
  pdl_wait();
  const int total = max_rows * row_elems;
  const int cnt = *count;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int r = t / row_elems, e = t - r * row_elems;
    float v = 0.f;
    if (r < cnt) {
      const int loc = cand_loc[idx[r]];
      v = cof_src[(size_t)loc_row(lm, loc) * cof_pitch + e];
      if (e == 0 && loc_out) loc_out[r] = loc;
    } else if (e == 0 && loc_out) {
      loc_out[r] = -1;
    }
    det_cofs[t] = v;
    if (e < 4) det_boxes[r * 4 + e] = (r < cnt) ? det[r * 5 + e] : 0.f;
  }
}

// SipMask-VIS: the 512-d tracking feature of every kept detection, taken at the box centre of res_det = det * scale_factor
// on the stride-8 track map: floor((x1 + x2) / 2 / 8) (VIS/mmdet/models/anchor_heads/sipmask_head.py:609-613,768-781).
// track [h,w,C] fp32 channel-last; out [max_rows,C], zeros after *count.  Indices are clamped into the map (the reference
// indexes unclamped and would raise on an out-of-range centre).
__global__ void gather_track_feats_kernel(const float* __restrict__ track, int h, int w, int C, const float* __restrict__ det,
                                          const int* __restrict__ count, int max_rows, GeomArg ga, float stride,
                                          float* __restrict__ out) {
  pdl_wait();
  const smb_img_geom_t g = load_geom(ga);
  const float sx = g.track_sx, sy = g.track_sy;
  const int total = max_rows * C;
  const int cnt = *count;
  for (int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
    const int r = t / C, e = t - r * C;
    float v = 0.f;
    if (r < cnt) {
      const float x1 = __fmul_rn(det[r * 5 + 0], sx), y1 = __fmul_rn(det[r * 5 + 1], sy);
      const float x2 = __fmul_rn(det[r * 5 + 2], sx), y2 = __fmul_rn(det[r * 5 + 3], sy);
      int cx = (int)floorf(__fdiv_rn(__fdiv_rn(__fadd_rn(x2, x1), 2.0f), stride));
      int cy = (int)floorf(__fdiv_rn(__fdiv_rn(__fadd_rn(y2, y1), 2.0f), stride));
      cx = min(max(cx, 0), w - 1);
      cy = min(max(cy, 0), h - 1);
      v = track[((size_t)cy * w + cx) * C + e];
    }
    out[t] = v;
  }
}

// ---------------------------------------------------------------------------------------------
// SipMask-benchmark post-processing (SipMask-benchmark/fcos_core/modeling/rpn/sipmask/inference.py:90-190,
// csrc/cuda/ml_nms.cu:13-72,132-135).  Candidates are (location, class) PAIRS, not locations.
// ---------------------------------------------------------------------------------------------
// Sigmoid with one rounding per step: exp in double rounded to float, then IEEE add and divide.  A CPU restatement
// (float64 exp -> float32, float32 arithmetic) gives the same bits, so the pair selection can be checked exactly.
__device__ __forceinline__ float sigmoid_rn(float x) {
  const float e = (float)exp(-(double)x);
  return __fdiv_rn(1.0f, __fadd_rn(1.0f, e));
}

struct PairLevels {
  smb_level_t lv[MAXLVL];
  int loc_off[MAXLVL + 1];    // level-concatenated location offsets
  long long pair_off[MAXLVL + 1];   // level-concatenated pair offsets (h*w*C per level)
  int sel_cap[MAXLVL];        // min(h*w*C, nms_pre): capacity of the level's slice of `sel`
  int sel_off[MAXLVL + 1];
  int num;
};

// key[pair] = bits(sigmoid(cls) * sigmoid(ctr)) + 1 if sigmoid(cls) > thr, else 0 (inference.py:90-95).  Positive floats
// order like their bit patterns, so a larger key is a larger score.  One warp per location.
__global__ void pair_key_kernel(PairLevels L, int C, float thr, unsigned* __restrict__ keys) {
  pdl_wait();
  const int total = L.loc_off[L.num];
  const int warps_per_block = blockDim.x >> 5;
  const int lane = threadIdx.x & 31;
  for (int loc = blockIdx.x * warps_per_block + (threadIdx.x >> 5); loc < total; loc += gridDim.x * warps_per_block) {
    int l = 0;
    while (loc >= L.loc_off[l + 1]) ++l;
    const int i = loc - L.loc_off[l];
    const smb_level_t& lv = L.lv[l];
    const float* row = lv.cls + (size_t)i * lv.cls_pitch;
    const float ct = sigmoid_rn(lv.ctr[(size_t)i * lv.ctr_pitch]);
    unsigned* out = keys + L.pair_off[l] + (size_t)i * C;
    for (int c = lane; c < C; c += 32) {
      const float s = sigmoid_rn(row[c]);
      out[c] = (s > thr) ? __float_as_uint(__fmul_rn(s, ct)) + 1u : 0u;
    }
  }
}

// One CTA per level: the pairs that pass, or, when more than nms_pre pass, the nms_pre largest keys with ties going to
// the lower pair index.  Writes the selected pair indices in ascending order and their number (<= sel_cap[l]).
constexpr int PAIR_RUN = 16;       // consecutive pairs per thread in the ordered compaction
__global__ void __launch_bounds__(NT) pair_select_kernel(PairLevels L, int nms_pre, const unsigned* __restrict__ keys,
                                                         int* __restrict__ sel, int* __restrict__ sel_count) {
  pdl_wait();
  __shared__ SelectSmem s_select;
  __shared__ int s_warp[32];
  const int l = blockIdx.x;
  const int n = (int)(L.pair_off[l + 1] - L.pair_off[l]);
  const unsigned* kl = keys + L.pair_off[l];
  const int cap = L.sel_cap[l];
  int* out = sel + L.sel_off[l];
  // number of passing pairs
  int mine = 0;
  for (int i = threadIdx.x; i < n; i += NT) mine += kl[i] != 0u;
  int n_pass;
  cta_inclusive_scan<NT>(mine, Sum(), s_warp, &n_pass);
  // threshold key T and the number of pairs equal to T that may still be taken (lowest indices first)
  unsigned T = 1u;
  int budget = 0x7fffffff;
  if (n_pass > cap) {
    // the cap-th smallest of ~key (= the cap-th largest key), and its rank among the keys equal to it
    const RadixKth<unsigned> kth = cta_radix_select<NT, unsigned>(n, cap, [&](int i) { return ~kl[i]; }, s_select);
    T = ~kth.key;
    budget = kth.rank;
  }
  // ordered compaction: thread t owns PAIR_RUN consecutive pairs of each chunk
  int running = 0, tie_running = 0;
  for (int base = 0; base < n; base += NT * PAIR_RUN) {
    const int i0 = base + threadIdx.x * PAIR_RUN;
    unsigned k[PAIR_RUN];
    int ties = 0;
#pragma unroll
    for (int j = 0; j < PAIR_RUN; ++j) {
      k[j] = (i0 + j < n) ? kl[i0 + j] : 0u;
      ties += k[j] == T;
    }
    int tie_tot;
    int tie_rank = tie_running + cta_exclusive_scan<NT>(ties, Sum(), 0, s_warp, &tie_tot);
    unsigned take = 0u;
    int cnt = 0;
#pragma unroll
    for (int j = 0; j < PAIR_RUN; ++j) {
      bool f = k[j] > T;
      if (k[j] == T && k[j] != 0u) { f = tie_rank < budget; ++tie_rank; }
      if (f) { take |= 1u << j; ++cnt; }
    }
    int tot;
    int pos = running + cta_exclusive_scan<NT>(cnt, Sum(), 0, s_warp, &tot);
#pragma unroll
    for (int j = 0; j < PAIR_RUN; ++j)
      if ((take >> j) & 1u) {
        if (pos < cap) out[pos] = i0 + j;
        ++pos;
      }
    running += tot;
    tie_running += tie_tot;
  }
  if (threadIdx.x == 0) sel_count[l] = min(running, cap);
}

// One thread per output slot: level-major, ascending pair index inside a level.  Box = location -/+ relu(box * scale) *
// mul, clipped to [0, w-1] x [0, h-1] (inference.py:125-141, bounding_box.py:214-224); score = sqrt(cls * ctr).
// Slots past the candidate count get zero boxes / scores and label -1.
__global__ void pair_decode_kernel(PairLevels L, int C, GeomArg ga, const int* __restrict__ sel,
                                   const int* __restrict__ sel_count, int n_slots, float* __restrict__ cand_boxes,
                                   float* __restrict__ cand_scores, int* __restrict__ cand_labels, int* __restrict__ cand_loc,
                                   int* __restrict__ n_cand) {
  pdl_wait();
  const smb_img_geom_t g = load_geom(ga);
  int off[MAXLVL + 1];
  off[0] = 0;
  for (int l = 0; l < L.num; ++l) off[l + 1] = off[l] + min(max(sel_count[l], 0), L.sel_cap[l]);
  const int total = off[L.num];
  if (blockIdx.x == 0 && threadIdx.x == 0) *n_cand = total;
  for (int q = blockIdx.x * blockDim.x + threadIdx.x; q < n_slots; q += gridDim.x * blockDim.x) {
    if (q >= total) {
      *reinterpret_cast<float4*>(cand_boxes + (size_t)q * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
      cand_scores[q] = 0.f;
      cand_labels[q] = -1;
      cand_loc[q] = -1;
      continue;
    }
    int l = 0;
    while (q >= off[l + 1]) ++l;
    const int p = sel[L.sel_off[l] + (q - off[l])];
    const int i = p / C, c = p - i * C;
    const smb_level_t& lv = L.lv[l];
    const float s = __fmul_rn(sigmoid_rn(lv.cls[(size_t)i * lv.cls_pitch + c]), sigmoid_rn(lv.ctr[(size_t)i * lv.ctr_pitch]));
    const int y = i / lv.w, x = i - y * lv.w;
    const float px = (float)(x * lv.stride + lv.stride / 2), py = (float)(y * lv.stride + lv.stride / 2);
    const float* d = lv.box + (size_t)i * lv.box_pitch;
    float dd[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) dd[k] = __fmul_rn(fmaxf(__fmul_rn(d[k], lv.box_scale), 0.f), lv.box_mul);
    const float mw = (float)(g.img_w - 1), mh = (float)(g.img_h - 1);
    const float x1 = fminf(fmaxf(__fsub_rn(px, dd[0]), 0.f), mw), y1 = fminf(fmaxf(__fsub_rn(py, dd[1]), 0.f), mh);
    const float x2 = fminf(fmaxf(__fadd_rn(px, dd[2]), 0.f), mw), y2 = fminf(fmaxf(__fadd_rn(py, dd[3]), 0.f), mh);
    *reinterpret_cast<float4*>(cand_boxes + (size_t)q * 4) = make_float4(x1, y1, x2, y2);
    cand_scores[q] = __fsqrt_rn(s);
    cand_labels[q] = c;
    cand_loc[q] = L.loc_off[l] + i;
  }
}

// Label-aware NMS, stage 1 (one CTA): n = clamp(*n_dev, 0, cap) candidates sorted by descending score, ties by ascending
// index.  Writes the mc_* layout of one list so that mc_sweep_kernel can run the sweep.
__global__ void __launch_bounds__(NT) ml_prepare_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                        const int* __restrict__ labels, const int* __restrict__ n_dev, int cap,
                                                        int* __restrict__ w_cidx, float* __restrict__ w_cscore,
                                                        unsigned long long* __restrict__ w_keys, float4* __restrict__ w_sbox,
                                                        int* __restrict__ w_slab, int* __restrict__ w_m) {
  pdl_wait();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);     // [next pow2 of MAXN]
  const int n = min(max(*n_dev, 0), cap);
  if (threadIdx.x == 0) *w_m = n;
  if (n == 0) return;
  int P = 1;
  while (P < n) P <<= 1;
  for (int i = threadIdx.x; i < P; i += NT) keys[i] = (i < n) ? desc_key(scores[i], (unsigned)i) : ~0ull;
  cta_bitonic_sort(keys, P, Less());
  for (int r = threadIdx.x; r < n; r += NT) {
    const unsigned long long k = keys[r];
    const int i = (int)(k & 0xffffffffu);
    w_keys[r] = k;
    w_sbox[r] = *reinterpret_cast<const float4*>(boxes + (size_t)i * 4);
    w_slab[r] = labels[i];
    w_cidx[r] = r;                   // positions are candidate indices: the sweep returns kept candidates ascending
    w_cscore[r] = scores[r];
  }
}

// Stage 2: suppression bit-matrix over 64x64 tiles of the upper triangle; IoU is 0 across labels (ml_nms.cu:13-24).
__global__ void __launch_bounds__(64) ml_mask_kernel(const float4* __restrict__ w_sbox, const int* __restrict__ w_slab,
                                                     const int* __restrict__ w_m, int nbmax, float iou_thr,
                                                     unsigned long long* __restrict__ mask) {
  pdl_wait();
  __shared__ float4 s_col[64];
  __shared__ int s_lab[64];
  const int m = min(*w_m, nbmax * 64);
  const int nb = (m + 63) >> 6;
  const int total = nb * (nb + 1) / 2;
  for (int t = blockIdx.x; t < total; t += gridDim.x) {
    int u = t, rb = 0;
    while (u >= nb - rb) { u -= nb - rb; ++rb; }
    const int cb = rb + u;
    const int col = cb * 64 + threadIdx.x;
    s_col[threadIdx.x] = (col < m) ? w_sbox[col] : make_float4(0.f, 0.f, 0.f, 0.f);
    s_lab[threadIdx.x] = (col < m) ? w_slab[col] : -1;
    __syncthreads();
    const int row = rb * 64 + threadIdx.x;
    if (row < m) {
      const float4 a = w_sbox[row];
      const int la = w_slab[row];
      unsigned long long bits = 0ull;
      const int lim = min(64, m - cb * 64);
      const int start = (rb == cb) ? threadIdx.x + 1 : 0;
      for (int q = start; q < lim; ++q) {
        const float v = (s_lab[q] != la) ? 0.f : iou_ref(a, s_col[q], 1.0f);
        if (v > iou_thr) bits |= 1ull << q;
      }
      mask[(size_t)row * nbmax + cb] = bits;
    }
    __syncthreads();
  }
}

// Stage 4 (one CTA): survivors (ascending candidate index) -> k-th-value cut at max_per_img (keep score >= the
// max_per_img-th largest, inference.py:182-190; ties can keep more) -> first out_cap rows, count = min(kept, out_cap),
// kept_total = kept.  Rows past the count: zeros, label / index -1.
__global__ void __launch_bounds__(NT) ml_finalize_kernel(const float* __restrict__ boxes, const int* __restrict__ labels,
                                                         const int* __restrict__ ws_idx, const float* __restrict__ ws_score,
                                                         const int* __restrict__ ws_count, int cap, int max_per_img,
                                                         int out_cap, float* __restrict__ det_out,
                                                         long long* __restrict__ label_out, long long* __restrict__ idx_out,
                                                         int* __restrict__ count_out, int* __restrict__ kept_total_out) {
  pdl_wait();
  __shared__ SelectSmem s_select;
  __shared__ int s_warp[32];
  const int K = min(max(*ws_count, 0), cap);
  float thr = -INFINITY;
  if (max_per_img > 0 && K > max_per_img) {
    // the max_per_img-th largest score: the max_per_img-th smallest key, resolved in its top 32 bits (the score)
    const auto key_at = [&](int g) { return desc_key(ws_score[g], 0u); };
    thr = key_score(cta_radix_select<NT, unsigned long long, 4>(K, max_per_img, key_at, s_select).key);
  }
  int running = 0;
  for (int base = 0; base < K; base += NT) {
    const int g = base + threadIdx.x;
    const float s = (g < K) ? ws_score[g] : 0.f;
    const int f = (g < K) && (s >= thr);
    int tot;
    const int pos = running + cta_exclusive_scan<NT>(f, Sum(), 0, s_warp, &tot);
    if (f && pos < out_cap) {
      const int i = ws_idx[g];
      const float4 b = *reinterpret_cast<const float4*>(boxes + (size_t)i * 4);
      det_out[pos * 5 + 0] = b.x; det_out[pos * 5 + 1] = b.y; det_out[pos * 5 + 2] = b.z; det_out[pos * 5 + 3] = b.w;
      det_out[pos * 5 + 4] = s;
      label_out[pos] = labels[i];
      idx_out[pos] = i;
    }
    running += tot;
  }
  const int count = min(running, out_cap);
  for (int r = count + threadIdx.x; r < out_cap; r += NT) {
    for (int q = 0; q < 5; ++q) det_out[r * 5 + q] = 0.f;
    label_out[r] = -1;
    idx_out[r] = -1;
  }
  if (threadIdx.x == 0) { *count_out = count; *kept_total_out = running; }
}

// ---------------------------------------------------------------------------------------------
// Soft-NMS (ops/nms/src/nms_cpu.cpp:70-209, nms_wrapper.py:63-118), one list per CTA, bit for bit in float32.
// The reference runs one O(n^2) loop per list: iteration i swaps the first maximum of [i, N) into slot i, then decays every
// score of [i+1, N) by a weight of its IoU with box i and removes a decayed score below min_score by copying the element at
// N-1 into its slot (N--).  Every element of [i+1, N) is decayed exactly once and its decay depends only on itself and box
// i, so the pass runs in parallel: with S survivors, those in [i+1, i+1+S) keep their slots and the k-th hole there
// (ascending) receives the k-th survivor of [i+1+S, N) counted from the back, which is the array the sequential
// swap-with-last leaves.  The next maximum is then the first maximum by new slot, reduced in the same pass.
// ---------------------------------------------------------------------------------------------
constexpr int SNT = 512;                     // threads per soft-NMS CTA
constexpr int SOFT_LINEAR = 1, SOFT_GAUSSIAN = 2;
static_assert(MAXN <= 32 * SNT, "a thread's slots of one pass are tracked in one 32-bit mask");

struct SoftSmem {
  float4 box[MAXN];
  float score[MAXN];
  int id[MAXN];                              // what the output reports for the element: input index or candidate row
  int hole[MAXN];                            // slots of removed elements in [i+1, i+1+S), ascending
  unsigned long long tab[32];
  float best_v[SNT / 32];
  int best_p[SNT / 32];
  int warp[SNT / 32];
  int sel;
};

// expf as glibc >= 2.27 computes it on an FMA host (the table-driven exp2 of Szabolcs Nagy's optimized routines): x / ln2
// scaled by 32, rounded to an integer k by the 1.5 * 2^52 shift, 2^(k/32) from a 32-entry table and a degree-3 polynomial
// of the remainder in double, one rounding to float at the end.  tab[j] = bits(2^(j/32)) - (j << 47).
__constant__ unsigned long long c_exp2_tab[32] = {
    0x3ff0000000000000ULL, 0x3fefd9b0d3158574ULL, 0x3fefb5586cf9890fULL, 0x3fef9301d0125b51ULL, 0x3fef72b83c7d517bULL,
    0x3fef54873168b9aaULL, 0x3fef387a6e756238ULL, 0x3fef1e9df51fdee1ULL, 0x3fef06fe0a31b715ULL, 0x3feef1a7373aa9cbULL,
    0x3feedea64c123422ULL, 0x3feece086061892dULL, 0x3feebfdad5362a27ULL, 0x3feeb42b569d4f82ULL, 0x3feeab07dd485429ULL,
    0x3feea47eb03a5585ULL, 0x3feea09e667f3bcdULL, 0x3fee9f75e8ec5f74ULL, 0x3feea11473eb0187ULL, 0x3feea589994cce13ULL,
    0x3feeace5422aa0dbULL, 0x3feeb737b0cdc5e5ULL, 0x3feec49182a3f090ULL, 0x3feed503b23e255dULL, 0x3feee89f995ad3adULL,
    0x3feeff76f2fb5e47ULL, 0x3fef199bdd85529cULL, 0x3fef3720dcef9069ULL, 0x3fef5818dcfba487ULL, 0x3fef7c97337b9b5fULL,
    0x3fefa4afa2a490daULL, 0x3fefd0765b6e4540ULL};

__device__ __forceinline__ float expf_host(float x, const unsigned long long* tab) {
  if (!(x >= -0x1.9fe368p6f)) return (x != x) ? x + x : 0.f;     // NaN; -inf and results below 2^-150 round to 0
  if (x > 0x1.62e42ep6f) return INFINITY;                         // above log(2^128)
  const double inv_ln2_n = 0x1.71547652b82fep+0 * 32, shift = 0x1.8p+52;
  const double c0 = 0x1.c6af84b912394p-5 / (32.0 * 32.0 * 32.0), c1 = 0x1.ebfce50fac4f3p-3 / (32.0 * 32.0),
               c2 = 0x1.62e42ff0c52d6p-1 / 32.0;
  const double xd = (double)x;
  // the FMA build contracts both uses of x * 32/ln2, so the product is never rounded on its own
  double kd = __fma_rn(inv_ln2_n, xd, shift);
  const unsigned long long ki = (unsigned long long)__double_as_longlong(kd);
  kd = __dsub_rn(kd, shift);
  const double r = __fma_rn(inv_ln2_n, xd, -kd);
  const double s = __longlong_as_double((long long)(tab[ki & 31] + (ki << 47)));
  const double p = __fma_rn(c0, r, c1);
  const double r2 = __dmul_rn(r, r);
  double y = __fma_rn(c2, r, 1.0);
  y = __fma_rn(p, r2, y);
  return __double2float_rn(__dmul_rn(y, s));
}

// nms_cpu.cpp's area and overlap: std::max / std::min comparisons, `+ 1`, every operation rounded on its own
__device__ __forceinline__ float soft_area(const float4 b) {
  return __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.f), __fadd_rn(__fsub_rn(b.w, b.y), 1.f));
}
__device__ __forceinline__ float soft_weight(const float4 a, float area_a, const float4 b, float thr, int method, float sigma,
                                             const unsigned long long* tab) {
  const float xx1 = (a.x < b.x) ? b.x : a.x, yy1 = (a.y < b.y) ? b.y : a.y;
  const float xx2 = (b.z < a.z) ? b.z : a.z, yy2 = (b.w < a.w) ? b.w : a.w;
  const float tw = __fadd_rn(__fsub_rn(xx2, xx1), 1.f), th = __fadd_rn(__fsub_rn(yy2, yy1), 1.f);
  const float w = (0.f < tw) ? tw : 0.f, h = (0.f < th) ? th : 0.f;
  const float inter = __fmul_rn(w, h);
  const float ovr = __fdiv_rn(inter, __fsub_rn(__fadd_rn(area_a, soft_area(b)), inter));
  if (method == SOFT_LINEAR) return (ovr > thr) ? __fsub_rn(1.f, ovr) : 1.f;
  return expf_host(__fdiv_rn(-__fmul_rn(ovr, ovr), sigma), tab);
}

// (v, p) beats the best so far when it is larger, or equal at an earlier slot; p == INT_MAX is "none".  NaN never enters.
__device__ __forceinline__ void soft_better(float& bv, int& bp, float v, int p) {
  if (p != INT_MAX && (bp == INT_MAX || v > bv || (v == bv && p < bp))) { bv = v; bp = p; }
}

// CTA-wide first maximum; the slot lands in S.sel (INT_MAX when no thread had a candidate).
__device__ __forceinline__ void soft_argmax(SoftSmem& S, float v, int p) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) soft_better(v, p, __shfl_down_sync(0xffffffffu, v, o), __shfl_down_sync(0xffffffffu, p, o));
  if (lane == 0) { S.best_v[wid] = v; S.best_p[wid] = p; }
  __syncthreads();
  if (wid == 0) {
    v = -INFINITY; p = INT_MAX;
    if (lane < SNT / 32) { v = S.best_v[lane]; p = S.best_p[lane]; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) soft_better(v, p, __shfl_down_sync(0xffffffffu, v, o), __shfl_down_sync(0xffffffffu, p, o));
    if (lane == 0) S.sel = p;
  }
  __syncthreads();
}

// Soft-NMS of the m elements in S (slots [0, m)); returns the number kept, in selection order in slots [0, return).
__device__ __forceinline__ int soft_nms_run(SoftSmem& S, int m, float thr, int method, float sigma, float min_score) {
  for (int k = threadIdx.x; k < 32; k += SNT) S.tab[k] = c_exp2_tab[k];
  {
    const int E = (m + SNT - 1) / SNT, j0 = threadIdx.x * E, j1 = min(j0 + E, m);
    float bv = -INFINITY;
    int bp = INT_MAX;
    for (int j = j0; j < j1; ++j) {
      const float s = S.score[j];
      if (s == s) soft_better(bv, bp, s, j);
    }
    soft_argmax(S, bv, bp);
  }
  int N = m;
  for (int i = 0; i < N; ++i) {
    if (threadIdx.x == 0) {
      // `if (max_score < scores[pos])` from max_score = scores[i]: a NaN at slot i is kept there, a NaN later never wins
      const int p = (S.score[i] != S.score[i] || S.sel == INT_MAX) ? i : S.sel;
      if (p != i) {
        const float4 b = S.box[i]; const float s = S.score[i]; const int d = S.id[i];
        S.box[i] = S.box[p]; S.score[i] = S.score[p]; S.id[i] = S.id[p];
        S.box[p] = b; S.score[p] = s; S.id[p] = d;
      }
    }
    __syncthreads();
    const int len = N - i - 1;
    if (len == 0) break;
    const float4 bi = S.box[i];
    const float ai = soft_area(bi);
    const int E = (len + SNT - 1) / SNT, j0 = i + 1 + threadIdx.x * E, j1 = min(j0 + E, N);
    unsigned rm = 0u;
    int surv = 0;
    float bv = -INFINITY;
    int bp = INT_MAX;
    for (int j = j0; j < j1; ++j) {
      // a NaN score stays the same NaN (x86 returns the NaN operand of a product; the device would canonicalise it)
      const float sj = S.score[j];
      const float s = (sj != sj) ? sj : __fmul_rn(soft_weight(bi, ai, S.box[j], thr, method, sigma, S.tab), sj);
      S.score[j] = s;
      if (s < min_score) {
        rm |= 1u << (j - j0);
      } else {
        ++surv;
        if (s == s) soft_better(bv, bp, s, j);
      }
    }
    int S_tot;
    cta_inclusive_scan<SNT>(surv, Sum(), S.warp, &S_tot);
    const int fend = i + 1 + S_tot;
    if (S_tot < len) {
      int holes = 0, backs = 0;
      for (int j = j0; j < j1; ++j) {
        const bool r = (rm >> (j - j0)) & 1u;
        holes += (r && j < fend);
        backs += (!r && j >= fend);
      }
      int tot;
      const int ex = cta_exclusive_scan<SNT>((holes << 16) | backs, Sum(), 0, S.warp, &tot);
      int hr = ex >> 16, br = ex & 0xffff;
      const int nback = tot & 0xffff;
      for (int j = j0; j < j1; ++j)
        if (((rm >> (j - j0)) & 1u) && j < fend) S.hole[hr++] = j;
      __syncthreads();
      bv = -INFINITY; bp = INT_MAX;
      for (int j = j0; j < j1; ++j) {
        if ((rm >> (j - j0)) & 1u) continue;
        int t = j;
        if (j >= fend) {
          t = S.hole[min(max(nback - 1 - br++, 0), MAXN - 1)];
          S.box[t] = S.box[j]; S.score[t] = S.score[j]; S.id[t] = S.id[j];
        }
        const float s = S.score[t];
        if (s == s) soft_better(bv, bp, s, t);
      }
    }
    N = fend;
    soft_argmax(S, bv, bp);
  }
  __syncthreads();
  return N;
}

// smb_soft_nms: one list dets [n,5] -> dets_out [n,5] (kept rows in selection order, decayed scores), inds_out [n].
__global__ void __launch_bounds__(SNT, 1) soft_nms_single_kernel(const float* __restrict__ dets, int n, float thr, int method,
                                                              float sigma, float min_score, float* __restrict__ dets_out,
                                                              long long* __restrict__ inds_out, int* __restrict__ count_out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SoftSmem& S = *reinterpret_cast<SoftSmem*>(smem_raw);
  const int m = min(n, MAXN);
  for (int j = threadIdx.x; j < m; j += SNT) {
    S.box[j] = make_float4(dets[j * 5], dets[j * 5 + 1], dets[j * 5 + 2], dets[j * 5 + 3]);
    S.score[j] = dets[j * 5 + 4];
    S.id[j] = j;
  }
  __syncthreads();
  const int k = soft_nms_run(S, m, thr, method, sigma, min_score);
  for (int j = threadIdx.x; j < k; j += SNT) {
    const float4 b = S.box[j];
    dets_out[j * 5 + 0] = b.x; dets_out[j * 5 + 1] = b.y; dets_out[j * 5 + 2] = b.z; dets_out[j * 5 + 3] = b.w;
    dets_out[j * 5 + 4] = S.score[j];
    inds_out[j] = S.id[j];
  }
  if (threadIdx.x == 0) *count_out = k;
}

// Multi-class soft-NMS, stage 1: one CTA per class.  The class list is mc_prepare_kernel's compaction (raw score > thr,
// score * ctr, ascending candidate row, bbox_nms.py:111-124); its survivors go to ws_idx / ws_score [C][n] in selection
// order with ws_count[c], the layout finalize_kernel reads.
__global__ void __launch_bounds__(SNT, 1) mc_soft_nms_kernel(const float* __restrict__ boxes, const float* __restrict__ scores,
                                                          const float* __restrict__ ctr, int n, int C, float score_thr,
                                                          float thr, int method, float sigma, float min_score,
                                                          int* __restrict__ ws_idx, float* __restrict__ ws_score,
                                                          int* __restrict__ ws_count) {
  pdl_wait();
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SoftSmem& S = *reinterpret_cast<SoftSmem*>(smem_raw);
  const int c = blockIdx.x;
  const int nn = min(n, MAXN);
  int m = 0;
  for (int base = 0; base < nn; base += SNT) {
    const int i = base + threadIdx.x;
    float s = 0.f;
    int f = 0;
    if (i < nn) { s = scores[(size_t)i * C + c]; f = s > score_thr; }
    int tot;
    const int ex = cta_exclusive_scan<SNT>(f, Sum(), 0, S.warp, &tot);
    if (f) {
      S.id[m + ex] = i;
      S.score[m + ex] = __fmul_rn(s, ctr[i]);
      S.box[m + ex] = *reinterpret_cast<const float4*>(boxes + (size_t)i * 4);
    }
    m += tot;
    __syncthreads();
  }
  const int k = soft_nms_run(S, m, thr, method, sigma, min_score);
  for (int j = threadIdx.x; j < k; j += SNT) {
    ws_idx[(size_t)c * n + j] = S.id[j];
    ws_score[(size_t)c * n + j] = S.score[j];
  }
  if (threadIdx.x == 0) ws_count[c] = k;
}

static int fill_levels(Levels* L, int num_levels, const smb_level_t* host_levels, int nms_pre) {
  if (num_levels < 1 || num_levels > MAXLVL) return -1;
  L->num = num_levels;
  L->loc_off[0] = 0;
  L->cand_off[0] = 0;
  for (int l = 0; l < num_levels; ++l) {
    L->lv[l] = host_levels[l];
    const int hw = host_levels[l].h * host_levels[l].w;
    if (hw <= 0) return -1;
    L->loc_off[l + 1] = L->loc_off[l] + hw;
    L->cand_off[l + 1] = L->cand_off[l] + ((nms_pre > 0 && hw > nms_pre) ? nms_pre : hw);
  }
  return 0;
}

}  // namespace smb

using namespace smb;

extern "C" int smb_nms(const float* dets, int n, float iou_thr, int cmp_ge, int plus_one, int64_t* keep_out,
                       int* n_keep_out, smb_stream_t stream) {
  SMB_CHECK_ARG(n >= 0 && n <= NMS1, "smb_nms: n=%d outside [0,%d]", n, NMS1);
  SMB_CHECK_ARG(keep_out && n_keep_out && (dets || n == 0), "smb_nms: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    SMB_CUDA_OK(cudaMemsetAsync(n_keep_out, 0, sizeof(int), st));
    return SMB_OK;
  }
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(nms_single_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(NmsSmem)));
  }
  nms_single_kernel<<<1, NT, sizeof(NmsSmem), st>>>(dets, n, iou_thr, cmp_ge, plus_one ? 1.f : 0.f,
                                                    (long long*)keep_out, n_keep_out);
  SMB_LAUNCH_OK("nms_single_kernel");
  return SMB_OK;
}

struct McWs {
  size_t idx, score, count, gkey, gval, cidx, cscore, keys, sbox, m, mask, total;
};

static McWs mc_ws_layout(int n, int C, bool with_mask) {
  McWs w;
  size_t off = 0;
  w.idx = off;    off = align_up(off + (size_t)C * n * sizeof(int), 256);
  w.score = off;  off = align_up(off + (size_t)C * n * sizeof(float), 256);
  w.count = off;  off = align_up(off + (size_t)(C + 1) * sizeof(int), 256);
  w.gkey = off;   off = align_up(off + (size_t)C * n * sizeof(unsigned long long), 256);
  w.gval = off;   off = align_up(off + (size_t)C * n * sizeof(int), 256);
  w.cidx = w.cscore = w.keys = w.sbox = w.m = w.mask = off;
  if (with_mask) {
    const int nbmax = (n + 63) / 64;
    w.cidx = off;   off = align_up(off + (size_t)C * n * sizeof(int), 256);
    w.cscore = off; off = align_up(off + (size_t)C * n * sizeof(float), 256);
    w.keys = off;   off = align_up(off + (size_t)C * n * sizeof(unsigned long long), 256);
    w.sbox = off;   off = align_up(off + (size_t)C * n * sizeof(float4), 256);
    w.m = off;      off = align_up(off + (size_t)(C + 1) * sizeof(int), 256);
    w.mask = off;   off = align_up(off + (size_t)C * n * nbmax * sizeof(unsigned long long), 256);
  }
  w.total = off;
  return w;
}

extern "C" size_t smb_multiclass_nms_workspace_bytes(int n, int num_classes) {
  return mc_ws_layout(n > 0 ? n : 1, num_classes, true).total;
}

extern "C" int smb_multiclass_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                                  float score_thr, float iou_thr, int max_num, int cmp_ge, float* det_out,
                                  int64_t* label_out, int64_t* idx_out, int* count_out, void* workspace,
                                  size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n >= 0 && n <= MAXN, "smb_multiclass_nms: n=%d outside [0,%d]", n, MAXN);
  SMB_CHECK_ARG(num_classes >= 1 && num_classes <= 1024, "smb_multiclass_nms: num_classes=%d", num_classes);
  SMB_CHECK_ARG(max_num >= 1 && max_num <= 1024, "smb_multiclass_nms: max_num=%d outside [1,1024]", max_num);
  SMB_CHECK_ARG(det_out && label_out && idx_out && count_out && workspace, "smb_multiclass_nms: null pointer");
  const int nn = n > 0 ? n : 1;
  const McWs w = mc_ws_layout(nn, num_classes, true);
  if (workspace_bytes < w.total) {
    set_error("smb_multiclass_nms: workspace %zu < %zu", workspace_bytes, w.total);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int* ws_count = (int*)(ws + w.count);
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(mc_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(McPrepSmem)));
  }
  if (n == 0) {
    SMB_CUDA_OK(cudaMemsetAsync(ws_count, 0, sizeof(int) * (num_classes + 1), st));
  } else {
    const int nbmax = (n + 63) / 64;
    mc_prepare_kernel<<<num_classes, NT, sizeof(McPrepSmem), st>>>(boxes, scores, ctr, n, num_classes, score_thr, (int*)(ws + w.cidx),
                                                                   (float*)(ws + w.cscore), (unsigned long long*)(ws + w.keys),
                                                                   (float4*)(ws + w.sbox), (int*)(ws + w.m));
    SMB_LAUNCH_OK("mc_prepare_kernel");
    mc_mask_kernel<<<132 * 16, 64, 0, st>>>((const float4*)(ws + w.sbox), (const int*)(ws + w.m), n, num_classes, nbmax, iou_thr,
                                            cmp_ge, (unsigned long long*)(ws + w.mask));
    SMB_LAUNCH_OK("mc_mask_kernel");
    mc_sweep_kernel<<<num_classes, NT, 0, st>>>((const unsigned long long*)(ws + w.mask), (const unsigned long long*)(ws + w.keys),
                                                (const int*)(ws + w.cidx), (const float*)(ws + w.cscore), (const int*)(ws + w.m), n,
                                                nbmax, (int*)(ws + w.idx), (float*)(ws + w.score), ws_count);
    SMB_LAUNCH_OK("mc_sweep_kernel");
  }
  finalize_kernel<<<1, NT, 0, st>>>(boxes, n, num_classes, max_num, 0, (const int*)(ws + w.idx), (const float*)(ws + w.score),
                                    ws_count, nn, (unsigned long long*)(ws + w.gkey), (int*)(ws + w.gval), det_out,
                                    (long long*)label_out, (long long*)idx_out, count_out);
  SMB_LAUNCH_OK("finalize_kernel");
  return SMB_OK;
}

static int soft_nms_attr() {
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(soft_nms_single_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SoftSmem)));
    SMB_CUDA_OK(cudaFuncSetAttribute(mc_soft_nms_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(SoftSmem)));
  }
  return SMB_OK;
}

extern "C" int smb_soft_nms(const float* dets, int n, float iou_thr, int method, float sigma, float min_score, float* dets_out,
                            int64_t* inds_out, int* count_out, smb_stream_t stream) {
  SMB_CHECK_ARG(n >= 0 && n <= MAXN, "smb_soft_nms: n=%d outside [0,%d]", n, MAXN);
  SMB_CHECK_ARG(method == SOFT_LINEAR || method == SOFT_GAUSSIAN, "smb_soft_nms: method=%d (1 linear, 2 gaussian)", method);
  SMB_CHECK_ARG(count_out && (n == 0 || (dets && dets_out && inds_out)), "smb_soft_nms: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  if (n == 0) {
    SMB_CUDA_OK(cudaMemsetAsync(count_out, 0, sizeof(int), st));
    return SMB_OK;
  }
  const int rc = soft_nms_attr();
  if (rc != SMB_OK) return rc;
  soft_nms_single_kernel<<<1, SNT, sizeof(SoftSmem), st>>>(dets, n, iou_thr, method, sigma, min_score, dets_out,
                                                           (long long*)inds_out, count_out);
  SMB_LAUNCH_OK("soft_nms_single_kernel");
  return SMB_OK;
}

extern "C" size_t smb_multiclass_soft_nms_workspace_bytes(int n, int num_classes) {
  return mc_ws_layout(n > 0 ? n : 1, num_classes, false).total;
}

extern "C" int smb_multiclass_soft_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                                       float score_thr, float iou_thr, int max_num, int method, float sigma, float min_score,
                                       float* det_out, int64_t* label_out, int64_t* idx_out, int* count_out, void* workspace,
                                       size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n >= 0 && n <= MAXN, "smb_multiclass_soft_nms: n=%d outside [0,%d]", n, MAXN);
  SMB_CHECK_ARG(num_classes >= 1 && num_classes <= 1024, "smb_multiclass_soft_nms: num_classes=%d", num_classes);
  SMB_CHECK_ARG(max_num >= 1 && max_num <= 1024, "smb_multiclass_soft_nms: max_num=%d outside [1,1024]", max_num);
  SMB_CHECK_ARG(method == SOFT_LINEAR || method == SOFT_GAUSSIAN, "smb_multiclass_soft_nms: method=%d (1 linear, 2 gaussian)",
                method);
  SMB_CHECK_ARG(det_out && label_out && idx_out && count_out && workspace, "smb_multiclass_soft_nms: null pointer");
  const int nn = n > 0 ? n : 1;
  const McWs w = mc_ws_layout(nn, num_classes, false);
  if (workspace_bytes < w.total) {
    set_error("smb_multiclass_soft_nms: workspace %zu < %zu", workspace_bytes, w.total);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int* ws_count = (int*)(ws + w.count);
  if (n == 0) {
    SMB_CUDA_OK(cudaMemsetAsync(ws_count, 0, sizeof(int) * (num_classes + 1), st));
  } else {
    const int rc = soft_nms_attr();
    if (rc != SMB_OK) return rc;
    mc_soft_nms_kernel<<<num_classes, SNT, sizeof(SoftSmem), st>>>(boxes, scores, ctr, n, num_classes, score_thr, iou_thr,
                                                                   method, sigma, min_score, (int*)(ws + w.idx),
                                                                   (float*)(ws + w.score), ws_count);
    SMB_LAUNCH_OK("mc_soft_nms_kernel");
  }
  finalize_kernel<<<1, NT, 0, st>>>(boxes, n, num_classes, max_num, 0, (const int*)(ws + w.idx), (const float*)(ws + w.score),
                                    ws_count, nn, (unsigned long long*)(ws + w.gkey), (int*)(ws + w.gval), det_out,
                                    (long long*)label_out, (long long*)idx_out, count_out);
  SMB_LAUNCH_OK("finalize_kernel");
  return SMB_OK;
}

extern "C" size_t smb_fast_nms_workspace_bytes(int n, int num_classes, int top_k) {
  (void)n;
  return mc_ws_layout(top_k, num_classes, false).total;
}

extern "C" int smb_fast_nms(const float* boxes, const float* scores, const float* ctr, int n, int num_classes,
                            float score_thr, float iou_thr, int top_k, int max_num, float* det_out, int64_t* label_out,
                            int64_t* idx_out, int* count_out, void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(n >= 1 && n <= MAXN, "smb_fast_nms: n=%d outside [1,%d]", n, MAXN);
  SMB_CHECK_ARG(top_k >= 1 && top_k <= 256, "smb_fast_nms: top_k=%d outside [1,256]", top_k);
  SMB_CHECK_ARG(num_classes >= 1 && num_classes <= 1024 && max_num >= 1 && max_num <= 1024, "smb_fast_nms: bad sizes");
  SMB_CHECK_ARG(det_out && label_out && idx_out && count_out && workspace, "smb_fast_nms: null pointer");
  const McWs w = mc_ws_layout(top_k, num_classes, false);
  const size_t o_idx = w.idx, o_score = w.score, o_count = w.count, o_gkey = w.gkey, o_gval = w.gval;
  if (workspace_bytes < w.total) {
    set_error("smb_fast_nms: workspace %zu < %zu", workspace_bytes, w.total);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(fast_nms_class_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(FastSmem)));
  }
  fast_nms_class_kernel<<<num_classes, NT, sizeof(FastSmem), st>>>(boxes, scores, ctr, n, num_classes, score_thr, iou_thr, top_k,
                                                                   (int*)(ws + o_idx), (float*)(ws + o_score), (int*)(ws + o_count));
  SMB_LAUNCH_OK("fast_nms_class_kernel");
  finalize_kernel<<<1, NT, 0, st>>>(boxes, n, num_classes, max_num, 1, (const int*)(ws + o_idx), (const float*)(ws + o_score),
                                    (const int*)(ws + o_count), top_k, (unsigned long long*)(ws + o_gkey), (int*)(ws + o_gval),
                                    det_out, (long long*)label_out, (long long*)idx_out, count_out);
  SMB_LAUNCH_OK("finalize_kernel");
  return SMB_OK;
}

extern "C" size_t smb_decode_workspace_bytes(int num_levels, const smb_level_t* host_levels, int nms_pre) {
  Levels L;
  if (fill_levels(&L, num_levels, host_levels, nms_pre)) return 0;
  return align_up((size_t)L.loc_off[L.num] * sizeof(float), 256) + align_up((size_t)L.cand_off[L.num] * sizeof(int), 256);
}

static int decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre, GeomArg ga,
                       float* cand_boxes, float* cand_scores, float* cand_ctr, int* cand_loc, void* workspace,
                       size_t workspace_bytes, smb_stream_t stream) {
  Levels L;
  SMB_CHECK_ARG(fill_levels(&L, num_levels, host_levels, nms_pre) == 0, "smb_decode_topk: bad levels");
  SMB_CHECK_ARG(nms_pre <= 1024, "smb_decode_topk: nms_pre=%d > 1024", nms_pre);
  SMB_CHECK_ARG(cand_boxes && cand_scores && cand_ctr && cand_loc && workspace, "smb_decode_topk: null pointer");
  const size_t s_bytes = align_up((size_t)L.loc_off[L.num] * sizeof(float), 256);
  const size_t need = s_bytes + align_up((size_t)L.cand_off[L.num] * sizeof(int), 256);
  if (workspace_bytes < need) {
    set_error("smb_decode_topk: workspace %zu < %zu", workspace_bytes, need);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  float* s = (float*)workspace;
  int* sel = (int*)((char*)workspace + s_bytes);
  const int total = L.loc_off[L.num];
  level_score_kernel<<<min(cdiv(total, 8), 132 * 8), 256, 0, st>>>(L, num_classes, s);
  SMB_LAUNCH_OK("level_score_kernel");
  level_topk_kernel<<<num_levels, NT, 0, st>>>(L, nms_pre, s, sel);
  SMB_LAUNCH_OK("level_topk_kernel");
  const int ncand = L.cand_off[L.num];
  gather_decode_kernel<<<min(cdiv(ncand, 8), 132 * 8), 256, 0, st>>>(L, num_classes, ga, sel, cand_boxes, cand_scores,
                                                                    cand_ctr, cand_loc);
  SMB_LAUNCH_OK("gather_decode_kernel");
  return SMB_OK;
}

extern "C" int smb_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre, int img_h,
                               int img_w, const float* host_scale4, float* cand_boxes, float* cand_scores,
                               float* cand_ctr, int* cand_loc, void* workspace, size_t workspace_bytes,
                               smb_stream_t stream) {
  smb_img_geom_t g;
  memset(&g, 0, sizeof(g));
  g.img_h = img_h; g.img_w = img_w;
  for (int k = 0; k < 4; ++k) g.scale[k] = host_scale4 ? host_scale4[k] : 1.f;
  return decode_topk(num_levels, host_levels, num_classes, nms_pre, geom_value(g), cand_boxes, cand_scores, cand_ctr,
                     cand_loc, workspace, workspace_bytes, stream);
}

extern "C" int smb_decode_topk_dev(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre,
                                   const smb_img_geom_t* geom, float* cand_boxes, float* cand_scores, float* cand_ctr,
                                   int* cand_loc, void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(geom, "smb_decode_topk_dev: null geometry");
  return decode_topk(num_levels, host_levels, num_classes, nms_pre, geom_device(geom), cand_boxes, cand_scores, cand_ctr,
                     cand_loc, workspace, workspace_bytes, stream);
}

extern "C" int smb_gather_det_inputs(const float* cof_src, int cof_pitch, const int* cand_loc, const int64_t* idx,
                                     const float* det, const int* count_dev, int max_rows, int row_elems, float* det_cofs,
                                     float* det_boxes, int64_t* loc_out, int num_levels, const int* host_level_hw, int n_img,
                                     int img, smb_stream_t stream) {
  SMB_CHECK_ARG(cof_src && cand_loc && idx && det && count_dev && det_cofs && det_boxes && max_rows > 0 && row_elems >= 4,
                "smb_gather_det_inputs: bad argument");
  SMB_CHECK_ARG(num_levels >= 0 && num_levels <= MAXLVL && (num_levels == 0 || (host_level_hw && n_img >= 1 && img >= 0 && img < n_img)),
                "smb_gather_det_inputs: bad level table");
  LocMap lm;
  memset(&lm, 0, sizeof(lm));
  lm.num = num_levels; lm.n_img = n_img; lm.img = img;
  for (int l = 0; l < num_levels; ++l) lm.loc_off[l + 1] = lm.loc_off[l] + host_level_hw[l];
  gather_det_inputs_kernel<<<cdiv(max_rows * row_elems, 256), 256, 0, (cudaStream_t)stream>>>(
      cof_src, cof_pitch, cand_loc, (const long long*)idx, det, count_dev, max_rows, row_elems, det_cofs, det_boxes,
      (long long*)loc_out, lm);
  SMB_LAUNCH_OK("gather_det_inputs_kernel");
  return SMB_OK;
}

static int gather_track_feats(const float* track, int h, int w, int C, const float* det, const int* count_dev, int max_rows,
                              GeomArg ga, float feat_stride, float* out, smb_stream_t stream) {
  SMB_CHECK_ARG(track && det && count_dev && out && h > 0 && w > 0 && C > 0 && max_rows > 0 && feat_stride > 0.f,
                "smb_gather_track_feats: bad argument");
  gather_track_feats_kernel<<<cdiv(max_rows * C, 256), 256, 0, (cudaStream_t)stream>>>(track, h, w, C, det, count_dev, max_rows,
                                                                                         ga, feat_stride, out);
  SMB_LAUNCH_OK("gather_track_feats_kernel");
  return SMB_OK;
}

extern "C" int smb_gather_track_feats(const float* track, int h, int w, int C, const float* det, const int* count_dev,
                                      int max_rows, float scale_x, float scale_y, float feat_stride, float* out,
                                      smb_stream_t stream) {
  smb_img_geom_t g;
  memset(&g, 0, sizeof(g));
  g.track_sx = scale_x; g.track_sy = scale_y;
  return gather_track_feats(track, h, w, C, det, count_dev, max_rows, geom_value(g), feat_stride, out, stream);
}

extern "C" int smb_gather_track_feats_dev(const float* track, int h, int w, int C, const float* det, const int* count_dev,
                                          int max_rows, const smb_img_geom_t* geom, float feat_stride, float* out,
                                          smb_stream_t stream) {
  SMB_CHECK_ARG(geom, "smb_gather_track_feats_dev: null geometry");
  return gather_track_feats(track, h, w, C, det, count_dev, max_rows, geom_device(geom), feat_stride, out, stream);
}

extern "C" int smb_gather_rows_f32(const float* src, int src_pitch, const int64_t* idx, const int* count_dev, int max_rows,
                                   int row_elems, float* dst, smb_stream_t stream) {
  SMB_CHECK_ARG(src && idx && count_dev && dst && max_rows > 0 && row_elems > 0, "smb_gather_rows_f32: bad argument");
  gather_rows_kernel<<<cdiv(max_rows * row_elems, 256), 256, 0, (cudaStream_t)stream>>>(src, src_pitch, (const long long*)idx,
                                                                                         count_dev, max_rows, row_elems, dst);
  SMB_LAUNCH_OK("gather_rows_kernel");
  return SMB_OK;
}

// ------------------------------------------------------------------------------------ SipMask-benchmark entry points
static int fill_pair_levels(PairLevels* L, int num_levels, const smb_level_t* host_levels, int C, int nms_pre) {
  if (num_levels < 1 || num_levels > MAXLVL || C < 1 || C > 1024 || nms_pre < 1 || nms_pre > MAXN) return -1;
  L->num = num_levels;
  L->loc_off[0] = 0;
  L->pair_off[0] = 0;
  L->sel_off[0] = 0;
  for (int l = 0; l < num_levels; ++l) {
    L->lv[l] = host_levels[l];
    const long long hw = (long long)host_levels[l].h * host_levels[l].w;
    const long long np = hw * C;
    if (host_levels[l].h <= 0 || host_levels[l].w <= 0 || np >= (1LL << 31) - (long long)NT * PAIR_RUN) return -1;
    if (!host_levels[l].cls || !host_levels[l].ctr || !host_levels[l].box) return -1;
    L->loc_off[l + 1] = L->loc_off[l] + (int)hw;
    L->pair_off[l + 1] = L->pair_off[l] + np;
    L->sel_cap[l] = (int)(np < nms_pre ? np : nms_pre);
    L->sel_off[l + 1] = L->sel_off[l] + L->sel_cap[l];
    if ((long long)L->loc_off[l + 1] >= (1LL << 31)) return -1;
  }
  return 0;
}

struct PairWs {
  size_t keys, sel, count, total;
};
static PairWs pair_ws_layout(const PairLevels& L) {
  PairWs w;
  size_t off = 0;
  w.keys = off;  off = align_up(off + (size_t)L.pair_off[L.num] * sizeof(unsigned), 256);
  w.sel = off;   off = align_up(off + (size_t)L.sel_off[L.num] * sizeof(int), 256);
  w.count = off; off = align_up(off + (size_t)MAXLVL * sizeof(int), 256);
  w.total = off;
  return w;
}

extern "C" int smb_pair_decode_slots(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre) {
  PairLevels L;
  if (!host_levels || fill_pair_levels(&L, num_levels, host_levels, num_classes, nms_pre)) return SMB_EINVAL;
  return L.sel_off[L.num];
}

extern "C" size_t smb_pair_decode_workspace_bytes(int num_levels, const smb_level_t* host_levels, int num_classes,
                                                  int nms_pre) {
  PairLevels L;
  if (!host_levels || fill_pair_levels(&L, num_levels, host_levels, num_classes, nms_pre)) return 0;
  return pair_ws_layout(L).total;
}

static int pair_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, float score_thr, int nms_pre,
                            GeomArg ga, float* cand_boxes, float* cand_scores, int* cand_labels, int* cand_loc, int* n_cand,
                            int n_slots, void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  PairLevels L;
  SMB_CHECK_ARG(host_levels && fill_pair_levels(&L, num_levels, host_levels, num_classes, nms_pre) == 0,
                "smb_pair_decode_topk: bad levels (1..%d levels, 1 <= C <= 1024, 1 <= nms_pre <= %d, h*w*C < 2^31)",
                MAXLVL, MAXN);
  SMB_CHECK_ARG(cand_boxes && cand_scores && cand_labels && cand_loc && n_cand && workspace,
                "smb_pair_decode_topk: null pointer");
  SMB_CHECK_ARG(ga.dev || (ga.v.img_h > 0 && ga.v.img_w > 0), "smb_pair_decode_topk: img %dx%d", ga.v.img_h, ga.v.img_w);
  SMB_CHECK_ARG(n_slots >= L.sel_off[L.num], "smb_pair_decode_topk: n_slots=%d < %d", n_slots, L.sel_off[L.num]);
  const PairWs w = pair_ws_layout(L);
  if (workspace_bytes < w.total) {
    set_error("smb_pair_decode_topk: workspace %zu < %zu", workspace_bytes, w.total);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  unsigned* keys = (unsigned*)(ws + w.keys);
  int* sel = (int*)(ws + w.sel);
  int* cnt = (int*)(ws + w.count);
  const int total = L.loc_off[L.num];
  pair_key_kernel<<<min(cdiv(total, 8), 132 * 16), 256, 0, st>>>(L, num_classes, score_thr, keys);
  SMB_LAUNCH_OK("pair_key_kernel");
  pair_select_kernel<<<num_levels, NT, 0, st>>>(L, nms_pre, keys, sel, cnt);
  SMB_LAUNCH_OK("pair_select_kernel");
  pair_decode_kernel<<<max(1, min(cdiv(n_slots, 256), 132 * 4)), 256, 0, st>>>(L, num_classes, ga, sel, cnt, n_slots,
                                                                             cand_boxes, cand_scores, cand_labels, cand_loc,
                                                                             n_cand);
  SMB_LAUNCH_OK("pair_decode_kernel");
  return SMB_OK;
}

extern "C" int smb_pair_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, float score_thr,
                                    int nms_pre, int img_h, int img_w, float* cand_boxes, float* cand_scores,
                                    int* cand_labels, int* cand_loc, int* n_cand, int n_slots, void* workspace,
                                    size_t workspace_bytes, smb_stream_t stream) {
  smb_img_geom_t g;
  memset(&g, 0, sizeof(g));
  g.img_h = img_h; g.img_w = img_w;
  return pair_decode_topk(num_levels, host_levels, num_classes, score_thr, nms_pre, geom_value(g), cand_boxes, cand_scores,
                          cand_labels, cand_loc, n_cand, n_slots, workspace, workspace_bytes, stream);
}

extern "C" int smb_pair_decode_topk_dev(int num_levels, const smb_level_t* host_levels, int num_classes, float score_thr,
                                        int nms_pre, const smb_img_geom_t* geom, float* cand_boxes, float* cand_scores,
                                        int* cand_labels, int* cand_loc, int* n_cand, int n_slots, void* workspace,
                                        size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(geom, "smb_pair_decode_topk_dev: null geometry");
  return pair_decode_topk(num_levels, host_levels, num_classes, score_thr, nms_pre, geom_device(geom), cand_boxes,
                          cand_scores, cand_labels, cand_loc, n_cand, n_slots, workspace, workspace_bytes, stream);
}

struct MlWs {
  size_t cidx, cscore, keys, sbox, slab, m, mask, idx, score, count, total;
};
static MlWs ml_ws_layout(int cap) {
  MlWs w;
  const int nbmax = (cap + 63) / 64;
  size_t off = 0;
  w.cidx = off;   off = align_up(off + (size_t)cap * sizeof(int), 256);
  w.cscore = off; off = align_up(off + (size_t)cap * sizeof(float), 256);
  w.keys = off;   off = align_up(off + (size_t)cap * sizeof(unsigned long long), 256);
  w.sbox = off;   off = align_up(off + (size_t)cap * sizeof(float4), 256);
  w.slab = off;   off = align_up(off + (size_t)cap * sizeof(int), 256);
  w.m = off;      off = align_up(off + sizeof(int), 256);
  w.mask = off;   off = align_up(off + (size_t)cap * nbmax * sizeof(unsigned long long), 256);
  w.idx = off;    off = align_up(off + (size_t)cap * sizeof(int), 256);
  w.score = off;  off = align_up(off + (size_t)cap * sizeof(float), 256);
  w.count = off;  off = align_up(off + sizeof(int), 256);
  w.total = off;
  return w;
}

extern "C" size_t smb_ml_nms_workspace_bytes(int cap) {
  if (cap < 1 || cap > MAXN) return 0;
  return ml_ws_layout(cap).total;
}

extern "C" int smb_ml_nms_topk(const float* boxes, const float* scores, const int* labels, const int* n_dev, int cap,
                               float iou_thr, int max_per_img, int out_cap, float* det_out, int64_t* label_out,
                               int64_t* idx_out, int* count_out, int* kept_total_out, void* workspace,
                               size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(cap >= 1 && cap <= MAXN, "smb_ml_nms_topk: cap=%d outside [1,%d]", cap, MAXN);
  SMB_CHECK_ARG(out_cap >= 1 && out_cap <= MAXN, "smb_ml_nms_topk: out_cap=%d outside [1,%d]", out_cap, MAXN);
  SMB_CHECK_ARG(boxes && scores && labels && n_dev && det_out && label_out && idx_out && count_out && kept_total_out &&
                workspace, "smb_ml_nms_topk: null pointer");
  const MlWs w = ml_ws_layout(cap);
  if (workspace_bytes < w.total) {
    set_error("smb_ml_nms_topk: workspace %zu < %zu", workspace_bytes, w.total);
    return SMB_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  int P = 1;
  while (P < cap) P <<= 1;
  const size_t prep_smem = (size_t)P * sizeof(unsigned long long);
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(ml_prepare_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (int)(8192 * sizeof(unsigned long long))));
  }
  const int nbmax = (cap + 63) / 64;
  ml_prepare_kernel<<<1, NT, prep_smem, st>>>(boxes, scores, labels, n_dev, cap, (int*)(ws + w.cidx), (float*)(ws + w.cscore),
                                              (unsigned long long*)(ws + w.keys), (float4*)(ws + w.sbox), (int*)(ws + w.slab),
                                              (int*)(ws + w.m));
  SMB_LAUNCH_OK("ml_prepare_kernel");
  ml_mask_kernel<<<132 * 8, 64, 0, st>>>((const float4*)(ws + w.sbox), (const int*)(ws + w.slab), (const int*)(ws + w.m), nbmax,
                                         iou_thr, (unsigned long long*)(ws + w.mask));
  SMB_LAUNCH_OK("ml_mask_kernel");
  mc_sweep_kernel<<<1, NT, 0, st>>>((const unsigned long long*)(ws + w.mask), (const unsigned long long*)(ws + w.keys),
                                    (const int*)(ws + w.cidx), (const float*)(ws + w.cscore), (const int*)(ws + w.m), cap, nbmax,
                                    (int*)(ws + w.idx), (float*)(ws + w.score), (int*)(ws + w.count));
  SMB_LAUNCH_OK("mc_sweep_kernel");
  ml_finalize_kernel<<<1, NT, 0, st>>>(boxes, labels, (const int*)(ws + w.idx), (const float*)(ws + w.score),
                                       (const int*)(ws + w.count), cap, max_per_img, out_cap, det_out, (long long*)label_out,
                                       (long long*)idx_out, count_out, kept_total_out);
  SMB_LAUNCH_OK("ml_finalize_kernel");
  return SMB_OK;
}
