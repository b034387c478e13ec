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

namespace smb {

constexpr int NT = 1024;          // threads per CTA for all kernels in this file
constexpr int MAXN = 5120;        // max candidates per class list held in shared memory (>= 5 levels x nms_pre = 1000)
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

// In-place ascending bitonic sort of P (power of two) keys in shared memory by the whole CTA.
__device__ void bitonic_sort(unsigned long long* keys, int P) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
        const int ixj = i | j;
        const bool up = (i & k) == 0;
        const unsigned long long a = keys[i], b = keys[ixj];
        if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
      }
    }
  }
  __syncthreads();
}

// CTA-wide exclusive scan of one int per thread (blockDim.x == NT); returns exclusive prefix, total in *total.
__device__ int block_exscan(int v, int* s_warp /* [33] */, int* total) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int inc = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const int t = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += t;
  }
  __syncthreads();
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    int w = (lane < (blockDim.x >> 5)) ? s_warp[lane] : 0;
    int winc = w;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, winc, o);
      if (lane >= o) winc += t;
    }
    s_warp[lane] = winc - w;
    if (lane == 31) s_warp[32] = winc;
  }
  __syncthreads();
  *total = s_warp[32];
  return s_warp[wid] + inc - v;
}


// Radix-select helper: given a 256-bin histogram in shared memory and the rank `need` (1-based) still wanted,
// warp 0 finds the digit d with sum(hist[0..d-1]) < need <= sum(hist[0..d]) and the rank inside that bin.
// All threads must call it (contains __syncthreads).
__device__ __forceinline__ void select_digit(const unsigned* s_hist, int* s_k, unsigned long long* s_prefix,
                                             unsigned long long prefix, int shift) {
  __syncthreads();
  if (threadIdx.x < 32) {
    const int lane = threadIdx.x;
    int c[8];
    int sum = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) { c[j] = (int)s_hist[lane * 8 + j]; sum += c[j]; }
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const int excl = incl - sum;
    const int need = *s_k;
    if (need > excl && need <= incl) {
      int r = need - excl, d = lane * 8;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        if (r > c[j]) { r -= c[j]; ++d; } else break;
      }
      *s_k = r;
      *s_prefix = prefix | ((unsigned long long)d << shift);
    }
  }
  __syncthreads();
}

// Greedy NMS sweep over `m` boxes already sorted by descending score in shared memory.
// On return bit r of rem[] is set iff sorted row r is suppressed.  `plus_one`/`cmp_ge` select the
// reference comparator (nms_kernel.cu:61 `>` vs nms_cpu.cpp:56 `>=`).
__device__ void greedy_sweep_n(const float4* sb, int m, float thr, int cmp_ge, float one,
                               unsigned long long* rem, int rem_words, unsigned long long* diag,
                               unsigned long long* s_keep);
__device__ __forceinline__ void greedy_sweep(const float4* sb, int m, float thr, int cmp_ge, float one,
                                             unsigned long long* rem /* [MAXN/64] */, unsigned long long* diag /* [64] */,
                                             unsigned long long* s_keep) {
  greedy_sweep_n(sb, m, thr, cmp_ge, one, rem, MAXN / 64, diag, s_keep);
}

// ---------------------------------------------------------------------------------------------
// Single-class NMS operator: dets [n,5]; keep ascending original indices.
// ---------------------------------------------------------------------------------------------
struct NmsSmem {
  unsigned long long keys[NMS1];
  float4 sb[NMS1];
  unsigned long long rem[NMS1 / 64];
  unsigned long long diag[64];
  unsigned long long keepbits;
  int warp[33];
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
  bitonic_sort(S.keys, P);
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
    const int ex = block_exscan(f, S.warp, &tot);
    if (f) keep_out[running + ex] = i;
    running += tot;
    __syncthreads();
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
  unsigned long long keys[MAXN];
  int cidx[MAXN];
  float cscore[MAXN];
  int warp[33];
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
    const int ex = block_exscan(f, S.warp, &tot);
    if (f) { S.cidx[m + ex] = i; S.cscore[m + ex] = __fmul_rn(s, ctr[i]); }  // bbox_nms.py:122
    m += tot;
    __syncthreads();
  }
  if (threadIdx.x == 0) w_m[c] = m;
  if (m == 0) return;
  int P = 1;
  while (P < m) P <<= 1;
  for (int i = threadIdx.x; i < P; i += NT) S.keys[i] = (i < m) ? desc_key(S.cscore[i], (unsigned)i) : ~0ull;
  bitonic_sort(S.keys, P);
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
  int warp[33];
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
    const int ex = block_exscan(f, S.warp, &tot);
    if (f) {
      ws_idx[(size_t)c * n + running + ex] = w_cidx[(size_t)c * n + p];
      ws_score[(size_t)c * n + running + ex] = w_cscore[(size_t)c * n + p];
    }
    running += tot;
    __syncthreads();
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
  __shared__ int s_warp[33];
  __shared__ unsigned s_hist[256];
  __shared__ unsigned long long s_sel[1024];
  __shared__ int s_nsel;
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k;
  // class offsets
  {
    const int v = (threadIdx.x < C) ? ws_count[threadIdx.x] : 0;
    int tot;
    const int ex = block_exscan(v, s_warp, &tot);
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
  __syncthreads();
  // radix-select the kout-th smallest key (keys are unique)
  if (threadIdx.x == 0) { s_prefix = 0ull; s_k = kout; }
  __syncthreads();
  if (K > kout) {
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int i = threadIdx.x; i < 256; i += NT) s_hist[i] = 0u;
      __syncthreads();
      const unsigned long long prefix = s_prefix;
      const unsigned long long himask = (shift == 56) ? 0ull : (~0ull << (shift + 8));
      for (int g = threadIdx.x; g < K; g += NT) {
        const unsigned long long k = gkey[g];
        if ((k & himask) == prefix) atomicAdd(&s_hist[(unsigned)(k >> shift) & 255u], 1u);
      }
      select_digit(s_hist, &s_k, &s_prefix, prefix, shift);
    }
  } else {
    if (threadIdx.x == 0) s_prefix = ~0ull;
    __syncthreads();
  }
  const unsigned long long kth = s_prefix;
  if (threadIdx.x == 0) s_nsel = 0;
  for (int i = threadIdx.x; i < 1024; i += NT) s_sel[i] = ~0ull;
  __syncthreads();
  for (int g = threadIdx.x; g < K; g += NT) {
    const unsigned long long k = gkey[g];
    if (k <= kth) { const int p = atomicAdd(&s_nsel, 1); if (p < 1024) s_sel[p] = k; }
  }
  __syncthreads();
  int P = 1;
  while (P < kout) P <<= 1;
  bitonic_sort(s_sel, P);
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
  unsigned long long keys[MAXN];
  float4 sb[256];
  float sscore[256];
  unsigned char kept[256];
  int warp[33];
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
  bitonic_sort(S.keys, P);
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
    const int ex = block_exscan(f, S.warp, &tot);
    if (f) {
      ws_idx[(size_t)c * top_k + running + ex] = (int)(S.keys[p] & 0xffffffffu);
      ws_score[(size_t)c * top_k + running + ex] = S.sscore[p];
    }
    running += tot;
    __syncthreads();
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
  __shared__ unsigned s_hist[256];
  __shared__ unsigned long long s_sel[1024];
  __shared__ int s_nsel;
  __shared__ unsigned long long s_prefix;
  __shared__ int s_k;
  const int l = blockIdx.x;
  const int hw = L.loc_off[l + 1] - L.loc_off[l];
  const float* sl = s + L.loc_off[l];
  int* out = sel + L.cand_off[l];
  if (nms_pre <= 0 || hw <= nms_pre) {
    for (int i = threadIdx.x; i < hw; i += NT) out[i] = i;
    return;
  }
  if (threadIdx.x == 0) { s_prefix = 0ull; s_k = nms_pre; }
  __syncthreads();
  for (int shift = 56; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += NT) s_hist[i] = 0u;
    __syncthreads();
    const unsigned long long prefix = s_prefix;
    const unsigned long long himask = (shift == 56) ? 0ull : (~0ull << (shift + 8));
    for (int i = threadIdx.x; i < hw; i += NT) {
      const unsigned long long k = desc_key(sl[i], (unsigned)i);
      if ((k & himask) == prefix) atomicAdd(&s_hist[(unsigned)(k >> shift) & 255u], 1u);
    }
    select_digit(s_hist, &s_k, &s_prefix, prefix, shift);
  }
  const unsigned long long kth = s_prefix;
  if (threadIdx.x == 0) s_nsel = 0;
  for (int i = threadIdx.x; i < 1024; i += NT) s_sel[i] = ~0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < hw; i += NT) {
    const unsigned long long k = desc_key(sl[i], (unsigned)i);
    if (k <= kth) { const int p = atomicAdd(&s_nsel, 1); if (p < 1024) s_sel[p] = k; }
  }
  __syncthreads();
  int P = 1;
  while (P < nms_pre) P <<= 1;
  bitonic_sort(s_sel, P);
  for (int r = threadIdx.x; r < nms_pre; r += NT) out[r] = (int)(s_sel[r] & 0xffffffffu);
}

// one warp per candidate: box decode + sigmoid scores
__global__ void gather_decode_kernel(Levels L, int C, int img_h, int img_w, float is0, float is1, float is2, float is3,
                                     int has_scale, const int* __restrict__ sel, float* __restrict__ cand_boxes,
                                     float* __restrict__ cand_scores, float* __restrict__ cand_ctr,
                                     int* __restrict__ cand_loc) {
  pdl_wait();
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
      const float mw = (float)(img_w - 1), mh = (float)(img_h - 1);
      x1 = fminf(fmaxf(x1, 0.f), mw); y1 = fminf(fmaxf(y1, 0.f), mh);
      x2 = fminf(fmaxf(x2, 0.f), mw); y2 = fminf(fmaxf(y2, 0.f), mh);
      if (has_scale) {  // mlvl_bboxes /= scale_factor (sipmask_head.py:587-588): true division
        x1 = __fdiv_rn(x1, is0); y1 = __fdiv_rn(y1, is1); x2 = __fdiv_rn(x2, is2); y2 = __fdiv_rn(y2, is3);
      }
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
                                          const int* __restrict__ count, int max_rows, float sx, float sy, float stride,
                                          float* __restrict__ out) {
  pdl_wait();
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

extern "C" int smb_decode_topk(int num_levels, const smb_level_t* host_levels, int num_classes, int nms_pre, int img_h,
                               int img_w, const float* host_scale4, float* cand_boxes, float* cand_scores,
                               float* cand_ctr, int* cand_loc, void* workspace, size_t workspace_bytes,
                               smb_stream_t stream) {
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
  const float i0 = host_scale4 ? host_scale4[0] : 1.f, i1 = host_scale4 ? host_scale4[1] : 1.f;
  const float i2 = host_scale4 ? host_scale4[2] : 1.f, i3 = host_scale4 ? host_scale4[3] : 1.f;
  gather_decode_kernel<<<min(cdiv(ncand, 8), 132 * 8), 256, 0, st>>>(L, num_classes, img_h, img_w, i0, i1, i2, i3,
                                                                    host_scale4 ? 1 : 0, sel, cand_boxes, cand_scores,
                                                                    cand_ctr, cand_loc);
  SMB_LAUNCH_OK("gather_decode_kernel");
  return SMB_OK;
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

extern "C" int smb_gather_track_feats(const float* track, int h, int w, int C, const float* det, const int* count_dev,
                                      int max_rows, float scale_x, float scale_y, float feat_stride, float* out,
                                      smb_stream_t stream) {
  SMB_CHECK_ARG(track && det && count_dev && out && h > 0 && w > 0 && C > 0 && max_rows > 0 && feat_stride > 0.f,
                "smb_gather_track_feats: bad argument");
  gather_track_feats_kernel<<<cdiv(max_rows * C, 256), 256, 0, (cudaStream_t)stream>>>(track, h, w, C, det, count_dev, max_rows,
                                                                                         scale_x, scale_y, feat_stride, out);
  SMB_LAUNCH_OK("gather_track_feats_kernel");
  return SMB_OK;
}

extern "C" int smb_gather_rows_f32(const float* src, int src_pitch, const int64_t* idx, const int* count_dev, int max_rows,
                                   int row_elems, float* dst, smb_stream_t stream) {
  SMB_CHECK_ARG(src && idx && count_dev && dst && max_rows > 0 && row_elems > 0, "smb_gather_rows_f32: bad argument");
  gather_rows_kernel<<<cdiv(max_rows * row_elems, 256), 256, 0, (cudaStream_t)stream>>>(src, src_pitch, (const long long*)idx,
                                                                                         count_dev, max_rows, row_elems, dst);
  SMB_LAUNCH_OK("gather_rows_kernel");
  return SMB_OK;
}
