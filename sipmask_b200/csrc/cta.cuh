// Block-wide (CTA) building blocks of the post-processing and evaluation kernels: scans, a bitonic sort in shared
// memory, a radix select of the k-th smallest key, and the k smallest keys in order.
//
// Sync contract, the same for every helper here: every thread of the CTA calls it (it contains __syncthreads()), and
// when it returns, its shared scratch is free for the next call.  The scans read no shared memory of the caller.  The
// sort and the selects synchronise before they first read or write the caller's memory (its keys, and the sel buffer
// of cta_smallest_sorted) and after their last write, so a caller may write the keys right before the call and read the
// result right after it, also when it calls again while other threads still read the previous result.  A helper with a
// kThreads template argument runs in CTAs of exactly kThreads threads (blockDim.x, a multiple of 32 up to 1024): its
// strides and warp count are then compile-time constants, which the select loops need to keep the speed of the code
// they replace.
#pragma once
#include <cuda_runtime.h>

namespace smb {

struct Sum {
  template <typename T> __device__ __forceinline__ T operator()(T a, T b) const { return a + b; }
};
struct Max {
  template <typename T> __device__ __forceinline__ T operator()(T a, T b) const { return a > b ? a : b; }
};
struct Xor {
  template <typename T> __device__ __forceinline__ T operator()(T a, T b) const { return a ^ b; }
};
struct Less {
  template <typename T> __device__ __forceinline__ bool operator()(T a, T b) const { return a < b; }
};

// Inclusive scan of v over lanes 0 .. kLanes - 1 of a warp: op(lane 0's v, ..., this lane's v).  All 32 lanes call it;
// what lanes kLanes and up return is not a prefix.
template <int kLanes = 32, typename T, typename Op>
__device__ __forceinline__ T warp_inclusive_scan(T v, Op op) {
  static_assert(kLanes >= 1 && kLanes <= 32, "a warp has 32 lanes");
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 1; o < kLanes; o <<= 1) {
    const T u = __shfl_up_sync(0xffffffffu, v, o);
    if (lane >= o) v = op(u, v);
  }
  return v;
}

// The part both CTA scans share.  `inc` is the thread's inclusive scan inside its warp and x its result inside the warp.
// Returns op(the totals of the warps before this one, x), x in warp 0; *total = the CTA's total.
template <int kThreads, typename T, typename Op>
__device__ __forceinline__ T cta_scan_warps(T inc, T x, Op op, T* s_warp, T* total) {
  static_assert(kThreads % 32 == 0 && kThreads >= 32 && kThreads <= 1024, "a multiple of 32 threads, at most 1024");
  constexpr int kWarps = kThreads / 32;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 31) s_warp[wid] = inc;
  __syncthreads();
  if (wid == 0) {
    const T w = warp_inclusive_scan<kWarps>(lane < kWarps ? s_warp[lane] : s_warp[0], op);
    if (lane < kWarps) s_warp[lane] = w;
  }
  __syncthreads();
  if (wid > 0) x = op(s_warp[wid - 1], x);
  *total = s_warp[kWarps - 1];
  __syncthreads();
  return x;
}

// CTA-wide inclusive scan of one T per thread: returns op(thread 0's v, ..., this thread's v) and *total = op over every
// thread.  s_warp holds kThreads / 32 values of T.
template <int kThreads, typename T, typename Op>
__device__ __forceinline__ T cta_inclusive_scan(T v, Op op, T* s_warp, T* total) {
  v = warp_inclusive_scan(v, op);
  return cta_scan_warps<kThreads>(v, v, op, s_warp, total);
}

// CTA-wide exclusive scan: op over the v of the threads before this one, `identity` (the identity of op) in thread 0.
template <int kThreads, typename T, typename Op>
__device__ __forceinline__ T cta_exclusive_scan(T v, Op op, T identity, T* s_warp, T* total) {
  const T inc = warp_inclusive_scan(v, op);
  const T prev = __shfl_up_sync(0xffffffffu, inc, 1);                          // the lane before's inclusive scan
  return cta_scan_warps<kThreads>(inc, (threadIdx.x & 31) ? prev : identity, op, s_warp, total);
}

// Ascending in-place bitonic sort of a[0 .. P) in shared memory (P a power of two) by the strict weak order `less`.
template <typename T, typename Cmp>
__device__ __forceinline__ void cta_bitonic_sort(T* a, int P, Cmp less) {
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      __syncthreads();
      for (int t = threadIdx.x; t < (P >> 1); t += blockDim.x) {
        const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1)), l = i | j;
        const bool up = (i & k) == 0;
        const T x = a[i], y = a[l];
        if (less(up ? y : x, up ? x : y)) { a[i] = y; a[l] = x; }
      }
    }
  }
  __syncthreads();
}

// Shared scratch of cta_radix_select and cta_smallest_sorted.
struct SelectSmem {
  unsigned hist[256];
  unsigned long long prefix;
  int rank;
  int count;
};

template <typename K>
struct RadixKth {
  K key;      // the k-th smallest key in its top kBytes bytes, the lower bytes 0
  int rank;   // the k-th key's rank (1-based) among the keys that share those bytes
};

// The k-th smallest (1 <= k <= n) of the n keys key_at(0 .. n - 1), 32- or 64-bit, resolved one byte per pass from the
// top, for kBytes bytes.
template <int kThreads, typename K, int kBytes = (int)sizeof(K), typename KeyAt>
__device__ __forceinline__ RadixKth<K> cta_radix_select(int n, int k, KeyAt key_at, SelectSmem& s) {
  static_assert(kThreads % 32 == 0 && kThreads >= 32 && kThreads <= 1024, "a multiple of 32 threads, at most 1024");
  static_assert(sizeof(K) == 4 || sizeof(K) == 8, "32- or 64-bit keys");
  static_assert(kBytes >= 1 && kBytes <= (int)sizeof(K), "resolve 1 .. sizeof(K) bytes");
  constexpr int kBits = 8 * (int)sizeof(K);
  K prefix = 0;
  int need = k;                                    // rank of the k-th key among the keys that share `prefix`
#pragma unroll                                     // constant shifts and masks in every pass
  for (int shift = kBits - 8; shift >= kBits - 8 * kBytes; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += kThreads) s.hist[i] = 0u;
    __syncthreads();
    const K himask = (shift == kBits - 8) ? K(0) : (~K(0) << (shift + 8));
    for (int i = threadIdx.x; i < n; i += kThreads) {
      const K key = key_at(i);
      if ((key & himask) == prefix) atomicAdd(&s.hist[(unsigned)(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    // warp 0: the digit d with sum(hist[0 .. d - 1]) < need <= sum(hist[0 .. d]), and the rank inside that bin
    if (threadIdx.x < 32) {
      const int lane = threadIdx.x;
      int c[8];
      int sum = 0;
#pragma unroll
      for (int j = 0; j < 8; ++j) { c[j] = (int)s.hist[lane * 8 + j]; sum += c[j]; }
      const int incl = warp_inclusive_scan(sum, Sum()), excl = incl - sum;
      if (need > excl && need <= incl) {
        int r = need - excl, d = lane * 8;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          if (r > c[j]) { r -= c[j]; ++d; } else break;
        }
        s.rank = r;
        s.prefix = (unsigned long long)prefix | ((unsigned long long)d << shift);
      }
    }
    __syncthreads();
    prefix = (K)s.prefix;                          // rewritten two barriers into the next pass or call
    need = s.rank;
  }
  return RadixKth<K>{prefix, need};
}

// The k smallest of the n distinct 64-bit keys key_at(0 .. n - 1), ascending, into sel[0 .. k).  sel holds cap keys and
// is padded with ~0 up to the next power of two of k, which must not exceed cap.  When n < k, sel[0 .. n) holds all n
// keys and the rest is padding.
template <int kThreads, typename KeyAt>
__device__ __forceinline__ void cta_smallest_sorted(int n, int k, KeyAt key_at, unsigned long long* sel, int cap,
                                                    SelectSmem& s) {
  // With n <= k no select runs, and the fill of sel below would otherwise be the first thing a thread does: wait for
  // every thread, so no thread overwrites sel (or s.count) while another still reads what a previous call left there.
  __syncthreads();
  const unsigned long long kth = (n > k) ? cta_radix_select<kThreads, unsigned long long>(n, k, key_at, s).key : ~0ull;
  if (threadIdx.x == 0) s.count = 0;
  for (int i = threadIdx.x; i < cap; i += kThreads) sel[i] = ~0ull;
  __syncthreads();
  for (int i = threadIdx.x; i < n; i += kThreads) {
    const unsigned long long key = key_at(i);
    if (key <= kth) {
      const int p = atomicAdd(&s.count, 1);
      if (p < cap) sel[p] = key;
    }
  }
  int P = 1;
  while (P < k) P <<= 1;
  cta_bitonic_sort(sel, P, Less());
}

}  // namespace smb
