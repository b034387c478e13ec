// Test harness of the block-wide primitives in sipmask_b200/csrc/cta.cuh, built into libsmb_cta_harness.so next to
// the product library (never into it).  Each kernel runs one primitive per CTA on that CTA's own segment, at every
// block size of kBlockSizes; tests/test_gpu_cta.py compares the results with numpy, bit for bit.
//
// Every entry point launches on the given stream and returns the launch's cudaError_t (cudaErrorInvalidValue for a
// block size, key width or mode outside the tables below).  Callers keep to each primitive's preconditions.
#include <cstdint>
#include <type_traits>

#include <cuda_runtime.h>

#include "cta.cuh"

namespace {

using u64 = unsigned long long;

constexpr int kBlockSizes[] = {32, 64, 96, 160, 256, 512, 992, 1024};
constexpr int kSelectCap = 1024;            // sel capacity of the cta_smallest_sorted kernels
constexpr int kContractKeys = 2048;         // keys a contract call stages in shared memory
constexpr int kContractSortP = 1024;

template <typename F>
cudaError_t with_threads(int threads, F&& f) {
  switch (threads) {
    case 32: return f(std::integral_constant<int, 32>{});
    case 64: return f(std::integral_constant<int, 64>{});
    case 96: return f(std::integral_constant<int, 96>{});
    case 160: return f(std::integral_constant<int, 160>{});
    case 256: return f(std::integral_constant<int, 256>{});
    case 512: return f(std::integral_constant<int, 512>{});
    case 992: return f(std::integral_constant<int, 992>{});
    case 1024: return f(std::integral_constant<int, 1024>{});
    default: return cudaErrorInvalidValue;
  }
}

// ---- scans: segment b is in[b * kThreads .. (b + 1) * kThreads); every thread writes its own totals ----
template <int kThreads, typename T, typename Op>
__global__ void __launch_bounds__(kThreads) scan_kernel(const T* in, T identity, T* inc, T* exc, T* tot_inc,
                                                        T* tot_exc) {
  __shared__ T s_warp[kThreads / 32];
  const size_t i = (size_t)blockIdx.x * kThreads + threadIdx.x;
  const T v = in[i];
  T ti, te;
  inc[i] = smb::cta_inclusive_scan<kThreads>(v, Op(), s_warp, &ti);   // the same s_warp for both: reusable on return
  exc[i] = smb::cta_exclusive_scan<kThreads>(v, Op(), identity, s_warp, &te);
  tot_inc[i] = ti;
  tot_exc[i] = te;
}

template <typename T, typename Op>
cudaError_t launch_scan(int threads, int blocks, const void* in, T identity, void* inc, void* exc, void* tot_inc,
                        void* tot_exc, cudaStream_t st) {
  return with_threads(threads, [&](auto t) {
    constexpr int kThreads = decltype(t)::value;
    scan_kernel<kThreads, T, Op><<<blocks, kThreads, 0, st>>>((const T*)in, identity, (T*)inc, (T*)exc, (T*)tot_inc,
                                                              (T*)tot_exc);
    return cudaGetLastError();
  });
}

// ---- warp_inclusive_scan<kLanes>: every warp scans its own 32 values ----
template <int kLanes>
__global__ void warp_scan_kernel(const int* in, int* out) {
  const int i = blockIdx.x * 32 + threadIdx.x;
  out[i] = smb::warp_inclusive_scan<kLanes>(in[i], smb::Sum());
}

// ---- bitonic sort: segment b is P keys; blockDim.x is free ----
__global__ void sort_u64_kernel(const u64* in, u64* out, int P) {
  extern __shared__ __align__(16) unsigned char smem[];
  u64* a = (u64*)smem;
  const size_t base = (size_t)blockIdx.x * P;
  for (int i = threadIdx.x; i < P; i += blockDim.x) a[i] = in[base + i];
  smb::cta_bitonic_sort(a, P, smb::Less());
  for (int i = threadIdx.x; i < P; i += blockDim.x) out[base + i] = a[i];
}

// Rows 0 .. n_valid[b] - 1 of segment b by descending key, ties by row; the padding rows (-1) last.  The comparator
// reads the keys from a table outside the sorted array, as match2_kernel's does.
__global__ void sort_index_kernel(const float* key, const int* n_valid, int* out, int P) {
  extern __shared__ __align__(16) unsigned char smem[];
  int* a = (int*)smem;
  const size_t base = (size_t)blockIdx.x * P;
  const float* kb = key + base;
  const int nv = n_valid[blockIdx.x];
  for (int i = threadIdx.x; i < P; i += blockDim.x) a[i] = i < nv ? i : -1;
  auto before = [&](int x, int y) -> bool {
    if (y < 0) return x >= 0;
    if (x < 0) return false;
    if (kb[x] != kb[y]) return kb[x] > kb[y];
    return x < y;
  };
  smb::cta_bitonic_sort(a, P, before);
  for (int i = threadIdx.x; i < P; i += blockDim.x) out[base + i] = a[i];
}

// ---- radix select: the CTAs share out the queries; each runs its queries back to back on one SelectSmem, with a
// cta_exclusive_scan between them as pair_select_kernel has.  Every thread writes what it got. ----
template <int kThreads, typename K, int kBytes>
__global__ void __launch_bounds__(kThreads) select_kernel(const K* keys, const long long* off, const int* nk, int nq,
                                                          K* out_key, int* out_rank, int* out_scan) {
  __shared__ smb::SelectSmem s;
  __shared__ int s_warp[kThreads / 32];
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const K* kq = keys + off[q];
    const smb::RadixKth<K> r =
        smb::cta_radix_select<kThreads, K, kBytes>(nk[2 * q], nk[2 * q + 1], [&](int i) { return kq[i]; }, s);
    const size_t o = (size_t)q * kThreads + threadIdx.x;
    out_key[o] = r.key;
    out_rank[o] = r.rank;
    int tot;
    out_scan[o] = smb::cta_exclusive_scan<kThreads>(r.rank, smb::Sum(), 0, s_warp, &tot);
  }
}

template <int kThreads, typename K, int kBytes = (int)sizeof(K)>
cudaError_t launch_select(int bytes, int blocks, const void* keys, const long long* off, const int* nk, int nq,
                          void* out_key, int* out_rank, int* out_scan, cudaStream_t st) {
  if (bytes == kBytes) {
    select_kernel<kThreads, K, kBytes><<<blocks, kThreads, 0, st>>>((const K*)keys, off, nk, nq, (K*)out_key, out_rank,
                                                                     out_scan);
    return cudaGetLastError();
  }
  if constexpr (kBytes > 1) {
    return launch_select<kThreads, K, kBytes - 1>(bytes, blocks, keys, off, nk, nq, out_key, out_rank, out_scan, st);
  } else {
    return cudaErrorInvalidValue;
  }
}

// ---- cta_smallest_sorted with cap = kSelectCap: the whole sel buffer of every query ----
template <int kThreads>
__global__ void __launch_bounds__(kThreads) smallest_kernel(const u64* keys, const long long* off, const int* nk,
                                                            int nq, u64* out) {
  __shared__ u64 s_sel[kSelectCap];
  __shared__ smb::SelectSmem s;
  for (int q = blockIdx.x; q < nq; q += gridDim.x) {
    const u64* kq = keys + off[q];
    smb::cta_smallest_sorted<kThreads>(nk[2 * q], nk[2 * q + 1], [&](int i) { return kq[i]; }, s_sel, kSelectCap, s);
    for (int i = threadIdx.x; i < kSelectCap; i += kThreads) out[(size_t)q * kSelectCap + i] = s_sel[i];
  }
}

// ---- the sync contract: keys go into shared memory right before each call and the result is read right after it,
// with no barrier of the caller's.  Warp 0 alone reads the whole first result (the select: its own copy), ~10 us late,
// while the other warps go on to the second call: a helper that touches the caller's memory before its first barrier
// corrupts that read on every run. ----
__device__ __forceinline__ void lag_warp0() {
  if (threadIdx.x < 32) {
    const long long t0 = clock64();
    while (clock64() - t0 < 20000) __nanosleep(256);
  }
}

template <typename T>
__device__ __forceinline__ void warp0_reads_late(const T* src, T* dst, int n) {
  lag_warp0();
  if (threadIdx.x < 32)
    for (int i = threadIdx.x; i < n; i += 32) dst[i] = src[i];
}

enum { kContractSort = 0, kContractSelect = 1, kContractSmallest = 2 };

// nk = {n1, k1, n2, k2}.  Sort: in1 / in2 are kContractSortP keys each, sorted in two buffers.  Select: out[t] is
// thread t's key and rank[t] its rank.  Smallest: out is the whole sel buffer.
template <int kThreads>
__global__ void __launch_bounds__(kThreads) contract_kernel(int mode, const u64* in1, const u64* in2, const int* nk,
                                                            u64* out1, u64* out2, int* rank1, int* rank2) {
  __shared__ u64 s_keys[kContractKeys];
  __shared__ u64 s_sel[kSelectCap];
  __shared__ smb::SelectSmem s;
  const int t = threadIdx.x;
  const int n1 = nk[0], k1 = nk[1], n2 = nk[2], k2 = nk[3];
  auto key_at = [&](int i) { return s_keys[i]; };
  if (mode == kContractSort) {
    u64* a1 = s_keys;
    u64* a2 = s_keys + kContractSortP;
    for (int i = t; i < kContractSortP; i += kThreads) a1[i] = in1[i];
    smb::cta_bitonic_sort(a1, kContractSortP, smb::Less());
    warp0_reads_late(a1, out1, kContractSortP);
    for (int i = t; i < kContractSortP; i += kThreads) a2[i] = in2[i];
    smb::cta_bitonic_sort(a2, kContractSortP, smb::Less());
    for (int i = t; i < kContractSortP; i += kThreads) out2[i] = a2[i];
  } else if (mode == kContractSelect) {
    for (int i = t; i < n1; i += kThreads) s_keys[i] = in1[i];
    const smb::RadixKth<u64> r1 = smb::cta_radix_select<kThreads, u64>(n1, k1, key_at, s);
    lag_warp0();
    out1[t] = r1.key;
    rank1[t] = r1.rank;
    for (int i = t; i < n2; i += kThreads) s_keys[i] = in2[i];
    const smb::RadixKth<u64> r2 = smb::cta_radix_select<kThreads, u64>(n2, k2, key_at, s);
    out2[t] = r2.key;
    rank2[t] = r2.rank;
  } else {
    for (int i = t; i < n1; i += kThreads) s_keys[i] = in1[i];
    smb::cta_smallest_sorted<kThreads>(n1, k1, key_at, s_sel, kSelectCap, s);
    warp0_reads_late(s_sel, out1, kSelectCap);
    for (int i = t; i < n2; i += kThreads) s_keys[i] = in2[i];
    smb::cta_smallest_sorted<kThreads>(n2, k2, key_at, s_sel, kSelectCap, s);
    for (int i = t; i < kSelectCap; i += kThreads) out2[i] = s_sel[i];
  }
}

}  // namespace

extern "C" {

// The block sizes every kernel is instantiated for; returns how many (at most cap are written).
int cta_h_block_sizes(int* out, int cap) {
  const int n = (int)(sizeof(kBlockSizes) / sizeof(kBlockSizes[0]));
  for (int i = 0; i < n && i < cap; ++i) out[i] = kBlockSizes[i];
  return n;
}

// op 0: int32 Sum, 1: uint64 Sum (mod 2^64), 2: double Max (identity -inf), 3: uint32 Xor.  All arrays hold
// blocks * threads elements.
int cta_h_scan(int op, int threads, int blocks, const void* in, void* inc, void* exc, void* tot_inc, void* tot_exc,
               cudaStream_t st) {
  switch (op) {
    case 0: return launch_scan<int32_t, smb::Sum>(threads, blocks, in, 0, inc, exc, tot_inc, tot_exc, st);
    case 1: return launch_scan<u64, smb::Sum>(threads, blocks, in, 0ull, inc, exc, tot_inc, tot_exc, st);
    case 2:
      return launch_scan<double, smb::Max>(threads, blocks, in, -__builtin_huge_val(), inc, exc, tot_inc, tot_exc, st);
    case 3: return launch_scan<uint32_t, smb::Xor>(threads, blocks, in, 0u, inc, exc, tot_inc, tot_exc, st);
    default: return cudaErrorInvalidValue;
  }
}

// int32 Sum over `warps` warps of 32 values; lanes >= kLanes of the output are unspecified.
int cta_h_warp_scan(int lanes, int warps, const int* in, int* out, cudaStream_t st) {
  switch (lanes) {
#define CTA_H_LANES(L) \
  case L: warp_scan_kernel<L><<<warps, 32, 0, st>>>(in, out); break;
    CTA_H_LANES(1) CTA_H_LANES(2) CTA_H_LANES(3) CTA_H_LANES(7) CTA_H_LANES(8) CTA_H_LANES(31) CTA_H_LANES(32)
#undef CTA_H_LANES
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// Ascending sort of blocks segments of P (a power of two, at most 8192) uint64 keys.
int cta_h_sort_u64(int P, int threads, int blocks, const u64* in, u64* out, cudaStream_t st) {
  const size_t smem = (size_t)P * sizeof(u64);
  cudaError_t e = cudaFuncSetAttribute(sort_u64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  sort_u64_kernel<<<blocks, threads, smem, st>>>(in, out, P);
  return cudaGetLastError();
}

// Index sort of blocks segments of P rows (see sort_index_kernel); out holds blocks * P row indices.
int cta_h_sort_index(int P, int threads, int blocks, const float* key, const int* n_valid, int* out, cudaStream_t st) {
  const size_t smem = (size_t)P * sizeof(int);
  cudaError_t e = cudaFuncSetAttribute(sort_index_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) return e;
  sort_index_kernel<<<blocks, threads, smem, st>>>(key, n_valid, out, P);
  return cudaGetLastError();
}

// Query q selects the nk[2q + 1]-th smallest of the nk[2q] keys at keys + off[q] (key_bits 32 or 64, resolving `bytes`
// bytes).  out_key / out_rank / out_scan hold nq * threads values: every thread's key, rank and the exclusive scan of
// the ranks.
int cta_h_radix_select(int key_bits, int bytes, int threads, int blocks, const void* keys, const long long* off,
                       const int* nk, int nq, void* out_key, int* out_rank, int* out_scan, cudaStream_t st) {
  return with_threads(threads, [&](auto t) {
    constexpr int kThreads = decltype(t)::value;
    if (key_bits == 32)
      return launch_select<kThreads, unsigned>(bytes, blocks, keys, off, nk, nq, out_key, out_rank, out_scan, st);
    if (key_bits == 64)
      return launch_select<kThreads, u64>(bytes, blocks, keys, off, nk, nq, out_key, out_rank, out_scan, st);
    return cudaErrorInvalidValue;
  });
}

// Query q: cta_smallest_sorted of the nk[2q] keys at keys + off[q] with k = nk[2q + 1]; out holds nq * 1024 keys.
int cta_h_smallest_sorted(int threads, int blocks, const u64* keys, const long long* off, const int* nk, int nq,
                          u64* out, cudaStream_t st) {
  return with_threads(threads, [&](auto t) {
    constexpr int kThreads = decltype(t)::value;
    smallest_kernel<kThreads><<<blocks, kThreads, 0, st>>>(keys, off, nk, nq, out);
    return cudaGetLastError();
  });
}

// One CTA of two back-to-back calls (mode 0: sort, 1: radix select, 2: cta_smallest_sorted); see contract_kernel.
int cta_h_contract(int mode, int threads, const u64* in1, const u64* in2, const int* nk, u64* out1, u64* out2,
                   int* rank1, int* rank2, cudaStream_t st) {
  if (mode < kContractSort || mode > kContractSmallest) return cudaErrorInvalidValue;
  return with_threads(threads, [&](auto t) {
    constexpr int kThreads = decltype(t)::value;
    contract_kernel<kThreads><<<1, kThreads, 0, st>>>(mode, in1, in2, nk, out1, out2, rank1, rank2);
    return cudaGetLastError();
  });
}

}  // extern "C"
