// COCO run-length encoding of the bit-packed instance masks on the device (SURVEY.md §8f-1).
//
// Replaces, per detection, `masks[i].cpu().numpy()` (a synchronous 4.3 MB copy) + `mask_util.encode(np.array(im_mask[:, :,
// np.newaxis], order='F'))` (single-threaded pycocotools on the host) - SipMask-mmdetection/mmdet/models/anchor_heads/
// sipmask_head.py:645-657.  The format is pycocotools' (not vendored in the reference): run lengths over the mask in
// COLUMN-major order, starting with the number of zeros; the compressed ASCII string has 5 data bits + a continuation
// bit per character, and counts[i] for i > 2 is stored as a delta against counts[i-2].
//
// One CTA per detection.  The masks are row-major bit planes (bit x&31 of word x>>5), the runs are column-major: every warp
// transposes 32x32-bit tiles with 32 ballots, so that lane c holds 32 vertically adjacent pixels of column 32*wq + c; a run
// boundary is a bit that differs from the pixel before it in column-major order (the bottom of the previous column for
// row 0; 0 for the very first pixel).  The columns are processed in blocks of RLE_COLS: pass 1 counts boundaries per
// column, a block scan orders them, pass 2 writes the boundary positions.  Then either
//   - rle_counts_kernel differences the positions into run lengths (smb_mask_rle_counts), or
//   - rle_encode_kernel turns them into the pycocotools string (per run: length, delta, character count, block scan of
//     the counts, characters), and rle_pack_kernel lays out each image's strings back to back behind a header in a
//     (pinned host) arena whose address it reads from a device word (smb_rle_encode_dev).
#include <stdint.h>
#include <string.h>

#include "common.cuh"
#include "cta.cuh"

namespace smb {

constexpr int RLE_THREADS = 1024;
constexpr int RLE_COLS = 2 * RLE_THREADS;          // columns per scan block (two per thread)
constexpr int RLE_MAX_CHARS = 7;                   // characters of one count: |delta| < 2^31 -> 7 x 5 bits
constexpr int RLE_MAX_DETS = RLE_THREADS;          // detections per image of the pack kernel (one per thread)

// 32 rows x 32 columns bit transpose: lane l supplies the word of row l, lane c receives the 32 row bits of column c
__device__ __forceinline__ uint32_t transpose32(uint32_t w, int lane) {
  uint32_t mine = 0u;
#pragma unroll
  for (int b = 0; b < 32; ++b) {
    const uint32_t t = __ballot_sync(0xffffffffu, (w >> b) & 1u);
    if (lane == b) mine = t;
  }
  return mine;
}

__device__ __forceinline__ uint32_t pixel_bit(const uint32_t* m, int words, int x, int y) {
  return (m[(size_t)y * words + (x >> 5)] >> (x & 31)) & 1u;
}

// The column-major run boundaries of column x = 32*wq + lane (the whole warp calls it): f(yc, t) receives, chunk by
// chunk, the boundary bits t of rows 32*yc .. 32*yc+31 (bit r = row 32*yc + r); t = 0 for columns at or past W.
template <typename F>
__device__ __forceinline__ void column_boundaries(const uint32_t* m, int words, int H, int W, int wq, int lane, F&& f) {
  const int x = wq * 32 + lane;
  uint32_t prev = (x > 0 && x < W) ? pixel_bit(m, words, x - 1, H - 1) : 0u;   // the pixel before (x, 0)
  const int ychunks = (H + 31) >> 5;
  for (int yc = 0; yc < ychunks; ++yc) {
    const int y = yc * 32 + lane;
    const uint32_t w = (y < H) ? m[(size_t)y * words + wq] : 0u;
    const uint32_t col = transpose32(w, lane);
    const int rows = min(32, H - yc * 32);
    const uint32_t valid = rows == 32 ? 0xffffffffu : ((1u << rows) - 1u);
    const uint32_t t = (col ^ ((col << 1) | prev)) & valid;
    prev = (col >> (rows - 1)) & 1u;
    f(yc, x < W ? t : 0u);
  }
}

// Boundary positions (column-major pixel index) of the H x W mask m, in order, into out[0, cap) (positions past cap are
// counted, not stored).  Returns the number of boundaries; the runs are that number + 1.  Every thread of the block calls
// it; s_cnt holds RLE_COLS ints.  Any width: the scan loops over blocks of RLE_COLS columns with a running carry.
__device__ int boundary_positions(const uint32_t* m, int words, int H, int W, uint32_t* out, int cap, int* s_cnt,
                                  int* s_warp) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int wcols = (W + 31) >> 5;
  int carry = 0;
  for (int wq0 = 0; wq0 < wcols; wq0 += RLE_COLS / 32) {
    const int nwq = min(RLE_COLS / 32, wcols - wq0);
    // ---- pass 1: run boundaries per column of this block
    for (int q = warp; q < nwq; q += RLE_THREADS / 32) {
      int c = 0;
      column_boundaries(m, words, H, W, wq0 + q, lane, [&](int, uint32_t t) { c += __popc(t); });
      s_cnt[q * 32 + lane] = c;
    }
    __syncthreads();
    // ---- exclusive scan over the block's columns, two per thread, after the boundaries of the blocks before it
    const int ncol = nwq * 32;
    const int i0 = 2 * threadIdx.x, i1 = i0 + 1;
    const int a0 = i0 < ncol ? s_cnt[i0] : 0, a1 = i1 < ncol ? s_cnt[i1] : 0;
    int total;
    const int base = carry + cta_exclusive_scan<RLE_THREADS>(a0 + a1, Sum(), 0, s_warp, &total);
    if (i0 < ncol) s_cnt[i0] = base;
    if (i1 < ncol) s_cnt[i1] = base + a0;
    __syncthreads();
    // ---- pass 2: boundary positions, in order
    for (int q = warp; q < nwq; q += RLE_THREADS / 32) {
      const int x = (wq0 + q) * 32 + lane;
      int o = s_cnt[q * 32 + lane];
      column_boundaries(m, words, H, W, wq0 + q, lane, [&](int yc, uint32_t t) {
        while (t) {
          const int r = __ffs(t) - 1;
          t &= t - 1;
          if (o < cap) out[o] = (uint32_t)(x * H + yc * 32 + r);
          ++o;
        }
      });
    }
    carry += total;
    __syncthreads();                               // s_cnt is rewritten by the next column block
  }
  return carry;
}

__global__ void __launch_bounds__(RLE_THREADS) rle_counts_kernel(const uint32_t* __restrict__ bits, int mask_h, int words, int H,
                                                                 int W, const int* __restrict__ n_valid, uint32_t* __restrict__ counts,
                                                                 int cap, int* __restrict__ n_counts) {
  __shared__ int s_cnt[RLE_COLS];
  __shared__ int s_warp[32];
  const int det = blockIdx.x;
  if (n_valid && det >= *n_valid) {
    if (threadIdx.x == 0) n_counts[det] = 0;
    return;
  }
  const uint32_t* m = bits + (size_t)det * mask_h * words;
  uint32_t* out = counts + (size_t)det * cap;
  const int total = boundary_positions(m, words, H, W, out, cap, s_cnt, s_warp);
  // ---- pass 3: positions -> run lengths, in place
  // counts[0] = pos[0] (zeros before the first one; 0 if the mask starts with a one), counts[k] = pos[k] - pos[k-1],
  // counts[T] = H*W - pos[T-1];  T == 0 -> the single run [H*W].
  const int T = min(total, cap - 1);
  const int P = H * W;
  // stripes run back to front: a stripe reads out[k0-1 .. k0+1023] and writes out[k0 .. k0+1023], so the stripes below it
  // still see positions
  for (int k0 = (T / RLE_THREADS) * RLE_THREADS; k0 >= 0; k0 -= RLE_THREADS) {
    const int k = k0 + threadIdx.x;
    uint32_t val = 0u;
    if (k <= T) {
      const uint32_t hi = (k < T) ? out[k] : (uint32_t)P;
      const uint32_t lo = (k > 0) ? out[k - 1] : 0u;
      val = hi - lo;
    }
    __syncthreads();                               // every position of this stripe (and out[k0-1]) has been read
    if (k <= T) out[k] = val;
    __syncthreads();
  }
  if (threadIdx.x == 0) n_counts[det] = (total >= cap) ? -(total + 1) : (T + 1);
}

// pycocotools rleToString, one count: writes its characters to out[0 ..) while they are below `room` (out may be null:
// count only); returns the number of characters (1..7 for |x| < 2^31)
__device__ __host__ __forceinline__ int rle_count_chars(long long x, char* out, int room) {
  int n = 0;
  bool more = true;
  while (more) {
    int c = (int)(x & 0x1f);
    x >>= 5;
    more = (c & 0x10) ? (x != -1) : (x != 0);
    if (more) c |= 0x20;
    if (out && n < room) out[n] = (char)(c + 48);
    ++n;
  }
  return n;
}

// One CTA per (detection, image).  Image img's canvas is (out_h, out_w) of its geometry row, clamped to the record.
// Writes the string of detection det into str_ws[slot * str_cap ..] and its length into lens[slot] (-1: more than run_cap
// runs); detections at or past the image's count do nothing.
__global__ void __launch_bounds__(RLE_THREADS) rle_encode_kernel(const uint32_t* __restrict__ bits, int max_num, int cap_h, int words,
                                                                 const int* __restrict__ count,
                                                                 const smb_img_geom_t* __restrict__ geom, int run_cap,
                                                                 uint32_t* __restrict__ pos_ws, char* __restrict__ str_ws,
                                                                 int str_cap, int* __restrict__ lens) {
  __shared__ int s_cnt[RLE_COLS];
  __shared__ int s_warp[32];
  const int det = blockIdx.x, img = blockIdx.y;
  const int cnt = min(max(count[img], 0), max_num);
  if (det >= cnt) return;
  const smb_img_geom_t g = geom[img];
  const int H = min(max(g.out_h, 0), cap_h), W = min(max(g.out_w, 0), words * 32);
  const size_t slot = (size_t)img * max_num + det;
  if (H == 0 || W == 0) {                          // an empty canvas has no runs: the empty string
    if (threadIdx.x == 0) lens[slot] = 0;
    return;
  }
  const uint32_t* m = bits + slot * cap_h * words;
  uint32_t* pos = pos_ws + slot * run_cap;
  char* str = str_ws + slot * str_cap;
  const int T = boundary_positions(m, words, H, W, pos, run_cap, s_cnt, s_warp);
  if (T >= run_cap) {                              // T + 1 runs do not fit (T is the same in every thread)
    if (threadIdx.x == 0) lens[slot] = -1;
    return;
  }
  // pass 2 wrote every position this block reads (boundary_positions ends with a barrier)
  const long long P = (long long)H * W;
  auto run = [&](int k) -> long long {             // length of run k of T + 1: counts[k]
    return (k < T ? (long long)pos[k] : P) - (k > 0 ? (long long)pos[k - 1] : 0ll);
  };
  int carry = 0;
  for (int k0 = 0; k0 <= T; k0 += RLE_THREADS) {
    const int k = k0 + threadIdx.x;
    long long x = 0;
    int nch = 0;
    if (k <= T) {
      x = run(k) - (k > 2 ? run(k - 2) : 0ll);
      nch = rle_count_chars(x, nullptr, 0);
    }
    int stripe;
    const int o = carry + cta_exclusive_scan<RLE_THREADS>(nch, Sum(), 0, s_warp, &stripe);
    if (k <= T && o < str_cap) rle_count_chars(x, str + o, str_cap - o);
    carry += stripe;
  }
  if (threadIdx.x == 0) lens[slot] = min(carry, str_cap);   // carry <= 7 * (T + 1) <= str_cap by construction
}

// One CTA per image: header {status, n, off[max_num + 1]} (int32) + the strings back to back into the image's img_bytes
// of the arena at *dst_word.  The strings are written only when the status is 0; header and strings stay inside the image's
// img_bytes.  Word stores: each thread gathers the 4 bytes of one destination word.
__global__ void __launch_bounds__(RLE_THREADS) rle_pack_kernel(const int* __restrict__ count, int max_num,
                                                               const int* __restrict__ lens, const char* __restrict__ str_ws,
                                                               int str_cap, const unsigned long long* __restrict__ dst_word,
                                                               int img_bytes) {
  __shared__ int s_off[RLE_MAX_DETS + 1];
  __shared__ int s_warp[32];
  __shared__ int s_bad;
  const int img = blockIdx.x;
  char* dst = reinterpret_cast<char*>(*dst_word);
  if (dst == nullptr) return;                      // no destination set: nothing to write
  const int cnt = min(max(count[img], 0), max_num);
  if (threadIdx.x == 0) s_bad = 0;
  __syncthreads();
  int len = 0;
  if ((int)threadIdx.x < cnt) {
    len = lens[(size_t)img * max_num + threadIdx.x];
    if (len < 0) {
      atomicOr(&s_bad, SMB_RLE_RUNS_OVERFLOW);
      len = 0;
    }
  }
  int total;
  const int off = cta_exclusive_scan<RLE_THREADS>(len, Sum(), 0, s_warp, &total);
  if ((int)threadIdx.x < max_num) s_off[threadIdx.x] = off;
  if (threadIdx.x == 0) s_off[max_num] = total;
  const int hdr_words = max_num + 3;
  const int str_bytes = img_bytes - 4 * hdr_words;
  const int status = s_bad | (total > str_bytes ? SMB_RLE_BYTES_OVERFLOW : 0);
  __syncthreads();
  int32_t* hdr = reinterpret_cast<int32_t*>(dst + (size_t)img * img_bytes);
  if (threadIdx.x == 0) {
    hdr[0] = status;
    hdr[1] = cnt;
  }
  for (int i = threadIdx.x; i <= max_num; i += RLE_THREADS) hdr[2 + i] = s_off[i];
  if (status != 0) return;
  uint32_t* out = reinterpret_cast<uint32_t*>(hdr + hdr_words);
  const int nw = (total + 3) >> 2;                 // <= str_bytes / 4: str_bytes is a multiple of 4
  for (int w = threadIdx.x; w < nw; w += RLE_THREADS) {
    const int p0 = 4 * w;
    int lo = 0, hi = cnt - 1;                      // the last detection whose string starts at or before p0
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (s_off[mid] <= p0) lo = mid; else hi = mid - 1;
    }
    int d = lo;
    uint32_t word = 0u;
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int p = p0 + b;
      if (p >= total) break;
      while (d + 1 < cnt && p >= s_off[d + 1]) ++d;
      const int r = p - s_off[d];
      if (r >= 0 && r < str_cap) word |= (uint32_t)(uint8_t)str_ws[((size_t)img * max_num + d) * str_cap + r] << (8 * b);
    }
    out[w] = word;
  }
}

inline size_t rle_str_cap(int run_cap) { return align_up((size_t)run_cap * RLE_MAX_CHARS, 4); }

inline void rle_ws_layout(int N, int max_num, int run_cap, size_t* off_pos, size_t* off_str, size_t* total) {
  const size_t slots = (size_t)N * max_num;
  *off_pos = align_up(slots * sizeof(int), 256);
  *off_str = *off_pos + align_up(slots * run_cap * sizeof(uint32_t), 256);
  *total = *off_str + align_up(slots * rle_str_cap(run_cap), 256);
}

}  // namespace smb

using namespace smb;

extern "C" int smb_mask_rle_counts(const uint32_t* mask_bits, int N, int mask_h, int words, int H, int W, const int* n_valid,
                                   uint32_t* counts, int cap, int* n_counts, smb_stream_t stream) {
  SMB_CHECK_ARG(mask_bits && counts && n_counts, "smb_mask_rle_counts: null pointer");
  SMB_CHECK_ARG(N >= 0 && H > 0 && W > 0 && H <= mask_h && W <= words * 32 && cap >= 2,
                "smb_mask_rle_counts: bad shape (N=%d H=%d W=%d mask_h=%d words=%d cap=%d)", N, H, W, mask_h, words, cap);
  SMB_CHECK_ARG((long long)H * W < (1ll << 31), "smb_mask_rle_counts: mask too large");
  if (N == 0) return SMB_OK;
  rle_counts_kernel<<<N, RLE_THREADS, 0, (cudaStream_t)stream>>>(mask_bits, mask_h, words, H, W, n_valid, counts, cap, n_counts);
  SMB_LAUNCH_OK("rle_counts_kernel");
  return SMB_OK;
}

extern "C" size_t smb_rle_encode_workspace_bytes(int N, int max_num, int run_cap) {
  if (N < 0 || max_num < 1 || run_cap < 1) return 0;
  size_t a, b, t;
  rle_ws_layout(N, max_num, run_cap, &a, &b, &t);
  return t;
}

extern "C" int smb_rle_encode_dev(const uint32_t* mask_bits, int N, int max_num, int cap_h, int words, const int* count,
                                  const smb_img_geom_t* geom, int run_cap, const uint64_t* dst, int img_bytes,
                                  void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(mask_bits && count && geom && dst && workspace, "smb_rle_encode_dev: null pointer");
  SMB_CHECK_ARG(N >= 0 && N <= 65535 && max_num >= 1 && max_num <= RLE_MAX_DETS && cap_h > 0 && words > 0 && run_cap >= 1 &&
                    run_cap <= (1 << 28),
                "smb_rle_encode_dev: bad shape (N=%d max_num=%d cap_h=%d words=%d run_cap=%d)", N, max_num, cap_h, words, run_cap);
  SMB_CHECK_ARG((long long)cap_h * words * 32 < (1ll << 31), "smb_rle_encode_dev: canvas too large");
  SMB_CHECK_ARG(img_bytes % 16 == 0 && img_bytes > 4 * (max_num + 3),
                "smb_rle_encode_dev: img_bytes %d must be a multiple of 16 above the %d-byte header", img_bytes, 4 * (max_num + 3));
  size_t off_pos, off_str, need;
  rle_ws_layout(N, max_num, run_cap, &off_pos, &off_str, &need);
  SMB_CHECK_ARG(workspace_bytes >= need, "smb_rle_encode_dev: workspace %zu < %zu bytes", workspace_bytes, need);
  if (N == 0) return SMB_OK;
  char* ws = static_cast<char*>(workspace);
  int* lens = reinterpret_cast<int*>(ws);
  uint32_t* pos = reinterpret_cast<uint32_t*>(ws + off_pos);
  char* str = ws + off_str;
  const int str_cap = (int)rle_str_cap(run_cap);
  rle_encode_kernel<<<dim3(max_num, N), RLE_THREADS, 0, (cudaStream_t)stream>>>(mask_bits, max_num, cap_h, words, count, geom, run_cap,
                                                                                pos, str, str_cap, lens);
  SMB_LAUNCH_OK("rle_encode_kernel");
  rle_pack_kernel<<<N, RLE_THREADS, 0, (cudaStream_t)stream>>>(count, max_num, lens, str, str_cap,
                                                               reinterpret_cast<const unsigned long long*>(dst), img_bytes);
  SMB_LAUNCH_OK("rle_pack_kernel");
  return SMB_OK;
}

extern "C" int smb_host_device_pointer(void* host_ptr, void** dev_ptr_out) {
  SMB_CHECK_ARG(host_ptr && dev_ptr_out, "smb_host_device_pointer: null pointer");
  SMB_CUDA_OK(cudaHostGetDevicePointer(dev_ptr_out, host_ptr, 0));
  return SMB_OK;
}

// pycocotools rleToString (host): returns the string length (without terminator), or -1 if `cap` is too small
extern "C" int smb_rle_to_string(const uint32_t* counts, int n, char* out, int cap) {
  int p = 0;
  for (int i = 0; i < n; ++i) {
    long x = (long)counts[i];
    if (i > 2) x -= (long)counts[i - 2];
    int more = 1;
    while (more) {
      char c = (char)(x & 0x1f);
      x >>= 5;
      more = (c & 0x10) ? (x != -1) : (x != 0);
      if (more) c |= 0x20;
      c += 48;
      if (p >= cap) return -1;
      out[p++] = c;
    }
  }
  if (p < cap) out[p] = 0;
  return p;
}
