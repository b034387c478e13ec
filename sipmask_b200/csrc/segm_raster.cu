// Segmentations to bit planes on the device: what pycocotools' rleFrPoly / rleFrBbox / rleFrString + rleDecode (and
// annToRLE's merge) compute, without run lengths ever being sorted or pixels touched by the host.
//
// A column-major mask is a list of boundary positions a_0 <= a_1 <= ...; pixel q = x * h + y is set iff the number of
// boundaries <= q is odd.  rleFrPoly's sort, differences and merging of zero-length runs only re-express that parity, and
// equal boundaries cancel in it, so the order the boundaries are produced in does not matter:
//   1. toggle_kernel : XOR one bit per boundary into the item's column-major scratch bitmap (h * w bits), and the
//                      parity of the boundaries of each column into one bit per column.
//                        run lengths: the boundaries are the inclusive prefix sums of the counts (block scan, 64 bit);
//                        polygons   : rleFrPoly's point generator in closed form, one warp per edge, each point against
//                                     the point before it (across edge joins, as the concatenated arrays on the host).
//   2. fill_kernel   : per (item, 32-column strip) the prefix XOR of every column (carry in = parity of the columns before
//                      it), transposed 32 x 32 bits at a time through shared memory and OR-ed into the row-major plane.
//                      Several items may share a plane: OR is annToRLE's merge.  Each item has its own scratch, because
//                      the XOR of two fills is not their union.
//   3. stats_kernel  : pixel count and extents of every plane, written where the caller's rows want them.
//
// Every float64 operation is an explicit _rn intrinsic so that nvcc cannot contract the host's multiply and add into an
// FMA (x86-64 pycocotools has none).
#include <limits.h>

#include "common.cuh"
#include "cta.cuh"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;

struct Launch {
  const smb_segm_item_t* items;
  int n_items;
  const double* xy;
  int64_t n_xy;                // vertices in the pool
  const uint32_t* counts;
  int64_t n_counts;
  uint32_t* planes;
  int n_planes;
  int64_t plane_stride;        // words
  int pitch;                   // words per plane row
  int64_t max_hw;
  int max_w;
  uint32_t* scratch;           // [n_items, scratch_stride] column-major toggles
  int64_t scratch_stride;
  uint32_t* colpar;            // [n_items, colpar_stride] parity of each column's toggles, one bit per column
  int colpar_stride;
};

inline int64_t scratch_words(int64_t max_hw) { return (int64_t)smb::align_up((size_t)((max_hw + 31) / 32), 32); }
inline int colpar_words(int max_w) { return (int)smb::align_up((size_t)((max_w + 31) / 32), 32); }

// Everything an item indexes with, bounded against what the launch owns.
__device__ __forceinline__ bool item_ok(const Launch& L, const smb_segm_item_t& it) {
  if (it.h < 0 || it.w < 0 || (int64_t)it.h * it.w > L.max_hw || it.w > L.max_w) return false;
  if (it.plane < 0 || it.plane >= L.n_planes) return false;
  if ((it.w + 31) / 32 > L.pitch || (int64_t)it.h * L.pitch > L.plane_stride) return false;
  if (it.off < 0 || it.n < 0) return false;
  if (it.kind == 0) return it.off <= L.n_xy && it.n <= L.n_xy - it.off;
  if (it.kind == 1) return it.off <= L.n_counts && it.n <= L.n_counts - it.off;
  return false;
}

__device__ __forceinline__ void toggle(uint32_t* scratch, uint32_t* colpar, int64_t pos, int col) {
  atomicXor(scratch + (pos >> 5), 1u << (pos & 31));
  atomicXor(colpar + (col >> 5), 1u << (col & 31));
}

// ------------------------------------------------------------------------------------------------ polygons
// One edge of rleFrPoly's upsampled polygon (vertices scaled by 5 and rounded): max(dx, dy) + 1 points, generated from
// the smaller end when `flip`.
struct Edge {
  int xs, ys, dx, dy, len;
  bool flip;
  double s;
};

__device__ __forceinline__ int scaled(double c) { return __double2int_rz(__dadd_rn(__dmul_rn(5.0, c), .5)); }

__device__ __forceinline__ Edge load_edge(const double* __restrict__ xy, int64_t k, int64_t j) {
  const int64_t jn = j + 1 < k ? j + 1 : 0;
  int xs = scaled(xy[2 * j]), ys = scaled(xy[2 * j + 1]), xe = scaled(xy[2 * jn]), ye = scaled(xy[2 * jn + 1]);
  Edge e;
  e.dx = abs(xe - xs);
  e.dy = abs(ys - ye);
  e.flip = (e.dx >= e.dy && xs > xe) || (e.dx < e.dy && ys > ye);
  if (e.flip) { int t = xs; xs = xe; xe = t; t = ys; ys = ye; ye = t; }
  e.xs = xs;
  e.ys = ys;
  e.len = max(e.dx, e.dy);
  e.s = e.len == 0 ? 0.0 : (e.dx >= e.dy ? __ddiv_rn((double)(ye - ys), (double)e.dx) : __ddiv_rn((double)(xe - xs), (double)e.dy));
  return e;
}

__device__ __forceinline__ void edge_point(const Edge& e, int d, int& u, int& v) {
  if (e.len == 0) {                                // s = 0 / 0: pycocotools stores (int)NaN, INT_MIN on x86-64
    u = e.xs;
    v = INT_MIN;
    return;
  }
  const int t = e.flip ? e.len - d : d;
  if (e.dx >= e.dy) {
    u = t + e.xs;
    v = __double2int_rz(__dadd_rn(__dadd_rn((double)e.ys, __dmul_rn(e.s, (double)t)), .5));
  } else {
    v = t + e.ys;
    u = __double2int_rz(__dadd_rn(__dadd_rn((double)e.xs, __dmul_rn(e.s, (double)t)), .5));
  }
}

// The boundary rleFrPoly derives from two consecutive points, toggled unless it filters it.
__device__ __forceinline__ void crossing(int u0, int v0, int u1, int v1, int h, int w, int64_t hw, uint32_t* scratch,
                                         uint32_t* colpar) {
  if (u1 == u0) return;
  double xd = (double)(u1 < u0 ? u1 : u1 - 1);
  xd = __dsub_rn(__ddiv_rn(__dadd_rn(xd, .5), 5.0), .5);
  if (floor(xd) != xd || xd < 0 || xd > (double)(w - 1)) return;
  double yd = (double)(v1 < v0 ? v1 : v0);
  yd = __dsub_rn(__ddiv_rn(__dadd_rn(yd, .5), 5.0), .5);
  if (yd < 0) yd = 0; else if (yd > h) yd = h;
  yd = ceil(yd);
  const int x = (int)xd, y = (int)yd;
  const int64_t pos = (int64_t)x * h + y;          // y == h is the first pixel of the next column
  if (pos < hw) toggle(scratch, colpar, pos, y == h ? x + 1 : x);
}

__global__ void __launch_bounds__(kThreads) segm_toggle_kernel(Launch L, int* __restrict__ status) {
  __shared__ uint64_t s_warp[kWarps];
  const int i = blockIdx.x, tid = threadIdx.x, lid = tid & 31, warp = tid >> 5;
  const smb_segm_item_t it = L.items[i];
  if (!item_ok(L, it)) {
    if (tid == 0) atomicOr(status, SMB_SEGM_RANGE);
    return;
  }
  const int h = it.h, w = it.w;
  const int64_t hw = (int64_t)h * w;
  if (hw == 0) return;
  uint32_t* scratch = L.scratch + (int64_t)i * L.scratch_stride;
  uint32_t* colpar = L.colpar + (int64_t)i * L.colpar_stride;
  if (it.kind == 0) {
    const double* xy = L.xy + 2 * it.off;
    for (int64_t j = warp; j < it.n; j += kWarps) {
      const Edge e = load_edge(xy, it.n, j);
      int up = 0, vp = 0;                          // the point before this edge's first: the last of the edge before
      if (j > 0) {
        const Edge p = load_edge(xy, it.n, j - 1);
        edge_point(p, p.len, up, vp);
      }
      for (int d0 = 0; d0 <= e.len; d0 += 32) {
        const int d = d0 + lid;
        if (d > e.len || (j == 0 && d == 0)) continue;
        int u0 = up, v0 = vp, u1, v1;
        if (d > 0) edge_point(e, d - 1, u0, v0);
        edge_point(e, d, u1, v1);
        crossing(u0, v0, u1, v1, h, w, hw, scratch, colpar);
      }
    }
  } else {
    const uint32_t* cnts = L.counts + it.off;
    uint64_t carry = 0;
    for (int64_t base = 0; base < it.n; base += kThreads) {
      const int64_t e = base + tid;
      const uint64_t v = e < it.n ? cnts[e] : 0;
      uint64_t total;
      const uint64_t pos = carry + smb::cta_inclusive_scan<kThreads>(v, smb::Sum(), s_warp, &total);
      if (e < it.n && pos < (uint64_t)hw) toggle(scratch, colpar, (int64_t)pos, (int)(pos / (uint64_t)h));
      carry += total;
    }
  }
}

// ------------------------------------------------------------------------------------------------ fill + transpose
__global__ void __launch_bounds__(kThreads) segm_fill_kernel(Launch L) {
  __shared__ uint32_t s_tile[32][33];              // [column of the strip][32-row word of the chunk]
  const int i = blockIdx.x, s = blockIdx.y, tid = threadIdx.x, lid = tid & 31, warp = tid >> 5;
  const smb_segm_item_t it = L.items[i];
  if (!item_ok(L, it)) return;                     // reported by toggle_kernel
  const int h = it.h, w = it.w;
  if (h == 0 || s * 32 >= w) return;
  const int64_t nwords = ((int64_t)h * w + 31) >> 5;
  const uint32_t* scratch = L.scratch + (int64_t)i * L.scratch_stride;
  const uint32_t* colpar = L.colpar + (int64_t)i * L.colpar_stride;
  uint32_t* plane = L.planes + (int64_t)it.plane * L.plane_stride;
  // carry into the strip: the parity of every boundary in the columns before it
  uint32_t base = 0;
  for (int q = lid; q < s; q += 32) base ^= colpar[q];
  base = __popc(base) & 1;
  for (int o = 16; o > 0; o >>= 1) base ^= __shfl_xor_sync(0xffffffffu, base, o);
  const uint32_t cp = colpar[s];
  uint32_t carry[4];                               // this warp's columns 4 * warp + k
  for (int k = 0; k < 4; ++k) carry[k] = base ^ (__popc(cp & ((1u << (warp * 4 + k)) - 1u)) & 1);
  for (int y0 = 0; y0 < h; y0 += 1024) {
    for (int k = 0; k < 4; ++k) {
      const int c = warp * 4 + k, x = s * 32 + c, y = y0 + lid * 32;
      uint32_t v = 0, valid = 0;
      if (x < w && y < h) {
        const int64_t b = (int64_t)x * h + y;
        const int64_t wi = b >> 5;
        const uint32_t lo = scratch[wi], hi = wi + 1 < nwords ? scratch[wi + 1] : 0u;
        valid = h - y >= 32 ? 0xffffffffu : (1u << (h - y)) - 1u;
        v = __funnelshift_r(lo, hi, (uint32_t)(b & 31)) & valid;
      }
      v ^= v << 1; v ^= v << 2; v ^= v << 4; v ^= v << 8; v ^= v << 16;      // bit r = parity of the toggles <= r
      v &= valid;
      const uint32_t par = valid ? (v >> (31 - __clz(valid))) & 1u : 0u;     // parity of the whole word
      const uint32_t incl = smb::warp_inclusive_scan(par, smb::Xor());
      if (carry[k] ^ incl ^ par) v ^= valid;
      carry[k] ^= __shfl_sync(0xffffffffu, incl, 31);
      s_tile[c][lid] = v;
    }
    __syncthreads();
    for (int r = warp; r < 32; r += kWarps) {      // 32 x 32 bit transpose: lane = column in, lane = row out
      const uint32_t v = s_tile[lid][r];
      uint32_t mine = 0;
      for (int b = 0; b < 32; ++b) {
        const uint32_t o = __ballot_sync(0xffffffffu, (v >> b) & 1u);
        if (lid == b) mine = o;
      }
      const int y = y0 + r * 32 + lid;
      if (y < h && mine) atomicOr(plane + (int64_t)y * L.pitch + s, mine);
    }
    __syncthreads();
  }
}

// ------------------------------------------------------------------------------------------------ stats
// One CTA per item; the first item of each plane (items of a plane are adjacent) reports the plane.
__global__ void __launch_bounds__(kThreads) segm_stats_kernel(Launch L, int32_t* __restrict__ area, int64_t area_stride,
                                                              int32_t* __restrict__ ext, int64_t ext_stride) {
  __shared__ int s_red[kWarps][5];
  const int i = blockIdx.x, tid = threadIdx.x, lid = tid & 31, warp = tid >> 5;
  const smb_segm_item_t it = L.items[i];
  if (!item_ok(L, it)) return;
  if (i > 0 && L.items[i - 1].plane == it.plane) return;
  const uint32_t* plane = L.planes + (int64_t)it.plane * L.plane_stride;
  const int words = (it.w + 31) >> 5;
  int v[5] = {0, INT_MAX, -1, INT_MAX, -1};        // area, row0, row1, word0, word1
  for (int e = tid; e < it.h * words; e += kThreads) {
    const int y = e / words, x = e - y * words;
    const uint32_t u = plane[(int64_t)y * L.pitch + x];
    if (u) { v[0] += __popc(u); v[1] = min(v[1], y); v[2] = max(v[2], y); v[3] = min(v[3], x); v[4] = max(v[4], x); }
  }
  for (int o = 16; o > 0; o >>= 1) {
    v[0] += __shfl_xor_sync(0xffffffffu, v[0], o);
    v[1] = min(v[1], __shfl_xor_sync(0xffffffffu, v[1], o));
    v[2] = max(v[2], __shfl_xor_sync(0xffffffffu, v[2], o));
    v[3] = min(v[3], __shfl_xor_sync(0xffffffffu, v[3], o));
    v[4] = max(v[4], __shfl_xor_sync(0xffffffffu, v[4], o));
  }
  if (lid == 0)
    for (int q = 0; q < 5; ++q) s_red[warp][q] = v[q];
  __syncthreads();
  if (tid != 0) return;
  for (int q = 1; q < kWarps; ++q) {
    v[0] += s_red[q][0];
    v[1] = min(v[1], s_red[q][1]); v[2] = max(v[2], s_red[q][2]);
    v[3] = min(v[3], s_red[q][3]); v[4] = max(v[4], s_red[q][4]);
  }
  if (area) area[(int64_t)it.plane * area_stride] = v[0];
  if (ext) {
    int32_t* e = ext + (int64_t)it.plane * ext_stride;
    if (v[0]) { e[0] = v[1]; e[1] = v[2] + 1; e[2] = v[3]; e[3] = v[4] + 1; }
    else e[0] = e[1] = e[2] = e[3] = 0;
  }
}

}  // namespace

extern "C" size_t smb_segm_raster_workspace_bytes(int n_items, int64_t max_hw, int max_w) {
  if (n_items <= 0 || max_hw < 0 || max_w < 0) return 0;
  return (size_t)n_items * (size_t)(scratch_words(max_hw) + colpar_words(max_w)) * sizeof(uint32_t);
}

extern "C" int smb_segm_raster_dev(const smb_segm_item_t* items, int n_items, const double* xy_pool, int64_t n_xy,
                                   const uint32_t* count_pool, int64_t n_counts, int64_t max_hw, int max_w, uint32_t* planes,
                                   int n_planes, int64_t plane_stride_words, int pitch, int32_t* area, int64_t area_stride,
                                   int32_t* ext, int64_t ext_stride, int* status, void* workspace, size_t workspace_bytes,
                                   smb_stream_t stream) {
  SMB_CHECK_ARG(n_items >= 0 && n_xy >= 0 && n_counts >= 0 && max_hw >= 0 && max_hw < (1ll << 31) && max_w >= 0 &&
                    n_planes >= 0 && plane_stride_words >= 0 && pitch >= 0 && max_w <= 32 * 65535,
                "smb_segm_raster_dev: bad sizes (n_items %d, n_xy %lld, n_counts %lld, max_hw %lld, max_w %d, n_planes %d)",
                n_items, (long long)n_xy, (long long)n_counts, (long long)max_hw, max_w, n_planes);
  cudaStream_t st = (cudaStream_t)stream;
  if (n_planes > 0 && plane_stride_words > 0) {
    SMB_CHECK_ARG(planes, "smb_segm_raster_dev: null planes");
    SMB_CUDA_OK(cudaMemsetAsync(planes, 0, (size_t)n_planes * plane_stride_words * sizeof(uint32_t), st));
  }
  if (n_items == 0) return SMB_OK;
  SMB_CHECK_ARG(items && status && workspace && (xy_pool || n_xy == 0) && (count_pool || n_counts == 0),
                "smb_segm_raster_dev: null pointer");
  const size_t need = smb_segm_raster_workspace_bytes(n_items, max_hw, max_w);
  SMB_CHECK_ARG(workspace_bytes >= need, "smb_segm_raster_dev: workspace of %zu bytes, %zu needed", workspace_bytes, need);
  Launch L;
  L.items = items; L.n_items = n_items;
  L.xy = xy_pool; L.n_xy = n_xy;
  L.counts = count_pool; L.n_counts = n_counts;
  L.planes = planes; L.n_planes = n_planes; L.plane_stride = plane_stride_words; L.pitch = pitch;
  L.max_hw = max_hw; L.max_w = max_w;
  L.scratch_stride = scratch_words(max_hw);
  L.colpar_stride = colpar_words(max_w);
  L.scratch = (uint32_t*)workspace;
  L.colpar = L.scratch + (size_t)n_items * L.scratch_stride;
  if (need) SMB_CUDA_OK(cudaMemsetAsync(workspace, 0, need, st));
  segm_toggle_kernel<<<n_items, kThreads, 0, st>>>(L, status);
  SMB_LAUNCH_OK("segm_toggle_kernel");
  if (max_w > 0) {
    segm_fill_kernel<<<dim3(n_items, (max_w + 31) / 32), kThreads, 0, st>>>(L);
    SMB_LAUNCH_OK("segm_fill_kernel");
  }
  if (area || ext) {
    segm_stats_kernel<<<n_items, kThreads, 0, st>>>(L, area, area_stride, ext, ext_stride);
    SMB_LAUNCH_OK("segm_stats_kernel");
  }
  return SMB_OK;
}
