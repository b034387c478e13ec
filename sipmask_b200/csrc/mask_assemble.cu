// Fused SipMask mask assembly for sm_90a.
//
// Reference (SipMask-mmdetection/mmdet/):
//   models/anchor_heads/sipmask_head.py:609-633   4x sgemm -> 4x sigmoid -> stack -> CropSplit -> permute
//   ops/crop/src/crop_split_cuda_kernel.cu:19-59  CropSplitKernelForward
// The reference materialises [4,H,W,N] sigmoid maps (~2.5 GB of HBM traffic for 142 MB of
// algorithmic bytes, SURVEY.md §8a-9).  Here one kernel reads every prototype pixel once into
// registers, and for each detection evaluates only the ONE 32-term dot product selected by the
// CropSplit cell of that pixel, and only for pixels inside the box; everything else is a zero store.
// HBM-bound: algorithmic bytes = protos (H*W*32*sizeof) + out (N*H*W*sizeof).
#include "common.cuh"

namespace smb {

struct __align__(16) BoxP {
  float x1, y1, x2, y2, roi_w, roi_h, pad0, pad1;
};

constexpr int MA_TW = 64;   // tile width  (16 threads x 4 pixels)
constexpr int MA_TH = 8;    // tile height

template <typename PT>
__device__ __forceinline__ float to_f(PT v);
template <>
__device__ __forceinline__ float to_f<float>(float v) { return v; }
template <>
__device__ __forceinline__ float to_f<__half>(__half v) { return __half2float(v); }

template <typename OT>
__device__ __forceinline__ void store4(OT* p, const float* o, bool vec, int nvalid);
template <>
__device__ __forceinline__ void store4<float>(float* p, const float* o, bool vec, int nvalid) {
  if (vec) {
    *reinterpret_cast<float4*>(p) = make_float4(o[0], o[1], o[2], o[3]);
  } else {
    for (int i = 0; i < nvalid; ++i) p[i] = o[i];
  }
}
template <>
__device__ __forceinline__ void store4<__half>(__half* p, const float* o, bool vec, int nvalid) {
  if (vec) {
    __half2 a = __floats2half2_rn(o[0], o[1]);
    __half2 b = __floats2half2_rn(o[2], o[3]);
    uint2 u;
    u.x = *reinterpret_cast<uint32_t*>(&a);
    u.y = *reinterpret_cast<uint32_t*>(&b);
    *reinterpret_cast<uint2*>(p) = u;
  } else {
    for (int i = 0; i < nvalid; ++i) p[i] = __float2half_rn(o[i]);
  }
}

template <typename OT>
__device__ __forceinline__ void store1(OT* p, float v);
template <>
__device__ __forceinline__ void store1<float>(float* p, float v) { *p = v; }
template <>
__device__ __forceinline__ void store1<__half>(__half* p, float v) { *p = __float2half_rn(v); }

// grid: (ceil(W/64), ceil(H/8)), block 256 (warp = tile row, lane = columns lane and lane + 32).  The output has been
// zero-filled by a memset node (the bulk of the 107 MB pos_masks tensor is zeros and a memset runs at store bandwidth); this
// kernel only touches pixels inside boxes: a CTA stages its 8 x 64 prototype pixels in shared memory ONCE (16-byte-chunk
// XOR swizzle: conflict-free LDS.128), lists the detections whose roi intersects the tile, then evaluates, per listed
// detection and in-box pixel, the ONE 32-term dot product selected by the CropSplit cell (coefficients: warp-uniform L1 reads).
constexpr int MA_LIST = 128;   // detections listed per pass
constexpr int MA_THREADS2 = 256;

template <typename PT> struct FusedCfg;
template <> struct FusedCfg<__half> { static constexpr int kChunks = 4; };   // 64 B / pixel
template <> struct FusedCfg<float> { static constexpr int kChunks = 8; };    // 128 B / pixel

template <typename PT>
__device__ __forceinline__ int swz(int p, int k);
template <>
__device__ __forceinline__ int swz<__half>(int p, int k) { return k ^ ((p >> 1) & 3); }
template <>
__device__ __forceinline__ int swz<float>(int p, int k) { return k ^ (p & 7); }

// 32-term dot product of shared-memory pixel p (swizzled 16-byte chunks) with cof[0..31]: sequential fmaf over channels,
// the same summation order in the dense and the fused kernel, so both give bit-identical mask values.
template <typename PT>
__device__ __forceinline__ float dot32_swz(const unsigned char* s_p, int p, const float* __restrict__ cof);
template <>
__device__ __forceinline__ float dot32_swz<__half>(const unsigned char* s_p, int p, const float* __restrict__ cof) {
  float acc = 0.f;
  const uint4* q = reinterpret_cast<const uint4*>(s_p + (size_t)p * 64);
  const float4* c4 = reinterpret_cast<const float4*>(cof);
#pragma unroll
  for (int v = 0; v < 4; ++v) {
    const uint4 u = q[swz<__half>(p, v)];
    const __half2* hh = reinterpret_cast<const __half2*>(&u);
    const float4 ca = __ldg(c4 + 2 * v), cb = __ldg(c4 + 2 * v + 1);
    const float2 f0 = __half22float2(hh[0]), f1 = __half22float2(hh[1]), f2 = __half22float2(hh[2]), f3 = __half22float2(hh[3]);
    acc = fmaf(f0.x, ca.x, acc); acc = fmaf(f0.y, ca.y, acc); acc = fmaf(f1.x, ca.z, acc); acc = fmaf(f1.y, ca.w, acc);
    acc = fmaf(f2.x, cb.x, acc); acc = fmaf(f2.y, cb.y, acc); acc = fmaf(f3.x, cb.z, acc); acc = fmaf(f3.y, cb.w, acc);
  }
  return acc;
}
template <>
__device__ __forceinline__ float dot32_swz<float>(const unsigned char* s_p, int p, const float* __restrict__ cof) {
  float acc = 0.f;
  const float4* q = reinterpret_cast<const float4*>(s_p + (size_t)p * 128);
  const float4* c4 = reinterpret_cast<const float4*>(cof);
#pragma unroll
  for (int v = 0; v < 8; ++v) {
    const float4 a = q[swz<float>(p, v)], c = __ldg(c4 + v);
    acc = fmaf(a.x, c.x, acc); acc = fmaf(a.y, c.y, acc); acc = fmaf(a.z, c.z, acc); acc = fmaf(a.w, c.w, acc);
  }
  return acc;
}

// stage an SRa x SCa window of prototype pixels (top-left source pixel (ys0, xs0)) into swizzled shared memory
template <typename PT, bool HWC>
__device__ __forceinline__ void stage_window(const PT* __restrict__ protos, unsigned char* s_p, int H, int W, int ys0, int xs0,
                                             int SRa, int SCa, int nthreads) {
  constexpr int CH = FusedCfg<PT>::kChunks, PX_BYTES = CH * 16;
  const int npx = SRa * SCa;
  if (HWC) {
    for (int i = threadIdx.x; i < npx * CH; i += nthreads) {
      const int p = i / CH, k = i - p * CH;
      const int r = p / SCa, c = p - r * SCa;
      const uint4 v = __ldg(reinterpret_cast<const uint4*>(protos + ((size_t)(ys0 + r) * W + xs0 + c) * 32) + k);
      *reinterpret_cast<uint4*>(s_p + (size_t)p * PX_BYTES + swz<PT>(p, k) * 16) = v;
    }
  } else {
    for (int i = threadIdx.x; i < npx * 32; i += nthreads) {
      const int ch = i / npx, p = i - ch * npx;
      const int r = p / SCa, c = p - r * SCa;
      const PT v = protos[((size_t)ch * H + ys0 + r) * W + xs0 + c];
      constexpr int EPC = 16 / (int)sizeof(PT);                              // elements per 16-byte chunk
      reinterpret_cast<PT*>(s_p + (size_t)p * PX_BYTES + swz<PT>(p, ch / EPC) * 16)[ch % EPC] = v;
    }
  }
}

template <typename OT>
__device__ __forceinline__ void store_zero4(OT* p);
template <>
__device__ __forceinline__ void store_zero4<float>(float* p) { *reinterpret_cast<float4*>(p) = make_float4(0.f, 0.f, 0.f, 0.f); }
template <>
__device__ __forceinline__ void store_zero4<__half>(__half* p) { *reinterpret_cast<uint2*>(p) = make_uint2(0u, 0u); }

// The kernel writes EVERY output element exactly once (no separate zero-fill pass): for a detection whose roi misses the
// tile the CTA stores 8 x 256 bytes of zeros (one 16-byte store per thread, 128 threads), for an intersecting one each warp
// stores its row (value inside the roi, 0 outside; 128 bytes per store instruction).  With seven CTAs per SM the stores of
// ~100 detections per tile are in flight concurrently - the r1 kernel had the same store pattern but 8 warps per SM and a
// serial per-thread detection loop.
template <typename PT, bool HWC, typename OT>
__global__ void __launch_bounds__(MA_THREADS2) mask_assemble_kernel(
    const PT* __restrict__ protos, const float* __restrict__ cofs, const float* __restrict__ boxes,
    GeomArg ga, OT* __restrict__ out, int H, int W, int N) {
  extern __shared__ __align__(16) unsigned char s_p[];        // [MA_TH * MA_TW] swizzled pixels (32 KB fp16 / 64 KB fp32)
  __shared__ BoxP s_box[MA_LIST];
  __shared__ int s_det[MA_LIST];
  __shared__ int s_cnt;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const smb_img_geom_t geom = load_geom(ga);
  const float sx1 = geom.roi_scale[0], sy1 = geom.roi_scale[1], sx2 = geom.roi_scale[2], sy2 = geom.roi_scale[3];
  const int y0t = blockIdx.y * MA_TH, x0t = blockIdx.x * MA_TW;
  const int SRa = min(MA_TH, H - y0t), SCa = min(MA_TW, W - x0t);
  stage_window<PT, HWC>(protos, s_p, H, W, y0t, x0t, SRa, SCa, MA_THREADS2);
  const int h = y0t + warp;
  const bool row_ok = warp < SRa;
  const float hf = (float)h;
  const float tile_x0 = (float)x0t, tile_x1 = (float)(x0t + SCa - 1), tile_y0 = (float)y0t, tile_y1 = (float)(y0t + SRa - 1);
  // zero-fill role: thread t < 128 owns the 4 pixels (row t / 16, columns 4 * (t % 16) ..) of the tile
  const int zr = threadIdx.x >> 4, zc = (threadIdx.x & 15) * 4;
  const bool z_vec = threadIdx.x < 128 && zr < SRa && zc + 3 < SCa && ((W & 3) == 0);
  const bool z_tail = threadIdx.x < 128 && zr < SRa && !z_vec && zc < SCa;

  for (int n0 = 0; n0 < N; n0 += MA_LIST) {
    const int nb = min(MA_LIST, N - n0);
    __syncthreads();                                   // window staged / previous pass done with the list
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    bool mine_listed = false;
    if (threadIdx.x < nb) {
      const float* b = boxes + (size_t)(n0 + threadIdx.x) * 4;
      BoxP bp;
      bp.x1 = b[0] * sx1; bp.y1 = b[1] * sy1; bp.x2 = b[2] * sx2; bp.y2 = b[3] * sy2;
      // some pixel (integer coordinates) of the tile satisfies x1 <= w < x2 and y1 <= h < y2 ?
      if (tile_x1 >= bp.x1 && tile_x0 < bp.x2 && tile_y1 >= bp.y1 && tile_y0 < bp.y2) {
        // (roi_x2-roi_x1+0.1)/num_cell: float difference, then double (0.1 is a double literal),
        // narrowed to float on assignment (crop_split_cuda_kernel.cu:46-47).
        bp.roi_w = (float)(((double)(bp.x2 - bp.x1) + 0.1) / 2);
        bp.roi_h = (float)(((double)(bp.y2 - bp.y1) + 0.1) / 2);
        bp.pad0 = bp.pad1 = 0.f;
        const int pos = atomicAdd(&s_cnt, 1);
        s_box[pos] = bp;
        s_det[pos] = n0 + threadIdx.x;
        mine_listed = true;
      }
    }
    // listed flags of this pass as four 32-bit ballots, broadcast through shared memory
    __shared__ unsigned s_listed[MA_LIST / 32];
    {
      const unsigned bal = __ballot_sync(0xffffffffu, mine_listed);
      if (lane == 0 && warp < MA_LIST / 32) s_listed[warp] = bal;
    }
    __syncthreads();
    const int cnt = s_cnt;
    // ---- detections whose roi misses the tile: zeros (16 bytes per thread, 8 rows x 256 B per detection)
    if (z_vec | z_tail) {
      for (int j = 0; j < nb; ++j) {
        if ((s_listed[j >> 5] >> (j & 31)) & 1u) continue;
        OT* dst = out + ((size_t)(n0 + j) * H + (y0t + zr)) * W + x0t + zc;
        if (z_vec) {
          store_zero4<OT>(dst);
        } else {
          for (int e = 0; e < 4 && zc + e < SCa; ++e) store1<OT>(dst + e, 0.f);
        }
      }
    }
    if (!row_ok) continue;
    // ---- listed detections: every pixel of the tile row is written (value inside the roi, 0 outside)
    for (int j = 0; j < cnt; ++j) {
      const BoxP b = s_box[j];
      const bool row_in = (hf >= b.y1) & (hf < b.y2);     // warp-uniform
      const int n = s_det[j];
      const float* cof = cofs + (size_t)n * 128;
      const int idx_h = row_in ? (int)__fdiv_rn(hf - b.y1, b.roi_h) : 0;
      OT* dst = out + ((size_t)n * H + h) * W + x0t;
#pragma unroll
      for (int q = 0; q < MA_TW / 32; ++q) {
        const int c = lane + q * 32;
        if (c < SCa) {
          const float wf = (float)(x0t + c);
          float v = 0.f;
          if (row_in & (wf >= b.x1) & (wf < b.x2)) {
            const int idx_w = (int)__fdiv_rn(wf - b.x1, b.roi_w);
            const int cell = min(max(idx_h * 2 + idx_w, 0), 3);
            v = sigmoidf_(dot32_swz<PT>(s_p, warp * SCa + c, cof + cell * 32));
          }
          store1<OT>(dst + c, v);
        }
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Bilinear resize (align_corners=False) + threshold of pos_masks, pasted top-left into [N,out_h,out_w]
// (sipmask_head.py:630-633,648-654).  The reference calls F.interpolate(scale_factor = 2 / scale_factor) (per axis on the
// SSD path): the interpolated size is (full_h, full_w) = floor(H * s), floor(W * s) and the source coordinate of output
// pixel y is ry * (y + 0.5) - 0.5 with ry = H / full_h (PyTorch's recompute_scale_factor=True rule, the behaviour of
// the PyTorch version the reference pins), clamped at 0; neighbours clamp at H - 1.  Pixels beyond (full_h, full_w) are 0.
struct Resize {
  int full_h, full_w;
  float ry, rx;
};

__device__ __forceinline__ void src_index(float r, int dst, int size, int& i0, int& i1, float& l) {
  float s = r * ((float)dst + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  i0 = min((int)s, size - 1);
  i1 = i0 + (i0 < size - 1 ? 1 : 0);
  l = s - (float)i0;
}

// One thread = 4 consecutive output pixels of one row.
template <typename PT>
__global__ void __launch_bounds__(256) resize_thresh_kernel(const PT* __restrict__ pos, uint8_t* __restrict__ out,
                                                            int N, int H, int W, int out_h, int out_w, Resize rs, float thr) {
  const int xq = blockIdx.x * blockDim.x + threadIdx.x;   // quad index along x
  const int y = blockIdx.y;
  const int n = blockIdx.z;
  const int x0 = xq * 4;
  if (x0 >= out_w) return;
  uint8_t r[4] = {0, 0, 0, 0};
  if (y < rs.full_h) {
    int y0, y1;
    float ly;
    src_index(rs.ry, y, H, y0, y1, ly);
    const float hy = 1.f - ly;
    const PT* r0 = pos + ((size_t)n * H + y0) * W;
    const PT* r1 = pos + ((size_t)n * H + y1) * W;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int x = x0 + i;
      if (x < out_w && x < rs.full_w) {
        int xa, xb;
        float lx;
        src_index(rs.rx, x, W, xa, xb, lx);
        const float hx = 1.f - lx;
        const float v = hy * (hx * to_f<PT>(r0[xa]) + lx * to_f<PT>(r0[xb])) +
                        ly * (hx * to_f<PT>(r1[xa]) + lx * to_f<PT>(r1[xb]));
        r[i] = v > thr ? 1 : 0;
      }
    }
  }
  uint8_t* o = out + ((size_t)n * out_h + y) * out_w + x0;
  if (x0 + 3 < out_w && ((out_w & 3) == 0)) {
    *reinterpret_cast<uchar4*>(o) = make_uchar4(r[0], r[1], r[2], r[3]);
  } else {
    for (int i = 0; i < 4 && x0 + i < out_w; ++i) o[i] = r[i];
  }
}

// Same, bit-packed: out_bits [N, out_h, words] uint32, bit (x & 31) of word (x >> 5), LSB first.  One warp = one word
// (lane = pixel, __ballot_sync packs): 13.4 MB instead of 107 MB per 100 masks at 800x1344 -> one small D2H.
template <typename PT>
__global__ void __launch_bounds__(256) resize_thresh_pack_kernel(const PT* __restrict__ pos, uint32_t* __restrict__ out,
                                                                 int N, int H, int W, int out_h, int out_w, int words,
                                                                 Resize rs, float thr) {
  const int lane = threadIdx.x & 31;
  const int wq = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int y = blockIdx.y;
  const int n = blockIdx.z;
  if (wq >= words) return;                                 // warp-uniform
  const int x = wq * 32 + lane;
  bool bit = false;
  if (y < rs.full_h && x < out_w && x < rs.full_w) {
    int y0, y1, xa, xb;
    float ly, lx;
    src_index(rs.ry, y, H, y0, y1, ly);
    src_index(rs.rx, x, W, xa, xb, lx);
    const float hy = 1.f - ly, hx = 1.f - lx;
    const PT* r0 = pos + ((size_t)n * H + y0) * W;
    const PT* r1 = pos + ((size_t)n * H + y1) * W;
    const float v = hy * (hx * to_f<PT>(r0[xa]) + lx * to_f<PT>(r0[xb])) + ly * (hx * to_f<PT>(r1[xa]) + lx * to_f<PT>(r1[xb]));
    bit = v > thr;
  }
  const uint32_t bits = __ballot_sync(0xffffffffu, bit);
  if (lane == 0) out[((size_t)n * out_h + y) * words + wq] = bits;
}

// ---------------------------------------------------------------------------------------------------------------
// Fully fused mask path: prototypes -> (selected sub-region dot product -> sigmoid -> crop) -> bilinear resize
// -> threshold -> bit-pack, without ever materialising pos_masks [N,H,W] (sipmask_head.py:609-633,648-654).
// Algorithmic HBM traffic = prototypes once + N*out_h*words*4 bytes of bits (13.4 MB for 100 masks at 800x1333).
//
// The bit planes are zero-filled by a memset node first (almost all words are zero).  The kernel is TILE-stationary and
// two-phase: a CTA owns TY output rows x TW output words, stages the prototype pixels those outputs can read (at most
// SR_CAP x SC_CAP, 16-byte-chunk XOR swizzle: conflict-free LDS.128) in shared memory ONCE, lists the detections whose
// roi intersects that source window, and for every listed detection
//   phase 1: one sigmoid-dot per source pixel (cell selected by CropSplit, 0 outside the box) -> s_val (fp32 tile),
//   phase 2: one lane per output pixel: 4-tap bilinear from s_val, `> thr`, __ballot_sync -> one 32-bit word per warp.
// (The previous kernel re-evaluated the dot product for up to four output pixels per source pixel: 2.8 % of HBM peak.)
constexpr int MF_THREADS = 256, MF_LIST = 128, MF_TY_MAX = 16;
struct RowC {
  int o0, o1;       // offsets of the two source rows inside the window (row * SCa)
  int y0, y1;       // the source rows themselves
  float ly;
  int pad_[3];
};

template <typename PT, bool HWC>
__global__ void __launch_bounds__(MF_THREADS) mask_fused_pack_kernel(
    const PT* __restrict__ protos, const float* __restrict__ cofs, const float* __restrict__ boxes, GeomArg ga,
    uint32_t* __restrict__ out, int H, int W, int N, int words, size_t plane, int TY, int TW, int win_cap, float thr) {
  constexpr int PX_BYTES = FusedCfg<PT>::kChunks * 16;
  extern __shared__ __align__(16) unsigned char mf_smem[];
  unsigned char* s_p = mf_smem;                                                        // [win_cap] swizzled pixels
  float* s_val = reinterpret_cast<float*>(mf_smem + (size_t)win_cap * PX_BYTES);        // [2][win_cap]
  BoxP* s_box = reinterpret_cast<BoxP*>(s_val + 2 * win_cap);                          // [MF_LIST]
  RowC* s_row = reinterpret_cast<RowC*>(s_box + MF_LIST);                              // [MF_TY_MAX]
  int* s_det = reinterpret_cast<int*>(s_row + MF_TY_MAX);                              // [MF_LIST]
  int* s_cnt = s_det + MF_LIST;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const smb_img_geom_t geom = load_geom(ga);
  const Resize rs = {geom.full_h, geom.full_w, geom.ry, geom.rx};
  const float sx1 = geom.roi_scale[0], sy1 = geom.roi_scale[1], sx2 = geom.roi_scale[2], sy2 = geom.roi_scale[3];
  const int y_first = blockIdx.y * TY, wq_first = blockIdx.x * TW;
  const int vh = min(geom.out_h, rs.full_h), vw = min(geom.out_w, rs.full_w);     // valid output frame; everything else stays 0
  const int y_last = min(y_first + TY, vh) - 1;
  const int x_first = wq_first * 32, x_last = min(x_first + TW * 32, vw) - 1;
  if (y_last < y_first || x_last < x_first) return;
  // source window read by this tile's outputs (bilinear neighbours included)
  int ys0, ys1, xs0, xs1, t0, t1;
  float tl;
  src_index(rs.ry, y_first, H, ys0, t1, tl);
  src_index(rs.ry, y_last, H, t0, ys1, tl);
  src_index(rs.rx, x_first, W, xs0, t1, tl);
  src_index(rs.rx, x_last, W, t0, xs1, tl);
  const int SRa = ys1 - ys0 + 1, SCa = xs1 - xs0 + 1;                    // SRa * SCa <= win_cap (tile sizes chosen by the host)
  if (SRa * SCa > win_cap) return;     // a device row steeper than the host declared: never overrun shared memory

  // ---- prototype window -> shared memory, read exactly once per CTA; per-row interpolation constants
  stage_window<PT, HWC>(protos, s_p, H, W, ys0, xs0, SRa, SCa, MF_THREADS);
  if (threadIdx.x <= y_last - y_first) {
    RowC rc;
    src_index(rs.ry, y_first + threadIdx.x, H, rc.y0, rc.y1, rc.ly);
    rc.o0 = (rc.y0 - ys0) * SCa;
    rc.o1 = (rc.y1 - ys0) * SCa;
    s_row[threadIdx.x] = rc;
  }

  // ---- per-lane column constants of phase 2 (warp -> one word column, rows strided by the warps sharing the column)
  const int wcol = warp % TW, rstep = (MF_THREADS / 32) / TW, rfirst = warp / TW;
  const int x = x_first + wcol * 32 + lane;
  int cx0, cx1;
  float lx;
  {
    int xa, xb;
    src_index(rs.rx, min(x, x_last), W, xa, xb, lx);
    cx0 = xa - xs0; cx1 = xb - xs0;
  }
  const float hx = 1.f - lx;
  const bool x_ok = x <= x_last;
  const bool word_ok = x_first + wcol * 32 <= x_last;                    // warp-uniform
  // source columns read by this warp's word (lane 0 .. last valid lane)
  const float wsrc_lo = (float)(xs0 + __shfl_sync(0xffffffffu, cx0, 0));
  const float wsrc_hi = (float)(xs0 + __shfl_sync(0xffffffffu, cx1, min(31, x_last - (x_first + wcol * 32))));
  const float win_x0 = (float)xs0, win_x1 = (float)xs1, win_y0 = (float)ys0, win_y1 = (float)ys1;

  for (int n0 = 0; n0 < N; n0 += MF_LIST) {
    const int nb = min(MF_LIST, N - n0);
    __syncthreads();                                   // window / row table staged; previous pass done with s_box, s_val
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    if (threadIdx.x < nb) {
      const float* b = boxes + (size_t)(n0 + threadIdx.x) * 4;
      BoxP bp;
      bp.x1 = b[0] * sx1; bp.y1 = b[1] * sy1; bp.x2 = b[2] * sx2; bp.y2 = b[3] * sy2;
      // some source pixel of the window lies inside the roi (x1 <= w < x2, y1 <= h < y2); otherwise every output of the
      // tile is 0 for this detection, which the memset already wrote
      if (win_x1 >= bp.x1 && win_x0 < bp.x2 && win_y1 >= bp.y1 && win_y0 < bp.y2) {
        bp.roi_w = (float)(((double)(bp.x2 - bp.x1) + 0.1) / 2);
        bp.roi_h = (float)(((double)(bp.y2 - bp.y1) + 0.1) / 2);
        bp.pad0 = bp.pad1 = 0.f;
        const int pos = atomicAdd(s_cnt, 1);
        s_box[pos] = bp;
        s_det[pos] = n0 + threadIdx.x;
      }
    }
    __syncthreads();
    const int cnt = *s_cnt;
    for (int j = 0; j < cnt; ++j) {
      const BoxP b = s_box[j];
      const int n = s_det[j];
      float* val = s_val + (j & 1) * win_cap;
      const float* cof = cofs + (size_t)n * 128;
      // ---- phase 1: one sigmoid-dot per source pixel of the window (warp = window row, lanes = columns); 0 outside the roi
      for (int r = warp; r < SRa; r += MF_THREADS / 32) {
        const float hf = (float)(ys0 + r);
        const bool row_in = (hf >= b.y1) & (hf < b.y2);
        const int idx_h = row_in ? (int)__fdiv_rn(hf - b.y1, b.roi_h) : 0;
        for (int c = lane; c < SCa; c += 32) {
          const float wf = (float)(xs0 + c);
          float v = 0.f;
          if (row_in & (wf >= b.x1) & (wf < b.x2)) {
            const int idx_w = (int)__fdiv_rn(wf - b.x1, b.roi_w);
            const int cell = min(max(idx_h * 2 + idx_w, 0), 3);
            v = sigmoidf_(dot32_swz<PT>(s_p, r * SCa + c, cof + cell * 32));
          }
          val[r * SCa + c] = v;
        }
      }
      __syncthreads();        // the only barrier per detection: s_val is double-buffered, see below
      // ---- phase 2: lane = output pixel of one word; rows of this warp's word column.  Words whose source columns, and
      // rows whose source rows, lie outside the roi are all-zero: skipped (the memset wrote them)
      if (word_ok && wsrc_hi >= b.x1 && wsrc_lo < b.x2) {
        uint32_t* o = out + (size_t)n * plane + wq_first + wcol;
        for (int y = y_first + rfirst; y <= y_last; y += rstep) {
          const RowC rc = s_row[y - y_first];
          if ((float)rc.y1 < b.y1 || (float)rc.y0 >= b.y2) continue;
          const float hy = 1.f - rc.ly;
          const float* r0 = val + rc.o0;
          const float* r1 = val + rc.o1;
          const float v = hy * (hx * r0[cx0] + lx * r0[cx1]) + rc.ly * (hx * r1[cx0] + lx * r1[cx1]);
          const uint32_t bits = __ballot_sync(0xffffffffu, x_ok && v > thr);
          if (lane == 0 && bits) o[(size_t)y * words] = bits;
        }
      }
      // no barrier here: phase 1 of detection j+1 writes the OTHER s_val buffer; buffer (j & 1) is rewritten by detection
      // j+2, whose phase 1 every warp enters only after the barrier of detection j+1, i.e. after all warps left this loop
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// Tensor-core variants of the two kernels above for fp16 prototypes (the engine's storage type).
//
// The 32-term dot products are evaluated by mma.sync.m16n8k16 (fp16 x fp16 -> fp32):
//   A  = 16 staged prototype pixels x 16 channels, read from the swizzled shared-memory window (two k-steps cover the 32
//        channels); row g / g + 8 of the fragment = pixel g / g + 8 of a 16-pixel run of one window row,
//   B  = 16 channels x 8 columns; column n = (detection slot n >> 1 of a group of FOUR listed detections, idx_w = n & 1):
//        the coefficients of CropSplit cell 2 * idx_h + idx_w, where idx_h is the half of the roi the pixel ROW lies in
//        (uniform along a row, so each B column is chosen per (detection, row) by the lanes that own it),
//   D  = for every pixel the logits of both idx_w halves of four detections; the epilogue keeps the one the pixel's own
//        cell selects, applies the sigmoid and the crop.
// The fp32 coefficients enter as fp16 hi + fp16 lo (two MMAs into one accumulator): c = hi + lo to 22 mantissa bits for
// |c| >= 0.125, below that lo is an fp16 subnormal and the error is absolute, <= 2^-25 per coefficient.  The prototypes
// are fp16 already, products and accumulation are fp32: the logit stays within 2^-21 * sum|p c| + 2^-24 * sum|p| of the
// exact dot product, the same order as the sequential-fmaf kernels (numpy model: tests/test_host_logic.py); the geometry
// (which pixels are inside, which cell) is computed exactly as before.
// Scalar kernels: ~140 instructions per in-box pixel and detection; here ~75 per 16 pixels x 4 detections.
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ uint32_t lds_u32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

__device__ __forceinline__ void mma_f16f32(float (&d)[4], const uint32_t (&a)[4], const uint32_t (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}

// A fragments (both k-steps) of window pixels p0 (fragment row g) and p0 + 8 (row g + 8).
// Register layout of m16n8k16: a0 = (row g, k 2t..2t+1), a1 = (row g+8, same k), a2 = (row g, k 2t+8..2t+9), a3 = (row g+8, ..);
// channel 16 * ks + 2t lives in 16-byte chunk 2 * ks at byte 4t, channel 16 * ks + 8 + 2t in chunk 2 * ks + 1 at byte 4t.
// `addr` = shared-window address of pixel p0 plus 4t, `sw` = swizzle key (p0 >> 1) & 3 of stage_window (chunk k sits at
// position k ^ sw; pixel p0 + 8 has the same key, 512 bytes further on).
__device__ __forceinline__ void load_a_frag(uint32_t addr, int sw, uint32_t (&a)[2][4]) {
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
    const uint32_t lo = addr + (((2 * ks) ^ sw) << 4), hi = addr + (((2 * ks + 1) ^ sw) << 4);
    a[ks][0] = lds_u32(lo);
    a[ks][1] = lds_u32(lo + 512);
    a[ks][2] = lds_u32(hi);
    a[ks][3] = lds_u32(hi + 512);
  }
}

// B fragments of column n = g: cof32 = the 32 fp32 coefficients of (detection, cell); b0 = (k 2t..2t+1, n), b1 = (k 2t+8..2t+9, n).
// hi = fp16(c), lo = fp16(c - hi).  fp16 holds |c| <= 65504 only: the MMA operands are clamped to +-65000 (no inf, so the
// other columns stay finite) and the return value flags a coefficient of this lane beyond that.  The callers send every
// pixel of such a detection to the scalar cold path, which reads the fp32 coefficients as they are: with small prototypes
// a coefficient of 1e5 gives an ordinary logit, and the clamped one would give a different mask.
__device__ __forceinline__ bool load_b_frag(const float* __restrict__ cof32, int t, bool valid, uint32_t (&bh)[2][2], uint32_t (&bl)[2][2]) {
  bool beyond = false;
#pragma unroll
  for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float2 v = make_float2(0.f, 0.f);
      if (valid) v = __ldg(reinterpret_cast<const float2*>(cof32 + ks * 16 + h * 8 + 2 * t));
      beyond |= fmaxf(fabsf(v.x), fabsf(v.y)) > 65000.f;
      v.x = fminf(fmaxf(v.x, -65000.f), 65000.f);
      v.y = fminf(fmaxf(v.y, -65000.f), 65000.f);
      const __half2 hi = __floats2half2_rn(v.x, v.y);
      const float2 hf = __half22float2(hi);
      const __half2 lo = __floats2half2_rn(v.x - hf.x, v.y - hf.y);
      bh[ks][h] = *reinterpret_cast<const uint32_t*>(&hi);
      bl[ks][h] = *reinterpret_cast<const uint32_t*>(&lo);
    }
  }
  return beyond;
}

// Detection slot t (accumulator columns 2t, 2t + 1) has a coefficient beyond the fp16 range in the B columns loaded by
// load_b_frag: those columns belong to lanes 8t .. 8t + 7 (g = 2t, 2t + 1).  All 32 lanes must call it.
__device__ __forceinline__ bool slot_beyond_fp16(bool lane_beyond, int t) {
  return ((__ballot_sync(0xffffffffu, lane_beyond) >> (8 * t)) & 0xffu) != 0u;
}

// sigmoid for the tensor-core kernels: ex2.approx + rcp.approx (4 instructions, |error| < 3e-7; the IEEE division of
// sigmoidf_ is ~12).  ex2 overflow -> rcp(inf) = 0, underflow -> rcp(1) = 1: the limits are right without special cases.
__device__ __forceinline__ float sigmoid_fast(float x) {
  float e, r;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(e) : "f"(x * -1.4426950408889634f));
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(1.0f + e));
  return r;
}

// (int)(a / b) of crop_split_cuda_kernel.cu:50-51 for a >= 0, b > 0.  IEEE division rounds to nearest; a < b implies
// a <= pred(b) and pred(b) / b <= 1 - 2^-24, which rounds below 1: the truncated quotient is >= 1 exactly when a >= b
// (and >= 2 exactly when a >= 2b, 2b being exact).  The kernels below use idx = (a >= b) inline and send a >= 2b - only
// reachable by rounding, the roi is two cells wide - to the generic path.
__device__ __forceinline__ int crop_idx(float a, float b) {
  return a >= b + b ? (int)__fdiv_rn(a, b) : (a >= b ? 1 : 0);
}

// Generic (cold, out of line) value of window pixel p at image position (wf, hf): the scalar kernel's arithmetic.
__device__ __noinline__ float pixel_value_cold(const unsigned char* s_p, int p, float wf, float hf, const BoxP* bp,
                                               const float* __restrict__ cof128) {
  const BoxP b = *bp;
  if (!((hf >= b.y1) & (hf < b.y2) & (wf >= b.x1) & (wf < b.x2))) return 0.f;
  const int cell = min(max(crop_idx(hf - b.y1, b.roi_h) * 2 + crop_idx(wf - b.x1, b.roi_w), 0), 3);
  return sigmoid_fast(dot32_swz<__half>(s_p, p, cof128 + cell * 32));
}

// Epilogue of one 16-pixel run for the detection whose accumulators this thread holds: acc[0] / acc[1] = pixel c0 (fragment
// row g), idx_w 0 / 1; acc[2] / acc[3] = pixel c0 + 8.  Straight-line and predicated; the never-in-practice cases (a
// quotient of 2) are recomputed out of line.
struct RowSel {
  bool row_in;      // row inside [y1, y2) of a valid detection
  bool rare;        // row_in and idx_h >= 2
  float x0f;        // image x of window column 0
};
__device__ __forceinline__ void run_values(const float (&acc)[4], const BoxP& b, const RowSel& rs, int c0, float& v0, float& v1,
                                           bool& rare) {
  const float roi_w2 = b.roi_w + b.roi_w;
  const float w0 = rs.x0f + (float)c0, w1 = w0 + 8.f;                 // exact: small integers
  const float a0 = w0 - b.x1, a1 = w1 - b.x1;
  const bool in0 = rs.row_in & (w0 >= b.x1) & (w0 < b.x2), in1 = rs.row_in & (w1 >= b.x1) & (w1 < b.x2);
  const float s0 = a0 >= b.roi_w ? acc[1] : acc[0], s1 = a1 >= b.roi_w ? acc[3] : acc[2];
  v0 = in0 ? sigmoid_fast(s0) : 0.f;
  v1 = in1 ? sigmoid_fast(s1) : 0.f;
  rare = rs.rare | (in0 & (a0 >= roi_w2)) | (in1 & (a1 >= roi_w2));
}

// Dense pos_masks, tensor-core dots.  Same tiling / listing / zero-fill as mask_assemble_kernel; a warp owns one tile row
// (its A fragments are re-read from shared memory per 16-pixel run and group: 8 LDS.32 against ~70 other instructions;
// keeping the row's 32 fragment registers live cost a CTA per SM).
// Tile = MA_TH rows x MA_TW pixels: a warp owns one 64-pixel segment of one tile row.
// 64 registers: four CTAs per SM (528 slots on 132 SMs for the 550 - 600 CTAs of a 400 x 672 prototype map; at three CTAs
// per SM the second wave would run on a fraction of the SMs).
template <bool HWC, typename OT>
__global__ void __launch_bounds__(MA_THREADS2, 4) mask_assemble_mma_kernel(
    const __half* __restrict__ protos, const float* __restrict__ cofs, const float* __restrict__ boxes,
    GeomArg ga, OT* __restrict__ out, int H, int W, int N) {
  static_assert(MA_TW % 64 == 0 && MA_TH * (MA_TW / 64) == MA_THREADS2 / 32, "one warp per 64-pixel row segment");
  constexpr int SEGS = MA_TW / 64;                            // 64-pixel segments (warps) per tile row
  extern __shared__ __align__(16) unsigned char s_p[];        // [MA_TH * MA_TW] swizzled pixels (32 KB)
  __shared__ BoxP s_box[MA_LIST];
  __shared__ int s_det[MA_LIST];
  __shared__ int s_cnt;
  __shared__ unsigned s_listed[MA_LIST / 32];

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const smb_img_geom_t geom = load_geom(ga);
  const float sx1 = geom.roi_scale[0], sy1 = geom.roi_scale[1], sx2 = geom.roi_scale[2], sy2 = geom.roi_scale[3];
  const int y0t = blockIdx.y * MA_TH, x0t = blockIdx.x * MA_TW;
  const int SRa = min(MA_TH, H - y0t), SCa = min(MA_TW, W - x0t);
  stage_window<__half, HWC>(protos, s_p, H, W, y0t, x0t, SRa, SCa, MA_THREADS2);
  const int wrow = warp / SEGS, wseg = (warp % SEGS) * 64;   // this warp's tile row and first tile column
  const int h = y0t + wrow;
  const bool row_ok = wrow < SRa && wseg < SCa;
  const float hf = (float)h;
  const float tile_x0 = (float)x0t, tile_x1 = (float)(x0t + SCa - 1), tile_y0 = (float)y0t, tile_y1 = (float)(y0t + SRa - 1);
  const float seg_x0 = (float)(x0t + wseg);
  // zero-fill role: thread t < 128 owns 4 pixels: row t / (MA_TW / 4), columns 4 * (t % (MA_TW / 4)) ..
  const int zr = threadIdx.x / (MA_TW / 4), zc = (threadIdx.x % (MA_TW / 4)) * 4;
  const bool z_vec = threadIdx.x < 128 && zr < SRa && zc + 3 < SCa && ((W & 3) == 0);
  const bool z_tail = threadIdx.x < 128 && zr < SRa && !z_vec && zc < SCa;
  const int MT = min(4, (SCa - wseg + 15) >> 4);            // 16-pixel runs of this warp's segment (the last one may be
                                                            // partial: its surplus rows read later pixels and are discarded)
  // fragment row g of run 0 of this warp's segment: pixel p_row (run m adds 16 pixels = 1024 bytes, same swizzle key)
  const int p_row = wrow * SCa + wseg + g;
  const uint32_t a_row = smem_addr(s_p) + (uint32_t)p_row * 64 + 4 * t;
  const int a_sw = (p_row >> 1) & 3;

  for (int n0 = 0; n0 < N; n0 += MA_LIST) {
    const int nb = min(MA_LIST, N - n0);
    __syncthreads();                                   // window staged / previous pass done with the list
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    bool mine_listed = false;
    if (threadIdx.x < nb) {
      const float* b = boxes + (size_t)(n0 + threadIdx.x) * 4;
      BoxP bp;
      bp.x1 = b[0] * sx1; bp.y1 = b[1] * sy1; bp.x2 = b[2] * sx2; bp.y2 = b[3] * sy2;
      if (tile_x1 >= bp.x1 && tile_x0 < bp.x2 && tile_y1 >= bp.y1 && tile_y0 < bp.y2) {
        bp.roi_w = (float)(((double)(bp.x2 - bp.x1) + 0.1) / 2);
        bp.roi_h = (float)(((double)(bp.y2 - bp.y1) + 0.1) / 2);
        bp.pad0 = bp.pad1 = 0.f;
        const int pos = atomicAdd(&s_cnt, 1);
        s_box[pos] = bp;
        s_det[pos] = n0 + threadIdx.x;
        mine_listed = true;
      }
    }
    {
      const unsigned bal = __ballot_sync(0xffffffffu, mine_listed);
      if (lane == 0 && warp < MA_LIST / 32) s_listed[warp] = bal;
    }
    __syncthreads();
    const int cnt = s_cnt;
    // ---- detections whose roi misses the tile: zeros (16 bytes per thread, 8 rows x 256 B per detection)
    if (z_vec | z_tail) {
      for (int j = 0; j < nb; ++j) {
        if ((s_listed[j >> 5] >> (j & 31)) & 1u) continue;
        OT* dst = out + ((size_t)(n0 + j) * H + (y0t + zr)) * W + x0t + zc;
        if (z_vec) {
          store_zero4<OT>(dst);
        } else {
          for (int e = 0; e < 4 && zc + e < SCa; ++e) store1<OT>(dst + e, 0.f);
        }
      }
    }
    if (!row_ok) continue;                               // warp-uniform
    // ---- listed detections, four at a time: every pixel of the tile row is written (value inside the roi, 0 outside)
    for (int j0 = 0; j0 < cnt; j0 += 4) {
      // B side: this lane feeds column n = g: detection slot g >> 1, idx_w = g & 1, row half of THIS row in that roi
      uint32_t bh[2][2], bl[2][2];
      bool beyond;
      {
        const int jb = j0 + (g >> 1);
        const bool vb = jb < cnt;
        const int js = vb ? jb : j0;
        const int hb = (hf - s_box[js].y1 >= s_box[js].roi_h) ? 1 : 0;          // min(idx_h, 1)
        beyond = load_b_frag(cofs + (size_t)s_det[js] * 128 + (hb * 2 + (g & 1)) * 32, t, vb, bh, bl);
      }
      beyond = slot_beyond_fp16(beyond, t);
      // C side: accumulator columns 2t, 2t+1 = detection slot t, idx_w 0 / 1
      const int jc = j0 + t;
      const bool vc = jc < cnt;
      const int js = vc ? jc : j0;
      const BoxP b = s_box[js];
      const int n = s_det[js];
      RowSel rsel;
      rsel.row_in = vc & (hf >= b.y1) & (hf < b.y2);
      rsel.rare = rsel.row_in & ((hf - b.y1 >= b.roi_h + b.roi_h) | beyond);
      rsel.x0f = seg_x0;
      OT* dst = out + ((size_t)n * H + h) * W + x0t + wseg + g;
#pragma unroll 1
      for (int m = 0; m < MT; ++m) {
        const float run_x0 = seg_x0 + (float)(m * 16), run_x1 = run_x0 + 15.f;
        const bool any_in = __any_sync(0xffffffffu, rsel.row_in & (run_x1 >= b.x1) & (run_x0 < b.x2));
        const int c0 = m * 16 + g;
        float v0 = 0.f, v1 = 0.f;
        if (any_in) {                                      // warp-uniform: the MMAs are executed by all 32 lanes
          uint32_t a[2][4];
          load_a_frag(a_row + m * 1024, a_sw, a);
          float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int ks = 0; ks < 2; ++ks) {
            mma_f16f32(acc, a[ks], bh[ks]);
            mma_f16f32(acc, a[ks], bl[ks]);
          }
          bool rare;
          run_values(acc, b, rsel, c0, v0, v1, rare);
          if (rare) {
            v0 = pixel_value_cold(s_p, p_row + m * 16, seg_x0 + (float)c0, hf, &s_box[js], cofs + (size_t)n * 128);
            v1 = pixel_value_cold(s_p, p_row + m * 16 + 8, seg_x0 + (float)(c0 + 8), hf, &s_box[js], cofs + (size_t)n * 128);
          }
        }
        if (vc) {
          if (wseg + c0 < SCa) store1<OT>(dst + m * 16, v0);
          if (wseg + c0 + 8 < SCa) store1<OT>(dst + m * 16 + 8, v1);
        }
      }
    }
  }
}

// Fused resize + threshold + bit-pack, tensor-core dots.  Same tiling / listing / phase 2 as mask_fused_pack_kernel; the
// listed detections are processed FOUR at a time: phase 1 walks (window row, 16-pixel run) units round-robin over the
// warps (the scalar kernel gave each warp whole rows: 10 rows on 8 warps, 66 columns on 32 lanes) and writes four value
// tiles, phase 2 packs them; two barriers per group of four instead of one per detection.
// 64 registers and a 64-entry list: four CTAs per SM (57 KB each), the ~550 CTAs of an 800 x 1344 canvas are one wave.
constexpr int MFM_LIST = 64;
template <bool HWC>
__global__ void __launch_bounds__(MF_THREADS, 4) mask_fused_pack_mma_kernel(
    const __half* __restrict__ protos, const float* __restrict__ cofs, const float* __restrict__ boxes, GeomArg ga,
    uint32_t* __restrict__ out, int H, int W, int N, int words, size_t plane, int TY, int TW, int win_cap, float thr) {
  extern __shared__ __align__(16) unsigned char mf_smem[];
  unsigned char* s_p = mf_smem;                                                        // [win_cap] swizzled pixels
  float* s_val = reinterpret_cast<float*>(mf_smem + (size_t)win_cap * 64);              // [4][win_cap]
  BoxP* s_box = reinterpret_cast<BoxP*>(s_val + 4 * win_cap);                          // [MFM_LIST]
  RowC* s_row = reinterpret_cast<RowC*>(s_box + MFM_LIST);                              // [MF_TY_MAX]
  int* s_det = reinterpret_cast<int*>(s_row + MF_TY_MAX);                              // [MFM_LIST]
  int* s_cnt = s_det + MFM_LIST;

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int g = lane >> 2, t = lane & 3;
  const smb_img_geom_t geom = load_geom(ga);
  const Resize rs = {geom.full_h, geom.full_w, geom.ry, geom.rx};
  const float sx1 = geom.roi_scale[0], sy1 = geom.roi_scale[1], sx2 = geom.roi_scale[2], sy2 = geom.roi_scale[3];
  const int y_first = blockIdx.y * TY, wq_first = blockIdx.x * TW;
  const int vh = min(geom.out_h, rs.full_h), vw = min(geom.out_w, rs.full_w);
  const int y_last = min(y_first + TY, vh) - 1;
  const int x_first = wq_first * 32, x_last = min(x_first + TW * 32, vw) - 1;
  if (y_last < y_first || x_last < x_first) return;
  int ys0, ys1, xs0, xs1, t0, t1;
  float tl;
  src_index(rs.ry, y_first, H, ys0, t1, tl);
  src_index(rs.ry, y_last, H, t0, ys1, tl);
  src_index(rs.rx, x_first, W, xs0, t1, tl);
  src_index(rs.rx, x_last, W, t0, xs1, tl);
  const int SRa = ys1 - ys0 + 1, SCa = xs1 - xs0 + 1;
  if (SRa * SCa > win_cap) return;     // a device row steeper than the host declared: never overrun shared memory
  const int MT = (SCa + 15) >> 4, n_units = SRa * MT;       // (window row, 16-pixel run) units; a partial last run reads
                                                            // the next row's (or the value tiles') bytes and discards them

  stage_window<__half, HWC>(protos, s_p, H, W, ys0, xs0, SRa, SCa, MF_THREADS);
  if (threadIdx.x <= y_last - y_first) {
    RowC rc;
    src_index(rs.ry, y_first + threadIdx.x, H, rc.y0, rc.y1, rc.ly);
    rc.o0 = (rc.y0 - ys0) * SCa;
    rc.o1 = (rc.y1 - ys0) * SCa;
    s_row[threadIdx.x] = rc;
  }

  const int wcol = warp % TW, rstep = (MF_THREADS / 32) / TW, rfirst = warp / TW;
  const int x = x_first + wcol * 32 + lane;
  int cx0, cx1;
  float lx;
  {
    int xa, xb;
    src_index(rs.rx, min(x, x_last), W, xa, xb, lx);
    cx0 = xa - xs0; cx1 = xb - xs0;
  }
  const float hx = 1.f - lx;
  const bool x_ok = x <= x_last;
  const bool word_ok = x_first + wcol * 32 <= x_last;
  const float wsrc_lo = (float)(xs0 + __shfl_sync(0xffffffffu, cx0, 0));
  const float wsrc_hi = (float)(xs0 + __shfl_sync(0xffffffffu, cx1, min(31, x_last - (x_first + wcol * 32))));
  const float win_x0 = (float)xs0, win_x1 = (float)xs1, win_y0 = (float)ys0, win_y1 = (float)ys1;
  const uint32_t sp_addr = smem_addr(s_p) + 4 * t;
  // first unit of this warp (units advance by the warp count)
  const int u_r0 = warp / MT, u_m0 = warp - u_r0 * MT;
  const int u_dr = (MF_THREADS / 32) / MT, u_dm = (MF_THREADS / 32) - u_dr * MT;

  for (int n0 = 0; n0 < N; n0 += MFM_LIST) {
    const int nb = min(MFM_LIST, N - n0);
    __syncthreads();                                   // window / row table staged; previous pass done with s_box, s_val
    if (threadIdx.x == 0) *s_cnt = 0;
    __syncthreads();
    if (threadIdx.x < nb) {
      const float* b = boxes + (size_t)(n0 + threadIdx.x) * 4;
      BoxP bp;
      bp.x1 = b[0] * sx1; bp.y1 = b[1] * sy1; bp.x2 = b[2] * sx2; bp.y2 = b[3] * sy2;
      if (win_x1 >= bp.x1 && win_x0 < bp.x2 && win_y1 >= bp.y1 && win_y0 < bp.y2) {
        bp.roi_w = (float)(((double)(bp.x2 - bp.x1) + 0.1) / 2);
        bp.roi_h = (float)(((double)(bp.y2 - bp.y1) + 0.1) / 2);
        bp.pad0 = bp.pad1 = 0.f;
        const int pos = atomicAdd(s_cnt, 1);
        s_box[pos] = bp;
        s_det[pos] = n0 + threadIdx.x;
      }
    }
    __syncthreads();
    const int cnt = *s_cnt;
    for (int j0 = 0; j0 < cnt; j0 += 4) {
      const int nd = min(4, cnt - j0);
      // ---- phase 1: value tiles of detections j0 .. j0 + nd - 1 (0 outside the roi)
      {
        // B side: column n = g -> detection slot g >> 1, idx_w = g & 1; both row halves, selected per unit
        uint32_t bh0[2][2], bl0[2][2], bh1[2][2], bl1[2][2];
        const int jb = j0 + (g >> 1);
        const bool vb = jb < cnt;
        const int jsb = vb ? jb : j0;
        const float bb_y1 = s_box[jsb].y1, bb_roi_h = s_box[jsb].roi_h;
        bool beyond;
        {
          const float* cb = cofs + (size_t)s_det[jsb] * 128 + (g & 1) * 32;
          beyond = load_b_frag(cb, t, vb, bh0, bl0);
          beyond |= load_b_frag(cb + 64, t, vb, bh1, bl1);
        }
        beyond = slot_beyond_fp16(beyond, t);
        // C side: detection slot t
        const int jc = j0 + t;
        const bool vc = jc < cnt;
        const int jsc = vc ? jc : j0;
        const BoxP b = s_box[jsc];
        const float roi_h2 = b.roi_h + b.roi_h;
        float* val = s_val + t * win_cap;
        int r = u_r0, m = u_m0;
        for (int u = warp; u < n_units; u += MF_THREADS / 32) {
          const float hf = win_y0 + (float)r;
          RowSel rsel;
          rsel.row_in = vc & (hf >= b.y1) & (hf < b.y2);
          rsel.rare = rsel.row_in & ((hf - b.y1 >= roi_h2) | beyond);
          rsel.x0f = win_x0;
          const float run_x0 = win_x0 + (float)(m * 16), run_x1 = run_x0 + 15.f;
          const bool any_in = __any_sync(0xffffffffu, rsel.row_in & (run_x1 >= b.x1) & (run_x0 < b.x2));
          const int c0 = m * 16 + g;
          const int p0 = r * SCa + c0;
          float v0 = 0.f, v1 = 0.f;
          if (any_in) {                                    // warp-uniform
            const bool hb = (hf - bb_y1) >= bb_roi_h;      // row half of this row in the roi of the B-side detection
            uint32_t a[2][4], bh[2][2], bl[2][2];
            load_a_frag(sp_addr + (uint32_t)p0 * 64, (p0 >> 1) & 3, a);
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
#pragma unroll
              for (int q = 0; q < 2; ++q) {
                bh[ks][q] = hb ? bh1[ks][q] : bh0[ks][q];
                bl[ks][q] = hb ? bl1[ks][q] : bl0[ks][q];
              }
            }
            float acc[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int ks = 0; ks < 2; ++ks) {
              mma_f16f32(acc, a[ks], bh[ks]);
              mma_f16f32(acc, a[ks], bl[ks]);
            }
            bool rare;
            run_values(acc, b, rsel, c0, v0, v1, rare);
            if (rare) {
              const float* cof128 = cofs + (size_t)s_det[jsc] * 128;
              v0 = pixel_value_cold(s_p, p0, win_x0 + (float)c0, hf, &s_box[jsc], cof128);
              v1 = pixel_value_cold(s_p, p0 + 8, win_x0 + (float)(c0 + 8), hf, &s_box[jsc], cof128);
            }
          }
          if (vc) {
            if (c0 < SCa) val[p0] = v0;
            if (c0 + 8 < SCa) val[p0 + 8] = v1;
          }
          r += u_dr; m += u_dm;
          if (m >= MT) { m -= MT; ++r; }
        }
      }
      __syncthreads();
      // ---- phase 2: lane = output pixel of one word; rows of this warp's word column (as in the scalar kernel)
      for (int d = 0; d < nd; ++d) {
        const BoxP b = s_box[j0 + d];
        if (word_ok && wsrc_hi >= b.x1 && wsrc_lo < b.x2) {
          const float* val = s_val + d * win_cap;
          uint32_t* o = out + (size_t)s_det[j0 + d] * plane + wq_first + wcol;
          for (int y = y_first + rfirst; y <= y_last; y += rstep) {
            const RowC rc = s_row[y - y_first];
            if ((float)rc.y1 < b.y1 || (float)rc.y0 >= b.y2) continue;
            const float hy = 1.f - rc.ly;
            const float* r0 = val + rc.o0;
            const float* r1 = val + rc.o1;
            const float v = hy * (hx * r0[cx0] + lx * r0[cx1]) + rc.ly * (hx * r1[cx0] + lx * r1[cx1]);
            const uint32_t bits = __ballot_sync(0xffffffffu, x_ok && v > thr);
            if (lane == 0 && bits) o[(size_t)y * words] = bits;
          }
        }
      }
      __syncthreads();                                   // the next group's phase 1 overwrites the value tiles
    }
  }
}

// CropSplit operator (ops/crop/src/crop_split_cuda_kernel.cu:19-59), c == 2.
template <typename T>
__global__ void crop_split_kernel(const T* __restrict__ data, const T* __restrict__ rois, T* __restrict__ out,
                                  long long count, int H, int W, int N) {
  for (long long index = blockIdx.x * (long long)blockDim.x + threadIdx.x; index < count;
       index += (long long)blockDim.x * gridDim.x) {
    const int n = (int)(index % N);
    const int pw = (int)((index / N) % W);
    const int ph = (int)(index / N / W);
    const float x1 = to_f<T>(rois[n * 4 + 0]), y1 = to_f<T>(rois[n * 4 + 1]);
    const float x2 = to_f<T>(rois[n * 4 + 2]), y2 = to_f<T>(rois[n * 4 + 3]);
    T v = T(0.f);
    if (((float)pw >= x1) & ((float)ph >= y1) & ((float)pw < x2) & ((float)ph < y2)) {
      const float roi_w = (float)(((double)(x2 - x1) + 0.1) / 2);
      const float roi_h = (float)(((double)(y2 - y1) + 0.1) / 2);
      const int idx_w = (int)__fdiv_rn((float)pw - x1, roi_w);
      const int idx_h = (int)__fdiv_rn((float)ph - y1, roi_h);
      const int cell = min(max(idx_h * 2 + idx_w, 0), 3);
      v = data[(long long)cell * count + index];
    }
    out[index] = v;
  }
}

// CropSplit backward (crop_split_cuda_kernel.cu:90-127): grad_in[cell(h,w,n), h, w, n] = grad_out[h,w,n] inside the roi, 0
// everywhere else.  Every (cell, index) target is written exactly once, so no atomics and no zero-init are needed.
template <typename T>
__global__ void crop_split_backward_kernel(const T* __restrict__ top, const T* __restrict__ rois, T* __restrict__ bottom,
                                           long long count, int H, int W, int N) {
  for (long long index = blockIdx.x * (long long)blockDim.x + threadIdx.x; index < count;
       index += (long long)blockDim.x * gridDim.x) {
    const int n = (int)(index % N);
    const int pw = (int)((index / N) % W);
    const int ph = (int)(index / N / W);
    const float x1 = to_f<T>(rois[n * 4 + 0]), y1 = to_f<T>(rois[n * 4 + 1]);
    const float x2 = to_f<T>(rois[n * 4 + 2]), y2 = to_f<T>(rois[n * 4 + 3]);
    int cell = -1;
    if (((float)pw >= x1) & ((float)ph >= y1) & ((float)pw < x2) & ((float)ph < y2)) {
      const float roi_w = (float)(((double)(x2 - x1) + 0.1) / 2);
      const float roi_h = (float)(((double)(y2 - y1) + 0.1) / 2);
      cell = min(max((int)__fdiv_rn((float)ph - y1, roi_h) * 2 + (int)__fdiv_rn((float)pw - x1, roi_w), 0), 3);
    }
    const T g = top[index];
#pragma unroll
    for (int k = 0; k < 4; ++k) bottom[(long long)k * count + index] = (k == cell) ? g : T(0.f);
  }
}

// CropSplitGt forward and backward (crop_split_gt_cuda_kernel.cu:19-49,76-104): out = data inside the roi, 0 outside.
template <typename T>
__global__ void crop_mask_kernel(const T* __restrict__ data, const T* __restrict__ rois, T* __restrict__ out, long long count,
                                 int H, int W, int N) {
  for (long long index = blockIdx.x * (long long)blockDim.x + threadIdx.x; index < count;
       index += (long long)blockDim.x * gridDim.x) {
    const int n = (int)(index % N);
    const int pw = (int)((index / N) % W);
    const int ph = (int)(index / N / W);
    const float x1 = to_f<T>(rois[n * 4 + 0]), y1 = to_f<T>(rois[n * 4 + 1]);
    const float x2 = to_f<T>(rois[n * 4 + 2]), y2 = to_f<T>(rois[n * 4 + 3]);
    const bool in = ((float)pw >= x1) & ((float)ph >= y1) & ((float)pw < x2) & ((float)ph < y2);
    out[index] = in ? data[index] : T(0.f);
  }
}

}  // namespace smb

using namespace smb;

// fp16 prototypes: tensor-core kernels (1, default) or the scalar-fmaf kernels (0)
static int g_mask_mma = 1;

extern "C" int smb_mask_set_tensor_dot(int on) {
  const int prev = g_mask_mma;
  if (on >= 0) g_mask_mma = on ? 1 : 0;
  return prev;
}

static int mask_assemble(const void* protos, int protos_dtype, int layout_hwc, const float* cofs, const float* boxes,
                         GeomArg ga, void* out, int out_dtype, int H, int W, int N, smb_stream_t stream) {
  SMB_CHECK_ARG(protos && cofs && boxes && out, "smb_mask_assemble: null pointer");
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0, "smb_mask_assemble: bad shape H=%d W=%d N=%d", H, W, N);
  SMB_CHECK_ARG((protos_dtype == SMB_F32 || protos_dtype == SMB_F16) && (out_dtype == SMB_F32 || out_dtype == SMB_F16),
                "smb_mask_assemble: bad dtype");
  if (N == 0) return SMB_OK;
  dim3 grid(cdiv(W, MA_TW), cdiv(H, MA_TH)), block(MA_THREADS2);
  cudaStream_t st = (cudaStream_t)stream;
  const size_t ma_smem = (size_t)MA_TH * MA_TW * (protos_dtype == SMB_F16 ? 64 : 128);
  static DeviceOnce ma_once;
  if (ma_once.first()) {
#define MA_ATTR(PT, HWC, OT) \
  SMB_CUDA_OK(cudaFuncSetAttribute(mask_assemble_kernel<PT, HWC, OT>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024))
    MA_ATTR(float, false, float); MA_ATTR(float, false, __half); MA_ATTR(float, true, float); MA_ATTR(float, true, __half);
    MA_ATTR(__half, false, float); MA_ATTR(__half, false, __half); MA_ATTR(__half, true, float); MA_ATTR(__half, true, __half);
#undef MA_ATTR
  }
#define MA_LAUNCH(PT, HWC, OT)                                                                                   \
  mask_assemble_kernel<PT, HWC, OT><<<grid, block, ma_smem, st>>>((const PT*)protos, cofs, boxes, ga, (OT*)out, \
                                                                  H, W, N)
  const int key = (protos_dtype << 2) | ((layout_hwc ? 1 : 0) << 1) | out_dtype;
  if (protos_dtype == SMB_F16 && g_mask_mma) {
#define MAM_LAUNCH(HWC, OT)                                                                                      \
  mask_assemble_mma_kernel<HWC, OT><<<grid, block, ma_smem, st>>>((const __half*)protos, cofs, boxes, ga,   \
                                                                  (OT*)out, H, W, N)
    switch (key & 3) {
      case 0: MAM_LAUNCH(false, float); break;
      case 1: MAM_LAUNCH(false, __half); break;
      case 2: MAM_LAUNCH(true, float); break;
      case 3: MAM_LAUNCH(true, __half); break;
    }
#undef MAM_LAUNCH
    SMB_LAUNCH_OK("mask_assemble_mma_kernel");
    return SMB_OK;
  }
  switch (key) {
    case 0: MA_LAUNCH(float, false, float); break;
    case 1: MA_LAUNCH(float, false, __half); break;
    case 2: MA_LAUNCH(float, true, float); break;
    case 3: MA_LAUNCH(float, true, __half); break;
    case 4: MA_LAUNCH(__half, false, float); break;
    case 5: MA_LAUNCH(__half, false, __half); break;
    case 6: MA_LAUNCH(__half, true, float); break;
    case 7: MA_LAUNCH(__half, true, __half); break;
  }
#undef MA_LAUNCH
  SMB_LAUNCH_OK("mask_assemble_kernel");
  return SMB_OK;
}

extern "C" int smb_mask_assemble(const void* protos, int protos_dtype, int layout_hwc, const float* cofs,
                                 const float* boxes, const float* host_box_scale4, void* out, int out_dtype,
                                 int H, int W, int N, smb_stream_t stream) {
  SMB_CHECK_ARG(host_box_scale4, "smb_mask_assemble: null pointer");
  smb_img_geom_t g;
  memset(&g, 0, sizeof(g));
  for (int k = 0; k < 4; ++k) g.roi_scale[k] = host_box_scale4[k];
  return mask_assemble(protos, protos_dtype, layout_hwc, cofs, boxes, geom_value(g), out, out_dtype, H, W, N, stream);
}

extern "C" int smb_mask_assemble_dev(const void* protos, int protos_dtype, int layout_hwc, const float* cofs,
                                     const float* boxes, const smb_img_geom_t* geom, void* out, int out_dtype,
                                     int H, int W, int N, smb_stream_t stream) {
  SMB_CHECK_ARG(geom, "smb_mask_assemble_dev: null geometry");
  return mask_assemble(protos, protos_dtype, layout_hwc, cofs, boxes, geom_device(geom), out, out_dtype, H, W, N, stream);
}

static int make_resize(int H, int W, int full_h, int full_w, float ry, float rx, Resize* rs, const char* who) {
  if (full_h <= 0 || full_w <= 0) { set_error("%s: interpolated size %dx%d must be positive", who, full_h, full_w); return SMB_EINVAL; }
  rs->full_h = full_h; rs->full_w = full_w;
  // source step per output pixel: the caller's 1/scale_factor (PyTorch >= 1.6 with scale_factor given), or in/out when the
  // caller passes <= 0 (recompute_scale_factor=True, the only behaviour of PyTorch <= 1.5)
  rs->ry = ry > 0.f ? ry : (float)H / (float)full_h;
  rs->rx = rx > 0.f ? rx : (float)W / (float)full_w;
  return SMB_OK;
}

extern "C" int smb_mask_resize_threshold(const void* pos, int pos_dtype, uint8_t* out_u8, int N, int H, int W, int full_h,
                                         int full_w, float ry, float rx, int out_h, int out_w, float thr, smb_stream_t stream) {
  SMB_CHECK_ARG(pos && out_u8, "smb_mask_resize_threshold: null pointer");
  SMB_CHECK_ARG(N >= 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0 && out_h <= 65535 && N <= 65535,
                "smb_mask_resize_threshold: bad shape");
  Resize rs;
  const int rc = make_resize(H, W, full_h, full_w, ry, rx, &rs, "smb_mask_resize_threshold");
  if (rc) return rc;
  if (N == 0) return SMB_OK;
  dim3 block(256), grid(cdiv(cdiv(out_w, 4), 256), out_h, N);
  cudaStream_t st = (cudaStream_t)stream;
  if (pos_dtype == SMB_F32)
    resize_thresh_kernel<float><<<grid, block, 0, st>>>((const float*)pos, out_u8, N, H, W, out_h, out_w, rs, thr);
  else
    resize_thresh_kernel<__half><<<grid, block, 0, st>>>((const __half*)pos, out_u8, N, H, W, out_h, out_w, rs, thr);
  SMB_LAUNCH_OK("resize_thresh_kernel");
  return SMB_OK;
}

extern "C" int smb_mask_resize_threshold_pack(const void* pos, int pos_dtype, uint32_t* out_bits, int N, int H, int W,
                                              int full_h, int full_w, float ry, float rx, int out_h, int out_w, float thr,
                                              smb_stream_t stream) {
  SMB_CHECK_ARG(pos && out_bits, "smb_mask_resize_threshold_pack: null pointer");
  SMB_CHECK_ARG(N >= 0 && H > 0 && W > 0 && out_h > 0 && out_w > 0 && out_h <= 65535 && N <= 65535,
                "smb_mask_resize_threshold_pack: bad shape");
  Resize rs;
  const int rc = make_resize(H, W, full_h, full_w, ry, rx, &rs, "smb_mask_resize_threshold_pack");
  if (rc) return rc;
  if (N == 0) return SMB_OK;
  const int words = cdiv(out_w, 32);
  dim3 block(256), grid(cdiv(words, 8), out_h, N);
  cudaStream_t st = (cudaStream_t)stream;
  if (pos_dtype == SMB_F32)
    resize_thresh_pack_kernel<float><<<grid, block, 0, st>>>((const float*)pos, out_bits, N, H, W, out_h, out_w, words, rs, thr);
  else
    resize_thresh_pack_kernel<__half><<<grid, block, 0, st>>>((const __half*)pos, out_bits, N, H, W, out_h, out_w, words, rs, thr);
  SMB_LAUNCH_OK("resize_thresh_pack_kernel");
  return SMB_OK;
}

extern "C" int smb_mask_upsample2_threshold(const void* pos, int pos_dtype, uint8_t* out_u8, int N, int H, int W,
                                            int out_h, int out_w, float thr, smb_stream_t stream) {
  return smb_mask_resize_threshold(pos, pos_dtype, out_u8, N, H, W, 2 * H, 2 * W, 0.5f, 0.5f, out_h, out_w, thr, stream);
}

extern "C" int smb_mask_upsample2_threshold_pack(const void* pos, int pos_dtype, uint32_t* out_bits, int N, int H, int W,
                                                 int out_h, int out_w, float thr, smb_stream_t stream) {
  return smb_mask_resize_threshold_pack(pos, pos_dtype, out_bits, N, H, W, 2 * H, 2 * W, 0.5f, 0.5f, out_h, out_w, thr, stream);
}

// The fused mask launch.  (tile_ry, tile_rx) size the tile (the steepest resize the geometry can hold), (grid_h, grid_w) the
// grid (the valid output frame, or the record's capacity when the geometry is a device row); the bit planes are
// [N, plane_h, words].
static int mask_assemble_pack(const void* protos, int protos_dtype, int layout_hwc, const float* cofs, const float* boxes,
                              GeomArg ga, float tile_ry, float tile_rx, uint32_t* out_bits, int H, int W, int N, int plane_h,
                              int words, int grid_h, int grid_w, float thr, smb_stream_t stream) {
  if (N == 0) return SMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t plane = (size_t)plane_h * words;
  SMB_CUDA_OK(cudaMemsetAsync(out_bits, 0, (size_t)N * plane * 4, st));      // zero background (memset node)
  // output tile (TY rows x TW words) whose source window fits the shared-memory caps: rows/cols <= ceil((n-1) * r) + 2
  // window budget in source pixels: ~48 KB of prototypes per CTA (4 CTAs / SM), e.g. 16 rows x 4 words at x2 = 10 x 66 px
  const size_t px_bytes = protos_dtype == SMB_F16 ? 64 : 128;
  const int px_budget = (int)((48 * 1024) / px_bytes);
  auto win_rows = [&](int ty) { return (int)ceilf((float)(ty - 1) * tile_ry) + 2; };
  auto win_cols = [&](int tw) { return (int)ceilf((float)(tw * 32 - 1) * tile_rx) + 2; };
  int TW = 4, TY = MF_TY_MAX;
  while (TW > 1 && win_rows(TY) * win_cols(TW) > px_budget) TW >>= 1;
  while (TY > 1 && win_rows(TY) * win_cols(TW) > px_budget) TY >>= 1;
  // rounded up to a multiple of 4 pixels: the arrays carved out of shared memory after the window (s_val, s_box, ...) are
  // read with 16-byte vector loads
  const int win_cap = (win_rows(TY) * win_cols(TW) + 3) & ~3;
  SMB_CHECK_ARG(win_cap <= px_budget + 3, "smb_mask_assemble_pack: resize %dx%d -> %dx%d shrinks too much for one tile (%d source "
                "pixels per 32-pixel word)", H, W, ga.v.full_h, ga.v.full_w, win_cap);
  dim3 grid(cdiv(cdiv(grid_w, 32), TW), cdiv(grid_h, TY)), block(MF_THREADS);
  const bool mma = protos_dtype == SMB_F16 && g_mask_mma;
  // value tiles: two (double-buffered, one detection each) for the scalar kernel, four (a group of detections) for the
  // tensor-core kernel
  const size_t smem = (size_t)win_cap * (px_bytes + (mma ? 16 : 8)) + (mma ? MFM_LIST : MF_LIST) * (sizeof(BoxP) + sizeof(int)) +
                      MF_TY_MAX * sizeof(RowC) + 16;
  static DeviceOnce attr_once;
  if (attr_once.first()) {
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_kernel<float, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_kernel<float, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_kernel<__half, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_kernel<__half, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 * 1024));
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_mma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024));
    SMB_CUDA_OK(cudaFuncSetAttribute(mask_fused_pack_mma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 72 * 1024));
  }
  if (mma) {
#define MFM_LAUNCH(HWC)                                                                                                  \
  mask_fused_pack_mma_kernel<HWC><<<grid, block, smem, st>>>((const __half*)protos, cofs, boxes, ga, out_bits, H, W, N, words, \
                                                             plane, TY, TW, win_cap, thr)
    if (layout_hwc) MFM_LAUNCH(true); else MFM_LAUNCH(false);
#undef MFM_LAUNCH
    SMB_LAUNCH_OK("mask_fused_pack_mma_kernel");
    return SMB_OK;
  }
#define MF_LAUNCH(PT, HWC)                                                                                          \
  mask_fused_pack_kernel<PT, HWC><<<grid, block, smem, st>>>((const PT*)protos, cofs, boxes, ga, out_bits, H, W, N, words, \
                                                           plane, TY, TW, win_cap, thr)
  if (protos_dtype == SMB_F16) {
    if (layout_hwc) MF_LAUNCH(__half, true); else MF_LAUNCH(__half, false);
  } else {
    if (layout_hwc) MF_LAUNCH(float, true); else MF_LAUNCH(float, false);
  }
#undef MF_LAUNCH
  SMB_LAUNCH_OK("mask_fused_pack_kernel");
  return SMB_OK;
}

extern "C" int smb_mask_assemble_pack(const void* protos, int protos_dtype, int layout_hwc, const float* cofs,
                                      const float* boxes, const float* host_box_scale4, uint32_t* out_bits, int H, int W, int N,
                                      int full_h, int full_w, float ry, float rx, int out_h, int out_w, float thr,
                                      smb_stream_t stream) {
  SMB_CHECK_ARG(protos && cofs && boxes && out_bits && host_box_scale4, "smb_mask_assemble_pack: null pointer");
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0 && out_h > 0 && out_w > 0, "smb_mask_assemble_pack: bad shape");
  SMB_CHECK_ARG(protos_dtype == SMB_F32 || protos_dtype == SMB_F16, "smb_mask_assemble_pack: bad dtype");
  Resize rs;
  const int rc = make_resize(H, W, full_h, full_w, ry, rx, &rs, "smb_mask_assemble_pack");
  if (rc) return rc;
  smb_img_geom_t g;
  memset(&g, 0, sizeof(g));
  for (int k = 0; k < 4; ++k) g.roi_scale[k] = host_box_scale4[k];
  g.full_h = rs.full_h; g.full_w = rs.full_w; g.ry = rs.ry; g.rx = rs.rx;
  g.out_h = out_h; g.out_w = out_w;
  const int vh = out_h < full_h ? out_h : full_h, vw = out_w < full_w ? out_w : full_w;
  return mask_assemble_pack(protos, protos_dtype, layout_hwc, cofs, boxes, geom_value(g), rs.ry, rs.rx, out_bits, H, W, N,
                            out_h, cdiv(out_w, 32), vh, vw, thr, stream);
}

extern "C" int smb_mask_assemble_pack_dev(const void* protos, int protos_dtype, int layout_hwc, const float* cofs,
                                          const float* boxes, const smb_img_geom_t* geom, float max_ry, float max_rx,
                                          uint32_t* out_bits, int H, int W, int N, int cap_h, int cap_w, float thr,
                                          smb_stream_t stream) {
  SMB_CHECK_ARG(protos && cofs && boxes && out_bits && geom, "smb_mask_assemble_pack_dev: null pointer");
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0 && cap_h > 0 && cap_w > 0, "smb_mask_assemble_pack_dev: bad shape");
  SMB_CHECK_ARG(protos_dtype == SMB_F32 || protos_dtype == SMB_F16, "smb_mask_assemble_pack_dev: bad dtype");
  SMB_CHECK_ARG(max_ry > 0.f && max_rx > 0.f, "smb_mask_assemble_pack_dev: max_ry=%g max_rx=%g must be positive", max_ry, max_rx);
  return mask_assemble_pack(protos, protos_dtype, layout_hwc, cofs, boxes, geom_device(geom), max_ry, max_rx, out_bits, H, W,
                            N, cap_h, cdiv(cap_w, 32), cap_h, cap_w, thr, stream);
}

extern "C" int smb_crop_split_forward(const void* data, const void* rois, void* out, int dtype, int H, int W, int c,
                                      int N, smb_stream_t stream) {
  SMB_CHECK_ARG(data && rois && out, "smb_crop_split_forward: null pointer");
  SMB_CHECK_ARG(c == 2, "smb_crop_split_forward: only c == 2 is used by SipMask (got %d)", c);
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0, "smb_crop_split_forward: bad shape");
  const long long count = (long long)H * W * N;
  if (count == 0) return SMB_OK;
  const int blocks = (int)min((long long)132 * 16, (count + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SMB_F32)
    crop_split_kernel<float><<<blocks, 256, 0, st>>>((const float*)data, (const float*)rois, (float*)out, count, H, W, N);
  else if (dtype == SMB_F16)
    crop_split_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)data, (const __half*)rois, (__half*)out, count, H, W, N);
  else
    SMB_CHECK_ARG(false, "smb_crop_split_forward: bad dtype %d", dtype);
  SMB_LAUNCH_OK("crop_split_kernel");
  return SMB_OK;
}

extern "C" int smb_crop_split_backward(const void* top_grad, const void* rois, void* bottom_grad, int dtype, int H, int W, int c,
                                       int N, smb_stream_t stream) {
  SMB_CHECK_ARG(top_grad && rois && bottom_grad, "smb_crop_split_backward: null pointer");
  SMB_CHECK_ARG(c == 2, "smb_crop_split_backward: only c == 2 is used by SipMask (got %d)", c);
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0, "smb_crop_split_backward: bad shape");
  const long long count = (long long)H * W * N;
  if (count == 0) return SMB_OK;
  const int blocks = (int)min((long long)132 * 16, (count + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SMB_F32)
    crop_split_backward_kernel<float><<<blocks, 256, 0, st>>>((const float*)top_grad, (const float*)rois, (float*)bottom_grad, count, H, W, N);
  else if (dtype == SMB_F16)
    crop_split_backward_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)top_grad, (const __half*)rois, (__half*)bottom_grad, count, H, W, N);
  else
    SMB_CHECK_ARG(false, "smb_crop_split_backward: bad dtype %d", dtype);
  SMB_LAUNCH_OK("crop_split_backward_kernel");
  return SMB_OK;
}

extern "C" int smb_crop_split_gt(const void* data, const void* rois, void* out, int dtype, int H, int W, int N,
                                 smb_stream_t stream) {
  SMB_CHECK_ARG(data && rois && out, "smb_crop_split_gt: null pointer");
  SMB_CHECK_ARG(H > 0 && W > 0 && N >= 0, "smb_crop_split_gt: bad shape");
  const long long count = (long long)H * W * N;
  if (count == 0) return SMB_OK;
  const int blocks = (int)min((long long)132 * 16, (count + 255) / 256);
  cudaStream_t st = (cudaStream_t)stream;
  if (dtype == SMB_F32)
    crop_mask_kernel<float><<<blocks, 256, 0, st>>>((const float*)data, (const float*)rois, (float*)out, count, H, W, N);
  else if (dtype == SMB_F16)
    crop_mask_kernel<__half><<<blocks, 256, 0, st>>>((const __half*)data, (const __half*)rois, (__half*)out, count, H, W, N);
  else
    SMB_CHECK_ARG(false, "smb_crop_split_gt: bad dtype %d", dtype);
  SMB_LAUNCH_OK("crop_mask_kernel");
  return SMB_OK;
}
