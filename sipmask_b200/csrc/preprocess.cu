// Test-time image pipeline on the device (SURVEY.md 8f-3): uint8 BGR HWC image -> keep-ratio bilinear resize ->
// mean subtraction -> zero pad -> the stem's space-to-depth fp16 layout, in one kernel.
//
// Reference: Resize(keep_ratio) / Normalize(std=1, to_rgb=False) / Pad(32) / ImageToTensor on the host CPU
// (SipMask-mmdetection/mmdet/datasets/pipelines/transforms.py:97-110, 274-300, 335-363), i.e. mmcv -> cv2.resize(INTER_LINEAR),
// followed by a 12.9 MB fp32 upload.  Here the upload is the raw uint8 image (<= 4 MB) and the arithmetic is OpenCV's
// 8-bit fixed-point bilinear restated exactly (11-bit coefficients, int32 horizontal pass, the two truncating shifts of
// the vertical pass), so the stem sees bit-identical input.  SipMask-benchmark checkpoints get their own kernel below
// (PIL bilinear on an RGB source).
#include <stdint.h>

#include <cuda_fp16.h>

#include "common.cuh"

namespace smb {

__device__ __forceinline__ uint4 pack8h(const float* f) {
  uint4 o;
  __half2* h = reinterpret_cast<__half2*>(&o);
#pragma unroll
  for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
  return o;
}

struct Coef {
  int s0, s1, a0, a1;
};

// OpenCV resize.cpp (INTER_LINEAR, 8U): fx = (float)((d + 0.5) * scale - 0.5); s = floor(fx); fx -= s; the x direction
// clamps the coefficient at the borders, the y direction only clamps the row index.
__device__ __forceinline__ Coef coef(int d, double scale, int sn, bool clamp_coef) {
  float f = (float)(((double)d + 0.5) * scale - 0.5);
  int s = (int)floorf(f);
  f = __fsub_rn(f, (float)s);
  if (clamp_coef) {
    if (s < 0) { f = 0.f; s = 0; }
    if (s >= sn - 1) { f = 0.f; s = sn - 1; }
  }
  Coef c;
  c.a1 = __float2int_rn(__fmul_rn(f, 2048.f));
  c.a0 = __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f));
  c.s0 = min(max(s, 0), sn - 1);
  c.s1 = min(max(s + 1, 0), sn - 1);
  return c;
}

// One resized + mean-subtracted pixel (x, y) of the dw x dh image, or zeros outside it (halo / padding).
struct PreArgs {
  const uint8_t* src;
  int sh, sw, pitch, dh, dw;
  double scale_y, scale_x;
  float m0, m1, m2;
};
// The per-pixel arguments of one source row.  A filler row (dst_h == 0 or dst_w == 0) gets dh = dw = 0: every pixel is
// outside the image, so nothing is read and its canvas is all zero.
__device__ __forceinline__ PreArgs pre_args(const smb_raw_src_t& r) {
  PreArgs a;
  const bool fill = r.dst_h <= 0 || r.dst_w <= 0;
  a.src = r.src; a.sh = r.src_h; a.sw = r.src_w; a.pitch = r.src_pitch_bytes;
  a.dh = fill ? 0 : r.dst_h; a.dw = fill ? 0 : r.dst_w;
  a.scale_y = fill ? 1.0 : 1.0 / ((double)r.dst_h / r.src_h);
  a.scale_x = fill ? 1.0 : 1.0 / ((double)r.dst_w / r.src_w);
  a.m0 = r.mean[0]; a.m1 = r.mean[1]; a.m2 = r.mean[2];
  return a;
}
__device__ __forceinline__ void pre_pixel(const PreArgs& a, int x, int y, float* f3) {
  f3[0] = f3[1] = f3[2] = 0.f;
  if (x >= 0 && x < a.dw && y >= 0 && y < a.dh) {
    int v[3];
    if (a.sh == a.dh && a.sw == a.dw) {                  // cv2.resize copies when the size does not change
      const uint8_t* p = a.src + (size_t)y * a.pitch + x * 3;
      v[0] = p[0]; v[1] = p[1]; v[2] = p[2];
    } else {
      const Coef cx = coef(x, a.scale_x, a.sw, true), cy = coef(y, a.scale_y, a.sh, false);
      const uint8_t* r0 = a.src + (size_t)cy.s0 * a.pitch;
      const uint8_t* r1 = a.src + (size_t)cy.s1 * a.pitch;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const int h0 = (int)r0[cx.s0 * 3 + c] * cx.a0 + (int)r0[cx.s1 * 3 + c] * cx.a1;
        const int h1 = (int)r1[cx.s0 * 3 + c] * cx.a0 + (int)r1[cx.s1 * 3 + c] * cx.a1;
        v[c] = (((cy.a0 * (h0 >> 4)) >> 16) + ((cy.a1 * (h1 >> 4)) >> 16) + 2) >> 2;
      }
    }
    f3[0] = __fsub_rn((float)v[0], a.m0);
    f3[1] = __fsub_rn((float)v[1], a.m1);
    f3[2] = __fsub_rn((float)v[2], a.m2);
  }
}

// Space-to-depth layout of the 7x7/2 stem: out [N, H/2+3, W/2+4, 16] fp16, element (n, Y, X, (dy*2+dx)*4 + c) = padded
// pixel (2Y+dy, 2X+dx) = pixel (2Y+dy-3, 2X+dx-3) of image n, channel c (c == 3: zero).  store_cell writes cell number
// `cell` (= (n * (H/2+3) + Y) * (W/2+4) + X) from its 16 floats f[(dy*2+dx)*4 + c] as two 16-byte stores.
__device__ __forceinline__ void store_cell(__half* __restrict__ out, long long cell, const float* f) {
  uint4* o = reinterpret_cast<uint4*>(out + cell * 16);
  o[0] = pack8h(f);
  o[1] = pack8h(f + 8);
}

// One thread = one 32-byte (n, Y, X) cell; image n's source row is rows[n] (device memory, rewritten between graph
// replays) or, with rows == nullptr (N == 1), row0 by value.  Write indices come from the canvas alone, so no row can make
// a thread write outside image n's canvas; reads stay inside the row's source image because pre_pixel clamps every source
// row / column index.
__global__ void preprocess_u8_s2d_kernel(const smb_raw_src_t* __restrict__ rows, smb_raw_src_t row0,
                                         __half* __restrict__ out, int N, int H, int W) {
  const int Hq = H / 2 + 3, Wq = W / 2 + 4;
  const long long cells = (long long)Hq * Wq, total = cells * N;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)blockDim.x * gridDim.x) {
    const int n = (int)(t / cells);
    const long long c = t - n * cells;
    const int X = (int)(c % Wq), Y = (int)(c / Wq);
    const PreArgs a = rows ? pre_args(rows[n]) : pre_args(row0);
    float f[16];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      pre_pixel(a, 2 * X + (d & 1) - 3, 2 * Y + (d >> 1) - 3, f + 4 * d);
      f[4 * d + 3] = 0.f;
    }
    store_cell(out, t, f);
  }
}

// ------------------------------------------------------------------------------------------------------------------------
// SipMask-benchmark's test transform (SipMask-benchmark/fcos_core/data/transforms/build.py:17-36, transforms.py:27-95):
// PIL RGB image -> torchvision F.resize = PIL Image.resize(BILINEAR) -> to_tensor -> to_bgr255 -> normalize(std = 1) ->
// zero pad to 32.  fl(fl(v / 255) * 255) == v for every uint8 v, so the network input is exactly float(v) - mean on the
// BGR channel, which this kernel computes from the RGB source.
//
// Pillow's resize (libImaging/Resample.c) is separable and antialiased, in 22-bit fixed point: per output index xx of an
// in -> out axis, scale = in / out, fs = max(scale, 1) (= the bilinear support), center = (xx + 0.5) * scale, taps
// [xmin, xmin + n) with xmin = max((int)(center - fs + 0.5), 0), xmin + n = min((int)(center + fs + 0.5), in), weights
// tri(((x + xmin) - center + 0.5) * (1 / fs)) summed in order in double, divided by the sum and stored as
// (int)(0.5 + k * 2^22).  The first pass clips to uint8; each pass is clamp((2^21 + sum v * k) >> 22, 0, 255).  The
// horizontal pass runs first, except where Image.resize runs the vertical one first: for an image more than 100 times
// taller than wide whose height shrinks.  The order changes the bits, because the intermediate image is clipped.  An axis
// whose size does not change gets the taps {2^22, 0}, which copy it exactly (Pillow skips that pass).
// Every double operation is an explicit _rn intrinsic: the reference (x86-64 Pillow) does not contract to FMA, nvcc would.
constexpr int PIL_TY = 8, PIL_TX = 32;                        // cells per CTA: 8 x 32 -> 16 output rows x 64 columns
constexpr int PIL_OY = 2 * PIL_TY, PIL_OX = 2 * PIL_TX;
constexpr int PIL_MAX_SCALE = 8;                              // steepest downscale per axis (validated by the host)
constexpr int PIL_KMAX = 2 * PIL_MAX_SCALE + 1;               // taps per output index at that scale (< 2 * fs + 1)
constexpr int PIL_RMAX = (PIL_OY - 1) * PIL_MAX_SCALE + PIL_KMAX;   // source rows the 16 output rows of a tile read
constexpr int PIL_CMAX = (PIL_OX - 1) * PIL_MAX_SCALE + PIL_KMAX;   // source columns the 64 output columns of a tile read
// The tile's intermediate image: horizontal pass first, PIL_RMAX source rows x PIL_OX output columns; vertical pass first,
// PIL_OY output rows x PIL_CMAX source columns.  One buffer holds either.
constexpr int PIL_HPASS_BYTES = PIL_RMAX * PIL_OX * 3, PIL_VPASS_BYTES = PIL_OY * PIL_CMAX * 3;
constexpr int PIL_PASS_BYTES = PIL_HPASS_BYTES > PIL_VPASS_BYTES ? PIL_HPASS_BYTES : PIL_VPASS_BYTES;

// Taps of output index xx of an in -> out axis: first source index, count, fixed-point weights.
__device__ void pil_taps(int xx, int in, int out, int* lo, int* cnt, int* w) {
  const double scale = __ddiv_rn((double)in, (double)out);
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn((double)xx, 0.5), scale);
  int xmin = __double2int_rz(__dadd_rn(__dsub_rn(center, fs), 0.5));
  int xmax = __double2int_rz(__dadd_rn(__dadd_rn(center, fs), 0.5));
  xmin = max(xmin, 0);
  xmax = min(min(xmax, in) - xmin, PIL_KMAX);
  double ww = 0.0;
  for (int x = 0; x < xmax; ++x) {
    const double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
    ww = __dadd_rn(ww, t < 1.0 ? __dsub_rn(1.0, t) : 0.0);
  }
  for (int x = 0; x < xmax; ++x) {                            // the same weights again, normalised
    const double t = fabs(__dmul_rn(__dadd_rn(__dsub_rn((double)(x + xmin), center), 0.5), ss));
    double k = t < 1.0 ? __dsub_rn(1.0, t) : 0.0;
    if (ww != 0.0) k = __ddiv_rn(k, ww);
    w[x] = __double2int_rz(__dadd_rn(0.5, __dmul_rn(k, 4194304.0)));
  }
  *lo = xmin;
  *cnt = xmax;
}

__device__ __forceinline__ int pil_clip8(int v) { return min(max(v >> 22, 0), 255); }

// One CTA = a tile of PIL_TY x PIL_TX cells of canvas blockIdx.z.  It computes the taps of the tile's output columns and
// rows once, runs the first pass into shared memory (uint8, as Pillow's intermediate image), then each thread runs the
// second pass for its cell's four pixels and writes the cell.  Horizontal first: the first pass covers the source rows
// the tile's output rows need, at its output columns.  Vertical first: it covers the tile's output rows, at the source
// columns its output columns need.  The order is a property of the canvas's row, so it is uniform over the CTA.  Write
// indices come from the canvas alone; source indices are clamped inside the row's image and shared-memory indices inside
// the tile's buffer, so an unvalidated row cannot make the kernel touch memory outside them.
struct PilSmem {
  int cx_lo[PIL_OX], cx_n[PIL_OX], cx_w[PIL_OX][PIL_KMAX];
  int cy_lo[PIL_OY], cy_n[PIL_OY], cy_w[PIL_OY][PIL_KMAX];
  uint8_t pass[PIL_PASS_BYTES];
};

// The tile with the passes in one order, compiled once per order so that neither pays for the other's branches.
template <bool VFIRST>
__device__ __forceinline__ void pil_tile(PilSmem& s, const smb_raw_src_t& r, int dh, int dw, __half* __restrict__ out,
                                         int H, int W) {
  auto& cx_lo = s.cx_lo; auto& cx_n = s.cx_n; auto& cx_w = s.cx_w;
  auto& cy_lo = s.cy_lo; auto& cy_n = s.cy_n; auto& cy_w = s.cy_w;
  uint8_t(*hpass)[PIL_OX * 3] = reinterpret_cast<uint8_t(*)[PIL_OX * 3]>(s.pass);       // [PIL_RMAX][PIL_OX * 3]
  uint8_t(*vpass)[PIL_CMAX * 3] = reinterpret_cast<uint8_t(*)[PIL_CMAX * 3]>(s.pass);   // [PIL_OY][PIL_CMAX * 3]
  const int Hq = H / 2 + 3, Wq = W / 2 + 4;
  const int n = blockIdx.z, Y0 = blockIdx.y * PIL_TY, X0 = blockIdx.x * PIL_TX, t = threadIdx.x;
  const int py0 = 2 * Y0 - 3, px0 = 2 * X0 - 3;               // output pixel of the tile's local (0, 0)
  // the tile's output pixels inside the resized image (everything else is halo / padding: zero)
  const int ya = max(py0, 0), yb = min(py0 + PIL_OY, dh), xa = max(px0, 0), xb = min(px0 + PIL_OX, dw);
  const bool any = ya < yb && xa < xb;                        // uniform over the CTA
  int ybase = 0, xbase = 0;
  if (any) {
    if (t < PIL_OX) {
      const int x = px0 + t;
      if (x >= xa && x < xb) pil_taps(x, r.src_w, dw, &cx_lo[t], &cx_n[t], cx_w[t]);
    } else if (t < PIL_OX + PIL_OY) {
      const int ly = t - PIL_OX, y = py0 + ly;
      if (y >= ya && y < yb) pil_taps(y, r.src_h, dh, &cy_lo[ly], &cy_n[ly], cy_w[ly]);
    }
    __syncthreads();
    if constexpr (!VFIRST) {                                  // horizontal pass over source rows [ybase, ybase + nrows)
      ybase = cy_lo[ya - py0];
      const int nrows = min(cy_lo[yb - 1 - py0] + cy_n[yb - 1 - py0] - ybase, PIL_RMAX);
      const int nx = xb - xa, lx0 = xa - px0;
      for (int i = t; i < nrows * nx; i += PIL_TY * PIL_TX) {
        const int rr = i / nx, lx = lx0 + i % nx;
        const uint8_t* p = r.src + (size_t)min(ybase + rr, r.src_h - 1) * r.src_pitch_bytes;
        const int lo = cx_lo[lx], cnt = cx_n[lx];
        int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
        for (int k = 0; k < cnt; ++k) {
          const uint8_t* q = p + 3 * min(lo + k, r.src_w - 1);
          const int w = cx_w[lx][k];
          a0 += (int)q[0] * w;
          a1 += (int)q[1] * w;
          a2 += (int)q[2] * w;
        }
        hpass[rr][lx * 3 + 0] = (uint8_t)pil_clip8(a0);
        hpass[rr][lx * 3 + 1] = (uint8_t)pil_clip8(a1);
        hpass[rr][lx * 3 + 2] = (uint8_t)pil_clip8(a2);
      }
    } else {                                                  // vertical pass over source columns [xbase, xbase + ncols)
      xbase = cx_lo[xa - px0];
      const int ncols = min(cx_lo[xb - 1 - px0] + cx_n[xb - 1 - px0] - xbase, PIL_CMAX);
      const int ny = yb - ya, ly0 = ya - py0;
      for (int i = t; i < ny * ncols; i += PIL_TY * PIL_TX) {
        const int ly = ly0 + i / ncols, cc = i % ncols;
        const uint8_t* p = r.src + 3 * min(xbase + cc, r.src_w - 1);
        const int lo = cy_lo[ly], cnt = cy_n[ly];
        int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
        for (int k = 0; k < cnt; ++k) {
          const uint8_t* q = p + (size_t)min(lo + k, r.src_h - 1) * r.src_pitch_bytes;
          const int w = cy_w[ly][k];
          a0 += (int)q[0] * w;
          a1 += (int)q[1] * w;
          a2 += (int)q[2] * w;
        }
        vpass[ly][cc * 3 + 0] = (uint8_t)pil_clip8(a0);
        vpass[ly][cc * 3 + 1] = (uint8_t)pil_clip8(a1);
        vpass[ly][cc * 3 + 2] = (uint8_t)pil_clip8(a2);
      }
    }
    __syncthreads();
  }
  const int ty = t / PIL_TX, tx = t % PIL_TX, Y = Y0 + ty, X = X0 + tx;
  if (Y >= Hq || X >= Wq) return;
  float f[16];
#pragma unroll
  for (int d = 0; d < 4; ++d) {
    const int ly = 2 * ty + (d >> 1), lx = 2 * tx + (d & 1), y = py0 + ly, x = px0 + lx;
    f[4 * d + 0] = f[4 * d + 1] = f[4 * d + 2] = f[4 * d + 3] = 0.f;
    if (any && y >= ya && y < yb && x >= xa && x < xb) {
      int a0 = 1 << 21, a1 = 1 << 21, a2 = 1 << 21;
      if constexpr (!VFIRST) {                                // vertical pass over the tile's rows of hpass
        const int lo = cy_lo[ly] - ybase, cnt = cy_n[ly];
        for (int k = 0; k < cnt; ++k) {
          const uint8_t* q = &hpass[min(lo + k, PIL_RMAX - 1)][lx * 3];
          const int w = cy_w[ly][k];
          a0 += (int)q[0] * w;
          a1 += (int)q[1] * w;
          a2 += (int)q[2] * w;
        }
      } else {                                                // horizontal pass along the output row ly of vpass
        const int lo = cx_lo[lx] - xbase, cnt = cx_n[lx];
        for (int k = 0; k < cnt; ++k) {
          const uint8_t* q = &vpass[ly][3 * min(lo + k, PIL_CMAX - 1)];
          const int w = cx_w[lx][k];
          a0 += (int)q[0] * w;
          a1 += (int)q[1] * w;
          a2 += (int)q[2] * w;
        }
      }
      // RGB source -> BGR network input
      f[4 * d + 0] = __fsub_rn((float)pil_clip8(a2), r.mean[0]);
      f[4 * d + 1] = __fsub_rn((float)pil_clip8(a1), r.mean[1]);
      f[4 * d + 2] = __fsub_rn((float)pil_clip8(a0), r.mean[2]);
    }
  }
  store_cell(out, ((long long)n * Hq + Y) * Wq + X, f);
}

__global__ void __launch_bounds__(PIL_TY * PIL_TX) preprocess_pil_u8_s2d_kernel(const smb_raw_src_t* __restrict__ rows,
                                                                               __half* __restrict__ out, int H, int W) {
  __shared__ PilSmem s;
  const smb_raw_src_t r = rows[blockIdx.z];
  const bool fill = r.dst_h <= 0 || r.dst_w <= 0;
  const int dh = fill ? 0 : r.dst_h, dw = fill ? 0 : r.dst_w;
  // Image.resize's order (PIL/Image.py): vertical first when the image is more than 100 times taller than wide and its
  // height shrinks.  64-bit: 100 * src_w overflows an int for widths a row admits.
  if ((long long)r.src_h > 100LL * r.src_w && dh < r.src_h)
    pil_tile<true>(s, r, dh, dw, out, H, W);
  else
    pil_tile<false>(s, r, dh, dw, out, H, W);
}

static int launch_preprocess(const smb_raw_src_t* rows, const smb_raw_src_t& row0, void* out, int N, int H, int W,
                             smb_stream_t stream) {
  const long long total = (long long)N * (H / 2 + 3) * (W / 2 + 4);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  preprocess_u8_s2d_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(rows, row0, (__half*)out, N, H, W);
  SMB_LAUNCH_OK("preprocess_u8_s2d_kernel");
  return SMB_OK;
}

}  // namespace smb

using namespace smb;

extern "C" int smb_preprocess_u8_s2d(const uint8_t* src, int src_h, int src_w, int src_pitch_bytes, int dst_h, int dst_w,
                                     const float* host_mean3, void* out, int H, int W, smb_stream_t stream) {
  SMB_CHECK_ARG(src && host_mean3 && out, "smb_preprocess_u8_s2d: null pointer");
  SMB_CHECK_ARG(src_h > 0 && src_w > 0 && src_pitch_bytes >= 3 * src_w && dst_h > 0 && dst_w > 0 && dst_h <= H && dst_w <= W,
                "smb_preprocess_u8_s2d: bad shape (src %dx%d -> %dx%d inside %dx%d)", src_h, src_w, dst_h, dst_w, H, W);
  SMB_CHECK_ARG(H % 2 == 0 && W % 2 == 0, "smb_preprocess_u8_s2d: H, W must be even");
  smb_raw_src_t r;
  r.src = src; r.src_h = src_h; r.src_w = src_w; r.src_pitch_bytes = src_pitch_bytes; r.dst_h = dst_h; r.dst_w = dst_w;
  r.mean[0] = host_mean3[0]; r.mean[1] = host_mean3[1]; r.mean[2] = host_mean3[2];
  return launch_preprocess(nullptr, r, out, 1, H, W, stream);
}

extern "C" int smb_preprocess_u8_s2d_dev(const smb_raw_src_t* rows, int N, void* out, int H, int W, smb_stream_t stream) {
  SMB_CHECK_ARG(rows && out, "smb_preprocess_u8_s2d_dev: null pointer");
  SMB_CHECK_ARG(N > 0 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                "smb_preprocess_u8_s2d_dev: bad canvas (N %d, %dx%d; H, W must be even)", N, H, W);
  smb_raw_src_t r;
  memset(&r, 0, sizeof(r));
  return launch_preprocess(rows, r, out, N, H, W, stream);
}

extern "C" int smb_preprocess_pil_u8_s2d_dev(const smb_raw_src_t* rows, int N, void* out, int H, int W,
                                             smb_stream_t stream) {
  SMB_CHECK_ARG(rows && out, "smb_preprocess_pil_u8_s2d_dev: null pointer");
  SMB_CHECK_ARG(N > 0 && N <= 65535 && H > 0 && W > 0 && H % 2 == 0 && W % 2 == 0,
                "smb_preprocess_pil_u8_s2d_dev: bad canvas (N %d, %dx%d; H, W must be even)", N, H, W);
  const dim3 grid(cdiv(W / 2 + 4, PIL_TX), cdiv(H / 2 + 3, PIL_TY), N);
  preprocess_pil_u8_s2d_kernel<<<grid, PIL_TY * PIL_TX, 0, (cudaStream_t)stream>>>(rows, (__half*)out, H, W);
  SMB_LAUNCH_OK("preprocess_pil_u8_s2d_kernel");
  return SMB_OK;
}
