// Test-time image pipeline on the device (SURVEY.md 8f-3): uint8 BGR HWC image -> keep-ratio bilinear resize ->
// mean subtraction -> zero pad -> the stem's NHWC8 fp16 layout, in one kernel.
//
// Reference: Resize(keep_ratio) / Normalize(std=1, to_rgb=False) / Pad(32) / ImageToTensor on the host CPU
// (SipMask-mmdetection/mmdet/datasets/pipelines/transforms.py:97-110, 274-300, 335-363), i.e. mmcv -> cv2.resize(INTER_LINEAR),
// followed by a 12.9 MB fp32 upload.  Here the upload is the raw uint8 image (<= 4 MB) and the arithmetic is OpenCV's
// 8-bit fixed-point bilinear restated exactly (11-bit coefficients, int32 horizontal pass, the two truncating shifts of
// the vertical pass), so the stem sees bit-identical input.
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

// out [H+6, W+8, 8] fp16: pixel (y, x) at (y+3, x+3); zeros in the halo, the padding and channels 3..7
__global__ void preprocess_u8_kernel(PreArgs a, __half* __restrict__ out, int H, int W) {
  const int Hp = H + 6, Wp = W + 8;
  const long long total = (long long)Hp * Wp;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)blockDim.x * gridDim.x) {
    const int xp = (int)(t % Wp), yp = (int)(t / Wp);
    float f[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    pre_pixel(a, xp - 3, yp - 3, f);
    *reinterpret_cast<uint4*>(out + t * 8) = pack8h(f);
  }
}

// Space-to-depth layout of the 7x7/2 stem: out [H/2+3, W/2+4, 16] fp16, element (Y, X, (dy*2+dx)*4 + c) = padded pixel
// (2Y+dy, 2X+dx) = image pixel (2Y+dy-3, 2X+dx-3), channel c (c == 3: zero).  One thread = one 32-byte (Y, X) cell.
__global__ void preprocess_u8_s2d_kernel(PreArgs a, __half* __restrict__ out, int H, int W) {
  const int Hq = H / 2 + 3, Wq = W / 2 + 4;
  const long long total = (long long)Hq * Wq;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)blockDim.x * gridDim.x) {
    const int X = (int)(t % Wq), Y = (int)(t / Wq);
    float f[16];
#pragma unroll
    for (int d = 0; d < 4; ++d) {
      pre_pixel(a, 2 * X + (d & 1) - 3, 2 * Y + (d >> 1) - 3, f + 4 * d);
      f[4 * d + 3] = 0.f;
    }
    uint4* o = reinterpret_cast<uint4*>(out + t * 16);
    o[0] = pack8h(f);
    o[1] = pack8h(f + 8);
  }
}

}  // namespace smb

using namespace smb;

static int preprocess_impl(const uint8_t* src, int src_h, int src_w, int src_pitch_bytes, int dst_h, int dst_w,
                           const float* host_mean3, void* out, int H, int W, int s2d, smb_stream_t stream) {
  SMB_CHECK_ARG(src && host_mean3 && out, "smb_preprocess_u8: null pointer");
  SMB_CHECK_ARG(src_h > 0 && src_w > 0 && src_pitch_bytes >= 3 * src_w && dst_h > 0 && dst_w > 0 && dst_h <= H && dst_w <= W,
                "smb_preprocess_u8: bad shape (src %dx%d -> %dx%d inside %dx%d)", src_h, src_w, dst_h, dst_w, H, W);
  SMB_CHECK_ARG(!s2d || (H % 2 == 0 && W % 2 == 0), "smb_preprocess_u8_s2d: H, W must be even");
  PreArgs a;
  a.src = src; a.sh = src_h; a.sw = src_w; a.pitch = src_pitch_bytes; a.dh = dst_h; a.dw = dst_w;
  a.scale_y = 1.0 / ((double)dst_h / src_h); a.scale_x = 1.0 / ((double)dst_w / src_w);
  a.m0 = host_mean3[0]; a.m1 = host_mean3[1]; a.m2 = host_mean3[2];
  const long long total = s2d ? (long long)(H / 2 + 3) * (W / 2 + 4) : (long long)(H + 6) * (W + 8);
  int blocks = (int)((total + 255) / 256);
  if (blocks > 132 * 16) blocks = 132 * 16;
  if (s2d) preprocess_u8_s2d_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a, (__half*)out, H, W);
  else preprocess_u8_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(a, (__half*)out, H, W);
  SMB_LAUNCH_OK("preprocess_u8_kernel");
  return SMB_OK;
}

extern "C" int smb_preprocess_u8(const uint8_t* src, int src_h, int src_w, int src_pitch_bytes, int dst_h, int dst_w,
                                 const float* host_mean3, void* out_nhwc8, int H, int W, smb_stream_t stream) {
  return preprocess_impl(src, src_h, src_w, src_pitch_bytes, dst_h, dst_w, host_mean3, out_nhwc8, H, W, 0, stream);
}

extern "C" int smb_preprocess_u8_s2d(const uint8_t* src, int src_h, int src_w, int src_pitch_bytes, int dst_h, int dst_w,
                                     const float* host_mean3, void* out_s2d16, int H, int W, smb_stream_t stream) {
  return preprocess_impl(src, src_h, src_w, src_pitch_bytes, dst_h, dst_w, host_mean3, out_s2d16, H, W, 1, stream);
}
