// Training-side operators for sm_90a: the DeformConv backward and the sigmoid focal loss.
//
// Reference (SipMask-mmdetection/mmdet/, identical in SipMask-VIS):
//   ops/dcn/src/deform_conv_cuda.cpp:262-470          deform_conv_backward_input_cuda / _parameters_cuda
//   ops/dcn/src/deform_conv_cuda_kernel.cu:117-188    get_gradient_weight / get_coordinate_weight
//   ops/dcn/src/deform_conv_cuda_kernel.cu:279-465    deformable_col2im / deformable_col2im_coord
//   ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu:23-100   SigmoidFocalLossForward / Backward
//
// The DeformConv backward of y[p, co] = sum_k col[p, k] W[co, k] (k = tap * C + c, col from smb_deform_im2col):
//   1. smb_deform_grad_scale: g16 = s * grad_out as fp16 NHWC, s a power of two chosen on the device from amax |grad_out|
//      (detection gradients sit far below fp16's normal range; s makes them representable, and dividing by s is exact);
//   2. grad_col[p, k] = g16[p, :] . W[:, k] through the convolution GEMM (a 1x1 ConvPlan over Cout input channels);
//   3. smb_deform_col2im: grad_offset (fixed-order reductions) and grad_input (atomics), both divided by s;
//   4. smb_deform_weight_grad: dW[co, k] = sum_p g16[p, co] col[p, k] / s, split over pixels, reduced in a fixed order.
#include <cooperative_groups.h>
#include <float.h>

#include "common.cuh"
#include "sm90.cuh"

namespace smb {

// ------------------------------------------------------------------------------------------- gradient scaling
// The scale puts amax |grad_out| into [2^14, 2^15): fp16 keeps 2^-14 relative to that as normal numbers and cannot
// overflow.  amax = 0 or a non-finite amax gives s = 1 (non-finite values stay non-finite).  The exponent is clamped so
// that s and 1/s are normal fp32 numbers.
__device__ __forceinline__ void scale_from_amax_bits(unsigned bits, float* scale) {
  int k = 0;
  if (bits != 0u && bits < 0x7f800000u) {
    const int e = (int)(bits >> 23) - 127;         // subnormal amax: e = -127, clamped below
    k = min(max(14 - e, -126), 126);
  }
  scale[0] = __int_as_float((k + 127) << 23);
  scale[1] = __int_as_float((127 - k) << 23);
}

// Cooperative grid: each block writes the largest |grad_out| bit pattern it saw (for non-negative floats the unsigned
// order is the float order, and NaN sorts above inf), the grid synchronises, every block derives s from all of them, and
// then writes g16[n, hw, c] = s * g[n, c, hw] (8 channels per thread: reads coalesced along hw, one 16-byte store).
__global__ void __launch_bounds__(256) grad_scale_kernel(const float* __restrict__ g, int n_img, int C, int HW,
                                                         __half* __restrict__ out, float* __restrict__ scale,
                                                         unsigned* __restrict__ block_max) {
  namespace cg = cooperative_groups;
  __shared__ unsigned s_max;
  __shared__ float s_scale[2];
  if (threadIdx.x == 0) s_max = 0u;
  __syncthreads();
  const size_t total = (size_t)n_img * C * HW;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  unsigned m = 0u;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += stride)
    m = max(m, __float_as_uint(g[i]) & 0x7fffffffu);
  atomicMax(&s_max, m);
  __syncthreads();
  if (threadIdx.x == 0) block_max[blockIdx.x] = s_max;
  cg::this_grid().sync();
  if (threadIdx.x == 0) {
    unsigned a = 0u;
    for (int b = 0; b < (int)gridDim.x; ++b) a = max(a, block_max[b]);
    scale_from_amax_bits(a, s_scale);
    if (blockIdx.x == 0) { scale[0] = s_scale[0]; scale[1] = s_scale[1]; }
  }
  __syncthreads();
  const float s = s_scale[0];
  const int vecs = C >> 3;
  const size_t P = (size_t)n_img * HW;
  for (size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x; t < P * vecs; t += stride) {
    const size_t pix = t % P;
    const int v = (int)(t / P);
    const size_t img = pix / HW, hw = pix % HW;
    const float* src = g + (img * C + (size_t)v * 8) * HW + hw;
    __align__(16) __half2 h[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = __floats2half2_rn(src[(2 * i) * HW] * s, src[(2 * i + 1) * HW] * s);
    *reinterpret_cast<uint4*>(out + pix * C + (size_t)v * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

// ------------------------------------------------------------------------------------------- col2im (fused)
constexpr int kCol2imWarps = 8;
constexpr int kCol2imMaxC = 1024;

__device__ __forceinline__ void load_h8(const __half* p, float* f) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const __half2* h = reinterpret_cast<const __half2*>(&u);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 t = __half22float2(h[i]);
    f[2 * i] = t.x;
    f[2 * i + 1] = t.y;
  }
}

__device__ __forceinline__ void atomic_add8(float* dst, const float* v) {
  atomicAdd(reinterpret_cast<float4*>(dst), make_float4(v[0], v[1], v[2], v[3]));
  atomicAdd(reinterpret_cast<float4*>(dst + 4), make_float4(v[4], v[5], v[6], v[7]));
}

// One warp per (pixel, tap), lanes over 8-channel vectors, as smb_deform_im2col.  The sample point and its four corners
// follow deform_conv_cuda_kernel.cu:313-331 and 421-426: nothing outside (-1, H) x (-1, W); a corner contributes when it
// lies inside the map and less than one pixel from the sample (so the far corners of an integer position do not).
//   grad_offset[pix, g*18 + 2*tap + d] = sum over the group's channels, in channel order, of
//       get_coordinate_weight(d) * grad_col  (kernel.cu:145-188; per-vector sums in shared memory, then one lane per group)
//   grad_input[img, corner, c] += get_gradient_weight(corner) * grad_col   (kernel.cu:117-143, float4 atomics)
// grad_col holds s * the gradient; both outputs are multiplied by 1/s (exact: a power of two).
__global__ void __launch_bounds__(32 * kCol2imWarps) deform_col2im_kernel(
    const float* __restrict__ gcol, const __half* __restrict__ x, const float* __restrict__ off, int off_pitch,
    const float* __restrict__ scale, float* __restrict__ grad_in, float* __restrict__ grad_off, int n_img, int H, int W,
    int C, int dg) {
  __shared__ float2 part[kCol2imWarps][kCol2imMaxC / 8];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long long total = (long long)n_img * H * W * 9;
  const int vecs = C >> 3, cpg = C / dg, vpg = cpg >> 3;
  const float inv = scale[1];
  for (long long wq = (long long)blockIdx.x * kCol2imWarps + wib; wq < total; wq += (long long)gridDim.x * kCol2imWarps) {
    const int tap = (int)(wq % 9);
    const long long pix = wq / 9;
    const int w_ = (int)(pix % W);
    const int h_ = (int)((pix / W) % H);
    const int img = (int)(pix / ((long long)W * H));
    const int i = tap / 3, j = tap - i * 3;
    const __half* xim = x + (size_t)img * H * W * C;
    float* gim = grad_in ? grad_in + (size_t)img * H * W * C : nullptr;
    for (int v = lane; v < vecs; v += 32) {
      const int g = v / vpg;
      const float* o = off + pix * off_pitch + g * 18 + 2 * tap;
      const float h_im = (float)(h_ - 1 + i) + o[0];
      const float w_im = (float)(w_ - 1 + j) + o[1];
      float ph = 0.f, pw = 0.f;
      if (h_im > -1.f && w_im > -1.f && h_im < (float)H && w_im < (float)W) {
        const int h_low = (int)floorf(h_im), w_low = (int)floorf(w_im);
        const int h_high = h_low + 1, w_high = w_low + 1;
        const float lh = h_im - (float)h_low, lw = w_im - (float)w_low;
        const float hh = 1.f - lh, hw = 1.f - lw;   // == (h_low + 1 - h_im), (w_low + 1 - w_im) bit for bit
        const bool ok1 = h_low >= 0 && w_low >= 0, ok2 = h_low >= 0 && w_high <= W - 1;
        const bool ok3 = h_high <= H - 1 && w_low >= 0, ok4 = h_high <= H - 1 && w_high <= W - 1;
        float gc[8];
        const float4* gp = reinterpret_cast<const float4*>(gcol + pix * 9 * C + (size_t)tap * C + v * 8);
        const float4 g0 = __ldg(gp), g1 = __ldg(gp + 1);
        gc[0] = g0.x; gc[1] = g0.y; gc[2] = g0.z; gc[3] = g0.w; gc[4] = g1.x; gc[5] = g1.y; gc[6] = g1.z; gc[7] = g1.w;
        if (grad_off) {
          float v1[8], v2[8], v3[8], v4[8];
#pragma unroll
          for (int e = 0; e < 8; ++e) v1[e] = v2[e] = v3[e] = v4[e] = 0.f;
          if (ok1) load_h8(xim + ((size_t)h_low * W + w_low) * C + v * 8, v1);
          if (ok2) load_h8(xim + ((size_t)h_low * W + w_high) * C + v * 8, v2);
          if (ok3) load_h8(xim + ((size_t)h_high * W + w_low) * C + v * 8, v3);
          if (ok4) load_h8(xim + ((size_t)h_high * W + w_high) * C + v * 8, v4);
#pragma unroll
          for (int e = 0; e < 8; ++e) {
            const float wh = -hw * v1[e] - lw * v2[e] + hw * v3[e] + lw * v4[e];   // bp_dir 0, kernel.cu:164-174
            const float ww = -hh * v1[e] + hh * v2[e] - lh * v3[e] + lh * v4[e];   // bp_dir 1, kernel.cu:175-185
            ph += wh * gc[e];
            pw += ww * gc[e];
          }
        }
        if (gim) {
          float t[8];
          const bool far_h = lh > 0.f, far_w = lw > 0.f;   // |h_im - h_high| < 1 (kernel.cu:325-326)
#define SMB_SCATTER(ok, wgt, hc, wc)                                                   \
  if (ok) {                                                                            \
    for (int e = 0; e < 8; ++e) t[e] = ((wgt) * gc[e]) * inv;                          \
    atomic_add8(gim + ((size_t)(hc) * W + (wc)) * C + v * 8, t);                       \
  }
          SMB_SCATTER(ok1, hh * hw, h_low, w_low)
          SMB_SCATTER(ok2 && far_w, hh * lw, h_low, w_high)
          SMB_SCATTER(ok3 && far_h, lh * hw, h_high, w_low)
          SMB_SCATTER(ok4 && far_h && far_w, lh * lw, h_high, w_high)
#undef SMB_SCATTER
        }
      }
      part[wib][v] = make_float2(ph, pw);
    }
    __syncwarp();
    if (grad_off) {
      for (int g = lane; g < dg; g += 32) {
        float sh = 0.f, sw = 0.f;
        for (int v = g * vpg; v < (g + 1) * vpg; ++v) { sh += part[wib][v].x; sw += part[wib][v].y; }
        float* go = grad_off + pix * (dg * 18) + g * 18 + 2 * tap;
        go[0] = sh * inv;
        go[1] = sw * inv;
      }
    }
    __syncwarp();
  }
}

// ------------------------------------------------------------------------------------------- weight gradient (wgmma)
// dW[co, k] = sum_p g16[p, co] col[p, k]: M = Cout, N = 9C, K = pixels.  Both operands are pixel-major, so a TMA box
// {64 (co or k), 64 pixels} lands as 64 rows of 128 bytes, one row per pixel: the MN-major 128-byte-swizzle wgmma layout
// (8 pixel rows per 1024-byte atom).  A CTA computes a 128 x 128 tile over one split of the pixels; the producer warp
// streams 32 KB stages, two consumer warpgroups issue m64n128k16 with both operands transposed.  Each split writes its
// fp32 tile to its own slice of the workspace; deform_wgrad_reduce sums the slices in split order and divides by s.
constexpr int kWgTile = 128;
constexpr int kWgKb = 64;                                 // pixels per stage
constexpr int kWgBox = 64 * kWgKb * 2;                    // one {64, 64} fp16 box, 8 KB
constexpr int kWgStageBytes = 4 * kWgBox;                 // A: two boxes (co), B: two boxes (k)
constexpr int kWgStages = 6;
constexpr int kWgThreads = 384;                           // consumer warpgroups 0, 1; warp 8 produces
constexpr size_t kWgSmem = (size_t)kWgStages * kWgStageBytes + 2 * kWgStages * 8 + 1024;
constexpr int kWgTargetCtas = 264;                        // split target: a fixed number, so dW's bits depend on the shape only

struct WgradParams {
  CUtensorMap amap, bmap;
  float* part;
  int Cout, Kc, kb_total, kb_per_split;
};

// MN-major, 128-byte swizzle: LBO = bytes between 64-element blocks along M / N, SBO = bytes between 8-row groups along K
__device__ __forceinline__ uint64_t make_sdesc_mn(uint32_t saddr, uint32_t lbo) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)((lbo >> 4) & 0x3FFFu) << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D[64 x 128] += A[64 x 16] * B[128 x 16]^T with A and B MN-major (imm-trans-a = imm-trans-b = 1)
__device__ __forceinline__ void wgmma_f16_mn128(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n.reg .pred p;\nsetp.ne.b32 p, 1, 0;\n"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {"
      "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 1, 1;\n}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(a), "l"(b)
      : "memory");
}

__global__ void __launch_bounds__(kWgThreads, 1) deform_wgrad_kernel(const __grid_constant__ WgradParams p) {
  extern __shared__ __align__(16) uint8_t smem_raw[];
  uint8_t* smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + (size_t)kWgStages * kWgStageBytes);
  uint64_t* empty_bar = full_bar + kWgStages;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int n0 = blockIdx.x * kWgTile, m0 = blockIdx.y * kWgTile;
  const int kb0 = blockIdx.z * p.kb_per_split, kb1 = min(kb0 + p.kb_per_split, p.kb_total);
  if (threadIdx.x == 0) {
    for (int i = 0; i < kWgStages; ++i) { mbar_init(&full_bar[i], 1); mbar_init(&empty_bar[i], 8); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (warp >= 8) {
    if (warp == 8 && lane == 0) {
      tma_prefetch_desc(&p.amap);
      tma_prefetch_desc(&p.bmap);
      int s = 0;
      uint32_t ph = 0;
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(&empty_bar[s], ph ^ 1);
        mbar_expect_tx(&full_bar[s], kWgStageBytes);
        uint8_t* st = smem + (size_t)s * kWgStageBytes;
        tma_load_2d(st, &p.amap, &full_bar[s], m0, kb * kWgKb);
        tma_load_2d(st + kWgBox, &p.amap, &full_bar[s], m0 + 64, kb * kWgKb);
        tma_load_2d(st + 2 * kWgBox, &p.bmap, &full_bar[s], n0, kb * kWgKb);
        tma_load_2d(st + 3 * kWgBox, &p.bmap, &full_bar[s], n0 + 64, kb * kWgKb);
        if (++s == kWgStages) { s = 0; ph ^= 1; }
      }
    }
    return;
  }
  const int wg = warp >> 2;
  float acc[64];
#pragma unroll
  for (int i = 0; i < 64; ++i) acc[i] = 0.f;
  int s = 0, prev = -1;
  uint32_t ph = 0;
  const uint32_t base = smem_u32(smem);
  for (int kb = kb0; kb < kb1; ++kb) {
    mbar_wait(&full_bar[s], ph);
    wgmma_fence();
    const uint32_t st = base + (uint32_t)s * kWgStageBytes;
    const uint64_t adesc = make_sdesc_mn(st + (uint32_t)wg * kWgBox, kWgBox);
    const uint64_t bdesc = make_sdesc_mn(st + 2 * kWgBox, kWgBox);
#pragma unroll
    for (int k = 0; k < kWgKb / 16; ++k)
      // 16 pixels = two 1024-byte atoms further along K: +2048 bytes, +128 in the >>4 start field
      wgmma_f16_mn128(acc, adesc + (uint64_t)(k * 128), bdesc + (uint64_t)(k * 128));
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = s;
    if (++s == kWgStages) { s = 0; ph ^= 1; }
  }
  wgmma_wait<0>();
  fence_regs<64>(acc);
  float* out = p.part + (size_t)blockIdx.z * p.Cout * p.Kc;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int row = m0 + wg * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
    if (row >= p.Cout) continue;
#pragma unroll
    for (int jn = 0; jn < 16; ++jn) {
      const int col = n0 + 8 * jn + 2 * (lane & 3);
      if (col < p.Kc)
        *reinterpret_cast<float2*>(out + (size_t)row * p.Kc + col) = make_float2(acc[4 * jn + 2 * i], acc[4 * jn + 2 * i + 1]);
    }
  }
}

// dW[i] = (part[0][i] + part[1][i] + ... + part[splits - 1][i]) / s, in that order
__global__ void deform_wgrad_reduce_kernel(const float4* __restrict__ part, int splits, size_t n4, const float* __restrict__ scale,
                                           float4* __restrict__ dw) {
  const float inv = scale[1];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (size_t)gridDim.x * blockDim.x) {
    float4 a = part[i];
    for (int sp = 1; sp < splits; ++sp) {
      const float4 b = part[(size_t)sp * n4 + i];
      a.x += b.x; a.y += b.y; a.z += b.z; a.w += b.w;
    }
    dw[i] = make_float4(a.x * inv, a.y * inv, a.z * inv, a.w * inv);
  }
}

static void wgrad_split(int Cout, int Kc, long long P, int* kb_total, int* kb_per_split, int* splits) {
  const int tiles = cdiv(Cout, kWgTile) * cdiv(Kc, kWgTile);
  *kb_total = (int)((P + kWgKb - 1) / kWgKb);
  int want = cdiv(kWgTargetCtas, tiles);
  want = want < 1 ? 1 : (want > *kb_total ? *kb_total : want);
  *kb_per_split = cdiv(*kb_total, want);
  *splits = cdiv(*kb_total, *kb_per_split);
}

// ------------------------------------------------------------------------------------------- sigmoid focal loss
// The reference's expressions, operation by operation, with its double-precision literals: 1. / (1. + expf(-x)) is a
// double division rounded to float, (1. - p) a double rounded to float by powf's parameter, term2's bracket a double.
// d = t == class + 1 (positive), t >= 0 and not that class (negative), t < 0 ignored.
__global__ void sigmoid_focal_loss_forward_kernel(const int nthreads, const float* logits, const int64_t* targets,
                                                  const int num_classes, const float gamma, const float alpha,
                                                  float* losses) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nthreads; i += blockDim.x * gridDim.x) {
    const int n = i / num_classes;
    const int d = i % num_classes;
    const int t = (int)targets[n];
    const float c1 = (float)(t == (d + 1));
    const float c2 = (float)((t >= 0) & (t != (d + 1)));
    const float zn = (float)(1.0 - (double)alpha);
    const float zp = alpha;
    const float x = logits[i];
    const float p = (float)(1. / (1. + (double)expf(-x)));
    const float term1 = powf((float)(1. - (double)p), gamma) * logf(fmaxf(p, FLT_MIN));
    const float term2 = (float)((double)powf(p, gamma) *
                                (-1. * (double)x * (double)(x >= 0) -
                                 (double)logf((float)(1. + (double)expf((float)((double)x - 2. * (double)x * (double)(x >= 0)))))));
    float l = 0.0f;
    l += -c1 * term1 * zp;
    l += -c2 * term2 * zn;
    losses[i] = l;
  }
}

__global__ void sigmoid_focal_loss_backward_kernel(const int nthreads, const float* logits, const int64_t* targets,
                                                   const float* d_losses, const int num_classes, const float gamma,
                                                   const float alpha, float* d_logits) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nthreads; i += blockDim.x * gridDim.x) {
    const int n = i / num_classes;
    const int d = i % num_classes;
    const int t = (int)targets[n];
    const float c1 = (float)(t == (d + 1));
    const float c2 = (float)((t >= 0) & (t != (d + 1)));
    const float zn = (float)(1.0 - (double)alpha);
    const float zp = alpha;
    const float x = logits[i];
    const float p = (float)(1. / (1. + (double)expf(-x)));
    const float term1 = (float)((double)powf((float)(1. - (double)p), gamma) *
                                (1. - (double)p - (double)(p * gamma * logf(fmaxf(p, FLT_MIN)))));
    const float term2 = (float)((double)powf(p, gamma) *
                                ((-1. * (double)x * (double)(x >= 0) -
                                  (double)logf((float)(1. + (double)expf((float)((double)x - 2. * (double)x * (double)(x >= 0)))))) *
                                     (1. - (double)p) * (double)gamma -
                                 (double)p));
    float g = 0.0f;
    g += -c1 * term1 * zp;
    g += -c2 * term2 * zn;
    g = g * d_losses[i];
    d_logits[i] = g;
  }
}

static dim3 focal_grid(long long n) {
  const long long b = (n + 511) / 512;
  return dim3((unsigned)(b < 4096 ? b : 4096));
}

}  // namespace smb

using namespace smb;

extern "C" size_t smb_deform_grad_scale_workspace_bytes(void) { return 4096 * sizeof(unsigned); }

extern "C" int smb_deform_grad_scale(const float* grad_out, int n_img, int C, int H, int W, void* out_f16, float* scale,
                                     void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(grad_out && out_f16 && scale && workspace, "smb_deform_grad_scale: null pointer");
  SMB_CHECK_ARG(n_img > 0 && C > 0 && C % 8 == 0 && H > 0 && W > 0, "smb_deform_grad_scale: bad shape %d x %d x %d x %d",
                n_img, C, H, W);
  SMB_CHECK_ARG((long long)n_img * C * H * W < (1ll << 31), "smb_deform_grad_scale: tensor too large");
  SMB_CHECK_ARG(((uintptr_t)out_f16 % 16) == 0, "smb_deform_grad_scale: out must be 16-byte aligned");
  int dev = 0, per_sm = 0;
  SMB_CUDA_OK(cudaGetDevice(&dev));
  SMB_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, grad_scale_kernel, 256, 0));
  int sms = 0;
  SMB_CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
  const long long want = ((long long)n_img * C * H * W / 8 + 255) / 256;
  int grid = per_sm * sms;
  if (grid > 4096) grid = 4096;
  if (want < grid) grid = (int)want;
  if (grid < 1) grid = 1;
  SMB_CHECK_ARG(workspace_bytes >= (size_t)grid * sizeof(unsigned), "smb_deform_grad_scale: workspace too small");
  int HW = H * W;
  unsigned* bm = (unsigned*)workspace;
  void* args[] = {(void*)&grad_out, (void*)&n_img, (void*)&C, (void*)&HW, (void*)&out_f16, (void*)&scale, (void*)&bm};
  SMB_CUDA_OK(cudaLaunchCooperativeKernel((const void*)grad_scale_kernel, dim3(grid), dim3(256), args, 0, (cudaStream_t)stream));
  return SMB_OK;
}

extern "C" int smb_deform_col2im(const float* grad_col, const void* x, const float* offset, int off_pitch, const float* scale,
                                 float* grad_input, float* grad_offset, int n_img, int H, int W, int C,
                                 int deformable_groups, smb_stream_t stream) {
  SMB_CHECK_ARG(grad_col && x && offset && scale && (grad_input || grad_offset), "smb_deform_col2im: null pointer");
  SMB_CHECK_ARG(C % 8 == 0 && C <= kCol2imMaxC && deformable_groups > 0 && C % deformable_groups == 0 &&
                    (C / deformable_groups) % 8 == 0,
                "smb_deform_col2im: C=%d dg=%d unsupported", C, deformable_groups);
  SMB_CHECK_ARG(n_img > 0 && H > 0 && W > 0 && off_pitch >= deformable_groups * 18, "smb_deform_col2im: bad shape");
  const long long warps = (long long)n_img * H * W * 9;
  long long blocks = (warps + kCol2imWarps - 1) / kCol2imWarps;
  if (blocks > 132 * 16) blocks = 132 * 16;
  deform_col2im_kernel<<<(unsigned)blocks, 32 * kCol2imWarps, 0, (cudaStream_t)stream>>>(
      grad_col, (const __half*)x, offset, off_pitch, scale, grad_input, grad_offset, n_img, H, W, C, deformable_groups);
  SMB_LAUNCH_OK("deform_col2im_kernel");
  return SMB_OK;
}

extern "C" size_t smb_deform_weight_grad_workspace_bytes(int Cout, int Kc, long long P) {
  if (Cout <= 0 || Kc <= 0 || P <= 0) return 0;
  int kb_total, kb_per_split, splits;
  wgrad_split(Cout, Kc, P, &kb_total, &kb_per_split, &splits);
  return (size_t)splits * Cout * Kc * sizeof(float);
}

extern "C" int smb_deform_weight_grad(const void* grad_f16, const void* col, long long P, int Cout, int Kc,
                                      const float* scale, float* grad_weight, void* workspace, size_t workspace_bytes,
                                      smb_stream_t stream) {
  SMB_CHECK_ARG(grad_f16 && col && scale && grad_weight && workspace, "smb_deform_weight_grad: null pointer");
  SMB_CHECK_ARG(P > 0 && P < (1ll << 31) && Cout > 0 && Cout % 8 == 0 && Kc > 0 && Kc % 8 == 0,
                "smb_deform_weight_grad: bad shape P=%lld Cout=%d K=%d", P, Cout, Kc);
  SMB_CHECK_ARG(((uintptr_t)grad_f16 % 16) == 0 && ((uintptr_t)col % 16) == 0 && ((uintptr_t)grad_weight % 16) == 0 &&
                    ((uintptr_t)workspace % 16) == 0,
                "smb_deform_weight_grad: pointers must be 16-byte aligned");
  SMB_CHECK_ARG(workspace_bytes >= smb_deform_weight_grad_workspace_bytes(Cout, Kc, P),
                "smb_deform_weight_grad: workspace too small");
  WgradParams p;
  memset(&p, 0, sizeof(p));
  p.Cout = Cout; p.Kc = Kc; p.part = (float*)workspace;
  int splits;
  wgrad_split(Cout, Kc, P, &p.kb_total, &p.kb_per_split, &splits);
  const uint32_t box[2] = {64, (uint32_t)kWgKb};
  const uint64_t adims[2] = {(uint64_t)Cout, (uint64_t)P}, astr[1] = {(uint64_t)Cout * 2};
  const uint64_t bdims[2] = {(uint64_t)Kc, (uint64_t)P}, bstr[1] = {(uint64_t)Kc * 2};
  int rc = encode_map(&p.amap, const_cast<void*>(grad_f16), 2, adims, astr, box);
  if (rc == SMB_OK) rc = encode_map(&p.bmap, const_cast<void*>(col), 2, bdims, bstr, box);
  if (rc != SMB_OK) return rc;
  static DeviceOnce attr_once;
  if (attr_once.first())
    SMB_CUDA_OK(cudaFuncSetAttribute(deform_wgrad_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kWgSmem));
  const dim3 grid(cdiv(Kc, kWgTile), cdiv(Cout, kWgTile), splits);
  deform_wgrad_kernel<<<grid, kWgThreads, kWgSmem, (cudaStream_t)stream>>>(p);
  SMB_LAUNCH_OK("deform_wgrad_kernel");
  const size_t n4 = (size_t)Cout * Kc / 4;
  deform_wgrad_reduce_kernel<<<(unsigned)((n4 + 255) / 256 < 4096 ? (n4 + 255) / 256 : 4096), 256, 0, (cudaStream_t)stream>>>(
      (const float4*)workspace, splits, n4, scale, (float4*)grad_weight);
  SMB_LAUNCH_OK("deform_wgrad_reduce_kernel");
  return SMB_OK;
}

extern "C" int smb_sigmoid_focal_loss_forward(const float* logits, const int64_t* targets, int N, int num_classes,
                                              float gamma, float alpha, float* losses, smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && num_classes > 0 && (long long)N * num_classes < (1ll << 31),
                "smb_sigmoid_focal_loss_forward: bad shape %d x %d", N, num_classes);
  const int n = N * num_classes;
  if (n == 0) return SMB_OK;
  SMB_CHECK_ARG(logits && targets && losses, "smb_sigmoid_focal_loss_forward: null pointer");
  sigmoid_focal_loss_forward_kernel<<<focal_grid(n), 512, 0, (cudaStream_t)stream>>>(n, logits, targets, num_classes, gamma,
                                                                                     alpha, losses);
  SMB_LAUNCH_OK("sigmoid_focal_loss_forward_kernel");
  return SMB_OK;
}

extern "C" int smb_sigmoid_focal_loss_backward(const float* logits, const int64_t* targets, const float* d_losses, int N,
                                               int num_classes, float gamma, float alpha, float* d_logits,
                                               smb_stream_t stream) {
  SMB_CHECK_ARG(N >= 0 && num_classes > 0 && (long long)N * num_classes < (1ll << 31),
                "smb_sigmoid_focal_loss_backward: bad shape %d x %d", N, num_classes);
  const int n = N * num_classes;
  if (n == 0) return SMB_OK;
  SMB_CHECK_ARG(logits && targets && d_losses && d_logits, "smb_sigmoid_focal_loss_backward: null pointer");
  sigmoid_focal_loss_backward_kernel<<<focal_grid(n), 512, 0, (cudaStream_t)stream>>>(n, logits, targets, d_losses,
                                                                                      num_classes, gamma, alpha, d_logits);
  SMB_LAUNCH_OK("sigmoid_focal_loss_backward_kernel");
  return SMB_OK;
}
