// SipMask++ mask rescoring (SURVEY.md 8a-10): six [conv3x3 stride 2 pad 0 + bias + ReLU] on the cropped stride-2 masks
// [N,1,Hm,Wm] (1 -> 16 -> 16 -> 16 -> 32 -> 64 -> 128 channels), conv1x1 -> classes, ReLU, global max-pool, pick the
// detection's class, times the box score (SipMask-mmdetection/mmdet/models/anchor_heads/sipmask_head.py:200-219 layers,
// :635-643 use).  3.7 GFLOP for 100 detections at 272x272.  Two implementations: fp32 CUDA-core direct convolutions, NCHW
// like the reference (operator API, drop-in head, the tests' reference), and the engine's fp16 tensor-core chain below.
#include <stdint.h>

#include "common.cuh"

namespace smb {

constexpr int RS_CO = 16;          // output channels per thread

// in [N,Cin,H,W] fp32, w [Cout,Cin,3,3], out [N,Cout,Ho,Wo], Ho = (H-3)/2+1.  blockIdx.y = group of 16 output channels.
__global__ void __launch_bounds__(128) conv3x3s2_relu_kernel(const float* __restrict__ in, const float* __restrict__ w,
                                                            const float* __restrict__ bias, float* __restrict__ out, int N, int Cin,
                                                            int H, int W, int Cout, int Ho, int Wo) {
  extern __shared__ float s_w[];                  // [RS_CO][Cin*9] weights of this channel group
  const int co0 = blockIdx.y * RS_CO;
  const int kk = Cin * 9;
  for (int i = threadIdx.x; i < RS_CO * kk; i += blockDim.x) {
    const int c = i / kk, r = i - c * kk;
    s_w[i] = (co0 + c < Cout) ? w[(size_t)(co0 + c) * kk + r] : 0.f;
  }
  __syncthreads();
  const long long total = (long long)N * Ho * Wo;
  for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)blockDim.x * gridDim.x) {
    const int ox = (int)(t % Wo), oy = (int)((t / Wo) % Ho), n = (int)(t / ((long long)Wo * Ho));
    float acc[RS_CO];
#pragma unroll
    for (int c = 0; c < RS_CO; ++c) acc[c] = (co0 + c < Cout) ? bias[co0 + c] : 0.f;
    const float* ip = in + ((size_t)n * Cin * H + 2 * oy) * W + 2 * ox;
    for (int ci = 0; ci < Cin; ++ci, ip += (size_t)H * W) {
      float x[9];
#pragma unroll
      for (int r = 0; r < 3; ++r)
#pragma unroll
        for (int s = 0; s < 3; ++s) x[r * 3 + s] = __ldg(ip + r * W + s);
      const float* wp = s_w + ci * 9;
#pragma unroll
      for (int c = 0; c < RS_CO; ++c) {
#pragma unroll
        for (int k = 0; k < 9; ++k) acc[c] = fmaf(wp[c * kk + k], x[k], acc[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < RS_CO; ++c)
      if (co0 + c < Cout) out[(((size_t)n * Cout + co0 + c) * Ho + oy) * Wo + ox] = fmaxf(acc[c], 0.f);
  }
}

// feat [N,C,h,w] fp32 -> mask_score[n] = det_score[n] * max_p relu(w1[label[n]] . feat[n,:,p] + b1[label[n]])
// one warp per detection (only the detection's own class row of the 1x1 conv is needed)
__global__ void rescore_final_kernel(const float* __restrict__ feat, int N, int C, int hw, const float* __restrict__ w1,
                                     const float* __restrict__ b1, const long long* __restrict__ labels,
                                     const float* __restrict__ det, const int* __restrict__ n_valid, float* __restrict__ scores) {
  const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= N) return;
  if (n_valid && n >= *n_valid) {
    if (lane == 0) scores[n] = 0.f;
    return;
  }
  const int c = (int)labels[n];
  const float* f = feat + (size_t)n * C * hw;
  const float* wr = w1 + (size_t)c * C;
  float best = 0.f;                                // ReLU output is >= 0, so 0 is the identity of the max
  for (int p = 0; p < hw; ++p) {
    float a = 0.f;
    for (int k = lane; k < C; k += 32) a = fmaf(wr[k], f[(size_t)k * hw + p], a);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    best = fmaxf(best, fmaxf(a + b1[c], 0.f));
  }
  if (lane == 0) scores[n] = best * det[(size_t)n * 5 + 4];
}

// ---------------------------------------------------------------------------------------------------------------
// Tensor-core chain (the engine's path): fp16 masks, weights and activations, fp32 accumulation, mma.sync.m16n8k16.
// Rows are r = img * max_rows + j; a row with j >= clamp(count[img], 0, max_rows) does no work.
//   rescore_l12_kernel       layers 1+2: one CTA = (row, 8 x 16 layer-2 outputs); the 35 x 67 input window and the 17 x 33
//                            x 16 layer-1 tile live in shared memory, layer 1 never reaches global memory
//   rescore_conv_kernel      layers 3-5: implicit GEMM straight from the NHWC fp16 input (L1 / L2 resident), one warp =
//                            16 output pixels x all output channels
//   rescore_score_kernel     layer 6 + the detection's mask_scoring row + ReLU + max over positions + x det[:, 4]: one
//                            CTA per row, the four warps split the 128 output channels
// The m16n8k16 fragments: A row g / g + 8 = output pixel, k = (tap, input channel); B column = output channel, read as
// 32-bit pairs from the [Cout, 9 * Cin] K-major weights; D row g / g + 8, columns 2t, 2t + 1.
__device__ __forceinline__ void rs_mma(float (&d)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile(
      "mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t ldg_h2(const __half* p) { return __ldg(reinterpret_cast<const unsigned int*>(p)); }
__device__ __forceinline__ uint32_t lds_h2(const __half* p) { return *reinterpret_cast<const uint32_t*>(p); }
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

__device__ __forceinline__ bool rs_row_live(const int* __restrict__ count, int r, int max_rows) {
  const int img = r / max_rows, j = r - img * max_rows;
  const int c = min(max(count[img], 0), max_rows);
  return j < c;
}

constexpr int L12_TH = 8, L12_TW = 16;                            // layer-2 outputs per CTA (8 M-tiles of 16)
constexpr int L12_IH = 4 * L12_TH + 3, L12_IW = 4 * L12_TW + 3;   // input window 35 x 67
constexpr int L12_AH = 2 * L12_TH + 1, L12_AW = 2 * L12_TW + 1;   // layer-1 tile 17 x 33
constexpr int L12_AP = 20;   // layer-1 pixel pitch in halves: 16 channels + 4 pad, so the A loads of the 8 rows g (pixels
                             // 2 apart = 20 words) hit 32 distinct banks

// masks [R,H,W] fp16 -> out [R,H2,W2,16] fp16.  blockIdx.x = row, blockIdx.y = tile.
__global__ void __launch_bounds__(128, 4) rescore_l12_kernel(const __half* __restrict__ masks, int max_rows, int H, int W,
                                                             const int* __restrict__ count, const __half* __restrict__ w1,
                                                             const float* __restrict__ b1, const __half* __restrict__ w2,
                                                             const float* __restrict__ b2, __half* __restrict__ out, int H2,
                                                             int W2, int tiles_x) {
  __shared__ __half s_in[L12_IH * L12_IW];
  __shared__ __align__(16) __half s_a[L12_AH * L12_AW * L12_AP];
  const int r = blockIdx.x;
  if (!rs_row_live(count, r, max_rows)) return;
  const int oy0 = (blockIdx.y / tiles_x) * L12_TH, ox0 = (blockIdx.y % tiles_x) * L12_TW;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  // layer-2 B fragments of all nine taps and both 8-channel halves, loaded before the layer-1 work hides their latency
  uint32_t b[9][2][2];
#pragma unroll
  for (int tap = 0; tap < 9; ++tap)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      const __half* wp = w2 + (nt * 8 + g) * 144 + tap * 16 + 2 * t;
      b[tap][nt][0] = ldg_h2(wp);
      b[tap][nt][1] = ldg_h2(wp + 8);
    }
  const __half* src = masks + (size_t)r * H * W;
  const int iy0 = 4 * oy0, ix0 = 4 * ox0;
  for (int i = threadIdx.x; i < L12_IH * L12_IW; i += 128) {
    const int y = i / L12_IW, x = i - y * L12_IW;
    const int gy = iy0 + y, gx = ix0 + x;     // past the map: zeros, which only reach outputs that are not stored
    s_in[i] = (gy < H && gx < W) ? src[(size_t)gy * W + gx] : __float2half(0.f);
  }
  // layer 1 (Cin = 1, K = 9): fp32 FMAs, + bias, ReLU, fp16 into the NHWC tile.  A thread owns 4 channels (36 weights in
  // registers) of every 32nd pixel.
  const int cq = 4 * (threadIdx.x & 3);
  float wl[4][9], bl[4];
#pragma unroll
  for (int c = 0; c < 4; ++c) {
    bl[c] = b1[cq + c];
#pragma unroll
    for (int k = 0; k < 9; ++k) wl[c][k] = __half2float(w1[(cq + c) * 9 + k]);
  }
  __syncthreads();
  for (int p = threadIdx.x >> 2; p < L12_AH * L12_AW; p += 32) {
    const int y = p / L12_AW, x = p - y * L12_AW;
    float v[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) v[k] = __half2float(s_in[(2 * y + k / 3) * L12_IW + 2 * x + k % 3]);
    float a[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      a[c] = bl[c];
#pragma unroll
      for (int k = 0; k < 9; ++k) a[c] = fmaf(wl[c][k], v[k], a[c]);
    }
    *reinterpret_cast<uint2*>(s_a + p * L12_AP + cq) =         // 40-byte pixels, 8-byte chunks
        make_uint2(pack_h2(fmaxf(a[0], 0.f), fmaxf(a[1], 0.f)), pack_h2(fmaxf(a[2], 0.f), fmaxf(a[3], 0.f)));
  }
  __syncthreads();
  // layer 2: warp w owns layer-2 rows 2w, 2w + 1 of the tile (one M-tile of 16 pixels each), K = 9 taps x 16 channels
#pragma unroll
  for (int mi = 0; mi < 2; ++mi) {
    const int ly = 2 * warp + mi;
    float acc[2][4];
#pragma unroll
    for (int nt = 0; nt < 2; ++nt) {
      acc[nt][0] = acc[nt][2] = b2[nt * 8 + 2 * t];
      acc[nt][1] = acc[nt][3] = b2[nt * 8 + 2 * t + 1];
    }
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) {
      const __half* lo = s_a + ((2 * ly + tap / 3) * L12_AW + 2 * g + tap % 3) * L12_AP + 2 * t;
      const __half* hi = lo + 16 * L12_AP;                     // pixel g + 8 = layer-1 column + 16
      const uint32_t a[4] = {lds_h2(lo), lds_h2(hi), lds_h2(lo + 8), lds_h2(hi + 8)};
      rs_mma(acc[0], a, b[tap][0][0], b[tap][0][1]);
      rs_mma(acc[1], a, b[tap][1][0], b[tap][1][1]);
    }
    const int oy = oy0 + ly;
    if (oy < H2) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int ox = ox0 + g + 8 * h;
        if (ox < W2) {
          __half* dst = out + (((size_t)r * H2 + oy) * W2 + ox) * 16 + 2 * t;
#pragma unroll
          for (int nt = 0; nt < 2; ++nt)
            *reinterpret_cast<uint32_t*>(dst + nt * 8) = pack_h2(fmaxf(acc[nt][2 * h], 0.f), fmaxf(acc[nt][2 * h + 1], 0.f));
        }
      }
    }
  }
}

// acc[j] += A (16 output pixels: rows g / g + 8 read from the 3x3 windows at pa / pb) x W^T (output channels n0 + 8j ..)
template <int CIN, int NT>
__device__ __forceinline__ void conv3x3s2_mma(const __half* pa, const __half* pb, int Wi, const __half* __restrict__ w, int n0,
                                              int g, int t, float (&acc)[NT][4]) {
  constexpr int K = 9 * CIN;
#pragma unroll 1   // unrolled, the pixel loop of rescore_score_kernel would hoist all 9 x CIN / 16 x NT B fragments (spills)
  for (int tap = 0; tap < 9; ++tap) {
    const int off = ((tap / 3) * Wi + tap % 3) * CIN + 2 * t;
#pragma unroll
    for (int c = 0; c < CIN; c += 16) {
      const uint32_t a[4] = {ldg_h2(pa + off + c), ldg_h2(pb + off + c), ldg_h2(pa + off + c + 8), ldg_h2(pb + off + c + 8)};
#pragma unroll
      for (int j = 0; j < NT; ++j) {
        const __half* wr = w + (size_t)(n0 + 8 * j + g) * K + tap * CIN + c + 2 * t;
        rs_mma(acc[j], a, ldg_h2(wr), ldg_h2(wr + 8));
      }
    }
  }
}

// in [R,Hi,Wi,CIN] -> out [R,Ho,Wo,COUT] (conv3x3 s2 p0 + bias + ReLU).  blockIdx.x = row, blockIdx.y = 64-pixel group.
template <int CIN, int COUT>
__global__ void __launch_bounds__(128) rescore_conv_kernel(const __half* __restrict__ in, int max_rows, int Hi, int Wi,
                                                           const int* __restrict__ count, const __half* __restrict__ w,
                                                           const float* __restrict__ bias, __half* __restrict__ out, int Ho,
                                                           int Wo) {
  const int r = blockIdx.x;
  if (!rs_row_live(count, r, max_rows)) return;
  const int Mo = Ho * Wo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int m0 = (blockIdx.y * 4 + warp) * 16;
  if (m0 >= Mo) return;                                        // no barriers below
  const __half* src = in + (size_t)r * Hi * Wi * CIN;
  const int ma = min(m0 + g, Mo - 1), mb = min(m0 + g + 8, Mo - 1);
  const int ya = ma / Wo, yb = mb / Wo;
  const __half* pa = src + ((size_t)(2 * ya) * Wi + 2 * (ma - ya * Wo)) * CIN;
  const __half* pb = src + ((size_t)(2 * yb) * Wi + 2 * (mb - yb * Wo)) * CIN;
  constexpr int NT = COUT / 8;
  float acc[NT][4];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    acc[j][0] = acc[j][2] = bias[8 * j + 2 * t];
    acc[j][1] = acc[j][3] = bias[8 * j + 2 * t + 1];
  }
  conv3x3s2_mma<CIN, NT>(pa, pb, Wi, w, 0, g, t, acc);
  __half* dst = out + (size_t)r * Mo * COUT + 2 * t;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = m0 + g + 8 * h;
    if (m < Mo) {
#pragma unroll
      for (int j = 0; j < NT; ++j)
        *reinterpret_cast<uint32_t*>(dst + (size_t)m * COUT + 8 * j) =
            pack_h2(fmaxf(acc[j][2 * h], 0.f), fmaxf(acc[j][2 * h + 1], 0.f));
    }
  }
}

// Layer 6 (64 -> 128) and the score.  scores[r] = det[r,4] * max_p relu(ws[label] . fp16(relu(conv6)[p]) + bs[label]);
// 0 for rows past the count and for labels outside [0, num_classes).
__global__ void __launch_bounds__(128) rescore_score_kernel(const __half* __restrict__ in, int max_rows, int Hi, int Wi,
                                                            const int* __restrict__ count, const __half* __restrict__ w,
                                                            const float* __restrict__ bias, const __half* __restrict__ ws,
                                                            const float* __restrict__ bs, int num_classes,
                                                            const long long* __restrict__ labels, const float* __restrict__ det,
                                                            float* __restrict__ scores, int Ho, int Wo) {
  constexpr int CIN = 64, COUT = 128, NT = COUT / 8 / 4;       // each warp: 32 output channels
  __shared__ float s_part[4][16];
  const int r = blockIdx.x;
  const long long lab = labels[r];
  if (!rs_row_live(count, r, max_rows) || lab < 0 || lab >= num_classes) {
    if (threadIdx.x == 0) scores[r] = 0.f;
    return;
  }
  const int Mo = Ho * Wo;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int n0 = warp * NT * 8;
  float wc[NT][2], bini[NT][2];
#pragma unroll
  for (int j = 0; j < NT; ++j) {
    const int c = n0 + 8 * j + 2 * t;
    wc[j][0] = __half2float(ws[(size_t)lab * COUT + c]);
    wc[j][1] = __half2float(ws[(size_t)lab * COUT + c + 1]);
    bini[j][0] = bias[c];
    bini[j][1] = bias[c + 1];
  }
  const float b_cls = bs[lab];
  const __half* src = in + (size_t)r * Hi * Wi * CIN;
  float best = 0.f;                                            // ReLU outputs are >= 0: 0 is the identity of the max
  for (int m0 = 0; m0 < Mo; m0 += 16) {
    const int ma = min(m0 + g, Mo - 1), mb = min(m0 + g + 8, Mo - 1);
    const int ya = ma / Wo, yb = mb / Wo;
    const __half* pa = src + ((size_t)(2 * ya) * Wi + 2 * (ma - ya * Wo)) * CIN;
    const __half* pb = src + ((size_t)(2 * yb) * Wi + 2 * (mb - yb * Wo)) * CIN;
    float acc[NT][4];
#pragma unroll
    for (int j = 0; j < NT; ++j) {
      acc[j][0] = acc[j][2] = bini[j][0];
      acc[j][1] = acc[j][3] = bini[j][1];
    }
    conv3x3s2_mma<CIN, NT>(pa, pb, Wi, w, n0, g, t, acc);
    float sa = 0.f, sb = 0.f;                                  // this lane's part of the 1x1 dot for pixels g, g + 8
#pragma unroll
    for (int j = 0; j < NT; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        sa = fmaf(wc[j][e], __half2float(__float2half_rn(fmaxf(acc[j][e], 0.f))), sa);
        sb = fmaf(wc[j][e], __half2float(__float2half_rn(fmaxf(acc[j][2 + e], 0.f))), sb);
      }
    sa += __shfl_xor_sync(0xffffffffu, sa, 1);
    sb += __shfl_xor_sync(0xffffffffu, sb, 1);
    sa += __shfl_xor_sync(0xffffffffu, sa, 2);
    sb += __shfl_xor_sync(0xffffffffu, sb, 2);
    if (t == 0) {
      s_part[warp][g] = sa;
      s_part[warp][g + 8] = sb;
    }
    __syncthreads();
    if (threadIdx.x < 16 && m0 + threadIdx.x < Mo) {
      const int i = threadIdx.x;
      const float s = b_cls + s_part[0][i] + s_part[1][i] + s_part[2][i] + s_part[3][i];
      best = fmaxf(best, fmaxf(s, 0.f));
    }
    __syncthreads();
  }
  if (warp == 0) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, o));
    if (lane == 0) scores[r] = best * det[(size_t)r * 5 + 4];
  }
}

// Shapes of the chain: layer l maps S[l-1] -> S[l] = (S[l-1] - 3) / 2 + 1, S[0] = the mask size.
struct RescoreShapes {
  int h[7], w[7];
  size_t off[4], bytes;        // workspace: layer-2..5 outputs [R,h,w,C] fp16 with C = 16, 16, 32, 64, 256-byte aligned
};
static RescoreShapes rescore_shapes(long long R, int H, int W) {
  RescoreShapes s;
  s.h[0] = H;
  s.w[0] = W;
  for (int l = 1; l < 7; ++l) {
    s.h[l] = (s.h[l - 1] - 3) / 2 + 1;
    s.w[l] = (s.w[l - 1] - 3) / 2 + 1;
  }
  const int ch[4] = {16, 16, 32, 64};
  size_t o = 0;
  for (int i = 0; i < 4; ++i) {
    s.off[i] = o;
    o = align_up(o + (size_t)R * s.h[i + 2] * s.w[i + 2] * ch[i] * sizeof(__half), 256);
  }
  s.bytes = o;
  return s;
}

}  // namespace smb

using namespace smb;

extern "C" int smb_conv3x3s2_relu_f32(const float* in, const float* weight, const float* bias, float* out, int N, int Cin, int H,
                                      int W, int Cout, smb_stream_t stream) {
  SMB_CHECK_ARG(in && weight && bias && out, "smb_conv3x3s2_relu_f32: null pointer");
  SMB_CHECK_ARG(N >= 0 && Cin > 0 && Cout > 0 && H >= 3 && W >= 3 && Cin <= 128, "smb_conv3x3s2_relu_f32: bad shape");
  if (N == 0) return SMB_OK;
  const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
  const long long total = (long long)N * Ho * Wo;
  int bx = (int)((total + 127) / 128);
  if (bx > 132 * 32) bx = 132 * 32;
  dim3 grid(bx, (Cout + RS_CO - 1) / RS_CO);
  const size_t smem = (size_t)RS_CO * Cin * 9 * sizeof(float);
  static bool attr_done = false;
  if (!attr_done) {
    SMB_CUDA_OK(cudaFuncSetAttribute(conv3x3s2_relu_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, RS_CO * 128 * 9 * 4));
    attr_done = true;
  }
  conv3x3s2_relu_kernel<<<grid, 128, smem, (cudaStream_t)stream>>>(in, weight, bias, out, N, Cin, H, W, Cout, Ho, Wo);
  SMB_LAUNCH_OK("conv3x3s2_relu_kernel");
  return SMB_OK;
}

extern "C" int smb_mask_rescore(const float* feat, int N, int C, int h, int w, const float* weight1x1, const float* bias1x1,
                                int num_classes, const int64_t* labels, const float* det, const int* n_valid, float* scores,
                                smb_stream_t stream) {
  SMB_CHECK_ARG(feat && weight1x1 && bias1x1 && labels && det && scores, "smb_mask_rescore: null pointer");
  SMB_CHECK_ARG(N >= 0 && C > 0 && h > 0 && w > 0 && num_classes > 0, "smb_mask_rescore: bad shape");
  if (N == 0) return SMB_OK;
  rescore_final_kernel<<<(N + 3) / 4, 128, 0, (cudaStream_t)stream>>>(feat, N, C, h * w, weight1x1, bias1x1,
                                                                       (const long long*)labels, det, n_valid, scores);
  SMB_LAUNCH_OK("rescore_final_kernel");
  return SMB_OK;
}

extern "C" size_t smb_mask_rescore_f16_workspace_bytes(int R, int H, int W) {
  if (R < 0 || H < 127 || W < 127) return 0;
  return rescore_shapes(R, H, W).bytes;
}

extern "C" int smb_mask_rescore_f16(const void* pos_masks, int n_img, int max_rows, int H, int W, const int* count,
                                    const smb_rescore_weights_t* host_weights, const int64_t* labels, const float* det,
                                    float* scores, void* workspace, size_t workspace_bytes, smb_stream_t stream) {
  SMB_CHECK_ARG(pos_masks && count && host_weights && labels && det && scores && workspace,
                "smb_mask_rescore_f16: null pointer");
  const smb_rescore_weights_t& wt = *host_weights;
  for (int i = 0; i < 6; ++i)
    SMB_CHECK_ARG(wt.conv_w[i] && wt.conv_b[i], "smb_mask_rescore_f16: null weight pointer (layer %d)", i + 1);
  SMB_CHECK_ARG(wt.score_w && wt.score_b && wt.num_classes > 0, "smb_mask_rescore_f16: bad mask_scoring weights");
  SMB_CHECK_ARG(n_img >= 0 && max_rows >= 0 && (long long)n_img * max_rows <= 0x7fffffffLL,
                "smb_mask_rescore_f16: bad n_img=%d max_rows=%d", n_img, max_rows);
  SMB_CHECK_ARG(H >= 127 && W >= 127, "smb_mask_rescore_f16: masks %dx%d are smaller than the 127x127 that six valid "
                "stride-2 3x3 convolutions need", H, W);
  const int R = n_img * max_rows;
  const RescoreShapes s = rescore_shapes(R, H, W);
  SMB_CHECK_ARG(workspace_bytes >= s.bytes, "smb_mask_rescore_f16: workspace %zu < %zu bytes", workspace_bytes, s.bytes);
  const int tiles_x = cdiv(s.w[2], L12_TW), tiles = tiles_x * cdiv(s.h[2], L12_TH);
  SMB_CHECK_ARG(tiles <= 65535 && cdiv(s.h[3] * s.w[3], 64) <= 65535, "smb_mask_rescore_f16: masks %dx%d too large", H, W);
  if (R == 0) return SMB_OK;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  __half* a2 = (__half*)(ws + s.off[0]);
  __half* a3 = (__half*)(ws + s.off[1]);
  __half* a4 = (__half*)(ws + s.off[2]);
  __half* a5 = (__half*)(ws + s.off[3]);
  const __half* const* w = (const __half* const*)wt.conv_w;
  rescore_l12_kernel<<<dim3(R, tiles), 128, 0, st>>>((const __half*)pos_masks, max_rows, H, W, count, w[0], wt.conv_b[0], w[1],
                                                     wt.conv_b[1], a2, s.h[2], s.w[2], tiles_x);
  SMB_LAUNCH_OK("rescore_l12_kernel");
  rescore_conv_kernel<16, 16><<<dim3(R, cdiv(s.h[3] * s.w[3], 64)), 128, 0, st>>>(a2, max_rows, s.h[2], s.w[2], count, w[2],
                                                                                  wt.conv_b[2], a3, s.h[3], s.w[3]);
  SMB_LAUNCH_OK("rescore_conv_kernel<16,16>");
  rescore_conv_kernel<16, 32><<<dim3(R, cdiv(s.h[4] * s.w[4], 64)), 128, 0, st>>>(a3, max_rows, s.h[3], s.w[3], count, w[3],
                                                                                  wt.conv_b[3], a4, s.h[4], s.w[4]);
  SMB_LAUNCH_OK("rescore_conv_kernel<16,32>");
  rescore_conv_kernel<32, 64><<<dim3(R, cdiv(s.h[5] * s.w[5], 64)), 128, 0, st>>>(a4, max_rows, s.h[4], s.w[4], count, w[4],
                                                                                  wt.conv_b[4], a5, s.h[5], s.w[5]);
  SMB_LAUNCH_OK("rescore_conv_kernel<32,64>");
  rescore_score_kernel<<<R, 128, 0, st>>>(a5, max_rows, s.h[5], s.w[5], count, w[5], wt.conv_b[5],
                                          (const __half*)wt.score_w, wt.score_b, wt.num_classes, (const long long*)labels,
                                          det, scores, s.h[6], s.w[6]);
  SMB_LAUNCH_OK("rescore_score_kernel");
  return SMB_OK;
}
