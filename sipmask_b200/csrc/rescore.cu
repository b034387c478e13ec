// SipMask++ mask rescoring (SURVEY.md 8a-10): six [conv3x3 stride 2 pad 0 + bias + ReLU] on the cropped stride-2 masks
// [N,1,Hm,Wm] (1 -> 16 -> 16 -> 16 -> 32 -> 64 -> 128 channels), conv1x1 -> classes, ReLU, global max-pool, pick the
// detection's class, times the box score (SipMask-mmdetection/mmdet/models/anchor_heads/sipmask_head.py:200-219 layers,
// :635-643 use).  3.7 GFLOP for 100 detections at 272x272: fp32 CUDA-core direct convolutions (the channel counts are far
// below a tensor-core tile and the reference computes them in fp32), NCHW like the reference.
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
