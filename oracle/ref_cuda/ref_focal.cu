// TEST INFRASTRUCTURE ONLY.  Compiles the reference's sigmoid focal loss CUDA source from where it lies
// (REF_SRC = /root/reference/SipMask-mmdetection/mmdet/ops/sigmoid_focal_loss/src/sigmoid_focal_loss_cuda.cu) and launches
// its kernel templates SigmoidFocalLossForward (:23-60) and SigmoidFocalLossBackward (:62-100) for float behind C entry
// points, with the reference launchers' configuration (:109-110: 512 threads, at most 4096 blocks).  The launchers
// themselves allocate through ATen, so they are renamed to unused static functions and never compiled into code.
#define SigmoidFocalLoss_forward_cuda static inline ref_unused_sigmoid_focal_loss_forward
#define SigmoidFocalLoss_backward_cuda static inline ref_unused_sigmoid_focal_loss_backward
#include REF_SRC

static dim3 ref_focal_grid(int n) { return dim3(std::min((n + 511) / 512, 4096)); }

extern "C" int ref_sigmoid_focal_loss_forward(const float* logits, const int64_t* targets, int N, int C, float gamma,
                                              float alpha, float* losses) {
  const int n = N * C;
  if (n == 0) return 0;
  SigmoidFocalLossForward<float><<<ref_focal_grid(n), 512>>>(n, logits, targets, C, gamma, alpha, N, losses);
  return (int)cudaDeviceSynchronize();
}

extern "C" int ref_sigmoid_focal_loss_backward(const float* logits, const int64_t* targets, const float* d_losses, int N,
                                               int C, float gamma, float alpha, float* d_logits) {
  const int n = N * C;
  if (n == 0) return 0;
  SigmoidFocalLossBackward<float><<<ref_focal_grid(n), 512>>>(n, logits, targets, d_losses, C, gamma, alpha, N, d_logits);
  return (int)cudaDeviceSynchronize();
}
