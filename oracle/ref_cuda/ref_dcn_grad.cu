// TEST INFRASTRUCTURE ONLY.  Compiles the reference's deformable-convolution CUDA source from where it lies
// (REF_SRC = /root/reference/SipMask-mmdetection/mmdet/ops/dcn/src/deform_conv_cuda_kernel.cu, passed by
// oracle/build_train.py) and exports its backward launchers behind C entry points:
//   deformable_col2im (:337-371; kernel :279-335, get_gradient_weight :117-143):
//     col [C*k*k, B, Ho, Wo] fp32 -> grad_im [B,C,H,W] (accumulated: the caller zeroes it, deform_conv_cuda.cpp:300)
//   deformable_col2im_coord (:438-465; kernel :373-436, get_coordinate_weight :145-188):
//     col, im [B,C,H,W], offset [B,dg*2*k*k,Ho,Wo] -> grad_offset [B,dg*2*k*k,Ho,Wo] (every element written)
#include REF_SRC

extern "C" int ref_deformable_col2im(const float* col, const float* offset, int C, int H, int W, int k, int pad, int stride,
                                     int dilation, int parallel_imgs, int dg, float* grad_im) {
  deformable_col2im(at::Tensor(col), at::Tensor(offset), C, H, W, k, k, pad, pad, stride, stride, dilation, dilation,
                    parallel_imgs, dg, at::Tensor(grad_im));
  return (int)cudaDeviceSynchronize();
}

extern "C" int ref_deformable_col2im_coord(const float* col, const float* im, const float* offset, int C, int H, int W,
                                           int k, int pad, int stride, int dilation, int parallel_imgs, int dg,
                                           float* grad_offset) {
  deformable_col2im_coord(at::Tensor(col), at::Tensor(im), at::Tensor(offset), C, H, W, k, k, pad, pad, stride, stride,
                          dilation, dilation, parallel_imgs, dg, at::Tensor(grad_offset));
  return (int)cudaDeviceSynchronize();
}
