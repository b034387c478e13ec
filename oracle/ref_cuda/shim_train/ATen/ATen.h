// TEST INFRASTRUCTURE ONLY - stand-in for <ATen/ATen.h> for the reference's training-side CUDA sources
// (deform_conv_cuda_kernel.cu's col2im launchers, sigmoid_focal_loss_cuda.cu), compiled with plain nvcc from where they
// lie under /root/reference by oracle/build_train.py; it is found before oracle/ref_cuda/shim/, which supplies the other
// headers.  No arithmetic lives here: at::Tensor is a raw device pointer, the dispatch macro instantiates the reference's
// lambda for scalar_t = float.  The members and functions that are only declared (dim, size, empty, ...) are used by
// launchers that the wrappers never compile into code (sigmoid_focal_loss_cuda.cu's, which oracle/ref_cuda/ref_focal.cu
// bypasses to launch the kernel templates itself).
#pragma once
#include <cuda_runtime.h>
#include <algorithm>
#include <cstdint>
#include <initializer_list>
namespace at {
struct Half {};
struct TensorOptions {};
struct TypeInfo {
  bool is_cuda() const { return true; }
};
struct Tensor {
  void* ptr;
  Tensor() : ptr(nullptr) {}
  explicit Tensor(const void* p) : ptr(const_cast<void*>(p)) {}
  template <typename T> T* data() const { return static_cast<T*>(ptr); }
  template <typename T> T* data_ptr() const { return static_cast<T*>(ptr); }
  TypeInfo type() const { return TypeInfo(); }
  int scalar_type() const { return 0; }
  int64_t dim() const;
  int64_t size(int64_t d) const;
  int64_t numel() const;
  TensorOptions options() const;
  Tensor contiguous() const;
};
Tensor empty(std::initializer_list<int64_t> sizes, const TensorOptions& options);
Tensor zeros(std::initializer_list<int64_t> sizes, const TensorOptions& options);
}  // namespace at
#define AT_ASSERTM(cond, msg) ((void)0)
#define AT_DISPATCH_FLOATING_TYPES_AND_HALF(TYPE, NAME, ...) \
  {                                                          \
    (void)(TYPE);                                            \
    using scalar_t = float;                                  \
    __VA_ARGS__();                                           \
  }
