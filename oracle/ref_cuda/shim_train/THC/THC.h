// TEST INFRASTRUCTURE ONLY - stand-in for <THC/THC.h>: THCudaCheck passes the CUDA status through unchecked (the
// wrappers in oracle/ref_cuda/ check cudaDeviceSynchronize themselves).
#pragma once
#include <cuda_runtime.h>
#define THCudaCheck(err) ((void)(err))
