// TEST INFRASTRUCTURE ONLY - stand-in for <THC/THCDeviceUtils.cuh>: THCCeilDiv is declared for the reference launchers
// that oracle/ref_cuda/ref_focal.cu never compiles into code, so it needs no definition.
#pragma once
template <typename T>
T THCCeilDiv(T a, T b);
