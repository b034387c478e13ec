#include "common.cuh"

namespace smb {
static thread_local char g_err[512] = "";
void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
}  // namespace smb

extern "C" const char* smb_last_error(void) { return smb::g_err; }
extern "C" int smb_version(void) { return 100; }

extern "C" int smb_check_device(void) {
  int dev = 0;
  SMB_CUDA_OK(cudaGetDevice(&dev));
  cudaDeviceProp p;
  SMB_CUDA_OK(cudaGetDeviceProperties(&p, dev));
  if (p.major != 9 || p.minor != 0) {
    smb::set_error("device %d is sm_%d%d; this library contains sm_90a code only", dev, p.major, p.minor);
    return SMB_EARCH;
  }
  return SMB_OK;
}
