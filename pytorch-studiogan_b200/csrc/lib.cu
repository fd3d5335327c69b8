// Library identity and device probe.
#include "common.cuh"

extern "C" int sgb_abi_version(void) { return 1; }

extern "C" int sgb_device_check(void) {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) { cudaGetLastError(); return SGB_ERR_CUDA; }
  int major = 0, minor = 0;
  if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return SGB_ERR_CUDA;
  if (cudaDeviceGetAttribute(&minor, cudaDevAttrComputeCapabilityMinor, dev) != cudaSuccess) return SGB_ERR_CUDA;
  if (major != 9 || minor != 0) {
    fprintf(stderr, "[sgb200] device is sm_%d%d; this library is built for sm_90a only\n", major, minor);
    return SGB_ERR_UNSUPPORTED;
  }
  return SGB_OK;
}

// Binds the calling host thread to ``device`` (primary context made current).  PyTorch's autograd engine runs backward
// on its own threads, where no context is current until some runtime call binds one; driver-level helpers used here
// (cuTensorMapEncodeTiled) need a current context, so the Python layer calls this once per thread.
extern "C" int sgb_bind_device(int32_t device) {
  SGB_CUDA(cudaSetDevice(device));
  SGB_CUDA(cudaFree(0));
  return SGB_OK;
}
