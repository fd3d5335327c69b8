// Host-side helpers shared by every translation unit of libsgb200: error codes, launch checks,
// TMA tensor-map encoding resolved through the runtime (no link-time libcuda dependency, so the
// library also loads on a GPU-less box for the C-ABI export test).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sgb200.h"

namespace sgb {

typedef __nv_bfloat16 bf16;

inline int cuda_fail(cudaError_t e, const char* what, const char* file, int line) {
  if (e == cudaSuccess) return 0;
  fprintf(stderr, "[sgb200] CUDA error %d (%s) at %s:%d in %s\n", (int)e, cudaGetErrorString(e), file, line, what);
  return SGB_ERR_CUDA;
}
#define SGB_CUDA(call)                                                   \
  do {                                                                   \
    int _rc = ::sgb::cuda_fail((call), #call, __FILE__, __LINE__);      \
    if (_rc) return _rc;                                                 \
  } while (0)
#define SGB_LAUNCH_CHECK() SGB_CUDA(cudaGetLastError())
#define SGB_REQUIRE(cond)                                                                        \
  do {                                                                                           \
    if (!(cond)) {                                                                               \
      fprintf(stderr, "[sgb200] invalid argument: %s at %s:%d\n", #cond, __FILE__, __LINE__);    \
      return SGB_ERR_ARG;                                                                        \
    }                                                                                            \
  } while (0)

typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

inline PFN_encodeTiled get_encode_tiled() {
  static PFN_encodeTiled fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = reinterpret_cast<PFN_encodeTiled>(p);
  return fn;
}

// bf16 tensor map, rank <= 5, SWIZZLE_128B, zero OOB fill. dims/box innermost first; strides in BYTES for dims 1..rank-1.
inline int make_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box, CUtensorMapSwizzle swz = CU_TENSOR_MAP_SWIZZLE_128B) {
  PFN_encodeTiled enc = get_encode_tiled();
  if (!enc) {
    fprintf(stderr, "[sgb200] cuTensorMapEncodeTiled unavailable (no CUDA driver?)\n");
    return SGB_ERR_CUDA;
  }
  cuuint64_t gd[5];
  cuuint64_t gs[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gd[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
    if (i > 0) gs[i - 1] = strides_bytes[i - 1];
  }
  CUresult r = enc(out, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void*>(base), gd, gs, bx, es,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    fprintf(stderr, "[sgb200] cuTensorMapEncodeTiled failed: %d (rank %d dims %llu %llu %llu %llu box %u %u %u %u)\n", (int)r,
            rank, (unsigned long long)gd[0], (unsigned long long)(rank > 1 ? gd[1] : 0),
            (unsigned long long)(rank > 2 ? gd[2] : 0), (unsigned long long)(rank > 3 ? gd[3] : 0), bx[0],
            rank > 1 ? bx[1] : 0, rank > 2 ? bx[2] : 0, rank > 3 ? bx[3] : 0);
    return SGB_ERR_CUDA;
  }
  return 0;
}

// NHWC bf16 activation [B][H][W][C] with channel stride cstride (elements); box = 64 channels x tw x th x nb pixels.
inline int make_act_tmap(CUtensorMap* m, const void* base, int B, int H, int W, int C, long long cstride, int tw, int th, int nb) {
  uint64_t dims[4] = {(uint64_t)C, (uint64_t)W, (uint64_t)H, (uint64_t)B};
  uint64_t strides[3] = {(uint64_t)cstride * 2, (uint64_t)cstride * 2 * W, (uint64_t)cstride * 2 * W * H};
  uint32_t box[4] = {64, (uint32_t)tw, (uint32_t)th, (uint32_t)nb};
  return make_tmap_bf16(m, base, 4, dims, strides, box);
}

// Launches Kernel with the full 227 KiB of opt-in shared memory available; the attribute is set once per kernel.
template <auto Kernel, typename... Args>
inline int launch_kernel(int grid, int threads, size_t smem, cudaStream_t stream, const Args&... args) {
  static bool attr_set = false;
  if (!attr_set) {
    SGB_CUDA(cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    attr_set = true;
  }
  Kernel<<<grid, threads, smem, stream>>>(args...);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

inline int sm_count() {
  static int n = 0;
  if (n) return n;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
  return n;
}

}  // namespace sgb
