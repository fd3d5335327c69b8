// Helpers shared by every translation unit of libsgb200.  Host side: error codes, launch checks, the grid size of the
// grid-stride kernels, TMA tensor-map encoding resolved through the runtime (no link-time libcuda dependency, so the
// library also loads on a GPU-less box for the C-ABI export test).  Device side: the packed bf16 pair / 16-byte vector
// format, warp reductions, and the 2x2 block of a nearest x2 upsample / 2x2 pool.
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

// Blocks of 256 threads for a grid-stride kernel over total_threads work items: one per 256 items, at most 16 per SM.
inline int ew_blocks(long long total_threads) {
  long long b = (total_threads + 255) / 256;
  const long long cap = 16LL * sm_count();
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (int)b;
}

// A bf16 pair in one 32-bit word, the first element in the low half.
__device__ __forceinline__ float bf16_bits_lo(uint32_t u) { return __uint_as_float(u << 16); }
__device__ __forceinline__ float bf16_bits_hi(uint32_t u) { return __uint_as_float(u & 0xFFFF0000u); }
__device__ __forceinline__ uint32_t pack_bf16x2(float a, float b) {
  __nv_bfloat162 t = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&t);
}

// 8 consecutive bf16 channels in one 16-byte vector (the streaming kernels' unit of access).
__device__ __forceinline__ void unpack8(const uint4& r, float (&f)[8]) {
  f[0] = bf16_bits_lo(r.x); f[1] = bf16_bits_hi(r.x);
  f[2] = bf16_bits_lo(r.y); f[3] = bf16_bits_hi(r.y);
  f[4] = bf16_bits_lo(r.z); f[5] = bf16_bits_hi(r.z);
  f[6] = bf16_bits_lo(r.w); f[7] = bf16_bits_hi(r.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(pack_bf16x2(f[0], f[1]), pack_bf16x2(f[2], f[3]), pack_bf16x2(f[4], f[5]), pack_bf16x2(f[6], f[7]));
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Pixel p = (b * h + y) * w + x of a [B][h][w] grid covers the 2x2 block {q, q + 1, q + 2w, q + 2w + 1} of the [B][2h][2w]
// grid, q = (b * 2h + 2y) * 2w + 2x = 4p - 2x (nearest x2 upsample, 2x2 pooling).  x = p % w is the caller's.
__device__ __forceinline__ void quad2x2(long long p, int x, int w, long long (&q)[4]) {
  q[0] = 4 * p - 2 * x;
  q[1] = q[0] + 1;
  q[2] = q[0] + 2 * w;
  q[3] = q[0] + 2 * w + 1;
}

}  // namespace sgb
