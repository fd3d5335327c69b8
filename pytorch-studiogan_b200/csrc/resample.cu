// Stride-2 helpers for the DCGAN layers (src/models/deep_conv.py:20,140: ConvTranspose2d / Conv2d with kernel 4, stride 2,
// padding 1), which run on the stride-1 wgmma conv engine through two exact identities:
//   conv_transpose(x, W; k4 s2 p1)  =  conv_same(zero_stuff(x), W~; k4, taps offset -2..+1)      zero_stuff: y[2h,2w] = x[h,w]
//   conv(x, W; k4 s2 p1)            =  subsample(conv_same(x, W; k4, taps offset -1..+2))        subsample:  y[h,w] = x[2h,2w]
// The sub-sampling is the conv engine's own out_sub = 2 store mode; its adjoint -- needed for the strided conv's gradients
// and as the transposed conv's input -- is the zero-stuffing below.  NHWC bf16, 8 channels (16 bytes) per thread.
#include "common.cuh"

namespace sgb {

// out[B][2H][2W][C]: out[b, 2h, 2w, :] = x[b, h, w, :], zero elsewhere.
__global__ void __launch_bounds__(256) zero_stuff2_kernel(const bf16* __restrict__ x, long long xs, bf16* __restrict__ y, long long ys,
                                                           int B, int H, int W, int C) {
  const int VG = C >> 3;
  const long long total = (long long)B * 2 * H * 2 * W * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;                       // output pixel
    const int ow = (int)(p % (2 * W)), oh = (int)((p / (2 * W)) % (2 * H));
    const int b = (int)(p / ((long long)4 * H * W));
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (((ow | oh) & 1) == 0)
      v = __ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + (oh >> 1)) * W + (ow >> 1)) * xs) + g);
    reinterpret_cast<uint4*>(y + p * ys)[g] = v;
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_zero_stuff2(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t H, int32_t W, int32_t C,
                               sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && ys % 8 == 0);
  zero_stuff2_kernel<<<ew_blocks((long long)B * 4 * H * W * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (bf16*)y, ys, B, H, W, C);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
