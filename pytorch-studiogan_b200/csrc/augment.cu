// Differentiable augmentation and consistency-regularisation augmentation on the device, one pass each.
//
// DiffAugment, policy "color,translation,cutout" (reference src/utils/diffaug.py:37-100; Zhao et al. 2020) is a chain of seven
// tensor-op passes over the image batch in the reference.  Per sample it is an affine map of the image followed by an integer
// shift and a box mask, so it collapses into ONE gather kernel given the per-sample parameters (drawn by the host wrapper in
// the reference's RNG order) and the per-sample mean of the input:
//   brightness  x1 = x + b                                     b  = rand - 0.5
//   saturation  x2 = (x1 - m1) * s + m1,  m1 = mean_c(x1)      s  = 2 rand
//   contrast    x3 = (x2 - m2) * c + m2,  m2 = mean_chw(x2)    c  = rand + 0.5     (m2 = mean_chw(x) + b: saturation keeps m1)
//   translation x4[h, w] = x3[h + tx, w + ty] inside the image, else 0            tx, ty in [-H/8, H/8]
//   cutout      x5 = x4 outside the box rows [ox - ch/2, ox - ch/2 + ch) x cols [oy - cw/2, ...) (clamped), 0 inside
// Its adjoint (generator phase: the gradient flows back into the fake images) is the same structure run backwards and needs
// the per-sample mean of the shifted, masked gradient.  params[b] = {b, s, c, tx, ty, ox, oy} as floats (integers exact).
//
// CR / bCR augmentation (src/utils/cr.py:13-50): random horizontal flip, then translation by up to H/8 with REFLECT padding.
#include "common.cuh"

namespace sgb {

// mean over (c, h, w) of each sample: one block per (sample, slice), atomics into out[b] (pre-zeroed); scaled by 1 / n_per.
__global__ void __launch_bounds__(256) sample_mean_kernel(const float* __restrict__ x, long long n_per, float* __restrict__ out,
                                                           int slices) {
  __shared__ float sh[8];
  const int b = blockIdx.x / slices, sl = blockIdx.x % slices;
  const float* xp = x + (long long)b * n_per;
  float acc = 0.f;
  for (long long i = (long long)sl * 256 + threadIdx.x; i < n_per; i += (long long)slices * 256) acc += __ldg(xp + i);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < 8; ++i) t += sh[i];
    atomicAdd(out + b, t / (float)n_per);
  }
}

struct AugGeom { int B, C, H, W, cut_h, cut_w; };

__device__ __forceinline__ bool in_cutout(int h, int w, int ox, int oy, const AugGeom& g) {
  // the reference zeroes mask[clamp(ox - ch/2 + i, 0, H-1), clamp(oy - cw/2 + j, 0, W-1)] for i < ch, j < cw: with
  // 0 <= ox <= H the clamped rows are exactly the contiguous range [max(h0, 0), min(h0 + ch - 1, H - 1)]
  const int h0 = ox - g.cut_h / 2, w0 = oy - g.cut_w / 2;
  const bool hin = h >= max(h0, 0) && h <= min(h0 + g.cut_h - 1, g.H - 1);
  const bool win = w >= max(w0, 0) && w <= min(w0 + g.cut_w - 1, g.W - 1);
  return hin && win;
}

// NCHW fp32, C == 3.  One thread per output pixel (all three channels: the saturation needs the channel mean).
__global__ void __launch_bounds__(256) diffaug_fwd_kernel(const float* __restrict__ x, const float* __restrict__ params,
                                                           const float* __restrict__ mean_x, float* __restrict__ y, AugGeom g,
                                                           int do_color, int do_trans, int do_cut) {
  const long long total = (long long)g.B * g.H * g.W;
  const long long plane = (long long)g.H * g.W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int w = (int)(i % g.W), h = (int)((i / g.W) % g.H), b = (int)(i / plane);
    const float* pr = params + (long long)b * 7;
    const int tx = do_trans ? (int)pr[3] : 0, ty = do_trans ? (int)pr[4] : 0;
    const int hs = h + tx, ws = w + ty;
    float o0 = 0.f, o1 = 0.f, o2 = 0.f;
    const bool cut = do_cut && in_cutout(h, w, (int)pr[5], (int)pr[6], g);
    if (!cut && hs >= 0 && hs < g.H && ws >= 0 && ws < g.W) {
      const float* xp = x + (long long)b * 3 * plane + (long long)hs * g.W + ws;
      float v0 = __ldg(xp), v1 = __ldg(xp + plane), v2 = __ldg(xp + 2 * plane);
      if (do_color) {
        const float bb = pr[0], s = pr[1], c = pr[2];
        v0 += bb; v1 += bb; v2 += bb;
        const float m1 = (v0 + v1 + v2) / 3.0f;
        v0 = (v0 - m1) * s + m1; v1 = (v1 - m1) * s + m1; v2 = (v2 - m1) * s + m1;
        const float m2 = mean_x[b] + bb;
        v0 = (v0 - m2) * c + m2; v1 = (v1 - m2) * c + m2; v2 = (v2 - m2) * c + m2;
      }
      o0 = v0; o1 = v1; o2 = v2;
    }
    float* yp = y + (long long)b * 3 * plane + (long long)h * g.W + w;
    yp[0] = o0; yp[plane] = o1; yp[2 * plane] = o2;
  }
}

// d3[b, :, hs, ws] = dy[b, :, hs - tx, ws - ty] * [not cut], zero where the source lies outside (adjoint of shift + mask);
// written to d3 (same shape) so that its per-sample mean can be taken, then the colour adjoint is applied in place.
__global__ void __launch_bounds__(256) diffaug_bwd_gather_kernel(const float* __restrict__ dy, const float* __restrict__ params,
                                                                  float* __restrict__ d3, AugGeom g, int do_trans, int do_cut) {
  const long long total = (long long)g.B * g.H * g.W;
  const long long plane = (long long)g.H * g.W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ws = (int)(i % g.W), hs = (int)((i / g.W) % g.H), b = (int)(i / plane);
    const float* pr = params + (long long)b * 7;
    const int tx = do_trans ? (int)pr[3] : 0, ty = do_trans ? (int)pr[4] : 0;
    const int h = hs - tx, w = ws - ty;                      // the output pixel that read this source pixel
    float g0 = 0.f, g1 = 0.f, g2 = 0.f;
    if (h >= 0 && h < g.H && w >= 0 && w < g.W && !(do_cut && in_cutout(h, w, (int)pr[5], (int)pr[6], g))) {
      const float* dp = dy + (long long)b * 3 * plane + (long long)h * g.W + w;
      g0 = __ldg(dp); g1 = __ldg(dp + plane); g2 = __ldg(dp + 2 * plane);
    }
    float* op = d3 + (long long)b * 3 * plane + (long long)hs * g.W + ws;
    op[0] = g0; op[plane] = g1; op[2 * plane] = g2;
  }
}

// colour adjoint, in place on d3: d2 = c d3 + (1 - c) mean_chw(d3);  d1 = s d2 + (1 - s) mean_c(d2);  dx = d1.
__global__ void __launch_bounds__(256) diffaug_bwd_color_kernel(float* __restrict__ d, const float* __restrict__ params,
                                                                 const float* __restrict__ mean_d3, AugGeom g) {
  const long long total = (long long)g.B * g.H * g.W;
  const long long plane = (long long)g.H * g.W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int b = (int)(i / plane);
    const long long hw = i % plane;
    const float s = params[(long long)b * 7 + 1], c = params[(long long)b * 7 + 2];
    float* p = d + (long long)b * 3 * plane + hw;
    const float md = mean_d3[b];
    float v0 = c * p[0] + (1.f - c) * md, v1 = c * p[plane] + (1.f - c) * md, v2 = c * p[2 * plane] + (1.f - c) * md;
    const float mc = (v0 + v1 + v2) / 3.0f;
    p[0] = s * v0 + (1.f - s) * mc; p[plane] = s * v1 + (1.f - s) * mc; p[2 * plane] = s * v2 + (1.f - s) * mc;
  }
}

__device__ __forceinline__ int reflect_idx(int i, int n) {     // F.pad(mode='reflect'): -1 -> 1, n -> n - 2
  if (i < 0) i = -i;
  if (i >= n) i = 2 * (n - 1) - i;
  return i;
}

// CR augmentation: y[b, c, h, w] = xf[b, c, reflect(h + tx), reflect(w + ty)], xf = x flipped along w where flip[b].
__global__ void __launch_bounds__(256) cr_aug_kernel(const float* __restrict__ x, const uint8_t* __restrict__ flip,
                                                      const int* __restrict__ tx, const int* __restrict__ ty, float* __restrict__ y,
                                                      int B, int C, int H, int W) {
  const long long total = (long long)B * C * H * W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int w = (int)(i % W), h = (int)((i / W) % H);
    const long long bc = i / ((long long)H * W);
    const int b = (int)(bc / C);
    const int hs = reflect_idx(h + (tx ? tx[b] : 0), H);
    int ws = reflect_idx(w + (ty ? ty[b] : 0), W);
    if (flip && flip[b]) ws = W - 1 - ws;
    y[i] = __ldg(x + bc * H * W + (long long)hs * W + ws);
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_sample_mean(const float* x, int32_t B, int64_t n_per, float* out, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && out && B > 0 && n_per > 0);
  SGB_CUDA(cudaMemsetAsync(out, 0, sizeof(float) * (size_t)B, stream));
  int slices = (int)((n_per + 256 * 64 - 1) / (256 * 64));
  if (slices < 1) slices = 1;
  if (slices > 64) slices = 64;
  sample_mean_kernel<<<B * slices, 256, 0, stream>>>(x, n_per, out, slices);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_diffaug_fwd(const float* x, const float* params, const float* mean_x, float* y, int32_t B, int32_t H, int32_t W,
                               int32_t do_color, int32_t do_translation, int32_t do_cutout, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && params && y && B > 0 && H > 0 && W > 0 && (!do_color || mean_x));
  AugGeom g = {B, 3, H, W, (int)(H * 0.5 + 0.5), (int)(W * 0.5 + 0.5)};
  diffaug_fwd_kernel<<<ew_blocks((long long)B * H * W), 256, 0, stream>>>(x, params, mean_x, y, g, do_color, do_translation, do_cutout);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_diffaug_bwd(const float* dy, const float* params, float* dx, float* mean_ws, int32_t B, int32_t H, int32_t W,
                               int32_t do_color, int32_t do_translation, int32_t do_cutout, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dy && params && dx && B > 0 && H > 0 && W > 0 && (!do_color || mean_ws));
  AugGeom g = {B, 3, H, W, (int)(H * 0.5 + 0.5), (int)(W * 0.5 + 0.5)};
  diffaug_bwd_gather_kernel<<<ew_blocks((long long)B * H * W), 256, 0, stream>>>(dy, params, dx, g, do_translation, do_cutout);
  SGB_LAUNCH_CHECK();
  if (do_color) {
    int rc = sgb_sample_mean(dx, B, (int64_t)3 * H * W, mean_ws, stream_);
    if (rc) return rc;
    diffaug_bwd_color_kernel<<<ew_blocks((long long)B * H * W), 256, 0, stream>>>(dx, params, mean_ws, g);
    SGB_LAUNCH_CHECK();
  }
  return SGB_OK;
}

extern "C" int sgb_cr_aug(const float* x, const uint8_t* flip, const int32_t* tx, const int32_t* ty, float* y, int32_t B, int32_t C,
                          int32_t H, int32_t W, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && B > 0 && C > 0 && H > 1 && W > 1);
  cr_aug_kernel<<<ew_blocks((long long)B * C * H * W), 256, 0, stream>>>(x, flip, tx, ty, y, B, C, H, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
