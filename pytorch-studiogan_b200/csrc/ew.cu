// Streaming element-wise / small-reduction kernels around the conv engine (all HBM-bound, 16-byte vectors on NHWC bf16).
// Reference call sites: ReLU / AvgPool2d / nearest-upsample / residual add in src/models/big_resnet_deep_legacy.py:49-73,
// 210-229,334-345; MaxPool2d + Softmax + sigma*attn in src/utils/ops.py:79-103; tanh at big_resnet_deep_legacy.py:183;
// Adam (src/config.py:541-563, eps 1e-6) and Ema.update (src/utils/ema.py:27-40).
#include "common.cuh"

namespace sgb {

// out = act(a*x + b*y) over [npix][C] with per-tensor channel strides; a may come from a device scalar.
// act: 0 none, 1 relu.  y may be null (b ignored).  mask (optional): out = mask > 0 ? out : 0.
__global__ void __launch_bounds__(256) axpby_kernel(const bf16* __restrict__ x, long long xs, const bf16* __restrict__ y,
                                                     long long ys, const bf16* __restrict__ mask, long long ms,
                                                     bf16* __restrict__ out, long long os, long long npix, int C, float a,
                                                     const float* __restrict__ a_dev, float b, int act) {
  const int VG = C >> 3;
  if (a_dev) a *= __ldg(a_dev);
  const long long total = npix * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    float f[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + p * xs) + g), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] *= a;
    if (y) {
      float t[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(y + p * ys) + g), t);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaf(b, t[j], f[j]);
    }
    if (act == 1) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
    }
    if (mask) {
      float t[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(mask + p * ms) + g), t);
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = t[j] > 0.f ? f[j] : 0.f;
    }
    reinterpret_cast<uint4*>(out + p * os)[g] = pack8(f);
  }
}

// 2x2 pooling.  mode 0: average, 1: max, 2: sum.  One thread = 8 channels of one OUTPUT pixel.
__global__ void __launch_bounds__(256) pool2_fwd_kernel(const bf16* __restrict__ x, long long xs, bf16* __restrict__ y,
                                                         long long ys, int B, int Ho, int Wo, int C, int mode) {
  const int VG = C >> 3;
  const long long total = (long long)B * Ho * Wo * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    long long qs[4];
    quad2x2(p, (int)(p % Wo), Wo, qs);
    float f[4][8], o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) unpack8(__ldg(reinterpret_cast<const uint4*>(x + qs[k] * xs) + g), f[k]);
#pragma unroll
    for (int j = 0; j < 8; ++j)
      o[j] = mode == 1 ? fmaxf(fmaxf(f[0][j], f[1][j]), fmaxf(f[2][j], f[3][j]))
                       : (mode == 0 ? 0.25f : 1.0f) * (f[0][j] + f[1][j] + f[2][j] + f[3][j]);  // 0 average, 2 sum
    reinterpret_cast<uint4*>(y + p * ys)[g] = pack8(o);
  }
}

// a0 = relu(x) at full resolution AND y = avgpool2(a0) in one pass (entry of a down-sampling discriminator block: the skip
// path pools the rectified input, big_resnet_deep_legacy.py:211-224); saves re-reading a0 for the pooling.
__global__ void __launch_bounds__(256) relu_pool2_kernel(const bf16* __restrict__ x, long long xs, bf16* __restrict__ a0,
                                                          long long as_, bf16* __restrict__ y, long long ys, int B, int Ho, int Wo,
                                                          int C) {
  const int VG = C >> 3;
  const long long total = (long long)B * Ho * Wo * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    long long qs[4];
    quad2x2(p, (int)(p % Wo), Wo, qs);
    float f[4][8], o[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) unpack8(__ldg(reinterpret_cast<const uint4*>(x + qs[k] * xs) + g), f[k]);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int k = 0; k < 4; ++k) f[k][j] = fmaxf(f[k][j], 0.f);
      o[j] = 0.25f * (f[0][j] + f[1][j] + f[2][j] + f[3][j]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) reinterpret_cast<uint4*>(a0 + qs[k] * as_)[g] = pack8(f[k]);
    reinterpret_cast<uint4*>(y + p * ys)[g] = pack8(o);
  }
}

// Backward of 2x2 pooling, one thread = 8 channels of one OUTPUT-resolution pixel, writes the 4 input-resolution pixels.
// mode 0 (avg): dx = 0.25*dy; mode 1 (max): dy routed to the first maximum in (h,w) scan order (torch MaxPool2d).
// Optional: add (same layout as dx) is summed in, relu_src masks the result where relu_src <= 0.
template <bool BITS>
__global__ void __launch_bounds__(256) pool2_bwd_kernel(const bf16* __restrict__ dy, long long dys, const bf16* __restrict__ x,
                                                         long long xs, const bf16* __restrict__ add, long long adds,
                                                         const bf16* __restrict__ relu_src, long long rs, bf16* __restrict__ dx,
                                                         long long dxs, int B, int Ho, int Wo, int C, int mode) {
  const int VG = C >> 3;
  const long long total = (long long)B * Ho * Wo * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    long long qs[4];
    quad2x2(p, (int)(p % Wo), Wo, qs);
    float d[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(dy + p * dys) + g), d);
    float o[4][8];
    if (mode == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
#pragma unroll
        for (int j = 0; j < 8; ++j) o[k][j] = 0.25f * d[j];
    } else {
      float f[4][8];
#pragma unroll
      for (int k = 0; k < 4; ++k) unpack8(__ldg(reinterpret_cast<const uint4*>(x + qs[k] * xs) + g), f[k]);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int arg = 0;
        float m = f[0][j];
#pragma unroll
        for (int k = 1; k < 4; ++k)
          if (f[k][j] > m) { m = f[k][j]; arg = k; }
#pragma unroll
        for (int k = 0; k < 4; ++k) o[k][j] = (k == arg) ? d[j] : 0.f;
      }
    }
    // issue every operand load (packed) before the arithmetic: up to eight 16-byte loads in flight per thread
    uint4 ra[4], rr[4];
    if (add) {
#pragma unroll
      for (int k = 0; k < 4; ++k) ra[k] = __ldg(reinterpret_cast<const uint4*>(add + qs[k] * adds) + g);
    }
    unsigned char rb[4];
    if (BITS) {                    // bit planes: one byte = these 8 channels of one pixel
#pragma unroll
      for (int k = 0; k < 4; ++k) rb[k] = __ldg(reinterpret_cast<const unsigned char*>(relu_src) + qs[k] * VG + g);
    } else if (relu_src) {
#pragma unroll
      for (int k = 0; k < 4; ++k) rr[k] = __ldg(reinterpret_cast<const uint4*>(relu_src + qs[k] * rs) + g);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if (add) {
        float t[8];
        unpack8(ra[k], t);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[k][j] += t[j];
      }
      if (BITS) {
#pragma unroll
        for (int j = 0; j < 8; ++j) o[k][j] = ((rb[k] >> j) & 1) ? o[k][j] : 0.f;
      } else if (relu_src) {
        float t[8];
        unpack8(rr[k], t);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[k][j] = t[j] > 0.f ? o[k][j] : 0.f;
      }
      reinterpret_cast<uint4*>(dx + qs[k] * dxs)[g] = pack8(o[k]);
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Discriminator head (src/models/big_resnet_deep_legacy.py:346-349,366-368; the same lines close big_resnet.py and
// resnet.py): adv[b] = <h_b, w1> / sigma1 + b1 + <h_b, E[y_b]> / sigmaE on the fp32 sum-pooled features.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dhead_fwd_kernel(const float* __restrict__ h, const float* __restrict__ w1,
                                                        const float* __restrict__ sigma1, const float* __restrict__ b1,
                                                        const float* __restrict__ E, const float* __restrict__ sigmaE,
                                                        const long long* __restrict__ labels, int B, int C, float* __restrict__ adv) {
  const int lane = threadIdx.x & 31;
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (b >= B) return;
  const float* hp = h + (size_t)b * C;
  const float* ep = E ? E + (size_t)labels[b] * C : nullptr;
  float a1 = 0.f, a2 = 0.f;
  for (int c = lane; c < C; c += 32) {
    const float hv = __ldg(hp + c);
    a1 = fmaf(hv, __ldg(w1 + c), a1);
    if (ep) a2 = fmaf(hv, __ldg(ep + c), a2);
  }
  a1 = warp_sum(a1);
  a2 = warp_sum(a2);
  if (lane == 0) {
    float r = sigma1 ? a1 / __ldg(sigma1) : a1;
    if (b1) r += __ldg(b1);
    if (ep) r += sigmaE ? a2 / __ldg(sigmaE) : a2;
    adv[b] = r;
  }
}

// dh[b][c] = dadv[b] * (w1[c] / sigma1 + E[y_b][c] / sigmaE); gE[y_b][c] += dadv[b] * h[b][c] (gradient of the EFFECTIVE table)
__global__ void __launch_bounds__(256) dhead_bwd_rows_kernel(const float* __restrict__ dadv, const float* __restrict__ h,
                                                             const float* __restrict__ w1, const float* __restrict__ sigma1,
                                                             const float* __restrict__ E, const float* __restrict__ sigmaE,
                                                             const long long* __restrict__ labels, int B, int C,
                                                             float* __restrict__ dh, float* __restrict__ gE) {
  const int b = blockIdx.y;
  const float d = __ldg(dadv + b);
  const float i1 = sigma1 ? 1.f / __ldg(sigma1) : 1.f;
  const float iE = sigmaE ? 1.f / __ldg(sigmaE) : 1.f;
  const long long y = E ? labels[b] : 0;
  for (int c = blockIdx.x * 256 + threadIdx.x; c < C; c += gridDim.x * 256) {
    float w = __ldg(w1 + c) * i1;
    if (E) w = fmaf(__ldg(E + (size_t)y * C + c), iE, w);
    if (dh) dh[(size_t)b * C + c] = d * w;
    if (E && gE) atomicAdd(gE + (size_t)y * C + c, d * __ldg(h + (size_t)b * C + c));
  }
}

// gw1[c] = sum_b dadv[b] * h[b][c] (gradient of the effective weight row), db1 = sum_b dadv[b]
__global__ void __launch_bounds__(256) dhead_bwd_w_kernel(const float* __restrict__ dadv, const float* __restrict__ h, int B, int C,
                                                          float* __restrict__ gw1, float* __restrict__ db1) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c < C) {
    float acc = 0.f;
    for (int b = 0; b < B; ++b) acc = fmaf(__ldg(dadv + b), __ldg(h + (size_t)b * C + c), acc);
    gw1[c] = acc;
  }
  if (db1 && blockIdx.x == 0 && threadIdx.x == 0) {
    float s = 0.f;
    for (int b = 0; b < B; ++b) s += __ldg(dadv + b);
    *db1 = s;
  }
}

// out[row] = sum_c x[row][c] * y[row][c]: delta = rowsum(dO * O) of the softmax backward; one warp per row.
__global__ void __launch_bounds__(256) rowdot_kernel(const bf16* __restrict__ x, long long xs, const bf16* __restrict__ y, long long ys,
                                                     long long rows, int C, float* __restrict__ out) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* xp = reinterpret_cast<const uint4*>(x + row * xs);
  const uint4* yp = reinterpret_cast<const uint4*>(y + row * ys);
  float acc = 0.f;
  for (int i = lane; i < (C >> 3); i += 32) {
    float a[8], b[8];
    unpack8(__ldg(xp + i), a);
    unpack8(__ldg(yp + i), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(a[j], b[j], acc);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[row] = acc;
}

// Row softmax over the last dim (bf16 in/out, fp32 math), one warp per row, in place allowed.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const bf16* __restrict__ s, bf16* __restrict__ p, long long rows, int n) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* sp = reinterpret_cast<const uint4*>(s + row * n);
  uint4* pp = reinterpret_cast<uint4*>(p + row * n);
  const int nv = n >> 3;
  float m = -INFINITY;
  for (int i = lane; i < nv; i += 32) {
    float f[8];
    unpack8(__ldg(sp + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) m = fmaxf(m, f[j]);
  }
  m = warp_max(m);
  float z = 0.f;
  for (int i = lane; i < nv; i += 32) {
    float f[8];
    unpack8(__ldg(sp + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) z += __expf(f[j] - m);
  }
  z = warp_sum(z);
  const float inv = 1.f / z;
  for (int i = lane; i < nv; i += 32) {
    float f[8];
    unpack8(__ldg(sp + i), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = __expf(f[j] - m) * inv;
    pp[i] = pack8(f);
  }
}

// dS = P * (dP - sum_j dP_j P_j), rowwise; writes into ds (may alias dp).
__global__ void __launch_bounds__(256) softmax_bwd_rows_kernel(const bf16* __restrict__ p, const bf16* __restrict__ dp,
                                                                bf16* __restrict__ ds, long long rows, int n) {
  const int lane = threadIdx.x & 31;
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const uint4* pp = reinterpret_cast<const uint4*>(p + row * n);
  const uint4* dpp = reinterpret_cast<const uint4*>(dp + row * n);
  uint4* dsp = reinterpret_cast<uint4*>(ds + row * n);
  const int nv = n >> 3;
  float dot = 0.f;
  for (int i = lane; i < nv; i += 32) {
    float a[8], b[8];
    unpack8(__ldg(pp + i), a);
    unpack8(__ldg(dpp + i), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) dot = fmaf(a[j], b[j], dot);
  }
  dot = warp_sum(dot);
  for (int i = lane; i < nv; i += 32) {
    float a[8], b[8];
    unpack8(__ldg(pp + i), a);
    unpack8(dpp[i], b);
#pragma unroll
    for (int j = 0; j < 8; ++j) b[j] = a[j] * (b[j] - dot);
    dsp[i] = pack8(b);
  }
}

// sum over a contiguous bf16 buffer of x*y -> fp32 scalar (atomic).
__global__ void __launch_bounds__(256) dot_kernel(const bf16* __restrict__ x, const bf16* __restrict__ y, long long nvec,
                                                   float* __restrict__ out) {
  __shared__ float sh[8];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < nvec; i += (long long)gridDim.x * 256) {
    float a[8], b[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x) + i), a);
    unpack8(__ldg(reinterpret_cast<const uint4*>(y) + i), b);
#pragma unroll
    for (int j = 0; j < 8; ++j) acc = fmaf(a[j], b[j], acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x < 8) {
    float r = sh[threadIdx.x];
    r += __shfl_xor_sync(0xffu, r, 4);
    r += __shfl_xor_sync(0xffu, r, 2);
    r += __shfl_xor_sync(0xffu, r, 1);
    if (threadIdx.x == 0) atomicAdd(out, r);
  }
}

// h[b,c] = sum_{hw} act(x[b,hw,c]) (fp32), act = relu if relu.  grid = (pixel chunks, B).
__global__ void __launch_bounds__(256) sum_hw_kernel(const bf16* __restrict__ x, long long xs, int HW, int C, int relu,
                                                      float* __restrict__ h, int pix_per_block) {
  extern __shared__ float acc_s[];
  const int b = blockIdx.y;
  for (int i = threadIdx.x; i < C; i += 256) acc_s[i] = 0.f;
  __syncthreads();
  const int VG = C >> 3;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(p0 + pix_per_block, HW);
  for (int g = threadIdx.x; g < VG; g += 256) {
    float a[8] = {0, 0, 0, 0, 0, 0, 0, 0};
    for (int hw = p0; hw < p1; ++hw) {
      float f[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(x + ((long long)b * HW + hw) * xs) + g), f);
#pragma unroll
      for (int j = 0; j < 8; ++j) a[j] += relu ? fmaxf(f[j], 0.f) : f[j];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) acc_s[g * 8 + j] += a[j];
  }
  __syncthreads();
  for (int i = threadIdx.x; i < C; i += 256) atomicAdd(h + (size_t)b * C + i, acc_s[i]);
}

// dx[b,hw,c] = dh[b,c] * (relu ? x > 0 : 1)
__global__ void __launch_bounds__(256) sum_hw_bwd_kernel(const float* __restrict__ dh, const bf16* __restrict__ x, long long xs,
                                                          bf16* __restrict__ dx, long long dxs, int B, int HW, int C, int relu) {
  const int VG = C >> 3;
  const long long total = (long long)B * HW * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    const int b = (int)(p / HW);
    float f[8], o[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + p * xs) + g), f);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float d = __ldg(dh + (size_t)b * C + g * 8 + j);
      o[j] = (!relu || f[j] > 0.f) ? d : 0.f;
    }
    reinterpret_cast<uint4*>(dx + p * dxs)[g] = pack8(o);
  }
}

// NCHW fp32 image -> NHWC bf16 with the channel dim zero-padded to Cp (multiple of 8).
__global__ void __launch_bounds__(256) img_to_nhwc_kernel(const float* __restrict__ img, bf16* __restrict__ out, int B, int C,
                                                           int HW, int Cp) {
  const long long total = (long long)B * HW;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
    const int b = (int)(p / HW), hw = (int)(p % HW);
    for (int c0 = 0; c0 < Cp; c0 += 8) {
      float f[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = (c0 + j < C) ? __ldg(img + ((size_t)b * C + c0 + j) * HW + hw) : 0.f;
      reinterpret_cast<uint4*>(out + p * Cp + c0)[0] = pack8(f);
    }
  }
}

// NHWC (fp32 or bf16, channel stride cs) -> NCHW fp32 for the first C channels; act: 0 none, 1 tanh.
__global__ void __launch_bounds__(256) nhwc_to_img_kernel(const void* __restrict__ in, int in_fp32, long long cs,
                                                           float* __restrict__ img, int B, int C, int HW, int act) {
  const long long total = (long long)B * HW;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
    const int b = (int)(p / HW), hw = (int)(p % HW);
    for (int c = 0; c < C; ++c) {
      float v = in_fp32 ? reinterpret_cast<const float*>(in)[p * cs + c]
                        : __bfloat162float(reinterpret_cast<const bf16*>(in)[p * cs + c]);
      if (act == 1) v = tanhf(v);
      img[((size_t)b * C + c) * HW + hw] = v;
    }
  }
}

// d(pre-tanh) in NHWC bf16 (padded to Cp) from d(image) and the tanh output, both NCHW fp32:  d * (1 - y^2).
// With y == null it is a plain NCHW fp32 -> NHWC bf16 gradient re-layout.
__global__ void __launch_bounds__(256) img_grad_to_nhwc_kernel(const float* __restrict__ dimg, const float* __restrict__ y,
                                                                bf16* __restrict__ out, int B, int C, int HW, int Cp) {
  const long long total = (long long)B * HW;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
    const int b = (int)(p / HW), hw = (int)(p % HW);
    for (int c0 = 0; c0 < Cp; c0 += 8) {
      float f[8];
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float v = 0.f;
        if (c0 + j < C) {
          const size_t idx = ((size_t)b * C + c0 + j) * HW + hw;
          v = __ldg(dimg + idx);
          if (y) { const float t = __ldg(y + idx); v *= (1.f - t * t); }
        }
        f[j] = v;
      }
      reinterpret_cast<uint4*>(out + p * Cp + c0)[0] = pack8(f);
    }
  }
}

// 3x3 / pad-1 patch gather for 3-channel images ("im2col27"): out[b,h,w, t*3+c] = src[b, c, h+th-1, w+tw-1] (zero outside),
// t = th*3+tw, k = 27..31 zero.  Turns the 3 -> C input convolution of the discriminators (src/models/*: input_conv /
// DiscOptBlock conv) and the dgrad of the generators' C -> 3 output convolution into a K = 32 1x1 GEMM for the tensor
// core (a 3-channel NHWC tensor would waste 8x of every TMA box and MMA).
// src: NCHW fp32 (src_nchw = 1) or NHWC bf16 with channel stride cs (first 3 channels used).
__global__ void __launch_bounds__(256) col27_kernel(const void* __restrict__ src, int src_nchw, long long cs, bf16* __restrict__ out,
                                                     int B, int H, int W) {
  const long long total = (long long)B * H * W;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
    const int w = (int)(p % W), h = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
    float v[4][8];                                   // k = t * 3 + c at v[k / 8][k % 8]
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h + t / 3 - 1, ww = w + t % 3 - 1;
      const bool in = (hh >= 0) && (hh < H) && (ww >= 0) && (ww < W);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float x = 0.f;
        if (in) {
          if (src_nchw) x = __ldg(reinterpret_cast<const float*>(src) + (((long long)b * 3 + c) * H + hh) * W + ww);
          else x = __bfloat162float(reinterpret_cast<const bf16*>(src)[(((long long)b * H + hh) * W + ww) * cs + c]);
        }
        v[(t * 3 + c) / 8][(t * 3 + c) % 8] = x;
      }
    }
#pragma unroll
    for (int k = 27; k < 32; ++k) v[3][k - 24] = 0.f;
#pragma unroll
    for (int j = 0; j < 4; ++j) reinterpret_cast<uint4*>(out + p * 32)[j] = pack8(v[j]);
  }
}

// Adjoint of col27: dimg[b,c,h,w] = sum_t dcol[b, h-th+1, w-tw+1, t*3+c]  (NCHW fp32 result).
__global__ void __launch_bounds__(256) col27_bwd_kernel(const bf16* __restrict__ dcol, float* __restrict__ dimg, int B, int H, int W) {
  const long long total = (long long)B * H * W;
  for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
    const int w = (int)(p % W), h = (int)((p / W) % H), b = (int)(p / ((long long)W * H));
    float acc[3] = {0.f, 0.f, 0.f};
#pragma unroll
    for (int t = 0; t < 9; ++t) {
      const int hh = h - (t / 3) + 1, ww = w - (t % 3) + 1;
      if (hh >= 0 && hh < H && ww >= 0 && ww < W) {
        const bf16* q = dcol + (((long long)b * H + hh) * W + ww) * 32 + t * 3;
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] += __bfloat162float(q[c]);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) dimg[(((long long)b * 3 + c) * H + h) * W + w] = acc[c];
  }
}

// 3x3 pooling of the Inception feature extractor (src/metrics/inception_net.py:81-107,135-249): max (stride 2, no padding:
// nn.MaxPool2d(3, 2); stride 1, padding 1 in FIDInceptionE_2) or average with count_include_pad=False (stride 1, padding 1).
__global__ void __launch_bounds__(256) pool3x3_kernel(const bf16* __restrict__ x, long long xs, bf16* __restrict__ y, long long ys,
                                                       int B, int H, int W, int Ho, int Wo, int C, int stride, int pad, int mode) {
  const int VG = C >> 3;
  const long long total = (long long)B * Ho * Wo * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    const int wo = (int)(p % Wo), ho = (int)((p / Wo) % Ho), b = (int)(p / ((long long)Wo * Ho));
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = mode == 1 ? -INFINITY : 0.f;
    int cnt = 0;
    for (int kh = 0; kh < 3; ++kh) {
      const int h = ho * stride + kh - pad;
      if (h < 0 || h >= H) continue;
      for (int kw = 0; kw < 3; ++kw) {
        const int w = wo * stride + kw - pad;
        if (w < 0 || w >= W) continue;
        float f[8];
        unpack8(__ldg(reinterpret_cast<const uint4*>(x + (((long long)b * H + h) * W + w) * xs) + g), f);
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = mode == 1 ? fmaxf(acc[j], f[j]) : acc[j] + f[j];
        ++cnt;
      }
    }
    if (mode == 0) {
      const float inv = 1.f / (float)cnt;
#pragma unroll
      for (int j = 0; j < 8; ++j) acc[j] *= inv;
    }
    reinterpret_cast<uint4*>(y + p * ys)[g] = pack8(acc);
  }
}

// Fused evaluation pre-processing (src/utils/ops.py:251-263 + src/utils/resize.py:83-91 "legacy" + InceptionV3_tf mean/std):
// float image in [-1,1] -> uint8 quantisation ((255*(x+1)/2 + 0.5) clamped, truncated) -> bilinear resize to S x S
// (align_corners = False, on the uint8 values, clipped to [0,255]) -> x/255 -> (x - 0.5)/0.5, all on the device; the
// reference does this on the host with a Python loop per image and two PCIe crossings.
// Output: the 3x3 / stride-2 / valid patches of the resized image, [B, So, So, 32] bf16 (So = (S-3)/2+1), i.e. the operand
// of Inception's first convolution as a K = 32 GEMM; also (optionally) the quantised uint8 image for bit-exact checks.
__device__ __forceinline__ float quant_u8(float x) {
  float q = 255.0f * ((x + 1.0f) / 2.0f) + 0.5f;
  q = fminf(fmaxf(q, 0.0f), 255.0f);
  return floorf(q);     // astype(np.uint8) truncates; q >= 0
}
__global__ void __launch_bounds__(256) quantize_kernel(const float* __restrict__ img, uint8_t* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    out[i] = (uint8_t)quant_u8(__ldg(img + i));
}
__device__ __forceinline__ float resized_pixel(const float* __restrict__ img, int quantize, int H, int W, int S, int oh, int ow,
                                               float scale_h, float scale_w) {
  // torch upsample_bilinear2d, align_corners=False: src = max(scale*(dst+0.5)-0.5, 0)
  const float sh = fmaxf(scale_h * (oh + 0.5f) - 0.5f, 0.f), sw = fmaxf(scale_w * (ow + 0.5f) - 0.5f, 0.f);
  const int h0 = (int)sh, w0 = (int)sw;
  const int h1 = h0 + (h0 < H - 1 ? 1 : 0), w1 = w0 + (w0 < W - 1 ? 1 : 0);
  const float lh = sh - h0, lw = sw - w0;
  float v00 = __ldg(img + (long long)h0 * W + w0), v01 = __ldg(img + (long long)h0 * W + w1);
  float v10 = __ldg(img + (long long)h1 * W + w0), v11 = __ldg(img + (long long)h1 * W + w1);
  if (quantize) { v00 = quant_u8(v00); v01 = quant_u8(v01); v10 = quant_u8(v10); v11 = quant_u8(v11); }
  const float r = (1.f - lh) * ((1.f - lw) * v00 + lw * v01) + lh * ((1.f - lw) * v10 + lw * v11);
  return fminf(fmaxf(r, 0.f), 255.f);
}
// "friendly" post-resizer = PIL bilinear on float32 ('F'-mode) channels (src/utils/resize.py:50-53,72-82).  Pillow's
// ImagingResample (Resample.c: precompute_coeffs + ImagingResampleHorizontal/Vertical_32bpc), restated: two separable
// passes, horizontal first; per output coordinate o: centre = (o + 0.5) * in/out, filterscale = max(in/out, 1),
// support = filterscale (triangle filter), taps [int(centre - support + 0.5), int(centre + support + 0.5)) clipped to the
// image, weight tri((x - centre + 0.5) / filterscale) normalised by the tap sum; coefficients and accumulation in double,
// the intermediate (after the horizontal pass) and the result rounded to float32.  Anti-aliased when down-scaling.
struct PilTaps { int lo, n; double w[8]; };
__device__ __forceinline__ PilTaps pil_taps(int o, int in_size, int out_size) {
  PilTaps t;
  const double scale = (double)in_size / (double)out_size;
  const double fs = scale < 1.0 ? 1.0 : scale;
  const double support = fs, center = (o + 0.5) * scale, ss = 1.0 / fs;
  int lo = (int)(center - support + 0.5); if (lo < 0) lo = 0;
  int hi = (int)(center + support + 0.5); if (hi > in_size) hi = in_size;
  t.lo = lo; t.n = hi - lo; if (t.n > 8) t.n = 8;          // 8 taps cover down-scaling by up to 3.5x
  double ww = 0.0;
  for (int x = 0; x < t.n; ++x) {
    double a = (x + lo - center + 0.5) * ss; if (a < 0.0) a = -a;
    const double w = a < 1.0 ? 1.0 - a : 0.0;
    t.w[x] = w; ww += w;
  }
  if (ww != 0.0) for (int x = 0; x < t.n; ++x) t.w[x] /= ww;
  return t;
}
__device__ __forceinline__ float resized_pixel_pil(const float* __restrict__ img, int quantize, int H, int W, int S, int oh, int ow) {
  const PilTaps tx = pil_taps(ow, W, S), ty = pil_taps(oh, H, S);
  double acc = 0.0;
  for (int y = 0; y < ty.n; ++y) {
    const float* row = img + (long long)(ty.lo + y) * W + tx.lo;
    double h = 0.0;
    for (int x = 0; x < tx.n; ++x) {
      float v = __ldg(row + x);
      if (quantize) v = quant_u8(v);
      h += (double)v * tx.w[x];
    }
    acc += (double)(float)h * ty.w[y];                       // the horizontal pass stores float32
  }
  return (float)acc;
}
// mode 0: write the normalised resized image as NCHW fp32 [B,3,S,S] (API parity / tests);
// mode 1: write the stride-2 valid 3x3 patch tensor [B,So,So,32] bf16 of the normalised resized image.
__global__ void __launch_bounds__(256) resize_norm_kernel(const float* __restrict__ img, int quantize, int B, int H, int W, int S,
                                                           float* __restrict__ out_img, bf16* __restrict__ out_col, int So,
                                                           int friendly) {
  const float scale_h = (float)H / (float)S, scale_w = (float)W / (float)S;
  if (out_img) {
    const long long total = (long long)B * 3 * S * S;
    for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
      const int ow = (int)(i % S), oh = (int)((i / S) % S);
      const long long bc = i / ((long long)S * S);
      const float r = friendly ? resized_pixel_pil(img + bc * H * W, quantize, H, W, S, oh, ow)
                               : resized_pixel(img + bc * H * W, quantize, H, W, S, oh, ow, scale_h, scale_w);
      out_img[i] = (r / 255.0f - 0.5f) / 0.5f;
    }
  }
  if (out_col) {
    const long long total = (long long)B * So * So;
    for (long long p = (long long)blockIdx.x * 256 + threadIdx.x; p < total; p += (long long)gridDim.x * 256) {
      const int wo = (int)(p % So), ho = (int)((p / So) % So), b = (int)(p / ((long long)So * So));
      float v[4][8];                                 // k = t * 3 + c at v[k / 8][k % 8], as in col27_kernel
#pragma unroll
      for (int t = 0; t < 9; ++t)
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float* src = img + ((long long)b * 3 + c) * H * W;
          const float r = friendly ? resized_pixel_pil(src, quantize, H, W, S, 2 * ho + t / 3, 2 * wo + t % 3)
                                   : resized_pixel(src, quantize, H, W, S, 2 * ho + t / 3, 2 * wo + t % 3, scale_h, scale_w);
          v[(t * 3 + c) / 8][(t * 3 + c) % 8] = (r / 255.0f - 0.5f) / 0.5f;
        }
#pragma unroll
      for (int k = 27; k < 32; ++k) v[3][k - 24] = 0.f;
#pragma unroll
      for (int j = 0; j < 4; ++j) reinterpret_cast<uint4*>(out_col + p * 32)[j] = pack8(v[j]);
    }
  }
}

// Data path (src/data_util.py:59-142): a uint8 NHWC batch as the datasets store it (HDF5 "imgs", decoded image folders)
// -> what the reference's per-sample CPU transform chain delivers: RandomHorizontalFlip, ToTensor (x / 255), Normalize(0.5, 0.5)
// ((x - 0.5) / 0.5), as NCHW fp32 in [-1, 1].  Same fp32 operations in the same order => bit-identical values; the host
// only ships 1 byte per value over PCIe / NVLink-C2C instead of 4.
__global__ void __launch_bounds__(256) u8_to_img_kernel(const uint8_t* __restrict__ u8, const uint8_t* __restrict__ flip,
                                                         float* __restrict__ img, int B, int H, int W) {
  const long long total = (long long)B * 3 * H * W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int w = (int)(i % W), h = (int)((i / W) % H);
    const int c = (int)((i / ((long long)W * H)) % 3), b = (int)(i / ((long long)3 * W * H));
    const int ws = (flip && flip[b]) ? W - 1 - w : w;
    const float v = (float)u8[(((long long)b * H + h) * W + ws) * 3 + c];
    img[i] = (v / 255.0f - 0.5f) / 0.5f;
  }
}

__global__ void __launch_bounds__(256) cast_f32_bf16_kernel(const float* __restrict__ in, bf16* __restrict__ out, long long n,
                                                             float scale) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    out[i] = __float2bfloat16_rn(__ldg(in + i) * scale);
}
__global__ void __launch_bounds__(256) cast_bf16_f32_kernel(const bf16* __restrict__ in, float* __restrict__ out, long long n) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256)
    out[i] = __bfloat162float(in[i]);
}

// Fused Adam (torch.optim.Adam semantics, no weight decay / amsgrad) + optional EMA lerp of the updated weights:
//   m = b1 m + (1-b1) g ; v = b2 v + (1-b2) g^2 ; p -= lr/bc1 * m / (sqrt(v)/sqrt(bc2) + eps)
//   ema = p + decay * (ema - p)                       (torch lerp: p.lerp(p_ema, decay), src/utils/ema.py:33-36)
__global__ void __launch_bounds__(256) adam_ema_kernel(float* __restrict__ p, const float* __restrict__ g, float* __restrict__ m,
                                                        float* __restrict__ v, long long n, float lr, float b1, float b2,
                                                        float eps, float bc1, float bc2_sqrt, float* __restrict__ ema,
                                                        float decay, float grad_scale, const int* __restrict__ step_dev) {
  if (step_dev) {                                   // step counter kept on the device (CUDA-graph replays advance it)
    const float t = (float)__ldg(step_dev);
    bc1 = 1.f - powf(b1, t);
    bc2_sqrt = sqrtf(1.f - powf(b2, t));
  }
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float gi = g[i] * grad_scale;
    const float mi = b1 * m[i] + (1.f - b1) * gi;
    const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
    m[i] = mi;
    v[i] = vi;
    const float denom = sqrtf(vi) / bc2_sqrt + eps;
    const float pi = p[i] - (lr / bc1) * (mi / denom);
    p[i] = pi;
    if (ema) ema[i] = pi + decay * (ema[i] - pi);
  }
}
__global__ void __launch_bounds__(256) lerp_kernel(float* __restrict__ ema, const float* __restrict__ p, long long n, float decay) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float pi = p[i];
    ema[i] = pi + decay * (ema[i] - pi);
  }
}


// ---------------------------------------------------------------------------------------------- gradient penalty
// losses.cal_grad_penalty (src/utils/losses.py:301-316): x_hat = alpha*real + (1-alpha)*fake (per-sample alpha, torch's
// operation order: two products, one sum, each rounded), per-sample ||grad||_2, and the seed of the second pass
// v_b = dP/dgrad_b = 2 (||g_b|| - 1) / (B ||g_b||) * g_b   for P = mean_b (||g_b|| - 1)^2.
__global__ void __launch_bounds__(256) gp_interpolate_kernel(const float* __restrict__ real, const float* __restrict__ fake,
                                                              const float* __restrict__ alpha, float* __restrict__ out,
                                                              long long n_per, long long total) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const float a = __ldg(alpha + i / n_per);
    out[i] = __fadd_rn(__fmul_rn(a, real[i]), __fmul_rn(__fsub_rn(1.f, a), fake[i]));
  }
}
__global__ void __launch_bounds__(256) gp_sumsq_kernel(const float* __restrict__ g, float* __restrict__ sumsq, long long n_per,
                                                        int blocks_per_sample) {
  const int b = blockIdx.x / blocks_per_sample, k = blockIdx.x % blocks_per_sample;
  const float* gb = g + (long long)b * n_per;
  float acc = 0.f;
  for (long long i = (long long)k * 256 + threadIdx.x; i < n_per; i += (long long)blocks_per_sample * 256) acc = fmaf(gb[i], gb[i], acc);
  __shared__ float red[8];
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < 8; ++w) t += red[w];
    atomicAdd(sumsq + b, t);
  }
}
__global__ void __launch_bounds__(256) gp_seed_kernel(const float* __restrict__ g, const float* __restrict__ sumsq,
                                                       float* __restrict__ v, long long n_per, long long total, float inv_B) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const float n = sqrtf(__ldg(sumsq + i / n_per));
    const float coef = n > 0.f ? 2.f * (n - 1.f) * inv_B / n : 0.f;
    v[i] = coef * g[i];
  }
}

// losses.cal_dra_penalty (src/utils/losses.py:319-335): sigma = real_images.std() (unbiased, over the whole batch) and
// x_hat = real + alpha_b * ((0.5 * sigma) * u), each product and the sum rounded once, in torch's order.  The standard
// deviation accumulates in fp64 around the first element (shifted sums keep the one-pass variance free of cancellation);
// one block per slice writes its two partial sums, then a single block adds them in a fixed order: deterministic.
__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ void block_sum2_f64(double& s, double& q) {    // 256 threads; the result lands in thread 0
  __shared__ double red[2][8];
  s = warp_sum_f64(s);
  q = warp_sum_f64(q);
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s;
    red[1][threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = q = 0.0;
    for (int w = 0; w < 8; ++w) {
      s += red[0][w];
      q += red[1][w];
    }
  }
}
__global__ void __launch_bounds__(256) dra_std_partial_kernel(const float* __restrict__ x, long long n, double* __restrict__ ws) {
  const double x0 = (double)__ldg(x);
  double s = 0.0, q = 0.0;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const double d = (double)__ldg(x + i) - x0;
    s += d;
    q = fma(d, d, q);
  }
  block_sum2_f64(s, q);
  if (threadIdx.x == 0) {
    ws[2 * blockIdx.x] = s;
    ws[2 * blockIdx.x + 1] = q;
  }
}
__global__ void __launch_bounds__(256) dra_std_final_kernel(const double* __restrict__ ws, int parts, long long n,
                                                             float* __restrict__ sigma) {
  double s = 0.0, q = 0.0;
  for (int k = threadIdx.x; k < parts; k += 256) {
    s += ws[2 * k];
    q += ws[2 * k + 1];
  }
  block_sum2_f64(s, q);
  if (threadIdx.x == 0) {
    const double var = fmax((q - s * s / (double)n) / (double)(n - 1), 0.0);
    *sigma = (float)sqrt(var);
  }
}
__global__ void __launch_bounds__(256) dra_perturb_kernel(const float* __restrict__ real, const float* __restrict__ sigma,
                                                           const float* __restrict__ alpha, const float* __restrict__ noise,
                                                           float* __restrict__ out, long long n_per, long long total) {
  const float half_sigma = __fmul_rn(0.5f, __ldg(sigma));
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const float a = __ldg(alpha + i / n_per);
    out[i] = __fadd_rn(real[i], __fmul_rn(a, __fmul_rn(half_sigma, noise[i])));
  }
}

// losses.cal_maxgrad_penalty (src/utils/losses.py:337-353): P = max_b ||g_b||^2 and its gradient w.r.t. g, which torch's
// backward of a full max() reduction spreads evenly over the tied arg-max samples: v_b = 2 g_b / n_ties there, 0
// elsewhere.  A NaN norm makes P NaN and the NaN samples the arg-max, as torch's max does.  Every block finds the maximum
// and the tie count over the [B] norms itself (B is small) before its slice of v.
__global__ void __launch_bounds__(256) gp_seed_max_kernel(const float* __restrict__ g, const float* __restrict__ sumsq,
                                                           float* __restrict__ v, float* __restrict__ penalty, int B,
                                                           long long n_per, long long total) {
  __shared__ float red[8];
  __shared__ float s_max;
  __shared__ int s_ties;
  float m = -INFINITY;
  int nan = 0;
  for (int b = threadIdx.x; b < B; b += 256) {
    const float s = __ldg(sumsq + b);
    nan |= isnan(s);
    m = fmaxf(m, s);
  }
  nan = __syncthreads_or(nan);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = red[0];
    for (int w = 1; w < 8; ++w) t = fmaxf(t, red[w]);
    s_max = nan ? __int_as_float(0x7fffffff) : t;
    s_ties = 0;
  }
  __syncthreads();
  m = s_max;
  int ties = 0;
  for (int b = threadIdx.x; b < B; b += 256) {
    const float s = __ldg(sumsq + b);
    ties += nan ? isnan(s) : s == m;
  }
  if (ties) atomicAdd(&s_ties, ties);
  __syncthreads();
  if (blockIdx.x == 0 && threadIdx.x == 0) *penalty = m;
  const float coef = 2.f / (float)s_ties;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const float s = __ldg(sumsq + i / n_per);
    v[i] = (nan ? isnan(s) : s == m) ? coef * g[i] : 0.f;
  }
}

// WGAN weight clipping (src/worker.py:490-492, p.data.clamp_(-c, c) over every discriminator parameter) as torch.clamp:
// NaN stays NaN, which fminf / fmaxf alone would replace by a bound.
__global__ void __launch_bounds__(256) clamp_kernel(float* __restrict__ x, long long n, float c) {
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float t = x[i];
    x[i] = isnan(t) ? t : fminf(fmaxf(t, -c), c);
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_axpby(const void* x, int64_t xs, const void* y, int64_t ys, const void* mask, int64_t ms, void* out,
                         int64_t os, int64_t npix, int32_t C, float a, const float* a_dev, float b, int32_t act,
                         sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && out && npix > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && os % 8 == 0);
  SGB_REQUIRE((!y || ys % 8 == 0) && (!mask || ms % 8 == 0));
  axpby_kernel<<<ew_blocks(npix * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (const bf16*)y, ys, (const bf16*)mask, ms,
                                                             (bf16*)out, os, npix, C, a, a_dev, b, act);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_pool2_fwd(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t Ho, int32_t Wo, int32_t C,
                             int32_t mode, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && B > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && ys % 8 == 0);
  pool2_fwd_kernel<<<ew_blocks((long long)B * Ho * Wo * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (bf16*)y, ys, B, Ho, Wo, C,
                                                                                  mode);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_relu_pool2(const void* x, int64_t xs, void* a0, int64_t as_, void* y, int64_t ys, int32_t B, int32_t Ho,
                              int32_t Wo, int32_t C, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && a0 && y && B > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && as_ % 8 == 0 && ys % 8 == 0);
  relu_pool2_kernel<<<ew_blocks((long long)B * Ho * Wo * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (bf16*)a0, as_, (bf16*)y, ys, B,
                                                                                    Ho, Wo, C);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_pool2_bwd(const void* dy, int64_t dys, const void* x, int64_t xs, const void* add, int64_t adds,
                             const void* relu_src, int64_t rs, void* dx, int64_t dxs, int32_t B, int32_t Ho, int32_t Wo,
                             int32_t C, int32_t mode, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dy && dx && B > 0 && Ho > 0 && Wo > 0 && C > 0 && C % 8 == 0 && dys % 8 == 0 && dxs % 8 == 0);
  SGB_REQUIRE(mode == 0 || (x && xs % 8 == 0));
  SGB_REQUIRE((!add || adds % 8 == 0) && (!relu_src || rs % 8 == 0 || (rs == -1 && C % 64 == 0)));   // rs == -1: relu_src = bit planes
  if (relu_src && rs == -1)
    pool2_bwd_kernel<true><<<ew_blocks((long long)B * Ho * Wo * (C / 8)), 256, 0, stream>>>(
        (const bf16*)dy, dys, (const bf16*)x, xs, (const bf16*)add, adds, (const bf16*)relu_src, rs, (bf16*)dx, dxs, B, Ho, Wo, C, mode);
  else
    pool2_bwd_kernel<false><<<ew_blocks((long long)B * Ho * Wo * (C / 8)), 256, 0, stream>>>(
        (const bf16*)dy, dys, (const bf16*)x, xs, (const bf16*)add, adds, (const bf16*)relu_src, rs, (bf16*)dx, dxs, B, Ho, Wo, C, mode);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_dhead_fwd(const float* h, const float* w1, const float* sigma1, const float* b1, const float* E,
                             const float* sigmaE, const int64_t* labels, int32_t B, int32_t C, float* adv, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(h && w1 && adv && B > 0 && C > 0 && (!E || labels));
  dhead_fwd_kernel<<<(B + 7) / 8, 256, 0, stream>>>(h, w1, sigma1, b1, E, sigmaE, (const long long*)labels, B, C, adv);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_dhead_bwd(const float* dadv, const float* h, const float* w1, const float* sigma1, const float* E,
                             const float* sigmaE, const int64_t* labels, int32_t B, int32_t C, float* dh, float* gw1, float* gE,
                             float* db1, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dadv && h && w1 && B > 0 && C > 0 && (!E || labels));
  if (dh || (E && gE)) {
    dhead_bwd_rows_kernel<<<dim3((C + 255) / 256, B), 256, 0, stream>>>(dadv, h, w1, sigma1, E, sigmaE, (const long long*)labels, B, C,
                                                                        dh, gE);
    SGB_LAUNCH_CHECK();
  }
  if (gw1) {
    dhead_bwd_w_kernel<<<(C + 255) / 256, 256, 0, stream>>>(dadv, h, B, C, gw1, db1);
    SGB_LAUNCH_CHECK();
  }
  return SGB_OK;
}

extern "C" int sgb_rowdot(const void* x, int64_t xs, const void* y, int64_t ys, int64_t rows, int32_t C, float* out, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && out && rows > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && ys % 8 == 0);
  rowdot_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>((const bf16*)x, xs, (const bf16*)y, ys, rows, C, out);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_softmax_rows(const void* s, void* p, int64_t rows, int32_t n, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(s && p && rows > 0 && n > 0 && n % 8 == 0);
  softmax_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>((const bf16*)s, (bf16*)p, rows, n);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_softmax_bwd_rows(const void* p, const void* dp, void* ds, int64_t rows, int32_t n, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(p && dp && ds && rows > 0 && n > 0 && n % 8 == 0);
  softmax_bwd_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, stream>>>((const bf16*)p, (const bf16*)dp, (bf16*)ds, rows, n);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_dot(const void* x, const void* y, int64_t n, float* out, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && out && n > 0 && n % 8 == 0);
  SGB_CUDA(cudaMemsetAsync(out, 0, sizeof(float), stream));
  dot_kernel<<<ew_blocks(n / 8), 256, 0, stream>>>((const bf16*)x, (const bf16*)y, n / 8, out);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_sum_hw(const void* x, int64_t xs, int32_t B, int32_t HW, int32_t C, int32_t relu, float* h,
                          sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && h && B > 0 && HW > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && C <= 8192);
  SGB_CUDA(cudaMemsetAsync(h, 0, sizeof(float) * (size_t)B * C, stream));
  int chunks = (4 * sm_count() + B - 1) / B;
  if (chunks > HW) chunks = HW;
  if (chunks < 1) chunks = 1;
  const int ppb = (HW + chunks - 1) / chunks;
  dim3 grid((HW + ppb - 1) / ppb, B);
  sum_hw_kernel<<<grid, 256, sizeof(float) * C, stream>>>((const bf16*)x, xs, HW, C, relu, h, ppb);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_sum_hw_bwd(const float* dh, const void* x, int64_t xs, void* dx, int64_t dxs, int32_t B, int32_t HW,
                              int32_t C, int32_t relu, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dh && x && dx && B > 0 && HW > 0 && C > 0 && C % 8 == 0 && xs % 8 == 0 && dxs % 8 == 0);
  sum_hw_bwd_kernel<<<ew_blocks((long long)B * HW * (C / 8)), 256, 0, stream>>>(dh, (const bf16*)x, xs, (bf16*)dx, dxs, B, HW, C,
                                                                              relu);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_img_to_nhwc(const float* img, void* out, int32_t B, int32_t C, int32_t HW, int32_t Cp, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(img && out && B > 0 && C > 0 && HW > 0 && Cp >= C && Cp % 8 == 0);
  img_to_nhwc_kernel<<<ew_blocks((long long)B * HW), 256, 0, stream>>>(img, (bf16*)out, B, C, HW, Cp);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_nhwc_to_img(const void* in, int32_t in_fp32, int64_t cs, float* img, int32_t B, int32_t C, int32_t HW,
                               int32_t act, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(in && img && B > 0 && C > 0 && HW > 0 && cs >= C);
  nhwc_to_img_kernel<<<ew_blocks((long long)B * HW), 256, 0, stream>>>(in, in_fp32, cs, img, B, C, HW, act);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_img_grad_to_nhwc(const float* dimg, const float* y, void* out, int32_t B, int32_t C, int32_t HW, int32_t Cp,
                                    sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dimg && out && B > 0 && C > 0 && HW > 0 && Cp >= C && Cp % 8 == 0);
  img_grad_to_nhwc_kernel<<<ew_blocks((long long)B * HW), 256, 0, stream>>>(dimg, y, (bf16*)out, B, C, HW, Cp);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_col27(const void* src, int32_t src_nchw_f32, int64_t cs, void* out, int32_t B, int32_t H, int32_t W,
                         sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(src && out && B > 0 && H > 0 && W > 0 && (src_nchw_f32 || cs >= 3));
  col27_kernel<<<ew_blocks((long long)B * H * W), 256, 0, stream>>>(src, src_nchw_f32, cs, (bf16*)out, B, H, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_col27_bwd(const void* dcol, float* dimg, int32_t B, int32_t H, int32_t W, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dcol && dimg && B > 0 && H > 0 && W > 0);
  col27_bwd_kernel<<<ew_blocks((long long)B * H * W), 256, 0, stream>>>((const bf16*)dcol, dimg, B, H, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_pool3x3(const void* x, int64_t xs, void* y, int64_t ys, int32_t B, int32_t H, int32_t W, int32_t C, int32_t stride,
                           int32_t pad, int32_t mode, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && B > 0 && H >= 3 && W >= 3 && C > 0 && C % 8 == 0 && xs % 8 == 0 && ys % 8 == 0);
  SGB_REQUIRE((stride == 1 || stride == 2) && (pad == 0 || pad == 1) && (mode == 0 || mode == 1));
  const int Ho = (H + 2 * pad - 3) / stride + 1, Wo = (W + 2 * pad - 3) / stride + 1;
  pool3x3_kernel<<<ew_blocks((long long)B * Ho * Wo * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (bf16*)y, ys, B, H, W, Ho, Wo, C,
                                                                                 stride, pad, mode);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_quantize_u8(const float* img, uint8_t* out, int64_t n, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(img && out && n > 0);
  quantize_kernel<<<ew_blocks(n), 256, 0, stream>>>(img, out, n);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_quantize_resize_normalize(const float* img, int32_t quantize, int32_t B, int32_t H, int32_t W, int32_t S,
                                             float* out_img, void* out_col, int32_t resizer, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(img && (out_img || out_col) && B > 0 && H > 0 && W > 0 && S >= 3);
  SGB_REQUIRE(resizer == 0 || resizer == 1);
  SGB_REQUIRE(resizer == 0 || (2 * H <= 7 * S && 2 * W <= 7 * S));   // PIL path: at most 8 taps per axis
  const int So = (S - 3) / 2 + 1;
  const long long work = out_img ? (long long)B * 3 * S * S : (long long)B * So * So;
  resize_norm_kernel<<<ew_blocks(work), 256, 0, stream>>>(img, quantize, B, H, W, S, out_img, (bf16*)out_col, So, resizer);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_u8_to_img(const uint8_t* u8, const uint8_t* flip, float* img, int32_t B, int32_t H, int32_t W, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(u8 && img && B > 0 && H > 0 && W > 0);
  u8_to_img_kernel<<<ew_blocks((long long)B * 3 * H * W), 256, 0, stream>>>(u8, flip, img, B, H, W);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_cast_f32_to_bf16(const float* in, void* out, int64_t n, float scale, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(in && out && n > 0);
  cast_f32_bf16_kernel<<<ew_blocks(n), 256, 0, stream>>>(in, (bf16*)out, n, scale);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_cast_bf16_to_f32(const void* in, float* out, int64_t n, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(in && out && n > 0);
  cast_bf16_f32_kernel<<<ew_blocks(n), 256, 0, stream>>>((const bf16*)in, out, n);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_adam_ema_step(float* p, const float* g, float* m, float* v, int64_t n, float lr, float beta1, float beta2,
                                 float eps, int32_t step, const int32_t* step_dev, float* ema, float ema_decay, float grad_scale,
                                 sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(p && g && m && v && n > 0 && (step >= 1 || step_dev));
  const float bc1 = 1.f - powf(beta1, (float)step);
  const float bc2 = 1.f - powf(beta2, (float)step);
  adam_ema_kernel<<<ew_blocks(n), 256, 0, stream>>>(p, g, m, v, n, lr, beta1, beta2, eps, bc1, sqrtf(bc2), ema, ema_decay,
                                                   grad_scale, step_dev);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_ema_lerp(float* ema, const float* p, int64_t n, float decay, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(ema && p && n > 0);
  lerp_kernel<<<ew_blocks(n), 256, 0, stream>>>(ema, p, n, decay);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_gp_interpolate(const float* real, const float* fake, const float* alpha, float* out, int32_t B, int64_t n_per,
                                  sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(real && fake && alpha && out && B > 0 && n_per > 0);
  const long long total = (long long)B * n_per;
  gp_interpolate_kernel<<<ew_blocks(total), 256, 0, stream>>>(real, fake, alpha, out, n_per, total);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_gp_sumsq(const float* g, float* sumsq, int32_t B, int64_t n_per, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(g && sumsq && B > 0 && n_per > 0);
  SGB_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float) * (size_t)B, stream));
  long long bps = (n_per + 256 * 16 - 1) / (256 * 16);
  const long long cap = (8LL * sm_count() + B - 1) / B;
  if (bps > cap) bps = cap;
  if (bps < 1) bps = 1;
  gp_sumsq_kernel<<<(unsigned)(B * bps), 256, 0, stream>>>(g, sumsq, n_per, (int)bps);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_gp_seed(const float* g, const float* sumsq, float* v, int32_t B, int64_t n_per, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(g && sumsq && v && B > 0 && n_per > 0);
  const long long total = (long long)B * n_per;
  gp_seed_kernel<<<ew_blocks(total), 256, 0, stream>>>(g, sumsq, v, n_per, total, 1.f / (float)B);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_gp_seed_max(const float* g, const float* sumsq, float* v, float* penalty, int32_t B, int64_t n_per,
                               sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(g && sumsq && v && penalty && B > 0 && n_per > 0);
  const long long total = (long long)B * n_per;
  gp_seed_max_kernel<<<ew_blocks(total), 256, 0, stream>>>(g, sumsq, v, penalty, B, n_per, total);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_dra_std(const float* x, int64_t n, double* ws, float* sigma, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && ws && sigma && n > 1);
  long long parts = (n + 256 * 16 - 1) / (256 * 16);
  if (parts > SGB_DRA_STD_PARTS) parts = SGB_DRA_STD_PARTS;
  dra_std_partial_kernel<<<(unsigned)parts, 256, 0, stream>>>(x, n, ws);
  SGB_LAUNCH_CHECK();
  dra_std_final_kernel<<<1, 256, 0, stream>>>(ws, (int)parts, n, sigma);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_dra_perturb(const float* real, const float* sigma, const float* alpha, const float* noise, float* out,
                               int32_t B, int64_t n_per, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(real && sigma && alpha && noise && out && B > 0 && n_per > 0);
  const long long total = (long long)B * n_per;
  dra_perturb_kernel<<<ew_blocks(total), 256, 0, stream>>>(real, sigma, alpha, noise, out, n_per, total);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_clamp(float* x, int64_t n, float c, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && n > 0 && c >= 0.f);
  clamp_kernel<<<ew_blocks(n), 256, 0, stream>>>(x, n, c);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
