// Batch-norm family on NHWC bf16 activations (HBM-bound streaming kernels, 16-byte vector accesses).
//   stats      : per-channel sum / sum-of-squares                         (F.batch_norm training statistics)
//   finalize   : mean / rstd, running-stat update, per-(image,channel) scale & shift for cBN or affine BN
//   apply      : y = [relu](x*scale + shift), optional fused nearest x2 upsample of the result
//   bwd_reduce : per-(image,channel) sums of dz and dz*xhat (+ channel totals weighted by the cBN gain)
//   bwd_apply  : dx = a*dz - k1 - k2*xhat
// Reference arithmetic: src/utils/ops.py:14-28 (ConditionalBatchNorm2d), :227-228 (batchnorm_2d, eps 1e-4,
// momentum 0.1), torch F.batch_norm; cross-rank reduction points follow torch/nn/modules/_functions.py:7-212.
#include "common.cuh"
#include <type_traits>

namespace sgb {

static constexpr int kChunkC = 2048;  // channels handled per block of the stats / backward kernels

// Thread layout of the stats / backward kernels over one chunk of kChunkC channels: thread threadIdx.x owns the 8-channel
// group g of the chunk and the pixel rows prow, prow + nrows, ... of the block's pixel range (threads with prow >= nrows idle).
struct ChanGroups {
  int c_base, cc;      // first channel of the chunk, channels in it
  int g, prow, nrows;
};
__device__ __forceinline__ ChanGroups chan_groups(int C, int chunk) {
  ChanGroups t;
  t.c_base = chunk * kChunkC;
  t.cc = min(C - t.c_base, kChunkC);
  const int VG = t.cc >> 3;
  const int VGb = VG < 256 ? VG : 256;
  t.nrows = 256 / VGb;
  t.g = threadIdx.x % VGb;
  t.prow = threadIdx.x / VGb;
  return t;
}

// ---------------------------------------------------------------------------------------------- stats
__global__ void __launch_bounds__(256) bn_stats_kernel(const bf16* __restrict__ x, long long npix, int C, long long cstride,
                                                        float* __restrict__ sum, float* __restrict__ sumsq,
                                                        long long pix_per_block) {
  __shared__ float s_sum[kChunkC];
  __shared__ float s_sq[kChunkC];
  const auto [c_base, cc, g, prow, nrows] = chan_groups(C, blockIdx.y);
  for (int i = threadIdx.x; i < cc; i += 256) { s_sum[i] = 0.f; s_sq[i] = 0.f; }
  __syncthreads();
  if (prow < nrows) {
    float a[8], q[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a[j] = 0.f; q[j] = 0.f; }
    const long long p0 = (long long)blockIdx.x * pix_per_block;
    const long long p1 = min(p0 + pix_per_block, npix);
    constexpr int U = 4;                         // four packed loads in flight per thread (latency-bound otherwise at small H*W)
    for (long long p = p0 + prow; p < p1; p += (long long)U * nrows) {
      uint4 r[U];
#pragma unroll
      for (int u = 0; u < U; ++u)
        if (p + (long long)u * nrows < p1) r[u] = __ldg(reinterpret_cast<const uint4*>(x + (p + (long long)u * nrows) * cstride + c_base) + g);
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (p + (long long)u * nrows < p1) {
          float f[8];
          unpack8(r[u], f);
#pragma unroll
          for (int j = 0; j < 8; ++j) { a[j] += f[j]; q[j] = fmaf(f[j], f[j], q[j]); }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { atomicAdd(&s_sum[g * 8 + j], a[j]); atomicAdd(&s_sq[g * 8 + j], q[j]); }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cc; i += 256) {
    atomicAdd(sum + c_base + i, s_sum[i]);
    atomicAdd(sumsq + c_base + i, s_sq[i]);
  }
}

// ---------------------------------------------------------------------------------------------- finalize
// mode 0: cBN     scale[b,c] = rstd*(1+gain[b,c]),  shift[b,c] = bias[b,c] - mean*scale[b,c]   (nb = B rows)
// mode 1: affine  scale[c]   = rstd*weight[c],      shift[c]   = bias[c]   - mean*scale[c]     (nb = 1 row)
// mode 2: plain   scale[c]   = rstd,                shift[c]   = -mean*rstd                    (nb = 1 row)
// use_batch_stats: 1 -> mean/var from sum/sumsq/count (and running stats updated if track), 0 -> running stats;
//                  2 -> as 1 with the DataParallel-mode SynchronizedBatchNorm's inverse std, bias_var.clamp(eps)^-0.5
//                       (src/sync_batchnorm/batchnorm.py:158-175) instead of torch's (var + eps)^-0.5.
__global__ void bn_finalize_kernel(const float* __restrict__ sum, const float* __restrict__ sumsq, float count,
                                   float* __restrict__ running_mean, float* __restrict__ running_var, float momentum,
                                   float eps, int use_batch_stats, int track, int mode, const float* __restrict__ gain,
                                   const float* __restrict__ bias, int nb, int C, float* __restrict__ mean_out,
                                   float* __restrict__ rstd_out, float* __restrict__ scale, float* __restrict__ shift, long long affine_ld) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  float mean, var;
  if (use_batch_stats) {
    mean = sum[c] / count;
    var = fmaxf(sumsq[c] / count - mean * mean, 0.f);
    if (track && running_mean && blockIdx.y == 0) {
      const float unbiased = count > 1.f ? var * (count / (count - 1.f)) : var;
      running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
      running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
    }
  } else {
    mean = running_mean[c];
    var = running_var[c];
  }
  const float rstd = use_batch_stats == 2 ? rsqrtf(fmaxf(var, eps)) : rsqrtf(var + eps);
  if (blockIdx.y == 0) {
    mean_out[c] = mean;
    rstd_out[c] = rstd;
  }
  for (int b = blockIdx.y; b < nb; b += gridDim.y) {   // images spread over blockIdx.y: no 256-deep serial loop for cBN
    float g = 1.f, be = 0.f;
    if (mode == 0) { g = 1.f + gain[(size_t)b * affine_ld + c]; be = bias[(size_t)b * affine_ld + c]; }
    else if (mode == 1) { g = gain[c]; be = bias[c]; }
    const float sc = rstd * g;
    scale[(size_t)b * C + c] = sc;
    shift[(size_t)b * C + c] = be - mean * sc;
  }
}

// ---------------------------------------------------------------------------------------------- apply
// One thread = 8 channels of one input pixel.  bstride = C for per-image scale/shift, 0 for per-channel.
__global__ void __launch_bounds__(256) scale_shift_act_kernel(const bf16* __restrict__ x, int B, int H, int W, int C,
                                                               long long x_cstride, const float* __restrict__ scale,
                                                               const float* __restrict__ shift, int bstride, int relu,
                                                               int up2, bf16* __restrict__ y, long long y_cstride) {
  const int VG = C >> 3;
  const long long total = (long long)B * H * W * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    const int b = (int)(p / ((long long)H * W));
    const uint4 r = __ldg(reinterpret_cast<const uint4*>(x + p * x_cstride) + g);
    float f[8];
    unpack8(r, f);
    const float4* sp = reinterpret_cast<const float4*>(scale + (size_t)b * bstride + g * 8);
    const float4* hp = reinterpret_cast<const float4*>(shift + (size_t)b * bstride + g * 8);
    const float4 s0 = __ldg(sp), s1 = __ldg(sp + 1), h0 = __ldg(hp), h1 = __ldg(hp + 1);
    f[0] = fmaf(f[0], s0.x, h0.x); f[1] = fmaf(f[1], s0.y, h0.y); f[2] = fmaf(f[2], s0.z, h0.z); f[3] = fmaf(f[3], s0.w, h0.w);
    f[4] = fmaf(f[4], s1.x, h1.x); f[5] = fmaf(f[5], s1.y, h1.y); f[6] = fmaf(f[6], s1.z, h1.z); f[7] = fmaf(f[7], s1.w, h1.w);
    if (relu) {
#pragma unroll
      for (int j = 0; j < 8; ++j) f[j] = fmaxf(f[j], 0.f);
    }
    const uint4 o = pack8(f);
    if (!up2) {
      reinterpret_cast<uint4*>(y + p * y_cstride)[g] = o;
    } else {
      long long qs[4];
      quad2x2(p, (int)(p % W), W, qs);
#pragma unroll
      for (int k = 0; k < 4; ++k) reinterpret_cast<uint4*>(y + qs[k] * y_cstride)[g] = o;
    }
  }
}

// ---------------------------------------------------------------------------------------------- backward
// The backward kernels run one template instance per value of UP2: whether the forward upsampled its output (nearest x2),
// so that the gradient dy is [B][2H][2W] and dz of a pixel is the sum of dy over its 2x2 block.  A thread owns one 8-channel
// group of one image; a step of its pixel loop covers U pixels (4, or 2 with UP2, which reads 4 dy vectors per pixel) and
// issues all of their 16-byte loads before the normalisation arithmetic (only the UP2 dz sums run as the vectors arrive):
// the kernels are pure streams and their speed is the number of bytes each SM keeps in flight.

// dz of 8 channels as a step holds it until its arithmetic, in the fewer registers: the packed dy vector (4), or with UP2
// the float sum of the four dy vectors of the 2x2 block (8, not 16).
template <bool UP2>
using DzRegs = std::conditional_t<UP2, float[8], uint4>;

// dz of 8 channels (group g) of pixel p = b * H * W + hw, x = hw % W.
template <bool UP2>
__device__ __forceinline__ void load_dz(const bf16* __restrict__ dy, long long dy_cstride, long long p, int x, int W, int g,
                                        DzRegs<UP2>& dz) {
  if constexpr (!UP2) {
    dz = __ldg(reinterpret_cast<const uint4*>(dy + p * dy_cstride) + g);
  } else {
    long long qs[4];
    quad2x2(p, x, W, qs);
    unpack8(__ldg(reinterpret_cast<const uint4*>(dy + qs[0] * dy_cstride) + g), dz);
#pragma unroll
    for (int k = 1; k < 4; ++k) {
      float t[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(dy + qs[k] * dy_cstride) + g), t);
#pragma unroll
      for (int j = 0; j < 8; ++j) dz[j] += t[j];
    }
  }
}

// Gradient at the normalised pre-activation z = x * sc + sh of 8 channels: dz, or 0 where a ReLU followed and z <= 0.
template <bool UP2>
__device__ __forceinline__ void relu_grad8(const float (&xv)[8], const DzRegs<UP2>& dz, const float (&sc)[8],
                                           const float (&sh)[8], int relu, float (&d)[8]) {
  float f[8];
  if constexpr (UP2) {
#pragma unroll
    for (int j = 0; j < 8; ++j) f[j] = dz[j];
  } else {
    unpack8(dz, f);
  }
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const float z = fmaf(xv[j], sc[j], sh[j]);
    d[j] = (relu && !(z > 0.f)) ? 0.f : f[j];
  }
}

// grid = (pixel chunks, B, channel chunks).  s1[b,c] += sum dz, s2[b,c] += sum dz*xhat (bn_bwd_total_kernel forms S1, S2).
template <bool UP2>
__global__ void __launch_bounds__(256) bn_bwd_reduce_kernel(const bf16* __restrict__ dy, long long dy_cstride,
                                                             const bf16* __restrict__ x, long long x_cstride, int H, int W, int C,
                                                             const float* __restrict__ scale, const float* __restrict__ shift,
                                                             int bstride, const float* __restrict__ mean,
                                                             const float* __restrict__ rstd, int relu, float* __restrict__ s1,
                                                             float* __restrict__ s2, int pix_per_block) {
  __shared__ float a1[kChunkC];
  __shared__ float a2[kChunkC];
  const int b = blockIdx.y;
  const auto [c_base, cc, g, prow, nrows] = chan_groups(C, blockIdx.z);
  for (int i = threadIdx.x; i < cc; i += 256) { a1[i] = 0.f; a2[i] = 0.f; }
  __syncthreads();
  if (prow < nrows) {
    // t2 accumulates sum(d * x) with the RAW input; sum(d * xhat) = rstd * (t2 - mean * t1) is formed once at the end, so the
    // loop carries no per-channel mean / rstd.
    float t1[8], t2[8], sc[8], sh[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      t1[j] = 0.f; t2[j] = 0.f;
      const int c = c_base + g * 8 + j;
      sc[j] = scale[(size_t)b * bstride + c]; sh[j] = shift[(size_t)b * bstride + c];
    }
    const int HW = H * W;
    const int p0 = blockIdx.x * pix_per_block, p1 = min(p0 + pix_per_block, HW);
    const int gg = (c_base >> 3) + g;
    constexpr int U = UP2 ? 2 : 4;
    for (int hw = p0 + prow; hw < p1; hw += U * nrows) {
      uint4 rx[U];
      DzRegs<UP2> dz[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const int h2 = hw + u * nrows;
        if (h2 < p1) {
          const long long p = (long long)b * HW + h2;
          rx[u] = __ldg(reinterpret_cast<const uint4*>(x + p * x_cstride) + gg);
          load_dz<UP2>(dy, dy_cstride, p, h2 % W, W, gg, dz[u]);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        if (hw + u * nrows < p1) {
          float xv[8], d[8];
          unpack8(rx[u], xv);
          relu_grad8<UP2>(xv, dz[u], sc, sh, relu, d);
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            t1[j] += d[j];
            t2[j] = fmaf(d[j], xv[j], t2[j]);
          }
        }
      }
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = c_base + g * 8 + j;
      atomicAdd(&a1[g * 8 + j], t1[j]);
      atomicAdd(&a2[g * 8 + j], rstd[c] * (t2[j] - mean[c] * t1[j]));
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < cc; i += 256) {
    const int c = c_base + i;
    const float v1 = a1[i], v2 = a2[i];
    atomicAdd(s1 + (size_t)b * C + c, v1);
    atomicAdd(s2 + (size_t)b * C + c, v2);
  }
}

// S1[c] = sum_b g1[b,c] * s1[b,c], S2 likewise, with g1 = scale / rstd (cBN: 1 + gain, affine: weight, plain: 1): d(xhat) = dz * g1.
// A separate C-thread pass over the [B][C] partials instead of B * blocks atomics per channel on two hot addresses.
__global__ void __launch_bounds__(256) bn_bwd_total_kernel(const float* __restrict__ s1, const float* __restrict__ s2,
                                                            const float* __restrict__ scale, int bstride,
                                                            const float* __restrict__ rstd, int B, int C, float* __restrict__ S1,
                                                            float* __restrict__ S2) {
  // one warp per channel, lanes stride over the images
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (c >= C) return;
  const float ir = 1.f / rstd[c];
  float a1 = 0.f, a2 = 0.f;
  for (int b = lane; b < B; b += 32) {
    const float g1 = scale[(size_t)b * bstride + c] * ir;
    a1 = fmaf(g1, s1[(size_t)b * C + c], a1);
    a2 = fmaf(g1, s2[(size_t)b * C + c], a2);
  }
  a1 = warp_sum(a1);
  a2 = warp_sum(a2);
  if (lane == 0) {
    S1[c] = a1;
    S2[c] = a2;
  }
}

// dx = scale[b,c]*dz - rstd*(S1/N) - rstd*(S2/N)*xhat   (train) ;   dx = scale[b,c]*dz   (eval: use_batch_stats = 0)
// grid = (pixel chunks, B, channel chunks) like the reduce kernel: a thread owns one 8-channel group of one image, so
// every per-(image, channel) constant lives in registers and the loop body is two 16-byte loads, 8 FMAs and one store.
template <bool UP2>
__global__ void __launch_bounds__(256) bn_bwd_apply_kernel(const bf16* __restrict__ dy, long long dy_cstride,
                                                            const bf16* __restrict__ x, long long x_cstride, int H, int W,
                                                            int C, const float* __restrict__ scale, const float* __restrict__ shift,
                                                            int bstride, const float* __restrict__ mean,
                                                            const float* __restrict__ rstd, const float* __restrict__ S1,
                                                            const float* __restrict__ S2, float inv_count, int relu,
                                                            int use_batch_stats, bf16* __restrict__ dx, long long dx_cstride,
                                                            int pix_per_block) {
  const int b = blockIdx.y;
  const auto [c_base, cc, g, prow, nrows] = chan_groups(C, blockIdx.z);
  if (prow >= nrows) return;
  const int gg = (c_base >> 3) + g;
  // dx = sc*d - ka - kb*(x - mu) = sc*d - k0 - kb*x with k0 = ka - kb*mu: four constants per channel.
  float sc[8], sh[8], k0[8], kb[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int c = c_base + g * 8 + j;
    sc[j] = scale[(size_t)b * bstride + c]; sh[j] = shift[(size_t)b * bstride + c];
    if (use_batch_stats) {
      const float rs = rstd[c];
      kb[j] = rs * rs * inv_count * S2[c];
      k0[j] = rs * inv_count * S1[c] - kb[j] * mean[c];
    } else {
      k0[j] = 0.f; kb[j] = 0.f;
    }
  }
  const int HW = H * W;
  const int p0 = blockIdx.x * pix_per_block, p1 = min(p0 + pix_per_block, HW);
  constexpr int U = UP2 ? 2 : 4;
  for (int hw = p0 + prow; hw < p1; hw += U * nrows) {
    uint4 rx[U];
    DzRegs<UP2> dz[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int h2 = hw + u * nrows;
      if (h2 < p1) {
        const long long p = (long long)b * HW + h2;
        rx[u] = __ldg(reinterpret_cast<const uint4*>(x + p * x_cstride) + gg);
        load_dz<UP2>(dy, dy_cstride, p, h2 % W, W, gg, dz[u]);
      }
    }
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const int h2 = hw + u * nrows;
      if (h2 < p1) {
        float xv[8], d[8], o[8];
        unpack8(rx[u], xv);
        relu_grad8<UP2>(xv, dz[u], sc, sh, relu, d);
#pragma unroll
        for (int j = 0; j < 8; ++j) o[j] = sc[j] * d[j] - k0[j] - kb[j] * xv[j];
        reinterpret_cast<uint4*>(dx + ((long long)b * HW + h2) * dx_cstride)[gg] = pack8(o);
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------- tangent (JVP) backward
// The gradient-penalty pass (sgb200/utils/gp.py) pushes a tangent a = dx/d(eps) through the discriminator.  For a
// training-mode batch norm the tangent map is  t = gamma * r * (a - mean(a) - xhat * mean(xhat * a))  (the same linear
// map as its backward, run by the bwd kernels above).  Differentiating t w.r.t. (x, a, gamma) for an incoming cotangent c
// (torch: batchnorm_double_backward, tools/autograd/templates/Functions.cpp) needs five per-channel sums
//   Sa = sum a, Sc = sum c, Sxa = sum xhat*a, Sxc = sum xhat*c, Sac = sum a*c            (M = pixels per channel)
//   dx = gamma r^2 / M * [ xhat * T + Sxc * (Sa/M - a) + Sxa * (Sc/M - c) ],  T = Sa*Sc/M - Sac + 3*Sxa*Sxc/M
//   da = gamma r * (c - Sc/M - xhat * Sxc/M)
//   dgamma = r * (Sac - Sa*Sc/M - Sxa*Sxc/M)                                              (host side, [C] vectors)
__global__ void __launch_bounds__(256) bn_tan_bwd_reduce_kernel(const bf16* __restrict__ x, long long xs,
                                                                 const bf16* __restrict__ a, long long as_,
                                                                 const bf16* __restrict__ c, long long cs, long long npix, int C,
                                                                 const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                 float* __restrict__ sums, long long pix_per_block) {
  __shared__ float acc[5][256];
  const int VG = C >> 3;
  const int VGb = VG < 32 ? VG : 32;          // channel groups handled per block (blockIdx.y strides the rest)
  const int nrows = 256 / VGb;
  const int gl = threadIdx.x % VGb, prow = threadIdx.x / VGb;
  const int g = blockIdx.y * VGb + gl;
  for (int i = threadIdx.x; i < 5 * 256; i += 256) acc[i / 256][i % 256] = 0.f;
  __syncthreads();
  if (prow < nrows && g < VG) {
    float t[5][8], mu[8], rs[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      mu[j] = mean[g * 8 + j]; rs[j] = rstd[g * 8 + j];
#pragma unroll
      for (int k = 0; k < 5; ++k) t[k][j] = 0.f;
    }
    const long long p0 = (long long)blockIdx.x * pix_per_block;
    const long long p1 = p0 + pix_per_block < npix ? p0 + pix_per_block : npix;
    for (long long p = p0 + prow; p < p1; p += nrows) {
      float xv[8], av[8], cv[8];
      unpack8(__ldg(reinterpret_cast<const uint4*>(x + p * xs) + g), xv);
      unpack8(__ldg(reinterpret_cast<const uint4*>(a + p * as_) + g), av);
      unpack8(__ldg(reinterpret_cast<const uint4*>(c + p * cs) + g), cv);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const float xh = (xv[j] - mu[j]) * rs[j];
        t[0][j] += av[j];
        t[1][j] += cv[j];
        t[2][j] = fmaf(xh, av[j], t[2][j]);
        t[3][j] = fmaf(xh, cv[j], t[3][j]);
        t[4][j] = fmaf(av[j], cv[j], t[4][j]);
      }
    }
#pragma unroll
    for (int k = 0; k < 5; ++k)
#pragma unroll
      for (int j = 0; j < 8; ++j) atomicAdd(&acc[k][gl * 8 + j], t[k][j]);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 5 * VGb * 8; i += 256) {
    const int k = i / (VGb * 8), cl = i % (VGb * 8);
    const int ch = blockIdx.y * VGb * 8 + cl;
    if (ch < C) atomicAdd(sums + (size_t)k * C + ch, acc[k][cl]);
  }
}

__global__ void __launch_bounds__(256) bn_tan_bwd_apply_kernel(const bf16* __restrict__ x, long long xs,
                                                                const bf16* __restrict__ a, long long as_,
                                                                const bf16* __restrict__ c, long long cs, long long npix, int C,
                                                                const float* __restrict__ gamma, const float* __restrict__ mean,
                                                                const float* __restrict__ rstd, const float* __restrict__ sums,
                                                                float inv_count, int use_batch_stats, bf16* __restrict__ dx,
                                                                long long dxs, bf16* __restrict__ da, long long das) {
  const int VG = C >> 3;
  const long long total = npix * VG;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int g = (int)(i % VG);
    const long long p = i / VG;
    float xv[8], av[8], cv[8], ox[8], oa[8];
    unpack8(__ldg(reinterpret_cast<const uint4*>(x + p * xs) + g), xv);
    unpack8(__ldg(reinterpret_cast<const uint4*>(a + p * as_) + g), av);
    unpack8(__ldg(reinterpret_cast<const uint4*>(c + p * cs) + g), cv);
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int ch = g * 8 + j;
      const float gm = gamma ? __ldg(gamma + ch) : 1.f;
      const float rs = __ldg(rstd + ch);
      if (use_batch_stats) {
        const float xh = (xv[j] - __ldg(mean + ch)) * rs;
        const float Sa = __ldg(sums + ch) * inv_count, Sc = __ldg(sums + C + ch) * inv_count;
        const float Sxa = __ldg(sums + 2 * C + ch) * inv_count, Sxc = __ldg(sums + 3 * C + ch) * inv_count;
        const float Sac = __ldg(sums + 4 * C + ch) * inv_count;
        const float T = Sa * Sc - Sac + 3.f * Sxa * Sxc;                      // all already divided by M once
        ox[j] = gm * rs * rs * (xh * T + Sxc * (Sa - av[j]) + Sxa * (Sc - cv[j]));
        oa[j] = gm * rs * (cv[j] - Sc - xh * Sxc);
      } else {
        ox[j] = 0.f;
        oa[j] = gm * rs * cv[j];
      }
    }
    if (dx) reinterpret_cast<uint4*>(dx + p * dxs)[g] = pack8(ox);
    if (da) reinterpret_cast<uint4*>(da + p * das)[g] = pack8(oa);
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_bn_stats(const void* x, int64_t npix, int32_t C, int64_t x_cstride, float* sum, float* sumsq,
                            sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && sum && sumsq && npix > 0 && C > 0 && C % 8 == 0 && x_cstride % 8 == 0);
  if (sumsq == sum + C) {                              // the usual case: one [2][C] buffer -> one memset node
    SGB_CUDA(cudaMemsetAsync(sum, 0, sizeof(float) * 2 * (size_t)C, stream));
  } else {
    SGB_CUDA(cudaMemsetAsync(sum, 0, sizeof(float) * C, stream));
    SGB_CUDA(cudaMemsetAsync(sumsq, 0, sizeof(float) * C, stream));
  }
  const int chunks = (C + kChunkC - 1) / kChunkC;
  long long target_blocks = 8LL * sm_count() / chunks;
  if (target_blocks < 1) target_blocks = 1;
  long long ppb = (npix + target_blocks - 1) / target_blocks;
  const int vgb = (C < kChunkC ? C : kChunkC) / 8 < 256 ? (C < kChunkC ? C : kChunkC) / 8 : 256;
  const long long ppb_min = 4LL * (256 / vgb);         // at least four pixels per thread row
  if (ppb < ppb_min) ppb = ppb_min;
  if (ppb < 16) ppb = 16;
  dim3 grid((unsigned)((npix + ppb - 1) / ppb), chunks);
  bn_stats_kernel<<<grid, 256, 0, stream>>>((const bf16*)x, npix, C, x_cstride, sum, sumsq, ppb);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_bn_finalize(const float* sum, const float* sumsq, float count, float* running_mean, float* running_var,
                               float momentum, float eps, int32_t use_batch_stats, int32_t track, int32_t mode,
                               const float* gain, const float* bias, int32_t nb, int32_t C, float* mean, float* rstd,
                               float* scale, float* shift, int64_t affine_ld, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(C > 0 && nb > 0 && mean && rstd && scale && shift && (affine_ld == 0 || affine_ld >= C));
  SGB_REQUIRE(use_batch_stats ? (sum && sumsq && count > 0.f) : (running_mean && running_var));
  SGB_REQUIRE(mode == 2 || (gain && bias));
  bn_finalize_kernel<<<dim3((C + 127) / 128, nb < 128 ? nb : 128), 128, 0, stream>>>(sum, sumsq, count, running_mean, running_var, momentum, eps,
                                                          use_batch_stats, track, mode, gain, bias, nb, C, mean, rstd, scale,
                                                          shift, affine_ld > 0 ? affine_ld : C);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_scale_shift_act(const void* x, int32_t B, int32_t H, int32_t W, int32_t C, int64_t x_cstride,
                                   const float* scale, const float* shift, int32_t per_image, int32_t relu, int32_t up2,
                                   void* y, int64_t y_cstride, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && y && scale && shift && B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0);
  SGB_REQUIRE(x_cstride % 8 == 0 && y_cstride % 8 == 0);
  SGB_REQUIRE(((uintptr_t)scale & 15) == 0 && ((uintptr_t)shift & 15) == 0);
  const long long total = (long long)B * H * W * (C / 8);
  scale_shift_act_kernel<<<ew_blocks(total), 256, 0, stream>>>((const bf16*)x, B, H, W, C, x_cstride, scale, shift,
                                                              per_image ? C : 0, relu, up2, (bf16*)y, y_cstride);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_bn_bwd_reduce(const void* dy, int64_t dy_cstride, const void* x, int64_t x_cstride, int32_t B, int32_t H,
                                 int32_t W, int32_t C, const float* scale, const float* shift, int32_t per_image,
                                 const float* mean, const float* rstd, int32_t relu, int32_t up2, float* s1, float* s2,
                                 float* S1, float* S2, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dy && x && scale && shift && mean && rstd && s1 && s2 && S1 && S2);
  SGB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && dy_cstride % 8 == 0 && x_cstride % 8 == 0);
  if (s2 == s1 + (size_t)B * C) {
    SGB_CUDA(cudaMemsetAsync(s1, 0, sizeof(float) * 2 * (size_t)B * C, stream));
  } else {
    SGB_CUDA(cudaMemsetAsync(s1, 0, sizeof(float) * (size_t)B * C, stream));
    SGB_CUDA(cudaMemsetAsync(s2, 0, sizeof(float) * (size_t)B * C, stream));
  }

  const int chunks = (C + kChunkC - 1) / kChunkC;
  const int HW = H * W;
  long long target = 8LL * sm_count() / ((long long)B * chunks);
  if (target < 1) target = 1;
  int ppb = (int)((HW + target - 1) / target);
  if (ppb < 32) ppb = 32;
  dim3 grid((HW + ppb - 1) / ppb, B, chunks);
  (up2 ? bn_bwd_reduce_kernel<true> : bn_bwd_reduce_kernel<false>)<<<grid, 256, 0, stream>>>(
      (const bf16*)dy, dy_cstride, (const bf16*)x, x_cstride, H, W, C, scale, shift, per_image ? C : 0, mean, rstd, relu, s1, s2,
      ppb);
  SGB_LAUNCH_CHECK();
  bn_bwd_total_kernel<<<(C + 7) / 8, 256, 0, stream>>>(s1, s2, scale, per_image ? C : 0, rstd, B, C, S1, S2);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_bn_bwd_apply(const void* dy, int64_t dy_cstride, const void* x, int64_t x_cstride, int32_t B, int32_t H,
                                int32_t W, int32_t C, const float* scale, const float* shift, int32_t per_image,
                                const float* mean, const float* rstd, const float* S1, const float* S2, float count,
                                int32_t relu, int32_t up2, int32_t use_batch_stats, void* dx, int64_t dx_cstride,
                                sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(dy && x && dx && scale && shift && mean && rstd);
  SGB_REQUIRE(!use_batch_stats || (S1 && S2 && count > 0.f));
  SGB_REQUIRE(B > 0 && H > 0 && W > 0 && C > 0 && C % 8 == 0 && dy_cstride % 8 == 0 && x_cstride % 8 == 0 && dx_cstride % 8 == 0);
  const int chunks = (C + kChunkC - 1) / kChunkC;
  const int HW = H * W;
  long long target = 16LL * sm_count() / ((long long)B * chunks);
  if (target < 1) target = 1;
  int ppb = (int)((HW + target - 1) / target);
  if (ppb < 64) ppb = 64;
  dim3 grid((HW + ppb - 1) / ppb, B, chunks);
  (up2 ? bn_bwd_apply_kernel<true> : bn_bwd_apply_kernel<false>)<<<grid, 256, 0, stream>>>(
      (const bf16*)dy, dy_cstride, (const bf16*)x, x_cstride, H, W, C, scale, shift, per_image ? C : 0, mean, rstd, S1, S2,
      use_batch_stats ? 1.f / count : 0.f, relu, use_batch_stats, (bf16*)dx, dx_cstride, ppb);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_bn_tangent_bwd_reduce(const void* x, int64_t xs, const void* a, int64_t as_, const void* c, int64_t cs,
                                         int64_t npix, int32_t C, const float* mean, const float* rstd, float* sums,
                                         sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && a && c && mean && rstd && sums && npix > 0 && C > 0 && C % 8 == 0);
  SGB_REQUIRE(xs % 8 == 0 && as_ % 8 == 0 && cs % 8 == 0);
  SGB_CUDA(cudaMemsetAsync(sums, 0, sizeof(float) * 5 * (size_t)C, stream));
  const int VG = C / 8, VGb = VG < 32 ? VG : 32;
  const int gy = (VG + VGb - 1) / VGb;
  long long target = 8LL * sm_count() / gy;
  if (target < 1) target = 1;
  long long ppb = (npix + target - 1) / target;
  if (ppb < 64) ppb = 64;
  dim3 grid((unsigned)((npix + ppb - 1) / ppb), gy);
  bn_tan_bwd_reduce_kernel<<<grid, 256, 0, stream>>>((const bf16*)x, xs, (const bf16*)a, as_, (const bf16*)c, cs, npix, C, mean, rstd,
                                                    sums, ppb);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_bn_tangent_bwd_apply(const void* x, int64_t xs, const void* a, int64_t as_, const void* c, int64_t cs,
                                        int64_t npix, int32_t C, const float* gamma, const float* mean, const float* rstd,
                                        const float* sums, float count, int32_t use_batch_stats, void* dx, int64_t dxs, void* da,
                                        int64_t das, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && a && c && mean && rstd && (dx || da) && npix > 0 && C > 0 && C % 8 == 0);
  SGB_REQUIRE(!use_batch_stats || (sums && count > 0.f));
  SGB_REQUIRE(xs % 8 == 0 && as_ % 8 == 0 && cs % 8 == 0 && (!dx || dxs % 8 == 0) && (!da || das % 8 == 0));
  bn_tan_bwd_apply_kernel<<<ew_blocks(npix * (C / 8)), 256, 0, stream>>>((const bf16*)x, xs, (const bf16*)a, as_, (const bf16*)c, cs,
                                                                        npix, C, gamma, mean, rstd, sums,
                                                                        use_batch_stats ? 1.f / count : 0.f, use_batch_stats,
                                                                        (bf16*)dx, dxs, (bf16*)da, das);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
