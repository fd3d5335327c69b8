// Weight gradient of 3x3 / pad 1 convolutions with 64 input channels (the widest-resolution layers of BigGAN-Deep: the
// generic wgrad kernel reloads dY and a shifted X tile for every one of the 9 taps).
//
//   dW[co][tap][ci] = sum_{b,h,w} dY[b,h,w,co] * X[b,h+dh,w+dw,ci]
//
// Formulation (pixels are the contraction dimension, all operands MN-major / SWIZZLE_128B):
//   A (M side) = X halo: one tile stages 4 halo rows x 130 pixels x 64 channels ONCE; tap (dh,dw) is the same buffer read
//                from pixel offset (dh+1)*130 + (dw+1) -- one 64-channel MN atom, M = 64.
//   B (N side) = dY tile, 2 rows x 128 pixels x Cout (<= 64) channels.
// Three consumer warpgroups, one filter row (kh) each: three taps x 64 x 64 fp32 accumulators in registers per warpgroup,
// accumulated over the CTA's whole pixel range and drained once with fp32 red.adds.  The bias gradient is one more small
// product on the first warpgroup: dY^T times a constant-ones operand.
#include "common.cuh"
#include "ptx.cuh"

namespace sgb {

static constexpr int kW3Consumers = 384;            // warpgroups 1..3: taps (kh, 0..2) for kh = warpgroup - 1
static constexpr int kW3Threads = 128 + kW3Consumers;   // warp 0 producer
static constexpr int kW3Px = 128;                   // pixels per tile row
static constexpr int kW3Halo = kW3Px + 2;           // halo row pitch in pixels
static constexpr uint32_t kW3DyBytes = 2 * kW3Px * 128;                       // 32 KB
static constexpr uint32_t kW3XBytes = 4 * kW3Halo * 128;                      // 66 560 B
static constexpr uint32_t kW3XAlloc = (kW3XBytes + 1023) / 1024 * 1024;
static constexpr uint32_t kW3Stage = kW3DyBytes + kW3XAlloc;
static constexpr int kW3Stages = 2;

struct W3Args {
  int H, W, Cin, Cout;           // Cin: channels of THIS launch's 64-wide input-channel block
  int dw_cin;                    // row pitch of dw (= the layer's full Cin)
  int tiles_w, tiles_h;          // tiles per row, row pairs per image
  long long tiles;               // B * tiles_h * tiles_w
  float* dw;
  float* dbias;                  // optional: sum of dY over all pixels
};

// Shared memory of wgrad3x3_c64_kernel: addresses from base, or offsets from the 1024-aligned base when base = 0.
struct W3Smem {
  uint32_t ring;                  // kW3Stages x (dY tile, X halo)
  uint32_t ones;                  // bf16 1.0 slab
  MbarRing ops;
  uint32_t total;
};
__host__ __device__ inline W3Smem w3_smem(uint32_t base = 0) {
  W3Smem L;
  L.ring = base;
  L.ones = L.ring + kW3Stages * kW3Stage;
  L.ops = {L.ones + kOnesSlabBytes, kW3Stages};
  L.total = L.ops.end() - base;
  return L;
}

// Consumer warpgroup of filter row kh: taps (kh, 0..2) over the CTA's tile range, then the red.add drain.  BIAS: this
// warpgroup also accumulates dY^T times a constant-ones operand (the bias gradient).
template <bool BIAS>
__device__ __forceinline__ void w3_consumer(const W3Args& p, const W3Smem& L, long long t_begin, long long t_end, int kh) {
  const int lane = threadIdx.x & 31;
  float acc[3][32], bacc[4];
#pragma unroll
  for (int k = 0; k < 3; ++k)
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[k][i] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) bacc[i] = 0.f;
  const uint64_t ones_desc = make_sdesc_sw128(L.ones, 16, 1024);   // K-major N = 8: every element is 1.0
  uint32_t it = 0;
  int prev = -1;
  for (long long t = t_begin; t < t_end; ++t, ++it) {
    const int s = L.ops.wait(it);
    const uint32_t ys = L.ring + s * kW3Stage;
    const uint32_t xs = ys + kW3DyBytes;
    wgmma_fence();
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const uint64_t bdesc = make_sdesc_sw128(ys + (uint32_t)(j * kW3Px) * 128u, 128 * kW3Px, 1024);
#pragma unroll
      for (int kw = 0; kw < 3; ++kw) {
        const uint64_t adesc = make_sdesc_sw128(xs + (uint32_t)((kh + j) * kW3Halo + kw) * 128u, 8192, 1024);
#pragma unroll
        for (int kk = 0; kk < kW3Px / 16; ++kk)   // 16 pixels (K) = two 8-row groups = 2048 bytes -> +128 in the (addr >> 4) field
          Wgmma<64>::mma<1, 1>(acc[kw], adesc + 128 * kk, bdesc + 128 * kk, 1u);
      }
      if constexpr (BIAS) {
#pragma unroll
        for (int kk = 0; kk < kW3Px / 16; ++kk) Wgmma<8>::mma<1, 0>(bacc, bdesc + 128 * kk, ones_desc, 1u);
      }
    }
    wgmma_commit();
    L.ops.release_prev(prev, s);
  }
  wgmma_wait<0>();
#pragma unroll
  for (int k = 0; k < 3; ++k) acc_fence(acc[k]);
  acc_fence(bacc);
  L.ops.release(prev);
  // drain: fragment rows = input channels, columns = output channels
  const int w = (threadIdx.x >> 5) & 3;
  const int ci0 = 16 * w + (lane >> 2), co0 = 2 * (lane & 3);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int ci = ci0 + 8 * hr;
    if (BIAS && (lane & 3) == 0 && ci < p.Cout) atomicAdd(p.dbias + ci, bacc[2 * hr]);   // bias fragment rows = output channels
    if (ci >= p.Cin) continue;
#pragma unroll
    for (int kw = 0; kw < 3; ++kw) {
      const int tap = kh * 3 + kw;
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int co = co0 + 8 * j + e;
          if (co < p.Cout) atomicAdd(p.dw + ((long long)co * 9 + tap) * p.dw_cin + ci, acc[kw][4 * j + 2 * hr + e]);
        }
    }
  }
}

__global__ void __launch_bounds__(kW3Threads, 1)
wgrad3x3_c64_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const W3Args p) {
  extern __shared__ uint8_t smem_raw[];
  const W3Smem L = w3_smem(smem_aligned(smem_raw));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
    L.ops.init(kW3Consumers / 32);
    fence_barrier_init();
  }
  if (p.dbias) fill_ones_slab(L.ones, kW3Threads);
  __syncthreads();

  // contiguous tile range of this CTA
  const long long t_begin = p.tiles * blockIdx.x / gridDim.x;
  const long long t_end = p.tiles * (blockIdx.x + 1) / gridDim.x;

  if (warp == 0) {
    if (lane == 0) {
      uint32_t it = 0;
      for (long long t = t_begin; t < t_end; ++t, ++it) {
        const int wt = (int)(t % p.tiles_w);
        const int ht = (int)((t / p.tiles_w) % p.tiles_h);
        const int b = (int)(t / ((long long)p.tiles_w * p.tiles_h));
        const int w0 = wt * kW3Px, h0 = ht * 2;
        const int s = L.ops.acquire(it, kW3DyBytes + kW3XBytes);
        const uint32_t sa = L.ring + s * kW3Stage;
        tma_load_4d(sa, &tmDY, L.ops.full(s), 0, w0, h0, b);
        tma_load_4d(sa + kW3DyBytes, &tmX, L.ops.full(s), 0, w0 - 1, h0 - 1, b);   // out-of-range halo = zero padding
      }
    }
  } else if (warp >= 4 && t_end > t_begin) {
    const int kh = (threadIdx.x - 128) >> 7;    // this warpgroup's filter row
    // the bias product is a compile-time property of the consumer body: a branch between the wgmmas would serialise them
    if (p.dbias != nullptr && kh == 0) w3_consumer<true>(p, L, t_begin, t_end, kh);
    else w3_consumer<false>(p, L, t_begin, t_end, kh);
  }
}

bool wgrad3x3_c64_eligible(const sgb_wgrad_desc* d) {
  // Cin > 64 (the generator's 128 -> 3 output convolution) runs as one launch per 64-channel block of the input
  return d->KH == 3 && d->KW == 3 && d->pad_h == 1 && d->pad_w == 1 && !d->per_image &&
         ((d->Cin <= 64 && d->Cin % 8 == 0) || (d->Cin % 64 == 0 && d->Cin <= 256 && d->Cout <= 16)) &&
         d->Cout <= 64 && d->Cout % 8 == 0 && d->W % kW3Px == 0 && d->H % 2 == 0 &&
         (long long)d->B * (d->H / 2) * (d->W / kW3Px) >= 64;
}

int launch_wgrad3x3_c64(const sgb_wgrad_desc* d, cudaStream_t stream) {
  if (!d->accumulate) {
    SGB_CUDA(cudaMemsetAsync(d->dw, 0, sizeof(float) * (size_t)d->Cout * 9 * d->Cin, stream));
    if (d->dbias) SGB_CUDA(cudaMemsetAsync(d->dbias, 0, sizeof(float) * (size_t)d->Cout, stream));
  }
  CUtensorMap tmDY;
  int rc = make_act_tmap(&tmDY, d->dy, d->B, d->H, d->W, d->Cout, d->dy_cstride, kW3Px, 2, 1);
  if (rc) return rc;
  const size_t smem = smem_request(w3_smem().total);
  for (int ci0 = 0; ci0 < d->Cin; ci0 += 64) {
    W3Args p;
    p.H = d->H; p.W = d->W; p.Cout = d->Cout;
    p.Cin = d->Cin - ci0 < 64 ? d->Cin - ci0 : 64;
    p.dw_cin = d->Cin;
    p.tiles_w = d->W / kW3Px;
    p.tiles_h = d->H / 2;
    p.tiles = (long long)d->B * p.tiles_h * p.tiles_w;
    p.dw = d->dw + ci0;
    p.dbias = ci0 == 0 ? d->dbias : nullptr;
    CUtensorMap tmX;
    rc = make_act_tmap(&tmX, (const bf16*)d->x + ci0, d->B, d->H, d->W, p.Cin, d->x_cstride, kW3Halo, 4, 1);
    if (rc) return rc;
    const int grid = p.tiles < sm_count() ? (int)p.tiles : sm_count();
    rc = launch_kernel<wgrad3x3_c64_kernel>(grid, kW3Threads, smem, stream, tmDY, tmX, p);
    if (rc) return rc;
  }
  return SGB_OK;
}

}  // namespace sgb
