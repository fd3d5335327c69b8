// Spectral normalisation: one power iteration, sigma, and emission of the tensor-core weight packs.
//
// Reference arithmetic (torch/nn/utils/spectral_norm.py:62-114, used by src/utils/ops.py:195-224 with eps=1e-6,
// n_power_iterations=1, dim=0):   v <- normalize(W^T u);  u <- normalize(W v);  sigma = u . (W v);  W_sn = W / sigma
// where W is the weight viewed as [R = out_channels, K = in_channels*kh*kw] and normalize(x) = x / max(||x||_2, eps).
// HBM-bound: two streaming passes over the fp32 weight for the iteration and one for the packs.
#include "common.cuh"

namespace sgb {

__device__ float block_sum(float v, float* sh) {
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = (threadIdx.x < (blockDim.x >> 5)) ? sh[threadIdx.x] : 0.f;
  if (w == 0) r = warp_sum(r);
  if (threadIdx.x == 0) sh[0] = r;
  __syncthreads();
  r = sh[0];
  return r;
}

// Every step below is written once, as a __device__ function of one layer, and runs in two kinds of launch:
//   per layer (sgb_sn_power_iter, sgb_weight_pack, sgb_sn_backward): the layer is a __grid_constant__ kernel parameter;
//   batched (sgb_sn_batch, sgb_sn_backward_batch): every layer of a network in one launch per step, layer
//     table[blockIdx.y] (the pack launch walks one work-unit index over all layers instead).  A BigGAN-Deep generator has
//     150+ such layers per forward, and dependent per-layer launches cost ~30 us each.
// A layer's blocks are those of grid.x; the power-iteration steps cap them at what the layer needs (its ticket counts them).

// ws layout (floats): [0..K) t = W^T u accumulator, [K..K+R) s = W v, [K+R] ticket A, [K+R+1] ticket B
// Step 1, t += W^T u: a block adds the (64-row x 256-column) tiles blockIdx.x, blockIdx.x + nblk, ... of the layer (the
// batched grid is capped at 4096 blocks, and a layer may have more tiles than that: an SN linear 16384 -> 4160 has 4160);
// the last block normalises t into v and clears t.
__device__ __forceinline__ void sn_wtu(const sgb_sn_layer& L, float eps) {
  __shared__ float sh[32];
  __shared__ bool last;
  const int R = L.R, K = L.K;
  const int col_blocks = (K + 255) / 256, rows_per_block = 64;
  const int row_blocks = (R + rows_per_block - 1) / rows_per_block;
  const unsigned total = (unsigned)col_blocks * row_blocks;
  const unsigned nblk = min((unsigned)gridDim.x, total);    // blocks taking part in this layer (and in its ticket)
  if (blockIdx.x >= nblk) return;
  const float* W = L.W;
  float* ws = L.ws;
  for (unsigned tile = blockIdx.x; tile < total; tile += nblk) {
    const int bx = (int)(tile % col_blocks), by = (int)(tile / col_blocks);
    const int c = bx * 256 + threadIdx.x;
    const int r0 = by * rows_per_block, r1 = min(r0 + rows_per_block, R);
    if (c < K) {
      float acc = 0.f;
      const float* wp = W + (size_t)r0 * K + c;
      for (int r = r0; r < r1; ++r, wp += K) acc = fmaf(__ldg(wp), __ldg(L.u + r), acc);
      atomicAdd(ws + c, acc);
    }
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned* ticket = reinterpret_cast<unsigned*>(ws + K + R);
    last = (atomicAdd(ticket, 1u) == nblk - 1);
    if (last) *ticket = 0u;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  float ss = 0.f;
  for (int i = threadIdx.x; i < K; i += 256) { const float t = __ldcg(ws + i); ss = fmaf(t, t, ss); }
  ss = block_sum(ss, sh);
  const float inv = 1.f / fmaxf(sqrtf(ss), eps);
  for (int i = threadIdx.x; i < K; i += 256) {
    L.v[i] = __ldcg(ws + i) * inv;
    ws[i] = 0.f;
  }
}

// Step 2, s = W v (one warp per row): the last block forms u = normalize(s) and *sigma = u . s, or (update_u = 0) only
// *sigma = u . s with the u the layer has.
__device__ __forceinline__ void sn_wv(const sgb_sn_layer& L, float* sigma, float eps, int update_u) {
  __shared__ float sh[32];
  __shared__ bool last;
  const int R = L.R, K = L.K;
  const unsigned nblk = min((unsigned)gridDim.x, (unsigned)((R + 7) / 8));
  if (blockIdx.x >= nblk) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* s = L.ws + K;
  for (int r = blockIdx.x * 8 + warp; r < R; r += nblk * 8) {
    const float* wp = L.W + (size_t)r * K;
    float acc = 0.f;
    for (int i = lane; i < K; i += 32) acc = fmaf(__ldg(wp + i), __ldcg(L.v + i), acc);
    acc = warp_sum(acc);
    if (lane == 0) s[r] = acc;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned* ticket = reinterpret_cast<unsigned*>(L.ws + K + R + 1);
    last = (atomicAdd(ticket, 1u) == nblk - 1);
    if (last) *ticket = 0u;
  }
  __syncthreads();
  if (!last) return;
  __threadfence();
  if (update_u) {
    float ss = 0.f;
    for (int i = threadIdx.x; i < R; i += 256) { const float t = __ldcg(s + i); ss = fmaf(t, t, ss); }
    ss = block_sum(ss, sh);
    const float inv = 1.f / fmaxf(sqrtf(ss), eps);
    for (int i = threadIdx.x; i < R; i += 256) L.u[i] = __ldcg(s + i) * inv;
    if (threadIdx.x == 0) *sigma = ss * inv;  // u . s = ||s||^2 / max(||s||, eps)
  } else {
    float d = 0.f;
    for (int i = threadIdx.x; i < R; i += 256) d = fmaf(__ldcg(s + i), L.u[i], d);
    d = block_sum(d, sh);
    if (threadIdx.x == 0) *sigma = d;
  }
}

// Packs: W is the module's weight [R = Cout][Cin][taps] (taps = kh*kw, row-major OIHW).
//   fprop pack  Wf[co][tap][ci]            = W[co][ci][tap] / sigma
//   dgrad pack  Wd[ci][taps-1-tap][co]     = W[co][ci][tap] / sigma     (180-degree rotated, in/out swapped)
// perm_S > 1 re-orders output rows for linear0, whose output is viewed as [C, S] by the reference
// (src/models/big_resnet_deep_legacy.py:167-168) but consumed here as NHWC [S, C]: packed row s*C + c <- row c*S + s.
// Tile t of a layer (taps <= 9) = 32 output channels x 32 input channels x all taps, (t / tiles_ci, t % tiles_ci), staged
// in shared memory so that the fp32 reads (one run of 32*taps floats per output channel) AND both bf16 writes are
// contiguous: the fprop pack [co][tap][ci] in runs of 32 ci, the dgrad pack [ci][taps-1-tap][co] in runs of 32 co.  A layer
// with more taps (4x4 filters of the DCGAN generator) has element-wise pseudo tiles of 4096 weights instead.
constexpr int kT = 32, kMaxTaps = 9;

__host__ __device__ inline int sn_pack_tiles(int Cout, int Cin, int taps) {
  return taps > kMaxTaps ? (int)(((unsigned)Cout * Cin * taps + 4095u) / 4096u) : ((Cout + kT - 1) / kT) * ((Cin + kT - 1) / kT);
}

__device__ __forceinline__ void sn_pack_tile(const sgb_sn_layer& L, int t, float inv, bf16* wf, bf16* wd) {
  __shared__ bf16 tile[kT][kT * kMaxTaps + 2];
  const int Cout = L.Cout, Cin = L.Cin, taps = L.taps, perm_S = L.perm_S;
  if (taps > kMaxTaps) {
    const unsigned total = (unsigned)Cout * Cin * taps;
    const unsigned e0 = (unsigned)t * 4096u, e1 = min(e0 + 4096u, total);
    for (unsigned i = e0 + threadIdx.x; i < e1; i += 256) {
      const int tap = (int)(i % taps);
      const int ci = (int)((i / taps) % Cin);
      int co = (int)(i / ((unsigned)taps * Cin));
      const bf16 v = __float2bfloat16_rn(__ldg(L.W + i) * inv);
      if (perm_S > 1) { const int C = Cout / perm_S; co = (co % perm_S) * C + co / perm_S; }
      if (wf) wf[((size_t)co * taps + tap) * L.Cin_p + ci] = v;
      if (wd) wd[((size_t)ci * taps + (taps - 1 - tap)) * L.Cout_p + co] = v;
    }
    return;
  }
  const int tiles_ci = (Cin + kT - 1) / kT;
  const int run = kT * taps;                      // source elements per output channel inside one tile
  const int co0 = (t / tiles_ci) * kT, ci0 = (t % tiles_ci) * kT;
  const int nci = min(kT, Cin - ci0), nco = min(kT, Cout - co0);
  __syncthreads();
  // read: row r of the tile = source channel co0 + r, elements (ci0*taps .. (ci0+nci)*taps) contiguous in memory
  for (int e = threadIdx.x; e < kT * run; e += 256) {
    const int r = e / run, k = e % run;
    if (r < nco && k < nci * taps)
      tile[r][k] = __float2bfloat16_rn(__ldg(L.W + ((size_t)(co0 + r) * Cin + ci0) * taps + k) * inv);
  }
  __syncthreads();
  if (wf) {   // [co][tap][ci]: runs of nci consecutive ci
    for (int e = threadIdx.x; e < kT * run; e += 256) {
      const int r = e / run, rem = e % run;
      const int tap = rem / kT, c = rem % kT;
      if (r < nco && c < nci) {
        int co = co0 + r;
        if (perm_S > 1) { const int C = Cout / perm_S; co = (co % perm_S) * C + co / perm_S; }
        wf[((size_t)co * taps + tap) * L.Cin_p + ci0 + c] = tile[r][c * taps + tap];
      }
    }
  }
  if (wd) {   // [ci][taps-1-tap][co]: runs of nco consecutive co (perm_S > 1 only permutes the rows of linear0: scattered there)
    for (int e = threadIdx.x; e < kT * run; e += 256) {
      const int k = e / kT, r = e % kT;          // k = c * taps + tap
      const int c = k / taps, tap = k % taps;
      if (r < nco && c < nci) {
        int co = co0 + r;
        if (perm_S > 1) { const int C = Cout / perm_S; co = (co % perm_S) * C + co / perm_S; }
        wd[((size_t)(ci0 + c) * taps + (taps - 1 - tap)) * L.Cout_p + co] = tile[r][k];
      }
    }
  }
}

// Backward of W_sn = W / sigma with u, v held constant (they are detached buffers in the reference):
//   dL/dW = (G - <G, W_sn> u v^T) / sigma,  G given in the fprop pack layout [co][tap][ci] (fp32, from wgrad).
// Both steps walk a layer row by row, block blockIdx.x taking rows blockIdx.x, blockIdx.x + gridDim.x, ... (row = one
// output channel: Cin * taps contiguous floats of W / dW, and the contiguous [taps][Cin_p] block of G).  For taps > 1 the G
// row is staged in shared memory so that the global reads of G, W and the read-modify-write of dW are all coalesced.
static constexpr int kSnRowFloats = 8192;          // 32 KiB: 512 channels x 16 taps

__device__ __forceinline__ int sn_g_row(const sgb_snbwd_layer& L, int co_orig) {
  if (L.perm_S > 1) { const int C = L.Cout / L.perm_S; return (co_orig % L.perm_S) * C + co_orig / L.perm_S; }
  return co_orig;
}

// The layer's G, u, v sit at g_flat + off_g, u_flat + off_u, v_flat + off_v (a per-layer launch passes them with zero offsets).
// *dot += <G, W> over the block's rows.
__device__ __forceinline__ void sn_bwd_dot(const sgb_snbwd_layer& L, const float* __restrict__ g_flat, float* dot) {
  __shared__ float sh[32];
  __shared__ float grow[kSnRowFloats];
  const int taps = L.taps, Cin = L.Cin, K = Cin * taps, GK = taps * L.Cin_p;
  const bool staged = taps > 1 && GK <= kSnRowFloats;
  float acc = 0.f;
  for (int r = blockIdx.x; r < L.Cout; r += gridDim.x) {
    const float* Gr = g_flat + L.off_g + (size_t)sn_g_row(L, r) * GK;
    const float* W = L.W + (size_t)r * K;
    if (taps == 1) {
      for (int k = threadIdx.x; k < K; k += 256) acc = fmaf(__ldg(Gr + k), __ldg(W + k), acc);
    } else if (staged) {
      __syncthreads();
      for (int k = threadIdx.x; k < GK; k += 256) grow[k] = __ldg(Gr + k);
      __syncthreads();
      for (int k = threadIdx.x; k < K; k += 256) {
        const int ci = k / taps, tap = k - ci * taps;
        acc = fmaf(grow[tap * L.Cin_p + ci], __ldg(W + k), acc);
      }
    } else {
      for (int k = threadIdx.x; k < K; k += 256) {
        const int ci = k / taps, tap = k - ci * taps;
        acc = fmaf(__ldg(Gr + (size_t)tap * L.Cin_p + ci), __ldg(W + k), acc);
      }
    }
  }
  acc = block_sum(acc, sh);
  if (threadIdx.x == 0 && acc != 0.f) atomicAdd(dot, acc);
}

// dW (=|+=) (G - (*dot / sigma) u v^T) / sigma over the block's rows; a layer without spectral norm (has_sn = 0) reads
// none of sigma, dot, u, v and re-lays G out.
__device__ __forceinline__ void sn_bwd_apply(const sgb_snbwd_layer& L, const float* __restrict__ g_flat, const float* __restrict__ sigma,
                                             const float* __restrict__ dot, const float* __restrict__ u_flat,
                                             const float* __restrict__ v_flat, bool accumulate) {
  __shared__ float grow[kSnRowFloats];
  const int taps = L.taps, Cin = L.Cin, K = Cin * taps, GK = taps * L.Cin_p;
  const bool staged = taps > 1 && GK <= kSnRowFloats;
  float inv = 1.f, coef = 0.f;
  const float* u = nullptr;
  const float* v = nullptr;
  if (L.has_sn) {
    inv = 1.f / __ldg(sigma);
    coef = __ldg(dot) * inv;  // <G, W> / sigma = <G, W_sn>
    u = u_flat + L.off_u;
    v = v_flat + L.off_v;
  }
  for (int r = blockIdx.x; r < L.Cout; r += gridDim.x) {
    const float* Gr = g_flat + L.off_g + (size_t)sn_g_row(L, r) * GK;
    float* dW = L.dW + (size_t)r * K;
    const float cu = L.has_sn ? coef * __ldg(u + r) : 0.f;
    if (staged) {
      __syncthreads();
      for (int k = threadIdx.x; k < GK; k += 256) grow[k] = __ldg(Gr + k);
      __syncthreads();
    }
    for (int k = threadIdx.x; k < K; k += 256) {
      float g;
      if (taps == 1) {
        g = __ldg(Gr + k);
      } else {
        const int ci = k / taps, tap = k - ci * taps;
        g = staged ? grow[tap * L.Cin_p + ci] : __ldg(Gr + (size_t)tap * L.Cin_p + ci);
      }
      if (L.has_sn) g = (g - cu * __ldg(v + k)) * inv;
      dW[k] = accumulate ? dW[k] + g : g;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------------
// Per-layer launches
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sn_wtu_layer_kernel(const __grid_constant__ sgb_sn_layer L, float eps) { sn_wtu(L, eps); }

__global__ void __launch_bounds__(256) sn_wv_layer_kernel(const __grid_constant__ sgb_sn_layer L, float* __restrict__ sigma,
                                                          float eps, int update_u) {
  sn_wv(L, sigma, eps, update_u);
}

__global__ void __launch_bounds__(256) sn_pack_layer_kernel(const __grid_constant__ sgb_sn_layer L, const float* __restrict__ sigma,
                                                            bf16* __restrict__ wf, bf16* __restrict__ wd) {
  const float inv = sigma ? 1.f / __ldg(sigma) : 1.f;
  const int tiles = sn_pack_tiles(L.Cout, L.Cin, L.taps);
  for (int t = blockIdx.x; t < tiles; t += gridDim.x) sn_pack_tile(L, t, inv, wf, wd);
}

__global__ void __launch_bounds__(256) sn_bwd_dot_layer_kernel(const __grid_constant__ sgb_snbwd_layer L, const float* __restrict__ G,
                                                               float* __restrict__ dot) {
  sn_bwd_dot(L, G, dot);
}

__global__ void __launch_bounds__(256) sn_bwd_apply_layer_kernel(const __grid_constant__ sgb_snbwd_layer L, const float* __restrict__ G,
                                                                 const float* __restrict__ sigma, const float* __restrict__ dot,
                                                                 const float* __restrict__ u, const float* __restrict__ v,
                                                                 int accumulate) {
  sn_bwd_apply(L, G, sigma, dot, u, v, accumulate != 0);
}

// ---------------------------------------------------------------------------------------------------------------------
// Batched launches (blockIdx.y = layer)
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) sn_wtu_batch_kernel(const sgb_sn_layer* __restrict__ table, float eps) {
  const sgb_sn_layer L = table[blockIdx.y];
  if (L.has_sn) sn_wtu(L, eps);
}

__global__ void __launch_bounds__(256) sn_wv_batch_kernel(const sgb_sn_layer* __restrict__ table, float* __restrict__ sigma_all,
                                                           float eps, int update_u) {
  const sgb_sn_layer L = table[blockIdx.y];
  if (!L.has_sn) {
    if (blockIdx.x == 0 && threadIdx.x == 0) sigma_all[blockIdx.y] = 1.f;
    return;
  }
  sn_wv(L, sigma_all + blockIdx.y, eps, update_u);
}

// Work decomposition: ONE global index over the work units of all layers (table[l].tile_start = units of the layers before
// l); a block owns a contiguous range of it.  A unit is ~1024 weights: a tile of a k-tap layer is k units, a pseudo tile 4,
// so that contiguous unit ranges are balanced; a tile belongs to the block whose range holds its first unit.  (A
// (max tiles) x (layers) grid launched ~300 k blocks of which most returned at once: most of the call's time.)
__global__ void __launch_bounds__(256) sn_pack_batch_kernel(const sgb_sn_layer* __restrict__ table, int n_layers, int total_tiles,
                                                             const float* __restrict__ sigma_all, bf16* __restrict__ pack_f,
                                                             bf16* __restrict__ pack_d) {
  const int u0 = (int)((long long)total_tiles * blockIdx.x / gridDim.x);
  const int u1 = (int)((long long)total_tiles * (blockIdx.x + 1) / gridDim.x);
  if (u0 >= u1) return;
  int lo = 0, hi = n_layers - 1;
  while (lo < hi) {                                // last layer whose first unit is <= u0
    const int mid = (lo + hi + 1) >> 1;
    if (table[mid].tile_start <= u0) lo = mid; else hi = mid - 1;
  }
  int l = lo;
  sgb_sn_layer L = table[l];
  int next_start = (l + 1 < n_layers) ? table[l + 1].tile_start : total_tiles;
  float inv = 1.f / __ldcg(sigma_all + l);
  int upt = L.taps > kMaxTaps ? 4 : L.taps;        // units per tile of the current layer
  int t = (u0 - L.tile_start + upt - 1) / upt;     // first tile starting at or after u0
  for (;;) {
    int ustart = L.tile_start + t * upt;
    while (ustart >= next_start && l + 1 < n_layers) {   // next layer (layers without tiles are skipped here)
      ++l;
      L = table[l];
      next_start = (l + 1 < n_layers) ? table[l + 1].tile_start : total_tiles;
      inv = 1.f / __ldcg(sigma_all + l);
      upt = L.taps > kMaxTaps ? 4 : L.taps;
      t = 0;
      ustart = L.tile_start;
    }
    if (ustart >= u1 || ustart >= next_start) break;
    sn_pack_tile(L, t, inv, pack_f ? pack_f + L.off_f : nullptr, pack_d ? pack_d + L.off_d : nullptr);
    ++t;
  }
}

// Chain rule of EVERY layer of a network pass.  G lives in one flat fp32 buffer laid out like the fprop packs (layer l at
// g_flat + off_g); u / v / sigma are the copies taken at that forward pass (flat arenas, per-layer offsets in the table).
// Layers that produced no weight gradient in this pass hold zeros in g_flat and add zero.
__global__ void __launch_bounds__(256) sn_bwd_dot_batch_kernel(const sgb_snbwd_layer* __restrict__ table,
                                                                const float* __restrict__ g_flat, float* __restrict__ dots) {
  const sgb_snbwd_layer L = table[blockIdx.y];
  if (!L.has_sn || !L.dW) return;
  sn_bwd_dot(L, g_flat, dots + blockIdx.y);
}

__global__ void __launch_bounds__(256) sn_bwd_apply_batch_kernel(const sgb_snbwd_layer* __restrict__ table,
                                                                  const float* __restrict__ g_flat, const float* __restrict__ dots,
                                                                  const float* __restrict__ sigma_all, const float* __restrict__ u_flat,
                                                                  const float* __restrict__ v_flat) {
  const sgb_snbwd_layer L = table[blockIdx.y];
  if (!L.dW) return;
  sn_bwd_apply(L, g_flat, sigma_all + blockIdx.y, dots + blockIdx.y, u_flat, v_flat, true);
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_sn_backward_batch(const sgb_snbwd_layer* table, int32_t n_layers, const float* g_flat, const float* sigma_all,
                                     const float* u_flat, const float* v_flat, float* dots, int32_t max_blocks,
                                     sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(table && n_layers > 0 && g_flat && dots && max_blocks > 0);
  SGB_CUDA(cudaMemsetAsync(dots, 0, sizeof(float) * (size_t)n_layers, stream));
  sn_bwd_dot_batch_kernel<<<dim3(max_blocks, n_layers), 256, 0, stream>>>(table, g_flat, dots);
  SGB_LAUNCH_CHECK();
  sn_bwd_apply_batch_kernel<<<dim3(max_blocks, n_layers), 256, 0, stream>>>(table, g_flat, dots, sigma_all, u_flat, v_flat);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_sn_batch(const sgb_sn_layer* table, int32_t n_layers, float* sigma_all, void* pack_f, void* pack_d, float eps,
                            int32_t do_power_iteration, int32_t max_blocks_wtu, int32_t max_blocks_wv, int32_t max_blocks_pack,
                            sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(table && n_layers > 0 && sigma_all && max_blocks_wtu > 0 && max_blocks_wv > 0 && max_blocks_pack > 0);
  if (do_power_iteration) {
    sn_wtu_batch_kernel<<<dim3(max_blocks_wtu, n_layers), 256, 0, stream>>>(table, eps);
    SGB_LAUNCH_CHECK();
  }
  sn_wv_batch_kernel<<<dim3(max_blocks_wv, n_layers), 256, 0, stream>>>(table, sigma_all, eps, do_power_iteration);
  SGB_LAUNCH_CHECK();
  if (pack_f || pack_d) {
    // max_blocks_pack carries the total tile count of the table (sum over layers, see sgb_sn_layer.tile_start)
    const int total_tiles = max_blocks_pack;
    const int blocks = total_tiles < 32 * sm_count() ? total_tiles : 32 * sm_count();   // 4 waves of resident blocks: dynamic balance
    sn_pack_batch_kernel<<<blocks, 256, 0, stream>>>(table, n_layers, total_tiles, sigma_all, (bf16*)pack_f, (bf16*)pack_d);
    SGB_LAUNCH_CHECK();
  }
  return SGB_OK;
}

extern "C" int64_t sgb_sn_workspace_floats(int32_t R, int32_t K) { return (int64_t)R + K + 4; }

extern "C" int sgb_sn_power_iter(const float* W, float* u, float* v, float* sigma, float* ws, int32_t R, int32_t K,
                                 float eps, int32_t do_power_iteration, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(W && u && v && sigma && ws && R > 0 && K > 0);
  sgb_sn_layer L = {};
  L.W = W;
  L.u = u;
  L.v = v;
  L.ws = ws;
  L.R = R;
  L.K = K;
  L.has_sn = 1;
  if (do_power_iteration) {
    sn_wtu_layer_kernel<<<((K + 255) / 256) * ((R + 63) / 64), 256, 0, stream>>>(L, eps);   // one block per W^T u tile
    SGB_LAUNCH_CHECK();
  }
  int blocks = (R + 7) / 8;
  if (blocks > 4 * sm_count()) blocks = 4 * sm_count();
  sn_wv_layer_kernel<<<blocks, 256, 0, stream>>>(L, sigma, eps, do_power_iteration);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_weight_pack(const float* W, const float* sigma, void* w_fprop, void* w_dgrad, int32_t Cout, int32_t Cin,
                               int32_t taps, int32_t perm_S, int32_t Cout_p, int32_t Cin_p, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(W && (w_fprop || w_dgrad) && Cout > 0 && Cin > 0 && taps > 0);
  SGB_REQUIRE(perm_S <= 1 || Cout % perm_S == 0);
  SGB_REQUIRE(Cout_p >= Cout && Cin_p >= Cin);
  SGB_REQUIRE((size_t)Cout * Cin * taps <= 0xffffffffu);   // pseudo tiles index the weight with 32-bit unsigned
  sgb_sn_layer L = {};
  L.W = W;
  L.Cout = Cout;
  L.Cin = Cin;
  L.taps = taps;
  L.perm_S = perm_S;
  L.Cout_p = Cout_p;
  L.Cin_p = Cin_p;
  const int tiles = sn_pack_tiles(Cout, Cin, taps);
  const int blocks = tiles < 32 * sm_count() ? tiles : 32 * sm_count();
  sn_pack_layer_kernel<<<blocks, 256, 0, stream>>>(L, sigma, (bf16*)w_fprop, (bf16*)w_dgrad);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_sn_backward(const float* G, const float* W, const float* u, const float* v, const float* sigma,
                               float* scratch_dot, float* dW, int32_t Cout, int32_t Cin, int32_t taps, int32_t perm_S,
                               int32_t Cin_p, int32_t accumulate, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(G && dW && Cout > 0 && Cin > 0 && taps > 0);
  SGB_REQUIRE(!sigma || (W && u && v && scratch_dot));
  SGB_REQUIRE(Cin_p >= Cin);
  sgb_snbwd_layer L = {};
  L.W = W;
  L.dW = dW;
  L.Cout = Cout;
  L.Cin = Cin;
  L.taps = taps;
  L.perm_S = perm_S;
  L.Cin_p = Cin_p;
  L.has_sn = sigma != nullptr;
  const int blocks = Cout < 4 * sm_count() ? Cout : 4 * sm_count();   // one block per row
  if (sigma) {
    SGB_CUDA(cudaMemsetAsync(scratch_dot, 0, sizeof(float), stream));
    sn_bwd_dot_layer_kernel<<<blocks, 256, 0, stream>>>(L, G, scratch_dot);
    SGB_LAUNCH_CHECK();
  }
  sn_bwd_apply_layer_kernel<<<blocks, 256, 0, stream>>>(L, G, sigma, scratch_dot, u, v, accumulate);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
