// Implicit-GEMM convolution / linear / dgrad / wgrad on Hopper tensor cores (wgmma).
//
//   fprop : D[pixel, co]   = sum_{tap, ci}  X[pixel + tap, ci] * Wp[co, tap, ci]
//           A = X  tile, TMA 4-D box (64 ch, tw, th, nb) over NHWC   -> smem [128 px][64 ch], K-major, SWIZZLE_128B
//           B = Wp tile, TMA 3-D box (64 ci, 1 tap, BN co)           -> smem [BN co][64 ci],  K-major, SWIZZLE_128B
//           padding = TMA out-of-bounds zero fill (negative / overflowing box coordinates).
//   wgrad : D[co, ci]      = sum_{pixel}    dY[pixel, co] * X[pixel + tap, ci]           (one tap per work item)
//           A = dY tile(s), B = X tile(s): same boxes, consumed as MN-major operands (the pixel axis is K).
//
// One persistent CTA per SM, 3 warpgroups: warp 0 = TMA producer (one lane), warp 2 = auxiliary-operand producer (fprop),
// warpgroups 1 and 2 = consumers.  The producer warpgroup drops to 40 registers (setmaxnreg), the consumers rise to 232.
// fprop, compile-time epilogue variants: ping-pong.  Each consumer warpgroup owns whole tiles (local tile i -> warpgroup
// i & 1), issues two m64 wgmmas per K step (rows 0..63 / 64..127, 128 accumulator registers at BN = 128) and, once its main
// loop is done, hands the tensor cores to the other warpgroup (named barriers) and runs the fused epilogue straight from its
// registers: per 64-channel chunk and 64-row half, bf16 pairs into its own staging tiles and one TMA store; residual / mask /
// softmax-P boxes arrive through its own aux ring; the attention softmax's row reductions run within the lane quads of the
// accumulator fragment.  The operand ring stays one ring in tile order.
// fprop, run-time flags (F = -1): both warpgroups run every tile (64 rows each), stage the accumulator tile in shared memory as
// fp32 rows and run the epilogue on it (one thread = one row).
// wgrad: each consumer warpgroup owns 64 of the tile's 128 rows; fp32 red.adds straight from the accumulator registers.
#include "common.cuh"
#include "ptx.cuh"
#include "conv_epilogue.cuh"

namespace sgb {

static constexpr int kConsumerThreads = 256;              // two consumer warpgroups, M = 64 rows each
static constexpr int kConsumerWarps = kConsumerThreads / 32;
static constexpr int kThreads = 128 + kConsumerThreads;   // warpgroup 0: producers (warps 0 / 2), warpgroups 1..2: MMA + epilogue
static constexpr int kWgradThreads = kThreads;
static constexpr int kTileM = 128;          // pixels (fprop) or output channels (wgrad) per tile
static constexpr int kBlockK = 64;          // bf16 elements per 128-byte swizzle row
static constexpr int kABytes = kTileM * kBlockK * 2;  // 16 KiB
static constexpr uint32_t kAccBar = 3;      // named barrier of the 256 consumer threads (1, 2: epilogue teams)

struct FpropArgs {
  int B, H, W, Cin, Cout, taps, KW, pad_h, pad_w;
  int tw, th, nb;                 // tile box: tw*th*nb == 128
  int tiles_w, tiles_h, tiles_b, tiles_n, num_tiles;
  int kblocks;                    // ceil(Cin / 64)
  int BN;                         // output-channel tile: 16, 32, 64 or 128
  int w_mode;                     // 0: shared weights [Cout][taps][Cin]; 1: per-image [B][N][K]; 2: per-image MN-major [B][K][N]
  int stages;
  int use_tma;                    // epilogue through staging tiles + TMA tensor stores
  int epi_nbuf;                   // staging tiles per epilogue team (2: stores overlap the next chunk's conversion)
  int b_resident;                 // 1: every weight tile of this CTA's channel tile stays in shared memory (loaded once)
  int aux_kind, aux_tw, aux_th;   // residual (1) / mask (2) / softmax P (3) tile staged by TMA; box aux_tw x aux_th x nb pixels
  int aux_depth;                  // aux tiles per epilogue team (ring filled by the aux producer warp)
  int out_sub;                    // 2: store only even (h, w) outputs at (h/2, w/2) -> stride-2 convolution (Inception reduction blocks)
  EpiArgs e;
};

// Tile index -> (channel tile, w / h / batch tile of the (tw, th, nb) box), channel tiles fastest.
struct FpropTile { int nt, wt, ht, bt; };
__device__ __forceinline__ FpropTile fprop_tile(const FpropArgs& p, int t) {
  FpropTile c;
  c.nt = t % p.tiles_n; t /= p.tiles_n;
  c.wt = t % p.tiles_w; t /= p.tiles_w;
  c.ht = t % p.tiles_h; t /= p.tiles_h;
  c.bt = t;
  return c;
}

__host__ __device__ constexpr bool fprop_is_pingpong(int f) { return f >= 0; }

// Shared memory of conv_fprop_kernel: addresses from base, or offsets from the 1024-aligned base when base = 0.  Every tile
// region is a multiple of 1024 bytes (b_bytes too: BN % 8 == 0).
struct FpropSmem {
  uint32_t epi;                   // staging tiles of the two epilogue teams (use_tma)
  uint32_t aux;                   // aux tiles, aux_depth per team (aux_kind)
  uint32_t bres;                  // resident weight tiles [tap][kb] (b_resident)
  uint32_t acc;                   // fp32 accumulator rows of the tile (staged schedule)
  uint32_t ring;                  // operand ring: stages x (A tile, B tile unless resident)
  uint32_t stage_bytes, b_bytes;
  MbarRing ops, bres_ready, aux0; // barriers: operand ring, resident filter (one slot, filled once), team 0's aux ring
  uint32_t total;
  __host__ __device__ MbarRing aux_ring(int team) const { return {aux0.bar + MbarRing::bytes(aux0.slots) * team, aux0.slots}; }
};
__host__ __device__ inline FpropSmem fprop_smem(const FpropArgs& p, bool pingpong, uint32_t base = 0) {
  FpropSmem L;
  L.b_bytes = (uint32_t)p.BN * kBlockK * 2;   // same size for K-major [BN][64] and MN-major (BN/64) x [64][64]
  L.stage_bytes = kABytes + (p.b_resident ? 0u : L.b_bytes);
  L.epi = base;
  L.aux = L.epi + (p.use_tma ? 2u * p.epi_nbuf * (pingpong ? kFragStageBytes : kEpiStageBytes) : 0u);
  L.bres = L.aux + (p.aux_kind ? 2u * p.aux_depth * kEpiStageBytes : 0u);
  L.acc = L.bres + (p.b_resident ? (uint32_t)(p.taps * p.kblocks) * L.b_bytes : 0u);
  L.ring = L.acc + (pingpong ? 0u : (uint32_t)kTileM * acc_row_bytes(p.BN));   // 128 rows x (16 mod 1024) B
  L.ops = {L.ring + (uint32_t)p.stages * L.stage_bytes, p.stages};
  L.bres_ready = {L.ops.end(), 1};
  L.aux0 = {L.bres_ready.end(), p.aux_depth};
  L.total = L.aux_ring(1).end() - base;
  return L;
}

// Main loop of one fprop tile on one consumer warpgroup: per 16-wide K step, M m64 wgmmas against the same B tile, row block h
// of the A tile at a_off + h * 8 KiB -> acc[h].  it = the tile's first position in the operand ring.
template <int BN, int M>
__device__ __forceinline__ void fprop_mma(const FpropArgs& p, const FpropSmem& L, float (&acc)[M][BN / 2], uint32_t a_off, uint32_t it) {
#pragma unroll
  for (int h = 0; h < M; ++h)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[h][i] = 0.f;
  const bool b_mn = (p.w_mode == 2);
  const int kiters = p.taps * p.kblocks;
  int prev = -1;
  for (int k = 0; k < kiters; ++k, ++it) {
    const int s = L.ops.wait(it);
    const uint32_t sa = L.ring + s * L.stage_bytes;
    const uint64_t adesc = make_sdesc_sw128(sa + a_off, 16, 1024);          // [128][64]; row block h is 8 KiB further
    // K-major B: rows = output channels, +32 B per 16-wide K step.
    // MN-major B: (BN/64) atoms of [64 k-rows][64 n] 8 KiB apart (LBO), 8-row groups 1 KiB apart (SBO), +2 KiB per K step.
    const uint32_t sb = p.b_resident ? L.bres + (uint32_t)k * L.b_bytes : sa + kABytes;     // k = tap * kblocks + kb
    wgmma_fence();
    if (b_mn) {
      const uint64_t bdesc = make_sdesc_sw128(sb, 8192, 1024);
#pragma unroll
      for (int kk = 0; kk < kBlockK / 16; ++kk)
#pragma unroll
        for (int h = 0; h < M; ++h)
          Wgmma<BN>::template mma<0, 1>(acc[h], adesc + 512 * h + 2 * kk, bdesc + 128 * kk, (k > 0 || kk > 0) ? 1u : 0u);
    } else {
      const uint64_t bdesc = make_sdesc_sw128(sb, 16, 1024);
#pragma unroll
      for (int kk = 0; kk < kBlockK / 16; ++kk)
#pragma unroll
        for (int h = 0; h < M; ++h)
          Wgmma<BN>::template mma<0, 0>(acc[h], adesc + 512 * h + 2 * kk, bdesc + 2 * kk, (k > 0 || kk > 0) ? 1u : 0u);
    }
    wgmma_commit();
    L.ops.release_prev(prev, s);              // the previous K block's MMAs have retired: its ring slot is free
  }
  wgmma_wait<0>();
#pragma unroll
  for (int h = 0; h < M; ++h) acc_fence(acc[h]);
  L.ops.release(prev);
}

// Staged schedule: the main loop of this consumer warpgroup's 64 rows (64 wg .. 64 wg + 63) of the tile, then its accumulators
// -> shared memory.
template <int BN>
__device__ __forceinline__ void fprop_staged_mma(const FpropArgs& p, const FpropSmem& L, uint32_t it, int wg) {
  float acc[1][BN / 2];
  fprop_mma<BN, 1>(p, L, acc, (uint32_t)wg * 8192u, it);
  named_bar_sync(kAccBar, kConsumerThreads);  // every consumer is done reading the previous tile's staged accumulators
  acc_store<BN>(acc[0], L.acc + (uint32_t)wg * 64u * acc_row_bytes(BN), acc_row_bytes(BN));
  named_bar_sync(kAccBar, kConsumerThreads);
}

// ------------------------------------------------------------------------------------------------ fprop, ping-pong schedule
// Compile-time epilogue variants: each consumer warpgroup owns whole 128-row tiles (local tile i goes to warpgroup i & 1) and
// runs the epilogue straight from its registers while the other warpgroup issues its MMAs.
static constexpr uint32_t kTurnBar = 4;       // named barriers 4 / 5: warpgroup 0 / 1 may start its next mainloop

// One consumer warpgroup of the ping-pong schedule.  The two warpgroups' main loops take turns (named barriers kTurnBar + wg),
// so warpgroup A's epilogue runs under warpgroup B's MMAs.  The epilogue stores the tile as two 64-row half boxes per
// 64-channel chunk through this warpgroup's staging tiles; a residual / mask / softmax-P chunk arrives in this warpgroup's aux
// ring as one box of the whole tile, read by both halves.  The softmax statistics pass stores only its row partials.
template <int F, int BN>
__device__ __forceinline__ void fprop_pp_consumer(const FpropArgs& p, const CUtensorMap* tmY, const FpropSmem& L, int wg) {
  constexpr int aux_kind = (F & kEpiAuxRes) ? 1 : ((F & kEpiAuxMask) ? 2 : ((F & kEpiSmBwd) ? 3 : 0));
  constexpr bool sm_stats = (F & kEpiSmStats) != 0, sm_apply = (F & kEpiSmApply) != 0, sm_bwd = (F & kEpiSmBwd) != 0;
  const uint32_t w = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const bool leader = (threadIdx.x & 127) == 0;
  const float alpha = epi_alpha(p.e);
  // the half box splits the outermost non-unit dimension of (tw, th, nb): 0 = w, 1 = h, 2 = b
  const int split = p.nb > 1 ? 2 : (p.th > 1 ? 1 : 0);
  // tile coordinates and aux-box row of this thread's four rows: half h, fragment row hr -> tile row 64 h + 16 w + lane / 4 + 8 hr
  int wi[2][2], hi[2][2], bi[2][2];
  uint32_t arow[2][2];
  const bool aux_half = aux_kind == 1 && p.e.res_up2;
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const int row = 64 * h + 16 * (int)w + (int)(lane >> 2) + 8 * hr;
      wi[h][hr] = row % p.tw; hi[h][hr] = (row / p.tw) % p.th; bi[h][hr] = row / (p.tw * p.th);
      arow[h][hr] = aux_half ? (uint32_t)((bi[h][hr] * p.aux_th + (p.aux_th == p.th ? hi[h][hr] : (hi[h][hr] >> 1))) * p.aux_tw + (wi[h][hr] >> 1))
                             : (uint32_t)row;
    }
  const uint32_t stage = L.epi + (uint32_t)(wg * p.epi_nbuf) * kFragStageBytes;
  const uint32_t aux_tiles = L.aux + (uint32_t)(wg * p.aux_depth) * kEpiStageBytes;
  const MbarRing aux = L.aux_ring(wg);
  const int kiters = p.taps * p.kblocks;
  const int n_local = (p.num_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // this CTA's tiles
  uint32_t sbuf = 0, aux_cnt = 0;
  if (p.b_resident) L.bres_ready.wait(0);
  for (int i = wg; i < n_local; i += 2) {
    const FpropTile tc = fprop_tile(p, (int)blockIdx.x + i * (int)gridDim.x);
    const int nt = tc.nt, wt = tc.wt, ht = tc.ht, bt = tc.bt;
    long long pix[2][2], rpix[2][2];
    bool valid[2][2];
    int c1[2], c2[2], c3[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      c1[h] = wt * p.tw + (split == 0 ? h * (p.tw >> 1) : 0);
      c2[h] = ht * p.th + (split == 1 ? h * (p.th >> 1) : 0);
      c3[h] = bt * p.nb + (split == 2 ? h * (p.nb >> 1) : 0);
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        const int x = wt * p.tw + wi[h][hr], y = ht * p.th + hi[h][hr], b = bt * p.nb + bi[h][hr];
        valid[h][hr] = x < p.W && y < p.H && b < p.B;
        pix[h][hr] = ((long long)b * p.H + y) * p.W + x;
        rpix[h][hr] = epi_rpix(p.e, b, y, x, p.H, p.W, pix[h][hr]);
      }
    }
    // softmax row operands of this thread's four rows, loaded before the turn barrier: the other warpgroup's MMAs and this
    // one's hide their latency.  sm: epi_pair's row constants (apply: merged after the main loop from the partials smt).
    float2 sm[2][2] = {}, smt[2][2][2];
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int hr = 0; hr < 2; ++hr) {
        if (sm_apply) sm_row_load(p.e, pix[h][hr], valid[h][hr], smt[h][hr]);
        if (sm_bwd) sm[h][hr].x = valid[h][hr] ? __ldg(p.e.sm_delta + pix[h][hr]) : 0.f;
      }
    float acc[2][BN / 2];
    if (i > 0) named_bar_sync(kTurnBar + wg, 256);          // the other warpgroup has issued tile i - 1
    fprop_mma<BN, 2>(p, L, acc, 0u, (uint32_t)(i * kiters));
    if (i + 1 < n_local) named_bar_arrive(kTurnBar + (wg ^ 1), 256);
    if constexpr (sm_stats) {
      const int nchunk = min(BN, p.e.Cout - nt * BN) / 64;   // (a chunk past Cout holds the zero-filled B rows)
      epilogue_frag_smstats<BN>(p.e, acc[0], nchunk, nt, pix[0], valid[0], alpha);
      epilogue_frag_smstats<BN>(p.e, acc[1], nchunk, nt, pix[1], valid[1], alpha);
      continue;
    }
    if (sm_apply) {
#pragma unroll
      for (int h = 0; h < 2; ++h)
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) sm[h][hr] = sm_row_apply(p.e, pix[h][hr], valid[h][hr], smt[h][hr]);
    }
#pragma unroll                                    // static accumulator indices: the fragments stay in registers
    for (int cc = 0; cc * 64 < BN; ++cc) {
      const int nbase = nt * BN + cc * 64;
      if (nbase >= p.e.Cout) break;                 // (the aux producer skips the same chunks)
      uint32_t aux_tile = 0u, aslot = 0u;
      if constexpr (aux_kind != 0) {
        aslot = aux.wait(aux_cnt);
        aux_tile = aux_tiles + aslot * kEpiStageBytes;
        ++aux_cnt;
      }
      epilogue_frag_chunk<F, BN>(p.e, tmY, acc[0], cc, nbase, c1[0], c2[0], c3[0], pix[0], rpix[0], valid[0], alpha, stage,
                                 p.epi_nbuf, sbuf, 1u + wg, leader, aux_tile, arow[0], sm[0]);
      epilogue_frag_chunk<F, BN>(p.e, tmY, acc[1], cc, nbase, c1[1], c2[1], c3[1], pix[1], rpix[1], valid[1], alpha, stage,
                                 p.epi_nbuf, sbuf, 1u + wg, leader, aux_tile, arow[1], sm[1]);
      // every thread of the warpgroup is past its last read of the aux box (the barrier before the second half's store)
      if (aux_kind != 0 && leader) mbar_arrive(aux.empty(aslot));
    }
  }
  if (leader) bulk_wait_all();                    // staging tiles must outlive the last tensor store
}

// Staged-epilogue consumer (the run-time general kernel, F = -1): both warpgroups run the MMAs of every tile, stage the
// accumulators in shared memory as fp32 rows, then run the epilogue on them.
__device__ __forceinline__ void fprop_staged_consumer(const FpropArgs& p, const CUtensorMap* tmY, const FpropSmem& L, int wg) {
  // Epilogue: team = which 64-channel chunks (even / odd) = consumer warpgroup, q = which 32 rows.
  const int ct = threadIdx.x - 128;
  const int lane = threadIdx.x & 31;
  const int q = (ct >> 5) & 3;
  const int team = wg;
  const int row = q * 32 + lane;
  const bool leader = (q == 0) && (lane == 0);
  const int wi = row % p.tw, hi = (row / p.tw) % p.th, bi = row / (p.tw * p.th);
  const bool vec_ok = epi_vec_ok(p.e);
  const float alpha = epi_alpha(p.e);
  const uint32_t stage = L.epi + team * p.epi_nbuf * kEpiStageBytes;
  const uint32_t t_row = L.acc + (uint32_t)row * acc_row_bytes(p.BN);
  const int kiters = p.taps * p.kblocks;
  uint32_t aux_cnt = 0, sbuf = 0, it = 0;
  EpiAux aux;
  aux.kind = p.aux_kind; aux.tiles = L.aux + (uint32_t)(team * p.aux_depth) * kEpiStageBytes;
  aux.ring = L.aux_ring(team); aux.cnt = &aux_cnt;
  const bool aux_half = p.aux_kind == 1 && p.e.res_up2;
  aux.arow = aux_half ? ((bi * p.aux_th + (p.aux_th == p.th ? hi : (hi >> 1))) * p.aux_tw + (wi >> 1)) : row;
  if (p.b_resident) L.bres_ready.wait(0);
  for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x, it += kiters) {
    const FpropTile tc = fprop_tile(p, tile);
    const int nt = tc.nt, wt = tc.wt, ht = tc.ht, bt = tc.bt;
    const int n0 = nt * p.BN;
    const int w = wt * p.tw + wi, h = ht * p.th + hi, b = bt * p.nb + bi;
    const bool valid = (w < p.W) && (h < p.H) && (b < p.B) && (p.out_sub == 1 || (((w | h) & 1) == 0));
    const long long pix = p.out_sub == 1 ? ((long long)b * p.H + h) * p.W + w
                                         : ((long long)b * ((p.H + 1) >> 1) + (h >> 1)) * ((p.W + 1) >> 1) + (w >> 1);
    const long long rpix = epi_rpix(p.e, b, h, w, p.H, p.W, pix);

    switch (p.BN) {
      case 16: fprop_staged_mma<16>(p, L, it, wg); break;
      case 32: fprop_staged_mma<32>(p, L, it, wg); break;
      case 64: fprop_staged_mma<64>(p, L, it, wg); break;
      default: fprop_staged_mma<128>(p, L, it, wg); break;
    }
    if (p.use_tma) {
      epilogue_tile_tma(p.e, tmY, t_row, p.BN, n0, wt * p.tw, ht * p.th, bt * p.nb, valid, pix, rpix, alpha, stage, p.epi_nbuf,
                        sbuf, team, row, leader, p.aux_kind ? &aux : nullptr);
    } else if (team == 0) {
      epilogue_row(p.e, t_row, p.BN, n0, valid, pix, rpix, alpha, vec_ok);
    }
  }
  if (p.use_tma && leader) bulk_wait_all();   // staging tiles must outlive the last tensor store
}

template <int F>      // epilogue variant (conv_epilogue.cuh: kEpi* bits fixed at compile time; -1 = run-time flags)
__global__ void __launch_bounds__(kThreads, 1)
conv_fprop_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                  const __grid_constant__ CUtensorMap tmY, const __grid_constant__ CUtensorMap tmAux, const FpropArgs p) {
  constexpr bool pingpong = fprop_is_pingpong(F);
  extern __shared__ uint8_t smem_raw[];
  const FpropSmem L = fprop_smem(p, pingpong, smem_aligned(smem_raw));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    L.ops.init(pingpong ? kConsumerWarps / 2 : kConsumerWarps);   // ping-pong: one warpgroup per stage
    L.bres_ready.init(1);
    L.aux_ring(0).init(1);
    L.aux_ring(1).init(1);
    fence_barrier_init();
    if (p.use_tma) tma_prefetch_desc(&tmY);
  }
  __syncthreads();

  if (warp >= 4) {
    reg_alloc<kConsumerRegs>();
    const int wg = (threadIdx.x - 128) >> 7;
    if constexpr (pingpong) {
      if (p.BN == 64) fprop_pp_consumer<F, 64>(p, &tmY, L, wg);
      else fprop_pp_consumer<F, 128>(p, &tmY, L, wg);
    } else {
      fprop_staged_consumer(p, &tmY, L, wg);
    }
    return;
  }
  reg_dealloc<kProducerRegs>();     // the whole producer warpgroup, idle warps 1 and 3 included
  if (warp == 0) {
    if (lane == 0) {
      // ------------------------------------------------------------- TMA producer: one operand ring in tile order
      uint32_t it = 0;
      if (p.b_resident) {       // tiles_n == 1: the whole (small) filter is fetched once per CTA instead of once per tile
        L.bres_ready.acquire(0, (uint32_t)(p.taps * p.kblocks) * L.b_bytes);
        for (int tap = 0; tap < p.taps; ++tap)
          for (int kb = 0; kb < p.kblocks; ++kb)
            tma_load_3d(L.bres + (uint32_t)(tap * p.kblocks + kb) * L.b_bytes, &tmB, L.bres_ready.full(0), kb * kBlockK, tap, 0);
      }
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const FpropTile tc = fprop_tile(p, tile);
        const int n0 = tc.nt * p.BN, w0 = tc.wt * p.tw, h0 = tc.ht * p.th, b0 = tc.bt * p.nb;
        for (int tap = 0; tap < p.taps; ++tap) {
          const int dh = tap / p.KW - p.pad_h, dw = tap % p.KW - p.pad_w;
          for (int kb = 0; kb < p.kblocks; ++kb, ++it) {
            const int s = L.ops.acquire(it, L.stage_bytes);
            const uint32_t sa = L.ring + s * L.stage_bytes, full = L.ops.full(s);
            tma_load_4d(sa, &tmA, full, kb * kBlockK, w0 + dw, h0 + dh, b0);
            if (p.b_resident) {
            } else if (p.w_mode == 0) {
              tma_load_3d(sa + kABytes, &tmB, full, kb * kBlockK, tap, n0);
            } else if (p.w_mode == 1) {
              tma_load_3d(sa + kABytes, &tmB, full, kb * kBlockK, b0, n0);
            } else {
              for (int j = 0; j < p.BN / 64; ++j)
                tma_load_3d(sa + kABytes + j * 8192, &tmB, full, n0 + j * 64, kb * kBlockK, b0);
            }
          }
        }
      }
    }
  } else if (warp == 2) {
    if (lane == 0 && p.aux_kind) {
      // ------------------------------------------------------------- aux producer: residual / mask / P boxes, in the order the
      // two rings are consumed (staged epilogue: team = chunk & 1; ping-pong: ring = local tile & 1), up to aux_depth boxes
      // ahead per ring
      const bool half = p.aux_kind == 1 && p.e.res_up2;
      const uint32_t bytes = (uint32_t)(p.aux_tw * p.aux_th * p.nb) * 128u;
      uint32_t cnt[2] = {0u, 0u};
      for (int tile = blockIdx.x, i = 0; tile < p.num_tiles; tile += gridDim.x, ++i) {
        const FpropTile tc = fprop_tile(p, tile);
        const int c1 = half ? (tc.wt * p.tw) >> 1 : tc.wt * p.tw, c2 = half ? (tc.ht * p.th) >> 1 : tc.ht * p.th, c3 = tc.bt * p.nb;
        for (int cc = 0; cc * 64 < p.BN; ++cc) {
          const int nbase = tc.nt * p.BN + cc * 64;
          if (nbase >= p.e.Cout) break;
          const int team = pingpong ? (i & 1) : (cc & 1);
          const MbarRing ring = L.aux_ring(team);
          const int slot = ring.acquire(cnt[team], bytes);
          tma_load_4d(L.aux + (uint32_t)(team * p.aux_depth + slot) * kEpiStageBytes, &tmAux, ring.full(slot), nbase, c1, c2, c3);
          ++cnt[team];
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ wgrad
struct WgradArgs {
  int B, H, W, Cin, Cout, taps, KW, pad_h, pad_w;
  int tw, th, nb;
  int tiles_w, tiles_h, tiles_b, pix_tiles;  // pix_tiles = tiles_w*tiles_h*tiles_b
  int tiles_m, tiles_n;                      // over Cout (128) and Cin (BN)
  int BN;                                    // 64 or 128 (input-channel tile)
  int groups, tiles_per_group;               // independent pixel groups (1, or B for per-image outputs)
  int splits, tiles_per_split;               // K-splits inside a group
  int num_items;                             // tiles_m*tiles_n*taps*groups*splits
  int stages;
  float* dw;
  long long dw_group_stride;
  float* dbias;                              // optional: sum over pixels of dy (bias gradient), from a constant-ones B operand
};

// Shared memory of conv_wgrad_kernel: addresses from base, or offsets from the 1024-aligned base when base = 0.
struct WgradSmem {
  uint32_t ones;                  // bf16 1.0 slab (dbias)
  uint32_t ring;                  // operand ring: stages x (two 64-channel dY boxes -> M = 128, BN / 64 X boxes)
  uint32_t stage_bytes;
  MbarRing ops;
  uint32_t total;
};
__host__ __device__ inline WgradSmem wgrad_smem(const WgradArgs& p, uint32_t base = 0) {
  WgradSmem L;
  L.stage_bytes = 2 * kABytes + (uint32_t)(p.BN / 64) * kABytes;
  L.ones = base;
  L.ring = L.ones + (p.dbias ? kOnesSlabBytes : 0u);
  L.ops = {L.ring + (uint32_t)p.stages * L.stage_bytes, p.stages};
  L.total = L.ops.end() - base;
  return L;
}

// work item -> (m tile, n tile, tap, split); n fastest so neighbouring CTAs share the dY tiles in L2
__device__ __forceinline__ void wgrad_decode(const WgradArgs& p, int item, int& mt, int& nt, int& tap, int& grp, int& pt_begin,
                                             int& pt_end) {
  int t = item;
  nt = t % p.tiles_n; t /= p.tiles_n;
  tap = t % p.taps; t /= p.taps;
  mt = t % p.tiles_m; t /= p.tiles_m;
  const int sp = t % p.splits; t /= p.splits;
  grp = t;
  const int g0 = grp * p.tiles_per_group;
  pt_begin = g0 + sp * p.tiles_per_split;
  pt_end = min(pt_begin + p.tiles_per_split, g0 + p.tiles_per_group);
}

// One wgrad work item for this consumer warpgroup (output channels mt*128 + 64 wg ..): MMAs over the item's pixel tiles, then
// fp32 red.adds straight from the accumulator registers.
template <int BN>
__device__ __forceinline__ void wgrad_item(const WgradArgs& p, const WgradSmem& L, int item, uint32_t& it, int wg) {
  int mt, nt, tap, grp, pb, pe;
  wgrad_decode(p, item, mt, nt, tap, grp, pb, pe);
  const uint32_t lane = threadIdx.x & 31, w = (threadIdx.x >> 5) & 3;
  const uint32_t a_bytes = 2 * kABytes;
  float acc[BN / 2], bacc[4];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) bacc[i] = 0.f;
  // bias gradient: the (first input-channel tile, first tap) items also multiply dY^T by a block of ones (K-major, N = 8)
  const bool with_bias = p.dbias != nullptr && nt == 0 && tap == 0;
  const uint64_t ones_desc = make_sdesc_sw128(L.ones, 16, 1024);
  int prev = -1;
  for (int pt = pb; pt < pe; ++pt, ++it) {
    const int s = L.ops.wait(it);
    const uint32_t sa = L.ring + s * L.stage_bytes;
    // MN-major: 64-wide MN atoms are kABytes apart (LBO), 8-row K groups are 1024 B apart (SBO); this warpgroup's M atom = wg
    const uint64_t adesc = make_sdesc_sw128(sa + (uint32_t)wg * kABytes, kABytes, 1024);
    const uint64_t bdesc = make_sdesc_sw128(sa + a_bytes, kABytes, 1024);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < kTileM / 16; ++kk)      // 16 pixels (K) = two 8-row groups = 2048 bytes -> +128 in the (addr >> 4) field
      Wgmma<BN>::template mma<1, 1>(acc, adesc + 128 * kk, bdesc + 128 * kk, 1u);
    if (with_bias) {
#pragma unroll
      for (int kk = 0; kk < kTileM / 16; ++kk) Wgmma<8>::template mma<1, 0>(bacc, adesc + 128 * kk, ones_desc, 1u);
    }
    wgmma_commit();
    L.ops.release_prev(prev, s);
  }
  wgmma_wait<0>();
  acc_fence(acc);
  acc_fence(bacc);
  if (prev >= 0) L.ops.release(prev);
  if (pe <= pb) return;
  const int co0 = mt * 128 + wg * 64 + (int)(16u * w + (lane >> 2));
  const int ci0 = nt * BN + 2 * (int)(lane & 3);
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int co = co0 + 8 * hr;
    if (co >= p.Cout) continue;
    float* dst = p.dw + grp * p.dw_group_stride + ((long long)co * p.taps + tap) * p.Cin;
    if (with_bias && (lane & 3) == 0) atomicAdd(p.dbias + co, bacc[2 * hr]);   // column 0 of the ones-product
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int ci = ci0 + 8 * j + e;
        if (ci < p.Cin) atomicAdd(dst + ci, acc[4 * j + 2 * hr + e]);
      }
  }
}

__global__ void __launch_bounds__(kWgradThreads, 1)
conv_wgrad_kernel(const __grid_constant__ CUtensorMap tmDY, const __grid_constant__ CUtensorMap tmX, const WgradArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const WgradSmem L = wgrad_smem(p, smem_aligned(smem_raw));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (p.dbias) fill_ones_slab(L.ones, kWgradThreads);
  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmDY);
    tma_prefetch_desc(&tmX);
    L.ops.init(kConsumerWarps);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp == 0) {
    if (lane == 0) {
      uint32_t it = 0;
      for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
        int mt, nt, tap, grp, pb, pe;
        wgrad_decode(p, item, mt, nt, tap, grp, pb, pe);
        const int dh = tap / p.KW - p.pad_h, dw = tap % p.KW - p.pad_w;
        for (int pt = pb; pt < pe; ++pt, ++it) {
          int t = pt;
          const int wt = t % p.tiles_w; t /= p.tiles_w;
          const int ht = t % p.tiles_h; t /= p.tiles_h;
          const int bt = t;
          const int w0 = wt * p.tw, h0 = ht * p.th, b0 = bt * p.nb;
          const int s = L.ops.acquire(it, L.stage_bytes);
          const uint32_t sa = L.ring + s * L.stage_bytes, full = L.ops.full(s);
          tma_load_4d(sa, &tmDY, full, mt * 128, w0, h0, b0);
          tma_load_4d(sa + kABytes, &tmDY, full, mt * 128 + 64, w0, h0, b0);
          for (int j = 0; j < p.BN / 64; ++j)
            tma_load_4d(sa + 2 * kABytes + j * kABytes, &tmX, full, nt * p.BN + j * 64, w0 + dw, h0 + dh, b0);
        }
      }
    }
  } else if (warp >= 4) {
    const int wg = (threadIdx.x - 128) >> 7;
    uint32_t it = 0;
    for (int item = blockIdx.x; item < p.num_items; item += gridDim.x) {
      if (p.BN == 64) wgrad_item<64>(p, L, item, it, wg);
      else wgrad_item<128>(p, L, item, it, wg);
    }
  }
}

// ------------------------------------------------------------------------------------------------ host side
// Tile box over (W, H, B) with tw*th*nb == 128. Power-of-two splits; edges are masked / zero-filled.
static void pick_tile(int H, int W, int B, int& tw, int& th, int& nb) {
  tw = 1;
  while (tw < W && tw < 128) tw <<= 1;   // smallest power of two >= W, capped at 128
  if (tw > 16 && (W % tw) != 0) {        // ragged widths (Inception): prefer narrower tiles to limit waste
    while (tw > 16 && (W % tw) != 0) tw >>= 1;
  }
  th = 1;
  while (th < H && tw * th < 128) th <<= 1;
  nb = 128 / (tw * th);
  (void)B;
}

// The epilogue can stage bf16 64-channel chunks and TMA-store them: a bf16 output, channel tiles of 64, 16-byte aligned
// channel strides of every tensor it reads or writes.
bool epi_tma_ok(const sgb_conv_desc* d, int BN) {
  return !d->y_fp32 && BN % 64 == 0 && d->Cout % 8 == 0 && d->y_cstride % 8 == 0 && (!d->residual || d->res_cstride % 8 == 0) &&
         (!d->mask || d->mask_cstride % 8 == 0);
}

void fill_epi(EpiArgs& e, const sgb_conv_desc* d) {
  e.Cout = d->Cout;
  e.alpha = d->alpha; e.alpha_ptr = d->alpha_ptr; e.bias = d->bias;
  e.residual = (const bf16*)d->residual; e.res_cstride = d->res_cstride; e.res_up2 = d->res_up2; e.res_after = d->res_after_mask;
  e.res_scale = d->res_scale != 0.f ? d->res_scale : 1.f;
  e.mask = (const bf16*)d->mask; e.mask_cstride = d->mask_cstride; e.relu = d->relu;
  e.y = d->y; e.y_cstride = d->y_cstride; e.y_fp32 = d->y_fp32;
  e.mask_bits = (const unsigned long long*)d->mask_bits;
  e.relu_bits = (unsigned long long*)d->relu_bits;
  e.sm_mode = d->sm_mode; e.sm_parts = 0; e.sm_stats = d->sm_stats; e.sm_delta = d->sm_delta;
}

// Output-channel tile of the fprop kernels (the halo-row kernel takes it too).
int pick_bn(const sgb_conv_desc* d) {
  int BN;
  if (d->Cout <= 16) BN = 16;
  else if (d->Cout <= 32) BN = 32;
  else if (d->Cout <= 64) BN = 64;
  else BN = 128;      // 128 x 128 fp32 accumulators: 64 registers per consumer thread, 66 KiB of staging rows
  if (d->w_mode == 2 && BN < 64) BN = 64;  // MN-major B is staged in 64-wide atoms
  return BN;
}

// The hot epilogue shapes of the training step get compile-time variants of the kernel; every other launch takes the
// general kernel (F = -1, run-time flags).
using FpropCompiled = EpiVariants<
    kEpiFull,                                                          // dgrad / attention GEMMs
    kEpiFull | kEpiBias,                                               // generator convs
    kEpiFull | kEpiBias | kEpiRelu,                                    // discriminator convs (no backward expected)
    kEpiFull | kEpiBias | kEpiRelu | kEpiBitsOut,                      // ... writing the ReLU bit plane
    kEpiFull | kEpiResPre | kEpiAuxRes,                                // concat-skip dgrad
    kEpiFull | kEpiBias | kEpiResPre | kEpiAuxRes,                     // block output + skip
    kEpiFull | kEpiBias | kEpiRelu | kEpiResPre | kEpiAuxRes,          // ... with the next block's ReLU
    kEpiFull | kEpiBias | kEpiRelu | kEpiResPre | kEpiAuxRes | kEpiBitsOut,
    kEpiFull | kEpiMask | kEpiMaskBits,                                // dgrad through a ReLU (bit plane)
    kEpiFull | kEpiMask | kEpiMaskBits | kEpiResPre | kEpiAuxRes,      // fused block entry (bit plane + pooled-skip gradient)
    kEpiFull | kEpiMask | kEpiAuxMask,                                 // dgrad through a ReLU (bf16 mask tile)
    kEpiFull | kEpiMask | kEpiResPre | kEpiAuxMask,                    // fused block entry (bf16 mask tile)
    kEpiFull | kEpiSmStats,                                            // attention: row (max, sum exp) partials of theta . phi^T
    kEpiFull | kEpiSmApply,                                            // attention: P = softmax(theta . phi^T) written directly
    kEpiFull | kEpiSmBwd>;                                             // attention: dS = P * (do . g^T - delta)

bool wgrad3x3_c64_eligible(const sgb_wgrad_desc* d);
int launch_wgrad3x3_c64(const sgb_wgrad_desc* d, cudaStream_t stream);
bool conv3x3_rows_eligible(const sgb_conv_desc* d);
int launch_conv3x3_rows(const sgb_conv_desc* d, cudaStream_t stream);

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_conv_softmax_parts(const sgb_conv_desc* d) {
  if (!d || d->Cout <= 0) return 0;
  const int BN = pick_bn(d);
  return (d->Cout + BN - 1) / BN;       // one (max, sum exp) partial per row and channel tile
}

extern "C" int sgb_conv_fprop(const sgb_conv_desc* d, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(d && d->x && d->w && d->y);
  SGB_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0);
  SGB_REQUIRE(d->Cin % 8 == 0 && d->x_cstride % 8 == 0 && d->x_cstride >= d->Cin);
  SGB_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->w & 15) == 0 && ((uintptr_t)d->y & 15) == 0);
  SGB_REQUIRE(!d->res_up2 || (d->H % 2 == 0 && d->W % 2 == 0));
  SGB_REQUIRE(d->w_mode >= 0 && d->w_mode <= 2);
  SGB_REQUIRE(d->w_mode == 0 || (d->KH == 1 && d->KW == 1 && d->H * d->W >= 128));
  SGB_REQUIRE(d->w_mode != 2 || d->Cout % 8 == 0);
  SGB_REQUIRE(((uintptr_t)d->bias & 15) == 0 && ((uintptr_t)d->residual & 15) == 0 && ((uintptr_t)d->mask & 15) == 0);
  // bit-plane ReLU masks: whole 64-channel words, vector epilogue paths only
  SGB_REQUIRE(!d->mask_bits || (!d->mask && d->Cout % 64 == 0 && !d->y_fp32 && d->out_sub != 2 && ((uintptr_t)d->mask_bits & 7) == 0));
  SGB_REQUIRE(!d->relu_bits || (d->relu && d->Cout % 64 == 0 && !d->y_fp32 && d->out_sub != 2 && d->y_cstride % 8 == 0 &&
                                ((uintptr_t)d->relu_bits & 7) == 0));
  SGB_REQUIRE(!(d->mask_bits || d->relu_bits) || ((!d->residual || d->res_cstride % 8 == 0) && d->y_cstride % 8 == 0));
  // attention softmax inside the epilogue: plain bf16 GEMM tiles only
  SGB_REQUIRE(d->sm_mode >= 0 && d->sm_mode <= 3);
  SGB_REQUIRE(!d->sm_mode || (d->Cout % 64 == 0 && !d->y_fp32 && d->out_sub != 2 && !d->bias && !d->residual && !d->mask && !d->mask_bits &&
                              !d->relu && d->KH == 1 && d->KW == 1 && d->Cin <= 640 && d->y_cstride % 8 == 0));
  SGB_REQUIRE(d->sm_mode != 1 || d->sm_stats);
  SGB_REQUIRE(d->sm_mode != 2 || d->sm_stats);
  SGB_REQUIRE(d->sm_mode != 3 || (d->sm_delta && d->sm_p && d->sm_p_cstride % 8 == 0 && ((uintptr_t)d->sm_p & 15) == 0));
  // wide, few-channel 3x3 layers: halo-row kernel (umma_conv3x3.cu)
  if (d->Hin <= 0 && d->Win <= 0 && d->out_sub != 2 && conv3x3_rows_eligible(d)) return launch_conv3x3_rows(d, stream);

  FpropArgs p;
  p.B = d->B; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout;
  p.taps = d->KH * d->KW; p.KW = d->KW; p.pad_h = d->pad_h; p.pad_w = d->pad_w;
  pick_tile(d->H, d->W, d->B, p.tw, p.th, p.nb);
  p.tiles_w = (d->W + p.tw - 1) / p.tw;
  p.tiles_h = (d->H + p.th - 1) / p.th;
  p.tiles_b = (d->B + p.nb - 1) / p.nb;
  const int BN = pick_bn(d);
  p.BN = BN;
  p.w_mode = d->w_mode;
  p.tiles_n = (d->Cout + BN - 1) / BN;
  p.num_tiles = p.tiles_n * p.tiles_w * p.tiles_h * p.tiles_b;
  p.kblocks = (d->Cin + kBlockK - 1) / kBlockK;
  const int Hin = d->Hin > 0 ? d->Hin : d->H, Win = d->Win > 0 ? d->Win : d->W;
  p.out_sub = d->out_sub == 2 ? 2 : 1;
  SGB_REQUIRE(p.out_sub == 1 || (!d->residual && !d->mask));
  p.use_tma = (p.out_sub == 1 && epi_tma_ok(d, BN)) ? 1 : 0;
  // auxiliary epilogue operand through TMA: exactly one of residual / mask, bf16 NHWC with 16-byte aligned channel stride
  p.aux_kind = 0; p.aux_tw = p.tw; p.aux_th = p.th;
  if (p.use_tma && (d->residual != nullptr || d->mask != nullptr)) {   // (mask_bits are 8-byte direct loads)
    // one operand rides TMA: the mask when both are present (full-resolution tile; the residual of such launches is the
    // quarter-size pooled-skip gradient, whose direct 16-byte loads are shared by 2x2 pixel neighbours through L1)
    if (d->mask) p.aux_kind = 2;
    else if (!d->residual) p.aux_kind = 0;                       // bit-plane mask only: nothing to stage
    else if (!d->res_up2) p.aux_kind = 1;
    else if (p.tw >= 2) { p.aux_kind = 1; p.aux_tw = p.tw / 2; p.aux_th = p.th >= 2 ? p.th / 2 : 1; }
  }
  if (d->sm_mode) {
    SGB_REQUIRE(p.use_tma);                                            // (the softmax variants exist only for the TMA-store epilogue)
    if (d->sm_mode == 3) p.aux_kind = 3;                               // P tile of the softmax backward
  }
  fill_epi(p.e, d);
  p.e.sm_parts = p.tiles_n;
  int f = p.use_tma ? epi_flags_of(p.e) : -1;
  SGB_REQUIRE(!d->sm_mode || f == (kEpiFull | (d->sm_mode == 1 ? kEpiSmStats : d->sm_mode == 2 ? kEpiSmApply : kEpiSmBwd)));
  if (f >= 0 && p.aux_kind == 1) f |= kEpiAuxRes;
  if (f >= 0 && p.aux_kind == 2) f |= kEpiAuxMask;
  if (!FpropCompiled::has(f)) f = -1;
  // ping-pong (every compiled variant): no fp32 accumulator staging; 8 KiB half-tile staging tiles per warpgroup.  The general
  // kernel (F = -1): fp32 rows of the whole tile plus 16 KiB staging tiles per epilogue team.
  const bool pingpong = fprop_is_pingpong(f);
  // short-K layers (one or two K blocks per tile) are store bound: their (small) filter stays resident in shared memory and the
  // space of the B halves of the ring buys more staging tiles per epilogue team = more store bytes in flight
  const uint32_t b_tile = (uint32_t)BN * kBlockK * 2;
  const int kt = p.taps * p.kblocks;
  p.b_resident = (d->w_mode == 0 && p.tiles_n == 1 && kt <= 2 && kt * b_tile <= 64u * 1024u) ? 1 : 0;
  p.epi_nbuf = !p.use_tma ? 1 : pingpong ? (kt <= 2 ? 4 : 2) : (kt <= 2 ? 2 : 1);
  // softmax backward (K = c/2 = 256, P through a 2-deep aux ring of 16 KiB boxes): one staging tile per warpgroup leaves room for
  // a 4th operand stage, measured 11 % faster at the flagship attention than 2 staging tiles and 3 stages
  if (d->sm_mode == 3) p.epi_nbuf = 1;
  p.aux_depth = p.aux_kind ? 2 : 1;
  p.stages = 0;
  // room for the operand ring: 216 KiB less the layout in front of it
  auto ring_room = [&] { return 216 * 1024 - (int)fprop_smem(p, pingpong).ring; };
  const int stage_bytes = (int)fprop_smem(p, pingpong).stage_bytes;
  // keep >= 3 operand ring stages: give back aux depth first, then staging tiles
  while (p.aux_kind && p.aux_depth > 1 && ring_room() < 3 * stage_bytes) --p.aux_depth;
  while (p.epi_nbuf > 1 && ring_room() < 3 * stage_bytes) --p.epi_nbuf;
  int stages = ring_room() / stage_bytes;
  if (stages > 8) stages = 8;
  if (stages < 2) stages = 2;
  p.stages = stages;

  CUtensorMap tmA, tmB;
  int rc = make_act_tmap(&tmA, d->x, d->B, Hin, Win, d->Cin, d->x_cstride, p.tw, p.th, p.nb);
  if (rc) return rc;
  if (d->w_mode == 0) {
    uint64_t dims[3] = {(uint64_t)d->Cin, (uint64_t)p.taps, (uint64_t)d->Cout};
    uint64_t strides[2] = {(uint64_t)d->Cin * 2, (uint64_t)d->Cin * 2 * p.taps};
    uint32_t box[3] = {64, 1, (uint32_t)BN};
    rc = make_tmap_bf16(&tmB, d->w, 3, dims, strides, box);
  } else if (d->w_mode == 1) {  // per-image [B][N = Cout][K = Cin]
    uint64_t dims[3] = {(uint64_t)d->Cin, (uint64_t)d->B, (uint64_t)d->Cout};
    uint64_t strides[2] = {(uint64_t)d->Cin * 2 * d->Cout, (uint64_t)d->Cin * 2};
    uint32_t box[3] = {64, 1, (uint32_t)BN};
    rc = make_tmap_bf16(&tmB, d->w, 3, dims, strides, box);
  } else {                      // per-image [B][K = Cin][N = Cout], N contiguous
    uint64_t dims[3] = {(uint64_t)d->Cout, (uint64_t)d->Cin, (uint64_t)d->B};
    uint64_t strides[2] = {(uint64_t)d->Cout * 2, (uint64_t)d->Cout * 2 * d->Cin};
    uint32_t box[3] = {64, 64, 1};
    rc = make_tmap_bf16(&tmB, d->w, 3, dims, strides, box);
  }
  if (rc) return rc;
  CUtensorMap tmY = tmA;
  if (p.use_tma) {
    // ping-pong: one store per 64-row half of the tile, whose box halves the outermost non-unit dimension of (tw, th, nb)
    const int split = p.nb > 1 ? 2 : (p.th > 1 ? 1 : 0);
    rc = make_act_tmap(&tmY, d->y, d->B, d->H, d->W, d->Cout, d->y_cstride, pingpong && split == 0 ? p.tw / 2 : p.tw,
                       pingpong && split == 1 ? p.th / 2 : p.th, pingpong && split == 2 ? p.nb / 2 : p.nb);
    if (rc) return rc;
  }
  CUtensorMap tmAux = tmA;
  if (p.aux_kind) {
    const bool half = (p.aux_kind == 1 && d->res_up2);
    const void* ap = p.aux_kind == 1 ? d->residual : (p.aux_kind == 3 ? d->sm_p : d->mask);
    const long long acs = p.aux_kind == 1 ? d->res_cstride : (p.aux_kind == 3 ? d->sm_p_cstride : d->mask_cstride);
    rc = make_act_tmap(&tmAux, ap, d->B, half ? d->H / 2 : d->H, half ? d->W / 2 : d->W, d->Cout, acs, p.aux_tw, p.aux_th, p.nb);
    if (rc) return rc;
  }
  const size_t smem = smem_request(fprop_smem(p, pingpong).total);
  SGB_REQUIRE(smem <= 227u * 1024u);
  int grid = p.num_tiles < sm_count() ? p.num_tiles : sm_count();
  return FpropCompiled::launch(f, [&](auto F) {
    return launch_kernel<conv_fprop_kernel<decltype(F)::value>>(grid, kThreads, smem, stream, tmA, tmB, tmY, tmAux, p);
  });
}

extern "C" int sgb_conv_wgrad_fuses_dbias(const sgb_wgrad_desc* d) {
  if (!d) return 0;
  if (wgrad3x3_c64_eligible(d)) return 1;
  return d->per_image ? 0 : 1;          // generic kernel: constant-ones B operand on its (first channel tile, first tap) items
}

extern "C" int sgb_conv_wgrad(const sgb_wgrad_desc* d, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(d && d->x && d->dy && d->dw);
  SGB_REQUIRE(d->B > 0 && d->H > 0 && d->W > 0 && d->Cin > 0 && d->Cout > 0 && d->KH > 0 && d->KW > 0);
  SGB_REQUIRE(d->Cin % 8 == 0 && d->x_cstride % 8 == 0 && d->Cout % 8 == 0 && d->dy_cstride % 8 == 0);
  SGB_REQUIRE(((uintptr_t)d->x & 15) == 0 && ((uintptr_t)d->dy & 15) == 0);
  if (wgrad3x3_c64_eligible(d)) return launch_wgrad3x3_c64(d, stream);
  SGB_REQUIRE(d->dbias == nullptr || !d->per_image);

  WgradArgs p;
  p.B = d->B; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout;
  p.taps = d->KH * d->KW; p.KW = d->KW; p.pad_h = d->pad_h; p.pad_w = d->pad_w;
  pick_tile(d->H, d->W, d->B, p.tw, p.th, p.nb);
  p.tiles_w = (d->W + p.tw - 1) / p.tw;
  p.tiles_h = (d->H + p.th - 1) / p.th;
  p.tiles_b = (d->B + p.nb - 1) / p.nb;
  p.pix_tiles = p.tiles_w * p.tiles_h * p.tiles_b;
  p.BN = (d->Cin <= 64) ? 64 : 128;
  p.tiles_m = (d->Cout + 127) / 128;
  p.tiles_n = (d->Cin + p.BN - 1) / p.BN;
  p.groups = d->per_image ? d->B : 1;
  SGB_REQUIRE(!d->per_image || (p.nb == 1));
  p.tiles_per_group = p.pix_tiles / p.groups;
  p.dw_group_stride = (long long)d->Cout * p.taps * d->Cin;
  const int base_items = p.tiles_m * p.tiles_n * p.taps * p.groups;
  // K-splits: the persistent grid runs ceil(items / SMs) rounds of one item (= tiles_per_split pixel tiles + a drain) each, so
  // pick the split count that minimises rounds x (tiles_per_split + drain): a last round with a handful of items leaves most
  // SMs idle.
  {
    const int sms = sm_count();
    const int max_splits = p.tiles_per_group < (4 * sms + base_items - 1) / base_items ? p.tiles_per_group : (4 * sms + base_items - 1) / base_items;
    const long long drain = 2;                      // accumulator drain (fp32 red.add of a 128 x BN block) in pixel-tile units
    long long best_cost = -1;
    int best = 1;
    for (int s = 1; s <= (max_splits < 1 ? 1 : max_splits); ++s) {
      const int tps = (p.tiles_per_group + s - 1) / s;
      const int eff = (p.tiles_per_group + tps - 1) / tps;
      const long long rounds = ((long long)base_items * eff + sms - 1) / sms;
      const long long cost = rounds * (tps + drain);
      if (best_cost < 0 || cost < best_cost) { best_cost = cost; best = s; }
    }
    // near-ties go to MORE splits: concurrent items of one split read the same dY / X tiles at the same moment (36 CTAs on
    // one set of L2 lines for a 256 -> 256 filter), more splits = more distinct streams and drains hidden behind the next item
    for (int s = best + 1; s <= (max_splits < 1 ? 1 : max_splits); ++s) {
      const int tps = (p.tiles_per_group + s - 1) / s;
      const int eff = (p.tiles_per_group + tps - 1) / tps;
      const long long rounds = ((long long)base_items * eff + sms - 1) / sms;
      if (50 * rounds * (tps + drain) <= 51 * best_cost) best = s;
    }
    p.tiles_per_split = (p.tiles_per_group + best - 1) / best;
    p.splits = (p.tiles_per_group + p.tiles_per_split - 1) / p.tiles_per_split;
  }
  p.num_items = base_items * p.splits;
  p.dw = d->dw;
  p.dbias = d->dbias;
  p.stages = 0;
  int stages = (int)((216 * 1024) / wgrad_smem(p).stage_bytes);
  if (stages > 6) stages = 6;
  p.stages = stages;
  if (d->dbias && !d->accumulate) SGB_CUDA(cudaMemsetAsync(d->dbias, 0, sizeof(float) * (size_t)d->Cout, stream));

  if (!d->accumulate)
    SGB_CUDA(cudaMemsetAsync(d->dw, 0, sizeof(float) * (size_t)d->Cout * p.taps * d->Cin * (d->per_image ? d->B : 1), stream));

  CUtensorMap tmDY, tmX;
  int rc = make_act_tmap(&tmDY, d->dy, d->B, d->H, d->W, d->Cout, d->dy_cstride, p.tw, p.th, p.nb);
  if (rc) return rc;
  rc = make_act_tmap(&tmX, d->x, d->B, d->H, d->W, d->Cin, d->x_cstride, p.tw, p.th, p.nb);
  if (rc) return rc;

  const size_t smem = smem_request(wgrad_smem(p).total);
  int grid = p.num_items < sm_count() ? p.num_items : sm_count();
  return launch_kernel<conv_wgrad_kernel>(grid, kWgradThreads, smem, stream, tmDY, tmX, p);
}
