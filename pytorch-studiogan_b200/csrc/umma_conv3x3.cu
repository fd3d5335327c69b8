// 3x3 / pad 1 convolution for wide feature maps with few channels (W % 64 == 0, Cin <= 256): the layers of BigGAN-Deep at
// 64x64 .. 256x256, where the generic per-tap kernel is bound by L2 -> smem traffic (each output tile re-fetches its input 9x
// and the whole filter once).  This variant stages HALO ROWS once and forms all nine taps from shared memory:
//   segment     = S = 128 output pixels of a row when W % 128 == 0, else S = 64, taken only when the layer has at least one
//                 work item per SM (rows_segment)
//   work item   = 256 output pixels x BN channels: R = 256 / S output rows of one S-pixel segment (S = 128: 2 rows, S = 64:
//                 4 rows); two register accumulators (two output rows of 64 pixels) per consumer warpgroup
//   A staging   = R + 2 input rows (h0 - 1 .. h0 + R) of S + 2 pixels x 64 channels per K block, one TMA box each, every row
//                 buffer rounded up to 1 KiB (S = 128: 4 x 17 KiB, S = 64: 6 x 9 KiB)
//                 (OOB rows / columns zero-filled = padding); tap (kh, kw) of output row r reads row buffer kh + r at a
//                 start address advanced by kw pixels (kw * 128 B): rows stay 128 B apart, and the 128-byte swizzle is a
//                 function of the absolute shared-memory address, so a row-shifted descriptor addresses exactly what TMA wrote
//   B staging   = filter taps; RESIDENT in smem for the whole persistent CTA when they fit (C = 64: 72 KiB), else a ring
//   L2 traffic  = 33 KiB per 128 output pixels at C = 64 (was 216 KiB), 210 KiB at C = 128 (was 576 KiB); S = 64, C = 256,
//                 BN = 128: 774 KiB per 256 pixels x 128 channels (198 KiB halo rows + 576 KiB filter), against 2304 KiB for the
//                 generic kernel's two 128-pixel tiles
// Warps: 0 = A producer, 2 = B producer (warpgroup 0 gives up registers with setmaxnreg); warpgroups 1 and 2 = consumers
// (wgmma M = 64; rows_slot: S = 128 pixels 0..63 / 64..127 of both rows, S = 64 rows 0, 1 / 2, 3).  Each consumer warpgroup
// runs the fused epilogue straight from its accumulator registers and TMA-stores its 64-pixel rows through its own bf16 staging
// tiles (epilogue_frag_tma), so no fp32 staging competes with the halo ring: the hot shapes (C = 64 resident taps, C = 128 / 256
// filter ring) get two halo stages, and the next item's halo rows load while this item computes.  fp32 outputs, N < 64 and
// unaligned strides take the staged-row epilogue.
#include "common.cuh"
#include "ptx.cuh"
#include "conv_epilogue.cuh"

namespace sgb {

static constexpr int kRowsItemPix = 256;                   // output pixels of a work item: R rows x S pixels
static constexpr int kRowsConsumers = 256;
static constexpr int kRowsThreads = 128 + kRowsConsumers;  // warps 0: A producer, 2: B producer, 4..11: MMA + epilogue
static constexpr uint32_t kRowsAccBar = 3;                 // named barrier of the consumers (1, 2: epilogue teams)

struct RowsArgs {
  int B, H, W, Cin, Cout;
  int S, R;                // segment width (128 or 64) and output rows of a work item (256 / S)
  int kblocks, BN, tiles_n, segs, hgroups, num_tiles;
  int resident, a_stages, b_stages;
  int use_tma, epi_nbuf;   // fragment epilogue with TMA stores; 8 KiB bf16 staging tiles per consumer warpgroup
  EpiArgs e;
};

// One halo row: S + 2 pixels x 64 channels loaded, the buffer rounded up to 1 KiB so every row buffer stays 1024-byte aligned.
__host__ __device__ inline uint32_t rows_load_bytes(const RowsArgs& p) { return (uint32_t)(p.S + 2) * 128u; }
__host__ __device__ inline uint32_t rows_buf_bytes(const RowsArgs& p) { return (rows_load_bytes(p) + 1023u) & ~1023u; }
// One halo stage: input rows h0 - 1 .. h0 + R of one K block (S = 128: 4 x 17 KiB, S = 64: 6 x 9 KiB).
__host__ __device__ inline uint32_t rows_stage_bytes(const RowsArgs& p) { return (uint32_t)(p.R + 2) * rows_buf_bytes(p); }

// Accumulator j (0, 1) of consumer warpgroup wg holds 64 pixels of one output row: the row of the item's R and the first pixel
// of the segment's S.  S = 128: pixels 64 wg .. 64 wg + 63 of rows 0 and 1; S = 64: rows 2 wg and 2 wg + 1.
struct RowsSlot { int row, px; };
__host__ __device__ inline RowsSlot rows_slot(const RowsArgs& p, int wg, int j) {
  return p.S == 128 ? RowsSlot{j, 64 * wg} : RowsSlot{2 * wg + j, 0};
}
// The A operand of tap (kh, kw) for slot s in the halo stage at sa: halo row s.row + kh from pixel s.px + kw.
__device__ __forceinline__ uint32_t rows_a_addr(const RowsArgs& p, uint32_t sa, RowsSlot s, int kh, int kw) {
  return sa + (uint32_t)(s.row + kh) * rows_buf_bytes(p) + (uint32_t)(s.px + kw) * 128u;
}

// Shared memory in front of the operand rings: the bf16 staging tiles of the fragment epilogue, or (staged-row epilogue) the
// fp32 accumulator rows of one output row.  A multiple of 1024 bytes.
__host__ __device__ inline uint32_t rows_epi_bytes(const RowsArgs& p) {
  return p.use_tma ? 2u * (uint32_t)p.epi_nbuf * 64u * 128u : 128u * acc_row_bytes(p.BN);
}

// Shared memory of conv3x3_rows_kernel: addresses from base, or offsets from the 1024-aligned base when base = 0.
struct RowsSmem {
  uint32_t epi;                   // rows_epi_bytes
  uint32_t a;                     // halo ring: a_stages x rows_stage_bytes
  uint32_t a_stage;               // rows_stage_bytes
  uint32_t b;                     // filter taps: resident [kb][kw][kh], or a ring of b_stages taps
  uint32_t bar;                   // first barrier = bytes of the tile regions
  uint32_t b_tile;
  MbarRing a_ring, b_ring;        // the resident filter is the b ring with one slot, filled once
  uint32_t total;
};
__host__ __device__ inline RowsSmem rows_smem(const RowsArgs& p, uint32_t base = 0) {
  RowsSmem L;
  L.b_tile = (uint32_t)p.BN * 128u;
  L.a_stage = rows_stage_bytes(p);
  L.epi = base;
  L.a = L.epi + rows_epi_bytes(p);
  L.b = L.a + (uint32_t)p.a_stages * L.a_stage;
  L.bar = L.b + (p.resident ? 9u * p.kblocks : (uint32_t)p.b_stages) * L.b_tile;
  L.a_ring = {L.bar, p.a_stages};
  L.b_ring = {L.a_ring.end(), p.b_stages};
  L.total = L.b_ring.end() - base;
  return L;
}

// Tile index -> (channel tile, S-pixel segment, group of R rows, image), channel tiles fastest.
struct RowsTile { int nt, ws, hg, b; };
__device__ __forceinline__ RowsTile rows_tile(const RowsArgs& p, int t) {
  RowsTile c;
  c.nt = t % p.tiles_n; t /= p.tiles_n;
  c.ws = t % p.segs; t /= p.segs;
  c.hg = t % p.hgroups; t /= p.hgroups;
  c.b = t;
  return c;
}

// One work item of a consumer warpgroup: its two slots' MMAs over every K block, accumulators of rows_slot(p, wg, j) in acc[j].
template <int BN>
__device__ __forceinline__ void rows_mma_tile(const RowsArgs& p, const RowsSmem& L, float (&acc)[2][BN / 2], uint32_t& ita,
                                              uint32_t& itb, int wg) {
#pragma unroll
  for (int j = 0; j < 2; ++j)
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[j][i] = 0.f;
  const RowsSlot slot[2] = {rows_slot(p, wg, 0), rows_slot(p, wg, 1)};
  for (int kb = 0; kb < p.kblocks; ++kb, ++ita) {
    const int sa_i = L.a_ring.wait(ita);
    const uint32_t sa = L.a + sa_i * L.a_stage;
    int bprev = -1;                              // filter-ring slot of the previous tap, released once its MMAs retire
    for (int tap = 0; tap < 9; ++tap) {
      const int kh = tap / 3, kw = tap % 3;
      uint32_t sb;
      int bslot = 0;
      if (p.resident) {
        sb = L.b + ((kb * 3 + kw) * 3 + kh) * L.b_tile;     // resident order [kb][kw][kh]
      } else {
        bslot = L.b_ring.wait(itb);
        sb = L.b + bslot * L.b_tile;
      }
      const uint64_t bdesc = make_sdesc_sw128(sb, 16, 1024);
      wgmma_fence();
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const uint64_t adesc = make_sdesc_sw128(rows_a_addr(p, sa, slot[j], kh, kw), 16, 1024);
#pragma unroll
        for (int kk = 0; kk < 4; ++kk) Wgmma<BN>::template mma<0, 0>(acc[j], adesc + 2 * kk, bdesc + 2 * kk, 1u);
      }
      wgmma_commit();
      if (!p.resident) {
        L.b_ring.release_prev(bprev, bslot);
        ++itb;
      }
    }
    wgmma_wait<0>();
    if (bprev >= 0) L.b_ring.release(bprev);
    L.a_ring.release(sa_i);
  }
  acc_fence(acc[0]);
  acc_fence(acc[1]);
}

// Stages output row j's accumulators of this warpgroup in shared memory (after every consumer is done with the previous ones).
template <int BN>
__device__ __forceinline__ void rows_stage(const float (&acc)[BN / 2], uint32_t acc_base, int wg) {
  named_bar_sync(kRowsAccBar, kRowsConsumers);
  acc_store<BN>(acc, acc_base + (uint32_t)wg * 64u * acc_row_bytes(BN), acc_row_bytes(BN));
  named_bar_sync(kRowsAccBar, kRowsConsumers);
}

template <int F, int BN>
__device__ __forceinline__ void rows_consumer(const RowsArgs& p, const CUtensorMap* tmY, const RowsSmem& L) {
  const int ct = threadIdx.x - 128;
  const int wg = ct >> 7;
  const int q = (ct >> 5) & 3;
  const int lane = threadIdx.x & 31;
  const float alpha = epi_alpha(p.e);
  uint32_t ita = 0, itb = 0;
  if (p.resident) L.b_ring.wait(0);
  if constexpr (F < 0 || BN < 64) {
    if (!p.use_tma) {
      // staged-row epilogue (fp32 output, N < 64, unaligned strides): both slots' accumulators go through shared memory and
      // warpgroup 1 runs epilogue_row, one thread per pixel (staged row t = slot j of warpgroup t / 64, pixel t % 64)
      const int row = q * 32 + lane;
      const bool vec_ok = epi_vec_ok(p.e);
      const uint32_t t_row = L.epi + (uint32_t)row * acc_row_bytes(BN);
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const RowsTile tc = rows_tile(p, tile);
        const int nt = tc.nt, ws = tc.ws, hg = tc.hg, b = tc.b;
        float acc[2][BN / 2];
        rows_mma_tile<BN>(p, L, acc, ita, itb, wg);
#pragma unroll 1
        for (int j = 0; j < 2; ++j) {
          if (j == 0) rows_stage<BN>(acc[0], L.epi, wg);    // static indices keep both accumulators in registers
          else rows_stage<BN>(acc[1], L.epi, wg);
          const RowsSlot sl = rows_slot(p, row >> 6, j);
          const int h = hg * p.R + sl.row, w = ws * p.S + sl.px + (row & 63);
          const long long pix = ((long long)b * p.H + h) * p.W + w;
          const long long rpix = epi_rpix(p.e, b, h, w, p.H, p.W, pix);
          if (wg == 0) epilogue_row(p.e, t_row, BN, nt * BN, true, pix, rpix, alpha, vec_ok);
        }
      }
      return;
    }
  }
  if constexpr (BN >= 64) {
    // fragment epilogue: each warpgroup stores its two 64-pixel slots from its registers through its own staging tiles
    const bool leader = (ct & 127) == 0;
    const uint32_t stage = L.epi + (uint32_t)(wg * p.epi_nbuf) * (64u * 128u);
    const uint32_t r0 = 16u * (uint32_t)q + ((uint32_t)lane >> 2);
    uint32_t sbuf = 0;
    for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
      const RowsTile tc = rows_tile(p, tile);
      const int nt = tc.nt, ws = tc.ws, hg = tc.hg, b = tc.b;
      float acc[2][BN / 2];
      rows_mma_tile<BN>(p, L, acc, ita, itb, wg);
#pragma unroll
      for (int j = 0; j < 2; ++j) {
        const RowsSlot sl = rows_slot(p, wg, j);
        const int h = hg * p.R + sl.row, w0 = ws * p.S + sl.px;
        long long pix[2], rpix[2];
#pragma unroll
        for (int hr = 0; hr < 2; ++hr) {
          const int w = w0 + (int)r0 + 8 * hr;
          pix[hr] = ((long long)b * p.H + h) * p.W + w;
          rpix[hr] = epi_rpix(p.e, b, h, w, p.H, p.W, pix[hr]);
        }
        epilogue_frag_tma<F, BN>(p.e, tmY, acc[j], nt * BN, w0, h, b, pix, rpix, alpha, stage, p.epi_nbuf, sbuf, 1u + wg, leader);
      }
    }
    if (leader) bulk_wait_all();                 // staging tiles must outlive the last tensor store
  }
}

template <int F>      // epilogue variant, see conv_epilogue.cuh
__global__ void __launch_bounds__(kRowsThreads, 1)
conv3x3_rows_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
                    const __grid_constant__ CUtensorMap tmY, const RowsArgs p) {
  extern __shared__ uint8_t smem_raw[];
  const RowsSmem L = rows_smem(p, smem_aligned(smem_raw));

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&tmA);
    tma_prefetch_desc(&tmB);
    L.a_ring.init(kRowsConsumers / 32);
    L.b_ring.init(kRowsConsumers / 32);
    fence_barrier_init();
  }
  __syncthreads();

  if (warp >= 4) {
    reg_alloc<kConsumerRegs>();
    switch (p.BN) {
      case 16: rows_consumer<F, 16>(p, &tmY, L); break;
      case 32: rows_consumer<F, 32>(p, &tmY, L); break;
      case 64: rows_consumer<F, 64>(p, &tmY, L); break;
      default: rows_consumer<F, 128>(p, &tmY, L); break;
    }
    return;
  }
  reg_dealloc<kProducerRegs>();     // the whole producer warpgroup, idle warps 1 and 3 included
  if (warp == 0) {
    if (lane == 0) {
      // ------------------------------------------------------------- A producer: R + 2 halo rows per K block
      const uint32_t row_buf = rows_buf_bytes(p);
      uint32_t it = 0;
      for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
        const RowsTile tc = rows_tile(p, tile);
        const int w0 = tc.ws * p.S, h0 = tc.hg * p.R, b = tc.b;
        for (int kb = 0; kb < p.kblocks; ++kb, ++it) {
          const int s = L.a_ring.acquire(it, (uint32_t)(p.R + 2) * rows_load_bytes(p));
          const uint32_t sa = L.a + s * L.a_stage;
          for (int r = 0; r < p.R + 2; ++r) tma_load_4d(sa + r * row_buf, &tmA, L.a_ring.full(s), kb * 64, w0 - 1, h0 - 1 + r, b);
        }
      }
    }
  } else if (warp == 2) {
    if (lane == 0) {
      // ------------------------------------------------------------- B producer: filter taps (resident or ring)
      if (p.resident) {
        L.b_ring.acquire(0, 9u * p.kblocks * L.b_tile);
        for (int tap = 0; tap < 9; ++tap)
          for (int kb = 0; kb < p.kblocks; ++kb)
            tma_load_3d(L.b + ((kb * 3 + tap % 3) * 3 + tap / 3) * L.b_tile, &tmB, L.b_ring.full(0), kb * 64, tap, 0);
      } else {
        uint32_t it = 0;
        for (int tile = blockIdx.x; tile < p.num_tiles; tile += gridDim.x) {
          const int nt = rows_tile(p, tile).nt;
          for (int kb = 0; kb < p.kblocks; ++kb)
            for (int tap = 0; tap < 9; ++tap, ++it) {
              const int s = L.b_ring.acquire(it, L.b_tile);
              tma_load_3d(L.b + s * L.b_tile, &tmB, L.b_ring.full(s), kb * 64, tap, nt * p.BN);
            }
        }
      }
    }
  }
}

void fill_epi(EpiArgs& e, const sgb_conv_desc* d);
int pick_bn(const sgb_conv_desc* d);
bool epi_tma_ok(const sgb_conv_desc* d, int BN);

using RowsCompiled = EpiVariants<
    kEpiFull | kEpiBias,                                               // generator 3x3
    kEpiFull | kEpiBias | kEpiRelu,                                    // discriminator 3x3
    kEpiFull | kEpiBias | kEpiRelu | kEpiBitsOut,                      // ... writing the ReLU bit plane
    kEpiFull | kEpiMask,                                               // dgrad through a ReLU (bf16 mask)
    kEpiFull | kEpiMask | kEpiMaskBits,                                // dgrad through a ReLU (bit plane)
    kEpiFull>;                                                         // plain dgrad

// Segment width S the halo-row kernel runs a layer at, or 0 where the generic kernel takes it.  S = 128 when W % 128 == 0;
// S = 64 when W % 64 == 0 only if its 256-pixel work items fill every SM at least once: below that, the generic kernel's
// 128-pixel tiles occupy twice as many SMs.
static int rows_segment(const sgb_conv_desc* d) {
  if (!(d->KH == 3 && d->KW == 3 && d->pad_h == 1 && d->pad_w == 1 && d->w_mode == 0 && d->Cin % 64 == 0 && d->Cin <= 256 &&
        d->Cout % 8 == 0))
    return 0;
  if (d->W % 128 == 0 && d->H % 2 == 0) return 128;
  if (d->W % 64 == 0 && d->H % 4 == 0) {
    const int BN = pick_bn(d);
    const long long items = (long long)((d->Cout + BN - 1) / BN) * (d->W / 64) * (d->H / 4) * d->B;
    if (items >= sm_count()) return 64;
  }
  return 0;
}

bool conv3x3_rows_eligible(const sgb_conv_desc* d) { return rows_segment(d) != 0; }

int launch_conv3x3_rows(const sgb_conv_desc* d, cudaStream_t stream) {
  RowsArgs p;
  p.B = d->B; p.H = d->H; p.W = d->W; p.Cin = d->Cin; p.Cout = d->Cout;
  p.S = rows_segment(d);
  SGB_REQUIRE(p.S == 128 || p.S == 64);
  p.R = kRowsItemPix / p.S;
  p.kblocks = d->Cin / 64;
  p.BN = pick_bn(d);      // Cout = 8 (padded image channels) runs as one N = 16 tile
  p.tiles_n = (d->Cout + p.BN - 1) / p.BN;
  p.segs = d->W / p.S;
  p.hgroups = d->H / p.R;
  p.num_tiles = p.tiles_n * p.segs * p.hgroups * d->B;
  const uint32_t budget = 227u * 1024u - 2048u;
  p.use_tma = epi_tma_ok(d, p.BN) ? 1 : 0;
  // tile bytes of the layout with a halo stages and b filter stages (the whole filter when resident)
  auto tiles = [&](int a, int b) { p.a_stages = a; p.b_stages = b; return rows_smem(p).bar; };
  // two staging tiles per warpgroup (a chunk's store overlaps the next chunk's packing), one where that would cost the
  // resident filter its second halo stage (C = 64: 72 KiB taps + 2 x 68 KiB halo + 16 KiB staging)
  p.epi_nbuf = 2;
  p.resident = 1;
  if (p.tiles_n != 1 || tiles(1, 1) > budget) p.resident = 0;
  if (p.resident && p.use_tma && tiles(2, 1) > budget) p.epi_nbuf = 1;
  if (p.resident) {
    const int a_stages = (int)((budget - tiles(0, 1)) / rows_stage_bytes(p));
    p.a_stages = a_stages > 3 ? 3 : a_stages;
    p.b_stages = 1;
  } else {
    const int a_stages = tiles(2, 2) > budget ? 1 : 2;
    const int b_stages = (int)((budget - tiles(a_stages, 0)) / rows_smem(p).b_tile);
    p.a_stages = a_stages;
    p.b_stages = b_stages > 6 ? 6 : b_stages;
    if (p.b_stages < 2) return SGB_ERR_UNSUPPORTED;
  }
  fill_epi(p.e, d);

  CUtensorMap tmA, tmB;
  int rc = make_act_tmap(&tmA, d->x, d->B, d->H, d->W, d->Cin, d->x_cstride, p.S + 2, 1, 1);   // one halo row
  if (rc) return rc;
  {
    uint64_t dims[3] = {(uint64_t)d->Cin, 9, (uint64_t)d->Cout};
    uint64_t strides[2] = {(uint64_t)d->Cin * 2, (uint64_t)d->Cin * 2 * 9};
    uint32_t box[3] = {64, 1, (uint32_t)p.BN};
    rc = make_tmap_bf16(&tmB, d->w, 3, dims, strides, box);
    if (rc) return rc;
  }
  CUtensorMap tmY = tmA;
  if (p.use_tma) {
    rc = make_act_tmap(&tmY, d->y, d->B, d->H, d->W, d->Cout, d->y_cstride, 64, 1, 1);   // one warpgroup's 64 pixels
    if (rc) return rc;
  }
  const size_t smem = smem_request(rows_smem(p).total);
  SGB_REQUIRE(smem <= 227u * 1024u);
  const int grid = p.num_tiles < sm_count() ? p.num_tiles : sm_count();
  const int f = p.use_tma ? epi_flags_of(p.e) : -1;
  return RowsCompiled::launch(f, [&](auto F) {
    return launch_kernel<conv3x3_rows_kernel<decltype(F)::value>>(grid, kRowsThreads, smem, stream, tmA, tmB, tmY, p);
  });
}

}  // namespace sgb
