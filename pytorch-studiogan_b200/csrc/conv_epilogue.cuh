// Fused conv epilogue shared by the wgmma conv kernels: accumulator -> alpha, bias, residual (optionally read from a
// half-resolution tensor = nearest x2 upsample), ReLU, ReLU-mask, post-mask residual -> bf16 / fp32 NHWC store; or the
// attention's row softmax (apply / backward) in place of those steps.
// The questions of a variant are EpiOps<F>; the TMA-store epilogues share the arithmetic epi_pair (one bf16 pair of channels)
// and only differ in where they load its operands from:
//   epilogue_tile_tma  : fp32 accumulator rows staged in shared memory, aux tile in shared memory (run-time flags)
//   epilogue_frag_chunk: straight from the wgmma accumulator registers (every compile-time variant)
// epilogue_row (direct stores, fp32 outputs, ragged channel tails) keeps 16-wide blocks per question: with run-time flags,
// per-pair tests of each question are if-converted into selects on every element.
#pragma once
#include "common.cuh"
#include "ptx.cuh"
#include <type_traits>

namespace sgb {

struct EpiArgs {
  int Cout;
  float alpha;
  const float* alpha_ptr;
  const float* bias;
  const bf16* residual; long long res_cstride; int res_up2; int res_after; float res_scale;
  const bf16* mask; long long mask_cstride;
  int relu;
  void* y; long long y_cstride; int y_fp32;
  // ReLU masks as bit planes (Cout % 64 == 0): one 64-bit word per (pixel, 64-channel chunk), bit j = channel 64 * chunk + j.
  // mask_bits replaces ``mask`` (1/16 of its bytes); relu_bits is written by a relu epilogue for the consumer's backward.
  const unsigned long long* mask_bits;
  unsigned long long* relu_bits;
  // Row softmax of the attention map inside the GEMM epilogues (a query row of a tile is held by the four lanes of a quad):
  //   sm_mode 1: no output; per row and per channel tile the partial (max, sum exp) of its columns -> sm_stats
  //   sm_mode 2: y = exp(acc - m) / l with (m, l) merged from the row's sm_parts partials
  //   sm_mode 3: y = P * (acc - delta[row]) (softmax backward; P arrives through the aux TMA ring, kind 3)
  int sm_mode, sm_parts;
  float* sm_stats;            // [rows][sm_parts = channel tiles][2]
  const float* sm_delta;      // [rows]
};

// Compile-time epilogue variants.  The per-piece loops run on 2 warps per scheduler with little latency hiding, so every
// run-time test of "is there a bias / residual / mask / ragged channel tail" costs issue slots on the critical path of the
// memory-bound layers (~150 SASS instructions per 16-column piece).  F >= 0 fixes those questions at compile time (bit 0
// bias, 1 ReLU, 2 residual before the activation, 3 residual after the mask, 4 mask, 5 Cout % 64 == 0 and every 16-byte
// alignment holds); F < 0 is the fully general run-time version.
static constexpr int kEpiBias = 1, kEpiRelu = 2, kEpiResPre = 4, kEpiResPost = 8, kEpiMask = 16, kEpiFull = 32;
// ... bit 6: the mask is a bit plane (mask_bits), 7 / 8: the residual / the bf16 mask tile arrives through the aux TMA ring,
// 9: the ReLU epilogue also writes its bit plane (relu_bits).  In the fused block-entry dgrad (mask + residual), with these
// three questions left to run time the compiler if-converts both sides of each and the piece loop issues 12 instructions per
// output element (the bias-only variant: 2).
static constexpr int kEpiMaskBits = 64, kEpiAuxRes = 128, kEpiAuxMask = 256, kEpiBitsOut = 512;
// attention: bit 10 softmax statistics (no store), 11 softmax apply, 12 softmax backward (P tile through the aux ring)
static constexpr int kEpiSmStats = 1024, kEpiSmApply = 2048, kEpiSmBwd = 4096;

__host__ __device__ inline int epi_flags_of(const EpiArgs& p) {
  int f = 0;
  if (p.bias) f |= kEpiBias;
  if (p.relu) f |= kEpiRelu;
  if (p.residual) f |= p.res_after ? kEpiResPost : kEpiResPre;
  if (p.mask || p.mask_bits) f |= kEpiMask;
  if (p.mask_bits) f |= kEpiMaskBits;
  if (p.relu && p.relu_bits) f |= kEpiBitsOut;
  if (p.Cout % 64 == 0) f |= kEpiFull;
  if (p.sm_mode == 1) f |= kEpiSmStats;
  if (p.sm_mode == 2) f |= kEpiSmApply;
  if (p.sm_mode == 3) f |= kEpiSmBwd;
  return f;
}

// The compiled variants of a kernel: launch(std::integral_constant<int, F>) runs variant F, or F = -1 (run-time flags) when f
// is not one of them.
template <int... Fs>
struct EpiVariants {
  static constexpr bool has(int f) { return ((f == Fs) || ...); }
  template <class Launch>
  static int launch(int f, Launch&& run) {
    int rc = 0;
    const bool hit = ((f == Fs && ((rc = run(std::integral_constant<int, Fs>{})), true)) || ...);
    return hit ? rc : run(std::integral_constant<int, -1>{});
  }
};

// The questions of epilogue variant F: fixed at compile time for F >= 0, read from the arguments for F < 0.
template <int F>
struct EpiOps {
  bool bias, relu, res_pre, res_post, mask, mask_bits, bits_out;
  bool full_c;                                   // no channel-tail tests (F >= 0 only)
  bool sm_apply, sm_bwd;                         // softmax apply / backward (F >= 0 only)
  __device__ __forceinline__ explicit EpiOps(const EpiArgs& p)
      : bias(F < 0 ? p.bias != nullptr : (F & kEpiBias) != 0),
        relu(F < 0 ? p.relu != 0 : (F & kEpiRelu) != 0),
        res_pre(F < 0 ? (p.residual != nullptr && !p.res_after) : (F & kEpiResPre) != 0),
        res_post(F < 0 ? (p.residual != nullptr && p.res_after) : (F & kEpiResPost) != 0),
        mask(F < 0 ? (p.mask != nullptr || p.mask_bits != nullptr) : (F & kEpiMask) != 0),
        mask_bits(F < 0 ? p.mask_bits != nullptr : (F & kEpiMaskBits) != 0),
        bits_out(F < 0 ? (p.relu != 0 && p.relu_bits != nullptr) : (F & kEpiBitsOut) != 0),
        full_c(F >= 0 && (F & kEpiFull) != 0),
        sm_apply(F >= 0 && (F & kEpiSmApply) != 0),
        sm_bwd(F >= 0 && (F & kEpiSmBwd) != 0) {}
};

// 2^x on the SFU (ex2.approx: 2^-22 relative error, far below the bf16 rounding of the softmax output); the accurate exp2f
// costs ~10 instructions per element and made the softmax epilogues issue bound
__device__ __forceinline__ float fast_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
static constexpr float kLog2e = 1.4426950408889634f;

// The arithmetic that follows acc * alpha, for two adjacent channels (c, c + 1): + bias, fmaf(residual, rs, .), ReLU, mask,
// fmaf(post-mask residual, rs, .).  res / msk: the packed bf16 residual / mask pair (low half = channel c); mbits: the pair's
// two mask bits (bit plane).  pos: bit 0 / 1 set iff the ReLU output of channel c / c + 1 is positive.
// Softmax variants instead: apply exp(f - m) / l with sm = (-m log2e, 1 / l) of the row; backward P * (f - delta) with
// sm.x = delta of the row and res = the packed bf16 P pair.
template <int F>
__device__ __forceinline__ float2 epi_pair(const EpiOps<F>& op, float f0, float f1, float2 b, uint32_t res, uint32_t msk,
                                           uint32_t mbits, float rs, float2 sm, uint32_t& pos) {
  pos = 0u;
  if (op.sm_apply) { f0 = fast_ex2(fmaf(f0, kLog2e, sm.x)) * sm.y; f1 = fast_ex2(fmaf(f1, kLog2e, sm.x)) * sm.y; }
  if (op.sm_bwd) { f0 = bf16_bits_lo(res) * (f0 - sm.x); f1 = bf16_bits_hi(res) * (f1 - sm.x); }
  if (op.bias) { f0 += b.x; f1 += b.y; }
  if (op.res_pre) { f0 = fmaf(bf16_bits_lo(res), rs, f0); f1 = fmaf(bf16_bits_hi(res), rs, f1); }
  if (op.relu) {
    f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f);
    pos = ((f0 > 0.f) ? 1u : 0u) | ((f1 > 0.f) ? 2u : 0u);
  }
  if (op.mask_bits) {
    f0 = (mbits & 1u) ? f0 : 0.f; f1 = (mbits & 2u) ? f1 : 0.f;
  } else if (op.mask) {
    f0 = bf16_bits_lo(msk) > 0.f ? f0 : 0.f; f1 = bf16_bits_hi(msk) > 0.f ? f1 : 0.f;
  }
  if (op.res_post) { f0 = fmaf(bf16_bits_lo(res), rs, f0); f1 = fmaf(bf16_bits_hi(res), rs, f1); }
  return make_float2(f0, f1);
}

// alpha, scaled by *alpha_ptr when it is given
__device__ __forceinline__ float epi_alpha(const EpiArgs& p) { return p.alpha_ptr ? p.alpha * __ldg(p.alpha_ptr) : p.alpha; }

// Residual pixel of output pixel pix = (b, h, w) of an H x W map: pix itself, or (res_up2) its nearest-x2 source pixel in the
// H/2 x W/2 residual.
__device__ __forceinline__ long long epi_rpix(const EpiArgs& p, int b, int h, int w, int H, int W, long long pix) {
  return p.res_up2 ? (((long long)b * (H >> 1) + (h >> 1)) * (W >> 1) + (w >> 1)) : pix;
}

__device__ __forceinline__ bool epi_vec_ok(const EpiArgs& p) {
  return (p.Cout % 8 == 0) && (p.y_cstride % 8 == 0) && (p.residual == nullptr || p.res_cstride % 8 == 0) &&
         (p.mask == nullptr || p.mask_cstride % 8 == 0);
}

// 16 accumulator values -> 16 mask bits (value > 0)
__device__ __forceinline__ uint32_t positive_bits16(const float (&f)[16]) {
  uint32_t b = 0u;
#pragma unroll
  for (int j = 0; j < 16; ++j) b |= (f[j] > 0.f) ? (1u << j) : 0u;
  return b;
}
__device__ __forceinline__ void apply_bits16(float (&f)[16], uint32_t mb) {
#pragma unroll
  for (int j = 0; j < 16; ++j) f[j] = ((mb >> j) & 1u) ? f[j] : 0.f;
}

// One thread = one accumulator row.  t_row: shared-memory address of this thread's accumulator row (acc_store layout);
// stores are predicated by valid.
__device__ __forceinline__ void epilogue_row(const EpiArgs& p, uint32_t t_row, int BN, int n0, bool valid, long long pix,
                                             long long rpix, float alpha, bool vec_ok) {
  const bool res_pre = p.residual != nullptr && !p.res_after;
  const bool res_post = p.residual != nullptr && p.res_after;
  const float rs = p.res_scale;
  for (int c0 = 0; c0 < BN; c0 += 16) {
    uint32_t v[16];
    acc_ld16(t_row + 4u * c0, v);
    const int n = n0 + c0;
    if (!valid || n >= p.Cout) continue;
    float f[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) f[j] = __uint_as_float(v[j]) * alpha;
    if (vec_ok && n + 16 <= p.Cout) {
      if (p.bias) {
        const float4* bp = reinterpret_cast<const float4*>(p.bias + n);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const float4 bb = __ldg(bp + j);
          f[4 * j + 0] += bb.x; f[4 * j + 1] += bb.y; f[4 * j + 2] += bb.z; f[4 * j + 3] += bb.w;
        }
      }
      if (res_pre) {
        const uint4* rp = reinterpret_cast<const uint4*>(p.residual + rpix * p.res_cstride + n);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint4 r = __ldg(rp + j);
          f[8 * j + 0] = fmaf(bf16_bits_lo(r.x), rs, f[8 * j + 0]); f[8 * j + 1] = fmaf(bf16_bits_hi(r.x), rs, f[8 * j + 1]);
          f[8 * j + 2] = fmaf(bf16_bits_lo(r.y), rs, f[8 * j + 2]); f[8 * j + 3] = fmaf(bf16_bits_hi(r.y), rs, f[8 * j + 3]);
          f[8 * j + 4] = fmaf(bf16_bits_lo(r.z), rs, f[8 * j + 4]); f[8 * j + 5] = fmaf(bf16_bits_hi(r.z), rs, f[8 * j + 5]);
          f[8 * j + 6] = fmaf(bf16_bits_lo(r.w), rs, f[8 * j + 6]); f[8 * j + 7] = fmaf(bf16_bits_hi(r.w), rs, f[8 * j + 7]);
        }
      }
      if (p.relu) {
#pragma unroll
        for (int j = 0; j < 16; ++j) f[j] = fmaxf(f[j], 0.f);
        if (p.relu_bits)
          reinterpret_cast<unsigned short*>(p.relu_bits)[(pix * (p.Cout >> 6) + (n >> 6)) * 4 + ((n >> 4) & 3)] =
              (unsigned short)positive_bits16(f);
      }
      if (p.mask_bits) {
        apply_bits16(f, __ldg(reinterpret_cast<const unsigned short*>(p.mask_bits) + (pix * (p.Cout >> 6) + (n >> 6)) * 4 + ((n >> 4) & 3)));
      } else if (p.mask) {
        const uint4* mp = reinterpret_cast<const uint4*>(p.mask + pix * p.mask_cstride + n);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint4 m = __ldg(mp + j);
          f[8 * j + 0] = bf16_bits_lo(m.x) > 0.f ? f[8 * j + 0] : 0.f;
          f[8 * j + 1] = bf16_bits_hi(m.x) > 0.f ? f[8 * j + 1] : 0.f;
          f[8 * j + 2] = bf16_bits_lo(m.y) > 0.f ? f[8 * j + 2] : 0.f;
          f[8 * j + 3] = bf16_bits_hi(m.y) > 0.f ? f[8 * j + 3] : 0.f;
          f[8 * j + 4] = bf16_bits_lo(m.z) > 0.f ? f[8 * j + 4] : 0.f;
          f[8 * j + 5] = bf16_bits_hi(m.z) > 0.f ? f[8 * j + 5] : 0.f;
          f[8 * j + 6] = bf16_bits_lo(m.w) > 0.f ? f[8 * j + 6] : 0.f;
          f[8 * j + 7] = bf16_bits_hi(m.w) > 0.f ? f[8 * j + 7] : 0.f;
        }
      }
      if (res_post) {
        const uint4* rp = reinterpret_cast<const uint4*>(p.residual + rpix * p.res_cstride + n);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          const uint4 r = __ldg(rp + j);
          f[8 * j + 0] = fmaf(bf16_bits_lo(r.x), rs, f[8 * j + 0]); f[8 * j + 1] = fmaf(bf16_bits_hi(r.x), rs, f[8 * j + 1]);
          f[8 * j + 2] = fmaf(bf16_bits_lo(r.y), rs, f[8 * j + 2]); f[8 * j + 3] = fmaf(bf16_bits_hi(r.y), rs, f[8 * j + 3]);
          f[8 * j + 4] = fmaf(bf16_bits_lo(r.z), rs, f[8 * j + 4]); f[8 * j + 5] = fmaf(bf16_bits_hi(r.z), rs, f[8 * j + 5]);
          f[8 * j + 6] = fmaf(bf16_bits_lo(r.w), rs, f[8 * j + 6]); f[8 * j + 7] = fmaf(bf16_bits_hi(r.w), rs, f[8 * j + 7]);
        }
      }
      if (p.y_fp32) {
        float4* yp = reinterpret_cast<float4*>(reinterpret_cast<float*>(p.y) + pix * p.y_cstride + n);
#pragma unroll
        for (int j = 0; j < 4; ++j) yp[j] = make_float4(f[4 * j], f[4 * j + 1], f[4 * j + 2], f[4 * j + 3]);
      } else {
        uint4* yp = reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(p.y) + pix * p.y_cstride + n);
#pragma unroll
        for (int j = 0; j < 2; ++j) {
          uint4 o;
          o.x = pack_bf16x2(f[8 * j + 0], f[8 * j + 1]);
          o.y = pack_bf16x2(f[8 * j + 2], f[8 * j + 3]);
          o.z = pack_bf16x2(f[8 * j + 4], f[8 * j + 5]);
          o.w = pack_bf16x2(f[8 * j + 6], f[8 * j + 7]);
          yp[j] = o;
        }
      }
    } else {
      // ragged / unaligned channel tail (e.g. Cout = 3): scalar path
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int nn = n + j;
        if (nn < p.Cout) {
          float x = f[j];
          if (p.bias) x += __ldg(p.bias + nn);
          if (res_pre) x = fmaf(__bfloat162float(p.residual[rpix * p.res_cstride + nn]), rs, x);
          if (p.relu) x = fmaxf(x, 0.f);
          if (p.mask) x = __bfloat162float(p.mask[pix * p.mask_cstride + nn]) > 0.f ? x : 0.f;
          if (res_post) x = fmaf(__bfloat162float(p.residual[rpix * p.res_cstride + nn]), rs, x);
          if (p.y_fp32) reinterpret_cast<float*>(p.y)[pix * p.y_cstride + nn] = x;
          else reinterpret_cast<bf16*>(p.y)[pix * p.y_cstride + nn] = __float2bfloat16_rn(x);
        }
      }
    }
  }
}


// -------------------------------------------------------------------------------------------------------------------
// Epilogue v2 (bf16 NHWC output, channel tile a multiple of 64): two teams of four warps take alternate 64-channel
// chunks; a team converts its 128 x 64 chunk into a SWIZZLE_128B staging tile in shared memory and one thread issues
// a TMA tensor store (full 128-byte lines, asynchronous, out-of-range rows / channels clipped by the hardware).  This
// replaces 16-byte-per-lane strided global stores, which bound every wide 1x1 layer (K = 64..128) at ~1/6 of HBM speed.
// -------------------------------------------------------------------------------------------------------------------
static constexpr int kEpiThreads = 256;           // 8 epilogue warps

// Optional auxiliary operand of the epilogue (the residual OR the ReLU-mask tensor) staged by TMA: one SWIZZLE_128B box of
// the same pixels (or of the half-resolution source pixels for the nearest-x2 residual) per 64-channel chunk.  The boxes are
// fetched by a dedicated producer warp into a per-team ring of ``depth`` tiles (full / empty mbarriers), in the order the team
// consumes its chunks, so their ~1-2 us latency under load overlaps ``depth`` chunks of epilogue work instead of one.
struct EpiAux {
  int kind;                 // 1 residual, 2 mask
  uint32_t tiles;           // this team's first aux tile (1024-byte aligned), tiles 16 KiB apart
  MbarRing ring;            // this team's ring, one slot per tile
  uint32_t* cnt;            // per-thread count of chunks consumed by this team
  int arow;                 // aux-tile row this thread reads
};

__device__ __forceinline__ uint4 ld_shared_v4(uint32_t addr) {
  uint4 r;
  asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "r"(addr));
  return r;
}
static constexpr int kEpiStageBytes = 128 * 128;  // one 128-row x 64-channel bf16 chunk

// The next of a team's nbuf (1..4) staging tiles, used round-robin (sbuf = its index), so a chunk only waits for the store
// issued nbuf chunks ago: the latency of the previous tensor stores is off the critical path and more bytes are in flight.
__device__ __forceinline__ uint32_t epi_stage_next(uint32_t stage, uint32_t tile_bytes, int nbuf, uint32_t& sbuf, bool leader) {
  const uint32_t cur = stage + sbuf * tile_bytes;
  if (leader) bulk_wait_read(nbuf);              // the store that last used this staging tile has finished reading it
  sbuf = (sbuf + 1u == (uint32_t)nbuf) ? 0u : sbuf + 1u;
  return cur;
}

// Staged epilogue of the run-time general kernel (F = -1).
// t_row : shared-memory address of this thread's accumulator row (first column of the accumulator).
// c1..c3: box coordinates (w0, h0, b0) of the tile in the output tensor map; channel coordinate = n0 + chunk * 64.
// stage : this team's first staging tile (1024-byte aligned), nbuf tiles used round-robin (sbuf = next one).
// team in {0,1}; row = accumulator row of this thread.  aux: the team's aux ring, or nullptr.
// A thread converts all four 16-column pieces of its row of the chunk; a team is 4 warps.
__device__ __forceinline__ void epilogue_tile_tma(const EpiArgs& p, const CUtensorMap* tmY, uint32_t t_row, int BN, int n0,
                                                  int c1, int c2, int c3, bool valid, long long pix, long long rpix, float alpha,
                                                  uint32_t stage, int nbuf, uint32_t& sbuf, int team, int row, bool leader,
                                                  const EpiAux* aux) {
  constexpr int kTeamThreads = 128;
  const EpiOps<-1> op(p);
  const long long nw = p.Cout >> 6;
  const float rs = p.res_scale;
  const uint32_t sw = (uint32_t)(row & 7);
  // 1: residual tile via TMA, 2: mask tile via TMA
  const int aux_kind = aux ? aux->kind : 0;
  const uint32_t asw = aux ? (uint32_t)(aux->arow & 7) : 0u;
  for (int cc = team; cc * 64 < BN; cc += 2) {
    const int nbase = n0 + cc * 64;
    if (nbase >= p.Cout) break;
    uint32_t mlo = 0u, mhi = 0u, olo = 0u, ohi = 0u;
    if (op.mask_bits && valid) {                 // 8 bytes instead of a 128-byte line of the bf16 activation
      const uint2 m = __ldg(reinterpret_cast<const uint2*>(p.mask_bits) + pix * nw + (nbase >> 6));
      mlo = m.x; mhi = m.y;
    }
    const uint32_t stage_cur = epi_stage_next(stage, kEpiStageBytes, nbuf, sbuf, leader);
    const uint32_t srow = stage_cur + (uint32_t)row * 128u;
    named_bar_sync(1 + team, kTeamThreads);
    uint32_t arow_addr = 0u, aslot = 0u;
    if (aux_kind) {                              // residual / mask chunk: one TMA box (fetched ahead by the aux producer warp)
      aslot = aux->ring.wait(*aux->cnt);
      arow_addr = aux->tiles + aslot * kEpiStageBytes + (uint32_t)aux->arow * 128u;
      *aux->cnt += 1u;
    }
    auto piece = [&](const int s, const uint32_t (&v)[16], const uint32_t mb) -> uint32_t {
        const int n = nbase + s * 16;
        float f[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) f[j] = __uint_as_float(v[j]) * alpha;
        const int nvalid = op.full_c ? 16 : p.Cout - n;   // channels of this 16-wide piece inside the tensor: >= 16, 8 (Cout % 16 == 8) or <= 0
        const bool in_c = op.full_c || nvalid > 0;
        // 16 bf16 values of this row: this piece's two 16-byte units of the aux tile, or global memory (zero past the tensor)
        auto load16 = [&](int kind, const bf16* src, uint32_t (&w)[8]) {
#pragma unroll
          for (int j = 0; j < 2; ++j)
            reinterpret_cast<uint4*>(w)[j] = (aux_kind == kind) ? ld_shared_v4(arow_addr + (((uint32_t)(2 * s + j) ^ asw) << 4))
                                             : ((op.full_c || 8 * j < nvalid) ? __ldg(reinterpret_cast<const uint4*>(src) + j)
                                                                             : make_uint4(0u, 0u, 0u, 0u));
        };
        float b[16] = {};
        uint32_t r[8] = {}, m[8] = {}, w[8];
        if (op.bias && in_c) {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (op.full_c || 4 * j < nvalid) reinterpret_cast<float4*>(b)[j] = __ldg(reinterpret_cast<const float4*>(p.bias + n) + j);
        }
        if ((op.res_pre || op.res_post) && in_c && valid) load16(1, p.residual + rpix * p.res_cstride + n, r);
        if (op.mask && !op.mask_bits && in_c && valid) load16(2, p.mask + pix * p.mask_cstride + n, m);
        uint32_t ob = 0u;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
          uint32_t pos;
          const float2 o = epi_pair(op, f[2 * k], f[2 * k + 1], make_float2(b[2 * k], b[2 * k + 1]), r[k], m[k], mb >> (2 * k), rs,
                                    make_float2(0.f, 1.f), pos);
          ob |= pos << (2 * k);
          w[k] = pack_bf16x2(o.x, o.y);
        }
        // 16 channels = two 16-byte units (2s, 2s+1) of this row's 128-byte line; unit u lives at (u ^ (row & 7))
        st_shared_v4(srow + (((uint32_t)(2 * s) ^ sw) << 4), w[0], w[1], w[2], w[3]);
        st_shared_v4(srow + (((uint32_t)(2 * s + 1) ^ sw) << 4), w[4], w[5], w[6], w[7]);
        return ob;
    };
#pragma unroll 1
    for (int s = 0; s < 4; ++s) {
      uint32_t v[16];
      acc_ld16(t_row + 4u * (cc * 64 + s * 16), v);
      const uint32_t ob = piece(s, v, ((s < 2 ? mlo : mhi) >> (16 * (s & 1))) & 0xFFFFu);
      if (s < 2) olo |= ob << (16 * (s & 1));
      else ohi |= ob << (16 * (s & 1));
    }
    if (op.bits_out && valid) {
      reinterpret_cast<uint2*>(p.relu_bits)[pix * nw + (nbase >> 6)] = make_uint2(olo, ohi);
    }
    fence_proxy_async_smem();                    // generic-proxy smem writes -> visible to the TMA (async proxy)
    named_bar_sync(1 + team, kTeamThreads);
    if (leader) {
      tma_store_4d(tmY, stage_cur, nbase, c1, c2, c3);
      bulk_commit();
      if (aux_kind) mbar_arrive(aux->ring.empty(aslot));   // every thread of the team is past its last read of the aux tile (barrier above)
    }
  }
}

// -------------------------------------------------------------------------------------------------------------------
// Epilogue straight from the wgmma accumulator registers of one warpgroup: 64 pixel rows x BN channels in the Wgmma
// fragment layout (thread = warp w, lane l of the warpgroup: rows 16w + l/4 and 16w + l/4 + 8, columns 8j + 2(l%4) + 0 / 1).
// No fp32 staging: per 64-channel chunk the warpgroup packs bf16 pairs (epi_pair) into a SWIZZLE_128B staging tile
// [64 rows][64 ch] (8 KiB; a thread's pair of column block j goes to 16-byte unit j ^ (row & 7), conflict-free) and one thread
// issues the TMA store of the box (64 ch, 64 px).  ReLU bit planes are OR-reduced over the four lanes that share a row.
//   cc         : 64-channel chunk of the accumulator (compile-time after unrolling: the fragments stay in registers).
//   pix / rpix : output / residual pixel of this thread's two rows; valid: the row lies inside the output (rows outside are
//                clipped by the TMA store; their global loads read pixel 0 and their bit-plane words are not written).
//   stage      : this warpgroup's first staging tile (1024-aligned), nbuf (1..4) tiles used round-robin (sbuf = next one).
//   bar        : named barrier of the warpgroup.
//   aux_tile   : F with kEpiAuxRes / kEpiAuxMask / kEpiSmBwd: the chunk's residual / mask / P box (SWIZZLE_128B, 128-byte
//                rows) filled by the aux producer; arow = the box row of each of this thread's two rows.  Other variants read
//                global memory.
//   sm         : softmax apply / backward: epi_pair's row constants of this thread's two rows (sm_row_apply, sm_delta).
static constexpr uint32_t kFragStageBytes = 64 * 128;

template <int F, int BN>
__device__ __forceinline__ void epilogue_frag_chunk(const EpiArgs& p, const CUtensorMap* tmY, const float (&acc)[BN / 2], int cc,
                                                    int nbase, int c1, int c2, int c3, const long long (&pix)[2],
                                                    const long long (&rpix)[2], const bool (&valid)[2], float alpha, uint32_t stage,
                                                    int nbuf, uint32_t& sbuf, uint32_t bar, bool leader, uint32_t aux_tile = 0u,
                                                    const uint32_t (&arow)[2] = {0u, 0u}, const float2 (&sm)[2] = {}) {
  constexpr int aux_kind = F < 0 ? 0 : ((F & kEpiAuxRes) ? 1 : ((F & kEpiAuxMask) ? 2 : ((F & kEpiSmBwd) ? 3 : 0)));
  // the ReLU is the last arithmetic of the pair (no mask, no post-mask residual): take the bits from the packed output word --
  // adding 0x7FFF to a post-ReLU bf16 half (+0 or a positive value <= 0x7F80) sets its bit 15 iff it is non-zero, without
  // carrying into its neighbour; fewer instructions than a compare per element, and the bit plane is paid for by write-bound layers
  constexpr bool bits_from_packed = F >= 0 && (F & kEpiBitsOut) != 0 && (F & (kEpiMask | kEpiResPost)) == 0;
  const EpiOps<F> op(p);
  const float rs = p.res_scale;
  const long long nw = p.Cout >> 6;
  const uint32_t w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31, q = l & 3;
  const uint32_t r0 = 16u * w + (l >> 2);
  const long long lpix[2] = {valid[0] ? pix[0] : 0ll, valid[1] ? pix[1] : 0ll};
  const long long lrpix[2] = {valid[0] ? rpix[0] : 0ll, valid[1] ? rpix[1] : 0ll};
  const uint32_t stage_cur = epi_stage_next(stage, kFragStageBytes, nbuf, sbuf, leader);
  named_bar_sync(bar, 128);
  uint32_t mb[2][2] = {{0u, 0u}, {0u, 0u}}, ob[2][2] = {{0u, 0u}, {0u, 0u}};
  if (op.mask_bits) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      const uint2 m = __ldg(reinterpret_cast<const uint2*>(p.mask_bits) + lpix[hr] * nw + (nbase >> 6));
      mb[hr][0] = m.x; mb[hr][1] = m.y;
    }
  }
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int j = cc * 8 + jj;                   // 8-column block of the accumulator
    const int n = nbase + 8 * jj + 2 * (int)q;
    const bool in_c = op.full_c || nbase + 8 * jj < p.Cout;   // Cout % 8 == 0: a column block is all in or all out
    const uint32_t bit = 8u * (jj & 3) + 2u * q;              // bit of column 0 of the pair in its 32-bit half of the word
    float2 bb = make_float2(0.f, 0.f);
    if (op.bias && in_c) bb = __ldg(reinterpret_cast<const float2*>(p.bias + n));
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      // this pair's 4 bytes in the aux box: 16-byte unit jj of row arow sits at jj ^ (arow & 7), conflict-free like the staging
      const uint32_t aaddr = aux_tile + arow[hr] * 128u + ((((uint32_t)jj) ^ (arow[hr] & 7u)) << 4) + 4u * q;
      uint32_t res = 0u, msk = 0u, pos;
      if ((op.res_pre || op.res_post || op.sm_bwd) && in_c)
        res = (aux_kind == 1 || aux_kind == 3) ? ld_shared_b32(aaddr)
                                               : __ldg(reinterpret_cast<const unsigned int*>(p.residual + lrpix[hr] * p.res_cstride + n));
      if (op.mask && !op.mask_bits && in_c)
        msk = aux_kind == 2 ? ld_shared_b32(aaddr) : __ldg(reinterpret_cast<const unsigned int*>(p.mask + lpix[hr] * p.mask_cstride + n));
      const float2 o = epi_pair(op, acc[4 * j + 2 * hr] * alpha, acc[4 * j + 2 * hr + 1] * alpha, bb, res, msk,
                                mb[hr][jj >> 2] >> bit, rs, sm[hr], pos);
      const uint32_t pk = pack_bf16x2(o.x, o.y);
      if (bits_from_packed) {
        const uint32_t t = pk + 0x7FFF7FFFu;
        ob[hr][jj >> 2] |= ((t >> 15) & 1u) << bit | (t >> 31) << (bit + 1);
      } else if (op.bits_out) {
        ob[hr][jj >> 2] |= pos << bit;
      }
      const uint32_t r = r0 + 8u * hr;
      st_shared_b32(stage_cur + r * 128u + ((((uint32_t)jj) ^ (r & 7u)) << 4) + 4u * q, pk);
    }
  }
  if (op.bits_out) {
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        ob[hr][k] |= __shfl_xor_sync(0xffffffffu, ob[hr][k], 1);
        ob[hr][k] |= __shfl_xor_sync(0xffffffffu, ob[hr][k], 2);
      }
      if (q == 0 && valid[hr]) reinterpret_cast<uint2*>(p.relu_bits)[pix[hr] * nw + (nbase >> 6)] = make_uint2(ob[hr][0], ob[hr][1]);
    }
  }
  fence_proxy_async_smem();                      // generic-proxy smem writes -> visible to the TMA (async proxy)
  named_bar_sync(bar, 128);
  if (leader) {
    tma_store_4d(tmY, stage_cur, nbase, c1, c2, c3);
    bulk_commit();
  }
}

// All 64-channel chunks of one 64-row accumulator block whose rows all lie inside the output (halo-row kernel).
template <int F, int BN>
__device__ __forceinline__ void epilogue_frag_tma(const EpiArgs& p, const CUtensorMap* tmY, const float (&acc)[BN / 2], int n0,
                                                  int c1, int c2, int c3, const long long (&pix)[2], const long long (&rpix)[2],
                                                  float alpha, uint32_t stage, int nbuf, uint32_t& sbuf, uint32_t bar, bool leader) {
  static_assert(F < 0 || (F & (kEpiAuxRes | kEpiAuxMask)) == 0, "the aux ring is read by callers of epilogue_frag_chunk");
  const bool full_c = F >= 0 && (F & kEpiFull) != 0;
  const bool valid[2] = {true, true};
#pragma unroll                                   // static accumulator indices: the fragments stay in registers
  for (int cc = 0; cc * 64 < BN; ++cc) {
    const int nbase = n0 + cc * 64;
    if (!full_c && nbase >= p.Cout) break;
    epilogue_frag_chunk<F, BN>(p, tmY, acc, cc, nbase, c1, c2, c3, pix, rpix, valid, alpha, stage, nbuf, sbuf, bar, leader);
  }
}

// ---------------------------------------------------------------------------------------- softmax rows in the fragment layout
// A row's columns of the tile are held by the four lanes of a quad (lane q: columns 8j + 2q + 0 / 1), so every row reduction
// is a reduction over this thread's columns and two xor shuffles (1, 2) within the quad; the results are the same in all four
// lanes.  Every thread of the warp executes the shuffles, whatever its rows' validity.

// Statistics pass (sm_mode 1) of one 64-row accumulator block: per row, (max, sum exp(. - max)) of the nchunk valid 64-column
// chunks of the tile (channel tile `part`), stored by lane 0 of the quad; rows outside the output store nothing.
template <int BN>
__device__ __forceinline__ void epilogue_frag_smstats(const EpiArgs& p, const float (&acc)[BN / 2], int nchunk, int part,
                                                      const long long (&pix)[2], const bool (&valid)[2], float alpha) {
  const float a2 = alpha * kLog2e;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    float m0 = -INFINITY, m1 = -INFINITY;       // two chains: one warp per scheduler runs this, so latency is not hidden
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      if (j < 8 * nchunk) { m0 = fmaxf(m0, acc[4 * j + 2 * hr] * alpha); m1 = fmaxf(m1, acc[4 * j + 2 * hr + 1] * alpha); }
    float m = fmaxf(m0, m1);
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
    const float m2 = -m * kLog2e;
    float l0 = 0.f, l1 = 0.f;
#pragma unroll
    for (int j = 0; j < BN / 8; ++j)
      if (j < 8 * nchunk) { l0 += fast_ex2(fmaf(acc[4 * j + 2 * hr], a2, m2)); l1 += fast_ex2(fmaf(acc[4 * j + 2 * hr + 1], a2, m2)); }
    float l = l0 + l1;
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    if ((threadIdx.x & 3) == 0 && valid[hr]) reinterpret_cast<float2*>(p.sm_stats)[pix[hr] * p.sm_parts + part] = make_float2(m, l);
  }
}

// Apply pass (sm_mode 2), first half: lane q of the quad merges the row's partials q, q + 4, q + 8, ...; this loads the first
// two of them ((-inf, 0) past sm_parts and for rows outside the output).  Issued before the main loop, whose MMAs hide the load.
__device__ __forceinline__ void sm_row_load(const EpiArgs& p, long long pix, bool valid, float2 (&t)[2]) {
  const int q = threadIdx.x & 3;
  const float2* st = reinterpret_cast<const float2*>(p.sm_stats) + pix * p.sm_parts;
#pragma unroll
  for (int k = 0; k < 2; ++k) t[k] = (valid && q + 4 * k < p.sm_parts) ? __ldcg(st + q + 4 * k) : make_float2(-INFINITY, 0.f);
}

// Apply pass, second half: merges t with this lane's further partials (sm_parts > 8) and across the quad into epi_pair's row
// constants (-m log2e, 1 / l); (0, 1) for rows outside the output.
__device__ __forceinline__ float2 sm_row_apply(const EpiArgs& p, long long pix, bool valid, const float2 (&t)[2]) {
  const int q = threadIdx.x & 3;
  const float2* st = reinterpret_cast<const float2*>(p.sm_stats) + pix * p.sm_parts;
  float m = fmaxf(t[0].x, t[1].x);
  for (int i = q + 8; valid && i < p.sm_parts; i += 4) m = fmaxf(m, __ldcg(&st[i].x));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 1));
  m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, 2));
  // an absent partial (-inf, 0) adds 0 * ex2(-inf) = 0
  float l = t[0].y * fast_ex2((t[0].x - m) * kLog2e) + t[1].y * fast_ex2((t[1].x - m) * kLog2e);
  for (int i = q + 8; valid && i < p.sm_parts; i += 4) {
    const float2 u = __ldcg(st + i);
    l += u.y * fast_ex2((u.x - m) * kLog2e);
  }
  l += __shfl_xor_sync(0xffffffffu, l, 1);
  l += __shfl_xor_sync(0xffffffffu, l, 2);
  return valid ? make_float2(-m * kLog2e, 1.f / l) : make_float2(0.f, 1.f);
}

}  // namespace sgb
