// sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), wgmma (warpgroup MMA with shared-memory descriptors).
// Hand-written for H100; nothing here compiles for an older arch and nothing here is a fallback.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>

namespace sgb {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init() {
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() {
  asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// Bounded spin: a descriptor / phase bug must surface as a trap, not as a hung GPU box.
#ifndef SGB_SPIN_LIMIT
#define SGB_SPIN_LIMIT (1u << 26)
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SGB_SPIN_LIMIT) { __trap(); }
  }
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2) {
  asm volatile(
      "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2)
      : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* m, uint32_t bar, int c0, int c1, int c2,
                                            int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(m)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
      : "memory");
}

__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, uint32_t src, int c0, int c1, int c2, int c3) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
               ::"l"(reinterpret_cast<uint64_t>(m)), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// Waits until the oldest of the last n (1..4) committed bulk groups has finished reading its shared-memory source: at most
// n - 1 groups are still reading.
__device__ __forceinline__ void bulk_wait_read(int n) {
  if (n == 1) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
  else if (n == 2) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");
  else if (n == 3) asm volatile("cp.async.bulk.wait_group.read 2;" ::: "memory");
  else asm volatile("cp.async.bulk.wait_group.read 3;" ::: "memory");
}
__device__ __forceinline__ void bulk_wait_all() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
// Counts this thread's warp at the barrier without waiting for it (the other side waits with named_bar_sync).
__device__ __forceinline__ void named_bar_arrive(uint32_t id, uint32_t nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ uint32_t ld_shared_b32(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(addr) : "memory");
  return v;
}
__device__ __forceinline__ void st_shared_v4(uint32_t addr, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(addr), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void st_shared_b32(uint32_t addr, uint32_t a) {
  asm volatile("st.shared.b32 [%0], %1;" ::"r"(addr), "r"(a) : "memory");
}

// ---------------------------------------------------------------- register reallocation between warpgroups
// Executed by all 128 threads of a warpgroup.  A 384-thread CTA launched at 168 registers per thread (the
// __launch_bounds__(384, 1) cap) can move 128 x (168 - 40) registers from the producer warpgroup to the two consumer
// warpgroups: 128 x 40 + 256 x 232 = 64 512 <= 65 536.
template <int R>
__device__ __forceinline__ void reg_dealloc() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void reg_alloc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
static constexpr int kProducerRegs = 40, kConsumerRegs = 232;

// ---------------------------------------------------------------- wgmma
// D[64 x N] (+)= A[64 x 16] * B[16 x N], bf16 inputs from shared-memory descriptors, f32 accumulators in registers; issued by
// all 128 threads of a warpgroup.  TA / TB = 1: the operand is MN-major (transposed), 0: K-major.
// Accumulator fragment of thread (warp w of the warpgroup, lane l): d[4j + 0 / 1] = row 16w + l/4, columns 8j + 2(l%4) + 0 / 1;
// d[4j + 2 / 3] = the same columns of row 16w + l/4 + 8.
template <int N> struct Wgmma;
template <> struct Wgmma<8> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[4], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %6, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n8k16.f32.bf16.bf16 {%0, %1, %2, %3}, %4, %5, p, 1, 1, %7, %8;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<16> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[8], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<32> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[16], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, %20;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<64> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, %35, %36;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
};
template <> struct Wgmma<128> {
  template <int TA, int TB>
  static __device__ __forceinline__ void mma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %67, %68;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(accumulate), "n"(TA), "n"(TB));
  }
};

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving reads / writes of the accumulator registers across an asynchronous wgmma.
template <int R>
__device__ __forceinline__ void acc_fence(float (&d)[R]) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------- mbarrier rings
// A ring of `slots` shared-memory buffers handed from a TMA producer to its consumers, guarded by one block of mbarriers
// [full x slots][empty x slots].  Both sides count the same running position it: slot it % slots, in round it / slots.
// A full barrier completes once per round (one producer arrival plus the TMA bytes), an empty barrier once the consumers
// are done with the slot, so a producer waits with the other parity (a fresh ring counts as released).
struct MbarRing {
  uint32_t bar;   // first full barrier
  int slots;
  __host__ __device__ static constexpr uint32_t bytes(int slots) { return 16u * (uint32_t)slots; }
  __host__ __device__ uint32_t end() const { return bar + bytes(slots); }
  __device__ uint32_t full(int s) const { return bar + 8u * s; }
  __device__ uint32_t empty(int s) const { return bar + 8u * (slots + s); }
  __device__ int slot(uint32_t it) const { return it % slots; }
  __device__ uint32_t phase(uint32_t it) const { return (it / slots) & 1; }
  // Thread 0, before the CTA-wide barrier that publishes the ring.
  __device__ void init(uint32_t consumer_arrivals) const {
    for (int s = 0; s < slots; ++s) {
      mbar_init(full(s), 1);
      mbar_init(empty(s), consumer_arrivals);
    }
  }
  // Producer: waits until position it's slot is released, then arms its full barrier for tx_bytes of TMA loads.
  __device__ int acquire(uint32_t it, uint32_t tx_bytes) const {
    const int s = slot(it);
    mbar_wait(empty(s), phase(it) ^ 1);
    mbar_arrive_expect_tx(full(s), tx_bytes);
    return s;
  }
  // Consumer: waits until position it's slot is filled.
  __device__ int wait(uint32_t it) const {
    const int s = slot(it);
    mbar_wait(full(s), phase(it));
    return s;
  }
  // Consumer warp (converged): one arrival on slot s's empty barrier, from lane 0.
  __device__ void release(int s) const {
    __syncwarp();
    if ((threadIdx.x & 31) == 0) mbar_arrive(empty(s));
  }
  // Consumer warp, after committing the MMAs that read slot s: once the previous group has retired, its slot (prev) is free.
  __device__ void release_prev(int& prev, int s) const {
    wgmma_wait<1>();
    if (prev >= 0) release(prev);
    prev = s;
  }
};

// Dynamic shared memory is carved from its first 1024-byte boundary (SWIZZLE_128B tiles need it), so the host requests a
// layout's total plus the worst-case padding.
__device__ __forceinline__ uint32_t smem_aligned(const void* smem_raw) { return (smem_u32(smem_raw) + 1023u) & ~1023u; }
inline size_t smem_request(uint32_t total) { return (size_t)total + 1024; }

// The constant B operand of the bias-gradient MMAs: 1 KiB of bf16 1.0 (8 K-major rows of 64), written by a CTA of nthreads and
// fenced for the tensor cores, which read it through the async proxy.  Precedes the CTA-wide barrier.
static constexpr uint32_t kOnesSlabBytes = 1024;
__device__ __forceinline__ void fill_ones_slab(uint32_t base, int nthreads) {
  for (int i = threadIdx.x; i < (int)kOnesSlabBytes / 4; i += nthreads) st_shared_b32(base + 4u * i, 0x3F803F80u);
  fence_proxy_async_smem();
}

// Accumulator staging in shared memory: fp32 rows of ``ld`` = acc_row_bytes(N) bytes, 16 more than the row (the padding
// staggers consecutive rows across the banks, so the one-row-per-thread 16-byte reads of the fused epilogues do not conflict).
__host__ __device__ inline uint32_t acc_row_bytes(int N) { return (uint32_t)N * 4u + 16u; }
// Stores this warpgroup's 64-row fragment at ``base`` (its first row).
template <int N>
__device__ __forceinline__ void acc_store(const float (&d)[N / 2], uint32_t base, uint32_t ld) {
  const uint32_t w = (threadIdx.x >> 5) & 3, l = threadIdx.x & 31;
  const uint32_t r0 = base + (16u * w + (l >> 2)) * ld + 8u * (l & 3);
#pragma unroll
  for (int j = 0; j < N / 8; ++j) {
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + 32u * j), "f"(d[4 * j]), "f"(d[4 * j + 1]) : "memory");
    asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(r0 + 8u * ld + 32u * j), "f"(d[4 * j + 2]), "f"(d[4 * j + 3]) : "memory");
  }
}
// 16 consecutive fp32 accumulator columns of one row, as raw bits.
__device__ __forceinline__ void acc_ld16(uint32_t addr, uint32_t (&v)[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[4 * i]), "=r"(v[4 * i + 1]), "=r"(v[4 * i + 2]), "=r"(v[4 * i + 3])
                 : "r"(addr + 16u * i)
                 : "memory");
}

// Shared-memory matrix descriptor (wgmma), SWIZZLE_128B.
//   K-major  operand tile [rows][64 bf16]: SBO = 1024 (8 rows x 128 B), LBO unused.
//   MN-major operand tile [k rows][64 bf16]: SBO = 1024 (8 k-rows), LBO = bytes between 64-wide MN atoms.
__device__ __forceinline__ uint64_t make_sdesc_sw128(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  uint64_t d = 0;
  d |= static_cast<uint64_t>((saddr & 0x3FFFFu) >> 4);
  d |= static_cast<uint64_t>((lbo_bytes >> 4) & 0x3FFFu) << 16;
  d |= static_cast<uint64_t>((sbo_bytes >> 4) & 0x3FFFu) << 32;
  d |= 1ull << 62;  // layout type = SWIZZLE_128B
  return d;
}

}  // namespace sgb
