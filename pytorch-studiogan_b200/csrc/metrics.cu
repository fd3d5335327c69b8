// Evaluation metrics on the device in fp64 (the reference computes them on the host in fp64 with numpy / scipy / sklearn):
//
//   * feature moments  [sum f, sum f f^T]  accumulated batch by batch (src/metrics/fid.py:65-98: np.mean + np.cov): the
//     [N, 2048] feature matrix never has to exist, and across ranks the 33.5 MB moment matrix is all-reduced instead of the
//     features being gathered (SURVEY 8e);
//   * PRDC (src/metrics/prdc.py:87-168): the three N x N euclidean distance matrices (20 GB each at N = 50 000 on the host)
//     are produced tile by tile as |x|^2 + |y|^2 - 2 x.y and reduced on the fly to what the four metrics need -- the
//     (k+1)-th smallest distance per row, per-row minimum / any, per-column counts -- and are never stored.
//
// One building block: a 64 x 64 output tile per CTA (256 threads, 4 x 4 register micro-tile each), operands staged through
// shared memory in 16-deep slices, double-precision FMA.  These are CUDA-core fp64 kernels: the arithmetic must track the
// host fp64 reference (threshold comparisons in PRDC, a 2048^2 covariance feeding a matrix square root in FID), and
// Hopper's tensor pipe has no fp64 advantage to offer here.
#include "common.cuh"

namespace sgb {

static constexpr int kMT = 64;     // tile edge
static constexpr int kMK = 16;     // slice depth
static constexpr int kMaxK1 = 8;   // nearest_k + 1 <= 8

// acc[a][b] += sum_k A[row0 + ty*4 + a][k] * B[col0 + tx*4 + b][k] for k in [0, D): both operands row-major [rows][D].
template <typename TA, typename TB>
__device__ __forceinline__ void tile_dot(const TA* __restrict__ A, long long lda, int rowsA, int row0, const TB* __restrict__ Bm,
                                         long long ldb, int rowsB, int col0, int D, double (&acc)[4][4], double (*As)[kMT + 1],
                                         double (*Bs)[kMT + 1]) {
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  for (int k0 = 0; k0 < D; k0 += kMK) {
    __syncthreads();
    for (int e = threadIdx.x; e < kMT * kMK; e += 256) {       // 64 rows x 16 k, k fastest in memory
      const int r = e / kMK, k = e % kMK;
      const int ra = row0 + r, rb = col0 + r;
      As[k][r] = (ra < rowsA && k0 + k < D) ? (double)A[(long long)ra * lda + k0 + k] : 0.0;
      Bs[k][r] = (rb < rowsB && k0 + k < D) ? (double)Bm[(long long)rb * ldb + k0 + k] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kMK; ++k) {
      double av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) av[a] = As[k][ty * 4 + a];
#pragma unroll
      for (int b = 0; b < 4; ++b) bv[b] = Bs[k][tx * 4 + b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
    }
  }
}

// ------------------------------------------------------------------------------------------------ feature moments
// outer[i][j] += sum_r f[r][i] * f[r][j] for the upper-triangular 64 x 64 blocks (bi <= bj); sum[i] += sum_r f[r][i].
__global__ void __launch_bounds__(256) moments_kernel(const float* __restrict__ f, int n, int D, double* __restrict__ sum,
                                                       double* __restrict__ outer, int nblk) {
  __shared__ double As[kMK][kMT + 1], Bs[kMK][kMT + 1];
  // linear block index -> (bi, bj) with bi <= bj
  int t = blockIdx.x, bi = 0;
  while (t >= nblk - bi) { t -= nblk - bi; ++bi; }
  const int bj = bi + t;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  double acc[4][4];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) acc[a][b] = 0.0;
  double colsum = 0.0;                                   // diagonal blocks also produce the column sums (thread = column)
  for (int r0 = 0; r0 < n; r0 += kMK) {
    __syncthreads();
    for (int e = threadIdx.x; e < kMT * kMK; e += 256) {         // 16 feature rows x 64 columns, columns fastest in memory
      const int k = e / kMT, c = e % kMT;
      const bool ok = r0 + k < n;
      As[k][c] = (ok && bi * kMT + c < D) ? (double)f[(long long)(r0 + k) * D + bi * kMT + c] : 0.0;
      Bs[k][c] = (ok && bj * kMT + c < D) ? (double)f[(long long)(r0 + k) * D + bj * kMT + c] : 0.0;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kMK; ++k) {
      double av[4], bv[4];
#pragma unroll
      for (int a = 0; a < 4; ++a) av[a] = As[k][ty * 4 + a];
#pragma unroll
      for (int b = 0; b < 4; ++b) bv[b] = Bs[k][tx * 4 + b];
#pragma unroll
      for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = fma(av[a], bv[b], acc[a][b]);
      if (bi == bj && threadIdx.x < kMT) colsum += As[k][threadIdx.x];
    }
  }
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int i = bi * kMT + ty * 4 + a, j = bj * kMT + tx * 4 + b;
      if (i < D && j < D) outer[(long long)i * D + j] += acc[a][b];
    }
  if (bi == bj && threadIdx.x < kMT && bi * kMT + threadIdx.x < D) sum[bi * kMT + threadIdx.x] += colsum;
}

// mu = sum / n;  sigma[i][j] = (outer[min][max] - n mu_i mu_j) / (n - 1)   (np.cov(rowvar=False))
__global__ void __launch_bounds__(256) moments_finalize_kernel(const double* __restrict__ sum, const double* __restrict__ outer, double n,
                                                                int D, double* __restrict__ mu, double* __restrict__ sigma) {
  const long long total = (long long)D * D;
  for (long long e = (long long)blockIdx.x * 256 + threadIdx.x; e < total; e += (long long)gridDim.x * 256) {
    const int i = (int)(e / D), j = (int)(e % D);
    const int lo = i < j ? i : j, hi = i < j ? j : i;
    const double mi = sum[i] / n, mj = sum[j] / n;
    sigma[e] = (outer[(long long)lo * D + hi] - n * mi * mj) / (n - 1.0);
    if (j == 0) mu[i] = mi;
  }
}

// ------------------------------------------------------------------------------------------------ PRDC
__global__ void __launch_bounds__(256) row_sqnorm_kernel(const double* __restrict__ x, int n, int D, double* __restrict__ out) {
  const int warp = (blockIdx.x * 256 + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  double s = 0.0;
  for (int k = lane; k < D; k += 32) { const double v = x[(long long)warp * D + k]; s = fma(v, v, s); }
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xFFFFFFFFu, s, o);
  if (lane == 0) out[warp] = s;
}

__device__ __forceinline__ void insert_sorted(double (&lst)[kMaxK1], int k1, double d) {
  if (d >= lst[k1 - 1]) return;
  lst[k1 - 1] = d;
#pragma unroll
  for (int i = kMaxK1 - 1; i > 0; --i)
    if (i < k1 && lst[i] < lst[i - 1]) { const double t = lst[i]; lst[i] = lst[i - 1]; lst[i - 1] = t; }
}

// radii[i] = (k1)-th smallest euclidean distance from x_i to the rows of x (self included): one CTA owns 64 rows and walks
// every column tile; each thread keeps the k1 smallest distances it has seen for each of its 4 rows, and the 16 threads that
// share a row (one half-warp) merge their lists by k1 rounds of "pop the global minimum".
__global__ void __launch_bounds__(256) prdc_radii_kernel(const double* __restrict__ x, const double* __restrict__ xn, int n, int D,
                                                          int k1, double* __restrict__ radii) {
  __shared__ double As[kMK][kMT + 1], Bs[kMK][kMT + 1];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int row0 = blockIdx.x * kMT;
  double lst[4][kMaxK1];
#pragma unroll
  for (int a = 0; a < 4; ++a)
#pragma unroll
    for (int i = 0; i < kMaxK1; ++i) lst[a][i] = 1e300;
  double rn[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) rn[a] = row0 + ty * 4 + a < n ? xn[row0 + ty * 4 + a] : 0.0;
  for (int col0 = 0; col0 < n; col0 += kMT) {
    double acc[4][4];
    tile_dot(x, D, n, row0, x, D, n, col0, D, acc, As, Bs);
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = col0 + tx * 4 + b;
      if (c >= n) continue;
      const double cn = xn[c];
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        const double d2 = rn[a] + cn - 2.0 * acc[a][b];
        insert_sorted(lst[a], k1, (row0 + ty * 4 + a == c) ? 0.0 : sqrt(d2 > 0.0 ? d2 : 0.0));   // sklearn zeroes the diagonal of X-vs-X
      }
    }
  }
  // merge across the 16 lanes of the half-warp that share these rows
  const unsigned lane = threadIdx.x & 31, half_base = lane & 16u;
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    int head = 0;
    double kth = 1e300;
    for (int round = 0; round < k1; ++round) {
      const double mine = head < k1 ? lst[a][0] : 1e300;      // lists are consumed by shifting (k1 <= 8: cheap)
      double m = mine;
      for (int o = 8; o > 0; o >>= 1) m = fmin(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
      const unsigned owners = __ballot_sync(0xFFFFFFFFu, mine == m) & (0xFFFFu << half_base);
      const unsigned owner = __ffs(owners) - 1;
      if (lane == owner) {
#pragma unroll
        for (int i = 0; i < kMaxK1 - 1; ++i) lst[a][i] = lst[a][i + 1];
        lst[a][kMaxK1 - 1] = 1e300;
        ++head;
      }
      kth = m;
    }
    const int r = row0 + ty * 4 + a;
    if (tx == 0 && r < n) radii[r] = kth;
  }
}

// Real-to-fake tile reductions: CTA = 64 real rows x all fake columns.
//   col_count[j] += #{i : d(i,j) < r_real[i]}     (density; precision = count > 0)
//   row_any[i]    = any_j d(i,j) < r_fake[j]       (recall)
//   row_cov[i]    = min_j d(i,j) < r_real[i]       (coverage)
__global__ void __launch_bounds__(256) prdc_cross_kernel(const double* __restrict__ real, const double* __restrict__ rn_all,
                                                          const double* __restrict__ fake, const double* __restrict__ fn_all,
                                                          const double* __restrict__ r_real, const double* __restrict__ r_fake, int nr,
                                                          int nf, int D, int* __restrict__ col_count, unsigned char* __restrict__ row_any,
                                                          unsigned char* __restrict__ row_cov) {
  __shared__ double As[kMK][kMT + 1], Bs[kMK][kMT + 1];
  __shared__ int ccount[kMT];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int row0 = blockIdx.x * kMT;
  double rn[4], rr[4], rmin[4];
  bool rany[4];
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    const int r = row0 + ty * 4 + a;
    rn[a] = r < nr ? rn_all[r] : 0.0;
    rr[a] = r < nr ? r_real[r] : -1.0;
    rmin[a] = 1e300;
    rany[a] = false;
  }
  for (int col0 = 0; col0 < nf; col0 += kMT) {
    double acc[4][4];
    tile_dot(real, D, nr, row0, fake, D, nf, col0, D, acc, As, Bs);
    if (threadIdx.x < kMT) ccount[threadIdx.x] = 0;
    __syncthreads();
#pragma unroll
    for (int b = 0; b < 4; ++b) {
      const int c = col0 + tx * 4 + b;
      if (c >= nf) continue;
      const double cn = fn_all[c], rf = r_fake[c];
      int cnt = 0;
#pragma unroll
      for (int a = 0; a < 4; ++a) {
        if (row0 + ty * 4 + a >= nr) continue;
        const double d2 = rn[a] + cn - 2.0 * acc[a][b];
        const double d = sqrt(d2 > 0.0 ? d2 : 0.0);
        cnt += d < rr[a] ? 1 : 0;
        rany[a] = rany[a] || d < rf;
        rmin[a] = fmin(rmin[a], d);
      }
      if (cnt) atomicAdd(&ccount[tx * 4 + b], cnt);
    }
    __syncthreads();
    if (threadIdx.x < kMT && col0 + threadIdx.x < nf && ccount[threadIdx.x]) atomicAdd(col_count + col0 + threadIdx.x, ccount[threadIdx.x]);
  }
#pragma unroll
  for (int a = 0; a < 4; ++a) {
    double m = rmin[a];
    unsigned any = rany[a] ? 1u : 0u;
    for (int o = 8; o > 0; o >>= 1) {
      m = fmin(m, __shfl_xor_sync(0xFFFFFFFFu, m, o));
      any |= __shfl_xor_sync(0xFFFFFFFFu, any, o);
    }
    const int r = row0 + ty * 4 + a;
    if (tx == 0 && r < nr) {
      row_any[r] = (unsigned char)any;
      row_cov[r] = m < rr[a] ? 1 : 0;
    }
  }
}

}  // namespace sgb

using namespace sgb;

extern "C" int sgb_feat_moments_accumulate(const float* feats, int32_t n, int32_t D, double* sum, double* outer, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(feats && sum && outer && n > 0 && D > 0);
  const int nblk = (D + kMT - 1) / kMT;
  moments_kernel<<<nblk * (nblk + 1) / 2, 256, 0, stream>>>(feats, n, D, sum, outer, nblk);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_feat_moments_finalize(const double* sum, const double* outer, double n, int32_t D, double* mu, double* sigma,
                                         sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(sum && outer && mu && sigma && n > 1.0 && D > 0);
  long long blocks = ((long long)D * D + 255) / 256;
  if (blocks > 8LL * sm_count()) blocks = 8LL * sm_count();
  moments_finalize_kernel<<<(int)blocks, 256, 0, stream>>>(sum, outer, n, D, mu, sigma);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_prdc_radii(const double* x, int32_t n, int32_t D, int32_t nearest_k, double* sqnorm_ws, double* radii,
                              sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(x && sqnorm_ws && radii && n > 0 && D > 0 && nearest_k >= 1 && nearest_k + 1 <= kMaxK1 && nearest_k + 1 <= n);
  row_sqnorm_kernel<<<(n * 32 + 255) / 256, 256, 0, stream>>>(x, n, D, sqnorm_ws);
  SGB_LAUNCH_CHECK();
  prdc_radii_kernel<<<(n + kMT - 1) / kMT, 256, 0, stream>>>(x, sqnorm_ws, n, D, nearest_k + 1, radii);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}

extern "C" int sgb_prdc_cross(const double* real, const double* real_sqnorm, const double* fake, const double* fake_sqnorm,
                              const double* radii_real, const double* radii_fake, int32_t n_real, int32_t n_fake, int32_t D,
                              int32_t* col_count, uint8_t* row_any, uint8_t* row_cov, sgb_stream_t stream_) {
  cudaStream_t stream = (cudaStream_t)stream_;
  SGB_REQUIRE(real && real_sqnorm && fake && fake_sqnorm && radii_real && radii_fake && col_count && row_any && row_cov);
  SGB_REQUIRE(n_real > 0 && n_fake > 0 && D > 0);
  SGB_CUDA(cudaMemsetAsync(col_count, 0, sizeof(int32_t) * (size_t)n_fake, stream));
  prdc_cross_kernel<<<(n_real + kMT - 1) / kMT, 256, 0, stream>>>(real, real_sqnorm, fake, fake_sqnorm, radii_real, radii_fake, n_real,
                                                                  n_fake, D, col_count, row_any, row_cov);
  SGB_LAUNCH_CHECK();
  return SGB_OK;
}
