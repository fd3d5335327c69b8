// Stand-alone bring-up harness for the wgmma conv engine: runs on the GPU without Python.
// Compares sgb_conv_fprop / sgb_conv_wgrad with a scalar host loop on small seeded cases, prints layout
// probes (delta inputs) so a descriptor mistake can be read off the log, and times a few BigGAN-Deep
// shaped layers.  Bring-up tooling only; the judged parity tests live in tests/ and go through Python.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#include "../../include/sgb200.h"

typedef __nv_bfloat16 bf16;

static uint32_t rng_state = 12345u;
static float frand() {
  rng_state = rng_state * 1664525u + 1013904223u;
  return ((rng_state >> 8) & 0xFFFF) / 65536.0f - 0.5f;
}
static float bfr(float x) { return __bfloat162float(__float2bfloat16_rn(x)); }

#define CK(x)                                                                     \
  do {                                                                            \
    cudaError_t e = (x);                                                          \
    if (e != cudaSuccess) {                                                       \
      printf("CUDA FAIL %s: %s (line %d)\n", #x, cudaGetErrorString(e), __LINE__); \
      exit(2);                                                                    \
    }                                                                             \
  } while (0)

struct Case {
  const char* name;
  int B, H, W, Cin, Cout, KH, KW, ph, pw;
  int bias, relu, res, res_up2, mask, fp32out;
};

static int run_fprop_case(const Case& c, bool verbose) {
  const int taps = c.KH * c.KW;
  const size_t nx = (size_t)c.B * c.H * c.W * c.Cin, nw = (size_t)c.Cout * taps * c.Cin, ny = (size_t)c.B * c.H * c.W * c.Cout;
  const int rH = c.res_up2 ? c.H / 2 : c.H, rW = c.res_up2 ? c.W / 2 : c.W;
  const size_t nr = (size_t)c.B * rH * rW * c.Cout;
  std::vector<float> x(nx), w(nw), bias(c.Cout), res(nr), msk(ny), ref(ny);
  for (auto& v : x) v = bfr(frand());
  for (auto& v : w) v = bfr(frand() * 0.25f);
  for (auto& v : bias) v = frand();
  for (auto& v : res) v = bfr(frand());
  for (auto& v : msk) v = bfr(frand());
  for (int b = 0; b < c.B; ++b)
    for (int h = 0; h < c.H; ++h)
      for (int ww = 0; ww < c.W; ++ww)
        for (int co = 0; co < c.Cout; ++co) {
          double acc = 0;
          for (int kh = 0; kh < c.KH; ++kh)
            for (int kw = 0; kw < c.KW; ++kw) {
              const int ih = h + kh - c.ph, iw = ww + kw - c.pw;
              if (ih < 0 || ih >= c.H || iw < 0 || iw >= c.W) continue;
              const float* xp = &x[(((size_t)b * c.H + ih) * c.W + iw) * c.Cin];
              const float* wp = &w[((size_t)co * taps + kh * c.KW + kw) * c.Cin];
              for (int ci = 0; ci < c.Cin; ++ci) acc += (double)xp[ci] * wp[ci];
            }
          float f = (float)acc * 0.5f;
          if (c.bias) f += bias[co];
          const size_t o = (((size_t)b * c.H + h) * c.W + ww) * c.Cout + co;
          if (c.res) f += res[(((size_t)b * rH + (c.res_up2 ? h / 2 : h)) * rW + (c.res_up2 ? ww / 2 : ww)) * c.Cout + co];
          if (c.relu) f = fmaxf(f, 0.f);
          if (c.mask) f = msk[o] > 0 ? f : 0.f;
          ref[o] = f;
        }
  std::vector<bf16> xb(nx), wb(nw), rb(nr), mb(ny);
  for (size_t i = 0; i < nx; ++i) xb[i] = __float2bfloat16_rn(x[i]);
  for (size_t i = 0; i < nw; ++i) wb[i] = __float2bfloat16_rn(w[i]);
  for (size_t i = 0; i < nr; ++i) rb[i] = __float2bfloat16_rn(res[i]);
  for (size_t i = 0; i < ny; ++i) mb[i] = __float2bfloat16_rn(msk[i]);
  bf16 *dx, *dw, *dr, *dm;
  void* dy;
  float* dbias;
  CK(cudaMalloc(&dx, nx * 2)); CK(cudaMalloc(&dw, nw * 2)); CK(cudaMalloc(&dr, nr * 2)); CK(cudaMalloc(&dm, ny * 2));
  CK(cudaMalloc(&dy, ny * 4)); CK(cudaMalloc(&dbias, c.Cout * 4));
  CK(cudaMemcpy(dx, xb.data(), nx * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dw, wb.data(), nw * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dr, rb.data(), nr * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dm, mb.data(), ny * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dbias, bias.data(), c.Cout * 4, cudaMemcpyHostToDevice));
  CK(cudaMemset(dy, 0xFF, ny * 4));
  sgb_conv_desc d;
  memset(&d, 0, sizeof(d));
  d.B = c.B; d.H = c.H; d.W = c.W; d.Cin = c.Cin; d.Cout = c.Cout; d.KH = c.KH; d.KW = c.KW; d.pad_h = c.ph; d.pad_w = c.pw;
  d.x = dx; d.x_cstride = c.Cin; d.w = dw; d.alpha = 0.5f; d.bias = c.bias ? dbias : nullptr;
  d.residual = c.res ? dr : nullptr; d.res_cstride = c.Cout; d.res_up2 = c.res_up2;
  d.mask = c.mask ? dm : nullptr; d.mask_cstride = c.Cout; d.relu = c.relu;
  d.y = dy; d.y_cstride = c.Cout; d.y_fp32 = c.fp32out;
  int rc = sgb_conv_fprop(&d, 0);
  cudaError_t se = cudaDeviceSynchronize();
  if (rc || se != cudaSuccess) {
    printf("[fprop %-28s] LAUNCH FAIL rc=%d cuda=%s\n", c.name, rc, cudaGetErrorString(se));
    return 1;
  }
  std::vector<float> got(ny);
  if (c.fp32out) {
    CK(cudaMemcpy(got.data(), dy, ny * 4, cudaMemcpyDeviceToHost));
  } else {
    std::vector<bf16> gb(ny);
    CK(cudaMemcpy(gb.data(), dy, ny * 2, cudaMemcpyDeviceToHost));
    for (size_t i = 0; i < ny; ++i) got[i] = __bfloat162float(gb[i]);
  }
  double maxerr = 0, maxref = 0;
  size_t bad = 0, first_bad = (size_t)-1;
  for (size_t i = 0; i < ny; ++i) {
    const double e = fabs((double)got[i] - ref[i]);
    const double tol = (c.fp32out ? 2e-3 : 1.5e-2) * (1.0 + fabs(ref[i]));
    if (!(e <= tol)) { if (!bad) first_bad = i; ++bad; }
    if (e > maxerr || e != e) maxerr = e;
    if (fabs(ref[i]) > maxref) maxref = fabs(ref[i]);
  }
  printf("[fprop %-28s] %s maxerr=%.4g maxref=%.3g bad=%zu/%zu\n", c.name, bad ? "FAIL" : "PASS", maxerr, maxref, bad, ny);
  if (bad && verbose) {
    for (size_t i = first_bad, k = 0; i < ny && k < 12; ++i) {
      const double e = fabs((double)got[i] - ref[i]);
      if (e > 1.5e-2 * (1 + fabs(ref[i])) || e != e) {
        const size_t pix = i / c.Cout;
        printf("    idx=%zu (b=%zu h=%zu w=%zu co=%zu) got=%g ref=%g\n", i, pix / ((size_t)c.H * c.W), (pix / c.W) % c.H, pix % c.W,
               i % c.Cout, got[i], ref[i]);
        ++k;
      }
    }
  }
  cudaFree(dx); cudaFree(dw); cudaFree(dr); cudaFree(dm); cudaFree(dy); cudaFree(dbias);
  return bad ? 1 : 0;
}

static int run_wgrad_case(const Case& c, bool verbose) {
  const int taps = c.KH * c.KW;
  const size_t nx = (size_t)c.B * c.H * c.W * c.Cin, nw = (size_t)c.Cout * taps * c.Cin, ny = (size_t)c.B * c.H * c.W * c.Cout;
  std::vector<float> x(nx), dy(ny);
  std::vector<double> ref(nw, 0.0);
  for (auto& v : x) v = bfr(frand());
  for (auto& v : dy) v = bfr(frand());
  for (int b = 0; b < c.B; ++b)
    for (int h = 0; h < c.H; ++h)
      for (int ww = 0; ww < c.W; ++ww)
        for (int kh = 0; kh < c.KH; ++kh)
          for (int kw = 0; kw < c.KW; ++kw) {
            const int ih = h + kh - c.ph, iw = ww + kw - c.pw;
            if (ih < 0 || ih >= c.H || iw < 0 || iw >= c.W) continue;
            const float* xp = &x[(((size_t)b * c.H + ih) * c.W + iw) * c.Cin];
            const float* gp = &dy[(((size_t)b * c.H + h) * c.W + ww) * c.Cout];
            for (int co = 0; co < c.Cout; ++co) {
              double* rp = &ref[((size_t)co * taps + kh * c.KW + kw) * c.Cin];
              const double g = gp[co];
              for (int ci = 0; ci < c.Cin; ++ci) rp[ci] += g * xp[ci];
            }
          }
  std::vector<bf16> xb(nx), yb(ny);
  for (size_t i = 0; i < nx; ++i) xb[i] = __float2bfloat16_rn(x[i]);
  for (size_t i = 0; i < ny; ++i) yb[i] = __float2bfloat16_rn(dy[i]);
  bf16 *dx, *ddy;
  float* ddw;
  CK(cudaMalloc(&dx, nx * 2)); CK(cudaMalloc(&ddy, ny * 2)); CK(cudaMalloc(&ddw, nw * 4));
  CK(cudaMemcpy(dx, xb.data(), nx * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ddy, yb.data(), ny * 2, cudaMemcpyHostToDevice));
  sgb_wgrad_desc d;
  memset(&d, 0, sizeof(d));
  d.B = c.B; d.H = c.H; d.W = c.W; d.Cin = c.Cin; d.Cout = c.Cout; d.KH = c.KH; d.KW = c.KW; d.pad_h = c.ph; d.pad_w = c.pw;
  d.x = dx; d.x_cstride = c.Cin; d.dy = ddy; d.dy_cstride = c.Cout; d.dw = ddw; d.accumulate = 0;
  float* ddb = nullptr;
  if (sgb_conv_wgrad_fuses_dbias(&d)) {
    CK(cudaMalloc(&ddb, c.Cout * 4));
    d.dbias = ddb;
  }
  int rc = sgb_conv_wgrad(&d, 0);
  cudaError_t se = cudaDeviceSynchronize();
  if (rc || se != cudaSuccess) {
    printf("[wgrad %-28s] LAUNCH FAIL rc=%d cuda=%s\n", c.name, rc, cudaGetErrorString(se));
    return 1;
  }
  size_t bad_b = 0;
  if (ddb) {                                     // fused bias gradient: sum of dy over all pixels
    std::vector<float> gb(c.Cout);
    CK(cudaMemcpy(gb.data(), ddb, c.Cout * 4, cudaMemcpyDeviceToHost));
    for (int co = 0; co < c.Cout; ++co) {
      double r = 0;
      for (size_t px = 0; px < (size_t)c.B * c.H * c.W; ++px) r += dy[px * c.Cout + co];
      if (!(fabs(gb[co] - r) <= 2e-3 * (1.0 + fabs(r)))) { if (!bad_b) printf("    dbias[%d] got=%g ref=%g\n", co, gb[co], r); ++bad_b; }
    }
    printf("[wgrad %-28s] fused dbias %s\n", c.name, bad_b ? "FAIL" : "PASS");
    cudaFree(ddb);
  }
  std::vector<float> got(nw);
  CK(cudaMemcpy(got.data(), ddw, nw * 4, cudaMemcpyDeviceToHost));
  double maxerr = 0, maxref = 0;
  size_t bad = 0, first_bad = 0;
  for (size_t i = 0; i < nw; ++i) {
    const double e = fabs((double)got[i] - ref[i]);
    if (!(e <= 2e-3 * (1.0 + fabs(ref[i])))) { if (!bad) first_bad = i; ++bad; }
    if (e > maxerr || e != e) maxerr = e;
    if (fabs(ref[i]) > maxref) maxref = fabs(ref[i]);
  }
  printf("[wgrad %-28s] %s maxerr=%.4g maxref=%.3g bad=%zu/%zu\n", c.name, bad ? "FAIL" : "PASS", maxerr, maxref, bad, nw);
  if (bad && verbose) {
    for (size_t i = first_bad, k = 0; i < nw && k < 12; ++i) {
      const double e = fabs((double)got[i] - ref[i]);
      if (e > 2e-3 * (1 + fabs(ref[i])) || e != e) {
        printf("    idx=%zu (co=%zu tap=%zu ci=%zu) got=%g ref=%g\n", i, i / ((size_t)taps * c.Cin), (i / c.Cin) % taps, i % c.Cin, got[i],
               ref[i]);
        ++k;
      }
    }
  }
  cudaFree(dx); cudaFree(ddy); cudaFree(ddw);
  return (bad || bad_b) ? 1 : 0;
}

// Layout probes: delta inputs, identity weights; prints where the energy lands.
static void probe_fprop() {
  const int B = 1, H = 16, W = 16, C = 128;
  const size_t n = (size_t)B * H * W * C;
  std::vector<bf16> x(n, __float2bfloat16_rn(0.f)), w((size_t)C * C, __float2bfloat16_rn(0.f));
  const int probes[4][2] = {{0, 0}, {5, 3}, {37, 70}, {200, 127}};  // (pixel, channel)
  for (auto& pr : probes) x[(size_t)pr[0] * C + pr[1]] = __float2bfloat16_rn(1.0f + pr[1] * 0.0078125f);
  for (int i = 0; i < C; ++i) w[(size_t)i * C + i] = __float2bfloat16_rn(1.f);
  bf16 *dx, *dw; float* dy;
  CK(cudaMalloc(&dx, n * 2)); CK(cudaMalloc(&dw, (size_t)C * C * 2)); CK(cudaMalloc(&dy, n * 4));
  CK(cudaMemcpy(dx, x.data(), n * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(dw, w.data(), (size_t)C * C * 2, cudaMemcpyHostToDevice));
  CK(cudaMemset(dy, 0, n * 4));
  sgb_conv_desc d; memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.Cin = C; d.Cout = C; d.KH = 1; d.KW = 1; d.x = dx; d.x_cstride = C; d.w = dw; d.alpha = 1.f;
  d.y = dy; d.y_cstride = C; d.y_fp32 = 1;
  int rc = sgb_conv_fprop(&d, 0);
  cudaError_t se = cudaDeviceSynchronize();
  printf("[probe fprop identity 1x1 C=128] rc=%d cuda=%s; expected nonzeros at (pix,ch): (0,0) (5,3) (37,70) (200,127)\n", rc, cudaGetErrorString(se));
  if (rc || se != cudaSuccess) return;
  std::vector<float> y(n);
  CK(cudaMemcpy(y.data(), dy, n * 4, cudaMemcpyDeviceToHost));
  int cnt = 0;
  for (size_t i = 0; i < n && cnt < 24; ++i)
    if (y[i] != 0.f) { printf("    y[pix=%zu][ch=%zu] = %g\n", i / C, i % C, y[i]); ++cnt; }
  if (!cnt) printf("    (all zero)\n");
  cudaFree(dx); cudaFree(dw); cudaFree(dy);
}

static void probe_wgrad() {
  const int B = 1, H = 16, W = 16, Ci = 128, Co = 128;
  const size_t nx = (size_t)B * H * W * Ci, ny = (size_t)B * H * W * Co, nw = (size_t)Co * Ci;
  std::vector<bf16> x(nx, __float2bfloat16_rn(0.f)), dy(ny, __float2bfloat16_rn(0.f));
  const int probes[4][3] = {{0, 0, 0}, {9, 3, 5}, {77, 70, 100}, {255, 127, 64}};  // (pixel, co, ci)
  for (auto& pr : probes) {
    dy[(size_t)pr[0] * Co + pr[1]] = __float2bfloat16_rn(1.f);
    x[(size_t)pr[0] * Ci + pr[2]] = __float2bfloat16_rn(1.0f + pr[2] * 0.0078125f);
  }
  bf16 *dx, *ddy; float* ddw;
  CK(cudaMalloc(&dx, nx * 2)); CK(cudaMalloc(&ddy, ny * 2)); CK(cudaMalloc(&ddw, nw * 4));
  CK(cudaMemcpy(dx, x.data(), nx * 2, cudaMemcpyHostToDevice));
  CK(cudaMemcpy(ddy, dy.data(), ny * 2, cudaMemcpyHostToDevice));
  sgb_wgrad_desc d; memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.Cin = Ci; d.Cout = Co; d.KH = 1; d.KW = 1; d.x = dx; d.x_cstride = Ci; d.dy = ddy; d.dy_cstride = Co; d.dw = ddw;
  int rc = sgb_conv_wgrad(&d, 0);
  cudaError_t se = cudaDeviceSynchronize();
  printf("[probe wgrad delta 1x1 128x128] rc=%d cuda=%s; expected nonzeros at (co,ci): (0,0) (3,5) (70,100) (127,64)\n", rc, cudaGetErrorString(se));
  if (rc || se != cudaSuccess) return;
  std::vector<float> g(nw);
  CK(cudaMemcpy(g.data(), ddw, nw * 4, cudaMemcpyDeviceToHost));
  int cnt = 0;
  for (size_t i = 0; i < nw && cnt < 24; ++i)
    if (g[i] != 0.f) { printf("    dw[co=%zu][ci=%zu] = %g\n", i / Ci, i % Ci, g[i]); ++cnt; }
  if (!cnt) printf("    (all zero)\n");
  cudaFree(dx); cudaFree(ddy); cudaFree(ddw);
}

static void time_fprop(const char* name, int B, int H, int W, int Cin, int Cout, int K) {
  const int taps = K * K;
  const size_t nx = (size_t)B * H * W * Cin, nw = (size_t)Cout * taps * Cin, ny = (size_t)B * H * W * Cout;
  bf16 *dx, *dw, *dy;
  CK(cudaMalloc(&dx, nx * 2)); CK(cudaMalloc(&dw, nw * 2)); CK(cudaMalloc(&dy, ny * 2));
  CK(cudaMemset(dx, 0x3c, nx * 2)); CK(cudaMemset(dw, 0x3c, nw * 2));
  sgb_conv_desc d; memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.KH = K; d.KW = K; d.pad_h = K / 2; d.pad_w = K / 2;
  d.x = dx; d.x_cstride = Cin; d.w = dw; d.alpha = 1.f; d.y = dy; d.y_cstride = Cout;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) sgb_conv_fprop(&d, 0);
  cudaEventRecord(e0);
  const int iters = 10;
  for (int i = 0; i < iters; ++i) sgb_conv_fprop(&d, 0);
  cudaEventRecord(e1);
  cudaError_t se = cudaEventSynchronize(e1);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1); ms /= iters;
  const double fl = 2.0 * B * H * W * (double)Cout * Cin * taps;
  printf("[time fprop %-30s] %s %.3f ms  %.1f TFLOP/s  (in %.1f MB out %.1f MB)\n", name, cudaGetErrorString(se), ms, fl / ms * 1e-9,
         nx * 2e-6, ny * 2e-6);
  cudaFree(dx); cudaFree(dw); cudaFree(dy);
}

static void time_wgrad(const char* name, int B, int H, int W, int Cin, int Cout, int K) {
  const int taps = K * K;
  const size_t nx = (size_t)B * H * W * Cin, nw = (size_t)Cout * taps * Cin, ny = (size_t)B * H * W * Cout;
  bf16 *dx, *dy; float* dw;
  CK(cudaMalloc(&dx, nx * 2)); CK(cudaMalloc(&dw, nw * 4)); CK(cudaMalloc(&dy, ny * 2));
  CK(cudaMemset(dx, 0x3c, nx * 2)); CK(cudaMemset(dy, 0x3c, ny * 2));
  sgb_wgrad_desc d; memset(&d, 0, sizeof(d));
  d.B = B; d.H = H; d.W = W; d.Cin = Cin; d.Cout = Cout; d.KH = K; d.KW = K; d.pad_h = K / 2; d.pad_w = K / 2;
  d.x = dx; d.x_cstride = Cin; d.dy = dy; d.dy_cstride = Cout; d.dw = dw;
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int i = 0; i < 3; ++i) sgb_conv_wgrad(&d, 0);
  cudaEventRecord(e0);
  const int iters = 10;
  for (int i = 0; i < iters; ++i) sgb_conv_wgrad(&d, 0);
  cudaEventRecord(e1);
  cudaError_t se = cudaEventSynchronize(e1);
  float ms = 0; cudaEventElapsedTime(&ms, e0, e1); ms /= iters;
  const double fl = 2.0 * B * H * W * (double)Cout * Cin * taps;
  printf("[time wgrad %-30s] %s %.3f ms  %.1f TFLOP/s\n", name, cudaGetErrorString(se), ms, fl / ms * 1e-9);
  cudaFree(dx); cudaFree(dw); cudaFree(dy);
}

int main(int argc, char** argv) {
  // modes (each run in its own process by the gpurun command so a trap in one does not hide the others):
  //   probe_f | probe_w | fprop | wgrad | time | all
  const char* mode = argc > 1 ? argv[1] : "all";
  auto on = [&](const char* m) { return strcmp(mode, m) == 0 || strcmp(mode, "all") == 0; };
  printf("sgb200 selftest[%s]: abi=%d device_check=%d\n", mode, sgb_abi_version(), sgb_device_check());
  int fails = 0;
  if (on("probe_f")) probe_fprop();
  if (on("probe_w")) probe_wgrad();
  const Case cases[] = {
      //  name                         B  H   W   Cin  Cout KH KW ph pw bias relu res up2 mask fp32
      {"1x1 c64->64 16x16",            2, 16, 16, 64,  64,  1, 1, 0, 0, 0, 0, 0, 0, 0, 1},
      {"1x1 c128->128 16x16",          2, 16, 16, 128, 128, 1, 1, 0, 0, 0, 0, 0, 0, 0, 1},
      {"1x1 c256->64 8x8 bias",        4, 8,  8,  256, 64,  1, 1, 0, 0, 1, 0, 0, 0, 0, 0},
      {"3x3 c64->64 8x8",              2, 8,  8,  64,  64,  3, 3, 1, 1, 0, 0, 0, 0, 0, 1},
      {"3x3 c128->256 32x32 b/r/res",  2, 32, 32, 128, 256, 3, 3, 1, 1, 1, 1, 1, 0, 0, 0},
      {"3x3 c64->3 16x16 bias",        2, 16, 16, 64,  3,   3, 3, 1, 1, 1, 0, 0, 0, 0, 1},
      {"3x3 c8->64 16x16 (Cin pad)",   2, 16, 16, 8,   64,  3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"linear 256->512 B=256",        256, 1, 1, 256, 512, 1, 1, 0, 0, 1, 0, 0, 0, 0, 1},
      {"3x3 4x4 nb=8 ragged B=12",     12, 4, 4,  64,  128, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"1x1 res_up2+mask 16x16",       2, 16, 16, 64,  64,  1, 1, 0, 0, 1, 1, 1, 1, 1, 0},
      {"1x7 c64->96 17x17 ragged",     2, 17, 17, 64,  96,  1, 7, 0, 3, 1, 1, 0, 0, 0, 0},
      {"3x3 c192->320 64x64",          1, 64, 64, 192, 320, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"3x3 c64->64 256x256 (tw=128)", 1, 256, 256, 64, 64, 3, 3, 1, 1, 0, 0, 0, 0, 0, 0},
      {"rows c64->64 128x128 b/r/res",  2, 128, 128, 64, 64, 3, 3, 1, 1, 1, 1, 1, 0, 0, 0},
      {"rows c128->128 128x128 mask",   1, 128, 128, 128, 128, 3, 3, 1, 1, 1, 0, 0, 0, 1, 0},
      {"rows c64->128 128x128 up2res",  1, 128, 128, 64, 128, 3, 3, 1, 1, 1, 0, 1, 1, 0, 0},
      {"rows c128->64 256x256 fp32",    1, 256, 256, 128, 64, 3, 3, 1, 1, 0, 0, 0, 0, 0, 1},
      {"rows c64->192 128x128",         1, 128, 128, 64, 192, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"rows c64->16 128x128",          3, 128, 128, 64, 16, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"rows c128->8 128x128",          2, 128, 128, 128, 8, 3, 3, 1, 1, 1, 0, 0, 0, 0, 0},
      {"aux 1x1 c64->256 32x32 res",    2, 32, 32, 64, 256, 1, 1, 0, 0, 1, 0, 1, 0, 0, 0},
      {"aux 1x1 c64->128 32x32 up2res", 2, 32, 32, 64, 128, 1, 1, 0, 0, 1, 0, 1, 1, 0, 0},
      {"aux 1x1 c128->64 16x16 mask",   3, 16, 16, 128, 64, 1, 1, 0, 0, 0, 0, 0, 0, 1, 0},
      {"aux 3x3 c64->64 16x16 res+relu", 2, 16, 16, 64, 64, 3, 3, 1, 1, 1, 1, 1, 0, 0, 0},
      {"aux 1x1 c64->256 4x4 up2 B=12", 12, 4, 4, 64, 256, 1, 1, 0, 0, 1, 0, 1, 1, 0, 0},
      {"aux 1x1 c64->192 8x8 res",      5, 8, 8, 64, 192, 1, 1, 0, 0, 1, 0, 1, 0, 0, 0},
      {"aux 1x1 c64->128 256x128 up2",  1, 256, 128, 64, 128, 1, 1, 0, 0, 0, 0, 1, 1, 0, 0},
      {"aux 1x1 c32->64 64x64 mask",    2, 64, 64, 32, 64, 1, 1, 0, 0, 1, 0, 0, 0, 1, 0},
  };
  if (on("fprop"))
    for (const auto& c : cases) fails += run_fprop_case(c, true);
  const Case wcases[] = {
      {"1x1 c64->64 16x16",            2, 16, 16, 64,  64,  1, 1, 0, 0},
      {"1x1 c128->128 16x16",          2, 16, 16, 128, 128, 1, 1, 0, 0},
      {"1x1 c256->64 8x8",             4, 8,  8,  256, 64,  1, 1, 0, 0},
      {"3x3 c64->64 8x8",              2, 8,  8,  64,  64,  3, 3, 1, 1},
      {"3x3 c128->256 32x32",          2, 32, 32, 128, 256, 3, 3, 1, 1},
      {"3x3 c64->8 16x16",             2, 16, 16, 64,  8,   3, 3, 1, 1},
      {"3x3 c8->64 16x16",             2, 16, 16, 8,   64,  3, 3, 1, 1},
      {"linear 256->512 B=256",        256, 1, 1, 256, 512, 1, 1, 0, 0},
      {"3x3 4x4 nb=8 ragged B=12",     12, 4, 4,  64,  128, 3, 3, 1, 1},
      {"1x7 c64->96 17x17 ragged",     2, 17, 17, 64,  96,  1, 7, 0, 3},
      {"3x3 c192->320 64x64",          1, 64, 64, 192, 320, 3, 3, 1, 1},
      {"w3 c64->64 128x128 B=2",       2, 128, 128, 64, 64, 3, 3, 1, 1},
      {"w3 c64->64 256x8 B=3",         3, 8, 256, 64, 64, 3, 3, 1, 1},
      {"w3 c64->32 128x128 B=1",       1, 128, 128, 64, 32, 3, 3, 1, 1},
      {"w3 c32->64 128x128 B=1",       1, 128, 128, 32, 64, 3, 3, 1, 1},
      {"w3 c64->64 128x128 B=5",       5, 128, 128, 64, 64, 3, 3, 1, 1},
      {"w3 c128->8 128x128 B=2",       2, 128, 128, 128, 8, 3, 3, 1, 1},
  };
  if (on("wgrad"))
    for (const auto& c : wcases) fails += run_wgrad_case(c, true);
  printf("selftest[%s]: %d failing case(s)\n", mode, fails);
  if (strcmp(mode, "one") == 0 && argc >= 8) {     // ./sgb_selftest one B H W Cin Cout K : time a single fprop shape (ncu target)
    time_fprop("one", atoi(argv[2]), atoi(argv[3]), atoi(argv[4]), atoi(argv[5]), atoi(argv[6]), atoi(argv[7]));
    return 0;
  }
  if (strcmp(mode, "time") == 0) {
    time_fprop("3x3 64->64 256^2 B=32", 32, 256, 256, 64, 64, 3);
    time_fprop("3x3 128->128 128^2 B=32", 32, 128, 128, 128, 128, 3);
    time_fprop("3x3 256->256 64^2 B=64", 64, 64, 64, 256, 256, 3);
    time_fprop("3x3 512->512 32^2 B=64", 64, 32, 32, 512, 512, 3);
    time_fprop("1x1 2048->512 8^2 B=256", 256, 8, 8, 2048, 512, 1);
    time_fprop("1x1 512->2048 8^2 B=256", 256, 8, 8, 512, 2048, 1);
    time_fprop("1x1 256->64 256^2 B=32", 32, 256, 256, 256, 64, 1);
    time_fprop("1x1 4096->4096 M=16384", 16384, 1, 1, 4096, 4096, 1);
    time_fprop("1x1 64->256 128^2 B=64", 64, 128, 128, 64, 256, 1);
    time_fprop("1x1 64->128 256^2 B=32", 32, 256, 256, 64, 128, 1);
    time_fprop("1x1 128->512 64^2 B=64", 64, 64, 64, 128, 512, 1);
    time_fprop("1x1 256->1024 32^2 B=64", 64, 32, 32, 256, 1024, 1);
    time_fprop("1x1 256->512 64^2 B=64", 64, 64, 64, 256, 512, 1);
    time_fprop("1x1 512->2048 16^2 B=64", 64, 16, 16, 512, 2048, 1);
    time_wgrad("3x3 64->64 256^2 B=32", 32, 256, 256, 64, 64, 3);
    time_wgrad("3x3 64->64 128^2 B=32", 32, 128, 128, 64, 64, 3);
    time_wgrad("3x3 256->256 64^2 B=64", 64, 64, 64, 256, 256, 3);
    time_wgrad("3x3 512->512 32^2 B=64", 64, 32, 32, 512, 512, 3);
    time_wgrad("1x1 2048->512 8^2 B=256", 256, 8, 8, 2048, 512, 1);
  }
  return fails ? 1 : 0;
}
