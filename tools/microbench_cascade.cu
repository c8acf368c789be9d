// Micro-benchmark: what does the H100 FP64 pipe deliver on the *actual* dependency
// structure of a 4-section monic biquad cascade (3 DFMA per section, 12 per sample, all
// operands distinct registers), as a function of resident warps per SM and of the
// schedule: plain (section after section, as the compiler sees the reference order)
// versus skewed (section k works on sample n-k: four independent chains per step)?
// No memory traffic: isolates the arithmetic pipe from the tile I/O.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench_cascade microbench_cascade.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

struct Coefs { double c1[4], na1[4], na2[4], G; };

template <bool SKEW, bool CVT>
__global__ void k_cascade(float* out, long long* cyc, int iters, Coefs cf_in, double x0) {
  Coefs cf = cf_in;
  // make the coefficients lane-dependent so that nothing is uniform / constant-bank
  const double eps = 1e-9 * (threadIdx.x + 1);
#pragma unroll
  for (int k = 0; k < 4; ++k) { cf.c1[k] += eps; cf.na1[k] -= eps; cf.na2[k] += eps; }
  double u[5][2];
#pragma unroll
  for (int k = 0; k < 5; ++k) { u[k][0] = 1e-3 * k; u[k][1] = 2e-3 * k; }
  double x = x0 + eps;
  float acc = 0.f;
  double dacc = 0.0;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      x = x * 0.999 + 1e-3;   // cheap input stand-in (adds 1 DFMA per sample, counted)
      if (!SKEW) {
        double in = x, in1 = u[0][0];
        u[0][0] = in;
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          const double y1 = u[k + 1][0], y2 = u[k + 1][1];
          double t = fma(cf.c1[k], in1, in);
          t = fma(cf.na2[k], y2, t);
          const double y = fma(cf.na1[k], y1, t);
          u[k + 1][1] = y1; u[k + 1][0] = y;
          in = y; in1 = y1;
        }
        if (CVT) acc += (float)(cf.G * in); else dacc += in;
      } else {
        // section k consumes u[k] history (= output of section k-1 up to the previous step)
        double y[4];
#pragma unroll
        for (int k = 3; k >= 0; --k) {
          const double in = (k == 0) ? x : u[k][0];
          const double in1 = (k == 0) ? u[0][0] : u[k][1];
          double t = fma(cf.c1[k], in1, in);
          t = fma(cf.na2[k], u[k + 1][1], t);
          y[k] = fma(cf.na1[k], u[k + 1][0], t);
        }
        u[0][0] = x;
#pragma unroll
        for (int k = 0; k < 4; ++k) { u[k + 1][1] = u[k + 1][0]; u[k + 1][0] = y[k]; }
        if (CVT) acc += (float)(cf.G * y[3]); else dacc += y[3];
      }
    }
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc + (float)dacc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}


struct UP { double c1[4], na1[4], na2[4], G; };
struct UParams { UP ch[64]; };
// INCVT: 0 = x already double in a register, 1 = F2F.F64.F32 per sample, 2 = integer widening per sample
template <int INCVT, bool OUTCVT>
__global__ void __launch_bounds__(32) k_uniform(const __grid_constant__ UParams P, float* out, long long* cyc, int iters, float x0) {
  const UP& cf = P.ch[blockIdx.x & 63];    // CTA-uniform -> uniform registers
  double u[5][2];
#pragma unroll
  for (int k = 0; k < 5; ++k) { u[k][0] = 1e-3 * k + threadIdx.x * 1e-6; u[k][1] = 2e-3 * k; }
  float xf = x0 + threadIdx.x * 1e-3f;
  double xd = xf;
  float acc = 0.f; double dacc = 0.0;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      double x;
      if (INCVT == 0) { xd = xd * 0.999 + 1e-3; x = xd; }
      else {
        xf = xf * 0.999f + 1e-3f;
        if (INCVT == 1) { asm volatile("cvt.f64.f32 %0, %1;" : "=d"(x) : "f"(xf)); }
        else {
          const unsigned b = __float_as_uint(xf);
          const unsigned e = b & 0x7f800000u;
          if (e != 0u && e != 0x7f800000u) {
            const unsigned hi = ((b & 0x7fffffffu) >> 3) + 0x38000000u | (b & 0x80000000u);
            x = __hiloint2double((int)hi, (int)(b << 29));
          } else x = (double)xf;
        }
      }
      double in = x, in1 = u[0][0];
      u[0][0] = in;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        const double y1 = u[k + 1][0], y2 = u[k + 1][1];
        double t = fma(cf.c1[k], in1, in);
        t = fma(cf.na2[k], y2, t);
        const double y = fma(cf.na1[k], y1, t);
        u[k + 1][1] = y1; u[k + 1][0] = y;
        in = y; in1 = y1;
      }
      if (OUTCVT) acc += (float)(cf.G * in); else dacc += in;
    }
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = acc + (float)dacc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  int nsm = p.multiProcessorCount;
  float* d_out; long long* d_cyc;
  CK(cudaMalloc(&d_out, sizeof(float) * nsm * 32 * 1024));
  CK(cudaMalloc(&d_cyc, sizeof(long long) * nsm * 64));
  Coefs cf;
  for (int k = 0; k < 4; ++k) { cf.c1[k] = -0.9 + 0.01 * k; cf.na1[k] = 1.2 - 0.02 * k; cf.na2[k] = -0.5 - 0.01 * k; }
  cf.G = 1e-3;
  const int iters = 2048;
  long long* h = (long long*)malloc(sizeof(long long) * nsm * 64);
  printf("%-10s %-6s %5s %5s %12s %10s\n", "schedule", "cvt", "warps", "ctas", "dfma/clk/SM", "cyc/sample");
#define RUN(SK, CV, threads, ctas_per_sm) do { \
    int grid = nsm * (ctas_per_sm); \
    k_cascade<SK, CV><<<grid, threads>>>(d_out, d_cyc, iters, cf, 0.5); CK(cudaDeviceSynchronize()); \
    k_cascade<SK, CV><<<grid, threads>>>(d_out, d_cyc, iters, cf, 0.5); CK(cudaDeviceSynchronize()); \
    CK(cudaMemcpy(h, d_cyc, sizeof(long long) * grid, cudaMemcpyDeviceToHost)); \
    double s = 0; for (int i = 0; i < grid; ++i) s += (double)h[i]; s /= grid; \
    double ops = (double)iters * 4 * (13 + (CV ? 1 : 0)); /* fp64-pipe ops per thread: 12 + input + (gain) */ \
    int warps = (threads) / 32 * (ctas_per_sm); \
    printf("%-10s %-6s %5d %5d %12.2f %10.1f\n", SK ? "skewed" : "plain", CV ? "yes" : "no", warps, ctas_per_sm, \
           ops * (threads) * (ctas_per_sm) / s, s / (iters * 4.0)); } while (0)
  int wl[] = {1, 2, 3, 4, 5, 6, 8};
  for (int wi = 0; wi < 7; ++wi) { int w = wl[wi]; RUN(false, false, 32 * 4, w); }
  for (int wi = 0; wi < 7; ++wi) { int w = wl[wi]; RUN(true, false, 32 * 4, w); }
  for (int wi = 0; wi < 7; ++wi) { int w = wl[wi]; RUN(false, true, 32 * 4, w); }
  for (int wi = 0; wi < 7; ++wi) { int w = wl[wi]; RUN(true, true, 32 * 4, w); }

  {
    UParams* hp = new UParams;
    for (int c = 0; c < 64; ++c) { for (int k = 0; k < 4; ++k) { hp->ch[c].c1[k] = -0.9 + 0.01 * k + 1e-4 * c; hp->ch[c].na1[k] = 1.2 - 0.02 * k; hp->ch[c].na2[k] = -0.5 - 0.01 * k; } hp->ch[c].G = 1e-3; }
    printf("uniform-coefficient variants (1 warp per CTA): incvt outcvt warps/SM  fp64ops/clk/SM cyc/sample\n");
#define RUNU(IC, OC, wps, nfp64) do { \
      int grid = nsm * (wps); \
      k_uniform<IC, OC><<<grid, 32>>>(*hp, d_out, d_cyc, iters, 0.5f); CK(cudaDeviceSynchronize()); \
      cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1); cudaEventRecord(e0); \
      k_uniform<IC, OC><<<grid, 32>>>(*hp, d_out, d_cyc, iters, 0.5f); cudaEventRecord(e1); CK(cudaDeviceSynchronize()); \
      float ms; cudaEventElapsedTime(&ms, e0, e1); \
      CK(cudaMemcpy(h, d_cyc, sizeof(long long) * grid, cudaMemcpyDeviceToHost)); \
      double s = 0; for (int i = 0; i < grid; ++i) s += (double)h[i]; s /= grid; \
      printf("  incvt %d outcvt %d warps %2d  %7.2f  %7.1f   (event %.3f ms -> %.1f cyc/sample/SMSP-warp @1.95GHz)\n", IC, (int)OC, wps, \
             (double)iters * 4 * (nfp64) * 32 * (wps) / s, s / (iters * 4.0), ms, ms * 1e-3 * 1.95e9 / (iters * 4.0) / ((wps) / 4.0)); } while (0)
    int ws[] = {8, 16, 20, 24, 32};
    for (int i = 0; i < 5; ++i) RUNU(0, false, ws[i], 14);
    for (int i = 0; i < 5; ++i) RUNU(0, true, ws[i], 14);
    for (int i = 0; i < 5; ++i) RUNU(1, true, ws[i], 13);
    for (int i = 0; i < 5; ++i) RUNU(2, true, ws[i], 13);
  }
  return 0;
}
