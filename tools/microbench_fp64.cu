// Micro-benchmarks that size the recurrence kernel's design on H100 (sm_90a):
//   * DFMA issue rate per SM (ILP x warps sweep) and dependent-chain latency
//   * F2F.F32.F64 / F2F.F64.F32 conversion rate, alone and mixed with DFMA
//   * FFMA rate for comparison
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o microbench_fp64 microbench_fp64.cu
// Prints one line per experiment: name, ops/clk/SM (SM clock measured with clock64).
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { \
  printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e), __FILE__, __LINE__); exit(1);} } while (0)

template <int ILP>
__global__ void k_dfma(double* out, long long* cyc, int iters, double a, double b) {
  double v[ILP];
#pragma unroll
  for (int i = 0; i < ILP; ++i) v[i] = threadIdx.x * 1e-3 + i;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int i = 0; i < ILP; ++i) v[i] = fma(v[i], a, b);
    }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < ILP; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

template <int ILP>
__global__ void k_ffma(float* out, long long* cyc, int iters, float a, float b) {
  float v[ILP];
#pragma unroll
  for (int i = 0; i < ILP; ++i) v[i] = threadIdx.x * 1e-3f + i;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int i = 0; i < ILP; ++i) v[i] = fmaf(v[i], a, b);
    }
  }
  long long t1 = clock64();
  float s = 0;
#pragma unroll
  for (int i = 0; i < ILP; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// double -> float -> double round trip chain: 1 F2F.F32.F64 + 1 F2F.F64.F32 per step
template <int ILP>
__global__ void k_cvt(double* out, long long* cyc, int iters, double a) {
  double v[ILP];
#pragma unroll
  for (int i = 0; i < ILP; ++i) v[i] = threadIdx.x * 1e-3 + i + a;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 8; ++r) {
#pragma unroll
      for (int i = 0; i < ILP; ++i) {
        float f;
        asm volatile("cvt.rn.f32.f64 %0, %1;" : "=f"(f) : "d"(v[i]));
        asm volatile("cvt.f64.f32 %0, %1;" : "=d"(v[i]) : "f"(f));
      }
    }
  }
  long long t1 = clock64();
  double s = 0;
#pragma unroll
  for (int i = 0; i < ILP; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

// Mixed: NF dfma chains plus one d->f conversion per NF dfma (the kernel's real mix ~12:1)
template <int NF>
__global__ void k_mix(double* out, float* outf, long long* cyc, int iters, double a, double b) {
  double v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) v[i] = threadIdx.x * 1e-3 + i;
  float acc = 0.f;
  long long t0 = clock64();
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < NF / 4; ++r) {
#pragma unroll
      for (int i = 0; i < 4; ++i) v[i] = fma(v[i], a, b);
    }
    float f;
    asm volatile("cvt.rn.f32.f64 %0, %1;" : "=f"(f) : "d"(v[0]));
    acc += f;
  }
  long long t1 = clock64();
  out[blockIdx.x * blockDim.x + threadIdx.x] = v[0] + v[1] + v[2] + v[3];
  outf[blockIdx.x * blockDim.x + threadIdx.x] = acc;
  if (threadIdx.x == 0) cyc[blockIdx.x] = t1 - t0;
}

static double avg_cycles(long long* d_cyc, int n) {
  long long* h = (long long*)malloc(n * sizeof(long long));
  CK(cudaMemcpy(h, d_cyc, n * sizeof(long long), cudaMemcpyDeviceToHost));
  double s = 0; for (int i = 0; i < n; ++i) s += (double)h[i];
  free(h); return s / n;
}

int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  int nsm = p.multiProcessorCount;
  printf("device %s sms %d clock %d kHz\n", p.name, nsm, p.clockRate);
  double* d_out; float* d_outf; long long* d_cyc;
  CK(cudaMalloc(&d_out, sizeof(double) * nsm * 2048));
  CK(cudaMalloc(&d_outf, sizeof(float) * nsm * 2048));
  CK(cudaMalloc(&d_cyc, sizeof(long long) * nsm * 2));
  const int iters = 4096;
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));

#define RUN(name, kern, threads, ops_per_thread, ...) do { \
    kern<<<nsm, threads>>>(__VA_ARGS__); CK(cudaDeviceSynchronize()); \
    CK(cudaEventRecord(e0)); kern<<<nsm, threads>>>(__VA_ARGS__); CK(cudaEventRecord(e1)); \
    CK(cudaDeviceSynchronize()); float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); \
    double cyc = avg_cycles(d_cyc, nsm); \
    printf("%-28s threads %4d  cycles %10.0f  ops/clk/SM %7.2f  ms %.3f  eff_MHz %.0f\n", name, threads, cyc, \
           (double)(ops_per_thread) * threads / cyc, ms, cyc / (ms * 1e3)); } while (0)

  // DFMA latency: 1 warp, ILP1
  RUN("dfma lat ilp1 1warp", k_dfma<1>, 32, iters * 8.0, d_out, d_cyc, iters, 1.0000001, 1e-9);
  RUN("ffma lat ilp1 1warp", k_ffma<1>, 32, iters * 8.0, d_outf, d_cyc, iters, 1.0000001f, 1e-9f);
  int tl[] = {128, 256, 512, 1024};
  for (int ti = 0; ti < 4; ++ti) {
    int t = tl[ti];
    RUN("dfma ilp1", k_dfma<1>, t, iters * 8.0 * 1, d_out, d_cyc, iters, 1.0000001, 1e-9);
    RUN("dfma ilp2", k_dfma<2>, t, iters * 8.0 * 2, d_out, d_cyc, iters, 1.0000001, 1e-9);
    RUN("dfma ilp4", k_dfma<4>, t, iters * 8.0 * 4, d_out, d_cyc, iters, 1.0000001, 1e-9);
    RUN("dfma ilp8", k_dfma<8>, t, iters * 8.0 * 8, d_out, d_cyc, iters, 1.0000001, 1e-9);
  }
  RUN("ffma ilp4", k_ffma<4>, 1024, iters * 8.0 * 4, d_outf, d_cyc, iters, 1.0000001f, 1e-9f);
  RUN("ffma ilp8", k_ffma<8>, 1024, iters * 8.0 * 8, d_outf, d_cyc, iters, 1.0000001f, 1e-9f);
  RUN("cvt d2f+f2d lat ilp1 1warp", k_cvt<1>, 32, iters * 8.0 * 2, d_out, d_cyc, iters, 0.5);
  RUN("cvt d2f+f2d ilp4", k_cvt<4>, 1024, iters * 8.0 * 4 * 2, d_out, d_cyc, iters, 0.5);
  RUN("cvt d2f+f2d ilp4", k_cvt<4>, 256, iters * 8.0 * 4 * 2, d_out, d_cyc, iters, 0.5);
  // mixes: count only dfma ops
  RUN("mix 12 dfma : 1 cvt", k_mix<12>, 1024, iters * 12.0, d_out, d_outf, d_cyc, iters, 1.0000001, 1e-9);
  RUN("mix 4 dfma : 1 cvt", k_mix<4>, 1024, iters * 4.0, d_out, d_outf, d_cyc, iters, 1.0000001, 1e-9);
  RUN("mix 12 dfma : 1 cvt", k_mix<12>, 512, iters * 12.0, d_out, d_outf, d_cyc, iters, 1.0000001, 1e-9);
  return 0;
}
