// Micro-benchmark: DFMA issue rate on H100 as a function of WHERE the three operands
// come from (fresh register pairs, registers shared with the previous instruction,
// uniform registers).  8 independent chains per thread, 16 warps/SM; event-timed.
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)
struct UP { double c[16]; };
// MODE 0: v = fma(v, a, b)        a,b shared by all 8 chains (2 of 3 operands repeat)
// MODE 1: v = fma(v, c_i, b)      multiplier distinct per chain, addend shared
// MODE 2: v = fma(v, c_i, d_i)    all three operands distinct registers
// MODE 3: v = fma(v, U_i, d_i)    multiplier in a uniform register, addend distinct register
// MODE 4: v = fma(c_i, w_i, v)    accumulate form: two distinct register multiplicands + own accumulator
// MODE 5: v = fma(U_i, w_i, v)    accumulate form with uniform multiplier
template <int MODE>
__global__ void __launch_bounds__(128) k(const __grid_constant__ UP P, double* out, int iters, double seed) {
  double v[8], c[8], d[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) { v[i] = seed + threadIdx.x * 1e-3 + i; c[i] = 1.0 + 1e-9 * (threadIdx.x + i); d[i] = 1e-9 * (i + 1) + threadIdx.x * 1e-12; }
  const double a = c[0], b = d[0];
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int r = 0; r < 4; ++r) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        if (MODE == 0) v[i] = fma(v[i], a, b);
        if (MODE == 1) v[i] = fma(v[i], c[i], b);
        if (MODE == 2) v[i] = fma(v[i], c[i], d[i]);
        if (MODE == 3) v[i] = fma(v[i], P.c[(blockIdx.x + i) & 15], d[i]);
        if (MODE == 4) v[i] = fma(c[i], d[(i + r) & 7], v[i]);
        if (MODE == 5) v[i] = fma(P.c[(blockIdx.x + i) & 15], d[(i + r) & 7], v[i]);
      }
    }
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += v[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}
int main() {
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  const int nsm = p.multiProcessorCount;
  double* d_out; CK(cudaMalloc(&d_out, sizeof(double) * nsm * 4 * 128));
  UP up; for (int i = 0; i < 16; ++i) up.c[i] = 1.0 + 1e-9 * i;
  const int iters = 8192;
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  // measure the SM clock with a known-rate kernel is circular; report ns and DFMA/ns/SM instead
#define RUN(M, name) do { \
    k<M><<<nsm * 4, 128>>>(up, d_out, iters, 0.5); CK(cudaDeviceSynchronize()); \
    CK(cudaEventRecord(e0)); k<M><<<nsm * 4, 128>>>(up, d_out, iters, 0.5); CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize()); \
    float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); \
    double ops = (double)iters * 32 * 128 * 4; /* per SM */ \
    printf("%-44s %8.3f ms  %7.2f DFMA/ns/SM  (= %5.1f /clk/SM at 1.95 GHz)\n", name, ms, ops / (ms * 1e6), ops / (ms * 1e6) / 1.95); } while (0)
  RUN(0, "v=fma(v,a,b)      2 shared operands");
  RUN(1, "v=fma(v,c_i,b)    1 shared operand");
  RUN(2, "v=fma(v,c_i,d_i)  3 distinct registers");
  RUN(3, "v=fma(v,U_i,d_i)  uniform-reg multiplier");
  RUN(4, "v=fma(c_i,w_j,v)  accumulate, 3 distinct");
  RUN(5, "v=fma(U_i,w_j,v)  accumulate, uniform mult");
  return 0;
}
