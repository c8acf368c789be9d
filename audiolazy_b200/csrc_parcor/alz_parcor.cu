// alz_parcor.cu -- the C ABI of include/alz_b200_parcor.h: the PARCOR step-down of many rows on sm_90a.
//
// A row's M steps form one dependent chain (a pow, a reciprocal and one update of every coefficient per step), and
// rows are independent, so the kernel is latency-bound and keeps each row in registers: a group of G lanes (8, 16 or
// 32, the smallest with 2 G >= L - 1) owns one row, lane l holding a[1 + l] and a[1 + l + G].  Each step broadcasts k
// = a[m] from its lane and pairs a[j] with a[m - j] by shuffle (a[1 + l + G] only ever pairs with a first-slot
// value).  The groups of a warp step in lockstep up to the warp's largest M, a finished row idling, so every shuffle
// is made by the full warp.  Lane t % G keeps the t-th emitted k, so the k row is stored once, coalesced, at the end.
//
// Every operation is spelled with a round-to-nearest intrinsic and the unit is compiled with -fmad=false: the only
// DFMAs are the pow restatement's own (alz_pow2.h) and the Newton steps of the correctly rounded reciprocal.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_parcor.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"
#include "alz_pow2.h"

#include <cuda_runtime.h>

#include <cstdint>

namespace {

constexpr int kThreads = 256;
constexpr unsigned kFull = 0xffffffffu;
constexpr long long kMaxGrid = 1 << 20;

// One coefficient of a step: a[j] - k a[m - j] times r, where a zero scalar or a missing term contributes nothing.
__device__ __forceinline__ double step(double x, double y, double k, double r) {
  const double t = (k == 0.0 || y == 0.0) ? x : __dsub_rn(x, __dmul_rn(k, y));
  return (r == 0.0 || t == 0.0) ? 0.0 : __dmul_rn(t, r);
}

}  // namespace

template <int G>
__global__ void __launch_bounds__(kThreads) alz_parcor_kernel(const double* __restrict__ coef, long long stride,
                                                              long long n, int L, double* __restrict__ k_out,
                                                              int32_t* __restrict__ count_out,
                                                              uint8_t* __restrict__ failed_out,
                                                              uint8_t* __restrict__ stable_out) {
  constexpr int rpc = kThreads / G;
  const int l = threadIdx.x % G;
  const int K = L - 1;
  const int i0 = 1 + l, i1 = 1 + l + G;
  const double nan = __longlong_as_double(0x7ff8000000000000LL);
  for (long long base = (long long)blockIdx.x * rpc; base < n; base += (long long)gridDim.x * rpc) {
    const long long row = base + threadIdx.x / G;
    const bool valid = row < n;
    const double* a = coef + row * stride;
    double v0 = valid && i0 < L ? a[i0] : 0.0;
    double v1 = valid && i1 < L ? a[i1] : 0.0;
    const bool monic = valid && a[0] == 1.0;
    int top = v1 != 0.0 ? i1 : (v0 != 0.0 ? i0 : 0);
#pragma unroll
    for (int o = G / 2; o; o >>= 1) top = max(top, __shfl_xor_sync(kFull, top, o, G));
    const int M = monic ? top : 0;
    const int steps = (int)__reduce_max_sync(kFull, (unsigned)M);
    int failed = valid && !monic ? 3 : 0, count = 0;
    bool stable = monic;
    double o0 = nan, o1 = nan;
    for (int t = 0; t < steps; ++t) {
      const int m = M - t;
      const bool active = failed == 0 && m >= 1;
      const int src = active ? (m - 1) & (G - 1) : 0;
      const double s0 = __shfl_sync(kFull, v0, src, G), s1 = __shfl_sync(kFull, v1, src, G);
      double k = m - 1 >= G ? s1 : s0;
      if (k == 0.0) k = 0.0;
      if (active) {
        if (l == (t & (G - 1))) {
          if (t < G) o0 = k;
          else o1 = k;
        }
        count = t + 1;
        if (!(fabs(k) < 1.0)) stable = false;
      }
      int overflow;
      const double d = __dsub_rn(1.0, alz_py_pow2(k, &overflow));
      if (active && overflow) failed = 2;
      else if (active && d == 0.0) failed = 1;
      const double r = __drcp_rn(d);
      const int p0 = m - i0, p1 = m - i1;   // partners; p1 - 1 < G always
      const int sl0 = p0 >= 1 ? (p0 - 1) & (G - 1) : 0;
      const int sl1 = p1 >= 1 ? p1 - 1 : 0;
      const double y0a = __shfl_sync(kFull, v0, sl0, G), y0b = __shfl_sync(kFull, v1, sl0, G);
      const double y1 = __shfl_sync(kFull, v0, sl1, G);
      if (active && failed == 0) {
        if (i0 < m) v0 = step(v0, p0 - 1 >= G ? y0b : y0a, k, r);
        if (i1 < m) v1 = step(v1, y1, k, r);
      }
    }
    if (valid) {
      if (k_out) {
        double* ko = k_out + row * K;
        if (l < K) ko[l] = o0;
        if (l + G < K) ko[l + G] = o1;
      }
      if (l == 0) {
        if (count_out) count_out[row] = count;
        if (failed_out) failed_out[row] = (uint8_t)failed;
        if (stable_out) stable_out[row] = (uint8_t)stable;
      }
    }
  }
}

namespace {

template <int G>
cudaError_t launch(const double* coef, long long stride, long long n, int L, double* k, int32_t* count,
                   uint8_t* failed, uint8_t* stable, cudaStream_t cs) {
  constexpr int rpc = kThreads / G;
  long long grid = (n + rpc - 1) / rpc;
  if (grid > kMaxGrid) grid = kMaxGrid;
  alz_parcor_kernel<G><<<(unsigned)grid, kThreads, 0, cs>>>(coef, stride, n, L, k, count, failed, stable);
  return cudaGetLastError();
}

}  // namespace

extern "C" {

const char* alz_parcor_last_error(void) { return g_err.c_str(); }

int32_t alz_parcor_f64(const double* coef_dev, int64_t row_stride, int64_t n_rows, int32_t L, double* k_dev,
                       int32_t* count_dev, uint8_t* failed_dev, uint8_t* stable_dev, void* cuda_stream) {
  if (L < 1 || L > ALZ_PARCOR_MAX_LEN)
    return fail(ALZ_PARCOR_ERR_INVALID, "L must be in 1 .. %d (got %d)", ALZ_PARCOR_MAX_LEN, L);
  if (n_rows < 0) return fail(ALZ_PARCOR_ERR_INVALID, "n_rows must be >= 0");
  if (n_rows == 0) return ALZ_PARCOR_OK;
  if (!coef_dev) return fail(ALZ_PARCOR_ERR_INVALID, "NULL coefficients");
  if (n_rows > 1 && row_stride < L) return fail(ALZ_PARCOR_ERR_INVALID, "row_stride < L");
  if (((uintptr_t)coef_dev & 7) || ((uintptr_t)k_dev & 7) || ((uintptr_t)count_dev & 3))
    return fail(ALZ_PARCOR_ERR_INVALID, "misaligned buffer");
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  const int K = L - 1;
  cudaError_t e;
  if (K <= 16) e = launch<8>(coef_dev, row_stride, n_rows, L, k_dev, count_dev, failed_dev, stable_dev, cs);
  else if (K <= 32) e = launch<16>(coef_dev, row_stride, n_rows, L, k_dev, count_dev, failed_dev, stable_dev, cs);
  else e = launch<32>(coef_dev, row_stride, n_rows, L, k_dev, count_dev, failed_dev, stable_dev, cs);
  ALZ_CUDA_CHECK(e, ALZ_PARCOR_ERR_CUDA);
  return ALZ_PARCOR_OK;
}

}  // extern "C"
