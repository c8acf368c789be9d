// alz_lpcfilt.cu -- frame-wise LPC analysis (FIR) and synthesis (all-pole) filtering of many streams, bit for bit as
// AudioLazy's time-varying ZFilters compute them (include/alz_b200_lpcfilt.h).
//
// Compiled with -fmad=false, and every product and sum is spelled __dmul_rn / __dadd_rn: the reference rounds each
// product and each addition once, left to right in ascending delay, so nothing may be contracted or reordered.  No
// kernel pads a row to a longer order: a padded 0 * inf term would turn a value into NaN.
//
// * alz_lpcfilt_analysis_kernel<In, Out>: sample-parallel.  A CTA owns kTile samples of one stream and stages them,
//   after the `order` samples before them (from the state on the stream's first tile), widened to float64 in shared
//   memory; each thread loads and stores its own kPer = 8 consecutive samples in 16-byte accesses when the rows are
//   aligned (else one at a time).  Each thread computes those 8 outputs.  It walks the taps k = 1 .. order once for
//   the eight, keeping the eight samples x[n + q - k] in registers and loading one new one per tap, so a tap costs one
//   shared load and one coefficient load (one row when its eight samples share it) for eight products and eight
//   additions.  The shared layout puts sample i at i + i / 8, so the eight-apart loads of a warp hit distinct banks
//   (8 outputs rather than 4 per thread took the order-16 flagship shape from 0.52 ms to 0.41 ms; DESIGN.md §5).
// * alz_lpcfilt_commit_kernel<In>: after the analysis, the state's last `order` inputs, one thread per stream.
// * Synthesis: serial per stream, one thread per stream: float64 addition in a fixed order has no time-parallel form
//   that keeps the bits.  alz_lpcfilt_synthesis_reg_kernel<ORDER> (orders 1 .. 32) keeps the last ORDER outputs and
//   the row's taps in registers and issues a sample's products ahead of its dependent additions;
//   alz_lpcfilt_synthesis_kernel<In, Out> (orders 0 and 33 .. 64) keeps the last 64 outputs in a ring in shared
//   memory (one column per thread), and the current row's negated taps too, copied once per row (the 32 streams of a
//   warp read distinct rows, which as global loads would cost one transaction per lane and tap); it walks the taps in
//   runs of 8.  Both write their last `order` outputs into the state.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_lpcfilt.h"
#pragma GCC visibility pop

#include <array>
#include <cstdint>
#include <utility>

#include "../csrc_common/alz_common.h"

namespace {

constexpr int kThreads = 256;
constexpr int kPer = 8;                        // consecutive outputs per thread
constexpr int kTile = kThreads * kPer;         // samples per analysis CTA
constexpr int kRing = 64;                      // synthesis ring: >= ALZ_LPCFILT_MAX_ORDER, a power of two
constexpr int kSynThreads = 32;

struct Args {
  const void* x;
  void* out;
  const double* coef;
  double* state;
  long long xs, os, crs, ccs;   // strides (elements): input row, output row, coefficient row, coefficient stream
  long long S, T, C, hop;       // streams, samples, samples consumed before the call, hop
  long long r0;                 // floor(C / hop): the stream row of the call's row 0
  long long nt;                 // analysis tiles per stream
  int order;
  int vec;                      // the rows of x and out start 16-byte aligned: the analysis moves 4 samples at a time
};

__host__ __device__ inline int sidx(int i) { return i + i / kPer; }

template <typename T>
__device__ __forceinline__ double widen(T v) { return (double)v; }

template <typename T>
__device__ __forceinline__ T narrow(double v);
template <>
__device__ __forceinline__ double narrow<double>(double v) { return v; }
template <>
__device__ __forceinline__ float narrow<float>(double v) { return __double2float_rn(v); }

// Four consecutive samples, 16-byte aligned (Args::vec), in 16-byte accesses.
__device__ __forceinline__ void load4(const float* p, double v[4]) {
  const float4 f = *reinterpret_cast<const float4*>(p);
  v[0] = f.x, v[1] = f.y, v[2] = f.z, v[3] = f.w;
}
__device__ __forceinline__ void load4(const double* p, double v[4]) {
  const double2 a = reinterpret_cast<const double2*>(p)[0], b = reinterpret_cast<const double2*>(p)[1];
  v[0] = a.x, v[1] = a.y, v[2] = b.x, v[3] = b.y;
}
__device__ __forceinline__ void store4(float* p, const double v[4]) {
  *reinterpret_cast<float4*>(p) =
      make_float4(__double2float_rn(v[0]), __double2float_rn(v[1]), __double2float_rn(v[2]), __double2float_rn(v[3]));
}
__device__ __forceinline__ void store4(double* p, const double v[4]) {
  reinterpret_cast<double2*>(p)[0] = make_double2(v[0], v[1]);
  reinterpret_cast<double2*>(p)[1] = make_double2(v[2], v[3]);
}

// The row (in the call) of stream sample C + n.
__device__ __forceinline__ long long row_of(const Args& a, long long n) { return (a.C + n) / a.hop - a.r0; }

}  // namespace

template <typename In, typename Out>
__global__ void __launch_bounds__(kThreads) alz_lpcfilt_analysis_kernel(Args a) {
  extern __shared__ double s_x[];              // samples tile0 - order .. tile0 + kTile - 1, at sidx(i)
  const long long s = blockIdx.x / a.nt;
  const long long n0 = (blockIdx.x % a.nt) * (long long)kTile;
  const int order = a.order;
  const In* x = static_cast<const In*>(a.x) + s * a.xs;
  const double* hist = a.state + s * order;
  for (int i = threadIdx.x; i < order; i += kThreads) {    // the `order` samples before the tile
    const long long n = n0 - order + i;
    s_x[sidx(i)] = n >= 0 ? widen(x[n]) : hist[order + n];
  }
  const long long n = n0 + kPer * threadIdx.x;  // this thread's first sample
  const int i0 = order + kPer * threadIdx.x;     // its shared index
  double acc[kPer], w[kPer];
  if (a.vec && n + kPer <= a.T) {
#pragma unroll
    for (int q = 0; q < kPer; q += 4) load4(x + n + q, acc + q);
  } else {
#pragma unroll
    for (int q = 0; q < kPer; ++q) acc[q] = n + q < a.T ? widen(x[n + q]) : 0.0;
  }
#pragma unroll
  for (int q = 0; q < kPer; ++q) s_x[sidx(i0 + q)] = acc[q];
  __syncthreads();

  if (n >= a.T) return;
#pragma unroll
  for (int q = 0; q < kPer; ++q) w[q] = order > 0 ? s_x[sidx(i0 + q - 1)] : 0.0;   // x[n + q - 1]
  const double* cs = a.coef + s * a.ccs;
  const long long last = n + kPer - 1 < a.T ? n + kPer - 1 : a.T - 1;   // rows past the call are not read
  const long long ra = row_of(a, n), rb = row_of(a, last);
  if (ra == rb) {
    const double* c = cs + ra * a.crs;
    for (int k = 1; k <= order; ++k) {
      const double ck = __ldg(c + k);
#pragma unroll
      for (int q = 0; q < kPer; ++q) acc[q] = __dadd_rn(acc[q], __dmul_rn(ck, w[q]));
#pragma unroll
      for (int q = kPer - 1; q > 0; --q) w[q] = w[q - 1];
      if (k < order) w[0] = s_x[sidx(i0 - k - 1)];
    }
  } else {
    const double* c[kPer];
#pragma unroll
    for (int q = 0; q < kPer; ++q) c[q] = cs + row_of(a, n + q <= last ? n + q : last) * a.crs;
    for (int k = 1; k <= order; ++k) {
#pragma unroll
      for (int q = 0; q < kPer; ++q) acc[q] = __dadd_rn(acc[q], __dmul_rn(__ldg(c[q] + k), w[q]));
#pragma unroll
      for (int q = kPer - 1; q > 0; --q) w[q] = w[q - 1];
      if (k < order) w[0] = s_x[sidx(i0 - k - 1)];
    }
  }
  Out* out = static_cast<Out*>(a.out) + s * a.os;
  if (a.vec && n + kPer <= a.T) {
#pragma unroll
    for (int q = 0; q < kPer; q += 4) store4(out + n + q, acc + q);
  } else {
#pragma unroll
    for (int q = 0; q < kPer; ++q)
      if (n + q < a.T) out[n + q] = narrow<Out>(acc[q]);
  }
}

// The state's last `order` inputs after the call: hist[j] = sample C + T - order + j.  In place, ascending: the new
// hist[j] reads the old hist[j + T], which no earlier j has written.
template <typename In>
__global__ void __launch_bounds__(kThreads) alz_lpcfilt_commit_kernel(Args a) {
  const long long s = blockIdx.x * (long long)kThreads + threadIdx.x;
  if (s >= a.S) return;
  const In* x = static_cast<const In*>(a.x) + s * a.xs;
  double* hist = a.state + s * a.order;
  for (int j = 0; j < a.order; ++j) {
    const long long n = a.T - a.order + j;
    hist[j] = n >= 0 ? widen(x[n]) : hist[j + a.T];
  }
}

template <typename In, typename Out>
__global__ void __launch_bounds__(kSynThreads) alz_lpcfilt_synthesis_kernel(Args a) {
  __shared__ double s_ring[kRing * kSynThreads];   // output n at slot ((C + n) & 63), column threadIdx.x
  __shared__ double s_nc[kRing * kSynThreads];     // -c_k of the current row at k - 1, column threadIdx.x
  const long long s = blockIdx.x * (long long)kSynThreads + threadIdx.x;
  if (s >= a.S) return;
  const int order = a.order;
  double* ring = s_ring + threadIdx.x;
  double* nc = s_nc + threadIdx.x;
  double* hist = a.state + s * order;
  const long long C = a.C;
  for (int j = 0; j < order; ++j) ring[((C - order + j) & (kRing - 1)) * kSynThreads] = hist[j];
  const In* x = static_cast<const In*>(a.x) + s * a.xs;
  Out* out = static_cast<Out*>(a.out) + s * a.os;
  const double* cs = a.coef + s * a.ccs;
  long long row_end = (a.r0 + 1) * a.hop - C;    // first sample of the next row
  const double* c = cs;
  for (int k = 1; k <= order; ++k) nc[(k - 1) * kSynThreads] = -__ldg(c + k);
  double xn = widen(x[0]);
  for (long long n = 0; n < a.T; ++n) {
    const double x0 = xn;
    if (n + 1 < a.T) xn = widen(x[n + 1]);
    if (n == row_end) {                          // a new row: its negated taps into this thread's column
      c += a.crs;
      row_end += a.hop;
      for (int k = 1; k <= order; ++k) nc[(k - 1) * kSynThreads] = -__ldg(c + k);
    }
    const int slot = (int)((C + n) & (kRing - 1));
    double acc = x0;
    int k = 1;
    for (; k + 7 <= order; k += 8) {
      double p[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        p[u] = __dmul_rn(nc[(k + u - 1) * kSynThreads], ring[((slot - k - u) & (kRing - 1)) * kSynThreads]);
#pragma unroll
      for (int u = 0; u < 8; ++u) acc = __dadd_rn(acc, p[u]);
    }
    for (; k <= order; ++k)
      acc = __dadd_rn(acc, __dmul_rn(nc[(k - 1) * kSynThreads], ring[((slot - k) & (kRing - 1)) * kSynThreads]));
    ring[slot * kSynThreads] = acc;
    out[n] = narrow<Out>(acc);
  }
  for (int j = 0; j < order; ++j) hist[j] = ring[((C + a.T - order + j) & (kRing - 1)) * kSynThreads];
}

// The synthesis at one exact order ORDER <= kRegMax, all in registers: the last ORDER outputs h[j] = y[n - 1 - j] and
// the current row's negated taps.  All ORDER products of a sample read outputs that are known when the sample starts,
// so they issue together, ahead of the dependent additions; only the first waits on the previous sample's chain.  The
// samples are loaded kAhead samples ahead.  The dtypes are run-time flags, uniform over the launch.
constexpr int kRegMax = 32;
constexpr int kAhead = 8;

template <int ORDER>
__global__ void __launch_bounds__(kSynThreads) alz_lpcfilt_synthesis_reg_kernel(Args a, int x64, int out64) {
  const long long s = blockIdx.x * (long long)kSynThreads + threadIdx.x;
  if (s >= a.S) return;
  double* hist = a.state + s * ORDER;
  double h[ORDER], nc[ORDER];
#pragma unroll
  for (int j = 0; j < ORDER; ++j) h[j] = hist[ORDER - 1 - j];
  const double* c = a.coef + s * a.ccs;
#pragma unroll
  for (int k = 0; k < ORDER; ++k) nc[k] = -__ldg(c + k + 1);
  const float* xf = static_cast<const float*>(a.x) + s * a.xs;
  const double* xd = static_cast<const double*>(a.x) + s * a.xs;
  float* of = static_cast<float*>(a.out) + s * a.os;
  double* od = static_cast<double*>(a.out) + s * a.os;
  const long long T = a.T;
  double q[kAhead];                              // samples n .. n + kAhead - 1
#pragma unroll
  for (int i = 0; i < kAhead; ++i) q[i] = i < T ? (x64 ? xd[i] : (double)xf[i]) : 0.0;
  long long row_end = (a.r0 + 1) * a.hop - a.C;
  for (long long n = 0; n < T; ++n) {
    const double x0 = q[0];
#pragma unroll
    for (int i = 0; i + 1 < kAhead; ++i) q[i] = q[i + 1];
    const long long nn = n + kAhead;
    q[kAhead - 1] = nn < T ? (x64 ? xd[nn] : (double)xf[nn]) : 0.0;
    if (n == row_end) {
      c += a.crs;
      row_end += a.hop;
#pragma unroll
      for (int k = 0; k < ORDER; ++k) nc[k] = -__ldg(c + k + 1);
    }
    double p[ORDER];
#pragma unroll
    for (int k = 0; k < ORDER; ++k) p[k] = __dmul_rn(nc[k], h[k]);
    double acc = x0;
#pragma unroll
    for (int k = 0; k < ORDER; ++k) acc = __dadd_rn(acc, p[k]);
#pragma unroll
    for (int j = ORDER - 1; j > 0; --j) h[j] = h[j - 1];
    h[0] = acc;
    if (out64) od[n] = acc;
    else of[n] = __double2float_rn(acc);
  }
#pragma unroll
  for (int j = 0; j < ORDER; ++j) hist[ORDER - 1 - j] = h[j];
}

namespace {

using RegKernel = void (*)(Args, int, int);

template <int... O>
constexpr std::array<RegKernel, sizeof...(O)> reg_kernels(std::integer_sequence<int, O...>) {
  return {&alz_lpcfilt_synthesis_reg_kernel<O + 1>...};
}

// alz_lpcfilt_synthesis_reg_kernel<order> for order 1 .. kRegMax, at [order - 1]
const std::array<RegKernel, kRegMax> kRegKernels = reg_kernels(std::make_integer_sequence<int, kRegMax>());

template <typename In, typename Out>
cudaError_t launch(const Args& a, int kind, cudaStream_t cs) {
  if (kind == ALZ_LPCFILT_SYNTHESIS) {
    const unsigned grid = (unsigned)((a.S + kSynThreads - 1) / kSynThreads);
    if (a.order >= 1 && a.order <= kRegMax) {
      kRegKernels[a.order - 1]<<<grid, kSynThreads, 0, cs>>>(a, (int)sizeof(In) == 8, (int)sizeof(Out) == 8);
      return cudaGetLastError();
    }
    alz_lpcfilt_synthesis_kernel<In, Out><<<(unsigned)((a.S + kSynThreads - 1) / kSynThreads), kSynThreads, 0, cs>>>(a);
    return cudaGetLastError();
  }
  const size_t smem = (size_t)(sidx(a.order + kTile - 1) + 1) * sizeof(double);
  alz_lpcfilt_analysis_kernel<In, Out><<<(unsigned)(a.S * a.nt), kThreads, smem, cs>>>(a);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || a.order == 0) return e;
  alz_lpcfilt_commit_kernel<In><<<(unsigned)((a.S + kThreads - 1) / kThreads), kThreads, 0, cs>>>(a);
  return cudaGetLastError();
}

bool bad_dtype(int32_t t) { return t != ALZ_LPCFILT_FLOAT32 && t != ALZ_LPCFILT_FLOAT64; }

long long elem_bytes(int32_t t) { return t == ALZ_LPCFILT_FLOAT64 ? 8 : 4; }

long long rows(long long consumed, long long n_samples, long long hop) {
  return n_samples > 0 ? (consumed + n_samples - 1) / hop - consumed / hop + 1 : 0;
}

}  // namespace

extern "C" {

const char* alz_lpcfilt_last_error(void) { return g_err.c_str(); }

int64_t alz_lpcfilt_state_bytes(int64_t n_streams, int32_t order) {
  if (n_streams < 0) return fail(ALZ_LPCFILT_ERR_INVALID, "need n_streams >= 0");
  if (order < 0 || order > ALZ_LPCFILT_MAX_ORDER)
    return fail(ALZ_LPCFILT_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPCFILT_MAX_ORDER, order);
  return n_streams * 8 * (int64_t)order;
}

int32_t alz_lpcfilt_state_init(void* state_dev, int64_t n_streams, int32_t order, void* cuda_stream) {
  const int64_t nbytes = alz_lpcfilt_state_bytes(n_streams, order);
  if (nbytes < 0) return (int32_t)nbytes;
  if (nbytes == 0) return ALZ_LPCFILT_OK;
  if (!state_dev) return fail(ALZ_LPCFILT_ERR_INVALID, "state is NULL");
  if ((uintptr_t)state_dev & 7) return fail(ALZ_LPCFILT_ERR_INVALID, "misaligned state");
  ALZ_CUDA_CHECK(cudaMemsetAsync(state_dev, 0, (size_t)nbytes, (cudaStream_t)cuda_stream), ALZ_LPCFILT_ERR_CUDA);
  return ALZ_LPCFILT_OK;
}

int64_t alz_lpcfilt_rows(int64_t consumed, int64_t n_samples, int64_t hop) {
  if (consumed < 0 || n_samples < 0) return fail(ALZ_LPCFILT_ERR_INVALID, "need consumed >= 0 and n_samples >= 0");
  if (hop < 1) return fail(ALZ_LPCFILT_ERR_INVALID, "hop must be >= 1 (got %lld)", (long long)hop);
  return rows(consumed, n_samples, hop);
}

int32_t alz_lpcfilt_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                          int64_t out_stride, const double* coef_dev, int64_t coef_row_stride,
                          int64_t coef_stream_stride, int64_t n_rows, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int64_t consumed, int32_t order, int64_t hop, int32_t kind,
                          void* cuda_stream) {
  if (kind != ALZ_LPCFILT_ANALYSIS && kind != ALZ_LPCFILT_SYNTHESIS)
    return fail(ALZ_LPCFILT_ERR_INVALID, "kind must be ALZ_LPCFILT_ANALYSIS or ALZ_LPCFILT_SYNTHESIS");
  if (order < 0 || order > ALZ_LPCFILT_MAX_ORDER)
    return fail(ALZ_LPCFILT_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPCFILT_MAX_ORDER, order);
  if (hop < 1) return fail(ALZ_LPCFILT_ERR_INVALID, "hop must be >= 1 (got %lld)", (long long)hop);
  if (n_streams < 0 || n_samples < 0 || consumed < 0)
    return fail(ALZ_LPCFILT_ERR_INVALID, "bad shape: n_streams %lld, n_samples %lld, consumed %lld",
                (long long)n_streams, (long long)n_samples, (long long)consumed);
  if (bad_dtype(x_dtype) || bad_dtype(out_dtype))
    return fail(ALZ_LPCFILT_ERR_INVALID, "dtype must be ALZ_LPCFILT_FLOAT32 or _FLOAT64");
  const long long need = rows(consumed, n_samples, hop);
  if (n_rows < need)
    return fail(ALZ_LPCFILT_ERR_INVALID, "coef holds %lld rows per stream, the call needs %lld", (long long)n_rows,
                need);
  if (n_streams == 0 || n_samples == 0) return ALZ_LPCFILT_OK;
  if (!x_dev || !out_dev || !coef_dev || (order > 0 && !state_dev)) return fail(ALZ_LPCFILT_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev % elem_bytes(x_dtype)) || ((uintptr_t)out_dev % elem_bytes(out_dtype)) ||
      ((uintptr_t)coef_dev & 7) || ((uintptr_t)state_dev & 7))
    return fail(ALZ_LPCFILT_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && (x_stride < n_samples || out_stride < n_samples))
    return fail(ALZ_LPCFILT_ERR_INVALID, "stride < n_samples");
  if (need > 1 && coef_row_stride < order + 1) return fail(ALZ_LPCFILT_ERR_INVALID, "coef row stride < order + 1");
  if (coef_stream_stride < 0) return fail(ALZ_LPCFILT_ERR_INVALID, "coef stream stride < 0");
  const long long nt = (n_samples + kTile - 1) / kTile;
  if (n_streams * nt > 0x7fffffffLL) return fail(ALZ_LPCFILT_ERR_UNSUPPORTED, "too many tiles for one launch");
  Args a{};
  a.x = x_dev;
  a.out = out_dev;
  a.coef = coef_dev;
  a.state = (double*)state_dev;
  a.xs = n_streams > 1 ? x_stride : n_samples;
  a.os = n_streams > 1 ? out_stride : n_samples;
  a.crs = coef_row_stride;
  a.ccs = coef_stream_stride;
  a.S = n_streams;
  a.T = n_samples;
  a.C = consumed;
  a.hop = hop;
  a.r0 = consumed / hop;
  a.nt = nt;
  a.order = order;
  a.vec = (uintptr_t)x_dev % 16 == 0 && (uintptr_t)out_dev % 16 == 0 && (a.xs * elem_bytes(x_dtype)) % 16 == 0 &&
          (a.os * elem_bytes(out_dtype)) % 16 == 0;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  const bool xd = x_dtype == ALZ_LPCFILT_FLOAT64, od = out_dtype == ALZ_LPCFILT_FLOAT64;
  const cudaError_t e = xd ? (od ? launch<double, double>(a, kind, cs) : launch<double, float>(a, kind, cs))
                           : (od ? launch<float, double>(a, kind, cs) : launch<float, float>(a, kind, cs));
  ALZ_CUDA_CHECK(e, ALZ_LPCFILT_ERR_CUDA);
  return ALZ_LPCFILT_OK;
}

}  // extern "C"
