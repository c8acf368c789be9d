// alz_lpcscan.cu -- time-parallel LPC synthesis of few long streams: chunk summaries, a carried-state scan and a rerun
// (include/alz_b200_lpcscan.h).
//
// Compiled with -fmad=false.  Every walk adds a sample's terms as alz_lpcfilt.cu's synthesis does: x[n] first, then
// __dmul_rn(-c_k, y[n - k]) for k = 1 .. order, each sum __dadd_rn.  So a walk from the call's state over the whole call
// (a flagged stream) or over chunk 0 gives alz_lpcfilt_apply's bits.  Only the scan contracts (explicit fma): it has no
// bit contract.
//
// * alz_lpcscan_walk_reg_kernel<ORDER> (orders 1 .. 32) keeps the last ORDER outputs and the row's negated taps in
//   registers; alz_lpcscan_walk_kernel (orders 0 and 33 .. 64) keeps them in shared memory, one column per thread, as
//   alz_lpcfilt_synthesis_kernel does.  Both run both walking passes:
//   - pass 0, the summaries: one thread per (stream, chunk, run), the run fastest, so that a warp's threads mostly share
//     a chunk and read the same row.  Run 0 walks the chunk's input from a zero state and stores its final state F_p;
//     run u >= 1 walks zero input from the unit state e_{u-1} and stores column u - 1 of M_p.  Within a warp the runs
//     differ by a predicate on the input load, not by a branch.
//   - pass 1, the rerun: one thread per (stream, chunk), from the scanned state s_p, storing outputs; the last chunk
//     writes the state.  A flagged stream's chunk-0 thread walks the whole call from the call's state instead.
// * alz_lpcscan_scan_kernel: one warp per stream; lane i owns state components i and i + 32.  Step p loads the lane's
//   rows of M_p (column-major, so that the loads of a column are one coalesced access) in blocks of 32 columns ahead
//   of the dependent products, and broadcasts s_p by shuffle.  Any NaN or infinity in F_p, M_p or s_p makes s_{p+1}
//   non-finite (inf * 0 is NaN), so testing the scanned states flags exactly the streams with a non-finite summary or
//   state.
//
// States inside this library are newest first, h[j] = y[n - 1 - j]; the caller's state is oldest first.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_lpcscan.h"
#pragma GCC visibility pop

#include <array>
#include <cmath>
#include <cstdint>
#include <utility>

#include "../csrc_common/alz_common.h"

namespace {

constexpr int kRegThreads = 128;
constexpr int kRegMax = 32;
constexpr int kAhead = 8;                      // samples loaded ahead of the register walk
constexpr int kSmemThreads = 32;
constexpr int kRing = 64;                      // shared-memory walk: >= ALZ_LPCSCAN_MAX_ORDER, a power of two
constexpr int kScanWarps = 4;                  // streams per scan CTA

struct Args {
  const void* x;
  void* out;
  const double* coef;
  double* state;
  double* F;                    // [S][P][order]: the chunks' zero-state final states
  double* M;                    // [S][P][order (column j)][order (component i)]: their unit-state responses
  double* st;                   // [S][P + 1][order]: the scanned start states s_p, s_P last
  int* flag;                    // [S]: 1 when the stream is walked sequentially
  long long xs, os, crs, ccs;   // strides (elements): input row, output row, coefficient row, coefficient stream
  long long S, T, C, hop;       // streams, samples, samples consumed before the call, hop
  long long r0;                 // floor(C / hop): the stream row of the call's row 0
  long long P;                  // chunks per stream
  int order;
  int x64, out64;
};

// First sample of chunk p (p = P: T).
__device__ __forceinline__ long long chunk_lo(const Args& a, long long p) {
  const long long q = a.T / a.P, r = a.T % a.P;
  return p * q + (p < r ? p : r);
}

__device__ __forceinline__ double load_x(const Args& a, long long s, long long n) {
  return a.x64 ? static_cast<const double*>(a.x)[s * a.xs + n] : (double)static_cast<const float*>(a.x)[s * a.xs + n];
}

__device__ __forceinline__ void store_y(const Args& a, long long s, long long n, double v) {
  if (a.out64) static_cast<double*>(a.out)[s * a.os + n] = v;
  else static_cast<float*>(a.out)[s * a.os + n] = __double2float_rn(v);
}

// The walk of thread g: its stream, chunk, run (pass 0) and samples.  Returns false when it has none.
struct Walk {
  long long s, p, n0, n1;
  int run;        // pass 0: 0 for the input run, u >= 1 for unit state e_{u - 1}; pass 1: 0
  bool seq;       // pass 1: a flagged stream walked whole by its chunk-0 thread
};

__device__ __forceinline__ bool walk_of(const Args& a, int pass, long long g, Walk& w) {
  const long long R = pass == 0 ? a.order + 1 : 1;
  if (g >= a.S * a.P * R) return false;
  w.run = (int)(g % R);
  w.p = (g / R) % a.P;
  w.s = g / (R * a.P);
  w.seq = pass == 1 && a.flag[w.s];
  if (w.seq && w.p > 0) return false;
  w.n0 = w.seq ? 0 : chunk_lo(a, w.p);
  w.n1 = w.seq ? a.T : chunk_lo(a, w.p + 1);
  return true;
}

}  // namespace

// Orders 1 .. 32, all in registers.  The products of a sample read outputs known when the sample starts, so they issue
// together ahead of the dependent additions; the input is loaded kAhead samples ahead.
template <int ORDER>
__global__ void __launch_bounds__(kRegThreads) alz_lpcscan_walk_reg_kernel(Args a, int pass) {
  Walk w;
  if (!walk_of(a, pass, blockIdx.x * (long long)kRegThreads + threadIdx.x, w)) return;
  const long long s = w.s;
  double h[ORDER], nc[ORDER];
  if (pass == 0) {
#pragma unroll
    for (int j = 0; j < ORDER; ++j) h[j] = j + 1 == w.run ? 1.0 : 0.0;
  } else if (w.seq) {
    const double* hist = a.state + s * ORDER;
#pragma unroll
    for (int j = 0; j < ORDER; ++j) h[j] = hist[ORDER - 1 - j];
  } else {
    const double* sp = a.st + (s * (a.P + 1) + w.p) * ORDER;
#pragma unroll
    for (int j = 0; j < ORDER; ++j) h[j] = sp[j];
  }
  const bool in = w.run == 0;
  const long long n0 = w.n0, n1 = w.n1;
  const long long row = (a.C + n0) / a.hop;
  const double* c = a.coef + s * a.ccs + (row - a.r0) * a.crs;
  long long row_end = (row + 1) * a.hop - a.C;   // first sample of the next row
#pragma unroll
  for (int k = 0; k < ORDER; ++k) nc[k] = -__ldg(c + k + 1);
  double q[kAhead];                              // samples n .. n + kAhead - 1 (the input run only)
#pragma unroll
  for (int i = 0; i < kAhead; ++i) q[i] = in && n0 + i < n1 ? load_x(a, s, n0 + i) : 0.0;
  for (long long n = n0; n < n1; ++n) {
    const double x0 = q[0];
#pragma unroll
    for (int i = 0; i + 1 < kAhead; ++i) q[i] = q[i + 1];
    const long long nn = n + kAhead;
    q[kAhead - 1] = in && nn < n1 ? load_x(a, s, nn) : 0.0;
    if (n == row_end) {
      c += a.crs;
      row_end += a.hop;
#pragma unroll
      for (int k = 0; k < ORDER; ++k) nc[k] = -__ldg(c + k + 1);
    }
    double pr[ORDER];
#pragma unroll
    for (int k = 0; k < ORDER; ++k) pr[k] = __dmul_rn(nc[k], h[k]);
    double acc = x0;
#pragma unroll
    for (int k = 0; k < ORDER; ++k) acc = __dadd_rn(acc, pr[k]);
#pragma unroll
    for (int j = ORDER - 1; j > 0; --j) h[j] = h[j - 1];
    h[0] = acc;
    if (pass == 1) store_y(a, s, n, acc);
  }
  if (pass == 0) {
    double* dst = w.run == 0 ? a.F + (s * a.P + w.p) * ORDER
                             : a.M + ((s * a.P + w.p) * ORDER + (w.run - 1)) * ORDER;
#pragma unroll
    for (int j = 0; j < ORDER; ++j) dst[j] = h[j];
  } else if (w.seq || w.p == a.P - 1) {
    double* hist = a.state + s * ORDER;
#pragma unroll
    for (int j = 0; j < ORDER; ++j) hist[ORDER - 1 - j] = h[j];
  }
}

// Orders 0 and 33 .. 64: the last 64 outputs in a ring in shared memory (output n at slot n & 63) and the row's
// negated taps, copied once per row, one column per thread; the taps are walked in runs of 8.
__global__ void __launch_bounds__(kSmemThreads) alz_lpcscan_walk_kernel(Args a, int pass) {
  __shared__ double s_ring[kRing * kSmemThreads];
  __shared__ double s_nc[kRing * kSmemThreads];
  Walk w;
  if (!walk_of(a, pass, blockIdx.x * (long long)kSmemThreads + threadIdx.x, w)) return;
  const long long s = w.s;
  const int order = a.order;
  double* ring = s_ring + threadIdx.x;
  double* nc = s_nc + threadIdx.x;
  const long long n0 = w.n0, n1 = w.n1;
  for (int j = 0; j < order; ++j) {              // y[n0 - 1 - j]
    double v;
    if (pass == 0) v = j + 1 == w.run ? 1.0 : 0.0;
    else if (w.seq) v = a.state[s * order + order - 1 - j];
    else v = a.st[(s * (a.P + 1) + w.p) * order + j];
    ring[((n0 - 1 - j) & (kRing - 1)) * kSmemThreads] = v;
  }
  const bool in = w.run == 0;
  const long long row = (a.C + n0) / a.hop;
  const double* c = a.coef + s * a.ccs + (row - a.r0) * a.crs;
  long long row_end = (row + 1) * a.hop - a.C;
  for (int k = 1; k <= order; ++k) nc[(k - 1) * kSmemThreads] = -__ldg(c + k);
  double xn = in && n0 < n1 ? load_x(a, s, n0) : 0.0;
  for (long long n = n0; n < n1; ++n) {
    const double x0 = xn;
    if (in && n + 1 < n1) xn = load_x(a, s, n + 1);
    if (n == row_end) {
      c += a.crs;
      row_end += a.hop;
      for (int k = 1; k <= order; ++k) nc[(k - 1) * kSmemThreads] = -__ldg(c + k);
    }
    const int slot = (int)(n & (kRing - 1));
    double acc = x0;
    int k = 1;
    for (; k + 7 <= order; k += 8) {
      double pr[8];
#pragma unroll
      for (int u = 0; u < 8; ++u)
        pr[u] = __dmul_rn(nc[(k + u - 1) * kSmemThreads], ring[((slot - k - u) & (kRing - 1)) * kSmemThreads]);
#pragma unroll
      for (int u = 0; u < 8; ++u) acc = __dadd_rn(acc, pr[u]);
    }
    for (; k <= order; ++k)
      acc = __dadd_rn(acc, __dmul_rn(nc[(k - 1) * kSmemThreads], ring[((slot - k) & (kRing - 1)) * kSmemThreads]));
    ring[slot * kSmemThreads] = acc;
    if (pass == 1) store_y(a, s, n, acc);
  }
  if (pass == 0) {
    double* dst = w.run == 0 ? a.F + (s * a.P + w.p) * order : a.M + ((s * a.P + w.p) * order + (w.run - 1)) * order;
    for (int j = 0; j < order; ++j) dst[j] = ring[((n1 - 1 - j) & (kRing - 1)) * kSmemThreads];
  } else if (w.seq || w.p == a.P - 1) {
    for (int j = 0; j < order; ++j)
      a.state[s * order + order - 1 - j] = ring[((n1 - 1 - j) & (kRing - 1)) * kSmemThreads];
  }
}

// s_0 = the call's state, s_{p+1} = F_p + M_p s_p; flag[s] = 1 when any s_p is not finite.
__global__ void __launch_bounds__(32 * kScanWarps) alz_lpcscan_scan_kernel(Args a) {
  const long long s = blockIdx.x * (long long)kScanWarps + threadIdx.x / 32;
  if (s >= a.S) return;
  const int lane = threadIdx.x & 31, order = a.order;
  const int i0 = lane, i1 = lane + 32;
  const bool has0 = i0 < order, has1 = i1 < order;
  const double* hist = a.state + s * order;
  double v0 = has0 ? hist[order - 1 - i0] : 0.0, v1 = has1 ? hist[order - 1 - i1] : 0.0;
  double* st = a.st + s * (a.P + 1) * order;
  if (has0) st[i0] = v0;
  if (has1) st[i1] = v1;
  bool bad = !isfinite(v0) || !isfinite(v1);
  for (long long p = 0; p < a.P; ++p) {
    const double* Fp = a.F + (s * a.P + p) * order;
    const double* Mp = a.M + (s * a.P + p) * order * order;
    double acc0 = has0 ? Fp[i0] : 0.0, acc1 = has1 ? Fp[i1] : 0.0;
    for (int jb = 0; jb < order; jb += 32) {     // columns jb .. jb + 31
      double m0[32], m1[32];
#pragma unroll
      for (int u = 0; u < 32; ++u) {
        const int j = jb + u;
        m0[u] = has0 && j < order ? Mp[j * order + i0] : 0.0;
        m1[u] = has1 && j < order ? Mp[j * order + i1] : 0.0;
      }
      const double vj = jb == 0 ? v0 : v1;     // component jb + lane of s_p
#pragma unroll
      for (int u = 0; u < 32; ++u) {
        const double sj = __shfl_sync(0xffffffffu, vj, u);
        acc0 = fma(m0[u], sj, acc0);
        acc1 = fma(m1[u], sj, acc1);
      }
    }
    v0 = acc0;
    v1 = acc1;
    bad |= !isfinite(v0) || !isfinite(v1);
    if (has0) st[(p + 1) * order + i0] = v0;
    if (has1) st[(p + 1) * order + i1] = v1;
  }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) a.flag[s] = bad ? 1 : 0;
}

namespace {

using RegKernel = void (*)(Args, int);

template <int... O>
constexpr std::array<RegKernel, sizeof...(O)> reg_kernels(std::integer_sequence<int, O...>) {
  return {&alz_lpcscan_walk_reg_kernel<O + 1>...};
}

// alz_lpcscan_walk_reg_kernel<order> for order 1 .. kRegMax, at [order - 1]
const std::array<RegKernel, kRegMax> kRegKernels = reg_kernels(std::make_integer_sequence<int, kRegMax>());

cudaError_t launch_walk(const Args& a, int pass, cudaStream_t cs) {
  const long long n = a.S * a.P * (pass == 0 ? a.order + 1 : 1);
  if (a.order >= 1 && a.order <= kRegMax) {
    kRegKernels[a.order - 1]<<<(unsigned)((n + kRegThreads - 1) / kRegThreads), kRegThreads, 0, cs>>>(a, pass);
  } else {
    alz_lpcscan_walk_kernel<<<(unsigned)((n + kSmemThreads - 1) / kSmemThreads), kSmemThreads, 0, cs>>>(a, pass);
  }
  return cudaGetLastError();
}

bool bad_dtype(int32_t t) { return t != ALZ_LPCSCAN_FLOAT32 && t != ALZ_LPCSCAN_FLOAT64; }

long long elem_bytes(int32_t t) { return t == ALZ_LPCSCAN_FLOAT64 ? 8 : 4; }

long long rows(long long consumed, long long n_samples, long long hop) {
  return n_samples > 0 ? (consumed + n_samples - 1) / hop - consumed / hop + 1 : 0;
}

long long max_chunks(long long n_samples, int order) {
  const long long m = n_samples / (order > 1 ? order : 1);
  return m > 1 ? m : 1;
}

// --- the cost model ---------------------------------------------------------------------------------------------
// Times in seconds, from the shape alone.  A walk is bound by its dependent chain: `order` additions per sample at
// kDep each, plus a tap reload per row, and by the card's FP64 issue rate over all walks (kOps, below the data sheet's
// 1.67e13 instructions/s).  On the H100 the sequential synthesis takes about 11 ns per addition; the chunk walks take
// 16 (summaries) to 32 ns (rerun: a warp's 32 threads load and store 32 distinct lines per sample), kDepChunk.
// Walks beyond the threads resident at once run in waves.  A scan step is an L2 round trip for its block of M_p plus a shuffle and
// a dependent fma per column.  The model is meant to tell "pays by far" from "does not", not to predict a time.
constexpr double kDep = 11e-9;
constexpr double kDepChunk = 24e-9;
constexpr double kRow = 0.3e-6;
constexpr double kOps = 1.2e13;
constexpr double kStep = 0.6e-6;
constexpr double kStepCol = 15e-9;
constexpr double kLaunch = 8e-6;
constexpr double kSMs = 132;
constexpr double kScratchMax = 1024.0 * 1024 * 1024;   // bytes of scratch the model may ask for

double resident_walks(int order) {             // walk threads resident at once
  if (order >= 1 && order <= kRegMax) {
    const double regs = 52 + 4.0 * order;        // registers per thread (ptxas: 117 at order 16, 182 at 32)
    const double per_sm = 65536.0 / regs;
    return kSMs * (per_sm < 2048 ? per_sm : 2048);
  }
  return kSMs * 7 * kSmemThreads;              // 32 KB of shared memory per 32 threads
}

double walk_time(double threads, double len, double hop, double ops, int order, double dep) {
  const double waves = std::ceil(threads / resident_walks(order));
  const double chain = (len * (order > 0 ? order : 1) * dep + std::ceil(len / hop) * kRow) * waves;
  const double issue = ops / kOps;
  return chain > issue ? chain : issue;
}

double sequential_time(double S, double T, int order, double hop) {
  return walk_time(S, T, hop, S * T * 2.0 * order, order, kDep);
}

double parallel_time(double S, double T, int order, double hop, double P) {
  const double L = std::ceil(T / P);
  const double pass0 = walk_time(S * P * (order + 1), L, hop, S * T * 2.0 * order * (order + 1), order, kDepChunk);
  const double scan = P * (kStep * std::ceil(order / 32.0) + kStepCol * order) * std::ceil(S / (kSMs * 64));
  const double pass1 = walk_time(S * P, L, hop, S * T * 2.0 * order, order, kDepChunk);
  return pass0 + scan + pass1 + 3 * kLaunch;
}

long long scratch_bytes(long long S, long long P, int order) {
  return 8 * (S * P * order * (long long)(order + 1) + S * (P + 1) * order) + 8 * ((S + 1) / 2);
}

}  // namespace

extern "C" {

const char* alz_lpcscan_last_error(void) { return g_err.c_str(); }

int64_t alz_lpcscan_chunks(int64_t n_streams, int64_t n_samples, int32_t order, int64_t hop) {
  if (n_streams < 0 || n_samples < 0) return fail(ALZ_LPCSCAN_ERR_INVALID, "need n_streams >= 0 and n_samples >= 0");
  if (order < 0 || order > ALZ_LPCSCAN_MAX_ORDER)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPCSCAN_MAX_ORDER, order);
  if (hop < 1) return fail(ALZ_LPCSCAN_ERR_INVALID, "hop must be >= 1 (got %lld)", (long long)hop);
  if (order == 0 || n_streams == 0 || n_samples == 0) return 1;
  const double S = (double)n_streams, T = (double)n_samples, H = (double)hop;
  const double seq = sequential_time(S, T, order, H);
  const long long top = max_chunks(n_samples, order);
  long long best = 1;
  double best_t = seq;
  for (double Pd = 2; Pd <= (double)top; Pd = std::ceil(Pd * 1.1)) {
    const long long P = (long long)Pd;
    if ((double)scratch_bytes(n_streams, P, order) > kScratchMax || S * Pd * (order + 1) > 4e9) break;
    const double t = parallel_time(S, T, order, H, Pd);
    if (t < best_t) best = P, best_t = t;
  }
  return best_t <= 0.5 * seq ? best : 1;
}

int64_t alz_lpcscan_scratch_bytes(int64_t n_streams, int64_t n_chunks, int32_t order) {
  if (n_streams < 0 || n_chunks < 1) return fail(ALZ_LPCSCAN_ERR_INVALID, "need n_streams >= 0 and n_chunks >= 1");
  if (order < 0 || order > ALZ_LPCSCAN_MAX_ORDER)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPCSCAN_MAX_ORDER, order);
  if ((double)n_streams * (double)n_chunks * (order + 1) * (order + 2) > 1e17)
    return fail(ALZ_LPCSCAN_ERR_UNSUPPORTED, "scratch too large");
  return scratch_bytes(n_streams, n_chunks, order);
}

int32_t alz_lpcscan_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                          int64_t out_stride, const double* coef_dev, int64_t coef_row_stride,
                          int64_t coef_stream_stride, int64_t n_rows, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int64_t consumed, int32_t order, int64_t hop, int64_t n_chunks,
                          void* scratch_dev, int64_t scratch_bytes_given, void* cuda_stream) {
  if (order < 0 || order > ALZ_LPCSCAN_MAX_ORDER)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPCSCAN_MAX_ORDER, order);
  if (hop < 1) return fail(ALZ_LPCSCAN_ERR_INVALID, "hop must be >= 1 (got %lld)", (long long)hop);
  if (n_streams < 0 || n_samples < 0 || consumed < 0)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "bad shape: n_streams %lld, n_samples %lld, consumed %lld",
                (long long)n_streams, (long long)n_samples, (long long)consumed);
  if (bad_dtype(x_dtype) || bad_dtype(out_dtype))
    return fail(ALZ_LPCSCAN_ERR_INVALID, "dtype must be ALZ_LPCSCAN_FLOAT32 or _FLOAT64");
  if (n_chunks < 1 || n_chunks > max_chunks(n_samples, order))
    return fail(ALZ_LPCSCAN_ERR_INVALID, "n_chunks must be in 1 .. %lld for %lld samples at order %d (got %lld)",
                max_chunks(n_samples, order), (long long)n_samples, order, (long long)n_chunks);
  const long long need = rows(consumed, n_samples, hop);
  if (n_rows < need)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "coef holds %lld rows per stream, the call needs %lld", (long long)n_rows,
                need);
  if (n_streams == 0 || n_samples == 0) return ALZ_LPCSCAN_OK;
  const int64_t nbytes = alz_lpcscan_scratch_bytes(n_streams, n_chunks, order);
  if (nbytes < 0) return (int32_t)nbytes;
  if (scratch_bytes_given < nbytes)
    return fail(ALZ_LPCSCAN_ERR_INVALID, "scratch holds %lld bytes, the call needs %lld", (long long)scratch_bytes_given,
                (long long)nbytes);
  if (!x_dev || !out_dev || !coef_dev || !scratch_dev || (order > 0 && !state_dev))
    return fail(ALZ_LPCSCAN_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev % elem_bytes(x_dtype)) || ((uintptr_t)out_dev % elem_bytes(out_dtype)) ||
      ((uintptr_t)coef_dev & 7) || ((uintptr_t)state_dev & 7) || ((uintptr_t)scratch_dev & 7))
    return fail(ALZ_LPCSCAN_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && (x_stride < n_samples || out_stride < n_samples))
    return fail(ALZ_LPCSCAN_ERR_INVALID, "stride < n_samples");
  if (need > 1 && coef_row_stride < order + 1) return fail(ALZ_LPCSCAN_ERR_INVALID, "coef row stride < order + 1");
  if (coef_stream_stride < 0) return fail(ALZ_LPCSCAN_ERR_INVALID, "coef stream stride < 0");
  const long long walks = n_streams * n_chunks * (order + 1);
  if ((walks + kSmemThreads - 1) / kSmemThreads > 0x7fffffffLL || (n_streams + kScanWarps - 1) / kScanWarps > 0x7fffffffLL)
    return fail(ALZ_LPCSCAN_ERR_UNSUPPORTED, "too many walks for one launch");
  Args a{};
  a.x = x_dev;
  a.out = out_dev;
  a.coef = coef_dev;
  a.state = (double*)state_dev;
  double* scratch = (double*)scratch_dev;
  a.F = scratch;
  a.M = a.F + n_streams * n_chunks * order;
  a.st = a.M + n_streams * n_chunks * order * order;
  a.flag = (int*)(a.st + n_streams * (n_chunks + 1) * order);
  a.xs = n_streams > 1 ? x_stride : n_samples;
  a.os = n_streams > 1 ? out_stride : n_samples;
  a.crs = coef_row_stride;
  a.ccs = coef_stream_stride;
  a.S = n_streams;
  a.T = n_samples;
  a.C = consumed;
  a.hop = hop;
  a.r0 = consumed / hop;
  a.P = n_chunks;
  a.order = order;
  a.x64 = x_dtype == ALZ_LPCSCAN_FLOAT64;
  a.out64 = out_dtype == ALZ_LPCSCAN_FLOAT64;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  ALZ_CUDA_CHECK(launch_walk(a, 0, cs), ALZ_LPCSCAN_ERR_CUDA);
  alz_lpcscan_scan_kernel<<<(unsigned)((n_streams + kScanWarps - 1) / kScanWarps), 32 * kScanWarps, 0, cs>>>(a);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPCSCAN_ERR_CUDA);
  ALZ_CUDA_CHECK(launch_walk(a, 1, cs), ALZ_LPCSCAN_ERR_CUDA);
  return ALZ_LPCSCAN_OK;
}

}  // extern "C"
