// alz_common.h -- host plumbing, block arithmetic and the compensated sum shared by the analysis libraries.
//
// Everything here is in an unnamed namespace: each library's unit gets its own copy, so the message a library's
// *_last_error() returns is that library's own last failure.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <string>

namespace {

thread_local std::string g_err;

// Records the message for the library's *_last_error() and returns `code`.
inline int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}

// Returns fail(code, ...) from the enclosing function when a CUDA runtime call fails.
#define ALZ_CUDA_CHECK(call, code)                                                         \
  do {                                                                                     \
    cudaError_t e_ = (call);                                                               \
    if (e_ != cudaSuccess) return fail((code), "%s: %s", #call, cudaGetErrorString(e_));   \
  } while (0)

__host__ __device__ inline long long floordiv(long long a, long long b) {   // b > 0
  return a >= 0 ? a / b : -((-a + b - 1) / b);
}

// Blocks are [k hop, k hop + size) for k = 0, 1, ...: the first block that is still open after n samples.
__host__ __device__ inline long long first_open_block(long long n, int size, int hop) {   // first k with k hop + size > n
  const long long k = floordiv(n - size, hop) + 1;
  return k > 0 ? k : 0;
}

// Blocks a call on n_samples samples emits after `consumed`: the ones it completes, plus, when it is the final call,
// the padded last block when the reference's Stream.blocks emits one.
inline long long emitted_blocks(long long consumed, long long n_samples, int size, int hop, bool final) {
  const long long ka = first_open_block(consumed, size, hop);
  const long long kc = floordiv(consumed + n_samples - size, hop);
  long long n = kc - ka + 1 > 0 ? kc - ka + 1 : 0;
  const long long kp = kc + 1 > 0 ? kc + 1 : 0;
  if (final && consumed + n_samples - kp * hop > (size > hop ? size - hop : 0)) ++n;
  return n;
}

// Running compensated sum: CPython 3.12's sum() of floats (Neumaier), started from 0.0 and compensated from the first
// term on, which gives the same value (see alz_lpc.cu).  The units that use it are compiled with -fmad=false.
struct Psum {
  double f = 0.0, c = 0.0;
  __device__ __forceinline__ void add(double x) {
    const double t = __dadd_rn(f, x);
    const bool big = fabs(f) >= fabs(x);
    const double hi = big ? f : x, lo = big ? x : f;
    c = __dadd_rn(c, __dadd_rn(__dsub_rn(hi, t), lo));
    f = t;
  }
  __device__ __forceinline__ double value() const { return (c != 0.0 && isfinite(c)) ? __dadd_rn(f, c) : f; }
};

}  // namespace
