// alz_common.h -- host plumbing, block arithmetic, the compensated sum and the carried-sample states shared by the
// analysis libraries.
//
// Everything here is in an unnamed namespace: each library's unit gets its own copy, so the message a library's
// *_last_error() returns is that library's own last failure.  The device functions are called from each library's own
// kernels, which keeps every kernel under its library's name.
#pragma once

#include <cuda_runtime.h>

#include <cstdarg>
#include <cstdio>
#include <mutex>
#include <set>
#include <string>
#include <utility>

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

// A kernel's dynamic shared-memory limit is an attribute of the function, shared by every caller and host thread.  It
// is raised once per (kernel, device) to the device's opt-in maximum and never set to one launch's size, which would
// make a concurrent launch that needs more fail; each launch asks for its own size.  Launches of at most the default
// 48 KB need nothing.
inline cudaError_t allow_dynamic_smem(const void* kernel, size_t bytes) {
  if (bytes <= 48 * 1024) return cudaSuccess;
  static std::mutex mu;
  static std::set<std::pair<const void*, int>> done;
  int dev = -1;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  std::lock_guard<std::mutex> lock(mu);
  if (done.count({kernel, dev})) return cudaSuccess;
  int max_smem = 0;
  cudaFuncAttributes fa;
  e = cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&fa, kernel);
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem - (int)fa.sharedSizeBytes);
  if (e == cudaSuccess) done.insert({kernel, dev});
  return e;
}

// The framed-sample state of the LPC and STFT analyses, per stream: the int64 count C of samples seen, then from byte
// 16 the last `size` of them as float32 (samples [C - size, C); zeros before the stream's first sample).  Every byte
// of a new state is zero.
inline long long framed_state_stride(int size) { return (16 + 4 * (long long)size + 7) / 8 * 8; }

// One stream's samples in a call on x[0, T): the state's tail, then the block, then zeros.
struct FramedSamples {
  const float* tail;   // samples [C - size, C)
  long long C;
  const float* x;      // samples [C, C + T)
  long long T;
  int size;

  // stream sample g, for g >= C - size
  __device__ __forceinline__ float operator()(long long g) const {
    if (g < C) return tail[g - (C - size)];
    if (g < C + T) return x[g - C];
    return 0.f;
  }
};

__device__ __forceinline__ FramedSamples framed_samples(const unsigned char* st, const float* x, long long T, int size) {
  return {reinterpret_cast<const float*>(st + 16), *reinterpret_cast<const long long*>(st), x, T, size};
}

// After a call on x[0, T): the last `size` samples become the tail and the count advances.  One CTA per stream; s_t
// is `size` floats of shared memory.
__device__ __forceinline__ void framed_commit(unsigned char* st, const float* x, long long T, int size, float* s_t) {
  const FramedSamples in = framed_samples(st, x, T, size);
  for (int j = threadIdx.x; j < size; j += blockDim.x) s_t[j] = in(in.C + T - size + j);
  __syncthreads();
  float* tail = reinterpret_cast<float*>(st + 16);
  for (int j = threadIdx.x; j < size; j += blockDim.x) tail[j] = s_t[j];
  if (threadIdx.x == 0) *reinterpret_cast<long long*>(st) = in.C + T;
}

// The float64 history hist[0, H) becomes the last H samples of (history, x[0, T)).  In place, ascending: new[i] reads
// old[i + T], which no earlier pass has written.  Every thread of the CTA calls it.
__device__ __forceinline__ void shift_history(double* hist, long long H, const float* x, long long T) {
  for (long long i0 = 0; i0 < H; i0 += blockDim.x) {
    const long long i = i0 + threadIdx.x, p = T - H + i;
    double v = 0.0;
    if (i < H) v = p >= 0 ? (double)x[p] : hist[i + T];
    __syncthreads();
    if (i < H) hist[i] = v;
    __syncthreads();
  }
}

}  // namespace
