// alz_lpc.cu -- the C ABI of include/alz_b200_lpc.h: frame-wise LPC of S streams on sm_90a.
//
// Three kernels per call, in stream order:
//   * alz_lpc_kernel: the autocorrelation.  A CTA stages the float64 values b[n] of up to kMaxFramesPerCta frames of
//     one stream in shared memory (samples before the call come from the state's last `size` samples), then each
//     thread owns one (frame, lag) pair and runs that lag's compensated sum sequentially in n order;
//   * alz_lpc_levinson_kernel: one thread per frame runs the recursion of the header, its lags and coefficients kept
//     in shared memory ([k][thread], so that a warp's accesses are consecutive); skipped for an acorr-only call;
//   * alz_lpc_commit_kernel: one CTA per stream shifts the last `size` samples into the state and counts the samples.
//
// The header's psum is CPython 3.12's sum() of floats.  Starting from f = 0.0 and compensating from the first term on
// is the same thing: the first term's compensation is 0, or NaN when it is infinite or NaN, and then f is no longer
// finite, so the compensation is never added.  The unit is compiled with -fmad=false and the arithmetic spelled with
// __dmul_rn / __dadd_rn / __dsub_rn, so nothing is contracted or reassociated.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_lpc.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace {

constexpr int kMaxFramesPerCta = 8;
constexpr int kThreadsAcorr = 128;          // target (frame, lag) pairs per CTA
constexpr int kSmemBudget = 48 * 1024;      // staging budget per CTA; one frame of a larger size opts in above it
constexpr int kThreadsCommit = 256;

struct LpcArgs {
  const float* x;
  const double* w;
  double* r;            // lags: acorr_dev, or the scratch
  double* coef;
  double* err;
  uint8_t* failed;
  unsigned char* state;
  long long xs, sstride, T, F;
  int order, size, hop, final_, fpc, blocks_per_stream;
};

long long state_stride(int size) { return (16 + 4 * (long long)size + 7) / 8 * 8; }

// Running compensated sum (the header's psum).
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

int frames_per_cta(int order, int size) {
  int fpc = kThreadsAcorr / (order + 1);
  const int by_smem = kSmemBudget / (8 * (size + 1));
  if (by_smem < fpc) fpc = by_smem;
  if (fpc > kMaxFramesPerCta) fpc = kMaxFramesPerCta;
  return fpc < 1 ? 1 : fpc;
}

int levinson_threads(int order) {
  int n = 128;
  while (n > 32 && 2 * 8 * (order + 1) * n > kSmemBudget) n /= 2;
  return n;
}

}  // namespace

// The lags of fpc consecutive frames of one stream per CTA (see the file comment).
__global__ void __launch_bounds__(kMaxFramesPerCta * 32) alz_lpc_kernel(const __grid_constant__ LpcArgs a) {
  extern __shared__ double s_b[];              // [fpc][size + 1]
  const long long s = blockIdx.x / a.blocks_per_stream;
  const long long i0 = (long long)(blockIdx.x % a.blocks_per_stream) * a.fpc;
  const unsigned char* st = a.state + s * a.sstride;
  const long long C = *reinterpret_cast<const long long*>(st);
  const float* tail = reinterpret_cast<const float*>(st + 16);    // samples [C - size, C)
  const float* xr = a.x + s * a.xs;
  const long long ka = first_open_block(C, a.size, a.hop);
  const int size = a.size, ld = size + 1;
  const int nf = (int)(a.F - i0 < a.fpc ? a.F - i0 : a.fpc);

  for (int e = threadIdx.x; e < nf * size; e += blockDim.x) {
    const int f = e / size, n = e - f * size;
    const long long g = (ka + i0 + f) * a.hop + n;                  // stream sample index
    float v = 0.f;
    if (g < C) {
      v = tail[g - (C - size)];
    } else if (g < C + a.T) {
      v = xr[g - C];
    }
    s_b[f * ld + n] = a.w ? __dmul_rn((double)v, a.w[n]) : (double)v;
  }
  __syncthreads();

  const int L = a.order + 1;
  const int f = threadIdx.x / L, tau = threadIdx.x - f * L;
  if (f >= nf) return;
  const double* b = s_b + f * ld;
  Psum acc;
  for (int n = 0; n + tau < size; ++n) acc.add(__dmul_rn(b[n], b[n + tau]));
  a.r[((s * a.F) + i0 + f) * L + tau] = acc.value();
}

// One frame per thread: the Levinson-Durbin recursion of the header.
__global__ void __launch_bounds__(128) alz_lpc_levinson_kernel(const __grid_constant__ LpcArgs a, long long n_frames) {
  extern __shared__ double s_m[];              // [order + 1][nt] lags, then [order + 1][nt] coefficients
  const int nt = blockDim.x, tid = threadIdx.x;
  const long long g = (long long)blockIdx.x * nt + tid;
  if (g >= n_frames) return;
  const int order = a.order, L = order + 1;
  double* R = s_m + tid;
  double* A = s_m + (long long)L * nt + tid;
#define RR(k) R[(k) * nt]
#define AA(k) A[(k) * nt]
  const double* rg = a.r + g * L;
  for (int k = 0; k < L; ++k) RR(k) = rg[k];
  AA(0) = 1.0;
  int hi = 0;                                  // last coefficient that is not zero
  bool failed = false;
  for (int m = 1; m <= order; ++m) {
    // den = inner(B, B), B[j] = j ? A[m - j] : 0
    Psum den;
    for (int i = 0; i <= m; ++i) {
      const double bi = i ? AA(m - i) : 0.0;
      for (int j = 0; j <= m; ++j) {
        const double bj = j ? AA(m - j) : 0.0;
        den.add(__dmul_rn(__dmul_rn(RR(i > j ? i - j : j - i), bi), bj));
      }
    }
    const double d = den.value();
    if (d == 0.0) {
      failed = true;
      break;
    }
    // num = inner(A', Z), Z[j] = j == m
    Psum num;
    for (int i = 0; i <= hi; ++i) {
      const double ai = AA(i);
      for (int j = 0; j <= m; ++j) num.add(__dmul_rn(__dmul_rn(RR(i > j ? i - j : j - i), ai), j == m ? 1.0 : 0.0));
    }
    const double c = __ddiv_rn(num.value(), d);
    AA(m) = 0.0;
    if (c != 0.0) {
      // A[k] -= c B[k] with B[k] = A[m - k] (old values, so the pair (k, m - k) is updated together); B[0] = 0
      for (int k = 0; 2 * k <= m; ++k) {
        const double ak = AA(k), amk = AA(m - k);
        const double bk = k ? amk : 0.0, bmk = ak;            // B[k], B[m - k] (m - k >= 1)
        double nk = ak, nmk = amk;
        if (bk != 0.0) {
          const double p = __dmul_rn(c, bk);
          if (p != 0.0) {
            const double v = __dsub_rn(ak, p);
            nk = v != 0.0 ? v : 0.0;
          }
        }
        if (bmk != 0.0) {
          const double p = __dmul_rn(c, bmk);
          if (p != 0.0) {
            const double v = __dsub_rn(amk, p);
            nmk = v != 0.0 ? v : 0.0;
          }
        }
        if (2 * k == m) {
          AA(k) = nk;
        } else {
          AA(k) = nk;
          AA(m - k) = nmk;
        }
      }
    }
    hi = 0;
    for (int k = m; k > 0; --k)
      if (AA(k) != 0.0) {
        hi = k;
        break;
      }
  }
  if (a.coef) {
    double* cg = a.coef + g * L;
    for (int k = 0; k < L; ++k) cg[k] = failed ? NAN : AA(k);
  }
  if (a.err) {
    double e = NAN;
    if (!failed) {
      Psum acc;
      for (int i = 0; i <= hi; ++i) {
        const double ai = AA(i);
        for (int j = 0; j <= hi; ++j) acc.add(__dmul_rn(__dmul_rn(RR(i > j ? i - j : j - i), ai), AA(j)));
      }
      e = acc.value();
    }
    a.err[g] = e;
  }
  if (a.failed) a.failed[g] = failed ? 1 : 0;
#undef RR
#undef AA
}

// After a call's frames: per stream (one CTA), the last `size` samples and the sample count.
__global__ void __launch_bounds__(kThreadsCommit) alz_lpc_commit_kernel(const __grid_constant__ LpcArgs a) {
  extern __shared__ float s_t[];
  const long long s = blockIdx.x;
  unsigned char* st = a.state + s * a.sstride;
  const long long C = *reinterpret_cast<const long long*>(st), C1 = C + a.T;
  float* tail = reinterpret_cast<float*>(st + 16);
  const float* xr = a.x + s * a.xs;
  for (int j = threadIdx.x; j < a.size; j += blockDim.x) {
    const long long g = C1 - a.size + j;
    s_t[j] = g >= C ? xr[g - C] : (g >= C - a.size ? tail[g - (C - a.size)] : 0.f);
  }
  __syncthreads();
  for (int j = threadIdx.x; j < a.size; j += blockDim.x) tail[j] = s_t[j];
  if (threadIdx.x == 0) *reinterpret_cast<long long*>(st) = C1;
}

__global__ void __launch_bounds__(kThreadsCommit) alz_lpc_init_kernel(unsigned char* state, long long n_words) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_words; i += (long long)gridDim.x * blockDim.x)
    reinterpret_cast<int*>(state)[i] = 0;
}

extern "C" {

const char* alz_lpc_last_error(void) { return g_err.c_str(); }

int64_t alz_lpc_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final) {
  if (consumed < 0 || n_samples < 0 || size < 1 || hop < 1)
    return fail(ALZ_LPC_ERR_INVALID, "need consumed >= 0, n_samples >= 0, size >= 1, hop >= 1");
  return emitted_blocks(consumed, n_samples, size, hop, final != 0);
}

int64_t alz_lpc_state_bytes(int64_t n_streams, int32_t size) {
  if (n_streams < 0 || size < 1 || size > ALZ_LPC_MAX_SIZE)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_LPC_MAX_SIZE);
  return n_streams * state_stride(size);
}

int32_t alz_lpc_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream) {
  if (n_streams < 0 || size < 1 || size > ALZ_LPC_MAX_SIZE)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_LPC_MAX_SIZE);
  if (n_streams == 0) return ALZ_LPC_OK;
  if (!state_dev || ((uintptr_t)state_dev & 7)) return fail(ALZ_LPC_ERR_INVALID, "state is NULL or not 8-byte aligned");
  const long long n = n_streams * (state_stride(size) / 4);
  const unsigned blocks = (unsigned)((n + kThreadsCommit - 1) / kThreadsCommit < 4096 ? (n + kThreadsCommit - 1) / kThreadsCommit : 4096);
  alz_lpc_init_kernel<<<blocks, kThreadsCommit, 0, (cudaStream_t)cuda_stream>>>((unsigned char*)state_dev, n);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
  return ALZ_LPC_OK;
}

int64_t alz_lpc_scratch_bytes(int64_t n_streams, int64_t n_frames, int32_t order) {
  if (n_streams < 0 || n_frames < 0 || order < 0 || order > ALZ_LPC_MAX_ORDER)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0, n_frames >= 0 and 0 <= order <= %d", ALZ_LPC_MAX_ORDER);
  return n_streams * n_frames * (order + 1) * 8;
}

int32_t alz_lpc_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, double* acorr_dev,
                          double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames, void* state_dev,
                          int64_t n_streams, int64_t n_samples, int32_t order, int32_t size, int32_t hop, int32_t final,
                          void* scratch_dev, int64_t scratch_bytes, void* cuda_stream) {
  if (order < 0 || order > ALZ_LPC_MAX_ORDER)
    return fail(ALZ_LPC_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPC_MAX_ORDER, order);
  if (size < 1 || size > ALZ_LPC_MAX_SIZE)
    return fail(ALZ_LPC_ERR_INVALID, "size must be in 1 .. %d (got %d)", ALZ_LPC_MAX_SIZE, size);
  if (hop < 1) return fail(ALZ_LPC_ERR_INVALID, "hop must be >= 1 (got %d)", hop);
  if (n_streams < 0 || n_samples < 0 || n_frames < 0) return fail(ALZ_LPC_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_LPC_OK;
  if (!state_dev || (n_samples > 0 && !x_dev)) return fail(ALZ_LPC_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev & 3) || ((uintptr_t)state_dev & 7) || ((uintptr_t)window_dev & 7))
    return fail(ALZ_LPC_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_LPC_ERR_INVALID, "stride < n_samples");
  const bool levinson = coef_dev || error_dev || failed_dev;
  double* r = acorr_dev;
  if (!r && levinson) {
    if (!scratch_dev || scratch_bytes < alz_lpc_scratch_bytes(n_streams, n_frames, order))
      return fail(ALZ_LPC_ERR_INVALID, "scratch of %lld bytes, %lld needed", (long long)scratch_bytes,
                  (long long)alz_lpc_scratch_bytes(n_streams, n_frames, order));
    if ((uintptr_t)scratch_dev & 7) return fail(ALZ_LPC_ERR_INVALID, "misaligned scratch");
    r = (double*)scratch_dev;
  }
  LpcArgs a{};
  a.x = x_dev;
  a.w = window_dev;
  a.r = r;
  a.coef = coef_dev;
  a.err = error_dev;
  a.failed = failed_dev;
  a.state = (unsigned char*)state_dev;
  a.xs = x_stride;
  a.sstride = state_stride(size);
  a.T = n_samples;
  a.F = n_frames;
  a.order = order;
  a.size = size;
  a.hop = hop;
  a.final_ = final != 0;
  a.fpc = frames_per_cta(order, size);
  a.blocks_per_stream = (int)((n_frames + a.fpc - 1) / a.fpc);
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  if (n_frames > 0 && r) {
    const long long grid = n_streams * a.blocks_per_stream;
    if (grid > 0x7fffffffLL || n_frames > 0x7fffffffLL) return fail(ALZ_LPC_ERR_UNSUPPORTED, "too many frames for one launch");
    const int threads = (a.fpc * (order + 1) + 31) / 32 * 32;
    const size_t smem = (size_t)a.fpc * (size + 1) * 8;
    if (smem > 48 * 1024)
      ALZ_CUDA_CHECK(cudaFuncSetAttribute(alz_lpc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem),
                     ALZ_LPC_ERR_CUDA);
    alz_lpc_kernel<<<(unsigned)grid, threads, smem, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
    if (levinson) {
      const long long total = n_streams * n_frames;
      const int nt = levinson_threads(order);
      const long long blocks = (total + nt - 1) / nt;
      if (blocks > 0x7fffffffLL) return fail(ALZ_LPC_ERR_UNSUPPORTED, "too many frames for one launch");
      alz_lpc_levinson_kernel<<<(unsigned)blocks, nt, (size_t)2 * 8 * (order + 1) * nt, cs>>>(a, total);
      ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
    }
  }
  if (n_samples > 0) {
    alz_lpc_commit_kernel<<<(unsigned)n_streams, kThreadsCommit, (size_t)4 * size, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
  }
  return ALZ_LPC_OK;
}

}  // extern "C"
