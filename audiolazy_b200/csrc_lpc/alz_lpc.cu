// alz_lpc.cu -- the C ABI of include/alz_b200_lpc.h: frame-wise LPC of S streams on sm_90a.
//
// Three kernels per call, in stream order, for both methods:
//   * alz_lpc_kernel: the frame statistics.  A CTA stages the float64 values b[n] of up to kMaxFramesPerCta frames
//     of one stream in shared memory (samples before the call come from the state's last `size` samples), then each
//     statistic's compensated sum runs sequentially in n order on one thread: kautocor's thread owns one (frame,
//     lag) pair, kcovar's threads take the (frame, lag-matrix cell) pairs of the CTA in turn (order 16 has 153 cells
//     a frame).  The two sums keep loops of their own: one loop over a generic cell (b[n + u] * b[n + v] for n in
//     [n0, n1)) cost the lags 5 % on H100 (DESIGN.md section 5);
//   * alz_lpc_levinson_kernel: the recursion, chosen by the call.  kautocor: one thread per frame runs
//     Levinson-Durbin, its lags and coefficients kept in shared memory ([k][thread], so that a warp's accesses are
//     consecutive).  kcovar: one warp per frame runs the Gram-Schmidt lattice on the frame's lag matrix, its lanes
//     sharing the independent sums of a step (the m + 1 divisions and the basis update) and each running the
//     sequential ones redundantly.  Both recursions take every quotient from one division in one loop, so the
//     kernel holds a single correctly rounded division.  Skipped for a statistics-only call;
//   * alz_lpc_commit_kernel: one CTA per stream shifts the last `size` samples into the state and counts the samples.
//
// The header's psum is CPython 3.12's sum() of floats.  Starting from f = 0.0 and compensating from the first term on
// is the same thing: the first term's compensation is 0, or NaN when it is infinite or NaN, and then f is no longer
// finite, so the compensation is never added.  Adding a +-0 term leaves (f, c) as they are (f never becomes -0.0, the
// compensation gains +0), which is what lets kcovar skip the products of a zero coefficient (see the header).  The
// unit is compiled with -fmad=false and the arithmetic spelled with __dmul_rn / __dadd_rn / __dsub_rn, so nothing is
// contracted or reassociated.
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
  double* r;            // statistics: acorr_dev or the scratch (kautocor), the lag-matrix triangle scratch (kcovar)
  double* lagm;         // kcovar: the full lag matrices, or NULL
  double* coef;
  double* err;
  uint8_t* failed;
  unsigned char* state;
  long long xs, sstride, T, F;
  int order, size, hop, final_, fpc, blocks_per_stream;
  int covar;            // 0: kautocor, 1: kcovar
  int ncell;            // statistics per frame: order + 1 lags, or the (order + 1)(order + 2) / 2 cells of a triangle
};

int frames_per_cta(int ncell, int size) {
  int fpc = kThreadsAcorr / ncell;
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

long long tri_cells(int order) { return (long long)(order + 1) * (order + 2) / 2; }

// kcovar: float64 values of one frame's shared memory: the full lag matrix (order + 1)^2, the basis B[q] (q = 0 ..
// order - 1, order + 2 values each), A (order + 1), beta, gamma and max|B[q]| (order each).
__host__ __device__ inline int covar_frame_doubles(int order) {
  const int L = order + 1;
  return L * L + order * (order + 2) + L + 3 * order + 1;
}

int covar_warps(int order) {
  const int bytes = 8 * covar_frame_doubles(order);
  int w = kSmemBudget / bytes;
  return w < 1 ? 1 : (w > 4 ? 4 : w);
}

}  // namespace

// The lags of fpc consecutive frames of one stream per CTA (see the file comment).
__global__ void __launch_bounds__(kMaxFramesPerCta * 32) alz_lpc_kernel(const __grid_constant__ LpcArgs a) {
  extern __shared__ double s_b[];              // [fpc][size + 1]
  const long long s = blockIdx.x / a.blocks_per_stream;
  const long long i0 = (long long)(blockIdx.x % a.blocks_per_stream) * a.fpc;
  const FramedSamples in = framed_samples(a.state + s * a.sstride, a.x + s * a.xs, a.T, a.size);
  const long long ka = first_open_block(in.C, a.size, a.hop);
  const int size = a.size, ld = size + 1;
  const int nf = (int)(a.F - i0 < a.fpc ? a.F - i0 : a.fpc);

  for (int e = threadIdx.x; e < nf * size; e += blockDim.x) {
    const int f = e / size, n = e - f * size;
    const float v = in((ka + i0 + f) * a.hop + n);
    s_b[f * ld + n] = a.w ? __dmul_rn((double)v, a.w[n]) : (double)v;
  }
  __syncthreads();

  const int L = a.order + 1;
  if (!a.covar) {                              // one lag per thread
    const int f = threadIdx.x / L, tau = threadIdx.x - f * L;
    if (f >= nf) return;
    const double* b = s_b + f * ld;
    Psum acc;
    for (int n = 0; n + tau < size; ++n) acc.add(__dmul_rn(b[n], b[n + tau]));
    a.r[((s * a.F) + i0 + f) * L + tau] = acc.value();
    return;
  }
  // the lag-matrix cells (i, j), i <= j, at c = j (j + 1) / 2 + i, taken in turn by the CTA's threads
  const int nc = a.ncell;
  for (int e = threadIdx.x; e < nf * nc; e += blockDim.x) {
    const int f = e / nc, c = e - f * nc;
    int j = (int)((sqrtf(8.f * c + 1.f) - 1.f) * .5f);
    while (j * (j + 1) / 2 > c) --j;
    while ((j + 1) * (j + 2) / 2 <= c) ++j;
    const int i = c - j * (j + 1) / 2;
    const double* bi = s_b + f * ld + a.order - i;      // b[n - i] for n = order .. size - 1
    const double* bj = s_b + f * ld + a.order - j;
    Psum acc;
    for (int n = 0; n < size - a.order; ++n) acc.add(__dmul_rn(bi[n], bj[n]));
    const double val = acc.value();
    const long long g = s * a.F + i0 + f;
    if (a.r) a.r[g * nc + c] = val;
    if (a.lagm) {
      a.lagm[(g * L + j) * L + i] = val;
      a.lagm[(g * L + i) * L + j] = val;
    }
  }
}

namespace {

// kautocor, one frame per thread: the Levinson-Durbin recursion of the header.  next() runs the sums of step m and
// hands over (num, den) for c = num / den, or returns false when the frame is done or fails; take(c) updates A.
struct Levinson {
  double* R;                                   // lags, [k * nt]
  double* A;                                   // coefficients, [k * nt]
  int nt, order, m, hi;                        // hi: last coefficient that is not zero
  bool failed;

  __device__ __forceinline__ double& r(int k) const { return R[k * nt]; }
  __device__ __forceinline__ double& c(int k) const { return A[k * nt]; }

  __device__ __forceinline__ bool init(const LpcArgs& a, long long n_frames, double* s_m) {
    nt = blockDim.x;
    const int tid = threadIdx.x;
    const long long g = (long long)blockIdx.x * nt + tid;
    if (g >= n_frames) return false;
    order = a.order;
    const int L = order + 1;
    R = s_m + tid;
    A = s_m + (long long)L * nt + tid;
    const double* rg = a.r + g * L;
    for (int k = 0; k < L; ++k) r(k) = rg[k];
    c(0) = 1.0;
    hi = 0;
    m = 1;
    failed = false;
    return true;
  }

  __device__ __forceinline__ bool next(double& num_out, double& den_out) {
    if (m > order) return false;
    // den = inner(B, B), B[j] = j ? A[m - j] : 0
    Psum den;
    for (int i = 0; i <= m; ++i) {
      const double bi = i ? c(m - i) : 0.0;
      for (int j = 0; j <= m; ++j) {
        const double bj = j ? c(m - j) : 0.0;
        den.add(__dmul_rn(__dmul_rn(r(i > j ? i - j : j - i), bi), bj));
      }
    }
    const double d = den.value();
    if (d == 0.0) {
      failed = true;
      return false;
    }
    // num = inner(A', Z), Z[j] = j == m
    Psum num;
    for (int i = 0; i <= hi; ++i) {
      const double ai = c(i);
      for (int j = 0; j <= m; ++j) num.add(__dmul_rn(__dmul_rn(r(i > j ? i - j : j - i), ai), j == m ? 1.0 : 0.0));
    }
    num_out = num.value();
    den_out = d;
    return true;
  }

  __device__ __forceinline__ void take(double cq) {
    c(m) = 0.0;
    if (cq != 0.0) {
      // A[k] -= c B[k] with B[k] = A[m - k] (old values, so the pair (k, m - k) is updated together); B[0] = 0
      for (int k = 0; 2 * k <= m; ++k) {
        const double ak = c(k), amk = c(m - k);
        const double bk = k ? amk : 0.0, bmk = ak;              // B[k], B[m - k] (m - k >= 1)
        double nk = ak, nmk = amk;
        if (bk != 0.0) {
          const double p = __dmul_rn(cq, bk);
          if (p != 0.0) {
            const double v = __dsub_rn(ak, p);
            nk = v != 0.0 ? v : 0.0;
          }
        }
        if (bmk != 0.0) {
          const double p = __dmul_rn(cq, bmk);
          if (p != 0.0) {
            const double v = __dsub_rn(amk, p);
            nmk = v != 0.0 ? v : 0.0;
          }
        }
        if (2 * k == m) {
          c(k) = nk;
        } else {
          c(k) = nk;
          c(m - k) = nmk;
        }
      }
    }
    hi = 0;
    for (int k = m; k > 0; --k)
      if (c(k) != 0.0) {
        hi = k;
        break;
      }
    ++m;
  }

  __device__ __forceinline__ void finish(const LpcArgs& a, long long n_frames) {
    const long long g = (long long)blockIdx.x * nt + threadIdx.x;
    const int L = order + 1;
    if (a.coef) {
      double* cg = a.coef + g * L;
      for (int k = 0; k < L; ++k) cg[k] = failed ? NAN : c(k);
    }
    if (a.err) {
      double e = NAN;
      if (!failed) {
        Psum acc;
        for (int i = 0; i <= hi; ++i) {
          const double ai = c(i);
          for (int j = 0; j <= hi; ++j) acc.add(__dmul_rn(__dmul_rn(r(i > j ? i - j : j - i), ai), c(j)));
        }
        e = acc.value();
      }
      a.err[g] = e;
    }
    if (a.failed) a.failed[g] = failed ? 1 : 0;
  }
};

__device__ __forceinline__ double abs_or_inf(double v) { return isfinite(v) ? fabs(v) : INFINITY; }

__device__ __forceinline__ double warp_max(double v) {
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// kcovar, one warp per frame: the Gram-Schmidt lattice of the header on the frame's lag matrix P.  Step m divides
// once per task: task 0 is k = -inner(A, z^-m) / beta[m - 1], task t = 1 .. m (while m < order) is gamma[t - 1] =
// inner(z^-(m+1), B[t - 1]) / beta[t - 1]; lane l takes tasks l, l + 32, ... in rounds, so next() / take() run
// ceil(tasks / 32) times per step and the last take() of a step finishes it.  Sums over a whole frame (beta, the
// error) run on every lane, which keeps the warp converged and leaves every lane with the value.
struct Covar {
  const double* P;                             // [L][L]
  double* B;                                   // B[q][p] at q * (order + 2) + p, p = 0 .. q + 1
  double* A;                                   // [L]
  double* beta;                                // [order]
  double* gam;                                 // [order]
  double* bmax;                                // [order]: max |B[q][p]|, inf when one is not finite
  long long g;
  int order, L, lane, m, round, la, failed;
  double maxphi, maxA, k;
  bool done;

  __device__ __forceinline__ double* b(int q) const { return B + q * (order + 2); }

  // psum(P[i][j] * x[i] * y[j] for i < lx, j < ly): the reference's inner() over two numlists
  __device__ __forceinline__ double inner(const double* x, int lx, const double* y, int ly) const {
    Psum acc;
    for (int i = 0; i < lx; ++i) {
      const double xi = x[i];
      const double* Pi = P + i * L;
      for (int j = 0; j < ly; ++j) acc.add(__dmul_rn(__dmul_rn(Pi[j], xi), y[j]));
    }
    return acc.value();
  }

  __device__ __forceinline__ bool init(const LpcArgs& a, long long n_frames, double* s_m) {
    const int warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
    lane = threadIdx.x & 31;
    g = (long long)blockIdx.x * nw + warp;
    if (g >= n_frames) return false;
    order = a.order;
    L = order + 1;
    double* base = s_m + (long long)warp * covar_frame_doubles(order);
    double* Pw = base;
    B = Pw + L * L;
    A = B + order * (order + 2);
    beta = A + L;
    gam = beta + order;
    bmax = gam + order;
    P = Pw;
    const int nc = L * (L + 1) / 2;
    const double* tri = a.r + g * nc;
    double mx = 0.0;
    for (int j = 0, c0 = 0; j < L; c0 += ++j)
      for (int i = lane; i <= j; i += 32) {
        const double v = tri[c0 + i];
        Pw[j * L + i] = v;
        Pw[i * L + j] = v;
        mx = fmax(mx, abs_or_inf(v));
      }
    maxphi = warp_max(mx);
    for (int p = lane; p < L; p += 32) A[p] = p ? 0.0 : 1.0;
    if (lane < 2) B[lane] = lane ? 1.0 : 0.0;
    if (lane == 0) bmax[0] = 1.0;
    __syncwarp();
    const double b0 = inner(B, 2, B, 2);
    if (lane == 0) beta[0] = b0;
    __syncwarp();
    m = 1;
    round = 0;
    la = 1;
    failed = 0;
    done = false;
    return true;
  }

  __device__ __forceinline__ int tasks() const { return m < order ? m + 1 : 1; }

  __device__ __forceinline__ bool next(double& num, double& den) {
    if (done) return false;
    if (round == 0) {
      if (beta[m - 1] == 0.0) {                // the reference's ZeroDivisionError
        failed = 1;
        done = true;
        return false;
      }
      double mx = 0.0;
      for (int i = 0; i < la; ++i) mx = fmax(mx, abs_or_inf(A[i]));
      maxA = mx;
    }
    const int t = round * 32 + lane;
    num = 0.0;
    den = 1.0;
    if (t == 0) {
      // inner(A, z^-m): only the products of j = m are summed; the others, (P[i][j] * A[i]) * 0.0, are +-0 unless
      // P[i][j] * A[i] is not finite, which makes the whole sum NaN
      Psum acc;
      for (int i = 0; i < la; ++i) acc.add(__dmul_rn(P[i * L + m], A[i]));
      double v = acc.value();
      if (!isfinite(__dmul_rn(maxphi, maxA)))
        for (int i = 0; i < la; ++i)
          for (int j = 0; j < m; ++j)
            if (!isfinite(__dmul_rn(P[i * L + j], A[i]))) v = NAN;
      num = -v;
      den = beta[m - 1];
    } else if (t < tasks()) {
      // inner(z^-(m+1), B[q]): only the products of i = m + 1 are summed; the others, (P[i][j] * 0.0) * B[q][j],
      // are +-0 unless P[i][j] or B[q][j] is not finite
      const int q = t - 1, lb = q + 2;
      const double* bq = b(q);
      const double* Pm = P + (m + 1) * L;
      Psum acc;
      for (int j = 0; j < lb; ++j) acc.add(__dmul_rn(Pm[j], bq[j]));
      double v = acc.value();
      if (!isfinite(__dmul_rn(maxphi, bmax[q])))
        for (int i = 0; i <= m; ++i)
          for (int j = 0; j < lb; ++j)
            if (!isfinite(P[i * L + j]) || !isfinite(bq[j])) v = NAN;
      num = v;
      den = beta[q];
    }
    return true;
  }

  __device__ __forceinline__ void take(double quot) {
    const int t = round * 32 + lane;
    if (t == 0) k = quot;
    else if (t < tasks()) gam[t - 1] = quot;
    if (++round * 32 < tasks()) return;
    round = 0;
    k = __shfl_sync(0xffffffffu, k, 0);
    __syncwarp();
    if (k >= 1.0 || k <= -1.0) {               // the reference's "Unstable filter"
      failed = 2;
      done = true;
      return;
    }
    // A += k B[m - 1], powers 1 .. m; a coefficient equal to zero is dropped (+0.0)
    const double* bm1 = b(m - 1);
    for (int p = lane + 1; p <= m; p += 32) {
      const double bp = bm1[p];
      if (bp != 0.0) {
        const double t2 = __dmul_rn(k, bp);
        if (t2 != 0.0) {
          const double v = __dadd_rn(A[p], t2);
          A[p] = v != 0.0 ? v : 0.0;
        }
      }
    }
    __syncwarp();
    la = 1;
    for (int p = m; p > 0; --p)
      if (A[p] != 0.0) {
        la = p + 1;
        break;
      }
    if (m >= order) {
      done = true;
      return;
    }
    // B[m] = z^-(m+1) - sum(gamma[q] B[q] for q < m): per power, plain additions in q order, zeros dropped
    double* bm = b(m);
    double mx = 0.0;
    for (int p = lane + 1; p <= m; p += 32) {
      double acc = 0.0;
      for (int q = p - 1; q < m; ++q) {
        const double bp = b(q)[p];
        if (bp != 0.0) {
          const double t2 = __dmul_rn(gam[q], bp);
          if (t2 != 0.0) {
            const double v = __dadd_rn(acc, t2);
            acc = v != 0.0 ? v : 0.0;
          }
        }
      }
      const double v = acc != 0.0 ? -acc : 0.0;
      bm[p] = v;
      mx = fmax(mx, abs_or_inf(v));
    }
    if (lane == 0) {
      bm[0] = 0.0;
      bm[m + 1] = 1.0;
    }
    mx = fmax(warp_max(mx), 1.0);
    if (lane == 0) bmax[m] = mx;
    __syncwarp();
    const double bt = inner(bm, m + 2, bm, m + 2);
    __syncwarp();
    if (lane == 0) beta[m] = bt;
    __syncwarp();
    ++m;
  }

  __device__ __forceinline__ void finish(const LpcArgs& a) {
    const double e = failed ? NAN : inner(A, la, A, la);
    if (a.coef)
      for (int p = lane; p < L; p += 32) a.coef[g * L + p] = failed ? NAN : A[p];
    if (lane == 0) {
      if (a.err) a.err[g] = e;
      if (a.failed) a.failed[g] = (uint8_t)failed;
    }
  }
};

}  // namespace

// The recursion of each frame (see the file comment): every quotient of both recursions comes from the one division
// of this loop.
__global__ void __launch_bounds__(128) alz_lpc_levinson_kernel(const __grid_constant__ LpcArgs a, long long n_frames) {
  extern __shared__ double s_m[];              // kautocor: [order + 1][nt] lags, then [order + 1][nt] coefficients;
                                               // kcovar: covar_frame_doubles(order) per warp
  const bool covar = a.covar != 0;
  Levinson lv;
  Covar cv;
  if (!(covar ? cv.init(a, n_frames, s_m) : lv.init(a, n_frames, s_m))) return;
  for (;;) {
    double num, den;
    if (!(covar ? cv.next(num, den) : lv.next(num, den))) break;
    const double q = __ddiv_rn(num, den);
    if (covar) cv.take(q);
    else lv.take(q);
  }
  if (covar) cv.finish(a);
  else lv.finish(a, n_frames);
}

// After a call's frames: per stream (one CTA), the last `size` samples and the sample count.
__global__ void __launch_bounds__(kThreadsCommit) alz_lpc_commit_kernel(const __grid_constant__ LpcArgs a) {
  extern __shared__ float s_t[];
  framed_commit(a.state + blockIdx.x * a.sstride, a.x + blockIdx.x * a.xs, a.T, a.size, s_t);
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
  return n_streams * framed_state_stride(size);
}

int32_t alz_lpc_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream) {
  if (n_streams < 0 || size < 1 || size > ALZ_LPC_MAX_SIZE)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_LPC_MAX_SIZE);
  if (n_streams == 0) return ALZ_LPC_OK;
  if (!state_dev || ((uintptr_t)state_dev & 7)) return fail(ALZ_LPC_ERR_INVALID, "state is NULL or not 8-byte aligned");
  ALZ_CUDA_CHECK(cudaMemsetAsync(state_dev, 0, n_streams * framed_state_stride(size), (cudaStream_t)cuda_stream),
                 ALZ_LPC_ERR_CUDA);
  return ALZ_LPC_OK;
}

int64_t alz_lpc_scratch_bytes(int64_t n_streams, int64_t n_frames, int32_t order) {
  if (n_streams < 0 || n_frames < 0 || order < 0 || order > ALZ_LPC_MAX_ORDER)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0, n_frames >= 0 and 0 <= order <= %d", ALZ_LPC_MAX_ORDER);
  return n_streams * n_frames * (order + 1) * 8;
}

int64_t alz_lpc_covar_scratch_bytes(int64_t n_streams, int64_t n_frames, int32_t order) {
  if (n_streams < 0 || n_frames < 0 || order < 0 || order > ALZ_LPC_MAX_ORDER)
    return fail(ALZ_LPC_ERR_INVALID, "need n_streams >= 0, n_frames >= 0 and 0 <= order <= %d", ALZ_LPC_MAX_ORDER);
  return n_streams * n_frames * tri_cells(order) * 8;
}

}  // extern "C"

namespace {

// Both entry points: stats is acorr_dev (kautocor) or lagm_dev (kcovar).
int32_t run(bool covar, const float* x_dev, int64_t x_stride, const double* window_dev, double* stats,
            double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames, void* state_dev,
            int64_t n_streams, int64_t n_samples, int32_t order, int32_t size, int32_t hop, int32_t final,
            void* scratch_dev, int64_t scratch_bytes, void* cuda_stream) {
  if (order < 0 || order > ALZ_LPC_MAX_ORDER)
    return fail(ALZ_LPC_ERR_INVALID, "order must be in 0 .. %d (got %d)", ALZ_LPC_MAX_ORDER, order);
  if (size < 1 || size > ALZ_LPC_MAX_SIZE)
    return fail(ALZ_LPC_ERR_INVALID, "size must be in 1 .. %d (got %d)", ALZ_LPC_MAX_SIZE, size);
  if (hop < 1) return fail(ALZ_LPC_ERR_INVALID, "hop must be >= 1 (got %d)", hop);
  const bool solve = coef_dev || error_dev || failed_dev;
  if (covar && order >= size)
    return fail(ALZ_LPC_ERR_INVALID, "the lag matrix needs order < size (got order %d, size %d)", order, size);
  if (covar && solve && order < 1) return fail(ALZ_LPC_ERR_INVALID, "the covariance method needs order >= 1");
  if (n_streams < 0 || n_samples < 0 || n_frames < 0) return fail(ALZ_LPC_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_LPC_OK;
  if (!state_dev || (n_samples > 0 && !x_dev)) return fail(ALZ_LPC_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev & 3) || ((uintptr_t)state_dev & 7) || ((uintptr_t)window_dev & 7) ||
      (covar && ((uintptr_t)stats & 7)))
    return fail(ALZ_LPC_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_LPC_ERR_INVALID, "stride < n_samples");
  // the statistics the recursion reads: acorr_dev or the scratch (kautocor), the triangle scratch (kcovar)
  double* r = covar ? nullptr : stats;
  if (!r && solve) {
    const int64_t need = covar ? alz_lpc_covar_scratch_bytes(n_streams, n_frames, order)
                               : alz_lpc_scratch_bytes(n_streams, n_frames, order);
    if (!scratch_dev || scratch_bytes < need)
      return fail(ALZ_LPC_ERR_INVALID, "scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
    if ((uintptr_t)scratch_dev & 7) return fail(ALZ_LPC_ERR_INVALID, "misaligned scratch");
    r = (double*)scratch_dev;
  }
  LpcArgs a{};
  a.x = x_dev;
  a.w = window_dev;
  a.r = r;
  a.lagm = covar ? stats : nullptr;
  a.coef = coef_dev;
  a.err = error_dev;
  a.failed = failed_dev;
  a.state = (unsigned char*)state_dev;
  a.xs = x_stride;
  a.sstride = framed_state_stride(size);
  a.T = n_samples;
  a.F = n_frames;
  a.order = order;
  a.size = size;
  a.hop = hop;
  a.final_ = final != 0;
  a.covar = covar;
  a.ncell = covar ? (int)tri_cells(order) : order + 1;
  a.fpc = frames_per_cta(a.ncell, size);
  a.blocks_per_stream = (int)((n_frames + a.fpc - 1) / a.fpc);
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  if (n_frames > 0 && (r || a.lagm)) {
    const long long grid = n_streams * a.blocks_per_stream;
    if (grid > 0x7fffffffLL || n_frames > 0x7fffffffLL) return fail(ALZ_LPC_ERR_UNSUPPORTED, "too many frames for one launch");
    int threads = (a.fpc * a.ncell + 31) / 32 * 32;
    if (threads > kMaxFramesPerCta * 32) threads = kMaxFramesPerCta * 32;
    const size_t smem = (size_t)a.fpc * (size + 1) * 8;
    ALZ_CUDA_CHECK(allow_dynamic_smem((const void*)alz_lpc_kernel, smem), ALZ_LPC_ERR_CUDA);
    alz_lpc_kernel<<<(unsigned)grid, threads, smem, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
    if (solve) {
      const long long total = n_streams * n_frames;
      int nt;
      size_t smem2;
      long long blocks;
      if (covar) {
        const int w = covar_warps(order);
        nt = 32 * w;
        smem2 = (size_t)w * covar_frame_doubles(order) * 8;
        blocks = (total + w - 1) / w;
      } else {
        nt = levinson_threads(order);
        smem2 = (size_t)2 * 8 * (order + 1) * nt;
        blocks = (total + nt - 1) / nt;
      }
      if (blocks > 0x7fffffffLL) return fail(ALZ_LPC_ERR_UNSUPPORTED, "too many frames for one launch");
      ALZ_CUDA_CHECK(allow_dynamic_smem((const void*)alz_lpc_levinson_kernel, smem2), ALZ_LPC_ERR_CUDA);
      alz_lpc_levinson_kernel<<<(unsigned)blocks, nt, smem2, cs>>>(a, total);
      ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
    }
  }
  if (n_samples > 0) {
    alz_lpc_commit_kernel<<<(unsigned)n_streams, kThreadsCommit, (size_t)4 * size, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_LPC_ERR_CUDA);
  }
  return ALZ_LPC_OK;
}

}  // namespace

extern "C" {

int32_t alz_lpc_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, double* acorr_dev,
                          double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames, void* state_dev,
                          int64_t n_streams, int64_t n_samples, int32_t order, int32_t size, int32_t hop, int32_t final,
                          void* scratch_dev, int64_t scratch_bytes, void* cuda_stream) {
  return run(false, x_dev, x_stride, window_dev, acorr_dev, coef_dev, error_dev, failed_dev, n_frames, state_dev,
             n_streams, n_samples, order, size, hop, final, scratch_dev, scratch_bytes, cuda_stream);
}

int32_t alz_lpc_covar_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, double* lagm_dev,
                                double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames,
                                void* state_dev, int64_t n_streams, int64_t n_samples, int32_t order, int32_t size,
                                int32_t hop, int32_t final, void* scratch_dev, int64_t scratch_bytes,
                                void* cuda_stream) {
  return run(true, x_dev, x_stride, window_dev, lagm_dev, coef_dev, error_dev, failed_dev, n_frames, state_dev,
             n_streams, n_samples, order, size, hop, final, scratch_dev, scratch_bytes, cuda_stream);
}

}  // extern "C"
