// alz_amdf.cu -- the C ABI of include/alz_b200_amdf.h: the AMDF of S streams x L lags in one sm_90a kernel.
//
// A CTA is (virtual stream, group of 128 lags); each thread owns one lag and walks the stream's samples in order,
// in tiles of B samples.  Per tile the CTA stages two windows of the input in shared memory, as float64: the recent
// one [p0 - K, p0 + B) for the new term and the one `size` samples earlier for the old term, which is recomputed
// from the samples instead of being stored (it is the same deterministic float64 value).  Positions before the block
// come from the history the state carries (the last size + K samples, float64: `zero` need not be a float32 value).
// Every decim-th running mean is staged per warp, 32 values per lag, and stored as 32 coalesced 128-byte rows.
//
// The arithmetic is float64 with __dmul_rn / __dadd_rn (and -fmad=false for this unit): no contraction, so the
// sequential evaluation is AudioLazy's float64 sequence bit for bit.  Lags are sorted by tap count and delay, so
// that a group of only 2-tap lags (integer lags, lags below 1) runs the 2-tap body; a body for a group that mixes tap
// counts (lags whose linearize leaves one tap) selects each lag's own partial sum.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_amdf.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <vector>

namespace {

constexpr int kThreads = 128;               // lags per CTA
constexpr int kWarps = kThreads / 32;
constexpr int kTile = 1024;                 // samples per staged tile
constexpr int kMinTimeParallel = 16384;     // shortest block evaluated time-parallel
constexpr int kObufFloats = kWarps * 32 * 33;

struct AmdfLag {
  double c[3];      // coefficients; taps past nt are 0 at delay 0 and never enter the sum
  int k[3];         // delays
  int nt;           // taps (0: d = zero)
  int row;          // index of the lag in the caller's table, -1 for padding
  int group_nt;     // taps the lag's group evaluates (2 or 3)
  int group_mixed;  // the group has a lag with 0 < nt < group_nt
};

struct AmdfArgs {
  const float* x;
  float* out;
  double* state;
  const AmdfLag* lags;
  long long T, xs, os, sstride, Lc;
  long long P;      // chunks per stream (1: sequential)
  int n_groups, L, size, K, H, decim, phase;
  double inv;       // 1. / size
};

struct AmdfPlan {
  int device, L, size, K, H, n_groups, sequential, sm_count, ctas_per_sm;
  size_t smem;
  double inv;
  AmdfLag* d_lags;
};

bool env_flag(const char* name) {
  const char* v = getenv(name);
  return v && *v && atoi(v) != 0;
}

// sum_j c_j w[-k_j] over the lag's nt taps, each product rounded, added left to right.  The body evaluates the group's
// NT taps.  In a group where some lag has fewer (MIXED), such a lag keeps its partial sum: a select rather than an
// added 0 * x, which an inf or NaN input would turn into NaN where the reference gives its own value.  Lags are sorted
// so that most groups are uniform and skip the selects (they cost ~10 % at 256 lags).
template <int NT, bool MIXED>
__device__ __forceinline__ double tap_sum(const double* w, const double (&c)[3], const int (&k)[3], int nt) {
  const double d0 = __dmul_rn(c[0], w[-k[0]]);
  const double d1 = __dadd_rn(d0, __dmul_rn(c[1], w[-k[1]]));
  double d = (!MIXED || nt > 1) ? d1 : d0;
  if (NT == 3) {
    const double d2 = __dadd_rn(d1, __dmul_rn(c[2], w[-k[2]]));
    d = (!MIXED || nt > 2) ? d2 : d;
  }
  return d;
}

template <int NT, bool MIXED>
__device__ __forceinline__ void amdf_run(const AmdfArgs& a, int g, long long v, double* sm) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long s = v / a.P, c = v % a.P;
  const AmdfLag lg = a.lags[(long long)g * kThreads + tid];
  const double cc[3] = {lg.c[0], lg.c[1], lg.c[2]};
  const int kk[3] = {lg.k[0], lg.k[1], lg.k[2]};
  const bool has = lg.nt > 0;
  double* st = a.state + s * a.sstride;
  const long long cnt = (long long)st[0];
  const double zero = st[1];
  const double* hist = st + 2;                         // hist[H + p]: block position p in [-H, 0)
  const double zinv = __dmul_rn(zero, a.inv);
  const float* xr = a.x + s * a.xs;
  const long long nb = c * a.Lc, ne = (c == a.P - 1) ? a.T : nb + a.Lc;
  const int K = a.K, W = kTile + K;
  double* wr = sm;                                     // [p0 - K, p0 + b): the new term's samples
  double* wo = sm + W;                                 // [p0 - size - K, p0 - size + b): the old term's
  float* ob = reinterpret_cast<float*>(sm + 2 * W) + warp * 32 * 33;

  auto sample = [&](long long p) -> double { return p >= 0 ? (double)__ldg(xr + p) : hist[a.H + p]; };

  double mean;
  if (c == 0) {
    mean = lg.row >= 0 ? st[2 + a.H + lg.row] : 0.0;
  } else {
    // a chunk of a time-parallel evaluation: the sum of the `size` terms before it (zero / size before the stream)
    mean = 0.0;
    for (long long p0 = nb - a.size; p0 < nb; p0 += kTile) {
      const int b = (int)min((long long)kTile, nb - p0);
      __syncthreads();
      for (int i = tid; i < b + K; i += kThreads) wr[i] = sample(p0 - K + i);
      __syncthreads();
      for (int n = 0; n < b; ++n) {
        const double d = has ? tap_sum<NT, MIXED>(wr + K + n, cc, kk, lg.nt) : zero;
        mean = __dadd_rn(mean, cnt + p0 + n < 0 ? zinv : __dmul_rn(fabs(d), a.inv));
      }
    }
  }

  long long m = (nb + a.phase) / a.decim;              // output index of the next stored value
  int cd = (int)(m * a.decim + a.decim - 1 - a.phase - nb) + 1;
  int k = 0;                                           // values staged in ob (uniform over the CTA)
  auto flush = [&](int n_vals) {
    __syncwarp();
    for (int r = 0; r < 32; ++r) {
      const int row = __shfl_sync(0xffffffffu, lg.row, r);
      if (lane < n_vals && row >= 0) a.out[(s * a.L + row) * a.os + m + lane] = ob[r * 33 + lane];
    }
    __syncwarp();
    m += n_vals;
  };

  for (long long p0 = nb; p0 < ne; p0 += kTile) {
    const int b = (int)min((long long)kTile, ne - p0);
    __syncthreads();
    for (int i = tid; i < b + K; i += kThreads) {
      wr[i] = sample(p0 - K + i);
      wo[i] = sample(p0 - a.size - K + i);
    }
    __syncthreads();
    for (int n = 0; n < b; ++n) {
      const double d = has ? tap_sum<NT, MIXED>(wr + K + n, cc, kk, lg.nt) : zero;
      const double dold = has ? tap_sum<NT, MIXED>(wo + K + n, cc, kk, lg.nt) : zero;
      const double nw = __dmul_rn(fabs(d), a.inv);
      const double od = cnt + p0 + n < a.size ? zinv : __dmul_rn(fabs(dold), a.inv);
      mean = __dadd_rn(__dsub_rn(mean, od), nw);
      if (--cd == 0) {
        cd = a.decim;
        ob[lane * 33 + k] = (float)mean;
        if (++k == 32) {
          flush(32);
          k = 0;
        }
      }
    }
  }
  if (k) flush(k);
  if (c == a.P - 1 && lg.row >= 0) st[2 + a.H + a.L + lg.row] = mean;   // committed by alz_amdf_commit_kernel
}

}  // namespace

__global__ void __launch_bounds__(kThreads) alz_amdf_kernel(const __grid_constant__ AmdfArgs a) {
  extern __shared__ __align__(16) double amdf_smem[];
  const int g = (int)(blockIdx.x % a.n_groups);
  const long long v = blockIdx.x / a.n_groups;
  const AmdfLag& first = a.lags[(long long)g * kThreads];   // group_nt / group_mixed: uniform over the CTA
  if (first.group_nt <= 2) {
    if (first.group_mixed) amdf_run<2, true>(a, g, v, amdf_smem);
    else amdf_run<2, false>(a, g, v, amdf_smem);
  } else {
    if (first.group_mixed) amdf_run<3, true>(a, g, v, amdf_smem);
    else amdf_run<3, false>(a, g, v, amdf_smem);
  }
}

// After a block: the history becomes the last H samples of (history, block), the running means those the last chunk
// left, and the count advances.
__global__ void __launch_bounds__(256) alz_amdf_commit_kernel(const __grid_constant__ AmdfArgs a) {
  double* st = a.state + (long long)blockIdx.x * a.sstride;
  shift_history(st + 2, a.H, a.x + (long long)blockIdx.x * a.xs, a.T);
  for (int l = threadIdx.x; l < a.L; l += blockDim.x) st[2 + a.H + l] = st[2 + a.H + a.L + l];
  if (threadIdx.x == 0) st[0] = st[0] + (double)a.T;
}

__global__ void __launch_bounds__(256) alz_amdf_init_kernel(double* state, long long n, long long sstride, double zero) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    state[i] = i % sstride == 0 ? 0.0 : zero;
}

namespace {

long long chunks(const AmdfPlan* p, long long S, long long T) {
  if (p->sequential || env_flag("ALZ_NO_TIME_PARALLEL") || T < kMinTimeParallel || S <= 0) return 1;
  const long long warps = S * p->n_groups * kWarps;
  const long long slots = (long long)p->sm_count * p->ctas_per_sm * kWarps;   // resident warp slots of this kernel
  if (warps * 2 > slots) return 1;
  // about two waves of CTAs, with chunks long enough that the seed sums (size samples each) cost <= 1/4 of a chunk
  const long long min_len = std::max(4LL * (p->size + p->K), 4096LL);
  long long P = std::min(T / min_len, (2 * slots + warps - 1) / warps);
  P = std::min(P, (long long)0x7fffffff / (S * p->n_groups));
  return P < 2 ? 1 : P;
}

}  // namespace

extern "C" {

const char* alz_amdf_last_error(void) { return g_err.c_str(); }

int32_t alz_amdf_plan_create(const int32_t* n_taps, const int32_t* delays, const double* coefs, int32_t n_lags,
                             int32_t size, int32_t flags, void** plan_out) {
  if (!plan_out) return fail(ALZ_AMDF_ERR_INVALID, "plan_out is NULL");
  *plan_out = nullptr;
  if (n_lags < 1 || !n_taps || !delays || !coefs) return fail(ALZ_AMDF_ERR_INVALID, "need at least one lag");
  if (size < 1) return fail(ALZ_AMDF_ERR_INVALID, "size must be >= 1 (got %d)", size);
  int K = 0;
  for (int l = 0; l < n_lags; ++l) {
    if (n_taps[l] < 0 || n_taps[l] > 3) return fail(ALZ_AMDF_ERR_INVALID, "lag %d has %d taps (0..3)", l, n_taps[l]);
    for (int j = 0; j < n_taps[l]; ++j) {
      if (delays[3 * l + j] < 0) return fail(ALZ_AMDF_ERR_NONCAUSAL, "Non-causal filter");
      K = std::max(K, (int)delays[3 * l + j]);
    }
  }
  auto p = new AmdfPlan{};
  p->L = n_lags;
  p->size = size;
  p->K = K;
  p->H = size + K;
  p->inv = 1. / size;
  p->sequential = (flags & ALZ_AMDF_PLAN_SEQUENTIAL) != 0;
  p->smem = (size_t)2 * (kTile + K) * sizeof(double) + kObufFloats * sizeof(float);
  int max_smem = 0;
  cudaError_t e = cudaGetDevice(&p->device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, p->device);
  if (e == cudaSuccess) e = cudaDeviceGetAttribute(&max_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, p->device);
  if (e != cudaSuccess) {
    delete p;
    cudaGetLastError();
    return fail(ALZ_AMDF_ERR_CUDA, "no usable CUDA device: %s", cudaGetErrorString(e));
  }
  if (p->smem > (size_t)max_smem) {
    delete p;
    return fail(ALZ_AMDF_ERR_UNSUPPORTED, "a tap delay of %d samples needs %zu bytes of shared memory (the device has %d): "
                "the longest supported delay is %d", K, (size_t)2 * (kTile + K) * 8 + kObufFloats * 4, max_smem,
                (int)((max_smem - kObufFloats * 4) / 16 - kTile));
  }
  // sort by (tap class, longest delay): 1-tap lags, then 0- and 2-tap lags, then 3-tap lags, so that groups are uniform
  // (groups of 2-tap lags run the 2-tap body, without selects); neighbouring threads read neighbouring samples
  std::vector<int> order(n_lags);
  for (int l = 0; l < n_lags; ++l) order[l] = l;
  auto key = [&](int l) {
    int kmax = 0;
    for (int j = 0; j < n_taps[l]; ++j) kmax = std::max(kmax, (int)delays[3 * l + j]);
    return std::make_pair(n_taps[l] == 1 ? 0 : n_taps[l] == 3 ? 2 : 1, kmax);
  };
  std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return key(a) < key(b); });
  p->n_groups = (n_lags + kThreads - 1) / kThreads;
  std::vector<AmdfLag> table((size_t)p->n_groups * kThreads);
  for (auto& t : table) t = AmdfLag{{0.0, 0.0, 0.0}, {0, 0, 0}, 0, -1, 2, 0};   // padding: no taps
  for (int i = 0; i < n_lags; ++i) {
    const int l = order[i];
    AmdfLag& t = table[i];
    t.nt = n_taps[l];
    t.row = l;
    for (int j = 0; j < n_taps[l]; ++j) {
      t.c[j] = coefs[3 * l + j];
      t.k[j] = delays[3 * l + j];
    }
  }
  for (int g = 0; g < p->n_groups; ++g) {
    int gnt = 2, mixed = 0;
    for (int i = 0; i < kThreads; ++i) gnt = std::max(gnt, table[(size_t)g * kThreads + i].nt);
    for (int i = 0; i < kThreads; ++i) {
      const int nt = table[(size_t)g * kThreads + i].nt;
      mixed |= nt > 0 && nt < gnt;
    }
    for (int i = 0; i < kThreads; ++i) {
      table[(size_t)g * kThreads + i].group_nt = gnt;
      table[(size_t)g * kThreads + i].group_mixed = mixed;
    }
  }
  e = allow_dynamic_smem((const void*)alz_amdf_kernel, p->smem);
  if (e == cudaSuccess) e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&p->ctas_per_sm, alz_amdf_kernel, kThreads, p->smem);
  if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_lags, table.size() * sizeof(AmdfLag));
  if (e == cudaSuccess) e = cudaMemcpy(p->d_lags, table.data(), table.size() * sizeof(AmdfLag), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) {
    if (p->d_lags) cudaFree(p->d_lags);
    delete p;
    cudaGetLastError();
    return fail(ALZ_AMDF_ERR_CUDA, "plan upload: %s", cudaGetErrorString(e));
  }
  p->ctas_per_sm = std::max(p->ctas_per_sm, 1);
  *plan_out = p;
  return ALZ_AMDF_OK;
}

void alz_amdf_plan_destroy(void* plan) {
  auto p = static_cast<AmdfPlan*>(plan);
  if (!p) return;
  // launches queued on any stream may still read the lag table: cudaFree only "may perform implicit synchronization"
  int cur = -1;
  cudaGetDevice(&cur);
  cudaSetDevice(p->device);
  cudaDeviceSynchronize();
  cudaFree(p->d_lags);
  if (cur >= 0) cudaSetDevice(cur);
  cudaGetLastError();
  delete p;
}

int64_t alz_amdf_state_doubles(const void* plan, int64_t n_streams) {
  auto p = static_cast<const AmdfPlan*>(plan);
  if (!p || n_streams < 0) return fail(ALZ_AMDF_ERR_INVALID, "bad plan or stream count");
  return n_streams * (2 + (int64_t)p->H + 2 * (int64_t)p->L);
}

int32_t alz_amdf_state_init(const void* plan, double* state_dev, int64_t n_streams, double zero, void* cuda_stream) {
  auto p = static_cast<const AmdfPlan*>(plan);
  if (!p || n_streams < 0 || (n_streams > 0 && !state_dev)) return fail(ALZ_AMDF_ERR_INVALID, "bad plan, state or stream count");
  if (n_streams == 0) return ALZ_AMDF_OK;
  const long long sstride = 2 + (long long)p->H + 2 * (long long)p->L, n = n_streams * sstride;
  const unsigned blocks = (unsigned)std::min<long long>((n + 255) / 256, 4096);
  alz_amdf_init_kernel<<<blocks, 256, 0, (cudaStream_t)cuda_stream>>>(state_dev, n, sstride, zero);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_AMDF_ERR_CUDA);
  return ALZ_AMDF_OK;
}

int64_t alz_amdf_plan_chunks(const void* plan, int64_t n_streams, int64_t n_samples) {
  auto p = static_cast<const AmdfPlan*>(plan);
  if (!p || n_streams < 0 || n_samples < 0) return fail(ALZ_AMDF_ERR_INVALID, "bad plan or shape");
  return chunks(p, n_streams, n_samples);
}

int32_t alz_amdf_apply_f32(const void* plan, const float* x_dev, float* out_dev, double* state_dev, int64_t n_streams,
                           int64_t n_samples, int64_t x_stride, int64_t out_stride, int32_t decim, int32_t phase,
                           void* cuda_stream) {
  auto p = static_cast<const AmdfPlan*>(plan);
  if (!p) return fail(ALZ_AMDF_ERR_INVALID, "plan is NULL");
  if (n_streams < 0 || n_samples < 0) return fail(ALZ_AMDF_ERR_INVALID, "negative shape");
  if (decim < 1 || phase < 0 || phase >= decim) return fail(ALZ_AMDF_ERR_INVALID, "need decim >= 1 and 0 <= phase < decim");
  if (n_streams == 0 || n_samples == 0) return ALZ_AMDF_OK;
  const long long n_out = (phase + n_samples) / decim;
  if (!x_dev || !state_dev || (n_out > 0 && !out_dev)) return fail(ALZ_AMDF_ERR_INVALID, "NULL buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_AMDF_ERR_INVALID, "x_stride < n_samples");
  if ((n_streams > 1 || p->L > 1) && out_stride < n_out) return fail(ALZ_AMDF_ERR_INVALID, "out_stride < n_out");
  int dev = -1;
  ALZ_CUDA_CHECK(cudaGetDevice(&dev), ALZ_AMDF_ERR_CUDA);
  if (dev != p->device) return fail(ALZ_AMDF_ERR_INVALID, "the plan lives on device %d, device %d is current", p->device, dev);
  const long long P = chunks(p, n_streams, n_samples);
  if (n_streams * P * p->n_groups > 0x7fffffffLL || n_streams > 0x7fffffffLL)
    return fail(ALZ_AMDF_ERR_UNSUPPORTED, "too many streams for one launch");
  AmdfArgs a{};
  a.x = x_dev;
  a.out = out_dev;
  a.state = state_dev;
  a.lags = p->d_lags;
  a.T = n_samples;
  a.xs = x_stride;
  a.os = out_stride;
  a.sstride = 2 + (long long)p->H + 2 * (long long)p->L;
  a.P = P;
  a.Lc = n_samples / P;
  a.n_groups = p->n_groups;
  a.L = p->L;
  a.size = p->size;
  a.K = p->K;
  a.H = p->H;
  a.decim = decim;
  a.phase = phase;
  a.inv = p->inv;
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  alz_amdf_kernel<<<(unsigned)(n_streams * P * p->n_groups), kThreads, p->smem, st>>>(a);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_AMDF_ERR_CUDA);
  alz_amdf_commit_kernel<<<(unsigned)n_streams, 256, 0, st>>>(a);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_AMDF_ERR_CUDA);
  return ALZ_AMDF_OK;
}

}  // extern "C"
