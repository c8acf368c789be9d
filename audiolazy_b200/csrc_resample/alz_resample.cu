// alz_resample.cu -- the C ABI of include/alz_b200_resample.h: Lagrange resampling of S streams on sm_90a.
//
// The host walks the schedule (alz_resample_schedule): it is control metadata, the same for every stream, like the
// block counts of alz_common.h.  A call then runs three kernels in stream order:
//   * alz_resample_weights_kernel: one thread per output computes the order + 1 weights of its idx, once for the
//     whole batch;
//   * alz_resample_kernel: a CTA takes a tile of kTile consecutive outputs for a group of up to kGroup streams.  It
//     stages the tile's weights in shared memory once ([j][t], so that a warp reads consecutive words), then each
//     thread evaluates its output for every stream of the group, two streams at a time: the compensated sum of the order + 1 products over
//     the samples before the output's position, read straight from global memory (neighbouring outputs read
//     neighbouring samples, so a warp's loads share sectors; a large step reads only the windows it needs) or, before
//     the block, from the float64 history;
//   * alz_resample_commit_kernel: one CTA per stream shifts the last order + 1 samples into the history.
// The unit is compiled with -fmad=false and spells its arithmetic with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn:
// nothing is contracted or reassociated, so every output is the reference's float64 value.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_resample.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

namespace {

constexpr int kTile = 128;                  // outputs per CTA (one per thread)
constexpr int kGroup = 8;                   // streams per CTA: the tile's weights are staged once for all of them
constexpr int kThreadsCommit = 64;

struct ResampleArgs {
  const float* x;
  void* out;
  double* state;
  const int64_t* pos;
  const double* w;
  long long n_out, S, T, xs, os;
  int L, group, out_f64;
};

bool valid_order(int order) { return order >= 1 && order <= ALZ_RESAMPLE_MAX_ORDER; }

}  // namespace

// w[i * L + j] = prod over r != j, in ascending r, of (idx[i] - r) / (j - r).
__global__ void __launch_bounds__(256) alz_resample_weights_kernel(const double* idx, double* w, long long n, int L) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
    const double k = idx[i];
    for (int j = 0; j < L; ++j) {
      double prod = 0.0;
      bool first = true;
      for (int r = 0; r < L; ++r) {
        if (r == j) continue;
        const double q = __ddiv_rn(__dsub_rn(k, (double)r), (double)(j - r));
        prod = first ? q : __dmul_rn(prod, q);
        first = false;
      }
      w[i * L + j] = prod;
    }
  }
}

__global__ void __launch_bounds__(kTile) alz_resample_kernel(const __grid_constant__ ResampleArgs a) {
  extern __shared__ double w_s[];           // [L][kTile]
  const int t = threadIdx.x, L = a.L;
  const long long m0 = (long long)blockIdx.x * kTile, m = m0 + t;
  const int nt = (int)min((long long)kTile, a.n_out - m0);
  for (int e = t; e < nt * L; e += kTile) {
    const int i = e / L, j = e - i * L;
    w_s[j * kTile + i] = a.w[(m0 + i) * L + j];
  }
  __syncthreads();
  if (t >= nt) return;
  const long long p0 = a.pos[m] - L;          // the output's first sample, in block coordinates
  const long long s0 = (long long)blockIdx.y * a.group, s1 = min(s0 + a.group, a.S);
  auto sample = [&](long long s, long long p) -> double {
    return p >= 0 ? (double)__ldg(a.x + s * a.xs + p) : a.state[s * L + L + p];   // history: p in [-L, 0)
  };
  auto store = [&](long long s, double v) {
    if (a.out_f64) static_cast<double*>(a.out)[s * a.os + m] = v;
    else static_cast<float*>(a.out)[s * a.os + m] = (float)v;
  };
  // two streams at a time: their loads are independent, so a thread has twice the loads in flight
  long long s = s0;
  for (; s + 1 < s1; s += 2) {
    Psum acc0, acc1;
#pragma unroll 4
    for (int j = 0; j < L; ++j) {
      const double w = w_s[j * kTile + t];
      const double y0 = sample(s, p0 + j), y1 = sample(s + 1, p0 + j);
      acc0.add(__dmul_rn(y0, w));
      acc1.add(__dmul_rn(y1, w));
    }
    store(s, acc0.value());
    store(s + 1, acc1.value());
  }
  if (s < s1) {
    Psum acc;
#pragma unroll 4
    for (int j = 0; j < L; ++j) acc.add(__dmul_rn(sample(s, p0 + j), w_s[j * kTile + t]));
    store(s, acc.value());
  }
}

// The history becomes the last L samples of (history, block).
__global__ void __launch_bounds__(kThreadsCommit) alz_resample_commit_kernel(const __grid_constant__ ResampleArgs a) {
  shift_history(a.state + (long long)blockIdx.x * a.L, a.L, a.x + (long long)blockIdx.x * a.xs, a.T);
}

__global__ void __launch_bounds__(256) alz_resample_init_kernel(double* state, long long n, double zero) {
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    state[i] = zero;
}

extern "C" {

const char* alz_resample_last_error(void) { return g_err.c_str(); }

int64_t alz_resample_state_doubles(int32_t order, int64_t n_streams) {
  if (!valid_order(order)) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "order must be in 1..%d (got %d)", ALZ_RESAMPLE_MAX_ORDER, order);
  if (n_streams < 0) return fail(ALZ_RESAMPLE_ERR_INVALID, "negative stream count");
  return n_streams * (order + 1);
}

int32_t alz_resample_state_init(double* state_dev, int64_t n_streams, int32_t order, double zero, void* cuda_stream) {
  if (!valid_order(order)) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "order must be in 1..%d (got %d)", ALZ_RESAMPLE_MAX_ORDER, order);
  if (n_streams < 0 || (n_streams > 0 && !state_dev)) return fail(ALZ_RESAMPLE_ERR_INVALID, "bad state or stream count");
  if (n_streams == 0) return ALZ_RESAMPLE_OK;
  const long long n = n_streams * (order + 1);
  const unsigned blocks = (unsigned)std::min<long long>((n + 255) / 256, 4096);
  alz_resample_init_kernel<<<blocks, 256, 0, (cudaStream_t)cuda_stream>>>(state_dev, n, zero);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_RESAMPLE_ERR_CUDA);
  return ALZ_RESAMPLE_OK;
}

int64_t alz_resample_schedule(int32_t order, double step, double idx, int64_t n_samples, int64_t capacity,
                              int64_t* pos, double* idx_out, double* idx_next) {
  if (!valid_order(order)) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "order must be in 1..%d (got %d)", ALZ_RESAMPLE_MAX_ORDER, order);
  if (!(std::isfinite(step) && step > 0)) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "the step must be finite and positive (got %g)", step);
  const double span = (double)(order + 1);
  if (span + step == span)
    return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "a step of %g never advances the position: the output would never consume its input", step);
  if (!std::isfinite(idx) || n_samples < 0 || capacity < 0 || !idx_next || (capacity > 0 && (!pos || !idx_out)))
    return fail(ALZ_RESAMPLE_ERR_INVALID, "bad idx, shape or buffer");
  const double threshold = .5 * span;
  int64_t consumed = 0, n = 0;
  for (;;) {
    while (idx > threshold) {
      if (consumed == n_samples) {
        *idx_next = idx;
        return n;
      }
      ++consumed;
      idx -= 1.0;
    }
    if (n == capacity) return fail(ALZ_RESAMPLE_ERR_CAPACITY, "the block yields more than %lld outputs", (long long)capacity);
    pos[n] = consumed;
    idx_out[n] = idx;
    ++n;
    idx += step;
  }
}

int32_t alz_resample_apply(const float* x_dev, void* out_dev, int32_t out_f64, double* state_dev,
                           const int64_t* pos_dev, const double* idx_dev, double* weights_dev, int64_t n_out,
                           int64_t n_streams, int64_t n_samples, int64_t x_stride, int64_t out_stride, int32_t order,
                           void* cuda_stream) {
  if (!valid_order(order)) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "order must be in 1..%d (got %d)", ALZ_RESAMPLE_MAX_ORDER, order);
  if (n_streams < 0 || n_samples < 0 || n_out < 0) return fail(ALZ_RESAMPLE_ERR_INVALID, "negative shape");
  if (n_streams == 0 || (n_samples == 0 && n_out == 0)) return ALZ_RESAMPLE_OK;
  if (!state_dev || (n_samples > 0 && !x_dev) || (n_out > 0 && (!out_dev || !pos_dev || !idx_dev || !weights_dev)))
    return fail(ALZ_RESAMPLE_ERR_INVALID, "NULL buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_RESAMPLE_ERR_INVALID, "x_stride < n_samples");
  if (n_streams > 1 && out_stride < n_out) return fail(ALZ_RESAMPLE_ERR_INVALID, "out_stride < n_out");
  ResampleArgs a{};
  a.x = x_dev;
  a.out = out_dev;
  a.state = state_dev;
  a.pos = pos_dev;
  a.w = weights_dev;
  a.n_out = n_out;
  a.S = n_streams;
  a.T = n_samples;
  a.xs = x_stride;
  a.os = out_stride;
  a.L = order + 1;
  a.out_f64 = out_f64 != 0;
  a.group = (int)std::min<long long>(n_streams, kGroup);
  long long groups = (n_streams + a.group - 1) / a.group;
  if (groups > 65535) {
    a.group = (int)((n_streams + 65534) / 65535);
    groups = (n_streams + a.group - 1) / a.group;
  }
  const long long tiles = (n_out + kTile - 1) / kTile;
  if (tiles > 0x7fffffffLL || n_streams > 0x7fffffffLL) return fail(ALZ_RESAMPLE_ERR_UNSUPPORTED, "too large a block for one launch");
  const cudaStream_t st = (cudaStream_t)cuda_stream;
  if (n_out > 0) {
    const unsigned wblocks = (unsigned)std::min<long long>((n_out + 255) / 256, 8192);
    alz_resample_weights_kernel<<<wblocks, 256, 0, st>>>(idx_dev, weights_dev, n_out, a.L);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_RESAMPLE_ERR_CUDA);
    const size_t smem = (size_t)a.L * kTile * sizeof(double);
    ALZ_CUDA_CHECK(allow_dynamic_smem((const void*)alz_resample_kernel, smem), ALZ_RESAMPLE_ERR_CUDA);
    alz_resample_kernel<<<dim3((unsigned)tiles, (unsigned)groups), kTile, smem, st>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_RESAMPLE_ERR_CUDA);
  }
  if (n_samples > 0) {
    alz_resample_commit_kernel<<<(unsigned)n_streams, kThreadsCommit, 0, st>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_RESAMPLE_ERR_CUDA);
  }
  return ALZ_RESAMPLE_OK;
}

}  // extern "C"
