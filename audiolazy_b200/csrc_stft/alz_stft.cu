// alz_stft.cu -- the C ABI of include/alz_b200_stft.h: short-time Fourier analysis, resynthesis and overlap-add of S
// streams on sm_90a.
//
// Kernels, in stream order:
//   * alz_stft_analysis_kernel: a CTA takes fpc consecutive frames of one stream (fpc = 1 from size 4096 on), tpf
//     threads per frame.  Each frame is loaded (samples before the call from the state's last `size` samples),
//     windowed, rotated and stored as complex float64 in shared memory, transformed there (see below), and
//     its bins 0 .. size / 2 stored, consecutive threads on consecutive bins;
//   * alz_stft_commit_kernel: one CTA per stream shifts the last `size` samples into the analysis state;
//   * alz_stft_synthesis_kernel: the same geometry the other way: the Hermitian spectrum of each frame is rebuilt in
//     shared memory from its size / 2 + 1 bins, inverse-transformed, scaled, rotated and stored as float64 frames;
//   * alz_ola_kernel: one thread per output sample of a stream sums the frames that cover it, oldest first, starting
//     from the open sum the state holds for the first size - hop samples; the sums still open after the call are
//     written to the state's other copy;
//   * alz_ola_commit_kernel: per stream, flips the state's copy and counts the frames.
// Both states start as zero bytes (cudaMemsetAsync).
//
// The transform is a mixed-radix decimation in time, in place in one shared buffer of N complex values (size 8192
// takes 128 KB): radices 4, 2, 3, 5, 7, then the other primes.  The frame is loaded in digit-reversed order
// (position()); with L the product of the radices before it, a stage of radix R combines R consecutive transforms of
// length L: butterfly (b, j), j < L, reads a[b L R + j + r L], multiplies input r by W^(r j N / (L R)) (W = exp(-+2
// pi i / N), the caller's table), takes its R-point DFT and writes output q back to a[b L R + j + q L].  Butterflies of
// radix <= 7 hold R values; a larger prime computes each output as a direct R-term sum, O(N R) for the stage, and holds
// its kOut outputs until the whole frame has been read.
//
// The unit is compiled with -fmad=false: the window products and the overlap-add sums are single roundings in the
// order of the header; the FFT spells its complex products with fma().
#pragma GCC visibility push(default)
#include "../../include/alz_b200_stft.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <cstdint>

namespace {

constexpr int kOut = 16;                 // outputs a thread holds in a stage: tpf = ceil(size / kOut)
constexpr int kMaxThreads = 512;
constexpr int kTargetThreads = 256;      // small sizes: frames per CTA until this many threads
constexpr int kMaxStages = 16;
constexpr int kSmemBudget = 64 * 1024;   // frames per CTA are capped by this much staging, one frame may take more
constexpr int kThreadsCommit = 256;
constexpr int kThreadsOla = 256;

struct Fft {
  int n, nst;
  int radix[kMaxStages];
};

struct StftArgs {
  const float* x;
  const double* w;
  const double2* tw;
  const void* spec_in;
  void* spec_out;
  double* frames;
  unsigned char* state;
  long long xs, sstride, T, F, fstride, sstride_spec;
  int size, hop, shift, c128, fpc, tpf, blocks_per_stream;
  Fft fft;
};

struct OlaArgs {
  const void* v;
  int f64;
  const double* w;
  float* y;
  unsigned char* state;
  long long fstride, sstride_v, ys, sstride, F, P;   // P: positions a stream's thread range covers
  int size, hop, final_;
};

long long ola_state_stride(int size, int hop) { return 16 + 16 * (long long)(size - hop); }

Fft factor(int n) {
  Fft f{};
  f.n = n;
  int m = n;
  while (m % 4 == 0) { f.radix[f.nst++] = 4; m /= 4; }
  while (m % 2 == 0) { f.radix[f.nst++] = 2; m /= 2; }
  for (int p = 3; m > 1; p += 2)
    while (m % p == 0) { f.radix[f.nst++] = p; m /= p; }
  return f;
}

int threads_per_frame(int size) { return (size + kOut - 1) / kOut; }

int frames_per_cta(int size) {
  const int tpf = threads_per_frame(size);
  int fpc = kTargetThreads / tpf;
  const int by_smem = kSmemBudget / (16 * size);
  if (by_smem < fpc) fpc = by_smem;
  return fpc < 1 ? 1 : fpc;
}

__device__ __forceinline__ double2 cmul(double2 a, double2 b) {
  return make_double2(fma(a.x, b.x, -(a.y * b.y)), fma(a.x, b.y, a.y * b.x));
}
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }

// W^m of the transform's direction: the table value, conjugated for the inverse
__device__ __forceinline__ double2 root(const double2* tw, int m, bool inv) {
  const double2 r = __ldg(tw + m);
  return inv ? make_double2(r.x, -r.y) : r;
}

// The R-point DFT of v in place of out: radix 2 and 4 by additions, 3, 5 and 7 by products with the R-th roots.
template <int R>
__device__ __forceinline__ void dft(const double2 (&v)[R], double2* out, const double2* tw, int M, bool inv) {
  if constexpr (R == 2) {
    out[0] = cadd(v[0], v[1]);
    out[1] = csub(v[0], v[1]);
  } else if constexpr (R == 4) {
    const double2 s02 = cadd(v[0], v[2]), d02 = csub(v[0], v[2]);
    const double2 s13 = cadd(v[1], v[3]), d13 = csub(v[1], v[3]);
    // -i d13 forward, +i d13 inverse
    const double2 jd = inv ? make_double2(-d13.y, d13.x) : make_double2(d13.y, -d13.x);
    out[0] = cadd(s02, s13);
    out[1] = cadd(d02, jd);
    out[2] = csub(s02, s13);
    out[3] = csub(d02, jd);
  } else {
#pragma unroll
    for (int q = 0; q < R; ++q) {
      double2 acc = v[0];
#pragma unroll
      for (int r = 1; r < R; ++r) {
        const double2 p = cmul(v[r], root(tw, ((r * q) % R) * M, inv));
        acc = cadd(acc, p);
      }
      out[q] = acc;
    }
  }
}

// Position of input n in the transform's buffer: n = d[m-1] + R[m-1] (d[m-2] + R[m-2] (... + R[1] d[0])) goes to
// sum(d[s] L[s]), L[s] the product of the radices before stage s (the mixed-radix digit reversal).
// Radices 4 and 2 (every stage of a power-of-two size) take shifts and masks instead of integer divisions.
__device__ __forceinline__ int position(int n, const Fft& fft) {
  int p = 0, L = fft.n;
  for (int s = fft.nst - 1; s >= 0; --s) {
    const int R = fft.radix[s];
    if (R == 4 || R == 2) {
      const int sh = R == 4 ? 2 : 1;
      L >>= sh;
      p += (n & (R - 1)) * L;
      n >>= sh;
    } else {
      L /= R;
      p += (n % R) * L;
      n /= R;
    }
  }
  return p;
}

// b = j / Lp and jj = j % Lp, by a shift and a mask when Lp is a power of two (every stage before the odd radices).
__device__ __forceinline__ void split(int j, int Lp, int& b, int& jj) {
  if ((Lp & (Lp - 1)) == 0) {
    b = j >> (__ffs(Lp) - 1);
    jj = j & (Lp - 1);
  } else {
    b = j / Lp;
    jj = j - b * Lp;
  }
}

// One stage of radix R <= 7 over the frame at buf, in place: butterfly j = tid, tid + tpf, ... (see the file comment).
template <int R>
__device__ __forceinline__ void stage_small(double2* buf, int tid, int tpf, int N, int Lp, const double2* tw,
                                            bool inv) {
  const int M = N / R, tstep = N / (Lp * R);
  for (int j = tid; j < M; j += tpf) {
    int b, jj;
    split(j, Lp, b, jj);
    const int base = b * Lp * R + jj;
    double2 v[R], out[R];
    v[0] = buf[base];
#pragma unroll
    for (int r = 1; r < R; ++r) v[r] = cmul(buf[base + r * Lp], root(tw, r * jj * tstep, inv));
    dft<R>(v, out, tw, M, inv);
#pragma unroll
    for (int q = 0; q < R; ++q) buf[base + q * Lp] = out[q];
  }
}

// One stage of any radix R: outputs o = tid, tid + tpf, ... (o = q M + j), each a direct R-term sum, held until the
// whole frame has been read.
__device__ __noinline__ void stage_generic(double2* buf, bool active, int tid, int tpf, int N, int Lp, int R,
                                           const double2* tw, bool inv) {
  const int M = N / R, tstep = N / (Lp * R);
  double2 out[kOut];
  if (active) {
#pragma unroll
    for (int i = 0; i < kOut; ++i) {
      const int o = tid + i * tpf;
      if (o < N) {
        const int q = o / M, j = o - q * M, b = j / Lp, jj = j - b * Lp, base = b * Lp * R + jj;
        const int step = (int)(((long long)jj * tstep + (long long)q * M) % N);
        double2 acc = buf[base];
        int m = 0;
        for (int r = 1; r < R; ++r) {
          m += step;
          if (m >= N) m -= N;
          acc = cadd(acc, cmul(buf[base + r * Lp], root(tw, m, inv)));
        }
        out[i] = acc;
      }
    }
  }
  __syncthreads();
  if (active) {
#pragma unroll
    for (int i = 0; i < kOut; ++i) {
      const int o = tid + i * tpf;
      if (o < N) {
        const int q = o / M, j = o - q * M, b = j / Lp, jj = j - b * Lp;
        buf[b * Lp * R + jj + q * Lp] = out[i];
      }
    }
  }
}

// The transform of the frame at buf (loaded at position(n)), in place and in natural order.  Every thread of the CTA
// calls it: the stages synchronise the CTA.
__device__ __forceinline__ void fft_frame(double2* buf, bool active, int tid, int tpf, const Fft& fft,
                                          const double2* tw, bool inv) {
  int Lp = 1;
  for (int s = 0; s < fft.nst; ++s) {
    const int R = fft.radix[s];
    if (R > 7) {
      stage_generic(buf, active, tid, tpf, fft.n, Lp, R, tw, inv);
    } else if (active) {
      switch (R) {
        case 2: stage_small<2>(buf, tid, tpf, fft.n, Lp, tw, inv); break;
        case 3: stage_small<3>(buf, tid, tpf, fft.n, Lp, tw, inv); break;
        case 4: stage_small<4>(buf, tid, tpf, fft.n, Lp, tw, inv); break;
        case 5: stage_small<5>(buf, tid, tpf, fft.n, Lp, tw, inv); break;
        default: stage_small<7>(buf, tid, tpf, fft.n, Lp, tw, inv); break;
      }
    }
    __syncthreads();
    Lp *= R;
  }
}

}  // namespace

// Spectra of fpc consecutive frames of one stream (see the file comment).
__global__ void __launch_bounds__(kMaxThreads) alz_stft_analysis_kernel(const __grid_constant__ StftArgs a) {
  extern __shared__ double2 s_buf[];           // [fpc][size]
  const long long s = blockIdx.x / a.blocks_per_stream;
  const long long i0 = (long long)(blockIdx.x % a.blocks_per_stream) * a.fpc;
  const FramedSamples in = framed_samples(a.state + s * a.sstride, a.x + s * a.xs, a.T, a.size);
  const long long ka = first_open_block(in.C, a.size, a.hop);
  const int N = a.size, half = N / 2;
  const int nf = (int)(a.F - i0 < a.fpc ? a.F - i0 : a.fpc);
  const int f = threadIdx.x / a.tpf, tid = threadIdx.x - f * a.tpf;
  const bool active = f < nf;
  double2* buf = s_buf + (long long)f * N;

  if (active) {
    const long long g0 = (ka + i0 + f) * a.hop;                     // stream index of the frame's sample 0
    for (int n = tid; n < N; n += a.tpf) {
      const float v = in(g0 + n);
      const double b = a.w ? __dmul_rn((double)v, a.w[n]) : (double)v;
      int p = n;
      if (a.shift) p = n >= half ? n - half : n + (N - half);     // b'[p] = b[(p + half) % N]
      buf[position(p, a.fft)] = make_double2(b, 0.0);
    }
  }
  __syncthreads();
  fft_frame(buf, active, tid, a.tpf, a.fft, a.tw, false);
  if (!active) return;
  const int B = half + 1;
  const long long o = (s * a.F + i0 + f) * B;
  if (a.c128) {
    double2* out = reinterpret_cast<double2*>(a.spec_out) + o;
    for (int k = tid; k < B; k += a.tpf) out[k] = buf[k];
  } else {
    float2* out = reinterpret_cast<float2*>(a.spec_out) + o;
    for (int k = tid; k < B; k += a.tpf) out[k] = make_float2((float)buf[k].x, (float)buf[k].y);
  }
}

// float64 frames of fpc consecutive spectra of one stream (see the file comment).
__global__ void __launch_bounds__(kMaxThreads) alz_stft_synthesis_kernel(const __grid_constant__ StftArgs a) {
  extern __shared__ double2 s_buf[];
  const long long s = blockIdx.x / a.blocks_per_stream;
  const long long i0 = (long long)(blockIdx.x % a.blocks_per_stream) * a.fpc;
  const int N = a.size, half = N / 2;
  const int nf = (int)(a.F - i0 < a.fpc ? a.F - i0 : a.fpc);
  const int f = threadIdx.x / a.tpf, tid = threadIdx.x - f * a.tpf;
  const bool active = f < nf;
  double2* buf = s_buf + (long long)f * N;

  if (active) {
    const long long o = s * a.sstride_spec + (i0 + f) * a.fstride;
    for (int k = tid; k <= half; k += a.tpf) {
      double2 X;
      if (a.c128) {
        X = reinterpret_cast<const double2*>(a.spec_in)[o + k];
      } else {
        const float2 v = reinterpret_cast<const float2*>(a.spec_in)[o + k];
        X = make_double2((double)v.x, (double)v.y);
      }
      if (k == 0 || 2 * k == N) X.y = 0.0;
      buf[position(k, a.fft)] = X;
      if (k > 0 && 2 * k < N) buf[position(N - k, a.fft)] = make_double2(X.x, -X.y);
    }
  }
  __syncthreads();
  fft_frame(buf, active, tid, a.tpf, a.fft, a.tw, true);
  if (!active) return;
  const double scale = 1.0 / N;
  double* out = a.frames + (s * a.F + i0 + f) * N;
  for (int n = tid; n < N; n += a.tpf) {
    int p = n;
    if (a.shift) p = n >= half ? n - half : n + (N - half);       // v[n] = v'[(n - half) mod N]
    out[n] = buf[p].x * scale;
  }
}

// Output samples and open sums of one stream's overlap-add (see the file comment).
__global__ void __launch_bounds__(kThreadsOla) alz_ola_kernel(const __grid_constant__ OlaArgs a) {
  const long long blocks = (a.P + kThreadsOla - 1) / kThreadsOla;
  const long long s = blockIdx.x / blocks;
  const long long t = (blockIdx.x % blocks) * kThreadsOla + threadIdx.x;
  if (t >= a.P) return;
  unsigned char* st = a.state + s * a.sstride;
  const int open = a.size - a.hop;
  const int par = *reinterpret_cast<const int*>(st + 8);
  double* const sums = reinterpret_cast<double*>(st + 16);
  const double* cur = sums + (long long)par * open;
  bool have = t < open;
  double acc = have ? cur[t] : 0.0;
  long long k0 = t - a.size + 1 <= 0 ? 0 : (t - a.size + a.hop) / a.hop;   // first frame with k hop + size > t
  long long k1 = t / a.hop;
  if (k1 > a.F - 1) k1 = a.F - 1;
  const double* v64 = reinterpret_cast<const double*>(a.v) + s * a.sstride_v;
  const float* v32 = reinterpret_cast<const float*>(a.v) + s * a.sstride_v;
  for (long long k = k0; k <= k1; ++k) {
    const int j = (int)(t - k * a.hop);
    double v = a.f64 ? v64[k * a.fstride + j] : (double)v32[k * a.fstride + j];
    if (a.w) v = __dmul_rn(a.w[j], v);
    acc = have ? __dadd_rn(acc, v) : v;
    have = true;
  }
  const long long emitted = a.F * a.hop;
  if (t < emitted || a.final_) {
    a.y[s * a.ys + t] = (float)acc;
  } else {
    sums[(long long)(1 - par) * open + (t - emitted)] = acc;
  }
}

__global__ void alz_ola_commit_kernel(unsigned char* state, long long sstride, long long n_streams, long long F) {
  const long long s = blockIdx.x * (long long)blockDim.x + threadIdx.x;
  if (s >= n_streams) return;
  unsigned char* st = state + s * sstride;
  *reinterpret_cast<long long*>(st) += F;
  int* par = reinterpret_cast<int*>(st + 8);
  *par = 1 - *par;
}

// After an analysis call: per stream (one CTA), the last `size` samples and the sample count.
__global__ void __launch_bounds__(kThreadsCommit) alz_stft_commit_kernel(const __grid_constant__ StftArgs a) {
  extern __shared__ float s_t[];
  framed_commit(a.state + blockIdx.x * a.sstride, a.x + blockIdx.x * a.xs, a.T, a.size, s_t);
}

namespace {

int check_shape(int32_t size, int32_t hop) {
  if (size < 1 || size > ALZ_STFT_MAX_SIZE)
    return fail(ALZ_STFT_ERR_INVALID, "size must be in 1 .. %d (got %d)", ALZ_STFT_MAX_SIZE, size);
  if (hop < 1 || hop > size) return fail(ALZ_STFT_ERR_INVALID, "hop must be in 1 .. size (got %d, size %d)", hop, size);
  return ALZ_STFT_OK;
}

int32_t init_state(void* state_dev, long long bytes, cudaStream_t cs) {
  if (bytes == 0) return ALZ_STFT_OK;
  if (!state_dev || ((uintptr_t)state_dev & 7)) return fail(ALZ_STFT_ERR_INVALID, "state is NULL or not 8-byte aligned");
  ALZ_CUDA_CHECK(cudaMemsetAsync(state_dev, 0, bytes, cs), ALZ_STFT_ERR_CUDA);
  return ALZ_STFT_OK;
}

// Launches a transform kernel over n_streams x n_frames frames with the geometry of `size`.
int32_t launch_frames(const void* kernel, StftArgs& a, long long n_streams, cudaStream_t cs) {
  a.fft = factor(a.size);
  a.tpf = threads_per_frame(a.size);
  a.fpc = frames_per_cta(a.size);
  a.blocks_per_stream = (int)((a.F + a.fpc - 1) / a.fpc);
  const long long grid = n_streams * a.blocks_per_stream;
  if (grid > 0x7fffffffLL || a.F > 0x7fffffffLL) return fail(ALZ_STFT_ERR_UNSUPPORTED, "too many frames for one launch");
  const size_t smem = (size_t)a.fpc * a.size * 16;
  ALZ_CUDA_CHECK(allow_dynamic_smem(kernel, smem), ALZ_STFT_ERR_CUDA);
  void* args[] = {&a};
  ALZ_CUDA_CHECK(cudaLaunchKernel(kernel, dim3((unsigned)grid), dim3(a.fpc * a.tpf), args, smem, cs), ALZ_STFT_ERR_CUDA);
  return ALZ_STFT_OK;
}

int32_t ola(const void* v, int f64, int64_t frame_stride, int64_t stream_stride, const double* window_dev,
            float* y_dev, int64_t y_stride, void* state_dev, int64_t n_streams, int64_t n_frames, int32_t size,
            int32_t hop, int32_t final, cudaStream_t cs) {
  if (int rc = check_shape(size, hop)) return rc;
  if (n_streams < 0 || n_frames < 0) return fail(ALZ_STFT_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_STFT_OK;
  const long long P = n_frames * hop + (size - hop);
  const long long emitted = n_frames * hop + (final ? size - hop : 0);
  if (!state_dev || (emitted > 0 && !y_dev) || (n_frames > 0 && !v)) return fail(ALZ_STFT_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)state_dev & 7) || ((uintptr_t)window_dev & 7) || ((uintptr_t)y_dev & 3) ||
      ((uintptr_t)v & (f64 ? 7 : 3)))
    return fail(ALZ_STFT_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && y_stride < emitted) return fail(ALZ_STFT_ERR_INVALID, "y_stride < the samples a stream emits");
  OlaArgs a{};
  a.v = v;
  a.f64 = f64;
  a.w = window_dev;
  a.y = y_dev;
  a.state = (unsigned char*)state_dev;
  a.fstride = frame_stride;
  a.sstride_v = stream_stride;
  a.ys = y_stride;
  a.sstride = ola_state_stride(size, hop);
  a.F = n_frames;
  a.P = P;
  a.size = size;
  a.hop = hop;
  a.final_ = final != 0;
  const long long blocks = n_streams * ((P + kThreadsOla - 1) / kThreadsOla);
  if (P > 0) {
    if (blocks > 0x7fffffffLL) return fail(ALZ_STFT_ERR_UNSUPPORTED, "too many samples for one launch");
    alz_ola_kernel<<<(unsigned)blocks, kThreadsOla, 0, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_STFT_ERR_CUDA);
  }
  alz_ola_commit_kernel<<<(unsigned)((n_streams + 255) / 256), 256, 0, cs>>>(a.state, a.sstride, n_streams, n_frames);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_STFT_ERR_CUDA);
  return ALZ_STFT_OK;
}

}  // namespace

extern "C" {

const char* alz_stft_last_error(void) { return g_err.c_str(); }

int64_t alz_stft_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final) {
  if (consumed < 0 || n_samples < 0) return fail(ALZ_STFT_ERR_INVALID, "need consumed >= 0 and n_samples >= 0");
  if (int rc = check_shape(size, hop)) return rc;
  return emitted_blocks(consumed, n_samples, size, hop, final != 0);
}

int64_t alz_stft_analysis_state_bytes(int64_t n_streams, int32_t size) {
  if (n_streams < 0 || size < 1 || size > ALZ_STFT_MAX_SIZE)
    return fail(ALZ_STFT_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_STFT_MAX_SIZE);
  return n_streams * framed_state_stride(size);
}

int32_t alz_stft_analysis_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream) {
  const int64_t n = alz_stft_analysis_state_bytes(n_streams, size);
  if (n < 0) return (int32_t)n;
  return init_state(state_dev, n, (cudaStream_t)cuda_stream);
}

int64_t alz_stft_ola_state_bytes(int64_t n_streams, int32_t size, int32_t hop) {
  if (n_streams < 0) return fail(ALZ_STFT_ERR_INVALID, "need n_streams >= 0");
  if (int rc = check_shape(size, hop)) return rc;
  return n_streams * ola_state_stride(size, hop);
}

int32_t alz_stft_ola_state_init(void* state_dev, int64_t n_streams, int32_t size, int32_t hop, void* cuda_stream) {
  const int64_t n = alz_stft_ola_state_bytes(n_streams, size, hop);
  if (n < 0) return (int32_t)n;
  return init_state(state_dev, n, (cudaStream_t)cuda_stream);
}

int32_t alz_stft_analysis(const float* x_dev, int64_t x_stride, const double* window_dev, const double* twiddle_dev,
                          void* spec_dev, int32_t spec_c128, int64_t n_frames, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int32_t size, int32_t hop, int32_t shift, int32_t final,
                          void* cuda_stream) {
  if (int rc = check_shape(size, hop)) return rc;
  if (n_streams < 0 || n_samples < 0 || n_frames < 0) return fail(ALZ_STFT_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_STFT_OK;
  if (!state_dev || !twiddle_dev || (n_samples > 0 && !x_dev) || (n_frames > 0 && !spec_dev))
    return fail(ALZ_STFT_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev & 3) || ((uintptr_t)state_dev & 7) || ((uintptr_t)window_dev & 7) ||
      ((uintptr_t)twiddle_dev & 15) || ((uintptr_t)spec_dev & (spec_c128 ? 15 : 7)))
    return fail(ALZ_STFT_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_STFT_ERR_INVALID, "stride < n_samples");
  StftArgs a{};
  a.x = x_dev;
  a.w = window_dev;
  a.tw = reinterpret_cast<const double2*>(twiddle_dev);
  a.spec_out = spec_dev;
  a.state = (unsigned char*)state_dev;
  a.xs = x_stride;
  a.sstride = framed_state_stride(size);
  a.T = n_samples;
  a.F = n_frames;
  a.size = size;
  a.hop = hop;
  a.shift = shift != 0;
  a.c128 = spec_c128 != 0;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  if (n_frames > 0)
    if (int32_t rc = launch_frames((const void*)alz_stft_analysis_kernel, a, n_streams, cs)) return rc;
  if (n_samples > 0) {
    if (n_streams > 0x7fffffffLL) return fail(ALZ_STFT_ERR_UNSUPPORTED, "too many streams for one launch");
    alz_stft_commit_kernel<<<(unsigned)n_streams, kThreadsCommit, (size_t)4 * size, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_STFT_ERR_CUDA);
  }
  return ALZ_STFT_OK;
}

int32_t alz_stft_synthesis(const void* spec_dev, int32_t spec_c128, int64_t frame_stride, int64_t stream_stride,
                           const double* twiddle_dev, int32_t shift, double* frames_dev, const double* ola_window_dev,
                           float* y_dev, int64_t y_stride, void* ola_state_dev, int64_t n_streams, int64_t n_frames,
                           int32_t size, int32_t hop, int32_t final, void* cuda_stream) {
  if (int rc = check_shape(size, hop)) return rc;
  if (n_streams < 0 || n_frames < 0) return fail(ALZ_STFT_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_STFT_OK;
  if (!twiddle_dev || (n_frames > 0 && (!spec_dev || !frames_dev))) return fail(ALZ_STFT_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)spec_dev & (spec_c128 ? 15 : 7)) || ((uintptr_t)twiddle_dev & 15) || ((uintptr_t)frames_dev & 7))
    return fail(ALZ_STFT_ERR_INVALID, "misaligned buffer");
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  if (n_frames > 0) {
    StftArgs a{};
    a.tw = reinterpret_cast<const double2*>(twiddle_dev);
    a.spec_in = spec_dev;
    a.frames = frames_dev;
    a.fstride = frame_stride;
    a.sstride_spec = stream_stride;
    a.F = n_frames;
    a.size = size;
    a.hop = hop;
    a.shift = shift != 0;
    a.c128 = spec_c128 != 0;
    if (int32_t rc = launch_frames((const void*)alz_stft_synthesis_kernel, a, n_streams, cs)) return rc;
  }
  if (!y_dev) return ALZ_STFT_OK;
  return ola(frames_dev, 1, size, n_frames * size, ola_window_dev, y_dev, y_stride, ola_state_dev, n_streams,
             n_frames, size, hop, final, cs);
}

int32_t alz_stft_ola_f64(const double* frames_dev, int64_t frame_stride, int64_t stream_stride,
                         const double* window_dev, float* y_dev, int64_t y_stride, void* ola_state_dev,
                         int64_t n_streams, int64_t n_frames, int32_t size, int32_t hop, int32_t final,
                         void* cuda_stream) {
  return ola(frames_dev, 1, frame_stride, stream_stride, window_dev, y_dev, y_stride, ola_state_dev, n_streams,
             n_frames, size, hop, final, (cudaStream_t)cuda_stream);
}

int32_t alz_stft_ola_f32(const float* frames_dev, int64_t frame_stride, int64_t stream_stride,
                         const double* window_dev, float* y_dev, int64_t y_stride, void* ola_state_dev,
                         int64_t n_streams, int64_t n_frames, int32_t size, int32_t hop, int32_t final,
                         void* cuda_stream) {
  return ola(frames_dev, 0, frame_stride, stream_stride, window_dev, y_dev, y_stride, ola_state_dev, n_streams,
             n_frames, size, hop, final, (cudaStream_t)cuda_stream);
}

}  // extern "C"
