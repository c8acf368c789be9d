// alz_dft.cu -- the C ABI of include/alz_b200_dft.h: the DFT of every frame of S streams at any frequencies, on sm_90a.
//
// Two kernels per call, in stream order:
//   * alz_dft_kernel: the frames x frequencies product of a (frames x samples) and a (samples x frequencies) matrix,
//     with the k order fixed.  A CTA owns a tile of kBM frames (rows of the whole batch, so a tile may span streams)
//     by kBN frequencies and walks the samples n in chunks of kc.  Each chunk stages the float64 frame values b[n]
//     (converted and windowed on the way in: the next chunk's float32 samples are loaded into registers while this
//     one is computed) and the chunk's twiddle rows (cp.async) in shared memory, double-buffered.  Each thread keeps a
//     4 x 4 tile of complex accumulators, rows ty + 16 r and columns tx + 16 c, and adds its terms strictly in n
//     order with __dmul_rn / __dadd_rn: per n it loads 4 frame values and 4 twiddles (12 doubles) and issues 64 FP64
//     instructions.  A frame inside the call's samples is read straight from x; one that starts before them (its first
//     samples are in the state's tail) or ends after them (the padded last frame) goes through FramedSamples;
//   * alz_dft_commit_kernel: one CTA per stream shifts the last `size` samples into the state and counts the samples.
//
// The unit is compiled with -fmad=false, and the host twiddles with -ffp-contract=off: nothing is contracted.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_dft.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace {

constexpr int kBM = 64;                      // frames per CTA tile
constexpr int kBN = 64;                      // frequencies per CTA tile
constexpr int kBK = 32;                      // samples per chunk (at most)
constexpr int kThreads = 256;                // 16 x 16 threads, each a 4 x 4 register tile
constexpr int kLoads = kBM * kBK / kThreads; // frame values a thread stages per chunk
constexpr int kThreadsCommit = 256;
constexpr long long kSlow = -1;              // row offsets: a frame read through FramedSamples
constexpr long long kNone = -2;              //              a row past the batch

struct DftArgs {
  const float* x;
  const double* w;
  const double2* tw;      // [size][nf]
  void* out;
  unsigned char* state;
  long long xs, sstride, T, F, R;   // R = streams * F rows
  int nf, size, hop, kc, normalize, c128;
};

// Chunk length: kBK, or the frame rounded up to 8 samples when it is shorter.
int chunk(int size) { return size < kBK ? (size + 7) / 8 * 8 : kBK; }

__host__ __device__ inline size_t stage_bytes(int kc) { return (size_t)kc * kBN * 16 + (size_t)kc * (kBM + 1) * 8; }

__device__ __forceinline__ void cp_async16(void* dst, const void* src, bool valid) {
  const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(src), "r"(valid ? 16 : 0));
}

// The one correctly rounded division of the library (CPython's `/`), kept out of line: its Newton steps are the only
// fused multiply-adds in the library, and they do not change its IEEE result.
__device__ __noinline__ double quot(double num, double den) { return __ddiv_rn(num, den); }

}  // namespace

// One kBM x kBN tile of frames x frequencies (see the file comment).
__global__ void __launch_bounds__(kThreads, 2) alz_dft_kernel(const __grid_constant__ DftArgs a) {
  extern __shared__ __align__(16) unsigned char s_raw[];   // per stage: twiddles [kc][kBN], then b [kc][kBM + 1]
  __shared__ long long s_off[kBM], s_str[kBM], s_g0[kBM];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const long long r0 = (long long)blockIdx.x * kBM;
  const int f0 = blockIdx.y * kBN;
  const int size = a.size, kc = a.kc;

  if (tid < kBM) {
    const long long r = r0 + tid;
    long long off = kNone, s = 0, g0 = 0;
    if (r < a.R) {
      s = r / a.F;
      const long long i = r - s * a.F;
      const long long C = *reinterpret_cast<const long long*>(a.state + s * a.sstride);
      g0 = (first_open_block(C, size, a.hop) + i) * a.hop;
      off = (g0 >= C && g0 + size <= C + a.T) ? s * a.xs + (g0 - C) : kSlow;
    }
    s_off[tid] = off;
    s_str[tid] = s;
    s_g0[tid] = g0;
  }
  __syncthreads();

  const size_t sbytes = stage_bytes(kc);
  double2* stw[2] = {reinterpret_cast<double2*>(s_raw), reinterpret_cast<double2*>(s_raw + sbytes)};
  double* sb[2] = {reinterpret_cast<double*>(s_raw + (size_t)kc * kBN * 16),
                   reinterpret_cast<double*>(s_raw + sbytes + (size_t)kc * kBN * 16)};

  // the twiddle rows n0 .. n0 + kc - 1 of the tile's columns; zeros past the table
  auto issue_twiddles = [&](double2* dst, int n0) {
    for (int e = tid; e < kc * kBN; e += kThreads) {
      const int kk = e / kBN, c = e - kk * kBN;
      const int n = n0 + kk, f = f0 + c;
      const bool ok = n < size && f < a.nf;
      cp_async16(dst + e, ok ? a.tw + (long long)n * a.nf + f : a.tw, ok);
    }
    asm volatile("cp.async.commit_group;\n" ::);
  };
  float v[kLoads];
  auto fetch = [&](int n0) {
#pragma unroll
    for (int j = 0; j < kLoads; ++j) {
      const int e = tid + j * kThreads;
      v[j] = 0.f;
      if (e < kBM * kc) {
        const int m = e / kc, n = n0 + e - m * kc;
        const long long off = s_off[m];
        if (n < size) {
          if (off >= 0) v[j] = a.x[off + n];
          else if (off == kSlow)
            v[j] = framed_samples(a.state + s_str[m] * a.sstride, a.x + s_str[m] * a.xs, a.T, size)(s_g0[m] + n);
        }
      }
    }
  };
  auto put = [&](double* dst, int n0) {
#pragma unroll
    for (int j = 0; j < kLoads; ++j) {
      const int e = tid + j * kThreads;
      if (e < kBM * kc) {
        const int m = e / kc, kk = e - m * kc, n = n0 + kk;
        double b = (double)v[j];
        if (a.w && n < size) b = __dmul_rn(b, a.w[n]);
        dst[kk * (kBM + 1) + m] = b;
      }
    }
  };

  double re[4][4], im[4][4];
#pragma unroll
  for (int r = 0; r < 4; ++r)
#pragma unroll
    for (int c = 0; c < 4; ++c) re[r][c] = im[r][c] = 0.0;

  issue_twiddles(stw[0], 0);
  fetch(0);
  put(sb[0], 0);
  asm volatile("cp.async.wait_group 0;\n" ::);
  __syncthreads();
  const int nchunks = (size + kc - 1) / kc;
  for (int ch = 0; ch < nchunks; ++ch) {
    const int cur = ch & 1;
    const bool more = ch + 1 < nchunks;
    if (more) issue_twiddles(stw[cur ^ 1], (ch + 1) * kc);
    const double* b = sb[cur];
    const double2* t = stw[cur];
    const int kmax = size - ch * kc < kc ? size - ch * kc : kc;
#pragma unroll 2
    for (int kk = 0; kk < kmax; ++kk) {
      double bv[4];
      double2 wv[4];
#pragma unroll
      for (int r = 0; r < 4; ++r) bv[r] = b[kk * (kBM + 1) + ty + 16 * r];
#pragma unroll
      for (int c = 0; c < 4; ++c) wv[c] = t[kk * kBN + tx + 16 * c];
#pragma unroll
      for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          re[r][c] = __dadd_rn(re[r][c], __dmul_rn(bv[r], wv[c].x));
          im[r][c] = __dadd_rn(im[r][c], __dmul_rn(bv[r], wv[c].y));
        }
    }
    if (more) {
      fetch((ch + 1) * kc);
      put(sb[cur ^ 1], (ch + 1) * kc);
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();
  }

  const double L = (double)size;
#pragma unroll
  for (int r = 0; r < 4; ++r) {
    const long long row = r0 + ty + 16 * r;
    if (row >= a.R) continue;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int f = f0 + tx + 16 * c;
      if (f >= a.nf) continue;
      double yr = re[r][c], yi = im[r][c];
      if (a.normalize) {                         // CPython's _Py_c_quot by complex(size, 0.0)
        const double qr = quot(__dadd_rn(yr, __dmul_rn(yi, 0.0)), L);
        const double qi = quot(__dsub_rn(yi, __dmul_rn(yr, 0.0)), L);
        yr = qr;
        yi = qi;
      }
      const long long o = row * a.nf + f;
      if (a.c128) reinterpret_cast<double2*>(a.out)[o] = make_double2(yr, yi);
      else reinterpret_cast<float2*>(a.out)[o] = make_float2(__double2float_rn(yr), __double2float_rn(yi));
    }
  }
}

// After a call's frames: per stream (one CTA), the last `size` samples and the sample count.
__global__ void __launch_bounds__(kThreadsCommit) alz_dft_commit_kernel(const __grid_constant__ DftArgs a) {
  extern __shared__ float s_t[];
  framed_commit(a.state + blockIdx.x * a.sstride, a.x + blockIdx.x * a.xs, a.T, a.size, s_t);
}

extern "C" {

const char* alz_dft_last_error(void) { return g_err.c_str(); }

int64_t alz_dft_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final) {
  if (consumed < 0 || n_samples < 0 || size < 1 || hop < 1)
    return fail(ALZ_DFT_ERR_INVALID, "need consumed >= 0, n_samples >= 0, size >= 1, hop >= 1");
  return emitted_blocks(consumed, n_samples, size, hop, final != 0);
}

int64_t alz_dft_state_bytes(int64_t n_streams, int32_t size) {
  if (n_streams < 0 || size < 1 || size > ALZ_DFT_MAX_SIZE)
    return fail(ALZ_DFT_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_DFT_MAX_SIZE);
  return n_streams * framed_state_stride(size);
}

int32_t alz_dft_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream) {
  if (n_streams < 0 || size < 1 || size > ALZ_DFT_MAX_SIZE)
    return fail(ALZ_DFT_ERR_INVALID, "need n_streams >= 0 and 1 <= size <= %d", ALZ_DFT_MAX_SIZE);
  if (n_streams == 0) return ALZ_DFT_OK;
  if (!state_dev || ((uintptr_t)state_dev & 7)) return fail(ALZ_DFT_ERR_INVALID, "state is NULL or not 8-byte aligned");
  ALZ_CUDA_CHECK(cudaMemsetAsync(state_dev, 0, n_streams * framed_state_stride(size), (cudaStream_t)cuda_stream),
                 ALZ_DFT_ERR_CUDA);
  return ALZ_DFT_OK;
}

int64_t alz_dft_twiddles(const double* freqs, int32_t n_freqs, int32_t size, double* table, uint8_t* unfilled) {
  if (n_freqs < 0 || size < 0) return fail(ALZ_DFT_ERR_INVALID, "need n_freqs >= 0 and size >= 0");
  if ((n_freqs > 0 && (!freqs || !unfilled)) || ((long long)n_freqs * size > 0 && !table))
    return fail(ALZ_DFT_ERR_INVALID, "NULL buffer");
  int64_t missing = 0;
  for (int j = 0; j < n_freqs; ++j) {
    const double f = freqs[j];
    bool ok = true;
    for (int n = 0; n < size && ok; ++n) {
      // -1j * n: (-0.0, -1.0) * (n, 0.0)
      const double nn = (double)n;
      const double ar = -0.0, ai = -1.0;
      const double z1r = ar * nn - ai * 0.0, z1i = ar * 0.0 + ai * nn;
      // * f: (z1r, z1i) * (f, 0.0)
      const double zr = z1r * f - z1i * 0.0, zi = z1r * 0.0 + z1i * f;
      // cmath.exp's finite path with z.real = 0.0 <= log(DBL_MAX) - 1: l = exp(0.0) = 1.0, (l cos(y), l sin(y))
      if (!(zr == 0.0 && !std::signbit(zr) && std::isfinite(zi))) {
        ok = false;
        break;
      }
      const double l = std::exp(zr);
      double* t = table + 2 * ((long long)n * n_freqs + j);
      t[0] = l * std::cos(zi);
      t[1] = l * std::sin(zi);
    }
    unfilled[j] = ok ? 0 : 1;
    missing += ok ? 0 : 1;
  }
  return missing;
}

int32_t alz_dft_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, const double* twiddles_dev,
                          int32_t n_freqs, int32_t normalize, void* out_dev, int32_t out_c128, int64_t n_frames,
                          void* state_dev, int64_t n_streams, int64_t n_samples, int32_t size, int32_t hop,
                          int32_t final, void* cuda_stream) {
  if (size < 1 || size > ALZ_DFT_MAX_SIZE)
    return fail(ALZ_DFT_ERR_INVALID, "size must be in 1 .. %d (got %d)", ALZ_DFT_MAX_SIZE, size);
  if (hop < 1) return fail(ALZ_DFT_ERR_INVALID, "hop must be >= 1 (got %d)", hop);
  if (n_freqs < 1 || n_freqs > ALZ_DFT_MAX_FREQS)
    return fail(ALZ_DFT_ERR_INVALID, "n_freqs must be in 1 .. %d (got %d)", ALZ_DFT_MAX_FREQS, n_freqs);
  if (n_streams < 0 || n_samples < 0 || n_frames < 0) return fail(ALZ_DFT_ERR_INVALID, "bad shape");
  if (n_streams == 0) return ALZ_DFT_OK;
  if (!state_dev || !twiddles_dev || (n_samples > 0 && !x_dev) || (n_frames > 0 && !out_dev))
    return fail(ALZ_DFT_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev & 3) || ((uintptr_t)state_dev & 7) || ((uintptr_t)window_dev & 7) ||
      ((uintptr_t)twiddles_dev & 15) || ((uintptr_t)out_dev & (out_c128 ? 15 : 7)))
    return fail(ALZ_DFT_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && x_stride < n_samples) return fail(ALZ_DFT_ERR_INVALID, "stride < n_samples");
  DftArgs a{};
  a.x = x_dev;
  a.w = window_dev;
  a.tw = reinterpret_cast<const double2*>(twiddles_dev);
  a.out = out_dev;
  a.state = (unsigned char*)state_dev;
  a.xs = x_stride;
  a.sstride = framed_state_stride(size);
  a.T = n_samples;
  a.F = n_frames;
  a.nf = n_freqs;
  a.size = size;
  a.hop = hop;
  a.kc = chunk(size);
  a.normalize = normalize != 0;
  a.c128 = out_c128 != 0;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  if (n_frames > 0) {
    if (n_frames > 0x7fffffffLL * kBM / n_streams) return fail(ALZ_DFT_ERR_UNSUPPORTED, "too many frames for one launch");
    a.R = n_streams * n_frames;
    const dim3 grid((unsigned)((a.R + kBM - 1) / kBM), (unsigned)((n_freqs + kBN - 1) / kBN));
    const size_t smem = 2 * stage_bytes(a.kc);
    ALZ_CUDA_CHECK(allow_dynamic_smem((const void*)alz_dft_kernel, smem), ALZ_DFT_ERR_CUDA);
    alz_dft_kernel<<<grid, kThreads, smem, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_DFT_ERR_CUDA);
  }
  if (n_samples > 0) {
    alz_dft_commit_kernel<<<(unsigned)n_streams, kThreadsCommit, (size_t)4 * size, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_DFT_ERR_CUDA);
  }
  return ALZ_DFT_OK;
}

}  // extern "C"
