// alz_capi.cu -- the C ABI of include/alz_b200.h: plan building, state seeding,
// kernel dispatch and the host-buffer pipeline.  No torch types, no CPU compute path.
#pragma GCC visibility push(default)
#include "../../include/alz_b200.h"
#pragma GCC visibility pop
#include "alz_biquad.cuh"
#include "alz_generic.cuh"
#include "alz_lane_tma.cuh"
#include "alz_plan.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstring>
#include <map>
#include <memory>
#include <thread>

#include <sys/mman.h>
#include <sys/syscall.h>
#include <unistd.h>

static std::mutex g_host_mu;
static std::map<void*, size_t> g_host_allocs;   // alz_host_alloc bookkeeping

static_assert(ALZI_OK == ALZ_OK && ALZI_ERR_CUDA == ALZ_ERR_CUDA && ALZI_ERR_UNSUPPORTED == ALZ_ERR_UNSUPPORTED, "status codes");

// ----------------------------------------------------------------------------------
// error plumbing
// ----------------------------------------------------------------------------------
static thread_local std::string g_err;
std::atomic<long long> alzi_launches{0};
#define g_launches alzi_launches

int alzi_fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define fail alzi_fail

int alzi_env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atoi(v) : dflt;
}
#define env_int alzi_env_int

static double env_double(const char* name, double dflt) {
  const char* v = getenv(name);
  return (v && *v) ? atof(v) : dflt;
}

// Keep the stream-ordered pool's memory across calls (its default trims at every sync).
void alzi_keep_async_pool() {
  static std::once_flag once[64];
  int dev = 0;
  cudaGetDevice(&dev);
  std::call_once(once[dev & 63], [dev] {
    cudaMemPool_t pool;
    if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
      unsigned long long keep = ~0ull;
      cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
    }
    cudaGetLastError();
  });
}
#define keep_async_pool alzi_keep_async_pool

static const int kCoefSmall = 512, kCoefLarge = 3584;   // as in alz_launch.cuh

__global__ void __launch_bounds__(32)
alz_generic_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzGenericArgs ca) {
  extern __shared__ __align__(16) float alz_smem[];
  alz_run_warp<AlzGenericCore>(a, ca, alz_smem);
}

__global__ void __launch_bounds__(32)
alz_generic_tma_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzGenericArgs ca,
                       const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy) {
  extern __shared__ __align__(1024) unsigned char alz_smem_tma[];
  alz_run_warp_tma<AlzGenericCore>(a, ca, &tmx, &tmy, alz_smem_tma);
}

// ---- tensor maps (driver entry point fetched through the runtime: no libcuda link) -------
typedef CUresult (*alz_encode_tiled_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                        const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                        CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static alz_encode_tiled_fn get_encode_tiled() {
  static alz_encode_tiled_fn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (alz_encode_tiled_fn)p;
    cudaGetLastError();
  });
  return fn;
}

template <class F>
static bool driver_fn(const char* name, F* out) {
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess || !p) {
    cudaGetLastError();
    return false;
  }
  *out = (F)p;
  return true;
}
static std::map<void*, CUgreenCtx> g_partitions;

// x[S][T] (row stride xs) and y[S][C][T] (row stride ys) as tiled tensor maps with 32-sample boxes.
bool alzi_make_tensor_maps(const AlzTileArgs& ta, CUtensorMap* tmx, CUtensorMap* tmy) {
  alz_encode_tiled_fn enc = get_encode_tiled();
  if (!enc || !ta.vec_in || !ta.vec_out || env_int("ALZ_NO_TMA", 0)) return false;
  if (ta.T >= (1ll << 31) || ta.S >= (1ll << 31)) return false;
  if ((unsigned long long)ta.xs * 4 >= (1ull << 40) || (unsigned long long)ta.ysS * 4 >= (1ull << 40)) return false;
  if (ta.ysS & 3) return false;
  const cuuint32_t estr[4] = {1, 1, 1, 1};
  if (ta.vP > 0) {
    // virtual streams: row v = chunk v % P of real stream v / P; T = chunk length, xs / ys / ysS = the REAL strides
    const cuuint64_t P = (cuuint64_t)ta.vP, Sreal = (cuuint64_t)(ta.S / ta.vP);
    const cuuint64_t xdims[3] = {(cuuint64_t)ta.T, P, Sreal};
    const cuuint64_t xstr[2] = {(cuuint64_t)ta.T * 4, (cuuint64_t)ta.xs * 4};
    const cuuint32_t xbox[3] = {32, 32, 1};
    if (enc(tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)ta.x, xdims, xstr, xbox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
    const cuuint64_t ydims[4] = {(cuuint64_t)ta.T, P, (cuuint64_t)ta.C, Sreal};
    const cuuint64_t ystr[3] = {(cuuint64_t)ta.T * 4, (cuuint64_t)ta.ys * 4, (cuuint64_t)ta.ysS * 4};
    const cuuint32_t ybox[4] = {32, 32, 1, 1};
    return enc(tmy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)ta.y, ydims, ystr, ybox, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
               CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
  }
  {
    // real streams, same ranks as the virtual case so that the kernels have ONE code path: x (T, S, 1), y (T, C, S, 1)
    const cuuint64_t dims[3] = {(cuuint64_t)ta.T, (cuuint64_t)ta.S, 1};
    const cuuint64_t strides[2] = {(cuuint64_t)ta.xs * 4, (cuuint64_t)ta.xs * 4};
    const cuuint32_t box[3] = {32, 32, 1};
    if (enc(tmx, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, (void*)ta.x, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
  }
  {
    const cuuint64_t dims[4] = {(cuuint64_t)ta.T, (cuuint64_t)ta.C, (cuuint64_t)ta.S, 1};
    const cuuint64_t strides[3] = {(cuuint64_t)ta.ys * 4, (cuuint64_t)ta.ysS * 4, (cuuint64_t)ta.ysS * 4};
    const cuuint32_t box[4] = {32, 1, 32, 1};
    if (enc(tmy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)ta.y, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
  }
  return true;
}

// rows[n_rows][T] float32 (row stride `stride` elements) with 32 x 32 boxes
static bool make_map_2d(const float* ptr, long long T, long long n_rows, long long stride, CUtensorMap* tm) {
  alz_encode_tiled_fn enc = get_encode_tiled();
  if (!enc || ((uintptr_t)ptr & 15) || (stride & 3) || T >= (1ll << 31) || n_rows >= (1ll << 31)) return false;
  const cuuint32_t estr[2] = {1, 1};
  const cuuint64_t dims[2] = {(cuuint64_t)T, (cuuint64_t)n_rows};
  const cuuint64_t strides[1] = {(cuuint64_t)stride * 4};
  const cuuint32_t box[2] = {32, 32};
  return enc(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)ptr, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
             CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int launch_biquad(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  if (p->NB0 == 8) {
    if (p->K == 1) return alzi_launch_headfir_k1(p, ta, st);
    if (p->K == 4) return alzi_launch_headfir_k4(p, ta, st);
    return fail(ALZ_ERR_UNSUPPORTED, "no head-FIR kernel for K=%d", p->K);
  }
  switch (p->K) {
    case 1: return alzi_launch_biquad_k1(p, ta, st);
    case 2: return alzi_launch_biquad_k2(p, ta, st);
    case 3: return alzi_launch_biquad_k3(p, ta, st);
    case 4: return alzi_launch_biquad_k4(p, ta, st);
    case 6: return alzi_launch_biquad_k6(p, ta, st);
    case 8: return alzi_launch_biquad_k8(p, ta, st);
  }
  return fail(ALZ_ERR_UNSUPPORTED, "no biquad kernel for K=%d", p->K);
}

static double probe_biquad(const alz_plan* p, const double* r64, const double* r32) {
  if (p->NB0 == 8) return p->K == 1 ? alzi_probe_headfir_k1(p, r64, r32) : alzi_probe_headfir_k4(p, r64, r32);
  switch (p->K) {
    case 1: return alzi_probe_biquad_k1(p, r64, r32);
    case 2: return alzi_probe_biquad_k2(p, r64, r32);
    case 3: return alzi_probe_biquad_k3(p, r64, r32);
    case 4: return alzi_probe_biquad_k4(p, r64, r32);
    case 6: return alzi_probe_biquad_k6(p, r64, r32);
    default: return alzi_probe_biquad_k8(p, r64, r32);
  }
}

static int launch_generic(const alz_plan* p, AlzTileArgs ta, cudaStream_t st, const double* tv = nullptr,
                          long long tv_stride = 0) {
  AlzGenericArgs ga{p->d_sec, p->d_tap_delay, p->d_coef, p->K, p->C, 0, tv, tv_stride};
  const long long groups = (ta.S + 31) / 32;
  CUtensorMap tmx, tmy;
  if (alzi_make_tensor_maps(ta, &tmx, &tmy))
    alz_generic_tma_kernel<<<dim3((unsigned)p->C, (unsigned)groups), 32, ALZ_TMA_SMEM, st>>>(ta, ga, tmx, tmy);
  else
    alz_generic_kernel<<<dim3((unsigned)p->C, (unsigned)groups), 32, ALZ_WARP_SMEM, st>>>(ta, ga);
  ALZ_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZ_OK;
}

static const int kBiquadKs[] = {1, 2, 3, 4, 6, 8};
// a channel with a pole farther out than this is never put on the float32 tier, whatever its probe measures
static const double kTierMaxRadius = 0.99;
// The time-parallel evaluation adds a chunk's zero-state response F to the free response M s of its true initial
// state.  When a numerator cancels (gammatone.sampled's head FIR at high rates: ~w^3 of its input) both are far larger
// than the output, and their float64 rounding does not cancel.  A plan whose measured chunk error exceeds this is
// always evaluated sequentially.  The error compounds over the chunks of a stream: over 10^6 samples the sampled
// 192 kHz bank measured 9.6e-7 here and 3.9e-4 (400 times) against the oracle, so the limit keeps 400 times it
// within the 1e-5 bar.  The 48 kHz sampled bank measures 2.1e-8 and stays within 3e-6 time-parallel.
static const double kChunkMaxErr = 2.5e-8;
static const long long kChunkProbeLen = 1024;          // about the chunk length the cost model picks for 10^6 samples
static const int kTileGroup4MaxFp64 = 16;               // most FP64 instructions per channel-sample for tile group 4

struct Sec { std::vector<double> b, a; };   // one section of a cascade; a[0] == 1 after normalisation (kept for indexing)

// One chunk transition of one channel (sections (b, a), a[0] == 1) in plain float64 Direct Form I, on noise: the state
// after 2L samples, F + M s as the time-parallel evaluation forms it, against the sequential state; both then filter the
// next L samples.  Returns max |difference| / max |sequential output| over those samples.
template <class Sec>
static double chunk_error(const std::vector<Sec>& secs, long long L) {
  const size_t K = secs.size();
  struct Hist { std::vector<std::vector<double>> x, y; };
  auto zero = [&]() {
    Hist h;
    for (const Sec& s : secs) { h.x.emplace_back(s.b.size() - 1, 0.0); h.y.emplace_back(s.a.size() - 1, 0.0); }
    return h;
  };
  auto step = [&](Hist& h, double v) {
    for (size_t k = 0; k < K; ++k) {
      const Sec& s = secs[k];
      std::vector<double>& xh = h.x[k];
      std::vector<double>& yh = h.y[k];
      double acc = s.b[0] * v;
      for (size_t j = 1; j < s.b.size(); ++j) acc += s.b[j] * xh[j - 1];
      for (size_t j = 1; j < s.a.size(); ++j) acc -= s.a[j] * yh[j - 1];
      if (!xh.empty()) { std::copy_backward(xh.begin(), xh.end() - 1, xh.end()); xh[0] = v; }
      if (!yh.empty()) { std::copy_backward(yh.begin(), yh.end() - 1, yh.end()); yh[0] = acc; }
      v = acc;
    }
    return v;
  };
  std::vector<double> x(3 * L);
  unsigned seed = 2024u;
  for (auto& v : x) { seed = seed * 1664525u + 1013904223u; v = (double)(float)((double)(seed >> 8) * (2.0 / 16777216.0) - 1.0); }
  Hist seq = zero();
  for (long long n = 0; n < L; ++n) step(seq, x[n]);
  Hist chunk = seq;                                   // -> M s: the state's response to L zero samples
  for (long long n = 0; n < L; ++n) step(chunk, 0.0);
  Hist f = zero();                                    // F: the second chunk from a zero state
  for (long long n = L; n < 2 * L; ++n) { step(seq, x[n]); step(f, x[n]); }
  for (size_t k = 0; k < K; ++k) {
    for (size_t j = 0; j < chunk.x[k].size(); ++j) chunk.x[k][j] += f.x[k][j];
    for (size_t j = 0; j < chunk.y[k].size(); ++j) chunk.y[k][j] += f.y[k][j];
  }
  double peak = 0.0, err = 0.0;
  for (long long n = 2 * L; n < 3 * L; ++n) {
    const double want = step(seq, x[n]), got = step(chunk, x[n]);
    peak = std::max(peak, std::fabs(want));
    const double d = std::fabs(got - want);
    err = std::max(err, d == d ? d : 1e300);
  }
  return peak > 0.0 ? err / peak : (err > 0.0 ? 1e300 : 0.0);
}

// Makes a plan's device current for the rest of the scope and gives the caller's device back on every return path.
struct DeviceScope {
  int prev = -1;
  bool switched = false;
  cudaError_t status;
  explicit DeviceScope(int device) {
    status = cudaGetDevice(&prev);
    if (status == cudaSuccess && prev != device) {
      status = cudaSetDevice(device);
      switched = status == cudaSuccess;
    }
  }
  ~DeviceScope() { if (switched) cudaSetDevice(prev); }
};

// Device scratch from the stream-ordered pool, freed on `st` when the scope ends (on every return path): after the
// work already queued there, so the caller only has to make sure every other stream that uses it is done.
template <class T>
struct StreamScratch {
  T* ptr = nullptr;
  cudaStream_t st;
  explicit StreamScratch(cudaStream_t s) : st(s) {}
  ~StreamScratch() { if (ptr) cudaFreeAsync(ptr, st); }
  StreamScratch(const StreamScratch&) = delete;
  StreamScratch& operator=(const StreamScratch&) = delete;
  cudaError_t alloc(size_t n) { return cudaMallocAsync((void**)&ptr, n * sizeof(T), st); }
};
// A buffer of cudaMalloc, freed when the scope ends.  The host entries size theirs by the whole batch: the pool, which
// keeps what it is given back once the time-parallel evaluation has run, would hold on to it after the call.
typedef std::unique_ptr<double, cudaError_t (*)(void*)> DeviceBuffer;

// A plan's host table and the device pointer of the plan that receives its copy.
struct Upload { void** dst; const void* src; size_t bytes; };
template <class T>
static Upload table(T** dst, const std::vector<T>& src) { return {(void**)dst, src.data(), src.size() * sizeof(T)}; }

// Copies a plan's tables to its device: sets every destination, or none of them when a step fails.  A design-only
// plan has no device and keeps them null.
static int upload_tables(const alz_plan* p, std::initializer_list<Upload> tables) {
  if (p->device < 0) return ALZ_OK;
  std::vector<void*> got;
  cudaError_t e = cudaSuccess;
  for (const Upload& t : tables) {
    void* d = nullptr;
    e = cudaMalloc(&d, std::max<size_t>(1, t.bytes));
    if (e != cudaSuccess) break;
    got.push_back(d);
    e = cudaMemcpy(d, t.src, t.bytes, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) break;
  }
  if (e != cudaSuccess) {
    for (void* d : got) cudaFree(d);
    return fail(ALZ_ERR_CUDA, "plan upload failed: %s", cudaGetErrorString(e));
  }
  size_t i = 0;
  for (const Upload& t : tables) *t.dst = got[i++];
  return ALZ_OK;
}

// ---- the plan's host staging pipeline (alz_apply_f32_host, envelope_host) ---------------------------------------------
// Creates the pipeline's streams and events on first use.  after_legacy: the ordering contract of include/alz_b200.h for
// a caller-supplied state, which must be complete or produced by work on the legacy default stream (where torch launches
// by default): the private pipeline streams are ordered after it.
static int pipe_open(AlzHostPipe& hp, bool after_legacy) {
  if (!hp.ready) {
    for (int i = 0; i < AlzHostPipe::NBUF; ++i) {
      ALZ_CUDA(cudaStreamCreateWithFlags(&hp.stream[i], cudaStreamNonBlocking));
      ALZ_CUDA(cudaEventCreateWithFlags(&hp.done[i], cudaEventDisableTiming));
    }
    hp.ready = true;
  }
  if (after_legacy) {
    ALZ_CUDA(cudaEventRecord(hp.done[0], cudaStreamLegacy));
    for (int i = 0; i < AlzHostPipe::NBUF; ++i) ALZ_CUDA(cudaStreamWaitEvent(hp.stream[i], hp.done[0], 0));
  }
  return ALZ_OK;
}

// Grows one staging buffer per pipeline stream to `need` bytes; they are kept in the plan between calls.
template <class T>
static int pipe_grow(AlzHostPipe& hp, T** bufs, size_t& have, size_t need) {
  if (have >= need) return ALZ_OK;
  for (int i = 0; i < AlzHostPipe::NBUF; ++i) {
    ALZ_CUDA(cudaStreamSynchronize(hp.stream[i]));
    cudaFree(bufs[i]);
    bufs[i] = nullptr;
  }
  have = 0;
  for (int i = 0; i < AlzHostPipe::NBUF; ++i) ALZ_CUDA(cudaMalloc((void**)&bufs[i], need));
  have = need;
  return ALZ_OK;
}

// Waits for every pipeline stream: returns rc, or the first error they report if rc is ALZ_OK.
static int pipe_finish(AlzHostPipe& hp, int rc) {
  for (int i = 0; i < AlzHostPipe::NBUF; ++i) {
    const cudaError_t e = cudaStreamSynchronize(hp.stream[i]);
    if (e != cudaSuccess && rc == ALZ_OK) rc = fail(ALZ_ERR_CUDA, "pipeline failed: %s", cudaGetErrorString(e));
  }
  return rc;
}

// ---- plan builders, one per kind: the tables of the normalised sections `secs` ([channel][section]) ----
static int build_biquad(alz_plan* p, const std::vector<std::vector<Sec>>& secs, int Kmax, int nbmax, int nb_rest,
                        bool headfir, int flags) {
  const int C = p->C;
  int K = 8;
  for (int kk : kBiquadKs) if (kk >= Kmax) { K = kk; break; }
  if (headfir) K = Kmax == 1 ? 1 : 4;
  p->kind = ALZ_KIND_BIQUAD;
  p->K = K;
  p->NB = headfir ? (nb_rest <= 1 ? 1 : 3) : nbmax;
  p->NB0 = headfir ? 8 : 0;
  p->xd = ALZ_H0(p->NB0); p->yd = 2;
  p->state_doubles = ALZ_STATE_SLOTS(K, p->NB0);
  // monic only if every b0 is a normal number and the running products stay normal
  bool monic = !p->parallel_sum;          // ParallelFilter plans keep plain sections: the channel outputs are summed in true units
  for (int c = 0; c < C && monic; ++c) {
    double g = 1.0;
    for (auto& s : secs[c]) {
      const double b0 = s.b[0];
      if (!(std::fabs(b0) > 1e-150 && std::fabs(b0) < 1e150)) { monic = false; break; }
      g *= b0;
      if (!(std::fabs(g) > 1e-250 && std::fabs(g) < 1e250)) { monic = false; break; }
    }
  }
  // input-side float32 gain (mode 2) when every channel's G is a normal float32 number
  bool gain_in = monic && !env_int("ALZ_EXACT_GAIN", 0);
  for (int c = 0; c < C && gain_in; ++c) {
    double g = 1.0;
    for (auto& s : secs[c]) g *= s.b[0];
    if (!(std::fabs(g) > 1e-30 && std::fabs(g) < 1e30)) gain_in = false;
  }
  p->monic = monic ? (gain_in ? 2 : 1) : 0;
  p->fp64_ops = (monic ? K * (p->NB - 1 + 2) + (gain_in ? 0 : 1) : K * (p->NB + 2)) + (headfir ? 8 - p->NB : 0);
  if (!headfir && !env_int("ALZ_NO_ZMASK", 0)) {   // taps 1 and 2 that no channel has (absent sections count as zero)
    int zm = (1 << (2 * K)) - 1;
    for (int c = 0; c < C; ++c)
      for (size_t k = 0; k < secs[c].size(); ++k)
        for (int j = 1; j <= 2; ++j)
          if ((int)secs[c][k].b.size() > j && secs[c][k].b[j] != 0.0) zm &= ~(1 << (2 * (int)k + j - 1));
    p->zmask = zm;
    if (K == 4 && p->NB == 3 && (zm & ALZ_ZMASK_KLAPURI) == ALZ_ZMASK_KLAPURI) p->fp64_ops -= 6;   // the kernel that skips them
  }
  const int stride = ALZ_COEF_STRIDE(K, p->NB0), nval = ALZ_COEF_NVAL(K, p->NB0);
  std::vector<double> tab((size_t)C * stride, 0.0);     // channel order, float64 records
  p->sc.assign((size_t)C * (K + 1), 1.0);
  for (int c = 0; c < C; ++c) {
    double* rec = tab.data() + (size_t)c * stride;
    double g = 1.0, sc = 1.0;
    if (p->monic == 2) {   // working units start at the (float32-rounded) gain applied to the input
      double gg = 1.0;
      for (auto& s : secs[c]) gg *= s.b[0];
      sc = (double)(float)gg;
      p->sc[(size_t)c * (K + 1)] = sc;
    }
    for (int k = 0; k < K; ++k) {
      double b[8] = {1.0, 0, 0, 0, 0, 0, 0, 0}, a[3] = {1.0, 0.0, 0.0};   // identity padding
      if (k < (int)secs[c].size()) {
        const Sec& s = secs[c][k];
        b[0] = 0.0;
        for (size_t i = 0; i < s.b.size(); ++i) b[i] = s.b[i];
        for (size_t i = 0; i < s.a.size(); ++i) a[i] = s.a[i];
      }
      if (k == 0 && p->NB0 == 8)
        for (int j = 3; j < 8; ++j) rec[5 * K + 1 + (j - 3)] = monic ? b[j] / b[0] : b[j];
      if (monic) {
        rec[5 * k + 0] = 1.0;
        rec[5 * k + 1] = b[1] / b[0];
        rec[5 * k + 2] = b[2] / b[0];
        g *= b[0];
        sc /= b[0];
      } else {
        rec[5 * k + 0] = b[0];
        rec[5 * k + 1] = b[1];
        rec[5 * k + 2] = b[2];
      }
      rec[5 * k + 3] = -a[1];
      rec[5 * k + 4] = -a[2];
      p->sc[(size_t)c * (K + 1) + k + 1] = sc;
    }
    rec[5 * K] = monic ? g : 1.0;
  }
  // ---- precision tier per channel: MEASURED, not guessed -----------------------------------
  // A channel runs its recurrence in float32 (FP32 pipe, no conversions) only if the float32 core,
  // executed here on the host with the kernel's own arithmetic, stays within tier_tol of the float64
  // core on the probe signals; tier_tol defaults to a quarter of the 1e-5 parity bar.  Poles close
  // to z = 1 (low ERB channels) fail by orders of magnitude and stay in float64.
  p->tier.assign(C, 0);
  p->tier_err.assign(C, -1.0);
  p->tier_tol = env_double("ALZ_TIER_TOL", 2.5e-6);
  p->probe_len = std::max(64, env_int("ALZ_TIER_PROBE", 8192));
  const bool tiering = !(flags & ALZ_PLAN_EXACT) && !p->parallel_sum && !env_int("ALZ_NO_FP32_TIER", 0) && p->tier_tol > 0.0;
  std::vector<double> tab32((size_t)C * stride, 0.0);   // the same records as packed floats
  for (int c = 0; c < C; ++c) {
    const double* rec = tab.data() + (size_t)c * stride;
    float* r32 = reinterpret_cast<float*>(tab32.data() + (size_t)c * stride);
    bool representable = true;
    for (int i = 0; i < nval; ++i) {
      r32[i] = (float)rec[i];
      if (rec[i] != 0.0 && !(std::fabs(rec[i]) > 1e-30 && std::fabs(rec[i]) < 1e30)) representable = false;
    }
    // Near the unit circle float32 state rounding is amplified by ~1 / (1 - r), and on it (a pole cancelled by a zero,
    // maverage.recursive(1)) the error random-walks with the length of the input, past any probe.
    double radius = 0.0;
    for (auto& s : secs[c]) {
      const double a1 = s.a.size() > 1 ? s.a[1] : 0.0, a2 = s.a.size() > 2 ? s.a[2] : 0.0, disc = a1 * a1 - 4.0 * a2;
      radius = std::max(radius, disc < 0.0 ? std::sqrt(a2) : 0.5 * (std::fabs(a1) + std::sqrt(disc)));
    }
    if (tiering && representable) {
      p->tier_err[c] = probe_biquad(p, rec, tab32.data() + (size_t)c * stride);
      if (p->tier_err[c] <= p->tier_tol && radius <= kTierMaxRadius) { p->tier[c] = 1; ++p->n_fp32; }
    }
  }
  if (!p->sequential)
    for (int c = 0; c < C; ++c) p->chunk_err = std::max(p->chunk_err, chunk_error(secs[c], kChunkProbeLen));
  // ---- positions: interleave the tiers along blockIdx.x so both kinds of warp share every SM ----
  {
    std::vector<int> lst[2];
    const int order = env_int("ALZ_TIER_ORDER", 1);   // 1: interleave the tiers; 0: channel order; 2: float32 channels first
    for (int c = 0; c < C; ++c) lst[order == 1 ? p->tier[c] : (order == 2 ? 1 - p->tier[c] : 0)].push_back(c);
    size_t i0 = 0, i1 = 0;
    p->pos_channel.clear();
    while (i0 < lst[0].size() || i1 < lst[1].size()) {   // Bresenham merge: the list that is less consumed goes next
      const bool take0 = i1 >= lst[1].size() || (i0 < lst[0].size() && i0 * lst[1].size() <= i1 * lst[0].size());
      p->pos_channel.push_back(take0 ? lst[0][i0++] : lst[1][i1++]);
    }
  }
  p->h_tab.assign((size_t)C * stride, 0.0);
  for (int pos = 0; pos < C; ++pos) {
    const int c = p->pos_channel[pos];
    const std::vector<double>& src = p->tier[c] ? tab32 : tab;
    double* rec = p->h_tab.data() + (size_t)pos * stride;
    memcpy(rec, src.data() + (size_t)c * stride, (size_t)nval * sizeof(double));
    rec[ALZ_COEF_META(K, p->NB0)] = (double)(c + 65536 * p->tier[c]);
  }
  p->fp64_ops_exact = p->fp64_ops;
  // ---- kernel-parameter blocks, built once (launches pass them by address) ---------------------
  p->coef_small = C * stride <= kCoefSmall;
  const int ncoef = p->coef_small ? kCoefSmall : kCoefLarge;
  const int per_launch = ncoef / stride;
  if (per_launch < 1) return fail(ALZ_ERR_UNSUPPORTED, "coefficient record too large");
  for (int p0 = 0; p0 < C; p0 += per_launch) {
    const int npos = std::min(per_launch, C - p0);
    char* blk = (char*)calloc(1, 2 * sizeof(int) + (size_t)ncoef * sizeof(double));
    if (!blk) return fail(ALZ_ERR_NOMEM, "out of host memory");
    reinterpret_cast<int*>(blk)[0] = stride;
    reinterpret_cast<int*>(blk)[1] = npos;
    memcpy(blk + 2 * sizeof(int), p->h_tab.data() + (size_t)p0 * stride, (size_t)npos * stride * sizeof(double));
    p->chunks.push_back({blk, npos});
  }
  // Tile group of the launches that fill the machine: 4 (512 B pieces of every output row, 13 CTAs per SM on an H100)
  // when the arithmetic hides under the output stores; a plan with more FP64 work per channel-sample is bound by
  // issue and keeps 2, whose 24 CTAs per SM hide more of it.  Measured at the same shape (4096 x 16384,
  // profiles/h100_tile_group4_ab.txt): klapuri (fp64_ops 10) and slaney (12) gain 3 % with 4, the head-FIR sampled
  // bank (19) loses 5 %; the bound lies between them.
  const int group = env_int("ALZ_TILE_GROUP", 0);
  p->tile_group_forced = group == 1 || group == 2 || group == 4;
  p->tile_group = p->tile_group_forced ? group : (p->fp64_ops <= kTileGroup4MaxFp64 ? 4 : 2);
  // How groups of 4 tiles leave the SM: warp-wide 512-byte row stores (default), or TMA box stores with ALZ_STORE_PATH=tma
  // (DESIGN.md section 3: measured on the H100).
  const char* store_path = getenv("ALZ_STORE_PATH");
  p->vec_store = !(store_path && !strcmp(store_path, "tma"));
  return ALZ_OK;
}

// window: one section per channel, dense near taps in registers + prefetched far taps (alz_window.cuh)
static int build_window(alz_plan* p, const std::vector<std::vector<Sec>>& secs, int nbmax) {
  const int C = p->C;
  p->kind = ALZ_KIND_GENERIC;
  p->window = true;
  p->K = 1;
  p->NB = nbmax;
  p->monic = 0;
  int near_x = 0, near_y = 0, maxd_x = 0, maxd_y = 0;
  std::vector<int> far_x, far_y;                    // union over the channels of the taps with delay >= 16
  for (int c = 0; c < C; ++c) {
    if (secs[c].empty()) continue;
    const Sec& s = secs[c][0];
    for (size_t d = 1; d < s.b.size(); ++d)
      if (s.b[d] != 0.0) {
        maxd_x = std::max(maxd_x, (int)d);
        if (d < 16) near_x = std::max(near_x, (int)d);
        else if (std::find(far_x.begin(), far_x.end(), (int)d) == far_x.end()) far_x.push_back((int)d);
      }
    for (size_t d = 1; d < s.a.size(); ++d)
      if (s.a[d] != 0.0) {
        maxd_y = std::max(maxd_y, (int)d);
        if (d < 16) near_y = std::max(near_y, (int)d);
        else if (std::find(far_y.begin(), far_y.end(), (int)d) == far_y.end()) far_y.push_back((int)d);
      }
  }
  std::sort(far_x.begin(), far_x.end());
  std::sort(far_y.begin(), far_y.end());
  auto slots_of = [](int nearest) { return nearest == 0 ? 0 : (nearest <= 3 ? 4 : 16); };
  auto pow2 = [](int n) { int q = 1; while (q < n) q <<= 1; return q; };
  p->win_mx = slots_of(near_x);
  p->win_my = slots_of(near_y);
  p->win_nfx = (int)far_x.size();
  p->win_nfy = (int)far_y.size();
  int slot = 1;                                     // slot 0: absolute sample count
  p->win_xwin = slot; slot += p->win_mx ? p->win_mx - 1 : 0;
  p->win_ywin = slot; slot += p->win_my ? p->win_my - 1 : 0;
  if (!far_x.empty()) { p->win_xbase = slot; p->win_xmask = pow2(far_x.back() + 16) - 1; slot += p->win_xmask + 1; }
  if (!far_y.empty()) { p->win_ybase = slot; p->win_ymask = pow2(far_y.back() + 16) - 1; slot += p->win_ymask + 1; }
  p->xd = maxd_x; p->yd = maxd_y;
  p->state_doubles = slot;
  p->fp64_ops = 1 + (p->win_mx ? p->win_mx - 1 : 0) + (p->win_my ? p->win_my - 1 : 0) + p->win_nfx + p->win_nfy;
  p->win_far_delay = far_x;
  p->win_far_delay.insert(p->win_far_delay.end(), far_y.begin(), far_y.end());
  p->h_tab.assign((size_t)C * 32, 0.0);             // [C][b0..b15, -a1..-a15, pad]
  std::vector<double> fcoef(std::max<size_t>(1, p->win_far_delay.size()) * C, 0.0);
  for (int c = 0; c < C; ++c) {
    double* rec = p->h_tab.data() + (size_t)c * 32;
    if (secs[c].empty()) { rec[0] = 1.0; continue; }   // empty cascade: identity
    const Sec& s = secs[c][0];
    for (size_t d = 0; d < s.b.size() && d < 16; ++d) rec[d] = s.b[d];
    for (size_t d = 1; d < s.a.size() && d < 16; ++d) rec[16 + d - 1] = -s.a[d];
    for (size_t f = 0; f < far_x.size(); ++f) fcoef[f * C + c] = (size_t)far_x[f] < s.b.size() ? s.b[far_x[f]] : 0.0;
    for (size_t f = 0; f < far_y.size(); ++f) fcoef[(far_x.size() + f) * C + c] = (size_t)far_y[f] < s.a.size() ? -s.a[far_y[f]] : 0.0;
  }
  p->coef_small = C * 32 <= 64;
  p->win_block = calloc(1, alzi_window_block_bytes(p->coef_small));
  if (!p->win_block) return fail(ALZ_ERR_NOMEM, "out of host memory");
  std::vector<int> fd(std::max<size_t>(1, p->win_far_delay.size()), 16);
  std::copy(p->win_far_delay.begin(), p->win_far_delay.end(), fd.begin());
  const int rc = upload_tables(p, {table(&p->d_far_delay, fd), table(&p->d_far_coef, fcoef)});
  if (rc != ALZ_OK) return rc;
  alzi_window_block_fill(p->win_block, p->coef_small, p->win_nfx, p->win_nfy, p->win_xbase, p->win_xmask, p->win_ybase,
                         p->win_ymask, p->win_xwin, p->win_ywin, C, p->d_far_delay, p->d_far_coef, p->h_tab.data());
  return ALZ_OK;
}

// generic: union tap structure per section
static int build_generic(alz_plan* p, const std::vector<std::vector<Sec>>& secs, int Kmax, int nbmax) {
  const int C = p->C;
  const int K = Kmax;
  p->kind = ALZ_KIND_GENERIC;
  p->K = K;
  p->NB = nbmax;
  p->monic = 0;
  std::vector<int> tap_delay;
  std::vector<std::vector<double>> tap_coef;   // [tap][C]
  p->h_sec.resize(K);
  p->h_xlen.assign(K, 0);
  p->h_ylen.assign(K, 0);
  int slot = 1;   // slot 0: absolute sample count
  int ops = 0, xdmax = 0, ydmax = 0;
  for (int k = 0; k < K; ++k) {
    size_t nb = 1, na = 1;
    for (int c = 0; c < C; ++c)
      if (k < (int)secs[c].size()) { nb = std::max(nb, secs[c][k].b.size()); na = std::max(na, secs[c][k].a.size()); }
    AlzGenSection gs{};
    gs.num_begin = (int)tap_delay.size();
    for (size_t d = 0; d < nb; ++d) {
      std::vector<double> col(C, 0.0);
      bool any = false;
      for (int c = 0; c < C; ++c) {
        double v;
        if (k < (int)secs[c].size()) v = d < secs[c][k].b.size() ? secs[c][k].b[d] : 0.0;
        else v = d == 0 ? 1.0 : 0.0;   // identity padding
        col[c] = v;
        any = any || v != 0.0;
      }
      if (any || d == 0) { tap_delay.push_back((int)d); tap_coef.push_back(std::move(col)); p->h_tap_is_den.push_back(0); }
    }
    gs.nnum = (int)tap_delay.size() - gs.num_begin;
    gs.den_begin = (int)tap_delay.size();
    for (size_t d = 1; d < na; ++d) {
      std::vector<double> col(C, 0.0);
      bool any = false;
      for (int c = 0; c < C; ++c) {
        double v = (k < (int)secs[c].size() && d < secs[c][k].a.size()) ? -secs[c][k].a[d] : 0.0;
        col[c] = v;
        any = any || v != 0.0;
      }
      if (any) { tap_delay.push_back((int)d); tap_coef.push_back(std::move(col)); p->h_tap_is_den.push_back(1); }
    }
    gs.nden = (int)tap_delay.size() - gs.den_begin;
    const int xlen = (int)nb - 1, ylen = (int)na - 1;
    auto pow2 = [](int n) { int q = 1; while (q < n) q <<= 1; return q; };
    if (xlen > 0) { gs.xbase = slot; gs.xmask = pow2(xlen) - 1; slot += gs.xmask + 1; } else { gs.xbase = 0; gs.xmask = -1; }
    if (ylen > 0) { gs.ybase = slot; gs.ymask = pow2(ylen) - 1; slot += gs.ymask + 1; } else { gs.ybase = 0; gs.ymask = -1; }
    p->h_sec[k] = gs;
    p->h_xlen[k] = xlen;
    p->h_ylen[k] = ylen;
    xdmax = std::max(xdmax, xlen);
    ydmax = std::max(ydmax, ylen);
    ops += gs.nnum + gs.nden;
  }
  p->xd = xdmax; p->yd = ydmax;
  p->state_doubles = slot;
  p->fp64_ops = ops;
  const size_t ntaps = tap_delay.size();
  p->h_tap_delay = tap_delay;
  std::vector<double> tab(ntaps * C);
  for (size_t t = 0; t < ntaps; ++t) memcpy(&tab[t * C], tap_coef[t].data(), C * sizeof(double));
  return upload_tables(p, {table(&p->d_coef, tab), table(&p->d_sec, p->h_sec), table(&p->d_tap_delay, tap_delay)});
}

// ----------------------------------------------------------------------------------
extern "C" {

const char* alz_last_error(void) { return g_err.c_str(); }
int32_t alz_abi_version(void) { return ALZ_ABI_VERSION; }
int64_t alz_launch_count(void) { return g_launches.load(); }

int32_t alz_device_count(void) {
  int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
  return n;
}

int32_t alz_set_device(int32_t device) {
  ALZ_CUDA(cudaSetDevice(device));
  return ALZ_OK;
}

int32_t alz_plan_create(const double* coef, const int32_t* desc, int32_t C, int32_t KM, alz_plan** out) {
  return alz_plan_create_ex(coef, desc, C, KM, 0, out);
}

int32_t alz_plan_create_ex(const double* coef, const int32_t* desc, int32_t C, int32_t KM, int32_t flags,
                           alz_plan** out) {
  if (!out) return fail(ALZ_ERR_INVALID, "out is null");
  *out = nullptr;
  if (!coef || !desc || C <= 0 || KM < 0) return fail(ALZ_ERR_INVALID, "bad plan arguments");
  const bool design_only = (flags & ALZ_PLAN_DESIGN_ONLY) != 0;   // tables and tier decision only: no device is touched
  int dev = -1;
  if (!design_only) ALZ_CUDA(cudaGetDevice(&dev));

  // ---- normalise every section: divide by a0, trim trailing zeros ------------------
  std::vector<std::vector<Sec>> secs(C);
  int Kmax = 0, nbmax = 1, namax = 1;
  int nb_first = 1, nb_rest = 1;   // numerator taps of the first section vs. of the later ones
  for (int c = 0; c < C; ++c) {
    bool ended = false;
    for (int k = 0; k < KM; ++k) {
      const int32_t* d = desc + ((size_t)c * KM + k) * 3;
      const int nb = d[0], na = d[1];
      if (nb == 0) { ended = true; continue; }
      if (ended) return fail(ALZ_ERR_INVALID, "channel %d: section %d follows an absent section", c, k);
      if (nb < 0 || na < 1 || d[2] < 0) return fail(ALZ_ERR_INVALID, "channel %d section %d: bad descriptor", c, k);
      const double* b = coef + d[2];
      const double* a = b + nb;
      if (a[0] == 0.0) return fail(ALZ_ERR_ZERO_GAIN, "channel %d section %d: Invalid filter gain (a0 == 0)", c, k);
      Sec s;
      s.b.assign(b, b + nb);
      s.a.assign(a, a + na);
      const double a0 = a[0];
      if (a0 != 1.0) {
        for (auto& v : s.b) v /= a0;
        for (auto& v : s.a) v /= a0;
        s.a[0] = 1.0;
      }
      while (s.b.size() > 1 && s.b.back() == 0.0) s.b.pop_back();
      while (s.a.size() > 1 && s.a.back() == 0.0) s.a.pop_back();
      for (double v : s.b) if (!std::isfinite(v)) return fail(ALZ_ERR_INVALID, "non-finite coefficient");
      for (double v : s.a) if (!std::isfinite(v)) return fail(ALZ_ERR_INVALID, "non-finite coefficient");
      nbmax = std::max(nbmax, (int)s.b.size());
      namax = std::max(namax, (int)s.a.size());
      int& nb_max = secs[c].empty() ? nb_first : nb_rest;
      nb_max = std::max(nb_max, (int)s.b.size());
      secs[c].push_back(std::move(s));
    }
    Kmax = std::max(Kmax, (int)secs[c].size());
  }
  if (Kmax == 0) Kmax = 1;   // bank of empty cascades: identity

  std::unique_ptr<alz_plan, void (*)(alz_plan*)> p(new (std::nothrow) alz_plan(), alz_plan_destroy);   // until handed out
  if (!p) return fail(ALZ_ERR_NOMEM, "out of host memory");
  p->C = C;
  p->device = dev;
  p->sequential = (flags & ALZ_PLAN_SEQUENTIAL) != 0;
  p->parallel_sum = (flags & ALZ_PLAN_PARALLEL) != 0;
  if (design_only || cudaDeviceGetAttribute(&p->sm_count, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || p->sm_count <= 0) {
    cudaGetLastError();
    p->sm_count = 132;
  }

  p->fr_desc.assign((size_t)C * Kmax * 3, 0);
  for (int c = 0; c < C; ++c)
    for (size_t k = 0; k < secs[c].size(); ++k) {
      int* d = &p->fr_desc[((size_t)c * Kmax + k) * 3];
      d[0] = (int)secs[c][k].b.size(); d[1] = (int)secs[c][k].a.size(); d[2] = (int)p->fr_coef.size();
      p->fr_coef.insert(p->fr_coef.end(), secs[c][k].b.begin(), secs[c][k].b.end());
      p->fr_coef.insert(p->fr_coef.end(), secs[c][k].a.begin(), secs[c][k].a.end());
    }
  p->fr_K = Kmax;

  const bool plain = nbmax <= 3 && namax <= 3 && Kmax <= 8;
  const bool headfir = !plain && namax <= 3 && nb_first <= 8 && nb_rest <= 3 && Kmax <= 4;
  const bool generic = (flags & ALZ_PLAN_FORCE_GENERIC) != 0;
  int rc;
  if ((plain || headfir) && !generic)
    rc = build_biquad(p.get(), secs, Kmax, nbmax, nb_rest, headfir, flags);
  else if (Kmax == 1 && !generic && C * 32 <= kCoefLarge && !env_int("ALZ_NO_WINDOW", 0))
    rc = build_window(p.get(), secs, nbmax);
  else
    rc = build_generic(p.get(), secs, Kmax, nbmax);
  if (rc != ALZ_OK) return rc;
  *out = p.release();
  return ALZ_OK;
}

void alz_plan_destroy(alz_plan* p) {
  if (!p) return;
  if (p->device >= 0) {   // a design-only plan holds host tables only
    DeviceScope dev(p->device);
    // Launches on any stream may still read the tables freed below (the window and generic kernels read d_coef, d_sec,
    // d_tap_delay and d_far_* from global memory, the scans the cached M): cudaFree only "may perform implicit
    // synchronization", so wait for the device (its green contexts included) first.
    cudaDeviceSynchronize();
    if (p->pipe.ready) {
      for (int i = 0; i < AlzHostPipe::NBUF; ++i) {
        if (p->pipe.stream[i]) { cudaStreamSynchronize(p->pipe.stream[i]); cudaStreamDestroy(p->pipe.stream[i]); }
        if (p->pipe.done[i]) cudaEventDestroy(p->pipe.done[i]);
        cudaFree(p->pipe.dx[i]);
        cudaFree(p->pipe.dy[i]);
        cudaFree(p->pipe.dst[i]);
        cudaFree(p->pipe.des[i]);
      }
    }
    for (auto* e : p->m_cache) { cudaFree(e->M); cudaEventDestroy(e->ready); delete e; }
    cudaFree(p->d_far_delay);
    cudaFree(p->d_far_coef);
    cudaFree(p->d_coef);
    cudaFree(p->d_sec);
    cudaFree(p->d_tap_delay);
    cudaFree(p->d_fr_coef);
    cudaFree(p->d_fr_desc);
    cudaGetLastError();
  }
  for (auto& ch : p->chunks) free(ch.block);
  free(p->win_block);
  delete p;
}

int32_t alz_plan_info_get(const alz_plan* p, alz_plan_info* out) {
  if (!p || !out) return fail(ALZ_ERR_INVALID, "null argument");
  memset(out, 0, sizeof *out);
  out->abi_version = ALZ_ABI_VERSION;
  out->kind = p->kind;
  out->n_channels = p->C;
  out->n_sections = p->K;
  out->num_taps = p->NB0 ? p->NB0 : p->NB;
  out->monic = p->monic;
  out->state_doubles = p->state_doubles;
  out->fp64_ops = p->fp64_ops;
  out->device = p->device;
  out->n_fp32_channels = p->n_fp32;
  out->tier_tol_e9 = (int32_t)std::min(2.0e9, p->tier_tol * 1e9 + 0.5);
  out->time_parallel = p->kind == ALZ_KIND_BIQUAD && !p->sequential && p->chunk_err <= kChunkMaxErr;
  return ALZ_OK;
}

int32_t alz_plan_tiers(const alz_plan* p, int32_t* tier, double* probe_err, int32_t cap) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  for (int c = 0; c < p->C && c < cap; ++c) {
    const bool have = c < (int)p->tier.size();
    if (tier) tier[c] = have ? p->tier[c] : 0;
    if (probe_err) probe_err[c] = have ? p->tier_err[c] : -1.0;
  }
  return p->C;
}

int64_t alz_plan_state_doubles(const alz_plan* p, int64_t S) {
  if (!p || S < 0) return fail(ALZ_ERR_INVALID, "bad argument");
  return (int64_t)p->state_doubles * S * p->C;
}

int32_t alz_plan_history(const alz_plan* p, int32_t* xd, int32_t* yd) {
  if (!p || !xd || !yd) return fail(ALZ_ERR_INVALID, "null argument");
  *xd = p->xd;
  *yd = p->yd;
  return ALZ_OK;
}

// Broadcast one per-channel row of slot values to all streams: state[slot*R + c*S + s].
static __global__ void alz_state_fill_kernel(double* state, const double* proto, long long R, int C, int slots) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * slots) return;
  const long long slot = i / R, r = i - slot * R, S = R / C;
  state[i] = proto[slot * C + (int)(r / S)];
}

int32_t alz_state_init(const alz_plan* p, double* state, int64_t S, const double* xinit, const double* yinit,
                       void* cuda_stream) {
  if (!p || S < 0) return fail(ALZ_ERR_INVALID, "bad argument");
  if (p->device < 0) return fail(ALZ_ERR_CUDA, "design-only plan: no device");
  if (S == 0) return ALZ_OK;
  if (!state) return fail(ALZ_ERR_INVALID, "state is null");
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  cudaStream_t st = (cudaStream_t)cuda_stream;
  const long long R = (long long)S * p->C;
  const size_t bytes = (size_t)p->state_doubles * R * sizeof(double);
  if (!xinit && !yinit) {
    ALZ_CUDA(cudaMemsetAsync(state, 0, bytes, st));
    return ALZ_OK;
  }
  const int C = p->C, K = p->K, slots = p->state_doubles;
  std::vector<double> proto((size_t)slots * C, 0.0);
  if (p->kind == ALZ_KIND_BIQUAD) {
    for (int c = 0; c < C; ++c)
      for (int k = 0; k < K; ++k) {
        const double sc_in = p->sc[(size_t)c * (K + 1) + k], sc_out = p->sc[(size_t)c * (K + 1) + k + 1];
        const int base = ALZ_STATE_BASE(k, p->NB0);
        const int nx = k == 0 ? ALZ_H0(p->NB0) : 2;
        for (int j = 0; j < nx; ++j) {
          const double xv = xinit ? xinit[((size_t)c * K + k) * p->xd + j] : 0.0;
          // mode 2 scales the float32 input by the float32 gain in FP32, exactly like the kernel
          proto[(size_t)(base + j) * C + c] = (p->monic == 2 && k == 0) ? (double)((float)xv * (float)sc_in) : xv * sc_in;
        }
        for (int j = 0; j < 2; ++j) {
          const double yv = yinit ? yinit[((size_t)c * K + k) * 2 + j] : 0.0;
          proto[(size_t)(base + nx + j) * C + c] = yv * sc_out;
        }
      }
  } else if (p->window) {
    for (int c = 0; c < C; ++c) {
      for (int j = 0; j < p->xd; ++j) {                 // entry j = delay j+1
        const double xv = xinit ? xinit[(size_t)c * p->xd + j] : 0.0;
        if (j + 1 < p->win_mx) proto[(size_t)(p->win_xwin + j) * C + c] = xv;
        if (p->win_xmask >= 0) proto[(size_t)(p->win_xbase + ((-(j + 1)) & p->win_xmask)) * C + c] = xv;
      }
      for (int j = 0; j < p->yd; ++j) {
        const double yv = yinit ? yinit[(size_t)c * p->yd + j] : 0.0;
        if (j + 1 < p->win_my) proto[(size_t)(p->win_ywin + j) * C + c] = yv;
        if (p->win_ymask >= 0) proto[(size_t)(p->win_ybase + ((-(j + 1)) & p->win_ymask)) * C + c] = yv;
      }
    }
  } else {
    for (int c = 0; c < C; ++c)
      for (int k = 0; k < K; ++k) {
        const AlzGenSection& gs = p->h_sec[k];
        for (int j = 0; j < p->h_xlen[k]; ++j) {   // delay j+1 lives at ring position (-(j+1)) & mask
          const double xv = xinit ? xinit[((size_t)c * K + k) * p->xd + j] : 0.0;
          proto[(size_t)(gs.xbase + ((-(j + 1)) & gs.xmask)) * C + c] = xv;
        }
        for (int j = 0; j < p->h_ylen[k]; ++j) {
          const double yv = yinit ? yinit[((size_t)c * K + k) * p->yd + j] : 0.0;
          proto[(size_t)(gs.ybase + ((-(j + 1)) & gs.ymask)) * C + c] = yv;
        }
      }
  }
  StreamScratch<double> d_proto(st);
  ALZ_CUDA(d_proto.alloc(proto.size()));
  ALZ_CUDA(cudaMemcpyAsync(d_proto.ptr, proto.data(), proto.size() * sizeof(double), cudaMemcpyHostToDevice, st));
  const long long n = R * slots;
  alz_state_fill_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(state, d_proto.ptr, R, C, slots);
  ALZ_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  ALZ_CUDA(cudaStreamSynchronize(st));   // proto (pageable host vector) must be consumed before return
  return ALZ_OK;
}

static int apply_launch(const alz_plan* p, AlzTileArgs ta, double* state, long long sstride, cudaStream_t st,
                        const double* tv, long long tv_stride) {
  ta.state = state;
  ta.sstride = sstride;
  if (p->kind == ALZ_KIND_BIQUAD) return launch_biquad(p, ta, st);
  if (p->window) return alzi_launch_window(p, ta, st);
  return launch_generic(p, ta, st, tv, tv_stride);
}

// ---- time-parallel evaluation of FEW long streams ------------------------------------------
// A recurrence is serial in time, so one stream keeps one lane busy.  For an LTI filter the
// state after a chunk is an affine function of the state before it:  s' = F + M s, where F is
// the chunk's zero-state final state and M = A^L depends only on the coefficients.  So:
//   pass 1  every chunk of L samples is filtered from a ZERO state, all chunks in parallel (a
//           chunk is a "virtual stream": same kernels, x row stride L)         -> F_p
//   basis   L zero samples from each unit state                                   -> M (d x d per channel)
//   scan    s_{p+1} = F_p + M s_p, sequential over the P chunks (tiny kernel)     -> every chunk's true initial state
//   pass 2  every chunk again, from its true initial state                        -> the output
// Exact in exact arithmetic; in float64 the chunk states differ from the sequential ones by
// rounding only (parity bar 1e-5; tests/test_gpu_parity.py::test_time_parallel_path).
static __global__ void alz_unit_state_kernel(double* m, int d, int C) {   // m[slot j][(c*d + i)] = (i == j)
  const long long n = (long long)d * d * C;
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const long long j = i / ((long long)d * C), rest = i - j * d * C;
  m[i] = (rest % d == j) ? 1.0 : 0.0;
}

// One WARP per (channel, stream) (d <= 32): lane j owns state slot j, keeps row j of M in registers and
// the running state is exchanged with shuffles; F of the next chunk is prefetched.
// F / init: [slot][C][S][P] (virtual stream v = s * P + p); user state: [slot][C][Stot_user], stream offset applied by the caller.
static __global__ void __launch_bounds__(32) alz_chunk_scan_kernel(const double* __restrict__ F, double* __restrict__ init,
                                                            const double* __restrict__ M, double* user_state,
                                                            long long user_stride, long long user_stot, int d, int C,
                                                            long long S, long long P) {
  const int c = blockIdx.x, j = threadIdx.x;
  const long long sidx = blockIdx.y;
  const bool on = j < d;
  double mrow[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) mrow[i] = (on && i < d) ? M[(long long)j * d * C + (long long)c * d + i] : 0.0;
  double* us = user_state + (long long)(on ? j : 0) * user_stride + (long long)c * user_stot + sidx;
  double cur = on ? *us : 0.0;
  const long long slot_stride = (long long)C * S * P;
  const double* Fj = F + (long long)(on ? j : 0) * slot_stride + ((long long)c * S + sidx) * P;
  double* Ij = init + (long long)(on ? j : 0) * slot_stride + ((long long)c * S + sidx) * P;
  double f_next = (on && P > 0) ? Fj[0] : 0.0;
  for (long long p = 0; p < P; ++p) {
    const double f = f_next;
    if (on) {
      Ij[p] = cur;
      if (p + 1 < P) f_next = Fj[p + 1];
    }
    double a0 = f, a1 = 0.0;                       // two partial sums: shorter dependency chain
#pragma unroll
    for (int i = 0; i < 32; i += 2) {
      a0 = fma(mrow[i], __shfl_sync(0xffffffffu, cur, i), a0);
      a1 = fma(mrow[i + 1], __shfl_sync(0xffffffffu, cur, i + 1), a1);
    }
    cur = a0 + a1;
  }
  if (on) *us = cur;
}

// Time-parallel evaluation pays when the plain launch (one warp per channel and 32 streams, serial in time)
// would leave most of the machine idle: few streams, long blocks.  P chunks per stream (a multiple of 32, so that
// a warp's 32 virtual streams are chunks of ONE real stream: 3-D / 4-D tensor maps), L samples each.  `passes`: the
// passes over all chunks the evaluation makes (2 for the bank, 3 for the bank with the envelope consumer).
static bool chunk_geometry(const alz_plan* p, long long S, long long T, int passes, long long* P_out, long long* L_out) {
  if (p->kind != ALZ_KIND_BIQUAD || p->sequential || p->chunk_err > kChunkMaxErr || env_int("ALZ_NO_TIME_PARALLEL", 0))
    return false;
  if (T < std::max(2048, env_int("ALZ_TIME_PARALLEL_MIN", 16384)) || p->state_doubles > 32) return false;
  if (T >= (1ll << 31) || S > 65535) return false;
  const long long slots = (long long)p->sm_count * 24;
  const long long warps = (long long)p->C * ((S + 31) / 32);
  if (warps * 2 > slots) return false;             // the plain launch already fills half of the machine
  // cost model (tools/time_small.py times both evaluations): a lone warp advances one sample per t_seq / T (12 FP64 ops
  // per channel-sample); the chunked evaluation runs `passes` passes + extras
  const double work = std::max(1, p->fp64_ops) / 12.0;
  const double t_seq = (double)T * 36e-9 * work;
  // Chunk count P (a multiple of 32, chunks of >= 256 samples, <= 1024 because the scan over a stream's chunks is
  // serial): the one with the smallest estimated time.  A pass over all chunks costs ceil(waves) x L samples at the
  // per-sample time of a warp on a machine `occ` full (from alone to all 24 warp slots of its SM busy);
  // chunks are whole tiles, so T mod 32 P samples are left over for a sequential tail.
  long long P = 0;
  double best = 1e30;
  for (long long q = 32; q <= 1024 && q * 256 <= T; q += 32) {
    const double waves = (double)p->C * S * q / 32.0 / (double)slots;
    const double occ = waves < 1.0 ? waves : 1.0;
    const long long Lq = T / q / 32 * 32, tail = T - q * Lq;
    const double t_sample = std::max(36e-9, 92e-9 * occ) * work;
    // + the chunk states: d doubles per (channel, virtual stream), written / scanned / read ~6 times;
    // + ~10 us per wave and pass of CTA start-up and wave-end imbalance; + the serial scan, ~0.1 us per chunk
    const double t_state = 6.0 * p->state_doubles * 8.0 * p->C * (double)S * (double)q / 4e12;
    const double t = passes * std::ceil(waves) * ((double)Lq * t_sample + 1e-5) + t_state + (double)tail * 36e-9 * work + (double)q * 1e-7;
    if (t < best) { best = t; P = q; }
  }
  if (P == 0 || 1.25 * best + 5e-5 > 0.8 * t_seq) return false;   // the estimate is optimistic
  const long long L = T / P / 32 * 32;
  if (L < 256) return false;
  *P_out = P;
  *L_out = L;
  return true;
}

// Frees a chunk-transition entry nobody holds.  Scans that read its M may still be queued on any stream (of any host
// thread, or of a green context): cudaFree promises no ordering for memory from cudaMalloc ("may perform implicit
// synchronization"), so the device is synchronised first (cudaDeviceSynchronize == cuCtxSynchronize on the primary
// context, which also waits for the green contexts created from it).
static void chunk_entry_free(alz_plan::MEntry* e) {
  cudaDeviceSynchronize();
  cudaFree(e->M);
  cudaEventDestroy(e->ready);
  cudaGetLastError();
  delete e;
}

// Ends a call's use of an entry of chunk_transition, once every launch that reads its M is queued.
static void chunk_release(const alz_plan* p, alz_plan::MEntry* e) {
  alz_plan* pm = const_cast<alz_plan*>(p);
  bool last;
  {
    std::lock_guard<std::mutex> lock(pm->m_mu);
    last = --e->users == 0 && e->evicted;
  }
  if (last) chunk_entry_free(e);
}

// M = A^L (the chunk transition matrices, d x d per channel) on the device, ordered before the next work on `st`.  It
// depends on the plan and the chunk length only: computed once per (plan, L), kept in the plan.  The entry is held
// for the caller, which hands it back with chunk_release after queuing its scan; until then no other call (thread)
// frees it.  The basis run is queued under the lock, so that calls that miss the same L at once compute it once.
static int chunk_transition(const alz_plan* p, long long L, cudaStream_t st, alz_plan::MEntry** out) {
  const int C = p->C, d = p->state_doubles;
  alz_plan* pm = const_cast<alz_plan*>(p);
  alz_plan::MEntry* e = nullptr;
  alz_plan::MEntry* victim = nullptr;
  *out = nullptr;
  {
    std::lock_guard<std::mutex> lock(pm->m_mu);
    for (auto* c : pm->m_cache)
      if (c->L == L) e = c;
    if (e) {
      ++e->users;
    } else {   // basis run: L zero samples from each unit state -> M = A^L, per channel (it does not depend on the stream)
      double* M = nullptr;
      StreamScratch<float> xz(st), ydum(st);
      cudaEvent_t ready = nullptr;
      ALZ_CUDA(cudaMalloc((void**)&M, (size_t)d * d * C * 8));
      cudaError_t ce = cudaEventCreateWithFlags(&ready, cudaEventDisableTiming);
      if (ce == cudaSuccess) ce = xz.alloc((size_t)d * L);
      if (ce == cudaSuccess) ce = ydum.alloc((size_t)d * C * L);
      if (ce == cudaSuccess) ce = cudaMemsetAsync(xz.ptr, 0, (size_t)d * L * 4, st);
      int rc = ALZ_OK;
      if (ce == cudaSuccess) {
        const long long n = (long long)d * d * C;
        alz_unit_state_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(M, d, C);
        g_launches.fetch_add(1, std::memory_order_relaxed);
        AlzTileArgs tb{};
        tb.x = xz.ptr; tb.y = ydum.ptr; tb.S = d; tb.T = L; tb.xs = L; tb.ys = L; tb.ysS = (long long)C * L; tb.C = C; tb.Stot = d;
        tb.vec_in = tb.vec_out = 1;
        tb.exp = 2;                                                             // its outputs are not needed: no tile stores
        rc = apply_launch(p, tb, M, (long long)d * C, st, nullptr, 0);
      }
      if (ce == cudaSuccess && rc == ALZ_OK) ce = cudaEventRecord(ready, st);
      if (ce != cudaSuccess || rc != ALZ_OK) {
        cudaStreamSynchronize(st);                 // the basis run may be queued: M stays allocated until it is done
        cudaFree(M);
        if (ready) cudaEventDestroy(ready);
        cudaGetLastError();
        return rc != ALZ_OK ? rc : fail(ALZ_ERR_CUDA, "chunk transition: %s", cudaGetErrorString(ce));
      }
      e = new alz_plan::MEntry{L, M, ready, 1, false};
      if (pm->m_cache.size() >= 8) {               // bounded: drop the oldest entry; calls that still hold it free it
        victim = pm->m_cache.front();
        pm->m_cache.erase(pm->m_cache.begin());
        victim->evicted = true;
        if (victim->users > 0) victim = nullptr;
      }
      pm->m_cache.push_back(e);
    }
  }
  if (victim) chunk_entry_free(victim);
  // held: nobody destroys e->ready before this wait is queued (for the call that computed M it orders nothing)
  const cudaError_t we = cudaStreamWaitEvent(st, e->ready, 0);
  if (we != cudaSuccess) {
    chunk_release(p, e);
    return fail(ALZ_ERR_CUDA, "cudaStreamWaitEvent failed: %s", cudaGetErrorString(we));
  }
  *out = e;
  return ALZ_OK;
}

// 16-byte output stores (st.v4) need every row start aligned: y, the row stride ys and the stream stride ysS.
// The cp.async engine steps between the 32 rows of a warp by ysS.
static int vec_out_ok(const float* y, long long ys, long long ysS) {
  return (((uintptr_t)y & 15) == 0 && (ys & 3) == 0 && (ysS & 3) == 0) ? 1 : 0;
}

// Pass 1 and the bank-state scan of the time-parallel evaluation, on the caller's virtual streams `ta` (P chunks of L
// samples per stream): every chunk runs from a zero state into `zero`, and the scan turns those final states into
// every chunk's true initial state, in `init` ([slot][V * C] each, allocated here), and carries `state` past the last
// chunk.  `zero` is free for other use afterwards.
static int chunk_states(const alz_plan* p, AlzTileArgs ta, double* state, long long sstride, long long P, long long L,
                        cudaStream_t st, StreamScratch<double>& zero, StreamScratch<double>& init) {
  const int C = p->C, d = p->state_doubles;
  const long long V = ta.S, S = V / P;
  const size_t nstate = (size_t)d * V * C;
  keep_async_pool();
  ALZ_CUDA(zero.alloc(nstate));
  ALZ_CUDA(init.alloc(nstate));
  ALZ_CUDA(cudaMemsetAsync(zero.ptr, 0, nstate * 8, st));
  alz_plan::MEntry* m = nullptr;
  int rc = chunk_transition(p, L, st, &m);
  if (rc != ALZ_OK) return rc;
  ta.exp = 2;                                      // zero-state chunks: only the final states matter, no tile stores
  rc = apply_launch(p, ta, zero.ptr, V * C, st, nullptr, 0);
  if (rc == ALZ_OK) {
    alz_chunk_scan_kernel<<<dim3((unsigned)C, (unsigned)S), 32, 0, st>>>(zero.ptr, init.ptr, m->M, state, sstride, sstride / C,
                                                                         d, C, S, P);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) rc = fail(ALZ_ERR_CUDA, "chunk scan launch failed: %s", cudaGetErrorString(e));
    else g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  chunk_release(p, m);
  return rc;
}

// The first P * L samples of every stream, time-parallel.
static int apply_chunked(const alz_plan* p, const float* x, float* y, double* state, long long sstride, long long S,
                         long long xs, long long ys, long long P, long long L, cudaStream_t st) {
  const int C = p->C;
  const long long V = S * P;                       // V virtual streams
  AlzTileArgs ta{};
  ta.x = x; ta.y = y; ta.S = V; ta.T = L; ta.xs = xs; ta.ys = ys; ta.ysS = (long long)C * ys; ta.C = C; ta.Stot = V;
  ta.vec_in = (((uintptr_t)x & 15) == 0 && (xs & 3) == 0) ? 1 : 0;          // L is a multiple of 32: chunk starts keep the alignment
  ta.vec_out = vec_out_ok(y, ys, ta.ysS);
  ta.vP = (int)P;
  StreamScratch<double> zero(st), init(st);
  const int rc = chunk_states(p, ta, state, sstride, P, L, st, zero, init);
  if (rc != ALZ_OK) return rc;
  return apply_launch(p, ta, init.ptr, V * C, st, nullptr, 0);              // pass 2: every chunk from its true initial state
}

// ysS: the distance between the output rows of consecutive streams.
static int apply_impl(const alz_plan* p, const float* x, float* y, double* state, long long sstride, long long S,
                      long long T, long long xs, long long ys, long long ysS, cudaStream_t st, const double* tv = nullptr,
                      long long tv_stride = 0) {
  long long P = 0, L = 0;
  while (!tv && ysS == (long long)p->C * ys && chunk_geometry(p, S, T, 2, &P, &L)) {
    const int rc = apply_chunked(p, x, y, state, sstride, S, xs, ys, P, L, st);
    if (rc != ALZ_OK || T == P * L) return rc;
    x += P * L; y += P * L; T -= P * L;            // left-over samples of all streams: the same decision again
  }
  AlzTileArgs ta{};
  ta.T = T; ta.xs = xs; ta.ys = ys; ta.ysS = ysS; ta.C = p->C;
  ta.Stot = sstride / p->C;
  ta.vec_in = (((uintptr_t)x & 15) == 0 && (xs & 3) == 0) ? 1 : 0;
  ta.vec_out = vec_out_ok(y, ys, ysS);   // channel-major rows (ysS = T) are 16-byte aligned only when T is a multiple of 4
  const long long kMaxStreams = 65535ll * 32;   // gridDim.y limit
  for (long long s0 = 0; s0 < S; s0 += kMaxStreams) {
    ta.S = std::min(kMaxStreams, S - s0);
    ta.x = x + s0 * xs;
    ta.y = y + s0 * ysS;
    double* stp = state + s0;
    const int rc = apply_launch(p, ta, stp, sstride, st, tv, tv_stride);
    if (rc != ALZ_OK) return rc;
  }
  return ALZ_OK;
}

// The argument checks of the apply-style entries, in this order.  False when the entry returns *rc at once: an error, or
// ALZ_OK for an empty block.  `buffers`: every buffer the entry needs is given.  `need_device`: a design-only plan is
// refused before the sizes are looked at.
static bool apply_check(const alz_plan* p, bool need_device, int64_t S, int64_t T, bool buffers, int64_t xs, int64_t ys,
                        int* rc) {
  *rc = ALZ_OK;
  if (!p) *rc = fail(ALZ_ERR_INVALID, "plan is null");
  else if (need_device && p->device < 0) *rc = fail(ALZ_ERR_CUDA, "design-only plan: no device");
  else if (S < 0 || T < 0) *rc = fail(ALZ_ERR_INVALID, "negative size");
  else if (S == 0 || T == 0) return false;
  else if (!buffers) *rc = fail(ALZ_ERR_INVALID, "null buffer");
  else if (xs < T || ys < T) *rc = fail(ALZ_ERR_INVALID, "row stride shorter than n_samples");
  return *rc == ALZ_OK;
}

int32_t alz_apply_f32(const alz_plan* p, const float* x, float* y, double* state, int64_t S, int64_t T,
                      int64_t xs, int64_t ys, void* cuda_stream) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  return alz_apply_f32_ex(p, x, y, state, S, T, xs, ys, (int64_t)p->C * ys, cuda_stream);
}

int32_t alz_apply_f32_ex(const alz_plan* p, const float* x, float* y, double* state, int64_t S, int64_t T,
                         int64_t xs, int64_t ys, int64_t y_stream_stride, void* cuda_stream) {
  int rc;
  if (!apply_check(p, true, S, T, x && y && state, xs, ys, &rc)) return rc;
  // rows must not overlap: stream-major (stream stride >= C rows) or channel-major (row stride >= S stream strides)
  if (y_stream_stride < T || !(y_stream_stride >= (int64_t)p->C * ys || ys >= S * y_stream_stride))
    return fail(ALZ_ERR_INVALID, "output rows overlap: need y_stream_stride >= n_channels * y_stride or y_stride >= n_streams * y_stream_stride");
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  return apply_impl(p, x, y, state, (long long)S * p->C, S, T, xs, ys, y_stream_stride, (cudaStream_t)cuda_stream);
}

// ---- the bank with the fused envelope consumer ----------------------------------------------------------------------
// The envelope parameters of one call: the lowpass e[n] = fma(R, e[n-1], g r[n]), decimation and rectifier.
struct EnvParams { int decim, phase, mode; double g, R; };

static int envelope_launch(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  return p->NB0 == 8 ? alzi_launch_envelope_headfir_k4(p, ta, st) : alzi_launch_envelope_k4(p, ta, st);
}

// Time-parallel evaluation of few long streams (the bank's is apply_chunked): every stream is cut into P chunks of L
// samples (virtual streams), and
//   pass 1  the bank runs every chunk from a zero state, no output                     -> F_p
//   scan    alz_chunk_scan_kernel                                                     -> the chunks' true bank states
//   pass 2  bank from the true states, lowpass from zero, nothing stored               -> Fe_p
//   scan    alz_chunk_scan_kernel again, on the lowpass: it is linear in its state, so the state after chunk p is
//           e_{p+1} = Fe_p + R^L e_p, the same affine scan with a one-value state        -> the chunks' true lowpass states
//   pass 3  bank and lowpass from their true states, values stored at each chunk's decimation phase and offset
// and the T - P L samples left over continue sequentially.  Exact in exact arithmetic; in float64 the chunk states
// differ from the sequential ones by rounding only.  This evaluates the first P L samples of every stream.
static int envelope_chunked(const alz_plan* p, const float* x, float* env, double* state, double* env_state, long long sstride,
                            long long S, long long xs, long long es, const EnvParams& ep, long long P, long long L,
                            cudaStream_t st) {
  const int C = p->C;
  const long long V = S * P;                       // V virtual streams
  const size_t nstate = (size_t)p->state_doubles * V * C, nenv = (size_t)V * C;
  AlzTileArgs ta{};
  // y feeds only the (unused) output tensor map: x stands in, as in the sequential launch
  ta.x = x; ta.y = const_cast<float*>(x); ta.S = V; ta.T = L; ta.xs = xs; ta.ys = xs; ta.ysS = (long long)C * xs; ta.C = C;
  ta.Stot = V;
  ta.vec_in = ta.vec_out = 1;
  ta.vP = (int)P;
  StreamScratch<double> zero(st), init(st), E(st), E2(st), RL(st);
  int rc = chunk_states(p, ta, state, sstride, P, L, st, zero, init);     // pass 1 and the bank-state scan
  if (rc != ALZ_OK) return rc;
  ALZ_CUDA(E.alloc(nenv));
  ALZ_CUDA(E2.alloc(nenv));
  ALZ_CUDA(RL.alloc(C));
  ALZ_CUDA(cudaMemsetAsync(E.ptr, 0, nenv * 8, st));
  {   // the lowpass's chunk transition R^L (float64), one 1 x 1 matrix per channel; pageable source: staged before return
    const std::vector<double> rl((size_t)C, std::pow(ep.R, (double)L));
    ALZ_CUDA(cudaMemcpyAsync(RL.ptr, rl.data(), (size_t)C * 8, cudaMemcpyHostToDevice, st));
  }
  ALZ_CUDA(cudaMemcpyAsync(zero.ptr, init.ptr, nstate * 8, cudaMemcpyDeviceToDevice, st));   // pass 2 overwrites init; pass 3 needs it
  ta.state = init.ptr; ta.sstride = V * C;
  ta.env_out = env; ta.env_es = es; ta.env_state = E.ptr; ta.env_g = ep.g; ta.env_R = ep.R; ta.env_decim = ep.decim;
  ta.env_mode = ep.mode; ta.env_phase = ep.phase;
  ta.env_store = 0;                                // pass 2: only the final lowpass states
  rc = envelope_launch(p, ta, st);
  if (rc != ALZ_OK) return rc;
  alz_chunk_scan_kernel<<<dim3((unsigned)C, (unsigned)S), 32, 0, st>>>(E.ptr, E2.ptr, RL.ptr, env_state, nenv, sstride / C, 1, C, S, P);
  ALZ_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  ta.state = zero.ptr;
  ta.env_state = E2.ptr;
  ta.env_store = 1;                                // pass 3: the output
  return envelope_launch(p, ta, st);
}

// One implementation for every envelope entry.  state: [slot][sstride] bank states; env_state: [C][sstride / C] lowpass
// states (stream-fastest, like the bank's); env rows [S][C], stride es, (phase + T) / decim values each.  T > 0.
static int envelope_impl(const alz_plan* p, const float* x, float* env, double* state, double* env_state, long long sstride,
                         long long S, long long T, long long xs, long long es, EnvParams ep, cudaStream_t st) {
  if (((uintptr_t)x & 15) || (xs & 3) || env_int("ALZ_NO_TMA", 0))
    return fail(ALZ_ERR_UNSUPPORTED, "envelope consumer needs 16-byte aligned x rows");
  long long P = 0, L = 0;
  while (chunk_geometry(p, S, T, 3, &P, &L)) {
    const int rc = envelope_chunked(p, x, env, state, env_state, sstride, S, xs, es, ep, P, L, st);
    if (rc != ALZ_OK || T == P * L) return rc;
    // left-over samples of all streams: the same decision again
    env += (ep.phase + P * L) / ep.decim;
    ep.phase = (int)((ep.phase + P * L) % ep.decim);
    x += P * L;
    T -= P * L;
  }
  AlzTileArgs ta{};
  // y only feeds the output tensor map, which the envelope consumer never uses; it must be 16-byte aligned for the map to
  // be encoded, and env need not be (a block of a longer envelope row starts anywhere), so x, which must be, stands in.
  ta.x = x; ta.y = const_cast<float*>(x);
  ta.S = S; ta.T = T; ta.xs = xs; ta.ys = (T + 3) & ~3LL; ta.ysS = (long long)p->C * ta.ys; ta.C = p->C; ta.Stot = sstride / p->C;
  ta.state = state; ta.sstride = sstride;
  ta.vec_in = 1;
  ta.vec_out = 1;
  ta.env_out = env; ta.env_es = es; ta.env_state = env_state; ta.env_g = ep.g; ta.env_R = ep.R; ta.env_decim = ep.decim;
  ta.env_mode = ep.mode; ta.env_phase = ep.phase; ta.env_store = 1;
  return envelope_launch(p, ta, st);
}

// whole: the block must hold whole decimation windows (the entries without a phase)
static int envelope_check(const alz_plan* p, int64_t S, int64_t T, int64_t xs, int64_t es, const EnvParams& ep, bool whole) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  if (p->device < 0) return fail(ALZ_ERR_CUDA, "design-only plan: no device");
  if (S < 0 || T < 0 || ep.decim < 1 || ep.mode < 0 || ep.mode > 2 || ep.phase < 0 || ep.phase >= ep.decim)
    return fail(ALZ_ERR_INVALID, "bad argument");
  if (whole && T % ep.decim) return fail(ALZ_ERR_INVALID, "n_samples must be a multiple of the decimation factor");
  if (xs < T || es < (ep.phase + T) / ep.decim) return fail(ALZ_ERR_INVALID, "row stride shorter than the row");
  if (p->kind != ALZ_KIND_BIQUAD || p->K != 4 || p->C * ALZ_COEF_STRIDE(4, p->NB0) <= 512 || S > 65535ll * 32)
    return fail(ALZ_ERR_UNSUPPORTED, "the envelope consumer is built for the gammatone banks (4 sections per channel)");
  return ALZ_OK;
}

static int envelope_device(const alz_plan* p, const float* x, float* env, double* state, double* env_state, int64_t S,
                           int64_t T, int64_t xs, int64_t es, const EnvParams& ep, bool whole, void* cuda_stream) {
  const int chk = envelope_check(p, S, T, xs, es, ep, whole);
  if (chk != ALZ_OK) return chk;
  if (S == 0 || T == 0) return ALZ_OK;
  if (!x || !state || !env_state || (!env && (ep.phase + T) / ep.decim > 0)) return fail(ALZ_ERR_INVALID, "null buffer");
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  return envelope_impl(p, x, env, state, env_state, (long long)S * p->C, S, T, xs, es, ep, (cudaStream_t)cuda_stream);
}

int32_t alz_apply_envelope_f32(const alz_plan* p, const float* x, float* env, double* state, double* env_state, int64_t S,
                               int64_t T, int64_t xs, int64_t es, int32_t decim, int32_t mode, double g, double R,
                               void* cuda_stream) {
  return envelope_device(p, x, env, state, env_state, S, T, xs, es, EnvParams{decim, 0, mode, g, R}, true, cuda_stream);
}

int32_t alz_apply_envelope_f32_ex(const alz_plan* p, const float* x, float* env, double* state, double* env_state, int64_t S,
                                  int64_t T, int64_t xs, int64_t es, int32_t decim, int32_t phase, int32_t mode, double g,
                                  double R, void* cuda_stream) {
  return envelope_device(p, x, env, state, env_state, S, T, xs, es, EnvParams{decim, phase, mode, g, R}, false, cuda_stream);
}

// Host buffers: chunks of whole streams through the plan's staging pipeline.  state / env_state: device, NULL = zero and
// discarded (per-chunk staging states when both are NULL).
static int envelope_host(const alz_plan* cp, const float* xh, float* eh, double* state, double* env_state, int64_t S, int64_t T,
                         int64_t xs, int64_t es, const EnvParams& ep, bool whole) {
  const int chk = envelope_check(cp, S, T, xs, es, ep, whole);
  if (chk != ALZ_OK) return chk;
  alz_plan* p = const_cast<alz_plan*>(cp);
  if (S == 0 || T == 0) return ALZ_OK;
  if (!xh || (!eh && (ep.phase + T) / ep.decim > 0)) return fail(ALZ_ERR_INVALID, "null buffer");
  std::lock_guard<std::mutex> lock(p->host_mu);
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  const int decim = ep.decim;
  const long long C = p->C, Td = (ep.phase + T) / decim, Tp = (T + 3) & ~3LL, Tdp = (Td + 3) & ~3LL;
  // chunks of whole streams: <= 64 MiB of input per chunk (the output is decim times smaller than the bank's)
  long long Sc = std::max<long long>(32, (64LL << 20) / (Tp * 4) / 32 * 32);
  if (Sc > S) Sc = S;
  AlzHostPipe& hp = p->pipe;
  const int NB = AlzHostPipe::NBUF;
  // Given states are indexed for all S streams ([slot][S * C], [C][S]).  When only one of the two is given, the other
  // gets a zeroed buffer of the same layout for this call.
  DeviceBuffer own(nullptr, cudaFree);
  if ((state != nullptr) != (env_state != nullptr)) {
    const size_t bytes = (size_t)(state ? 1 : p->state_doubles) * S * C * 8;
    double* buf = nullptr;
    ALZ_CUDA(cudaMalloc((void**)&buf, bytes));
    own.reset(buf);
    ALZ_CUDA(cudaMemset(buf, 0, bytes));
    (state ? env_state : state) = buf;
  }
  const bool given = state != nullptr;
  int rc = pipe_open(hp, given);
  if (rc != ALZ_OK) return rc;
  rc = pipe_grow(hp, hp.dx, hp.dx_bytes, (size_t)Sc * Tp * 4);
  if (rc == ALZ_OK) rc = pipe_grow(hp, hp.dy, hp.dy_bytes, (size_t)Sc * C * Tdp * 4);
  if (rc == ALZ_OK && !given) rc = pipe_grow(hp, hp.dst, hp.dst_bytes, (size_t)p->state_doubles * Sc * C * 8);
  if (rc == ALZ_OK && !given) rc = pipe_grow(hp, hp.des, hp.des_bytes, (size_t)Sc * C * 8);
  int i = 0;
  for (long long s0 = 0; s0 < S && rc == ALZ_OK; s0 += Sc, ++i) {
    const long long n = std::min<long long>(Sc, S - s0);
    const int b = i % NB;
    cudaStream_t st = hp.stream[b];
    double* sb = given ? state + s0 : hp.dst[b];
    double* eb = given ? env_state + s0 : hp.des[b];
    const long long sstride = given ? S * C : n * C;
    if (!given) {
      cudaMemsetAsync(hp.dst[b], 0, (size_t)p->state_doubles * n * C * 8, st);
      cudaMemsetAsync(hp.des[b], 0, (size_t)n * C * 8, st);
    }
    cudaError_t e = cudaMemcpy2DAsync(hp.dx[b], Tp * 4, xh + s0 * xs, xs * 4, T * 4, n, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) { rc = fail(ALZ_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(e)); break; }
    rc = envelope_impl(p, hp.dx[b], hp.dy[b], sb, eb, sstride, n, T, Tp, Tdp, ep, st);
    if (rc != ALZ_OK) break;
    if (Td > 0) {
      e = cudaMemcpy2DAsync(eh + s0 * C * es, es * 4, hp.dy[b], Tdp * 4, Td * 4, n * C, cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) { rc = fail(ALZ_ERR_CUDA, "D2H copy failed: %s", cudaGetErrorString(e)); break; }
    }
  }
  return pipe_finish(hp, rc);
}

int32_t alz_apply_envelope_f32_host(const alz_plan* p, const float* xh, float* eh, int64_t S, int64_t T, int64_t xs, int64_t es,
                                    int32_t decim, int32_t mode, double g, double R) {
  return envelope_host(p, xh, eh, nullptr, nullptr, S, T, xs, es, EnvParams{decim, 0, mode, g, R}, true);
}

int32_t alz_apply_envelope_f32_host_ex(const alz_plan* p, const float* xh, float* eh, double* state, double* env_state,
                                       int64_t S, int64_t T, int64_t xs, int64_t es, int32_t decim, int32_t phase, int32_t mode,
                                       double g, double R) {
  return envelope_host(p, xh, eh, state, env_state, S, T, xs, es, EnvParams{decim, phase, mode, g, R}, false);
}

int32_t alz_apply_sum_f32(const alz_plan* p, const float* x, float* out, double* state, int64_t S, int64_t T,
                          int64_t xs, int64_t os, void* cuda_stream) {
  int rc;
  if (!apply_check(p, true, S, T, x && out && state, xs, os, &rc)) return rc;
  if (p->kind != ALZ_KIND_BIQUAD || !p->parallel_sum || p->NB0 != 0 || p->monic != 0 || p->chunks.size() != 1)
    return fail(ALZ_ERR_UNSUPPORTED, "alz_apply_sum_f32 needs a biquad plan created with ALZ_PLAN_PARALLEL");
  if (S > 65535ll * 32) return fail(ALZ_ERR_UNSUPPORTED, "too many streams for one launch");
  CUtensorMap tmx, tmo;
  if (env_int("ALZ_NO_TMA", 0) || !make_map_2d(x, T, S, xs, &tmx) || !make_map_2d(out, T, S, os, &tmo))
    return fail(ALZ_ERR_UNSUPPORTED, "alz_apply_sum_f32 needs 16-byte aligned rows (use alz_apply_f32 + alz_sum_channels_f32)");
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  AlzTileArgs ta{};
  ta.x = x; ta.y = out; ta.S = S; ta.T = T; ta.xs = xs; ta.ys = os; ta.ysS = os; ta.C = p->C; ta.Stot = S;
  ta.state = state; ta.sstride = (long long)S * p->C;
  ta.vec_in = ta.vec_out = 1;
  return alzi_launch_parallel(p, ta, tmx, tmo, (cudaStream_t)cuda_stream);
}

int32_t alz_plan_taps(const alz_plan* p, int32_t* delay, int32_t* is_den, int32_t cap) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  if (p->kind != ALZ_KIND_GENERIC || p->window) return fail(ALZ_ERR_UNSUPPORTED, "tap list exists only for plans built with ALZ_PLAN_FORCE_GENERIC");
  const int n = (int)p->h_tap_delay.size();
  for (int i = 0; i < n && i < cap; ++i) {
    if (delay) delay[i] = p->h_tap_delay[i];
    if (is_den) is_den[i] = p->h_tap_is_den[i];
  }
  return n;
}

int32_t alz_apply_tv_f32(const alz_plan* p, const float* x, float* y, double* state, int64_t S, int64_t T,
                         int64_t xs, int64_t ys, const double* coef_dev, int64_t coef_stride, void* cuda_stream) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  if (p->kind != ALZ_KIND_GENERIC || p->C != 1 || p->window)
    return fail(ALZ_ERR_UNSUPPORTED, "time-varying coefficients need a single-channel generic plan (alz_plan_create_ex with ALZ_PLAN_FORCE_GENERIC)");
  int rc;
  if (!apply_check(p, false, S, T, x && y && state && coef_dev, xs, std::min(ys, coef_stride), &rc)) return rc;
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  return apply_impl(p, x, y, state, (long long)S, S, T, xs, ys, ys, (cudaStream_t)cuda_stream, coef_dev, coef_stride);
}

int32_t alz_apply_f32_host(const alz_plan* cp, const float* xh, float* yh, double* state, int64_t S, int64_t T,
                           int64_t xs, int64_t ys) {
  alz_plan* p = const_cast<alz_plan*>(cp);
  int rc;
  if (!apply_check(p, true, S, T, xh && yh, xs, ys, &rc)) return rc;
  std::lock_guard<std::mutex> lock(p->host_mu);
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  AlzHostPipe& hp = p->pipe;
  const long long C = p->C;
  const long long kChunkBytes = 128LL << 20;   // <= 128 MiB of output per staged chunk
  // a chunk is (streams [s0, s0+Sc)) x (samples [t0, t0+Tc)): whole streams when they are short,
  // time segments of one stream (state carried on the device) when a single stream is long
  long long Tc = T;
  if (C * ((T + 3) & ~3LL) * 4 > kChunkBytes) {
    Tc = (kChunkBytes / (C * 4)) & ~31LL;
    if (Tc < 32) Tc = 32;
  }
  const long long Tp = (Tc + 3) & ~3LL;         // device row pitch: keeps every row 16-byte aligned
  long long Sc = kChunkBytes / (C * Tp * 4);
  if (Sc < 1) Sc = 1;
  if (Sc > S) Sc = S;
  rc = pipe_open(hp, state != nullptr);
  if (rc == ALZ_OK) rc = pipe_grow(hp, hp.dx, hp.dx_bytes, (size_t)Sc * Tp * 4);
  if (rc == ALZ_OK) rc = pipe_grow(hp, hp.dy, hp.dy_bytes, (size_t)Sc * C * Tp * 4);
  if (rc != ALZ_OK) return rc;
  DeviceBuffer own(nullptr, cudaFree);   // zero initial state when none is given
  double* st_buf = state;
  if (!st_buf) {
    const size_t bytes = (size_t)p->state_doubles * S * C * sizeof(double);
    ALZ_CUDA(cudaMalloc(&st_buf, bytes));
    own.reset(st_buf);
    ALZ_CUDA(cudaMemsetAsync(st_buf, 0, bytes, hp.stream[0]));
    ALZ_CUDA(cudaStreamSynchronize(hp.stream[0]));
  }
  int i = 0;
  for (long long s0 = 0; s0 < S && rc == ALZ_OK; s0 += Sc) {
    const long long n = std::min<long long>(Sc, S - s0);
    cudaEvent_t prev = nullptr;   // time segments of the same streams must run in order (state dependency)
    for (long long t0 = 0; t0 < T && rc == ALZ_OK; t0 += Tc, ++i) {
      const long long nt = std::min<long long>(Tc, T - t0);
      const int b = i % AlzHostPipe::NBUF;
      cudaStream_t st = hp.stream[b];
      if (prev) { cudaStreamWaitEvent(st, prev, 0); cudaEventDestroy(prev); prev = nullptr; }
      cudaError_t e = cudaMemcpy2DAsync(hp.dx[b], Tp * 4, xh + s0 * xs + t0, xs * 4, nt * 4, n, cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) { rc = fail(ALZ_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(e)); break; }
      rc = apply_impl(p, hp.dx[b], hp.dy[b], st_buf + s0, (long long)S * C, n, nt, Tp, Tp, C * Tp, st);
      if (rc != ALZ_OK) break;
      if (t0 + Tc < T) {
        cudaEventCreateWithFlags(&prev, cudaEventDisableTiming);
        cudaEventRecord(prev, st);
      }
      e = cudaMemcpy2DAsync(yh + s0 * C * ys + t0, ys * 4, hp.dy[b], Tp * 4, nt * 4, n * C, cudaMemcpyDeviceToHost, st);
      if (e != cudaSuccess) { rc = fail(ALZ_ERR_CUDA, "D2H copy failed: %s", cudaGetErrorString(e)); break; }
    }
    if (prev) cudaEventDestroy(prev);
  }
  return pipe_finish(hp, rc);
}

static __global__ void alz_sum_channels_kernel(const float* y, float* out, long long S, int C, long long T, long long ys,
                                        long long os) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= S * T) return;
  const long long s = i / T, t = i - s * T;
  const float* row = y + (s * C) * ys + t;
  double acc = row[0];
  for (int c = 1; c < C; ++c) acc += (double)row[(long long)c * ys];
  out[s * os + t] = (float)acc;
}

int32_t alz_sum_channels_f32(const float* y, float* out, int64_t S, int32_t C, int64_t T, int64_t ys, int64_t os,
                             void* cuda_stream) {
  if (S < 0 || T < 0 || C <= 0) return fail(ALZ_ERR_INVALID, "bad size");
  if (S == 0 || T == 0) return ALZ_OK;
  if (!y || !out) return fail(ALZ_ERR_INVALID, "null buffer");
  const long long n = (long long)S * T;
  alz_sum_channels_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)cuda_stream>>>(y, out, S, C, T, ys, os);
  ALZ_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZ_OK;
}

// H_c(e^{jw}) = prod_k B_ck(z^-1) / A_ck(z^-1) at z^-1 = e^{-jw}: one thread per (channel, frequency),
// Horner in complex float64 (reference lazy_filters.py:267-301 evaluates numpoly / denpoly the same way).
static __global__ void alz_freq_response_kernel(const double* __restrict__ coef, const int* __restrict__ desc, int C, int K,
                                         const double* __restrict__ w, long long n, double* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int c = blockIdx.y;
  if (i >= n) return;
  double zi, zr;
  sincos(-w[i], &zi, &zr);
  double hr = 1.0, hi = 0.0;
  for (int k = 0; k < K; ++k) {
    const int* d = desc + ((size_t)c * K + k) * 3;
    if (d[0] == 0) break;
    const double* b = coef + d[2];
    const double* a = b + d[0];
    double nr = b[d[0] - 1], ni = 0.0;
    for (int j = d[0] - 2; j >= 0; --j) {
      const double tr = nr * zr - ni * zi + b[j];
      ni = nr * zi + ni * zr;
      nr = tr;
    }
    double dr = a[d[1] - 1], di = 0.0;
    for (int j = d[1] - 2; j >= 0; --j) {
      const double tr = dr * zr - di * zi + a[j];
      di = dr * zi + di * zr;
      dr = tr;
    }
    const double den = dr * dr + di * di;      // 0 -> NaN, like the reference's nan for a pole on the grid
    const double qr = (nr * dr + ni * di) / den, qi = (ni * dr - nr * di) / den;
    const double tr = hr * qr - hi * qi;
    hi = hr * qi + hi * qr;
    hr = tr;
  }
  out[((size_t)c * n + i) * 2 + 0] = hr;
  out[((size_t)c * n + i) * 2 + 1] = hi;
}

int32_t alz_freq_response_f64(alz_plan* p, const double* w, double* out, int64_t n, void* cuda_stream) {
  if (!p) return fail(ALZ_ERR_INVALID, "plan is null");
  if (p->device < 0) return fail(ALZ_ERR_CUDA, "design-only plan: no device");
  if (n < 0) return fail(ALZ_ERR_INVALID, "negative size");
  if (n == 0) return ALZ_OK;
  if (!w || !out) return fail(ALZ_ERR_INVALID, "null buffer");
  DeviceScope dev(p->device);
  ALZ_CUDA(dev.status);
  {
    std::lock_guard<std::mutex> lock(p->host_mu);
    if (!p->d_fr_desc) {
      const int rc = upload_tables(p, {table(&p->d_fr_desc, p->fr_desc), table(&p->d_fr_coef, p->fr_coef)});
      if (rc != ALZ_OK) return rc;
    }
  }
  alz_freq_response_kernel<<<dim3((unsigned)((n + 127) / 128), (unsigned)p->C), 128, 0, (cudaStream_t)cuda_stream>>>(
      p->d_fr_coef, p->d_fr_desc, p->C, p->fr_K, w, n, out);
  ALZ_CUDA(cudaGetLastError());
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZ_OK;
}

// ---- pinned host buffers on the GPU's NUMA node ------------------------------------------------
// alz_apply_f32_host moves 260 B per input sample over PCIe; on a two-socket box a pinned buffer that
// lives on the other socket lowers that rate once several GPUs copy at the same time.  No libnuma in the image: the node comes from sysfs, the policy is set
// with the mbind system call, the pages are touched here and then registered with CUDA.
static int gpu_numa_node(int device) {
  char bus[32] = {0};
  if (cudaDeviceGetPCIBusId(bus, sizeof bus, device) != cudaSuccess) { cudaGetLastError(); return -1; }
  for (char* c = bus; *c; ++c) *c = (char)tolower(*c);
  char path[128];
  snprintf(path, sizeof path, "/sys/bus/pci/devices/%s/numa_node", bus);
  FILE* f = fopen(path, "r");
  if (!f) return -1;
  int node = -1;
  if (fscanf(f, "%d", &node) != 1) node = -1;
  fclose(f);
  return node;
}

int32_t alz_host_alloc(void** out, int64_t bytes, int32_t device, int32_t* numa_node) {
  if (!out || bytes <= 0) return fail(ALZ_ERR_INVALID, "bad argument");
  *out = nullptr;
  int dev = device;
  if (dev < 0) ALZ_CUDA(cudaGetDevice(&dev));
  const int node = env_int("ALZ_NO_NUMA", 0) ? -1 : gpu_numa_node(dev);
  const size_t len = ((size_t)bytes + (2u << 20) - 1) & ~((size_t)(2u << 20) - 1);
  void* ptr = mmap(nullptr, len, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  if (ptr == MAP_FAILED) return fail(ALZ_ERR_NOMEM, "mmap of %lld bytes failed", (long long)bytes);
  int bound = -1;
  if (node >= 0 && node < 1024) {
    unsigned long mask[16] = {0};
    mask[node / (8 * sizeof(unsigned long))] |= 1ul << (node % (8 * sizeof(unsigned long)));
    // MPOL_PREFERRED = 1: allocate on `node` while it has memory, never fail because of it
    if (syscall(SYS_mbind, ptr, len, 1 /* MPOL_PREFERRED */, mask, 1025ul, 0u) == 0) bound = node;
  }
  madvise(ptr, len, MADV_HUGEPAGE);
  {   // first touch with a few threads (page faults of tens of GB on one thread take seconds)
    const int nt = 8;
    std::vector<std::thread> th;
    const size_t per = ((len / nt) + 4095) & ~(size_t)4095;
    for (int i = 0; i < nt; ++i)
      th.emplace_back([=] {
        const size_t lo = (size_t)i * per, hi = std::min(len, lo + per);
        for (size_t o = lo; o < hi; o += 4096) ((volatile char*)ptr)[o] = 0;
      });
    for (auto& t : th) t.join();
  }
  cudaError_t e = cudaSetDevice(dev);
  if (e == cudaSuccess) e = cudaHostRegister(ptr, len, cudaHostRegisterPortable);
  if (e != cudaSuccess) {
    munmap(ptr, len);
    return fail(ALZ_ERR_CUDA, "cudaHostRegister of %lld bytes failed: %s", (long long)bytes, cudaGetErrorString(e));
  }
  {
    std::lock_guard<std::mutex> lock(g_host_mu);
    g_host_allocs[ptr] = len;
  }
  if (numa_node) *numa_node = bound;
  *out = ptr;
  return ALZ_OK;
}

int32_t alz_host_free(void* ptr) {
  if (!ptr) return ALZ_OK;
  size_t len = 0;
  {
    std::lock_guard<std::mutex> lock(g_host_mu);
    auto it = g_host_allocs.find(ptr);
    if (it == g_host_allocs.end()) return fail(ALZ_ERR_INVALID, "not an alz_host_alloc pointer");
    len = it->second;
    g_host_allocs.erase(it);
  }
  cudaHostUnregister(ptr);
  cudaGetLastError();
  munmap(ptr, len);
  return ALZ_OK;
}

// ---- a stream confined to a partition of the SMs (green context) ----------------------------------------
// Channel-sharded multi-GPU: every rank's bank kernel is short and its one-warp CTAs sit on ALL SMs for the whole
// kernel; an NCCL kernel (hundreds of threads x ~100 registers per CTA) needs an SM that is nearly EMPTY, so a broadcast
// issued on a side stream waits for the bank kernel to end (a step then costs kernel + broadcast).  A stream of a green
// context that owns only `sm_count` SMs keeps the bank kernel off the others, which NCCL's CTAs then find free.
int32_t alz_stream_create_partition(int32_t device, int32_t sm_count, void** stream_out, int32_t* sm_granted) {
  if (!stream_out || sm_count < 8) return fail(ALZ_ERR_INVALID, "bad argument");
  *stream_out = nullptr;
  int dev = device;
  if (dev < 0) ALZ_CUDA(cudaGetDevice(&dev));
  ALZ_CUDA(cudaSetDevice(dev));
  ALZ_CUDA(cudaFree(nullptr));                           // the primary context exists
  CUresult (*devGet)(CUdevice*, int) = nullptr;
  CUresult (*getRes)(CUdevice, CUdevResource*, CUdevResourceType) = nullptr;
  CUresult (*split)(CUdevResource*, unsigned int*, const CUdevResource*, CUdevResource*, unsigned int, unsigned int) = nullptr;
  CUresult (*genDesc)(CUdevResourceDesc*, CUdevResource*, unsigned int) = nullptr;
  CUresult (*ctxCreate)(CUgreenCtx*, CUdevResourceDesc, CUdevice, unsigned int) = nullptr;
  CUresult (*ctxDestroy)(CUgreenCtx) = nullptr;
  CUresult (*streamCreate)(CUstream*, CUgreenCtx, unsigned int, int) = nullptr;
  if (!driver_fn("cuDeviceGet", &devGet) || !driver_fn("cuDeviceGetDevResource", &getRes) ||
      !driver_fn("cuDevSmResourceSplitByCount", &split) || !driver_fn("cuDevResourceGenerateDesc", &genDesc) ||
      !driver_fn("cuGreenCtxCreate", &ctxCreate) || !driver_fn("cuGreenCtxDestroy", &ctxDestroy) ||
      !driver_fn("cuGreenCtxStreamCreate", &streamCreate))
    return fail(ALZ_ERR_UNSUPPORTED, "this driver has no green contexts");
  CUdevice cudev;
  CUdevResource all, part, rest;
  unsigned int groups = 1;
  CUdevResourceDesc desc;
  CUgreenCtx gctx;
  CUstream stream;
  CUresult r = devGet(&cudev, dev);
  if (r == CUDA_SUCCESS) r = getRes(cudev, &all, CU_DEV_RESOURCE_TYPE_SM);
  if (r == CUDA_SUCCESS) r = split(&part, &groups, &all, &rest, 0, (unsigned)sm_count);
  if (r == CUDA_SUCCESS && groups < 1) r = CUDA_ERROR_INVALID_VALUE;
  if (r == CUDA_SUCCESS) r = genDesc(&desc, &part, 1);
  if (r == CUDA_SUCCESS) r = ctxCreate(&gctx, desc, cudev, CU_GREEN_CTX_DEFAULT_STREAM);
  if (r != CUDA_SUCCESS) return fail(ALZ_ERR_CUDA, "green context with %d SMs failed (CUresult %d)", sm_count, (int)r);
  r = streamCreate(&stream, gctx, CU_STREAM_NON_BLOCKING, 0);
  if (r != CUDA_SUCCESS) { ctxDestroy(gctx); return fail(ALZ_ERR_CUDA, "green-context stream failed (CUresult %d)", (int)r); }
  {
    std::lock_guard<std::mutex> lock(g_host_mu);
    g_partitions[(void*)stream] = gctx;
  }
  if (sm_granted) *sm_granted = (int32_t)part.sm.smCount;
  *stream_out = (void*)stream;
  return ALZ_OK;
}

int32_t alz_stream_destroy_partition(void* stream) {
  if (!stream) return ALZ_OK;
  CUgreenCtx gctx;
  {
    std::lock_guard<std::mutex> lock(g_host_mu);
    auto it = g_partitions.find(stream);
    if (it == g_partitions.end()) return fail(ALZ_ERR_INVALID, "not a partition stream");
    gctx = it->second;
    g_partitions.erase(it);
  }
  cudaStreamSynchronize((cudaStream_t)stream);
  cudaStreamDestroy((cudaStream_t)stream);
  CUresult (*ctxDestroy)(CUgreenCtx) = nullptr;
  if (driver_fn("cuGreenCtxDestroy", &ctxDestroy)) ctxDestroy(gctx);
  cudaGetLastError();
  return ALZ_OK;
}

}  // extern "C"
