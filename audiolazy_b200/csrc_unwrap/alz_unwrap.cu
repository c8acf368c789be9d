// alz_unwrap.cu -- the C ABI of include/alz_b200_unwrap.h: phase unwrapping of S streams in one sm_90a launch, and
// clipping.
//
// delta is a float64 running sum over a stream's jumps, and float64 addition is not associative, so no tile can fold
// its jumps into an aggregate that a later tile combines: every stream's delta is chained from jump to jump in sample
// order.  Everything else is sample-parallel.  The unwrap kernel is a single-pass chained scan over tiles of kTile
// samples:
//   * a CTA takes its tile from an atomic ticket.  Tickets run over tile columns first (tile j of every row group, then
//     tile j + 1), so the predecessor a tile may wait on has a smaller ticket and is already running or done;
//   * each thread loads its samples (sample o of the tile is chunk o / kThreads, thread o % kThreads: every load and
//     store is coalesced), forms its diffs and jump tests and the jump terms, and the tile compacts its entries into
//     shared memory in sample order.  An entry is a jump's term, or the start of a row, which resets delta to a value
//     known without the chain (the state's delta, plus the term of a jump on that sample; d - d on a stream's first);
//   * one thread then walks the entries: d = reset ? v : d + v, one dependent __dadd_rn per jump, the only serial
//     part.  A tile that continues a row (tile j > 0) needs its predecessor's inclusive delta first: it publishes
//     "no entries" at once when it has none (a tile without a jump passes delta through unchanged, exactly), and warp 0
//     looks back over its predecessors, 32 at a time, to the nearest published inclusive delta (acquire / release);
//   * the tile publishes its inclusive delta before its stores; each sample then takes the value of the last entry at
//     or before it (its inclusive entry count), or the carry-in, and the thread of a row's last sample writes the
//     row's state.
// Rows of fewer than kTile samples are packed, kTile / T of them per tile, so a tile of short rows never waits.
//
// The unit is compiled with -fmad=false (nothing here multiplies, but no add may be contracted either) and without
// -ftz: subnormal samples are themselves.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_unwrap.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunks = 8;                       // samples per thread
constexpr int kTile = kChunks * kThreads;        // 2048 samples
constexpr unsigned kAgg = 1, kInc = 2;           // tile status: no entries (passes delta through) / inclusive delta

// Per stream: consumed (int64), previous sample (float64), delta (float64), and the bitwise complement of the first
// failing jump's index (0: none), so that an all-zero state is a new one and atomicMax keeps the first failure.
struct StreamState {
  long long consumed;
  double prev;
  double delta;
  unsigned long long fail;
};
static_assert(sizeof(StreamState) == 32, "state layout");

// Tiles of one call: R rows of L samples each (R > 1 only when a row fits in half a tile), nt tiles per row, G row groups.
struct Geometry {
  long long R, L, nt, G;
};

Geometry geometry(long long S, long long T) {
  Geometry g{};
  if (S <= 0 || T <= 0) return g;
  g.R = T >= kTile ? 1 : kTile / T;
  g.L = g.R == 1 ? kTile : T;
  g.nt = g.R == 1 ? (T + kTile - 1) / kTile : 1;
  g.G = (S + g.R - 1) / g.R;
  return g;
}

struct UwArgs {
  const void* x;
  void* out;
  StreamState* state;
  unsigned* ticket;
  double* val;               // [G][nt] inclusive delta of each tile
  unsigned* status;          // [G][nt] 0 while nothing is published, kAgg, kInc
  long long xs, os, S, T, R, L, nt, G;
  double M, P;
};

// the term of a jump with step 0: the reference raises there; here delta becomes NaN
__device__ __forceinline__ double step0_term() { return __longlong_as_double(0x7ff8000000000000LL); }

template <typename V> __device__ __forceinline__ double widen(V v) { return (double)v; }

template <typename V> __device__ __forceinline__ V narrow(double v) { return (V)v; }

// CPython 3.12's float_rem(v, w) for w != 0
__device__ __forceinline__ double py_rem(double v, double w) {
  double mod = fmod(v, w);
  if (mod != 0.0) {
    if ((w < 0.0) != (mod < 0.0)) mod = __dadd_rn(mod, w);
  } else {
    mod = copysign(0.0, w);
  }
  return mod;
}

// (-diff) + min(diff % P, diff % -P, key=abs); P != 0.  Out of line: fmod is long, and only jumps call it
__device__ __noinline__ double jump_term(double diff, double P) {
  const double a = py_rem(diff, P), b = py_rem(diff, -P);
  return __dadd_rn(-diff, fabs(b) < fabs(a) ? b : a);
}

__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ void st_release(unsigned* p, unsigned v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// The inclusive delta of the nearest predecessor of tile j that has one, looking back over tiles without entries
// (warp 0).  Tile 0 of a row always publishes one, so the walk ends there at the latest.
__device__ double look_back(const unsigned* status, const double* val, long long j, int lane) {
  long long base = j - 1;
  while (true) {
    const long long q = base - lane;
    const unsigned st = q >= 0 ? ld_acquire(status + q) : kAgg;
    const unsigned not_ready = __ballot_sync(0xffffffffu, st == 0);
    const unsigned stop = __ballot_sync(0xffffffffu, st == kInc);
    if (stop) {
      const int first = __ffs(stop) - 1;
      if ((not_ready & ((1u << first) - 1)) == 0) {
        const double v = lane == first ? *(const volatile double*)(val + q) : 0.0;
        return __shfl_sync(0xffffffffu, v, first);
      }
    } else if (!not_ready) {
      base -= 32;
      continue;
    }
    __nanosleep(64);
  }
}

}  // namespace

template <typename In, typename Out>
__global__ void __launch_bounds__(kThreads, 3) alz_unwrap_kernel(const __grid_constant__ UwArgs a) {
  __shared__ double s_val[kTile];                 // entry values, then the walked delta after each entry
  __shared__ unsigned char s_rst[kTile];          // 1: the entry resets delta to its value
  __shared__ int s_base[kChunks * kWarps];        // entries before each (chunk, warp) of the tile
  __shared__ unsigned s_tile;
  __shared__ int s_J;                             // entries of the tile
  __shared__ double s_carry;

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(a.ticket, 1u);
  __syncthreads();
  const long long t = s_tile, j = t / a.G, grp = t % a.G;
  const In* __restrict__ x = static_cast<const In*>(a.x);
  const double M = a.M, P = a.P;
  const int L = (int)a.L;                         // <= kTile

  double d[kChunks], ev[kChunks];
  int cnt[kChunks];             // entries of the tile at or before the sample
  unsigned first = 0, valid = 0, has = 0, rst = 0;
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    const int o = k * kThreads + tid;
    const int r = o / L;
    const long long s = grp * a.R + r, n = j * L + o % L;
    d[k] = ev[k] = 0.0;
    if (r < a.R && s < a.S && n < a.T) {
      valid |= 1u << k;
      const In* xr = x + s * a.xs;
      StreamState* st = a.state + s;
      d[k] = widen(xr[n]);
      if (n == 0) {                               // a row start: delta from the state, without the chain
        has |= 1u << k;
        rst |= 1u << k;
        if (st->consumed == 0) {
          ev[k] = __dsub_rn(d[k], d[k]);
          first |= 1u << k;
        } else {
          const double diff = __dsub_rn(d[k], st->prev);
          ev[k] = st->delta;
          if (fabs(diff) > M) {
            if (P == 0.0) atomicMax(&st->fail, ~(unsigned long long)st->consumed);
            ev[k] = __dadd_rn(ev[k], P == 0.0 ? step0_term() : jump_term(diff, P));
          }
        }
      } else {
        const double diff = __dsub_rn(d[k], widen(xr[n - 1]));
        if (fabs(diff) > M) {
          has |= 1u << k;
          if (P == 0.0) {
            atomicMax(&st->fail, ~(unsigned long long)(st->consumed + n));
            ev[k] = step0_term();
          } else {
            ev[k] = jump_term(diff, P);
          }
        }
      }
    }
    const unsigned mask = __ballot_sync(0xffffffffu, (has >> k) & 1u);
    cnt[k] = __popc(mask & ((2u << lane) - 1));   // entries of this warp's chunk at or before the sample
    if (lane == 0) s_base[k * kWarps + warp] = __popc(mask);
  }
  __syncthreads();
  if (warp == 0) {                                // exclusive scan of the 64 (chunk, warp) counts, 2 per lane
    const int c0 = s_base[2 * lane], c1 = s_base[2 * lane + 1];
    int c = c0 + c1;
#pragma unroll
    for (int dd = 1; dd < 32; dd <<= 1) {
      const int y = __shfl_up_sync(0xffffffffu, c, dd);
      if (lane >= dd) c += y;
    }
    s_base[2 * lane] = c - c0 - c1;
    s_base[2 * lane + 1] = c - c1;
    if (lane == 31) s_J = c;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {             // compaction: entries in sample order
    cnt[k] += s_base[k * kWarps + warp];
    if ((has >> k) & 1u) {
      s_val[cnt[k] - 1] = ev[k];
      s_rst[cnt[k] - 1] = (rst >> k) & 1u;
    }
  }
  __syncthreads();

  if (warp == 0) {
    const int n_entries = s_J;
    const long long di = grp * a.nt + j;
    double dl = 0.0;
    if (j > 0) {
      if (lane == 0 && n_entries == 0) st_release(a.status + di, kAgg);
      dl = look_back(a.status + grp * a.nt, a.val + grp * a.nt, j, lane);
    }
    if (lane == 0) {
      if (j > 0) s_carry = dl;
      int i = 0;
      for (; i + 8 <= n_entries; i += 8) {        // the loads do not wait on the chain
        double v[8];
        bool r[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = s_val[i + e], r[e] = s_rst[i + e];
#pragma unroll
        for (int e = 0; e < 8; ++e) dl = r[e] ? v[e] : __dadd_rn(dl, v[e]), v[e] = dl;
#pragma unroll
        for (int e = 0; e < 8; ++e) s_val[i + e] = v[e];
      }
      for (; i < n_entries; ++i) {
        dl = s_rst[i] ? s_val[i] : __dadd_rn(dl, s_val[i]);
        s_val[i] = dl;
      }
      if (a.nt > 1) {
        a.val[di] = dl;
        st_release(a.status + di, kInc);
      }
    }
  }
  __syncthreads();

  Out* __restrict__ out = static_cast<Out*>(a.out);
  const double carry = j > 0 ? s_carry : 0.0;
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    if (!((valid >> k) & 1u)) continue;
    const int o = k * kThreads + tid;
    const int r = o / L;
    const long long s = grp * a.R + r, n = j * L + o % L;
    const double delta = cnt[k] > 0 ? s_val[cnt[k] - 1] : carry;
    out[s * a.os + n] = narrow<Out>((first >> k) & 1u ? d[k] : __dadd_rn(d[k], delta));
    if (n == a.T - 1) {
      StreamState* st = a.state + s;
      st->consumed += a.T;
      st->prev = d[k];
      st->delta = delta;
    }
  }
}

template <typename In, typename Out>
__global__ void __launch_bounds__(kThreads) alz_clip_kernel(const In* __restrict__ x, long long xs,
                                                            Out* __restrict__ out, long long os, long long S,
                                                            long long T, double low, int has_low, double high,
                                                            int has_high) {
  for (long long s = blockIdx.y; s < S; s += gridDim.y) {
    const In* xr = x + s * xs;
    Out* orow = out + s * os;
    for (long long n = blockIdx.x * (long long)kThreads + threadIdx.x; n < T; n += (long long)gridDim.x * kThreads) {
      const double v = widen(xr[n]);
      double y;
      if (has_low && has_high) y = v > high ? high : (v < low ? low : v);
      else if (has_low) y = v > low ? v : low;
      else if (has_high) y = v < high ? v : high;
      else y = v;
      orow[n] = narrow<Out>(y);
    }
  }
}

namespace {

template <typename In, typename Out>
cudaError_t launch_unwrap(const UwArgs& a, cudaStream_t cs) {
  alz_unwrap_kernel<In, Out><<<(unsigned)(a.G * a.nt), kThreads, 0, cs>>>(a);
  return cudaGetLastError();
}

template <typename In, typename Out>
cudaError_t launch_clip(const void* x, long long xs, void* out, long long os, long long S, long long T, double low,
                        int has_low, double high, int has_high, cudaStream_t cs) {
  // contiguous rows are one row of S * T samples
  if (S > 1 && xs == T && os == T) T *= S, S = 1;
  const long long per_row = (T + kThreads * 4 - 1) / (kThreads * 4);
  const long long gx = per_row < 65535 * 16 ? per_row : 65535 * 16;
  const long long gy = S < 65535 ? S : 65535;
  alz_clip_kernel<In, Out><<<dim3((unsigned)gx, (unsigned)gy), kThreads, 0, cs>>>(
      static_cast<const In*>(x), xs, static_cast<Out*>(out), os, S, T, low, has_low, high, has_high);
  return cudaGetLastError();
}

bool bad_dtype(int32_t t) { return t != ALZ_UNWRAP_FLOAT32 && t != ALZ_UNWRAP_FLOAT64; }

long long elem_bytes(int32_t t) { return t == ALZ_UNWRAP_FLOAT64 ? 8 : 4; }

// The checks alz_unwrap_apply and alz_clip_apply share.
int check_io(const void* x, int32_t xt, int64_t xs, const void* out, int32_t ot, int64_t os, int64_t S, int64_t T) {
  if (S < 0 || T < 0) return fail(ALZ_UNWRAP_ERR_INVALID, "bad shape: n_streams %lld, n_samples %lld", (long long)S,
                                  (long long)T);
  if (bad_dtype(xt) || bad_dtype(ot)) return fail(ALZ_UNWRAP_ERR_INVALID, "dtype must be ALZ_UNWRAP_FLOAT32 or _FLOAT64");
  if (S == 0 || T == 0) return ALZ_UNWRAP_OK;
  if (!x || !out) return fail(ALZ_UNWRAP_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x % elem_bytes(xt)) || ((uintptr_t)out % elem_bytes(ot)))
    return fail(ALZ_UNWRAP_ERR_INVALID, "misaligned buffer");
  if (S > 1 && (xs < T || os < T)) return fail(ALZ_UNWRAP_ERR_INVALID, "stride < n_samples");
  return ALZ_UNWRAP_OK;
}

}  // namespace

extern "C" {

const char* alz_unwrap_last_error(void) { return g_err.c_str(); }

int64_t alz_unwrap_state_bytes(int64_t n_streams) {
  if (n_streams < 0) return fail(ALZ_UNWRAP_ERR_INVALID, "need n_streams >= 0");
  return n_streams * (int64_t)sizeof(StreamState);
}

int32_t alz_unwrap_state_init(void* state_dev, int64_t n_streams, void* cuda_stream) {
  if (n_streams < 0) return fail(ALZ_UNWRAP_ERR_INVALID, "need n_streams >= 0");
  if (n_streams == 0) return ALZ_UNWRAP_OK;
  if (!state_dev) return fail(ALZ_UNWRAP_ERR_INVALID, "state is NULL");
  if ((uintptr_t)state_dev & 7) return fail(ALZ_UNWRAP_ERR_INVALID, "misaligned state");
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  ALZ_CUDA_CHECK(cudaMemsetAsync(state_dev, 0, (size_t)n_streams * sizeof(StreamState), cs), ALZ_UNWRAP_ERR_CUDA);
  return ALZ_UNWRAP_OK;
}

int64_t alz_unwrap_scratch_bytes(int64_t n_streams, int64_t n_samples) {
  if (n_streams < 0 || n_samples < 0) return fail(ALZ_UNWRAP_ERR_INVALID, "bad shape");
  const Geometry g = geometry(n_streams, n_samples);
  return 16 + (g.G * g.nt * 12 + 7) / 8 * 8;
}

int32_t alz_unwrap_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                         int64_t out_stride, void* state_dev, int64_t n_streams, int64_t n_samples, double max_delta,
                         double step, void* scratch_dev, int64_t scratch_bytes, void* cuda_stream) {
  const int rc = check_io(x_dev, x_dtype, x_stride, out_dev, out_dtype, out_stride, n_streams, n_samples);
  if (rc != ALZ_UNWRAP_OK) return rc;
  if (n_streams == 0) return ALZ_UNWRAP_OK;
  if (!state_dev || !scratch_dev) return fail(ALZ_UNWRAP_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)state_dev & 7) || ((uintptr_t)scratch_dev & 7)) return fail(ALZ_UNWRAP_ERR_INVALID, "misaligned buffer");
  const int64_t need = alz_unwrap_scratch_bytes(n_streams, n_samples);
  if (scratch_bytes < need)
    return fail(ALZ_UNWRAP_ERR_INVALID, "scratch of %lld bytes, %lld needed", (long long)scratch_bytes, (long long)need);
  if (n_samples == 0) return ALZ_UNWRAP_OK;
  if (n_samples > 0x7fffffffLL - kTile) return fail(ALZ_UNWRAP_ERR_UNSUPPORTED, "n_samples too large for one launch");
  const Geometry g = geometry(n_streams, n_samples);
  if (g.G * g.nt > 0x7fffffffLL) return fail(ALZ_UNWRAP_ERR_UNSUPPORTED, "too many tiles for one launch");
  UwArgs a{};
  a.x = x_dev;
  a.out = out_dev;
  a.state = (StreamState*)state_dev;
  a.ticket = (unsigned*)scratch_dev;
  a.val = (double*)((char*)scratch_dev + 16);
  a.status = (unsigned*)(a.val + g.G * g.nt);
  a.xs = n_streams > 1 ? x_stride : n_samples;
  a.os = n_streams > 1 ? out_stride : n_samples;
  a.S = n_streams;
  a.T = n_samples;
  a.R = g.R;
  a.L = g.L;
  a.nt = g.nt;
  a.G = g.G;
  a.M = max_delta;
  a.P = step;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  ALZ_CUDA_CHECK(cudaMemsetAsync(scratch_dev, 0, (size_t)need, cs), ALZ_UNWRAP_ERR_CUDA);
  const bool xd = x_dtype == ALZ_UNWRAP_FLOAT64, od = out_dtype == ALZ_UNWRAP_FLOAT64;
  const cudaError_t e = xd ? (od ? launch_unwrap<double, double>(a, cs) : launch_unwrap<double, float>(a, cs))
                           : (od ? launch_unwrap<float, double>(a, cs) : launch_unwrap<float, float>(a, cs));
  ALZ_CUDA_CHECK(e, ALZ_UNWRAP_ERR_CUDA);
  return ALZ_UNWRAP_OK;
}

int32_t alz_clip_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                       int64_t out_stride, int64_t n_streams, int64_t n_samples, double low, int32_t has_low,
                       double high, int32_t has_high, void* cuda_stream) {
  const int rc = check_io(x_dev, x_dtype, x_stride, out_dev, out_dtype, out_stride, n_streams, n_samples);
  if (rc != ALZ_UNWRAP_OK) return rc;
  if (has_low && has_high && high < low)
    return fail(ALZ_UNWRAP_ERR_INVALID, "higher clipping limit is smaller than lower one");
  if (n_streams == 0 || n_samples == 0) return ALZ_UNWRAP_OK;
  const long long xs = n_streams > 1 ? x_stride : n_samples, os = n_streams > 1 ? out_stride : n_samples;
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  const bool xd = x_dtype == ALZ_UNWRAP_FLOAT64, od = out_dtype == ALZ_UNWRAP_FLOAT64;
  const int hl = has_low != 0, hh = has_high != 0;
  const cudaError_t e =
      xd ? (od ? launch_clip<double, double>(x_dev, xs, out_dev, os, n_streams, n_samples, low, hl, high, hh, cs)
               : launch_clip<double, float>(x_dev, xs, out_dev, os, n_streams, n_samples, low, hl, high, hh, cs))
         : (od ? launch_clip<float, double>(x_dev, xs, out_dev, os, n_streams, n_samples, low, hl, high, hh, cs)
               : launch_clip<float, float>(x_dev, xs, out_dev, os, n_streams, n_samples, low, hl, high, hh, cs));
  ALZ_CUDA_CHECK(e, ALZ_UNWRAP_ERR_CUDA);
  return ALZ_UNWRAP_OK;
}

}  // extern "C"
