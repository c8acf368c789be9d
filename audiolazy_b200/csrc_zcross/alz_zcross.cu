// alz_zcross.cu -- the C ABI of include/alz_b200_zcross.h: zero crossings of S streams in one sm_90a launch.
//
// The carried sign is a "last decisive sample" scan: s[n] is the sign of the last sample at or before n with
// |x| beyond the hysteresis.  It has no arithmetic, so it is evaluated as a single-pass chained scan over tiles of
// kTile samples, bit-identical to the sequential recursion whatever the tiling:
//   * a CTA takes its tile from an atomic ticket, so the tiles it looks back on are already running;
//   * it loads the tile with 16-byte loads (tiles are aligned to the row's address, so only a row's first and last
//     quads are loaded per sample) and finds each sample's nearest earlier decisive sample with __ballot_sync;
//   * it publishes the tile's own last decisive sign (which does not depend on the carry-in) at once, and as the
//     tile's inclusive value when the tile has a decisive sample;
//   * warp 0 resolves the carry-in from its predecessors' descriptors, 32 at a time, and publishes the inclusive value;
//   * the flags are stored, and in counts mode each block's crossings in the tile are the difference of two prefix
//     counts of the tile, added to the block's counter with one integer atomic (exact in any order).
// alz_zcross_finish_kernel then adds the partial counts the state carries, stores the completed blocks and carries
// the open ones, the sign and the sample count to the next call.
//
// Comparisons are made in float32 against hf, the largest float32 <= h (NaN for a NaN h): for a float32 y,
// y > h <=> y > hf and y < -h <=> y < -hf, so they equal the float64 comparisons of the reference for every h.  The
// unit is compiled without -ftz: subnormal samples compare as themselves.
#pragma GCC visibility push(default)
#include "../../include/alz_b200_zcross.h"
#pragma GCC visibility pop
#include "../csrc_common/alz_common.h"

#include <cuda_runtime.h>

#include <cmath>
#include <cstdint>

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kChunks = 4;                      // quads per thread; a chunk is kThreads consecutive quads
constexpr int kTile = kChunks * kThreads * 4;   // 4096 samples
constexpr unsigned kAgg = 1, kInc = 2;          // descriptor status: tile aggregate / inclusive value published

struct ZcArgs {
  const float* x;
  uint8_t* flags;
  int32_t* counts;
  unsigned char* state;
  unsigned* ticket;
  unsigned* desc;          // [S][nt]: status | (sign + 1) << 4, 0 while nothing is published
  int32_t* acc;            // [S][nacc]: crossings of blocks ka + i in this call (counts mode)
  long long xs, fs, cs, sstride, T, nt, nacc;
  int size, hop, R, final_;
  float hf;
};

long long ring_slots(int size, int hop) { return size > 0 ? (size + (long long)hop - 1) / hop : 0; }

long long state_stride(int size, int hop) { return (16 + 4 * ring_slots(size, hop) + 7) / 8 * 8; }

long long tiles_per_stream(long long T) { return T > 0 ? (T + 3 + kTile - 1) / kTile : 0; }

long long acc_per_stream(long long T, int size, int hop) { return size > 0 ? (T + size - 1) / hop + 2 : 0; }

__device__ __forceinline__ int sign_of_last(unsigned nz, unsigned pos) {   // nz != 0
  return (pos >> (31 - __clz(nz))) & 1u ? 1 : -1;
}

__device__ __forceinline__ unsigned ld_volatile(const unsigned* p) { return *(const volatile unsigned*)p; }

__device__ __forceinline__ void st_volatile(unsigned* p, unsigned v) { *(volatile unsigned*)p = v; }

__device__ __forceinline__ unsigned descriptor(unsigned status, int sign) { return status | (unsigned)(sign + 1) << 4; }

// The carried sign at the start of tile j of a stream (warp 0): the inclusive value of the nearest predecessor that
// has one, or the aggregate of the nearest predecessor with a decisive sample (that is its inclusive value), looking
// back over tiles without a decisive sample; before tile 0, the state's sign.
__device__ int look_back(const unsigned* desc, long long j, int state_sign, int lane) {
  long long base = j - 1;
  while (true) {
    const long long q = base - lane;
    const unsigned w = q >= 0 ? ld_volatile(desc + q) : descriptor(kInc, state_sign);
    const unsigned status = w & 15u;
    const int val = (int)(w >> 4) - 1;
    const unsigned not_ready = __ballot_sync(0xffffffffu, status == 0);
    const unsigned stop = __ballot_sync(0xffffffffu, status == kInc || (status == kAgg && val != 0));
    if (stop) {
      const int first = __ffs(stop) - 1;
      if ((not_ready & ((1u << first) - 1)) == 0) return __shfl_sync(0xffffffffu, val, first);
    } else if (!not_ready) {
      base -= 32;
    }
  }
}

}  // namespace

__global__ void __launch_bounds__(kThreads, 5) alz_zcross_kernel(const __grid_constant__ ZcArgs a) {
  __shared__ unsigned s_tile;
  __shared__ int s_agg[kChunks * kWarps];     // last decisive sign of each (chunk, warp), 0: none
  __shared__ int s_excl[kChunks * kWarps];    // carried sign at the start of each (chunk, warp)
  __shared__ int s_wtot[kChunks * kWarps];    // crossings of each (chunk, warp)
  __shared__ int s_wpre[kChunks * kWarps];
  __shared__ unsigned s_quad[kChunks * kThreads];   // crossings before the quad in the tile << 4 | the quad's crossings

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) s_tile = atomicAdd(a.ticket, 1u);
  __syncthreads();
  const long long t = s_tile, s = t / a.nt, j = t % a.nt;
  const float* xr = a.x + s * a.xs;
  const long long off = (long long)(((uintptr_t)xr >> 2) & 3);   // the tile grid starts at the aligned address xr - off
  const long long T = a.T;
  const float hf = a.hf;
  const unsigned char* st = a.state + s * a.sstride;
  const long long consumed = *reinterpret_cast<const long long*>(st);
  const int state_sign = *reinterpret_cast<const int*>(st + 8);

  // per quad, 4 bits each: lt = x < -hf, gt = x > hf (decisive = lt | gt; a crossing from +1 is lt, from -1 gt) and
  // pos = !(x < 0), the sign a decisive sample sets; samples outside the stream are neither lt nor gt
  unsigned lt[kChunks], gt[kChunks], pos[kChunks];
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    const long long p = j * kTile + (k * kThreads + tid) * 4 - off;
    float v[4];
    unsigned valid = 15u;
    if (p >= 0 && p + 3 < T) {
      const float4 q = __ldg(reinterpret_cast<const float4*>(xr + p));
      v[0] = q.x, v[1] = q.y, v[2] = q.z, v[3] = q.w;
    } else {
      valid = 0;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const bool in = p + e >= 0 && p + e < T;
        v[e] = in ? __ldg(xr + p + e) : 0.f;
        valid |= (unsigned)in << e;
      }
    }
    lt[k] = gt[k] = pos[k] = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      lt[k] |= (unsigned)(v[e] < -hf) << e;
      gt[k] |= (unsigned)(v[e] > hf) << e;
      pos[k] |= (unsigned)!(v[e] < 0.f) << e;
    }
    lt[k] &= valid;
    gt[k] &= valid;
  }

  int pin[kChunks];
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    const unsigned dec = lt[k] | gt[k];
    const bool has = dec != 0;
    const unsigned nz = __ballot_sync(0xffffffffu, has);
    const unsigned ps = __ballot_sync(0xffffffffu, has && ((pos[k] >> (31 - __clz(dec))) & 1u));
    const unsigned before = nz & ((1u << lane) - 1);
    pin[k] = before ? sign_of_last(before, ps) : 0;
    if (lane == 0) s_agg[k * kWarps + warp] = nz ? sign_of_last(nz, ps) : 0;
  }
  __syncthreads();

  if (warp == 0) {
    unsigned* desc = a.desc + s * a.nt;
    const int ag = s_agg[lane];
    const unsigned nz = __ballot_sync(0xffffffffu, ag != 0), ps = __ballot_sync(0xffffffffu, ag > 0);
    const int agg = nz ? sign_of_last(nz, ps) : 0;
    int carry;
    if (j == 0) {
      carry = state_sign;
      if (lane == 0) st_volatile(desc, descriptor(kInc, agg ? agg : carry));
    } else {
      if (lane == 0) st_volatile(desc + j, agg ? descriptor(kInc, agg) : descriptor(kAgg, 0));
      carry = look_back(desc, j, state_sign, lane);
      if (lane == 0 && !agg) st_volatile(desc + j, descriptor(kInc, carry));
    }
    const unsigned before = nz & ((1u << lane) - 1);
    s_excl[lane] = before ? sign_of_last(before, ps) : carry;
  }
  __syncthreads();

  uint8_t* fr = a.flags ? a.flags + s * a.fs : nullptr;
  unsigned cm[kChunks];
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    int sp = pin[k] ? pin[k] : s_excl[k * kWarps + warp];
    cm[k] = 0;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      cm[k] |= (sp > 0 ? (lt[k] >> e) & 1u : (sp < 0 ? (gt[k] >> e) & 1u : 0u)) << e;
      if (((lt[k] | gt[k]) >> e) & 1u) sp = ((pos[k] >> e) & 1u) ? 1 : -1;
    }
    if (fr) {
      const long long p = j * kTile + (k * kThreads + tid) * 4 - off;
      const bool full = p >= 0 && p + 3 < T;
      if (full && (((uintptr_t)(fr + p)) & 3) == 0) {
        *reinterpret_cast<uint32_t*>(fr + p) = (cm[k] & 1u) | ((cm[k] >> 1) & 1u) << 8 | ((cm[k] >> 2) & 1u) << 16 |
                                               ((cm[k] >> 3) & 1u) << 24;
      } else {
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (p + e >= 0 && p + e < T) fr[p + e] = (uint8_t)((cm[k] >> e) & 1u);
      }
    }
  }
  if (a.size == 0) return;

  // counts (kept in the state even when they are not stored): the tile's prefix counts of crossings, per quad
  int incl[kChunks];
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    int c = __popc(cm[k]);
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, c, d);
      if (lane >= d) c += o;
    }
    incl[k] = c;
    if (lane == 31) s_wtot[k * kWarps + warp] = c;
  }
  __syncthreads();
  if (warp == 0) {
    const int w = s_wtot[lane];
    int c = w;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const int o = __shfl_up_sync(0xffffffffu, c, d);
      if (lane >= d) c += o;
    }
    s_wpre[lane] = c - w;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < kChunks; ++k) {
    const int pre = s_wpre[k * kWarps + warp] + incl[k] - __popc(cm[k]);
    s_quad[k * kThreads + tid] = (unsigned)pre << 4 | cm[k];
  }
  __syncthreads();
  const int total = s_wpre[kChunks * kWarps - 1] + s_wtot[kChunks * kWarps - 1];
  const long long v0 = j * kTile - off;                           // sample index of the tile's first position
  const long long p0 = v0 > 0 ? v0 : 0, p1 = v0 + kTile < T ? v0 + kTile : T;
  if (p0 >= p1) return;
  auto before = [&](long long p) -> int {                         // crossings at samples [v0, p) of the tile
    const long long l = p - v0;
    if (l >= kTile) return total;
    const unsigned w = s_quad[l >> 2];
    return (int)(w >> 4) + __popc(w & 15u & ((1u << (l & 3)) - 1));
  };
  const long long A0 = consumed + p0, A1 = consumed + p1;
  const long long ka = first_open_block(consumed, a.size, a.hop);
  const long long kmin = first_open_block(A0, a.size, a.hop), kmax = floordiv(A1 - 1, a.hop);
  int32_t* acc = a.acc + s * a.nacc;
  for (long long k = kmin + tid; k <= kmax; k += kThreads) {
    const long long b0 = k * a.hop, b1 = b0 + a.size;
    const long long lo = (b0 > A0 ? b0 : A0) - consumed, hi = (b1 < A1 ? b1 : A1) - consumed;
    if (lo >= hi) continue;
    const int c = before(hi) - before(lo);
    if (c) atomicAdd(acc + (k - ka), c);
  }
}

// After the tiles of a call: per stream (one CTA), the carried sign, the completed and open blocks, the sample count.
__global__ void __launch_bounds__(kThreads) alz_zcross_finish_kernel(const __grid_constant__ ZcArgs a) {
  const long long s = blockIdx.x;
  unsigned char* st = a.state + s * a.sstride;
  const long long C0 = *reinterpret_cast<const long long*>(st), C1 = C0 + a.T;
  if (a.size > 0) {
    int32_t* part = reinterpret_cast<int32_t*>(st + 16);
    int32_t* acc = a.acc + s * a.nacc;
    const long long ka = first_open_block(C0, a.size, a.hop);
    const long long kb = floordiv(C1 - 1, a.hop);                  // last block with a sample before C1
    const long long kopen = floordiv(C0 - 1, a.hop);               // blocks ka..kopen started before the call
    for (long long k = ka + threadIdx.x; k <= kopen; k += blockDim.x) acc[k - ka] += part[k % a.R];
    __syncthreads();
    const long long kc = floordiv(C1 - a.size, a.hop);             // last completed block
    const long long n_done = kc - ka + 1 > 0 ? kc - ka + 1 : 0;
    for (long long k = ka + threadIdx.x; k <= kb; k += blockDim.x) {
      if (k <= kc) {
        if (a.counts) a.counts[s * a.cs + (k - ka)] = acc[k - ka];
      } else if (!a.final_) {
        part[k % a.R] = acc[k - ka];
      }
    }
    if (a.final_ && a.counts && threadIdx.x == 0) {
      const long long kp = kc + 1 > 0 ? kc + 1 : 0;
      const long long over = a.size > a.hop ? a.size - a.hop : 0;
      if (C1 - kp * a.hop > over) a.counts[s * a.cs + n_done] = acc[kp - ka];
    }
  }
  if (threadIdx.x == 0) {
    if (a.nt > 0) {
      const unsigned w = *(const volatile unsigned*)(a.desc + s * a.nt + a.nt - 1);
      *reinterpret_cast<int*>(st + 8) = (int)(w >> 4) - 1;
    }
    *reinterpret_cast<long long*>(st) = C1;
  }
}

__global__ void __launch_bounds__(kThreads) alz_zcross_init_kernel(unsigned char* state, long long n_streams,
                                                                   long long sstride, int sign) {
  const long long words = sstride / 4;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n_streams * words;
       i += (long long)gridDim.x * blockDim.x)
    reinterpret_cast<int*>(state)[i] = i % words == 2 ? sign : 0;
}

extern "C" {

const char* alz_zcross_last_error(void) { return g_err.c_str(); }

int64_t alz_zcross_state_bytes(int64_t n_streams, int32_t size, int32_t hop) {
  if (n_streams < 0 || size < 0 || hop < 1) return fail(ALZ_ZCROSS_ERR_INVALID, "need n_streams >= 0, size >= 0, hop >= 1");
  return n_streams * state_stride(size, hop);
}

int32_t alz_zcross_state_init(void* state_dev, int64_t n_streams, double first_sign, int32_t size, int32_t hop,
                              void* cuda_stream) {
  if (n_streams < 0 || size < 0 || hop < 1) return fail(ALZ_ZCROSS_ERR_INVALID, "need n_streams >= 0, size >= 0, hop >= 1");
  if (n_streams == 0) return ALZ_ZCROSS_OK;
  if (!state_dev) return fail(ALZ_ZCROSS_ERR_INVALID, "state is NULL");
  const int sign = first_sign == 0 ? 0 : (first_sign < 0 ? -1 : 1);
  const long long n = n_streams * (state_stride(size, hop) / 4);
  const unsigned blocks = (unsigned)((n + kThreads - 1) / kThreads < 4096 ? (n + kThreads - 1) / kThreads : 4096);
  alz_zcross_init_kernel<<<blocks, kThreads, 0, (cudaStream_t)cuda_stream>>>((unsigned char*)state_dev, n_streams,
                                                                            state_stride(size, hop), sign);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_ZCROSS_ERR_CUDA);
  return ALZ_ZCROSS_OK;
}

int64_t alz_zcross_scratch_bytes(int64_t n_streams, int64_t n_samples, int32_t size, int32_t hop) {
  if (n_streams < 0 || n_samples < 0 || size < 0 || hop < 1) return fail(ALZ_ZCROSS_ERR_INVALID, "bad shape");
  return 16 + 4 * n_streams * (tiles_per_stream(n_samples) + acc_per_stream(n_samples, size, hop));
}

int32_t alz_zcross_apply_f32(const float* x_dev, int64_t x_stride, uint8_t* flags_dev, int64_t flags_stride,
                             int32_t* counts_dev, int64_t counts_stride, void* state_dev, int64_t n_streams,
                             int64_t n_samples, int32_t size, int32_t hop, double hysteresis, int32_t final,
                             void* scratch_dev, int64_t scratch_bytes, void* cuda_stream) {
  if (n_streams < 0 || n_samples < 0 || size < 0 || hop < 1) return fail(ALZ_ZCROSS_ERR_INVALID, "bad shape");
  if (counts_dev && size < 1) return fail(ALZ_ZCROSS_ERR_INVALID, "counts need size >= 1");
  if (n_streams == 0) return ALZ_ZCROSS_OK;
  if (!state_dev || !scratch_dev || (n_samples > 0 && !x_dev)) return fail(ALZ_ZCROSS_ERR_INVALID, "NULL buffer");
  if (((uintptr_t)x_dev & 3) || ((uintptr_t)state_dev & 7) || ((uintptr_t)scratch_dev & 3))
    return fail(ALZ_ZCROSS_ERR_INVALID, "misaligned buffer");
  if (n_streams > 1 && (x_stride < n_samples || (flags_dev && flags_stride < n_samples)))
    return fail(ALZ_ZCROSS_ERR_INVALID, "stride < n_samples");
  if (scratch_bytes < alz_zcross_scratch_bytes(n_streams, n_samples, size, hop))
    return fail(ALZ_ZCROSS_ERR_INVALID, "scratch of %lld bytes, %lld needed", (long long)scratch_bytes,
                (long long)alz_zcross_scratch_bytes(n_streams, n_samples, size, hop));
  const long long nt = tiles_per_stream(n_samples);
  if (n_streams * nt > 0x7fffffffLL || n_streams > 0x7fffffffLL)
    return fail(ALZ_ZCROSS_ERR_UNSUPPORTED, "too many tiles for one launch");
  ZcArgs a{};
  a.x = x_dev;
  a.flags = flags_dev;
  a.counts = counts_dev;
  a.state = (unsigned char*)state_dev;
  a.ticket = (unsigned*)scratch_dev;
  a.desc = a.ticket + 4;
  a.acc = (int32_t*)(a.desc + n_streams * nt);
  a.xs = x_stride;
  a.fs = flags_stride;
  a.cs = counts_stride;
  a.sstride = state_stride(size, hop);
  a.T = n_samples;
  a.nt = nt;
  a.nacc = acc_per_stream(n_samples, size, hop);
  a.size = size;
  a.hop = hop;
  a.R = (int)ring_slots(size, hop);
  a.final_ = final != 0;
  if (std::isnan(hysteresis)) {
    a.hf = NAN;
  } else {
    a.hf = (float)hysteresis;                                     // the largest float32 <= hysteresis
    if ((double)a.hf > hysteresis) a.hf = std::nextafter(a.hf, -INFINITY);
  }
  const cudaStream_t cs = (cudaStream_t)cuda_stream;
  ALZ_CUDA_CHECK(cudaMemsetAsync(scratch_dev, 0, (size_t)alz_zcross_scratch_bytes(n_streams, n_samples, size, hop), cs),
                 ALZ_ZCROSS_ERR_CUDA);
  if (nt > 0) {
    alz_zcross_kernel<<<(unsigned)(n_streams * nt), kThreads, 0, cs>>>(a);
    ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_ZCROSS_ERR_CUDA);
  }
  alz_zcross_finish_kernel<<<(unsigned)n_streams, kThreads, 0, cs>>>(a);
  ALZ_CUDA_CHECK(cudaGetLastError(), ALZ_ZCROSS_ERR_CUDA);
  return ALZ_ZCROSS_OK;
}

}  // extern "C"
