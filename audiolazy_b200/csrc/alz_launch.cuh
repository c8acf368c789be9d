// alz_launch.cuh -- the biquad kernels and their launch / probe code, as templates over the
// cascade length K.  Included by the alz_inst_*.cu translation units (one per K, compiled in
// parallel); alz_capi.cu reaches them through the alzi_* functions declared in alz_plan.h.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstring>

#include "alz_biquad.cuh"
#include "alz_lane_tma.cuh"
#include "alz_plan.h"

// Kernel-parameter coefficient capacity (doubles).  CUDA 12.1+ allows 32764 bytes of
// parameters; two sizes so that small filters do not push 28 KB per launch.
static const int kCoefSmall = 512, kCoefLarge = 3584;
static const int kWarpsPerSm = 22;      // cp.async engine: 2 x 4608 B tile buffers + 1 KB CTA reserve -> 22 CTAs per SM
static const int kWarpsPerSmTma = 24;   // TMA engine launch bounds: 80 registers, 24 CTAs per SM (bank launches query it)
static const double kSegTailIdle = 0.02;   // largest share of a bank launch's warp slots its last wave may leave idle

// Both precision tiers live in one kernel: the tier of a grid position is warp (= CTA) uniform,
// read from the position's coefficient record.  Float64 and float32 warps of different channels
// are co-resident on every SM (the plan interleaves the tiers along blockIdx.x), so the FP32 pipe
// works in the issue slots the 2-cycle DFMAs leave free.
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
__global__ void __launch_bounds__(32, kWarpsPerSm)
alz_biquad_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzBiquadArgs<NCOEF> ca) {
  extern __shared__ __align__(16) float alz_smem[];
  if (ca.tier(blockIdx.x) == 0) alz_run_warp<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, double>>(a, ca, alz_smem);
  else alz_run_warp<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, float>>(a, ca, alz_smem);
}

// Instantiations with the vector store path of tile groups of 4 (alz_run_warp_tma): all but the head-FIR ones, whose
// plans (19 FP64 instructions per channel-sample) keep tile group 2 unless ALZ_TILE_GROUP forces 4.
template <int NB0>
constexpr bool kVecStore = NB0 != 8;

// TMA variant: same cores, tiles moved by cp.async.bulk.tensor (16-byte aligned rows only).
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
__global__ void __launch_bounds__(32, kWarpsPerSmTma)
alz_biquad_tma_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzBiquadArgs<NCOEF> ca,
                      const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy) {
  extern __shared__ __align__(1024) unsigned char alz_smem_tma[];
  if (ca.tier(blockIdx.x) == 0)
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, double>, AlzStoreY, kVecStore<NB0>>(a, ca, &tmx, &tmy, alz_smem_tma);
  else
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, float>, AlzStoreY, kVecStore<NB0>>(a, ca, &tmx, &tmy, alz_smem_tma);
}

// Envelope consumer (AlzEnvelopePost): the bank's outputs are rectified / squared, lowpassed and decimated in the kernel;
// instantiated for the gammatone banks only (K = 4, input-side gain, one parameter block).
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
__global__ void __launch_bounds__(32, kWarpsPerSmTma)
alz_biquad_envelope_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzBiquadArgs<NCOEF> ca,
                           const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy) {
  extern __shared__ __align__(1024) unsigned char alz_smem_tma[];
  if (ca.tier(blockIdx.x) == 0)
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, double>, AlzEnvelopePost>(a, ca, &tmx, &tmy, alz_smem_tma);
  else
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, float>, AlzEnvelopePost>(a, ca, &tmx, &tmy, alz_smem_tma);
}

template <int K, int NB, int NB0, int ZMASK>
static int launch_envelope_t(const alz_plan* p, AlzTileArgs ta, cudaStream_t st) {
  if (p->coef_small || p->chunks.size() != 1)
    return alzi_fail(ALZI_ERR_UNSUPPORTED, "envelope consumer: gammatone-bank plans only");
  CUtensorMap tmx, tmy;
  if (!alzi_make_tensor_maps(ta, &tmx, &tmy)) return alzi_fail(ALZI_ERR_UNSUPPORTED, "envelope consumer needs 16-byte aligned x rows");
  const long long groups = (ta.S + 31) / 32;
  ta.paired = (long long)p->chunks[0].npos * groups >= (long long)p->sm_count * kWarpsPerSmTma ? 2 : 1;
  ta.groups = (int)groups;
  void* args[4] = {(void*)&ta, p->chunks[0].block, (void*)&tmx, (void*)&tmy};
  const void* kern = p->monic == 2 ? (const void*)alz_biquad_envelope_kernel<K, NB, 2, kCoefLarge, NB0, ZMASK>
                   : p->monic == 1 ? (const void*)alz_biquad_envelope_kernel<K, NB, 1, kCoefLarge, NB0, ZMASK>
                                   : (const void*)alz_biquad_envelope_kernel<K, NB, 0, kCoefLarge, NB0, ZMASK>;
  ALZ_CUDA(cudaLaunchKernel(kern, dim3((unsigned)p->chunks[0].npos, (unsigned)groups), dim3(32), args, ALZ_TMA_SMEM_FOR(ta.paired), st));
  ALZ_CUDA(cudaGetLastError());
  alzi_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZI_OK;
}

// CTAs of the TMA bank kernel `kern` resident per SM with the tile buffers of group size `ng`: the occupancy of the
// instantiation on the plan's device (registers, shared memory, the 1 KB reserve per CTA), queried once per plan and
// buffer count.  The shared-memory carveout is asked for at its maximum, so that on an H100 13 CTAs of 4 tiles (17.4 KB
// each with the reserve) share the 228 KB of an SM.
static int tma_ctas_per_sm(const alz_plan* p, const void* kern, int ng, long long* out) {
  std::atomic<int>& cached = p->tma_ctas_per_sm[ng >= 4 ? 1 : 0];
  int n = cached.load(std::memory_order_relaxed);
  if (n == 0) {
    ALZ_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    ALZ_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, 32, ALZ_TMA_SMEM_FOR(ng)));
    if (n < 1) return alzi_fail(ALZI_ERR_UNSUPPORTED, "bank kernel: no CTA of %d tiles fits on an SM", ng < 2 ? 2 : ng);
    cached.store(n, std::memory_order_relaxed);
  }
  *out = n;
  return ALZI_OK;
}

// One launch: positions [p0, p0+npos) x stream groups of `ta` (ta.S <= 65535*32 streams).  `block` is
// the plan's pre-built AlzBiquadArgs<NCOEF> for this chunk.
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
static int launch_biquad_chunk(const alz_plan* p, AlzTileArgs ta, const void* block, int npos, cudaStream_t st) {
  const long long groups = (ta.S + 31) / 32;
  CUtensorMap tmx, tmy;
  if (alzi_make_tensor_maps(ta, &tmx, &tmy)) {
    const void* kern = (const void*)alz_biquad_tma_kernel<K, NB, MONIC, NCOEF, NB0, ZMASK>;
    const long long warps = (long long)npos * groups;
    const long long min_len = std::max(32, alzi_env_int("ALZ_SEG_MIN", 1024));
    const bool can_segment = ta.vP == 0 && ta.T >= 2 * min_len && !alzi_env_int("ALZ_NO_SEGMENT", 0);
    // Tile group: the plan's (alz_capi.cu) when the launch fills the machine at that group's occupancy.  A launch that
    // fits in one wave of the one-tile pipeline and cannot be cut into time segments stays there: with 4 tiles (13 CTAs
    // per SM instead of 24 on an H100) it would run a second, mostly idle wave.
    long long per_one = 0, per_group = 0;
    int rc = tma_ctas_per_sm(p, kern, 1, &per_one);
    if (rc == ALZI_OK) rc = tma_ctas_per_sm(p, kern, p->tile_group, &per_group);
    if (rc != ALZI_OK) return rc;
    const bool fills = warps >= p->sm_count * per_group && (can_segment || warps >= p->sm_count * per_one);
    int ng = p->tile_group_forced || fills ? p->tile_group : 1;
    ng = alzi_env_int("ALZ_TMA_PAIRED", ng);     // 0/1 = prefetch pipeline, 2 / 4 = tile groups
    if (ng != 2 && ng != 4) ng = 1;
    ta.paired = ng;
    // Groups of 4 tiles leave as warp-wide row stores where y allows 16-byte vectors (the TMA map already needs that
    // of its base and strides; checked here so that the kernel's addressing does not depend on it).
    ta.vec_store = ng == 4 && kVecStore<NB0> && p->vec_store && ((uintptr_t)ta.y & 15) == 0 && (ta.ys & 3) == 0 && (ta.ysS & 3) == 0 &&
                   (ta.vP == 0 || (ta.T & 3) == 0);
    ta.exp |= alzi_env_int("ALZ_EXP", 0);
    const size_t smem = ALZ_TMA_SMEM_FOR(ng);
    long long per_sm = 0;
    if ((rc = tma_ctas_per_sm(p, kern, ng, &per_sm)) != ALZI_OK) return rc;
    const long long slots = (long long)p->sm_count * per_sm;
    // Time segments chained through the state (alz_lane_tma.cuh).  The warps run in waves of `slots`, and a partly
    // filled last wave idles the rest of the slots for a whole wave: a share ceil(n w / s) s - n w of ceil(n w / s) s
    // when the launch is cut into n segments, n w warps of 1 / n the length.  A launch that would idle more than
    // kSegTailIdle of its slots is cut into the fewest segments (whole tile groups, >= min_len samples) that stay
    // within it, else into the count that idles least.  A count that idles no less than the whole launch is not taken:
    // it would pay for the segment flags and the chained waits and gain nothing.
    auto idle = [&](long long n) {
      const long long cap = (n * warps + slots - 1) / slots * slots;
      return (double)(cap - n * warps) / (double)cap;
    };
    long long nseg = 1, len = ta.T;
    if (can_segment && warps > slots && idle(1) > kSegTailIdle) {
      const long long quantum = 32ll * ng;
      double best = idle(1);
      for (long long n = 2; n <= ta.T / min_len && groups * n <= 65535; ++n) {
        const long long ln = ((ta.T + n - 1) / n + quantum - 1) / quantum * quantum;
        if ((ta.T + ln - 1) / ln != n) continue;   // fewer segments once rounded: that count is weighed on its own
        const double f = idle(n);
        if (f < best) { best = f; nseg = n; len = ln; }
        if (f <= kSegTailIdle) break;
      }
    }
    if (alzi_env_int("ALZ_LOG_LAUNCH", 0))
      fprintf(stderr, "alz bank launch: %lld warps, tile group %d, %lld CTAs per SM (%lld slots), %lld segment(s) of %lld samples, "
              "%s stores, %d chunks per stream\n", warps, ng, per_sm, slots, nseg, len, ta.vec_store ? "vector" : "TMA",
              ta.vP > 0 ? ta.vP : 1);
    if (nseg > 1) {
      const size_t words = (size_t)npos + (size_t)npos * groups;
      unsigned* sync = nullptr;
      alzi_keep_async_pool();
      ALZ_CUDA(cudaMallocAsync(&sync, words * 4, st));
      if (cudaMemsetAsync(sync, 0, words * 4, st) != cudaSuccess) {
        cudaFreeAsync(sync, st);
        ALZ_CUDA(cudaGetLastError());
      }
      ta.nseg = (int)nseg; ta.seg_len = len; ta.sync = sync;
    }
    ta.groups = (int)groups;
    if (smem > 48 * 1024) return alzi_fail(ALZI_ERR_UNSUPPORTED, "tile group too large");
    void* args[4] = {(void*)&ta, const_cast<void*>(block), (void*)&tmx, (void*)&tmy};
    const cudaError_t e = cudaLaunchKernel(kern, dim3((unsigned)npos, (unsigned)(groups * nseg)), dim3(32), args, smem, st);
    if (ta.sync) cudaFreeAsync(ta.sync, st);
    ALZ_CUDA(e);
  } else {
    if (ta.exp & 2) ta.y = nullptr;   // cp.async engine: "no tile stores" is expressed by a null output (see alz_run_warp)
    auto kern = alz_biquad_kernel<K, NB, MONIC, NCOEF, NB0, ZMASK>;
    void* args[2] = {(void*)&ta, const_cast<void*>(block)};
    ALZ_CUDA(cudaLaunchKernel((const void*)kern, dim3((unsigned)npos, (unsigned)groups), dim3(32), args, ALZ_WARP_SMEM, st));
  }
  ALZ_CUDA(cudaGetLastError());
  alzi_launches.fetch_add(1, std::memory_order_relaxed);
  return ALZI_OK;
}

template <int K, int NB, int MONIC, int NB0, int ZMASK>
static int launch_biquad_t(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  for (const auto& ch : p->chunks) {
    const int rc = p->coef_small ? launch_biquad_chunk<K, NB, MONIC, kCoefSmall, NB0, ZMASK>(p, ta, ch.block, ch.npos, st)
                                 : launch_biquad_chunk<K, NB, MONIC, kCoefLarge, NB0, ZMASK>(p, ta, ch.block, ch.npos, st);
    if (rc != ALZI_OK) return rc;
  }
  return ALZI_OK;
}

template <int K, int NB, int NB0, int ZMASK = 0>
static int launch_biquad_nb(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  if (p->monic == 2) return launch_biquad_t<K, NB, 2, NB0, ZMASK>(p, ta, st);
  if (p->monic == 1) return launch_biquad_t<K, NB, 1, NB0, ZMASK>(p, ta, st);
  return launch_biquad_t<K, NB, 0, NB0, ZMASK>(p, ta, st);
}

template <int K>
static int launch_biquad_k(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  switch (p->NB) {
    case 1: return launch_biquad_nb<K, 1, 0>(p, ta, st);
    case 2: return launch_biquad_nb<K, 2, 0>(p, ta, st);
    default:
      if constexpr (K == 4) {
        if ((p->zmask & ALZ_ZMASK_KLAPURI) == ALZ_ZMASK_KLAPURI) return launch_biquad_nb<4, 3, 0, ALZ_ZMASK_KLAPURI>(p, ta, st);
      }
      return launch_biquad_nb<K, 3, 0>(p, ta, st);
  }
}

// head-FIR plans: first section with up to 8 numerator taps (K in {1, 4}, NB in {1, 3}).  NB counts the taps of the
// sections AFTER the first, so a one-section plan always has NB = 1: K = 1 is instantiated for NB = 1 only.
template <int K>
static int launch_headfir_k(const alz_plan* p, const AlzTileArgs& ta, cudaStream_t st) {
  if constexpr (K == 1) return launch_biquad_nb<1, 1, 8>(p, ta, st);
  else {
    if (p->NB <= 1) return launch_biquad_nb<K, 1, 8>(p, ta, st);
    return launch_biquad_nb<K, 3, 8>(p, ta, st);
  }
}

// ---- plan-time tier probe (host) -------------------------------------------------------------
// Runs ONE channel through the float64 core and through the float32 core -- the very code the
// kernels execute (fma / fmaf are correctly rounded on the host as on the device) -- on three
// deterministic probe signals from a zero state -- uniform white noise; a unit step; a unit impulse;
// white noise with a full-scale Nyquist tone on top; the pure Nyquist sequence (a narrow low channel
// answers it 100+ dB down: any float32 recurrence's in-band rounding noise is then large relative to
// THAT output, and such a channel stays in float64) -- and returns max over the signals of
// max|y32 - y64| / max|y64|.
static inline float alzi_probe_noise(unsigned& s) {   // uniform in [-1, 1), LCG (Numerical Recipes constants)
  s = s * 1664525u + 1013904223u;
  return (float)((double)(s >> 8) * (2.0 / 16777216.0) - 1.0);
}

template <int K, int NB, int MONIC, int NB0, int ZMASK>
static double probe_biquad_t(const double* rec64, const double* rec32, int n) {
  double worst = 0.0;
  for (int sig = 0; sig < 5; ++sig) {
    AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, double> c64;
    AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, float> c32;
    c64.load_coef(rec64); c64.zero_state();
    c32.load_coef(rec32); c32.zero_state();
    unsigned seed = 12345u;
    double peak = 0.0, err = 0.0;
    for (int i = 0; i < n; ++i) {
      const float nyq = (i & 1) ? -1.0f : 1.0f;
      const float x = sig == 0 ? alzi_probe_noise(seed) : sig == 1 ? 1.0f : sig == 2 ? (i == 0 ? 1.0f : 0.0f)
                      : sig == 3 ? 0.5f * alzi_probe_noise(seed) + 0.5f * nyq : nyq;
      float y64, y32;
      if (i < 2) { y64 = c64.step_explicit(c64.widen(x)); y32 = c32.step_explicit(c32.widen(x)); }
      else { y64 = c64.step_alias(c64.widen(x)); y32 = c32.step_alias(c32.widen(x)); }
      peak = std::max(peak, std::fabs((double)y64));
      const double d = std::fabs((double)y32 - (double)y64);
      err = std::max(err, d == d ? d : 1e300);   // NaN counts as a failure
    }
    if (peak > 0.0) worst = std::max(worst, err / peak);
    else if (err > 0.0) worst = 1e300;
  }
  return worst;
}

template <int K, int NB, int NB0, int ZMASK = 0>
static double probe_biquad_nb(const alz_plan* p, const double* r64, const double* r32, int n) {
  if (p->monic == 2) return probe_biquad_t<K, NB, 2, NB0, ZMASK>(r64, r32, n);
  if (p->monic == 1) return probe_biquad_t<K, NB, 1, NB0, ZMASK>(r64, r32, n);
  return probe_biquad_t<K, NB, 0, NB0, ZMASK>(r64, r32, n);
}

template <int K>
static double probe_biquad_k(const alz_plan* p, const double* r64, const double* r32) {
  const int n = p->probe_len;
  switch (p->NB) {
    case 1: return probe_biquad_nb<K, 1, 0>(p, r64, r32, n);
    case 2: return probe_biquad_nb<K, 2, 0>(p, r64, r32, n);
    default:
      if constexpr (K == 4) {
        if ((p->zmask & ALZ_ZMASK_KLAPURI) == ALZ_ZMASK_KLAPURI) return probe_biquad_nb<4, 3, 0, ALZ_ZMASK_KLAPURI>(p, r64, r32, n);
      }
      return probe_biquad_nb<K, 3, 0>(p, r64, r32, n);
  }
}

template <int K>
static double probe_headfir_k(const alz_plan* p, const double* r64, const double* r32) {
  if constexpr (K == 1) return probe_biquad_nb<1, 1, 8>(p, r64, r32, p->probe_len);
  else {
    if (p->NB <= 1) return probe_biquad_nb<K, 1, 8>(p, r64, r32, p->probe_len);
    return probe_biquad_nb<K, 3, 8>(p, r64, r32, p->probe_len);
  }
}
