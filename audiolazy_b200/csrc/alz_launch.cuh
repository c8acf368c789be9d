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
static const int kWarpsPerSmTma = 24;   // TMA engine: 2 x 4096 B + barriers + reserve -> 24 CTAs per SM

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

// TMA variant: same cores, tiles moved by cp.async.bulk.tensor (16-byte aligned rows only).
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
__global__ void __launch_bounds__(32, kWarpsPerSmTma)
alz_biquad_tma_kernel(const __grid_constant__ AlzTileArgs a, const __grid_constant__ AlzBiquadArgs<NCOEF> ca,
                      const __grid_constant__ CUtensorMap tmx, const __grid_constant__ CUtensorMap tmy) {
  extern __shared__ __align__(1024) unsigned char alz_smem_tma[];
  if (ca.tier(blockIdx.x) == 0)
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, double>>(a, ca, &tmx, &tmy, alz_smem_tma);
  else
    alz_run_warp_tma<AlzBiquadCore<K, NB, MONIC, NB0, ZMASK, float>>(a, ca, &tmx, &tmy, alz_smem_tma);
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

// One launch: positions [p0, p0+npos) x stream groups of `ta` (ta.S <= 65535*32 streams).  `block` is
// the plan's pre-built AlzBiquadArgs<NCOEF> for this chunk.
template <int K, int NB, int MONIC, int NCOEF, int NB0, int ZMASK>
static int launch_biquad_chunk(const alz_plan* p, AlzTileArgs ta, const void* block, int npos, cudaStream_t st) {
  const long long groups = (ta.S + 31) / 32;
  CUtensorMap tmx, tmy;
  if (alzi_make_tensor_maps(ta, &tmx, &tmy)) {
    // A launch of only a few waves of warps loses its last, partly filled wave: cut time into
    // segments chained through the state (alz_lane_tma.cuh) so the next segment fills the tail.
    const long long warps = (long long)npos * groups;
    int ng = warps >= (long long)p->sm_count * kWarpsPerSmTma ? p->tile_group : 1;
    ng = alzi_env_int("ALZ_TMA_PAIRED", ng);     // 0/1 = prefetch pipeline, 2 / 4 = tile groups
    if (ng != 2 && ng != 4) ng = 1;
    ta.paired = ng;
    ta.exp |= alzi_env_int("ALZ_EXP", 0);
    const size_t smem = ALZ_TMA_SMEM_FOR(ng);
    const long long per_sm = std::min<long long>(kWarpsPerSmTma, (228 * 1024) / (long long)(smem + 1024));
    const long long slots = (long long)p->sm_count * per_sm;
    long long nseg = 1;
    if (ta.vP == 0 && warps > slots && warps < 8 * slots && ta.T >= 2048 && !alzi_env_int("ALZ_NO_SEGMENT", 0)) {
      const long long waves = std::max(1, alzi_env_int("ALZ_SEG_WAVES", 16)), min_len = std::max(32, alzi_env_int("ALZ_SEG_MIN", 1024));
      nseg = std::min((waves * slots + warps - 1) / warps, ta.T / min_len);
      const long long quantum = 32ll * ng;     // whole tile groups per segment
      const long long len = ((ta.T + nseg - 1) / nseg + quantum - 1) / quantum * quantum;
      nseg = (ta.T + len - 1) / len;
      if (nseg > 1 && groups * nseg <= 65535) {
        const size_t words = (size_t)npos + (size_t)npos * groups;
        unsigned* sync = nullptr;
        alzi_keep_async_pool();
        ALZ_CUDA(cudaMallocAsync(&sync, words * 4, st));
        if (cudaMemsetAsync(sync, 0, words * 4, st) != cudaSuccess) {
          cudaFreeAsync(sync, st);
          ALZ_CUDA(cudaGetLastError());
        }
        ta.nseg = (int)nseg; ta.seg_len = len; ta.sync = sync;
      } else {
        nseg = 1;
      }
    }
    ta.groups = (int)groups;
    auto kern = alz_biquad_tma_kernel<K, NB, MONIC, NCOEF, NB0, ZMASK>;
    if (smem > 48 * 1024) return alzi_fail(ALZI_ERR_UNSUPPORTED, "tile group too large");
    void* args[4] = {(void*)&ta, const_cast<void*>(block), (void*)&tmx, (void*)&tmy};
    const cudaError_t e = cudaLaunchKernel((const void*)kern, dim3((unsigned)npos, (unsigned)(groups * nseg)), dim3(32), args, smem, st);
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
