// alz_plan.h -- private to the library: the plan object and the helpers shared by the
// translation units (alz_capi.cu = the C ABI; alz_inst_*.cu = the biquad kernel instantiations,
// split by cascade length so that they compile in parallel).  Nothing here is exported.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>
#include <atomic>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <vector>

#include "alz_generic.cuh"
#include "alz_lane.cuh"

// status codes of include/alz_b200.h (kept in sync by a static_assert in alz_capi.cu)
#define ALZI_OK 0
#define ALZI_ERR_CUDA (-4)
#define ALZI_ERR_UNSUPPORTED (-6)

int alzi_fail(int code, const char* fmt, ...);
int alzi_env_int(const char* name, int dflt);
void alzi_keep_async_pool();
extern std::atomic<long long> alzi_launches;

#define ALZ_CUDA(expr)                                                                        \
  do {                                                                                        \
    cudaError_t e__ = (expr);                                                                 \
    if (e__ != cudaSuccess)                                                                   \
      return alzi_fail(ALZI_ERR_CUDA, "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
  } while (0)

struct AlzHostPipe {   // lazily created resources of alz_apply_f32_host
  static const int NBUF = 4;
  cudaStream_t stream[NBUF] = {};
  cudaEvent_t done[NBUF] = {};
  float* dx[NBUF] = {};
  float* dy[NBUF] = {};
  double* dst[NBUF] = {};     // envelope entry: per-chunk recurrence states and lowpass states
  double* des[NBUF] = {};
  size_t dx_bytes = 0, dy_bytes = 0, dst_bytes = 0, des_bytes = 0;
  bool ready = false;
};

struct alz_plan {
  int kind = 0, C = 0, K = 0, NB = 0, NB0 = 0, monic = 0, device = 0, sm_count = 132;
  int zmask = 0;               // biquad: numerator taps that are zero in every channel (AlzBiquadCore ZMASK)
  int xd = 0, yd = 0;          // history depths exposed to alz_state_init
  int state_doubles = 0;       // per recurrence
  int fp64_ops = 0;            // FP64 instructions per channel-sample of a float64-tier channel
  int fp64_ops_exact = 0;
  int n_fp32 = 0;              // biquad: channels on the float32 tier
  double tier_tol = 0.0;       // measured-error threshold the tier decision used
  int probe_len = 8192;        // samples per probe signal of the tier decision
  int tile_group = 4;          // TMA engine: tiles moved together by launches that fill the machine (1, 2, 4; alz_capi.cu)
  bool tile_group_forced = false;   // ALZ_TILE_GROUP: tile_group on every TMA launch, whatever its size
  bool vec_store = true;       // TMA launches of tile group 4 store rows with st.global.v4 (ALZ_STORE_PATH=tma: TMA boxes)
  // TMA bank kernel: CTAs resident per SM with 2 / 4 tile buffers (occupancy query on the plan's first TMA launch; 0 = not
  // yet).  Host threads that race on the first launch store the same value.
  mutable std::atomic<int> tma_ctas_per_sm[2] = {};
  bool parallel_sum = false;   // ALZ_PLAN_PARALLEL: plain float64 records, usable by alz_apply_sum_f32
  bool sequential = false;     // ALZ_PLAN_SEQUENTIAL: never evaluate time-parallel (bit-reproducible blocking)
  double chunk_err = 0.0;      // biquad: measured error of one chunk transition of the time-parallel evaluation
  bool coef_small = false;     // kernel-parameter block size (kCoefSmall / kCoefLarge doubles)
  struct Chunk { void* block; int npos; };
  std::vector<Chunk> chunks;   // biquad: pre-built AlzBiquadArgs<NCOEF> blocks, <= NCOEF / stride positions each
  // generic plans of ONE section per channel run on the window kernels (alz_window.cuh)
  bool window = false;
  int win_mx = 0, win_my = 0;           // near-window slots per history (0, 4, 16)
  int win_xwin = 0, win_ywin = 0;       // state slots of the near windows
  int win_xbase = 0, win_xmask = -1, win_ybase = 0, win_ymask = -1;   // far rings
  std::vector<int> win_far_delay;       // numerator taps first
  int win_nfx = 0, win_nfy = 0;
  void* win_block = nullptr;            // host AlzWindowArgs<NCOEF>
  int* d_far_delay = nullptr;
  double* d_far_coef = nullptr;
  // device tables
  double* d_coef = nullptr;
  AlzGenSection* d_sec = nullptr;
  int* d_tap_delay = nullptr;
  // host copies used by alz_state_init
  std::vector<double> h_tab;              // biquad: [position][ALZ_COEF_STRIDE] coefficient records (kernel parameters)
  std::vector<int> pos_channel;           // biquad: position -> channel
  std::vector<int> tier;                  // biquad: per CHANNEL precision tier (0 float64, 1 float32)
  std::vector<double> tier_err;           // biquad: per channel measured float32 error (probe), < 0 = not probed
  std::vector<double> sc;                 // biquad: [C][K+1] working-unit scales
  std::vector<AlzGenSection> h_sec;       // generic
  std::vector<int> h_xlen, h_ylen;        // generic: true max delays per section
  std::vector<int> h_tap_delay, h_tap_is_den;   // generic: tap order of the coefficient table
  // normalised sections as given (a0 == 1), for alz_freq_response_f64
  std::vector<double> fr_coef;            // b then a of every (channel, section), concatenated
  std::vector<int> fr_desc;               // [C][K][3] = nb, na, offset (nb == 0: absent)
  double* d_fr_coef = nullptr;
  int fr_K = 0;
  int* d_fr_desc = nullptr;
  // users: calls that hold the entry between their lookup and the launch of their last reader of M (chunk_release);
  // an entry evicted while held is freed by the call that drops its last user
  struct MEntry { long long L; double* M; cudaEvent_t ready; int users; bool evicted; };
  std::mutex m_mu;                // guards m_cache and every entry's users / evicted (NOT host_mu: alz_apply_f32_host
                                  // holds that one across its launches)
  std::vector<MEntry*> m_cache;   // time-parallel evaluation: chunk transition matrices A^L per chunk length (device)
  std::mutex host_mu;
  AlzHostPipe pipe;
};

// Biquad launches, one translation unit per cascade length (alz_inst_*.cu).
int alzi_launch_biquad_k1(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_biquad_k2(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_biquad_k3(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_biquad_k4(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_biquad_k6(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_biquad_k8(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_headfir_k1(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_headfir_k4(const alz_plan*, const AlzTileArgs&, cudaStream_t);

int alzi_launch_envelope_k4(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_envelope_headfir_k4(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_window(const alz_plan*, const AlzTileArgs&, cudaStream_t);
int alzi_launch_parallel(const alz_plan*, const AlzTileArgs&, const CUtensorMap& tmx, const CUtensorMap& tmo, cudaStream_t);
size_t alzi_window_block_bytes(bool small);
void alzi_window_block_fill(void* blk, bool small, int n_far_x, int n_far_y, int xbase, int xmask, int ybase, int ymask, int xwin,
                            int ywin, int C, const int* far_delay, const double* far_coef, const double* coef);

// Plan-time tier probe (host): runs channel records through the SAME core arithmetic in float64
// and float32 on probe signals, returns the float32 tier's error relative to the row peak.
// rec64 / rec32: one record each (ALZ_COEF_STRIDE doubles).
double alzi_probe_biquad_k1(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_biquad_k2(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_biquad_k3(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_biquad_k4(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_biquad_k6(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_biquad_k8(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_headfir_k1(const alz_plan*, const double* rec64, const double* rec32);
double alzi_probe_headfir_k4(const alz_plan*, const double* rec64, const double* rec32);

// tensor maps of x[S][T] / y[S][C][T] (alz_capi.cu)
bool alzi_make_tensor_maps(const AlzTileArgs& ta, CUtensorMap* tmx, CUtensorMap* tmy);
