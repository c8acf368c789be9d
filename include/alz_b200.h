/*
 * alz_b200.h -- C ABI of the H100-native AudioLazy filter hot path.
 *
 * This is the drop-in boundary for ONE path of danilobellini/audiolazy: the
 * sample-by-sample linear filter evaluator and its composites.  The reference
 * has no FFI; its operator contract is "a filter is any callable that receives
 * an iterable and returns a Stream" (reference audiolazy/lazy_filters.py:975-978,
 * :1033-1036).  The entry points below are what a ctypes binding of that path
 * binds (see INTEGRATION.md for the stub a reference maintainer would add):
 *
 *   alz_plan_create      <- the per-call source generation + exec of
 *                           LinearFilter.__call__ (lazy_filters.py:197-260):
 *                           "compile" a filter (or a bank of cascades) once.
 *   alz_state_init       <- memory=/zero= seeding (lazy_filters.py:181-195,
 *                           :243-250).
 *   alz_apply_f32        <- the generated `for d0 in seq:` loop
 *                           (lazy_filters.py:251-257), CascadeFilter.__call__
 *                           (:988-990) and the bank fan-out loop
 *                           (examples/gammatone_plots.py:63-71), on DEVICE buffers.
 *   alz_apply_f32_host   <- the same through HOST buffers (what a Stream block
 *                           pump or any host caller uses); copies are inside.
 *   alz_sum_channels_f32 <- ParallelFilter.__call__'s left-associated
 *                           elementwise sum (lazy_filters.py:1048-1054).
 *   alz_freq_response_f64 <- LinearFilter.freq_response / CascadeFilter.freq_response
 *                           (lazy_filters.py:267-301, :1000-1003) for a whole bank
 *                           on a frequency grid.
 *
 * Conventions: plain pointers and sizes only; no exceptions cross the ABI; every
 * function returns 0 on success or a negative alz_status; alz_last_error() gives a
 * thread-local message for the last failure.  The caller owns every buffer.  Calls
 * are asynchronous with respect to the given CUDA stream unless stated otherwise.
 * A plan is immutable after creation and may be used concurrently from several
 * host threads / CUDA streams as long as each call uses its own state buffer.
 *
 * There is NO CPU implementation behind this ABI.  Every compute entry point
 * fails (ALZ_ERR_CUDA) when no CUDA device is usable.
 */
#ifndef ALZ_B200_H
#define ALZ_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_ABI_VERSION 2

typedef enum alz_status {
  ALZ_OK = 0,
  ALZ_ERR_INVALID = -1,    /* bad argument (null pointer, negative size, ...)          */
  ALZ_ERR_NONCAUSAL = -2,  /* reserved: host layer raises ValueError("Non-causal filter") */
  ALZ_ERR_ZERO_GAIN = -3,  /* a0 == 0: reference raises ZeroDivisionError (lazy_filters.py:177-178) */
  ALZ_ERR_CUDA = -4,       /* CUDA runtime failure or no device                        */
  ALZ_ERR_NOMEM = -5,
  ALZ_ERR_UNSUPPORTED = -6
} alz_status;

/* Which kernel family a plan dispatches to. */
typedef enum alz_kind {
  ALZ_KIND_BIQUAD = 1,   /* every section has <=3 numerator and <=3 denominator taps  */
  ALZ_KIND_GENERIC = 2   /* arbitrary (sparse) taps, ring-buffer history              */
} alz_kind;

typedef struct alz_plan alz_plan;

typedef struct alz_plan_info {
  int32_t abi_version;
  int32_t kind;              /* alz_kind                                              */
  int32_t n_channels;        /* C: independent cascades fed by the same input stream  */
  int32_t n_sections;        /* K: sections per cascade after padding                 */
  int32_t num_taps;          /* NB template value (biquad kind) or max nb (generic)   */
  int32_t monic;             /* 0 plain; 1 b0 factored out, gain on the float64 output; 2 gain on the float32 input */
  int32_t state_doubles;     /* doubles of state per (stream, channel)                */
  int32_t fp64_ops;          /* FP64 instructions per channel-sample in the hot loop  */
  int32_t device;            /* CUDA device ordinal the plan lives on                 */
  int32_t n_fp32_channels;   /* channels whose recurrence runs on the float32 tier (see alz_plan_tiers) */
  int32_t tier_tol_e9;       /* the tier decision's error threshold, in units of 1e-9 */
  int32_t time_parallel;     /* 1: a call on few long streams may be evaluated time-parallel (biquad kind, its
                                measured chunk error within the bar, not ALZ_PLAN_SEQUENTIAL)                  */
  int32_t reserved[4];
} alz_plan_info;

/* Thread-local description of the last error returned on this thread. */
const char* alz_last_error(void);

/* ABI version of the loaded library (== ALZ_ABI_VERSION it was built with). */
int32_t alz_abi_version(void);

/* Number of usable CUDA devices (0 if none; never fails). */
int32_t alz_device_count(void);

/* Make `device` the current CUDA device of the calling thread for this library
 * (plans are created on the current device; apply calls use the plan's device). */
int32_t alz_set_device(int32_t device);

/*
 * Build a plan for a bank of `n_channels` cascades of up to `max_sections`
 * direct-form-I sections on the CURRENT CUDA device.
 *
 *   section_desc[(c*max_sections + k)*3 + 0] = nb  (numerator taps, 0 => section absent)
 *   section_desc[(c*max_sections + k)*3 + 1] = na  (denominator taps incl. a0, >= 1)
 *   section_desc[(c*max_sections + k)*3 + 2] = offset into coef[]
 *   coef[offset .. offset+nb)        = b[0..nb)   (ascending delay, zeros allowed)
 *   coef[offset+nb .. offset+nb+na)  = a[0..na)   (a[0] is the gain divisor)
 *
 * Each section computes, per sample (reference lazy_filters.py:197-257):
 *   y[n] = (sum_k b[k] x[n-k] - sum_{k>=1} a[k] y[n-k]) / a[0]
 * Absent sections (nb == 0) must be trailing; a channel with no sections is the
 * identity (empty CascadeFilter, reference tests/test_filters.py:557-561).
 */
int32_t alz_plan_create(const double* coef, const int32_t* section_desc,
                        int32_t n_channels, int32_t max_sections, alz_plan** out);

/* Same with flags.  ALZ_PLAN_FORCE_GENERIC keeps every listed tap (also zero-valued ones are
 * kept if non-zero in any channel) on the generic kernel: required for time-varying plans. */
#define ALZ_PLAN_FORCE_GENERIC 1
/* ALZ_PLAN_EXACT: every channel's recurrence in float64 (no float32 precision tier, below). */
#define ALZ_PLAN_EXACT 2
/* ALZ_PLAN_DESIGN_ONLY: build the plan's tables and tier decision without touching any device
 * (works on a host without a GPU); only alz_plan_info_get / alz_plan_tiers / alz_plan_history /
 * alz_plan_state_doubles / alz_plan_destroy accept such a plan, every compute entry fails. */
#define ALZ_PLAN_DESIGN_ONLY 4
/* ALZ_PLAN_SEQUENTIAL: never use the time-parallel evaluation (see alz_apply_f32): every call is
 * evaluated sample by sample, so ANY blocking of a stream gives the same bits. */
#define ALZ_PLAN_SEQUENTIAL 8
/* ALZ_PLAN_PARALLEL: the plan is the member list of a ParallelFilter (reference lazy_filters.py:1024-1084):
 * plain float64 sections, every channel on the float64 tier; alz_apply_sum_f32 evaluates the sum in one kernel. */
#define ALZ_PLAN_PARALLEL 16
int32_t alz_plan_create_ex(const double* coef, const int32_t* section_desc, int32_t n_channels,
                           int32_t max_sections, int32_t flags, alz_plan** out);

void alz_plan_destroy(alz_plan* plan);

int32_t alz_plan_info_get(const alz_plan* plan, alz_plan_info* out);

/*
 * Precision tiers (biquad plans).  The reference evaluates everything in float64
 * (lazy_filters.py:197-257 on Python floats); the parity bar of this path is 1e-5 relative to
 * each output row's peak for float32 I/O.  At plan creation every channel is run, on the host,
 * through the kernel's own arithmetic in float64 AND in float32 on probe signals (white noise,
 * step, impulse, noise + Nyquist tone, pure Nyquist); a channel whose float32 result stays within the threshold (default 2.5e-6 =
 * a quarter of the bar; ALZ_TIER_TOL) is evaluated in float32 on the device (tier 1: FP32 pipe,
 * no conversions), all others in float64 (tier 0).  Poles near z = 1 -- low ERB channels -- fail
 * the probe by orders of magnitude and stay on tier 0.  ALZ_PLAN_EXACT or ALZ_NO_FP32_TIER=1
 * keep every channel on tier 0.  Fills tier[c] / probe_err[c] (measured float32 error, < 0 when
 * not probed) for c < min(cap, n_channels); returns n_channels.  Either array may be NULL.
 */
int32_t alz_plan_tiers(const alz_plan* plan, int32_t* tier, double* probe_err, int32_t cap);

/* Doubles of device state needed for `n_streams` input streams (>= 0), or <0 on error. */
int64_t alz_plan_state_doubles(const alz_plan* plan, int64_t n_streams);

/*
 * Initialise a device state buffer.  xinit / yinit are HOST arrays (or NULL for
 * zeros) shaped [n_channels][n_sections][xd] and [n_channels][n_sections][yd]
 * where xd / yd are returned by alz_plan_history(): entry j is the value the
 * reference would hold in d{j+1} (input pre-history, `zero`) and m{j+1}
 * (`memory`), lazy_filters.py:243-250.  The same initial history is given to
 * every stream.  Asynchronous on `cuda_stream` (the host arrays are consumed
 * before return).
 */
int32_t alz_state_init(const alz_plan* plan, double* state_dev, int64_t n_streams,
                       const double* xinit, const double* yinit, void* cuda_stream);

/* History depths (per section) of the xinit / yinit arrays above. */
int32_t alz_plan_history(const alz_plan* plan, int32_t* xd, int32_t* yd);

/*
 * Filter a block.  x_dev: [n_streams] rows of n_samples float32, row stride
 * x_stride elements.  y_dev: [n_streams * n_channels] rows (stream-major,
 * channel-minor) of n_samples float32, row stride y_stride elements.
 * state_dev: in/out, carries every recurrence across blocks, so that
 * apply(block0) ; apply(block1) == apply(block0 ++ block1) bit for bit.  (Exception: a call
 * whose sequential launch would leave more than half of the GPU idle -- n_channels * ceil(n_streams / 32)
 * warps < half the resident warp slots -- with n_samples >= 16384 (ALZ_TIME_PARALLEL_MIN) is
 * evaluated time-parallel: every stream is cut into chunks, all chunks run from a zero state, the
 * chunk transition matrices are scanned, all chunks run again from their true initial states.  The
 * result agrees with the sequential one to float64 rounding of the chunk states, ~1e-6 relative
 * at worst.  A plan created with ALZ_PLAN_SEQUENTIAL, or ALZ_NO_TIME_PARALLEL=1, never does this.)
 * Asynchronous on `cuda_stream`.
 */
int32_t alz_apply_f32(const alz_plan* plan, const float* x_dev, float* y_dev,
                      double* state_dev, int64_t n_streams, int64_t n_samples,
                      int64_t x_stride, int64_t y_stride, void* cuda_stream);

/*
 * Same as alz_apply_f32 with an explicit distance (in elements) between the output rows of
 * consecutive STREAMS: row (s, c) starts at y_dev + s * y_stream_stride + c * y_stride.  Lets a
 * plan that holds a SLICE of a bank's channels (channel-sharded multi-GPU, audiolazy_b200/parallel.py)
 * write its rows straight into the full y[S][C_total][T] tensor -- local, or a peer GPU's over
 * NVLink -- with y_dev offset to its first channel; y_stream_stride >= n_channels * y_stride.  It also
 * expresses the CHANNEL-MAJOR layout y[C][S][T]: y_stream_stride = T, y_stride = n_streams * T (then
 * y_stride >= n_streams * y_stream_stride): the 32 rows a warp stores are 64 KB apart instead of C * 64 KB.
 * The time-parallel evaluation of few long streams is not used on this entry.
 */
int32_t alz_apply_f32_ex(const alz_plan* plan, const float* x_dev, float* y_dev, double* state_dev,
                         int64_t n_streams, int64_t n_samples, int64_t x_stride, int64_t y_stride,
                         int64_t y_stream_stride, void* cuda_stream);

/*
 * Time-varying coefficients (reference lazy_filters.py:200-216: Stream-valued b_k / a_k are
 * advanced once per input sample).  For a single-channel GENERIC plan, alz_plan_taps() lists
 * the taps in the order of the coefficient table: delay[i], is_den[i] (1 for feedback taps).
 * alz_apply_tv_f32() filters a block with per-sample coefficients coef_dev[i * coef_stride + n]
 * (device, float64): b_k[n] / a_0[n] for numerator taps, -a_k[n] / a_0[n] for feedback taps.
 * All streams of the batch share the coefficient sequences.
 */
int32_t alz_plan_taps(const alz_plan* plan, int32_t* delay, int32_t* is_den, int32_t cap);
int32_t alz_apply_tv_f32(const alz_plan* plan, const float* x_dev, float* y_dev, double* state_dev,
                         int64_t n_streams, int64_t n_samples, int64_t x_stride, int64_t y_stride,
                         const double* coef_dev, int64_t coef_stride, void* cuda_stream);

/*
 * Same with HOST buffers: host->device copy of x, the kernel, device->host copy
 * of y, chunked over streams and pipelined on internal CUDA streams.  The host
 * buffers may be pageable or pinned (pinned is faster; alz_host_alloc below).  state_dev may
 * be NULL (zero initial state, discarded afterwards).  Synchronous: y_host is complete on
 * return.  ORDERING: the copies and kernels run on private non-blocking streams that are ordered
 * after the LEGACY DEFAULT stream at entry; a state_dev produced on any other stream must be
 * complete (synchronised) before the call.
 */
int32_t alz_apply_f32_host(const alz_plan* plan, const float* x_host, float* y_host,
                           double* state_dev, int64_t n_streams, int64_t n_samples,
                           int64_t x_stride, int64_t y_stride);

/*
 * The bank with a fused envelope consumer (reference lazy_analysis.py:440-520: envelope.abs / .squared / .rms are
 * lowpass(cutoff)(abs(sig)), lowpass(cutoff)(sig ** 2), (...) ** .5): every channel output y is rectified (mode 0: |y|)
 * or squared (mode 1; mode 2 = squared, square root on output), followed by the one-pole lowpass
 * e[n] = g r[n] + R e[n-1] in float64, and only every decim-th value is stored: env_dev[s][c][n / decim].  The bank's
 * 256 bytes of output per input sample never leave the SM; a host caller receives 256 / decim bytes per input sample.
 * Same values as alz_apply_f32 followed by that lowpass on the float32 y.  For gammatone-bank plans (4 sections per
 * channel); n_samples % decim == 0; x rows 16-byte aligned (else ALZ_ERR_UNSUPPORTED).  env_state_dev:
 * n_channels * n_streams doubles (in/out, index c * n_streams + s), state_dev as alz_apply_f32.  (Exception: a call
 * whose sequential launch would leave more than half of the GPU idle -- n_channels * ceil(n_streams / 32) warps < half
 * the resident warp slots -- with n_samples >= 16384 (ALZ_TIME_PARALLEL_MIN) is evaluated time-parallel: every stream is
 * cut into chunks, all chunks run from a zero state, the chunk transition matrices are scanned, all chunks run again from
 * their true bank states to give the lowpass's chunk transitions, those are scanned, and all chunks run a third time
 * from their true bank and lowpass states.  The result agrees with the sequential one to float64 rounding of the chunk
 * states, ~1e-6 relative at worst.  A plan created with ALZ_PLAN_SEQUENTIAL, or ALZ_NO_TIME_PARALLEL=1, never does this.)
 * The _host variant takes host buffers (zero initial state), copies inside, synchronous.
 */
int32_t alz_apply_envelope_f32(const alz_plan* plan, const float* x_dev, float* env_dev, double* state_dev,
                               double* env_state_dev, int64_t n_streams, int64_t n_samples, int64_t x_stride,
                               int64_t env_stride, int32_t decim, int32_t mode, double g, double R, void* cuda_stream);
int32_t alz_apply_envelope_f32_host(const alz_plan* plan, const float* x_host, float* env_host, int64_t n_streams,
                                    int64_t n_samples, int64_t x_stride, int64_t env_stride, int32_t decim, int32_t mode,
                                    double g, double R);

/*
 * The same for a block of an endless stream: any n_samples >= 0.  `phase` (0 <= phase < decim) is the number of samples
 * of the current decimation window consumed before this block; the block yields n_out = (phase + n_samples) / decim
 * values per row, the first of them at block sample decim - 1 - phase, and the next block's phase is
 * (phase + n_samples) % decim.  env_stride >= n_out.  So a stream cut into blocks of any lengths, with state_dev /
 * env_state_dev / the phase carried from call to call, gives the same values as one call over the whole stream (bit
 * for bit when no call is evaluated time-parallel, see above).  alz_apply_envelope_f32 is the phase = 0 case.
 * The _host variant takes host x / env and DEVICE state_dev / env_state_dev (either may be NULL: zero initial state,
 * discarded afterwards; ordering as alz_apply_f32_host), synchronous.
 */
int32_t alz_apply_envelope_f32_ex(const alz_plan* plan, const float* x_dev, float* env_dev, double* state_dev,
                                  double* env_state_dev, int64_t n_streams, int64_t n_samples, int64_t x_stride,
                                  int64_t env_stride, int32_t decim, int32_t phase, int32_t mode, double g, double R,
                                  void* cuda_stream);
int32_t alz_apply_envelope_f32_host_ex(const alz_plan* plan, const float* x_host, float* env_host, double* state_dev,
                                       double* env_state_dev, int64_t n_streams, int64_t n_samples, int64_t x_stride,
                                       int64_t env_stride, int32_t decim, int32_t phase, int32_t mode, double g, double R);

/*
 * Pinned host buffers for alz_apply_f32_host, placed on the NUMA node of CUDA device `device`
 * (< 0: the current device) so that several GPUs can run their PCIe copies at full rate at the same
 * time.  *numa_node (may be NULL) receives the node the pages were bound to, or -1 when the
 * topology is not visible.  Free with alz_host_free.
 */
int32_t alz_host_alloc(void** out, int64_t bytes, int32_t device, int32_t* numa_node);
int32_t alz_host_free(void* ptr);

/*
 * ParallelFilter.__call__ in ONE kernel (reference lazy_filters.py:1048-1054): out[s][t] =
 * ((y_0[s][t] + y_1[s][t]) + ...) over the plan's channels, summed left to right in float64 over the
 * float64 channel results, rounded to float32 once.  The channel outputs never reach memory: 8 bytes
 * of HBM traffic per input sample.  Needs a biquad plan created with ALZ_PLAN_PARALLEL and 16-byte
 * aligned x / out rows (else ALZ_ERR_UNSUPPORTED: use alz_apply_f32 + alz_sum_channels_f32).
 * x_dev [n_streams][n_samples], out_dev [n_streams][n_samples]; state as alz_apply_f32.
 */
int32_t alz_apply_sum_f32(const alz_plan* plan, const float* x_dev, float* out_dev, double* state_dev,
                          int64_t n_streams, int64_t n_samples, int64_t x_stride, int64_t out_stride,
                          void* cuda_stream);

/*
 * A CUDA stream whose kernels run on a partition of `sm_count` SMs only (green context; the granted count -- a
 * multiple of 8 on this architecture -- is returned in *sm_granted).  For the channel-sharded multi-GPU pipeline: the
 * bank kernel's one-warp CTAs otherwise occupy every SM for the whole kernel and an NCCL kernel issued on a side stream
 * (its CTAs need a nearly empty SM) waits for it; launched on a partition stream the bank kernel leaves the other SMs to
 * NCCL and the broadcast of the next input block really overlaps.  Pass the handle as `cuda_stream` to the apply entries.
 */
int32_t alz_stream_create_partition(int32_t device, int32_t sm_count, void** stream_out, int32_t* sm_granted);
int32_t alz_stream_destroy_partition(void* stream);

/*
 * ParallelFilter reduction: out[s][t] = ((y[s][0][t] + y[s][1][t]) + ...) over
 * the channel axis, left associated as reference lazy_filters.py:1053-1054.
 * Device buffers; asynchronous on `cuda_stream`.
 */
int32_t alz_sum_channels_f32(const float* y_dev, float* out_dev, int64_t n_streams,
                             int32_t n_channels, int64_t n_samples, int64_t y_stride,
                             int64_t out_stride, void* cuda_stream);

/*
 * Frequency response of every channel of the plan on a grid: out[c][i] =
 * prod_k B_ck(e^{-j w[i]}) / A_ck(e^{-j w[i]}) as interleaved (re, im) float64,
 * out_dev sized [n_channels][n][2]; w_dev in rad/sample.  A pole exactly on the
 * grid gives NaN (reference lazy_filters.py:267-301 evaluates numpoly/denpoly at
 * exp(-1j*freq); CascadeFilter multiplies the sections' responses, :1000-1003).
 * Device buffers; asynchronous on `cuda_stream`.
 */
int32_t alz_freq_response_f64(alz_plan* plan, const double* w_dev, double* out_dev, int64_t n,
                              void* cuda_stream);

/* Number of kernel launches issued by this library since load (bench bookkeeping). */
int64_t alz_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* ALZ_B200_H */
