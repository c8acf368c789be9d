/* alz_b200_amdf.h -- plain-C ABI of libalz_b200_amdf.so: the average magnitude difference function (AMDF) of many
 * streams at many lags, evaluated by one sm_90a kernel.
 *
 * For one lag with taps (c_j, k_j) (the terms of (1 - z^-lag).linearize(): at most 3, ascending delay, no zero
 * coefficient) and one stream x (float32 samples, x[j] = zero for j < 0):
 *
 *   d[n]    = c_0 x[n - k_0] + c_1 x[n - k_1] + ...   float64, each product rounded, summed left to right
 *                                                     (no taps: d[n] = zero)
 *   new[n]  = |d[n]| * (1. / size)
 *   old[n]  = new[n - size], or zero * (1. / size) for n < size
 *   mean[n] = (mean[n - 1] - old[n]) + new[n]         mean[-1] = zero
 *
 * which is AudioLazy's amdf(lag, size)(x, zero=zero): maverage(size) over abs((1 - z^-lag).linearize()(x)).  The
 * arithmetic is float64 without contraction, so a sequential evaluation reproduces that float64 sequence bit for bit;
 * it is stored as float32.  All lags of a plan share one `size`.
 *
 * All pointers passed to alz_amdf_apply_f32 are device pointers; the call is asynchronous on `cuda_stream`
 * (a cudaStream_t, NULL = legacy default stream) and must be made with the plan's device current.
 */
#ifndef ALZ_B200_AMDF_H
#define ALZ_B200_AMDF_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_AMDF_OK 0
#define ALZ_AMDF_ERR_INVALID (-1)      /* bad argument */
#define ALZ_AMDF_ERR_NONCAUSAL (-2)    /* a tap with a negative delay */
#define ALZ_AMDF_ERR_CUDA (-4)         /* a CUDA call failed; alz_amdf_last_error() has the message */
#define ALZ_AMDF_ERR_NOMEM (-5)
#define ALZ_AMDF_ERR_UNSUPPORTED (-6)  /* a tap delay longer than the kernel's shared-memory window allows */

/* Plan flags. */
#define ALZ_AMDF_PLAN_SEQUENTIAL 8     /* never evaluate time-parallel (as ALZ_PLAN_SEQUENTIAL of alz_b200.h) */

/* Message of the last failed call on this thread. */
const char* alz_amdf_last_error(void);

/* Plan for n_lags lags on the current device.  Lag l has n_taps[l] (0..3) taps: delays[3 l + j] (>= 0) and
 * coefs[3 l + j], j < n_taps[l], in the order they are summed.  size >= 1. */
int32_t alz_amdf_plan_create(const int32_t* n_taps, const int32_t* delays, const double* coefs, int32_t n_lags,
                             int32_t size, int32_t flags, void** plan_out);
void alz_amdf_plan_destroy(void* plan);

/* Doubles of device state for n_streams streams: per stream the samples consumed, `zero`, the last size + K input
 * samples (K: the longest tap delay) and the running mean of every lag. */
int64_t alz_amdf_state_doubles(const void* plan, int64_t n_streams);

/* Sets the state of n_streams streams to the start of a stream with pre-history `zero`. */
int32_t alz_amdf_state_init(const void* plan, double* state_dev, int64_t n_streams, double zero, void* cuda_stream);

/* Chunks per stream alz_amdf_apply_f32 cuts a block of n_streams x n_samples into (1: sequential evaluation). */
int64_t alz_amdf_plan_chunks(const void* plan, int64_t n_streams, int64_t n_samples);

/* The next n_samples >= 0 samples of n_streams streams: x_dev[s * x_stride + n] (float32, any alignment) ->
 * out_dev[(s * n_lags + l) * out_stride + m] (float32), continuing state_dev.  Every decim-th mean is stored: `phase`
 * (0 <= phase < decim) samples of the current decimation window were consumed before this block, which yields
 * n_out = (phase + n_samples) / decim values per row, the first at block sample decim - 1 - phase; the next block's
 * phase is (phase + n_samples) % decim and out_stride >= n_out.  A stream cut into blocks of any lengths gives the
 * same values as one call over the whole stream.
 *
 * Few long streams (the sequential launch would fill less than half of the device's resident warp slots, and
 * n_samples >= 16384) are evaluated time-parallel unless the plan has ALZ_AMDF_PLAN_SEQUENTIAL or the environment
 * sets ALZ_NO_TIME_PARALLEL=1: each stream is cut into chunks that run as streams of their own, and the running mean
 * at the start of a chunk is the float64 sum of the `size` terms before it.  It differs from the sequential
 * recursion by that recursion's own rounding drift (~1e-13 relative), so outputs may differ in the last float32 bit. */
int32_t alz_amdf_apply_f32(const void* plan, const float* x_dev, float* out_dev, double* state_dev, int64_t n_streams,
                           int64_t n_samples, int64_t x_stride, int64_t out_stride, int32_t decim, int32_t phase,
                           void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_AMDF_H */
