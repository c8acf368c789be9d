/* alz_b200_unwrap.h -- plain-C ABI of libalz_b200_unwrap.so: phase unwrapping and clipping of many streams, each
 * evaluated by one sm_90a kernel.
 *
 * Unwrap.  For one stream d[0..N) (float32 or float64 samples, widened to float64), a float64 max_delta M and step P:
 *
 *   out[0] = d[0]                       delta = d[0] - d[0]      (+0.0, or NaN when d[0] is +-inf or NaN)
 *   for n >= 1:  diff   = d[n] - d[n-1]
 *                if |diff| > M:  delta = delta + ((-diff) + pick(rem(diff, P), rem(diff, -P)))
 *                out[n] = d[n] + delta
 *
 * with every operation a float64 operation rounded to nearest (no contraction), delta a sequential sum in sample order,
 * and, restating CPython 3.12:
 *
 *   rem(v, w)    float `%` (float_rem): w == 0 is an error (ZeroDivisionError "float modulo").  Otherwise
 *                mod = fmod(v, w), which is exact; if mod != 0 (NaN counts as nonzero) and (w < 0) != (mod < 0),
 *                mod = mod + w (a rounded add); a zero mod becomes copysign(0.0, w).
 *   pick(a, b)   min(a, b, key=abs): b when |b| < |a|, else a (a tie or a NaN keeps a).
 *
 * which is AudioLazy's unwrap(d, max_delta=M, step=P) bit for bit.  Consequences worth naming: a NaN diff is never a
 * jump (a NaN sample only spoils itself and its successor's diff); an infinite diff makes delta NaN from then on;
 * d[n] + delta turns -0.0 into +0.0 for n >= 1 but out[0] keeps it; M < 0 makes every non-NaN diff a jump, M = NaN
 * none.  With P == 0 (or -0.0) the first jump raises in the reference, after the values before it were yielded: here
 * its term is NaN (so delta and every later output are NaN) and the state records the jump's sample index.
 *
 * Clip.  out = x, clipped as AudioLazy's clip(x, low, high) does, in float64 (x widened, limits as given):
 *
 *   both limits      high if x > high else (low if x < low else x)
 *   low only         x if x > low else low             (a NaN sample becomes low)
 *   high only        x if x < high else high           (a NaN sample becomes high)
 *   none             x
 *
 * A clipped value is the limit itself, so signed zeros and NaN limits follow from the comparisons.  high < low is an
 * error.
 *
 * Samples are float32 or float64 (ALZ_UNWRAP_FLOAT32 / ALZ_UNWRAP_FLOAT64), the output of either kind: float64 holds
 * the values above, float32 their rounding.  All pointers are device pointers aligned to their element size; calls are
 * asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default stream) and must be made with the device of the
 * buffers current.  The library keeps no state between calls: the stream state and the scratch come from the caller.
 */
#ifndef ALZ_B200_UNWRAP_H
#define ALZ_B200_UNWRAP_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_UNWRAP_OK 0
#define ALZ_UNWRAP_ERR_INVALID (-1)      /* bad argument */
#define ALZ_UNWRAP_ERR_CUDA (-4)         /* a CUDA call failed; alz_unwrap_last_error() has the message */
#define ALZ_UNWRAP_ERR_UNSUPPORTED (-6)  /* a shape too large for one launch */

#define ALZ_UNWRAP_FLOAT32 0
#define ALZ_UNWRAP_FLOAT64 1

/* Message of the last failed call on this thread. */
const char* alz_unwrap_last_error(void);

/* Bytes of device state for n_streams streams, 32 per stream: the samples consumed (int64), the previous sample
 * (float64), delta (float64) and the bitwise complement of the sample index of the first jump taken with step == 0
 * (int64; 0, the complement of -1: none).  A state of all zero bytes is a new one. */
int64_t alz_unwrap_state_bytes(int64_t n_streams);

/* Sets the state of n_streams streams to the start of a stream: nothing consumed, delta +0.0, no failure.  The buffer
 * is 8-byte aligned. */
int32_t alz_unwrap_state_init(void* state_dev, int64_t n_streams, void* cuda_stream);

/* Bytes of scratch alz_unwrap_apply needs for a block of n_streams x n_samples (8-byte aligned). */
int64_t alz_unwrap_scratch_bytes(int64_t n_streams, int64_t n_samples);

/* The next n_samples >= 0 samples of n_streams streams, x_dev[s * x_stride + n], unwrapped into
 * out_dev[s * out_stride + n], continuing state_dev (made by alz_unwrap_state_init).  A stream cut into blocks of any
 * lengths (0 included) gives the bits of one call.  scratch_dev holds scratch_bytes >= alz_unwrap_scratch_bytes(...)
 * bytes of device memory that no other work in flight uses; it is cleared on cuda_stream before the kernel reads it. */
int32_t alz_unwrap_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                         int64_t out_stride, void* state_dev, int64_t n_streams, int64_t n_samples, double max_delta,
                         double step, void* scratch_dev, int64_t scratch_bytes, void* cuda_stream);

/* out_dev[s * out_stride + n] = clip(x_dev[s * x_stride + n]) for n_streams x n_samples samples; has_low / has_high
 * = 0 stand for a limit of None (its value is then ignored). */
int32_t alz_clip_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                       int64_t out_stride, int64_t n_streams, int64_t n_samples, double low, int32_t has_low,
                       double high, int32_t has_high, void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_UNWRAP_H */
