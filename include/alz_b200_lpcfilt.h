/* alz_b200_lpcfilt.h -- plain-C ABI of libalz_b200_lpcfilt.so: frame-wise LPC analysis and synthesis filtering of many
 * streams on sm_90a kernels, bit for bit as AudioLazy evaluates the time-varying ZFilters
 *
 *   analysis:   1 + sum(held(k) * z ** -k for k in 1 .. order)
 *   synthesis:  1 / (1 + sum(held(k) * z ** -k for k in 1 .. order))
 *
 * where held(k) is the Stream of each row's c_k repeated `hop` times, with the filters' default memory (zeros).
 * AudioLazy writes the generator
 *
 *   analysis:   y[n] = x[n] + c_1 * x[n - 1] + c_2 * x[n - 2] + ... + c_order * x[n - order]
 *   synthesis:  y[n] = x[n] + (-c_1) * y[n - 1] + (-c_2) * y[n - 2] + ... + (-c_order) * y[n - order]
 *
 * a left-to-right float64 sum of single-rounded products in ascending delay, nothing contracted, with c the row of
 * sample n.  Every tap is a term on every sample, even where its coefficient is 0.0 (0 * inf is NaN).  Samples before
 * a stream's first are 0.0.
 *
 * Rows: stream s's row r covers its samples [r * hop, (r + 1) * hop), counted across calls, and is
 * coef_dev[s * coef_stream_stride + r' * coef_row_stride + k] (float64) with r' = r - floor(consumed / hop) the row's
 * index in the call; column 0 is not read (the rows are monic).  A call on n_samples reads
 * alz_lpcfilt_rows(consumed, n_samples, hop) rows.
 *
 * State, per stream: the last `order` inputs (analysis) or outputs (synthesis) as float64, oldest first.  A new state
 * is zero: AudioLazy's default memory and zero.  The caller counts the samples a state has consumed and passes the
 * count to every call.
 *
 * All pointers are device pointers; a call is asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default
 * stream) and must be made with the device of the buffers current.  The library keeps no state between calls.
 */
#ifndef ALZ_B200_LPCFILT_H
#define ALZ_B200_LPCFILT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_LPCFILT_OK 0
#define ALZ_LPCFILT_ERR_INVALID (-1)      /* bad argument; alz_lpcfilt_last_error() has the message */
#define ALZ_LPCFILT_ERR_UNSUPPORTED (-2)  /* a shape beyond one launch */
#define ALZ_LPCFILT_ERR_CUDA (-4)         /* a CUDA call failed */

#define ALZ_LPCFILT_MAX_ORDER 64

#define ALZ_LPCFILT_ANALYSIS 0            /* kind: the FIR residual filter A(z) */
#define ALZ_LPCFILT_SYNTHESIS 1           /* kind: the all-pole filter 1 / A(z) */

#define ALZ_LPCFILT_FLOAT32 0             /* sample dtypes */
#define ALZ_LPCFILT_FLOAT64 1

/* Message of the last failed call on this thread. */
const char* alz_lpcfilt_last_error(void);

/* Bytes of the state of n_streams streams at `order` (0 .. ALZ_LPCFILT_MAX_ORDER): n_streams * 8 * order. */
int64_t alz_lpcfilt_state_bytes(int64_t n_streams, int32_t order);

/* Zeroes a state (8-byte aligned). */
int32_t alz_lpcfilt_state_init(void* state_dev, int64_t n_streams, int32_t order, void* cuda_stream);

/* Rows a call on n_samples reads after `consumed` samples: floor((consumed + n_samples - 1) / hop) -
 * floor(consumed / hop) + 1, and 0 for an empty call. */
int64_t alz_lpcfilt_rows(int64_t consumed, int64_t n_samples, int64_t hop);

/* Filters x[s * x_stride + n] (x_dtype, n < n_samples) of streams that have consumed `consumed` samples into
 * out[s * out_stride + n] (out_dtype: the float64 value or its float32 rounding) and advances the state.  n_rows is
 * the rows the coefficient table holds per stream, at least alz_lpcfilt_rows(consumed, n_samples, hop);
 * coef_row_stride >= order + 1 when n_rows > 1, coef_stream_stride >= 0 (0 shares one table).  The strides count
 * elements.  kind is ALZ_LPCFILT_ANALYSIS or ALZ_LPCFILT_SYNTHESIS. */
int32_t alz_lpcfilt_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                          int64_t out_stride, const double* coef_dev, int64_t coef_row_stride,
                          int64_t coef_stream_stride, int64_t n_rows, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int64_t consumed, int32_t order, int64_t hop, int32_t kind,
                          void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_LPCFILT_H */
