/* alz_b200_lpcscan.h -- plain-C ABI of libalz_b200_lpcscan.so: time-parallel LPC synthesis (the all-pole 1 / A(z) of
 * include/alz_b200_lpcfilt.h) for few long streams on sm_90a kernels
 *
 * The synthesis of a stream is a linear recurrence on its state, the last `order` outputs.  A call cuts each stream's
 * n_samples into n_chunks chunks (chunk p holds samples [p q + min(p, r), (p + 1) q + min(p + 1, r)) with q, r the
 * quotient and remainder of n_samples / n_chunks) and evaluates it in three passes:
 *
 *   1. summaries: every chunk is walked from a zero state with its input, giving its final state F_p, and `order`
 *      times from a unit state with zero input, giving the columns of M_p, so that the chunk maps a start state s to
 *      F_p + M_p s (exactly, in real arithmetic);
 *   2. scan: s_{p+1} = F_p + M_p s_p from the call's state s_0, one warp per stream;
 *   3. rerun: every chunk is walked from s_p and stores its outputs; the last chunk writes the state.
 *
 * Every walk is alz_lpcfilt_apply's arithmetic (ascending taps, every tap a term, __dmul_rn / __dadd_rn); the scan
 * contracts freely.  So chunk 0 gives the sequential bits and the other chunks differ from them by the float64
 * rounding drift of the scan.  A stream whose summaries or scanned states hold a NaN or an infinity (NaN or infinite
 * samples or rows, unstable rows that overflow) is walked sequentially instead, in the rerun launch, from the call's
 * state: its outputs and final state are alz_lpcfilt_apply's, bit for bit.
 *
 * Rows, state (the last `order` outputs as float64, oldest first) and the sample count are alz_lpcfilt_apply's, so
 * calls of the two libraries can be mixed on one state.  All pointers are device pointers; a call is asynchronous on
 * `cuda_stream` (a cudaStream_t, NULL = legacy default stream) and must be made with the device of the buffers
 * current.  The library keeps no state between calls.
 */
#ifndef ALZ_B200_LPCSCAN_H
#define ALZ_B200_LPCSCAN_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_LPCSCAN_OK 0
#define ALZ_LPCSCAN_ERR_INVALID (-1)      /* bad argument; alz_lpcscan_last_error() has the message */
#define ALZ_LPCSCAN_ERR_UNSUPPORTED (-2)  /* a shape beyond one launch */
#define ALZ_LPCSCAN_ERR_CUDA (-4)         /* a CUDA call failed */

#define ALZ_LPCSCAN_MAX_ORDER 64

#define ALZ_LPCSCAN_FLOAT32 0             /* sample dtypes, as ALZ_LPCFILT_FLOAT32 / _FLOAT64 */
#define ALZ_LPCSCAN_FLOAT64 1

/* Message of the last failed call on this thread. */
const char* alz_lpcscan_last_error(void);

/* The chunk count the cost model picks for a synthesis of n_streams x n_samples at `order` with rows switching every
 * `hop` samples: 1 (evaluate sequentially, with alz_lpcfilt_apply) unless the three passes are estimated to take at
 * most half the sequential time.  Never more than n_samples / max(order, 1). */
int64_t alz_lpcscan_chunks(int64_t n_streams, int64_t n_samples, int32_t order, int64_t hop);

/* Bytes of the scratch alz_lpcscan_apply needs for n_streams streams cut into n_chunks chunks at `order`: the
 * summaries, the scanned states and one flag per stream. */
int64_t alz_lpcscan_scratch_bytes(int64_t n_streams, int64_t n_chunks, int32_t order);

/* The synthesis of alz_lpcfilt_apply (same arguments, kind ALZ_LPCFILT_SYNTHESIS) in n_chunks chunks per stream,
 * 1 <= n_chunks <= max(1, n_samples / max(order, 1)), so that every chunk but a lone one holds at least `order`
 * samples.  scratch_dev (8-byte aligned) holds scratch_bytes >= alz_lpcscan_scratch_bytes(n_streams, n_chunks,
 * order) bytes; the caller must not touch it until the call is done on cuda_stream. */
int32_t alz_lpcscan_apply(const void* x_dev, int32_t x_dtype, int64_t x_stride, void* out_dev, int32_t out_dtype,
                          int64_t out_stride, const double* coef_dev, int64_t coef_row_stride,
                          int64_t coef_stream_stride, int64_t n_rows, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int64_t consumed, int32_t order, int64_t hop, int64_t n_chunks,
                          void* scratch_dev, int64_t scratch_bytes, void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_LPCSCAN_H */
