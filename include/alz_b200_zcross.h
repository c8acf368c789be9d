/* alz_b200_zcross.h -- plain-C ABI of libalz_b200_zcross.so: zero crossings of many streams, with per-block counts,
 * evaluated by one sm_90a kernel.
 *
 * For one stream x (float32 samples) and a float64 hysteresis h, with the carried sign s[-1] in {-1, 0, +1}:
 *
 *   decisive(x) = x > h or x < -h                      (compared in float64: x widened, h as given)
 *   sgn(x)      = -1 if x < 0 else 1
 *   out[n]      = 1 if s[n-1] != 0 and x[n] * s[n-1] < -h else 0
 *   s[n]        = sgn(x[n]) if decisive(x[n]) else s[n-1]
 *
 * which is AudioLazy's zcross(x, hysteresis=h, first_sign) for every h (negative, +-inf and NaN included), with
 * s[-1] = 0 when first_sign == 0 (the first decisive sample sets the sign and is not a crossing), else its sign
 * (NaN: +1).  s[n] is the sign of the last decisive sample at or before n, so any tiling of time gives the same bits.
 *
 * Block counts follow zcross(...).blocks(size, hop) and sum(block): block k covers stream samples
 * [k hop, k hop + size) (samples between blocks are skipped when hop > size) and is emitted once its last sample has
 * been consumed.  At the end of a stream of N samples the first incomplete block k is emitted too, counting
 * [k hop, N), if N - k hop > max(size - hop, 0) (AudioLazy's padded last block).
 *
 * All pointers are device pointers; calls are asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default
 * stream) and must be made with the device of the buffers current.  The library keeps no state between calls: the
 * stream state and the scratch both come from the caller.
 */
#ifndef ALZ_B200_ZCROSS_H
#define ALZ_B200_ZCROSS_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_ZCROSS_OK 0
#define ALZ_ZCROSS_ERR_INVALID (-1)      /* bad argument */
#define ALZ_ZCROSS_ERR_CUDA (-4)         /* a CUDA call failed; alz_zcross_last_error() has the message */
#define ALZ_ZCROSS_ERR_UNSUPPORTED (-6)  /* a shape too large for one launch */

/* Message of the last failed call on this thread. */
const char* alz_zcross_last_error(void);

/* Bytes of device state for n_streams streams: per stream the samples consumed (int64), the carried sign (int32) and,
 * when size >= 1, the partial counts of the at most ceil(size / hop) open blocks (int32).  size = 0: no counts. */
int64_t alz_zcross_state_bytes(int64_t n_streams, int32_t size, int32_t hop);

/* Sets the state of n_streams streams to the start of a stream: no sample consumed, carried sign 0 if
 * first_sign == 0, else -1 if first_sign < 0, else +1 (NaN: +1), no open block.  The buffer is 8-byte aligned. */
int32_t alz_zcross_state_init(void* state_dev, int64_t n_streams, double first_sign, int32_t size, int32_t hop,
                              void* cuda_stream);

/* Bytes of scratch alz_zcross_apply_f32 needs for a block of n_streams x n_samples (4-byte aligned). */
int64_t alz_zcross_scratch_bytes(int64_t n_streams, int64_t n_samples, int32_t size, int32_t hop);

/* The next n_samples >= 0 samples of n_streams streams, x_dev[s * x_stride + n] (float32, any 4-byte alignment),
 * continuing state_dev (made by alz_zcross_state_init with the same size and hop):
 *
 *   flags_dev  (NULL: not stored)  uint8 out[n] of every sample at flags_dev[s * flags_stride + n];
 *   counts_dev (NULL: not stored)  int32 counts[s * counts_stride + i] of the blocks completed by this call, in order
 *                                  (the first is block ka, the first block that ends after the samples consumed
 *                                  before it), then, if `final`, the padded last block when it is emitted.
 *                                  With C the samples consumed before the call and C' = C + n_samples:
 *                                  ka = max(0, floor((C - size) / hop) + 1), kc = floor((C' - size) / hop), and the
 *                                  call stores max(0, kc - ka + 1) counts, plus one when final and
 *                                  C' - max(kc + 1, 0) hop > max(size - hop, 0).  Needs size >= 1.
 *
 * A stream cut into blocks of any lengths gives the same flags and counts as one call.  `final` != 0 ends the
 * streams (the state must not be continued).  scratch_dev holds scratch_bytes >= alz_zcross_scratch_bytes(...) bytes
 * of device memory that no other work in flight uses; it is cleared on cuda_stream before the kernel reads it. */
int32_t alz_zcross_apply_f32(const float* x_dev, int64_t x_stride, uint8_t* flags_dev, int64_t flags_stride,
                             int32_t* counts_dev, int64_t counts_stride, void* state_dev, int64_t n_streams,
                             int64_t n_samples, int32_t size, int32_t hop, double hysteresis, int32_t final,
                             void* scratch_dev, int64_t scratch_bytes, void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_ZCROSS_H */
