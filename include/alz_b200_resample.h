/* alz_b200_resample.h -- plain-C ABI of libalz_b200_resample.so: Lagrange sample-rate conversion of many streams,
 * evaluated by sm_90a kernels.
 *
 * AudioLazy's resample(sig, old, new, order, zero) with a constant step = old / new, restated as a walk over one
 * pending position `idx` (float64) and a history of the last L = order + 1 samples (float64, `zero` before the
 * stream).  With threshold = .5 * L, a stream starts at idx = int(threshold) + rint(threshold) (rint: halves away
 * from zero) with every history sample `zero`; then, repeatedly:
 *
 *   while idx > threshold: consume the next sample into the history, idx -= 1    (exact: idx >= 1 there)
 *   emit y = psum(h[j] * w_j(idx) for j in 0 .. order)                          h[0] is the oldest sample
 *   idx += step                                                                  (float64, rounded)
 *
 *   w_j(idx) = ((idx - r_0) / (j - r_0)) * ((idx - r_1) / (j - r_1)) * ...      r_k in 0 .. order, r_k != j, left
 *                                                                                to right, each operation rounded
 *
 * psum is CPython 3.12's sum() of floats (a Neumaier compensated sum), each product h[j] * w_j rounded.  This is the
 * reference's float64 arithmetic without contraction, so the outputs are its values bit for bit.  The schedule (how
 * many outputs a block yields, at which input position and idx) depends on the step only, never on the samples: it
 * is walked on the host by alz_resample_schedule and shared by every stream of a batch that started together.  A
 * call stops when it needs a sample it does not have and carries idx to the next call, so a stream cut into blocks
 * of any lengths gives the outputs of one call.
 *
 * Device pointers are passed to alz_resample_state_init and alz_resample_apply; both are asynchronous on
 * `cuda_stream` (a cudaStream_t, NULL = legacy default stream) and run on the current device.
 */
#ifndef ALZ_B200_RESAMPLE_H
#define ALZ_B200_RESAMPLE_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_RESAMPLE_OK 0
#define ALZ_RESAMPLE_ERR_INVALID (-1)      /* bad argument */
#define ALZ_RESAMPLE_ERR_CUDA (-4)         /* a CUDA call failed; alz_resample_last_error() has the message */
#define ALZ_RESAMPLE_ERR_UNSUPPORTED (-6)  /* an order above 64, or a step that is not finite and positive or
                                            * too small to advance the position */
#define ALZ_RESAMPLE_ERR_CAPACITY (-7)     /* the block yields more outputs than the schedule arrays hold */

#define ALZ_RESAMPLE_MAX_ORDER 64

/* Message of the last failed call on this thread. */
const char* alz_resample_last_error(void);

/* Doubles of device state for n_streams streams of the given order: the last order + 1 samples of each stream. */
int64_t alz_resample_state_doubles(int32_t order, int64_t n_streams);

/* Sets the history of n_streams streams to `zero` (the start of a stream). */
int32_t alz_resample_state_init(double* state_dev, int64_t n_streams, int32_t order, double zero, void* cuda_stream);

/* The schedule of the next n_samples >= 0 samples, starting from the pending position `idx` (host memory, no device
 * needed).  Output i of the block uses block samples [pos[i] - order - 1, pos[i]) (negative positions: the
 * history) at position idx_out[i].  Returns the number of outputs n, and the idx to carry to the next block in
 * *idx_next.  ALZ_RESAMPLE_ERR_CAPACITY when n would exceed `capacity` (pos / idx_out are then partly written). */
int64_t alz_resample_schedule(int32_t order, double step, double idx, int64_t n_samples, int64_t capacity,
                              int64_t* pos, double* idx_out, double* idx_next);

/* Interpolates one block of n_streams streams: x_dev[s * x_stride + n] (float32, n < n_samples, any alignment) ->
 * out_dev[s * out_stride + i] (float32, the rounding of the float64 value, or float64 with out_f64), i < n_out, and
 * advances state_dev past the block.  pos_dev / idx_dev are the n_out schedule entries of alz_resample_schedule, in
 * device memory; weights_dev is device scratch of n_out * (order + 1) doubles, which the call fills with w_j(idx). */
int32_t alz_resample_apply(const float* x_dev, void* out_dev, int32_t out_f64, double* state_dev,
                           const int64_t* pos_dev, const double* idx_dev, double* weights_dev, int64_t n_out,
                           int64_t n_streams, int64_t n_samples, int64_t x_stride, int64_t out_stride, int32_t order,
                           void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_RESAMPLE_H */
