/* alz_b200_lpc.h -- plain-C ABI of libalz_b200_lpc.so: frame-wise linear prediction of many streams, evaluated by
 * sm_90a kernels: the autocorrelation method through Levinson-Durbin (AudioLazy's lpc.kautocor) and the covariance
 * method through a Gram-Schmidt lattice (lpc.kcovar).
 *
 * For one stream x (float32 samples), frame k covers stream samples [k hop, k hop + size) and is emitted once its last
 * sample has been consumed (samples between frames are skipped when hop > size).  At the end of a stream of N samples
 * (`final`) the first incomplete frame k is emitted too if N - k hop > max(size - hop, 0), its missing samples 0.0
 * (AudioLazy's padded last block of Stream.blocks(size, hop)).  Frame values are float64:
 *
 *   b[n] = (double)x[k hop + n]              without a window
 *   b[n] = (double)x[k hop + n] * w[n]       with a window w of `size` float64 values (one rounding)
 *
 * Every sum below is psum: a sequential sum in the order given, f = 0.0 + first term, then for each later term t'
 * = f + x, c += (|f| >= |x| ? (f - t') + x : (x - t') + f), f = t'; at the end f += c when c is finite and nonzero.
 * That is CPython >= 3.12's builtin sum() of floats, so the results equal AudioLazy's lpc.kautocor(block, order) and
 * acorr(block, order) bit for bit (NaN results are any NaN):
 *
 *   acorr[tau] = psum(b[n] * b[n + tau] for n in 0 .. size - tau - 1),  tau = 0 .. order  (0.0 when tau >= size)
 *   inner(a, b) = psum(acorr[|i - j|] * a[i] * b[j] for i over a, j over b)          (products left to right)
 *   A = [1];  for m = 1 .. order:
 *     B = [0] + reversed(A)  (length m + 1);  Z = [0] * m + [1]
 *     den = inner(B, B);  den == 0 -> the frame fails (AudioLazy's ParCorError)
 *     c = inner(A', Z) / den
 *     A[k] (k = 0 .. m, A[m] = 0 before) -= c * B[k], skipped where c == 0, B[k] == 0 or c * B[k] == 0; a result
 *     equal to zero is stored as +0.0
 *   error = inner(A', A')
 *
 * where A' is A up to its last coefficient that is not zero (AudioLazy's ZFilter drops zero coefficients; a[0] = 1).
 * coef holds A (order + 1 values, coef[0] = 1); a failed frame has failed = 1 and NaN coef and error.
 *
 * The covariance method (alz_lpc_covar_apply_f32, 1 <= order < size) equals AudioLazy's lpc.kcovar(block, order) and
 * lag_matrix(block, order) bit for bit.  A polynomial is a dense list with +0.0 for a missing power, and its numlist
 * stops at its highest power that is not zero:
 *
 *   phi[j][i] = psum(b[n - i] * b[n - j] for n in order .. size - 1)      (symmetric bit for bit)
 *   inner(x, y) = psum(phi[i][j] * x[i] * y[j] for i over x, j over y)     (numlists, products left to right)
 *   A = [1];  B[0] = z^-1 = [0, 1];  beta[0] = inner(B[0], B[0])
 *   for m = 1 .. order:
 *     beta[m - 1] == 0 -> the frame fails with 1 (AudioLazy's ZeroDivisionError("Can't find next coefficient"))
 *     k = -inner(A, z^-m) / beta[m - 1];  k >= 1 or k <= -1 -> the frame fails with 2 ("Unstable filter");
 *     a NaN k goes on
 *     A[p] += k * B[m - 1][p] for p = 1 .. m, skipped where B[m - 1][p] == 0 or k * B[m - 1][p] == 0
 *     m == order: error = inner(A, A), done
 *     gamma[q] = inner(z^-(m+1), B[q]) / beta[q] for q = 0 .. m - 1
 *     S[p] = 0, then S[p] += gamma[q] * B[q][p] for q = p - 1 .. m - 1 in order, skipped as above (powers 1 .. m)
 *     B[m] = [0, -S[1], .., -S[m], 1];  beta[m] = inner(B[m], B[m])
 *
 * where every sum or update result equal to zero is stored as +0.0 (AudioLazy's polynomials drop it).  In inner(A,
 * z^-m) and inner(z^-(m+1), B[q]) the products of a 0.0 coefficient of the unit polynomial are +-0, which leaves psum
 * as it is, unless the partial product they multiply is not finite: such a sum is NaN.  coef holds A (order + 1
 * values, coef[0] = 1); a failed frame has NaN coef and error.
 *
 * All pointers are device pointers; calls are asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default
 * stream) and must be made with the device of the buffers current.  The library keeps no state between calls: the
 * stream state and the scratch both come from the caller.
 */
#ifndef ALZ_B200_LPC_H
#define ALZ_B200_LPC_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_LPC_OK 0
#define ALZ_LPC_ERR_INVALID (-1)      /* bad argument; alz_lpc_last_error() has the message */
#define ALZ_LPC_ERR_CUDA (-4)         /* a CUDA call failed */
#define ALZ_LPC_ERR_UNSUPPORTED (-6)  /* a shape too large for one launch */

#define ALZ_LPC_MAX_ORDER 64
#define ALZ_LPC_MAX_SIZE 8192

/* Message of the last failed call on this thread. */
const char* alz_lpc_last_error(void);

/* Frames one call emits: with C samples consumed before it and C' = C + n_samples, ka = max(0, floor((C - size) /
 * hop) + 1), kc = floor((C' - size) / hop): max(0, kc - ka + 1) frames ka .. kc, plus one when final and
 * C' - max(kc + 1, 0) hop > max(size - hop, 0).  Negative on a bad argument. */
int64_t alz_lpc_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final);

/* Bytes of device state for n_streams streams of one size: per stream the samples consumed (int64) and the last
 * `size` samples (float32), which hold every sample an open frame still needs.  8-byte aligned. */
int64_t alz_lpc_state_bytes(int64_t n_streams, int32_t size);

/* Sets the state of n_streams streams to the start of a stream (no sample consumed). */
int32_t alz_lpc_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream);

/* Bytes of scratch alz_lpc_apply_f32 needs when acorr_dev is NULL and coef_dev, error_dev or failed_dev is not:
 * n_streams * n_frames * (order + 1) float64 values.  Otherwise no scratch is needed. */
int64_t alz_lpc_scratch_bytes(int64_t n_streams, int64_t n_frames, int32_t order);

/* Bytes of scratch alz_lpc_covar_apply_f32 needs when coef_dev, error_dev or failed_dev is not NULL: one triangle
 * of each lag matrix, n_streams * n_frames * (order + 1) * (order + 2) / 2 float64 values. */
int64_t alz_lpc_covar_scratch_bytes(int64_t n_streams, int64_t n_frames, int32_t order);

/* The next n_samples >= 0 samples of n_streams streams, x_dev[s * x_stride + n] (float32, 4-byte aligned, any 16-byte
 * alignment), continuing state_dev (made by alz_lpc_state_init with the same size).  window_dev: `size` float64
 * values, or NULL for none.  n_frames is alz_lpc_frames(C, n_samples, size, hop, final) for the C samples the state
 * has consumed; the frames are stored in order at frame index i = 0 .. n_frames - 1, each output NULL when not wanted:
 *
 *   acorr_dev   float64 [n_streams][n_frames][order + 1]
 *   coef_dev    float64 [n_streams][n_frames][order + 1]
 *   error_dev   float64 [n_streams][n_frames]
 *   failed_dev  uint8   [n_streams][n_frames]
 *
 * When only acorr_dev is given, the Levinson-Durbin stage does not run.  Limits: 0 <= order <= ALZ_LPC_MAX_ORDER,
 * 1 <= size <= ALZ_LPC_MAX_SIZE, hop >= 1.  A stream cut into blocks of any lengths gives the same bits as one call.
 * `final` != 0 ends the streams (the state must not be continued).  scratch_dev holds scratch_bytes >=
 * alz_lpc_scratch_bytes(...) bytes of device memory no other work in flight uses. */
int32_t alz_lpc_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, double* acorr_dev,
                          double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames, void* state_dev,
                          int64_t n_streams, int64_t n_samples, int32_t order, int32_t size, int32_t hop, int32_t final,
                          void* scratch_dev, int64_t scratch_bytes, void* cuda_stream);

/* As alz_lpc_apply_f32, for the covariance method: the same frames, state and arguments, with the outputs
 *
 *   lagm_dev    float64 [n_streams][n_frames][order + 1][order + 1]   the full (symmetric) lag matrix phi
 *   coef_dev    float64 [n_streams][n_frames][order + 1]
 *   error_dev   float64 [n_streams][n_frames]
 *   failed_dev  uint8   [n_streams][n_frames]   0, or 1 / 2 as above
 *
 * each NULL when not wanted.  Limits: 0 <= order < size, and order >= 1 when coef_dev, error_dev or failed_dev is
 * given (AudioLazy raises IndexError at order 0).  scratch_dev holds scratch_bytes >= alz_lpc_covar_scratch_bytes(...)
 * bytes of device memory no other work in flight uses. */
int32_t alz_lpc_covar_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, double* lagm_dev,
                                double* coef_dev, double* error_dev, uint8_t* failed_dev, int64_t n_frames,
                                void* state_dev, int64_t n_streams, int64_t n_samples, int32_t order, int32_t size,
                                int32_t hop, int32_t final, void* scratch_dev, int64_t scratch_bytes,
                                void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_LPC_H */
