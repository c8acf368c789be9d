/* alz_b200_dft.h -- plain-C ABI of libalz_b200_dft.so: the discrete Fourier transform of every frame of many streams
 * at any list of frequencies, evaluated by an sm_90a kernel, equal to AudioLazy's dft(blk, freqs, normalize) bit for
 * bit (a NaN part is any NaN).
 *
 * For one stream x (float32 samples), frame k covers stream samples [k hop, k hop + size) and is emitted once its last
 * sample has been consumed (samples between frames are skipped when hop > size).  At the end of a stream of N samples
 * (`final`) the first incomplete frame k is emitted too if N - k hop > max(size - hop, 0), its missing samples 0.0
 * (AudioLazy's padded last block of Stream.blocks(size, hop)).  Frame values are float64:
 *
 *   b[n] = (double)x[k hop + n]              without a window
 *   b[n] = (double)x[k hop + n] * w[n]       with a window w of `size` float64 values (one rounding)
 *
 * AudioLazy computes sum(xn * cexp(-1j * n * f) for n, xn in enumerate(blk)) for each f, then v / len(blk) when
 * normalizing.  Under CPython 3.12 that is, per frequency column j with twiddles W[n][j] = (wr, wi):
 *
 *   re = +0.0, im = +0.0;  for n = 0 .. size - 1 in order:  re = re + b[n] * wr;  im = im + b[n] * wi
 *   normalize:  re' = (re + im * 0.0) / size,  im' = (im - re * 0.0) / size        (CPython's _Py_c_quot)
 *
 * every product and sum rounded on its own (no fused multiply-add).  The reference's term complex(b, 0.0) * W has the
 * parts b wr - 0.0 wi and b wi + 0.0 wr; for a finite twiddle the extra products are +-0, which can only change the
 * sign of a zero term, and a sum that starts at +0.0 never becomes -0.0 under round-to-nearest, so the bits are the
 * same.  A twiddle with a NaN part (a frequency that is +-inf or NaN) gives NaN parts either way.
 *
 * The twiddles are cmath.exp(-1j * n * f), which the device cannot reproduce (its cos / sin are not the host's): the
 * caller fills the table on the host with alz_dft_twiddles and uploads it.  It is n-major, [size][n_freqs] pairs of
 * float64 (re, im).
 *
 * All device pointers; calls are asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default stream) and must
 * be made with the device of the buffers current.  The library keeps no state between calls.
 */
#ifndef ALZ_B200_DFT_H
#define ALZ_B200_DFT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_DFT_OK 0
#define ALZ_DFT_ERR_INVALID (-1)      /* bad argument; alz_dft_last_error() has the message */
#define ALZ_DFT_ERR_CUDA (-4)         /* a CUDA call failed */
#define ALZ_DFT_ERR_UNSUPPORTED (-6)  /* a shape too large for one launch */

#define ALZ_DFT_MAX_SIZE 8192
#define ALZ_DFT_MAX_FREQS 4096

/* Message of the last failed call on this thread. */
const char* alz_dft_last_error(void);

/* Frames one call emits: with C samples consumed before it and C' = C + n_samples, ka = max(0, floor((C - size) /
 * hop) + 1), kc = floor((C' - size) / hop): max(0, kc - ka + 1) frames ka .. kc, plus one when final and
 * C' - max(kc + 1, 0) hop > max(size - hop, 0).  Negative on a bad argument. */
int64_t alz_dft_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final);

/* Bytes of device state for n_streams streams of one size: per stream the samples consumed (int64) and the last
 * `size` samples (float32), which hold every sample an open frame still needs.  8-byte aligned. */
int64_t alz_dft_state_bytes(int64_t n_streams, int32_t size);

/* Sets the state of n_streams streams to the start of a stream (no sample consumed). */
int32_t alz_dft_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream);

/* HOST function.  Fills table[n][j] (n = 0 .. size - 1, j = 0 .. n_freqs - 1; host memory, 2 * size * n_freqs
 * float64) with cmath.exp(-1j * n * freqs[j]) for every column j whose twiddles it can restate: CPython's products
 * (-0.0 - 1.0j) * complex(n, 0.0) and then * complex(f, 0.0), which give z = (+0.0, 0.0 + (-n * f)) for a finite f,
 * and cmath.exp's finite path, (exp(0.0) cos(z.imag), exp(0.0) sin(z.imag)) with the host's libm.  A column where z is
 * not of that form for some n (f not finite, or n f overflowing) is left as it is and marked with unfilled[j] = 1
 * (else 0): there cmath.exp returns NaNs or raises ValueError, which the caller takes from cmath itself.  Returns the
 * number of unfilled columns, negative on a bad argument. */
int64_t alz_dft_twiddles(const double* freqs, int32_t n_freqs, int32_t size, double* table, uint8_t* unfilled);

/* The next n_samples >= 0 samples of n_streams streams, x_dev[s * x_stride + n] (float32, 4-byte aligned),
 * continuing state_dev (made by alz_dft_state_init with the same size).  window_dev: `size` float64 values, or NULL.
 * twiddles_dev: the table above for these size and n_freqs, 16-byte aligned.  n_frames is alz_dft_frames(C,
 * n_samples, size, hop, final) for the C samples the state has consumed; the frames are stored in order:
 *
 *   out_dev  [n_streams][n_frames][n_freqs] complex128 (out_c128 != 0, 16-byte aligned) or complex64 (each part the
 *            float32 rounding of the complex128 value, 8-byte aligned)
 *
 * normalize != 0 divides by size as above.  Limits: 1 <= size <= ALZ_DFT_MAX_SIZE, 1 <= n_freqs <= ALZ_DFT_MAX_FREQS,
 * hop >= 1; ALZ_DFT_ERR_UNSUPPORTED for more frames than one launch takes.  A stream cut into blocks of any lengths
 * gives the same bits as one call.  `final` != 0 ends the streams (the state must not be continued). */
int32_t alz_dft_apply_f32(const float* x_dev, int64_t x_stride, const double* window_dev, const double* twiddles_dev,
                          int32_t n_freqs, int32_t normalize, void* out_dev, int32_t out_c128, int64_t n_frames,
                          void* state_dev, int64_t n_streams, int64_t n_samples, int32_t size, int32_t hop,
                          int32_t final, void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_DFT_H */
