/* alz_b200_stft.h -- plain-C ABI of libalz_b200_stft.so: short-time Fourier analysis, resynthesis and overlap-add of
 * many streams, evaluated by sm_90a kernels (AudioLazy's stft and overlap_add).
 *
 * Frames.  For one stream x (float32 samples), frame k covers stream samples [k hop, k hop + size) and is emitted once
 * its last sample has been consumed; at the end of a stream of N samples (`final`) the first incomplete frame k is
 * emitted too if N - k hop > max(size - hop, 0), its missing samples 0.0 (AudioLazy's padded last block of
 * Stream.blocks(size, hop), the rule of alz_b200_lpc.h).
 *
 * Analysis.  Frame k becomes the float64 block
 *
 *   b[n] = (double)x[k hop + n]              without a window
 *   b[n] = (double)x[k hop + n] * w[n]       with a window w of `size` float64 values (one rounding, no fma)
 *
 * which, when `shift` is set, is rotated as numpy.fft.ifftshift does (b'[n] = b[(n + size / 2) % size]), and then
 * goes through a float64 real FFT: X[j] = sum(b'[n] exp(-2 pi i j n / size)) for j = 0 .. size / 2.  The FFT is an
 * in-place shared-memory mixed-radix transform with radix 4, 2, 3, 5 and 7 butterflies and a direct DFT of O(p) per output for
 * any other prime factor p; its roots come from the caller's table twiddle_dev, `size` complex float64 values with
 * twiddle[m] = exp(-2 pi i m / size) (re, im interleaved), and its complex products may use fma.  It is accurate to a
 * few float64 ulps of the frame's peak |X| times log(size), not bit-identical to numpy's pocketfft.  A complex64
 * output is the complex128 result rounded to float32 per component.
 *
 * Synthesis.  Each frame of spectra, size / 2 + 1 bins, goes through numpy.fft.irfft(X, size): the imaginary parts of
 * bin 0 and, for an even size, of bin size / 2 are ignored, the result is scaled by 1 / size, then rotated back as
 * numpy.fft.fftshift does when `shift` is set (v[n] = v'[(n - size / 2) mod size]).  The float64 frames v are stored,
 * and then optionally overlap-added.
 *
 * Overlap-add.  With w' a float64 window (or none: the frame values as they are), output sample t of the stream is
 * the sum of w'[j] * v_k[j], j = t - k hop, over the frames k that cover it, oldest frame first, each newer term added
 * to the running sum; the samples t < size - hop also start from +0.0 (so -0.0 comes out +0.0 there).  That is
 * AudioLazy's overlap_add (numpy and list strategies) exactly, for the same float64 frames and window.  A call on F
 * frames emits F hop float32 samples (the float32 of those float64 sums) and keeps the size - hop sums still open in
 * the state; the final call also emits those size - hop sums (so a stream with no frames at all gives size - hop
 * zeros).
 *
 * All pointers are device pointers; calls are asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default
 * stream) and must be made with the device of the buffers current.  The library keeps no state between calls: the
 * stream state and the buffers both come from the caller.  A stream cut into blocks of any lengths gives the same bits
 * as one call.  Limits: 1 <= size <= ALZ_STFT_MAX_SIZE, 1 <= hop <= size.
 */
#ifndef ALZ_B200_STFT_H
#define ALZ_B200_STFT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_STFT_OK 0
#define ALZ_STFT_ERR_INVALID (-1)      /* bad argument; alz_stft_last_error() has the message */
#define ALZ_STFT_ERR_CUDA (-4)         /* a CUDA call failed */
#define ALZ_STFT_ERR_UNSUPPORTED (-6)  /* a shape too large for one launch */

#define ALZ_STFT_MAX_SIZE 8192

/* Message of the last failed call on this thread. */
const char* alz_stft_last_error(void);

/* Frames an analysis call emits with `consumed` samples before it (the rule of alz_lpc_frames).  Negative on a bad
 * argument. */
int64_t alz_stft_frames(int64_t consumed, int64_t n_samples, int32_t size, int32_t hop, int32_t final);

/* Bytes of analysis state for n_streams streams: per stream the samples consumed (int64) and the last `size` samples
 * (float32).  8-byte aligned. */
int64_t alz_stft_analysis_state_bytes(int64_t n_streams, int32_t size);

/* Sets the analysis state of n_streams streams to the start of a stream (no sample consumed). */
int32_t alz_stft_analysis_state_init(void* state_dev, int64_t n_streams, int32_t size, void* cuda_stream);

/* Bytes of overlap-add state for n_streams streams: per stream the frames consumed (int64) and the size - hop open
 * float64 sums (twice: the call reads one copy and writes the other).  8-byte aligned. */
int64_t alz_stft_ola_state_bytes(int64_t n_streams, int32_t size, int32_t hop);

/* Sets the overlap-add state of n_streams streams to the start of a stream (no frame consumed, every open sum +0.0). */
int32_t alz_stft_ola_state_init(void* state_dev, int64_t n_streams, int32_t size, int32_t hop, void* cuda_stream);

/* The next n_samples >= 0 samples of n_streams streams, x_dev[s * x_stride + n] (float32, 4-byte aligned),
 * continuing state_dev.  window_dev: `size` float64 values or NULL.  n_frames is alz_stft_frames(C, n_samples, size,
 * hop, final) for the C samples the state has consumed.  The spectra go to spec_dev [n_streams][n_frames][size / 2 +
 * 1], complex128 (interleaved float64) when spec_c128 != 0, else complex64.  `final` != 0 ends the streams. */
int32_t alz_stft_analysis(const float* x_dev, int64_t x_stride, const double* window_dev, const double* twiddle_dev,
                          void* spec_dev, int32_t spec_c128, int64_t n_frames, void* state_dev, int64_t n_streams,
                          int64_t n_samples, int32_t size, int32_t hop, int32_t shift, int32_t final,
                          void* cuda_stream);

/* Resynthesis of n_frames frames of spectra of n_streams streams: bin j of frame f of stream s at spec_dev[s *
 * stream_stride + f * frame_stride + j] (in complex elements; complex128 when spec_c128 != 0, else complex64).  The
 * float64 frames go to frames_dev [n_streams][n_frames][size] (always given).  When y_dev is not NULL they are then
 * overlap-added as alz_stft_ola_f64 does, with ola_window_dev, ola_state_dev, y_dev and y_stride. */
int32_t alz_stft_synthesis(const void* spec_dev, int32_t spec_c128, int64_t frame_stride, int64_t stream_stride,
                           const double* twiddle_dev, int32_t shift, double* frames_dev, const double* ola_window_dev,
                           float* y_dev, int64_t y_stride, void* ola_state_dev, int64_t n_streams, int64_t n_frames,
                           int32_t size, int32_t hop, int32_t final, void* cuda_stream);

/* Overlap-add of n_frames float64 frames of n_streams streams, value j of frame f of stream s at frames_dev[s *
 * stream_stride + f * frame_stride + j], continuing ola_state_dev.  window_dev: `size` float64 values w', or NULL for
 * none.  y_dev[s * y_stride + t] receives n_frames * hop samples, plus size - hop when `final` != 0 (which ends the
 * streams). */
int32_t alz_stft_ola_f64(const double* frames_dev, int64_t frame_stride, int64_t stream_stride,
                         const double* window_dev, float* y_dev, int64_t y_stride, void* ola_state_dev,
                         int64_t n_streams, int64_t n_frames, int32_t size, int32_t hop, int32_t final,
                         void* cuda_stream);

/* As alz_stft_ola_f64, for float32 frames (each value widened to float64 exactly). */
int32_t alz_stft_ola_f32(const float* frames_dev, int64_t frame_stride, int64_t stream_stride,
                         const double* window_dev, float* y_dev, int64_t y_stride, void* ola_state_dev,
                         int64_t n_streams, int64_t n_frames, int32_t size, int32_t hop, int32_t final,
                         void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_STFT_H */
