/* alz_b200_parcor.h -- plain-C ABI of libalz_b200_parcor.so: the reflection (PARCOR) coefficients of many FIR rows,
 * evaluated by an sm_90a kernel, bit for bit as AudioLazy's parcor(ZFilter(row)) and parcor_stable(1 / ZFilter(row))
 * compute them under CPython 3.12 on x86-64 glibc 2.39.
 *
 * For a row a[0 .. L-1] (float64) with a[0] == 1, M is the index of its last coefficient that is not zero (-0.0 is
 * zero, NaN is not), because AudioLazy's ZFilter keeps only nonzero terms.  For m = M .. 1, in that order:
 *
 *   k = a[m], or +0.0 when it is zero; k is emitted
 *   q = k ** 2, CPython's float pow: NaN -> NaN, +-inf -> inf, 0 -> +0.0, |k| == 1 -> 1.0, else glibc's pow(|k|, 2.0),
 *       which is not correctly rounded (see csrc_parcor/alz_pow2.h); an infinite result of a finite k is
 *       OverflowError: failure code 2
 *   d = 1 - q;  d == 0 is ParCorError: failure code 1 (both failures after k was emitted)
 *   r = 1 / d   (a ZFilter divides by a number through its reciprocal)
 *   for j = 1 .. m - 1:  t = a[j] when k == 0 or a[m - j] == 0, else a[j] - k * a[m - j]
 *                        a[j] = +0.0 when r == 0 or t == 0, else t * r
 *
 * (a zero scalar times a polynomial is the zero polynomial, and a missing term is not multiplied; a[0] is set back to
 * 1 each step and never feeds a k).  Every operation is one IEEE round-to-nearest operation; nothing is contracted.
 * parcor_stable is "every emitted k has |k| < 1": a failure only follows a k with |k| >= 1, a NaN k is not stable,
 * and a row with M == 0 is stable.  A row with a[0] != 1 (NaN included) takes another path in AudioLazy (its top term
 * is not cancelled) and is not evaluated here: it gets failure code 3, count 0, stable 0 and NaN k.
 *
 * All pointers are device pointers; the call is asynchronous on `cuda_stream` (a cudaStream_t, NULL = legacy default
 * stream) and must be made with the device of the buffers current.  The library keeps no state between calls.
 */
#ifndef ALZ_B200_PARCOR_H
#define ALZ_B200_PARCOR_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ALZ_PARCOR_OK 0
#define ALZ_PARCOR_ERR_INVALID (-1)      /* bad argument; alz_parcor_last_error() has the message */
#define ALZ_PARCOR_ERR_CUDA (-4)         /* a CUDA call failed */

#define ALZ_PARCOR_MAX_LEN 65            /* rows of LPC filters up to order 64 */

/* Message of the last failed call on this thread. */
const char* alz_parcor_last_error(void);

/* The step-down of n_rows >= 0 rows coef_dev[i * row_stride + j], j = 0 .. L - 1 (float64, 8-byte aligned,
 * row_stride >= L when n_rows > 1), 1 <= L <= ALZ_PARCOR_MAX_LEN.  Outputs, each NULL when not wanted:
 *
 *   k_dev       float64 [n_rows][L - 1]   the emitted k in emission order (highest order first), NaN past count
 *   count_dev   int32   [n_rows]          how many k were emitted
 *   failed_dev  uint8   [n_rows]          0, or the failure code 1 / 2 / 3 above
 *   stable_dev  uint8   [n_rows]          parcor_stable: 1 or 0
 */
int32_t alz_parcor_f64(const double* coef_dev, int64_t row_stride, int64_t n_rows, int32_t L, double* k_dev,
                       int32_t* count_dev, uint8_t* failed_dev, uint8_t* stable_dev, void* cuda_stream);

#ifdef __cplusplus
}
#endif

#endif /* ALZ_B200_PARCOR_H */
