/*
 * alz_oracle.c -- TEST INFRASTRUCTURE ONLY.  CPU restatement of the reference's
 * sample-by-sample linear filter evaluator, used as the parity checker by tests/,
 * __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
 * Nothing under audiolazy_b200/ may import, link or call this file.
 *
 * Restates (file:line relative to the reference checkout /root/reference):
 *   - LinearFilter.__call__, audiolazy/lazy_filters.py:141-264: Direct-Form-I,
 *       m0 = (sum_k b_k * d_k  +  sum_{k>=1} -a_k * m_k) / a0
 *     terms added left to right, numerator first then denominator, ascending delay
 *     (:197-237); zero coefficients contribute no term (Poly drops them,
 *     audiolazy/lazy_poly.py:132-139); the division by a0 is applied to the whole sum
 *     (:234-237) and skipped when a0 == 1; every product and sum is a separately
 *     rounded IEEE float64 operation (CPython floats): this file must be compiled with
 *     -ffp-contract=off so that gcc does not fuse them.
 *   - memory / zero seeding, lazy_filters.py:181-195 and :243-250: m_k (k>=1) start from
 *     `memory` (missing entries = zero), d_k (k>=1) start from `zero`.
 *   - CascadeFilter.__call__, lazy_filters.py:988-990: sections applied in series, each
 *     with its own m/d history, float64 between sections.
 *   - the bank fan-out loop of examples/gammatone_plots.py:63-71: the same input goes
 *     through every channel's cascade.
 *
 * Parity pin: tests/test_oracle.py checks this file against golden vectors generated
 * by running the reference itself (tests/golden/make_golden.py) and, when
 * /root/reference is present, against the live reference.
 *
 * Coefficient layout is the one of include/alz_b200.h (alz_plan_create).
 */
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_MAX_TAPS 8192

/* One DF-I section over n samples, in place on a float64 buffer.
 * xh[j] = d_{j+1}, yh[j] = m_{j+1} on entry (histories), updated on exit. */
static void orc_section(const double* b, int nb, const double* a, int na, double* buf, int64_t n, double* xh,
                        double* yh) {
  const double a0 = a[0];
  for (int64_t i = 0; i < n; ++i) {
    const double d0 = buf[i];
    double acc = 0.0;
    int first = 1;
    /* numerator terms, ascending delay */
    for (int k = 0; k < nb; ++k) {
      const double c = b[k];
      if (c == 0.0) continue;
      const double d = (k == 0) ? d0 : xh[k - 1];
      const double term = (c == 1.0) ? d : (c == -1.0) ? -d : c * d;
      if (first) { acc = term; first = 0; } else acc = acc + term;
    }
    /* denominator terms: "-a_k * m_k" */
    for (int k = 1; k < na; ++k) {
      const double c = a[k];
      if (c == 0.0) continue;
      const double m = yh[k - 1];
      const double term = (c == -1.0) ? m : (c == 1.0) ? -m : (-c) * m;
      if (first) { acc = term; first = 0; } else acc = acc + term;
    }
    double m0;
    if (first) m0 = 0.0;                 /* no term at all: reference yields `zero` (0.0 here) */
    else if (a0 == -1.0) m0 = -acc;
    else if (a0 != 1.0) m0 = acc / a0;
    else m0 = acc;
    buf[i] = m0;
    for (int k = na - 2; k > 0; --k) yh[k] = yh[k - 1];
    if (na > 1) yh[0] = m0;
    for (int k = nb - 2; k > 0; --k) xh[k] = xh[k - 1];
    if (nb > 1) xh[0] = d0;
  }
}

/*
 * Bank of cascades on float32 input, float64 output.
 *   x      : [S][T] float32 (row stride xs)
 *   y      : [S][C][T] float64 (row stride ys), the reference's float64 result
 *   coef / desc / C / KM: as alz_plan_create
 *   xinit / yinit : [C][KM][hx] / [C][KM][hy] initial histories or NULL (zeros)
 *   s_begin, s_end : stream range to process (lets a caller thread over streams)
 * Returns 0, or -1 on bad arguments / allocation failure.
 */
int orc_bank_apply(const float* x, double* y, const double* coef, const int32_t* desc, int32_t C, int32_t KM,
                   int64_t S, int64_t T, int64_t xs, int64_t ys, const double* xinit, int32_t hx, const double* yinit,
                   int32_t hy, int64_t s_begin, int64_t s_end) {
  if (!x || !y || !coef || !desc || C <= 0 || KM < 0 || T < 0 || s_begin < 0 || s_end > S) return -1;
  double* buf = (double*)malloc(sizeof(double) * (size_t)(T > 0 ? T : 1));
  double* xh = (double*)calloc(ORC_MAX_TAPS, sizeof(double));
  double* yh = (double*)calloc(ORC_MAX_TAPS, sizeof(double));
  if (!buf || !xh || !yh) { free(buf); free(xh); free(yh); return -1; }
  int rc = 0;
  for (int64_t s = s_begin; s < s_end && rc == 0; ++s) {
    for (int c = 0; c < C && rc == 0; ++c) {
      for (int64_t i = 0; i < T; ++i) buf[i] = (double)x[s * xs + i];
      for (int k = 0; k < KM; ++k) {
        const int32_t* d = desc + ((size_t)c * KM + k) * 3;
        const int nb = d[0], na = d[1];
        if (nb == 0) break;
        if (nb < 0 || na < 1 || nb > ORC_MAX_TAPS || na > ORC_MAX_TAPS) { rc = -1; break; }
        const double* b = coef + d[2];
        const double* a = b + nb;
        for (int j = 0; j < nb - 1; ++j) xh[j] = (xinit && j < hx) ? xinit[((size_t)c * KM + k) * hx + j] : 0.0;
        for (int j = 0; j < na - 1; ++j) yh[j] = (yinit && j < hy) ? yinit[((size_t)c * KM + k) * hy + j] : 0.0;
        orc_section(b, nb, a, na, buf, T, xh, yh);
      }
      memcpy(y + ((size_t)s * C + c) * ys, buf, sizeof(double) * (size_t)T);
    }
  }
  free(buf); free(xh); free(yh);
  return rc;
}

/* Same, rounding the result to float32 (what the device path stores in HBM). */
int orc_bank_apply_f32(const float* x, float* y, const double* coef, const int32_t* desc, int32_t C, int32_t KM,
                       int64_t S, int64_t T, int64_t xs, int64_t ys, int64_t s_begin, int64_t s_end) {
  if (!x || !y || !coef || !desc || C <= 0 || KM < 0 || T < 0 || s_begin < 0 || s_end > S) return -1;
  double* buf = (double*)malloc(sizeof(double) * (size_t)(T > 0 ? T : 1));
  double* xh = (double*)calloc(ORC_MAX_TAPS, sizeof(double));
  double* yh = (double*)calloc(ORC_MAX_TAPS, sizeof(double));
  if (!buf || !xh || !yh) { free(buf); free(xh); free(yh); return -1; }
  int rc = 0;
  for (int64_t s = s_begin; s < s_end && rc == 0; ++s) {
    for (int c = 0; c < C && rc == 0; ++c) {
      for (int64_t i = 0; i < T; ++i) buf[i] = (double)x[s * xs + i];
      for (int k = 0; k < KM; ++k) {
        const int32_t* d = desc + ((size_t)c * KM + k) * 3;
        const int nb = d[0], na = d[1];
        if (nb == 0) break;
        if (nb < 0 || na < 1 || nb > ORC_MAX_TAPS || na > ORC_MAX_TAPS) { rc = -1; break; }
        memset(xh, 0, sizeof(double) * (size_t)nb);
        memset(yh, 0, sizeof(double) * (size_t)na);
        orc_section(coef + d[2], nb, coef + d[2] + nb, na, buf, T, xh, yh);
      }
      float* out = y + ((size_t)s * C + c) * ys;
      for (int64_t i = 0; i < T; ++i) out[i] = (float)buf[i];
    }
  }
  free(buf); free(xh); free(yh);
  return rc;
}
