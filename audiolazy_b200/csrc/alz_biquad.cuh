// alz_biquad.cuh -- cascade-of-biquads recurrence core (the hot kernel).
//
// Math (reference LinearFilter.__call__, lazy_filters.py:197-257, composed by
// CascadeFilter.__call__, :988-990).  Section k of a cascade computes
//     u_k[n] = (b0 u_{k-1}[n] + b1 u_{k-1}[n-1] + b2 u_{k-1}[n-2]
//               - a1 u_k[n-1] - a2 u_k[n-2]) / a0 ,      u_0 = x,  y = u_K.
// The reference evaluates this in float64 with separately rounded products.  Here:
//   * the whole cascade stays in FLOAT64 REGISTERS (state) and UNIFORM REGISTERS
//     (coefficients); float32 exists only in HBM and in the shared-memory tile.
//     SURVEY.md section 7: float32 coefficients/state miss the 1e-5 parity bar by up to
//     6 orders of magnitude on low ERB channels.
//   * a0 is folded into the coefficients on the host, products are fused (DFMA).
//   * MONIC form: b0 of every section is factored out (floating point is scale
//     invariant, so this costs no accuracy): in working units u'_k = u_k * sc_k with
//     sc_k = 1/(b0_1...b0_k),
//         u'_k[n] = u'_{k-1}[n] + c1 u'_{k-1}[n-1] + c2 u'_{k-1}[n-2]
//                   + na1 u'_k[n-1] + na2 u'_k[n-2]          (NB-1+2 DFMA)
//     and y = G * u'_K with G = b0_1...b0_K (one DMUL).  For the gammatone "slaney"
//     cascade (4 sections, 2 numerator taps): 4*3 + 1 = 13 FP64 ops per
//     channel-sample instead of the reference's 28 flops / 16 fused ops.
//   * once two samples have been processed, the input history of section k IS the
//     output history of section k-1, so the steady-state loop keeps only K+1 signal
//     histories (aliased form).  The first two samples of every launch use explicit
//     per-section input histories so that memory=/zero= seeding
//     (lazy_filters.py:181-195, :243-250) is honoured exactly; when the state comes
//     from a previous launch the two forms see identical operands, so splitting a
//     stream into blocks is bit-exact.
//   * the state buffer holds WORKING-unit values (the host scales memory=/zero= once
//     in alz_state_init), so no rounding happens at block boundaries.
//
// Cost model: a float64-tier warp-sample of the slaney bank issues 12 DFMA/DMUL (uniform-
// register coefficient) and 2 F2F conversions (MONIC mode 2; mode 1 costs more): the kernel
// is FP64-issue bound below the HBM roofline, by construction of the arithmetic the parity
// bar demands (DESIGN.md section 3).
#pragma once
#include "alz_lane.cuh"

#ifndef ALZ_GROUP_UNROLL
#define ALZ_GROUP_UNROLL 8   // groups of 4 samples unrolled in the steady-state loop (8 = the whole tile)
#endif
constexpr int kAlzGroupUnroll = ALZ_GROUP_UNROLL;

// Per-POSITION coefficient record inside the kernel parameters (constant bank); position =
// blockIdx.x of the launch, the plan orders channels so that precision tiers interleave:
//   [k*5 + 0..4] = b0 (1 when monic), b1|c1, b2|c2, -a1, -a2   (all / a0);  [5K] = G;
//   head-FIR plans (NB0 = 8): [5K+1 .. 5K+5] = taps 3..7 of the FIRST section;
//   last slot (ALZ_COEF_META) = channel index + 65536 * tier, as a double.
// Tier 0 records hold doubles; tier 1 (float32 recurrence) records hold the SAME entries as
// floats packed from the start of the record (entry i at float index i).
#define ALZ_COEF_NVAL(K, NB0) (5 * (K) + 1 + ((NB0) > 3 ? (NB0) - 3 : 0))
#define ALZ_COEF_STRIDE(K, NB0) (ALZ_COEF_NVAL(K, NB0) + 1)
#define ALZ_COEF_META(K, NB0) ALZ_COEF_NVAL(K, NB0)
// State: state[slot * sstride + r], r = c*Stot + s (working units; consecutive lanes = consecutive
// streams touch consecutive doubles).  Section 0: H0 input
// delays (H0 = max(NB0 - 1, 2)) then yd1, yd2; section k >= 1: xd1, xd2, yd1, yd2.
#define ALZ_H0(NB0) ((NB0) > 3 ? (NB0) - 1 : 2)
#define ALZ_STATE_BASE(k, NB0) ((k) == 0 ? 0 : ALZ_H0(NB0) + 2 + 4 * ((k) - 1))
#define ALZ_STATE_SLOTS(K, NB0) (ALZ_H0(NB0) + 2 + 4 * ((K) - 1))
// Built ONCE per plan (one block per launch chunk) and handed to cudaLaunchKernel by address: no
// per-launch copy on the host, no lock, any number of host threads / devices.
template <int NCOEF>
struct AlzBiquadArgs {
  int rec_stride;      // ALZ_COEF_STRIDE of the plan
  int n_pos;           // positions (channels) of this launch chunk
  double coef[NCOEF];  // [positions of this launch][rec_stride]
  __device__ __forceinline__ int meta(int pos) const { return (int)coef[pos * rec_stride + rec_stride - 1]; }
  __device__ __forceinline__ int channel(int pos) const { return meta(pos) & 0xffff; }
  __device__ __forceinline__ int tier(int pos) const { return meta(pos) >> 16; }
};

// fused multiply-add in the working type (host versions: the plan-time tier probe runs the
// SAME arithmetic on the CPU, fma/fmaf are correctly rounded there too)
__host__ __device__ __forceinline__ double alz_fma(double a, double b, double c) { return fma(a, b, c); }
__host__ __device__ __forceinline__ float alz_fma(float a, float b, float c) { return fmaf(a, b, c); }

// MONIC: 0 = plain sections; 1 = b0 factored out, gain applied to the float64 OUTPUT (one
// DMUL per sample, bit-faithful); 2 = b0 factored out, gain applied to the float32 INPUT
// (an FP32 multiply before the widening conversion: the FP64 pipe does one op less per
// sample; costs two extra float32 roundings, <= 1.8e-7 relative, still 50x inside the bar).
// NB0: numerator taps of the FIRST section when it is longer than a biquad's (head FIR on
// the input, e.g. gammatone.sampled's 8-tap first section); 0 = same as NB.
// ZMASK: numerator taps that are zero in EVERY channel and are not computed at all (the
// reference's Poly drops zero coefficients too): bit 2k = tap 1 of section k, bit 2k+1 = tap 2.
// ALZ_ZMASK_KLAPURI is gammatone.klapuri's cascade [1 - z^-2, const, 1 - z^-2, const] / poles.
#define ALZ_ZMASK_KLAPURI 0xDD
// W: working type of the recurrence.  double = tier 0 (every channel qualifies); float = tier 1,
// only for channels whose float32 evaluation was MEASURED at plan creation to stay well inside
// the parity bar (alz_capi.cu: tier probe) -- high ERB channels with poles far from z = 1.  The
// float32 warps use the FP32 pipe and no conversions, and run in the issue slots the FP64 warps
// of the same SM leave free.
template <int K, int NB, int MONIC, int NB0 = 0, int ZMASK = 0, typename W = double>
struct AlzBiquadCore {
  static constexpr int H0 = ALZ_H0(NB0);
  static constexpr int NBF = NB0 > 3 ? NB0 : NB;   // taps of section 0
  W b0[K], c1[K], c2[K], na1[K], na2[K];
  W ch[NB0 > 3 ? NB0 - 3 : 1];                // taps 3.. of section 0
  W G;
  float Gf;
  W u[K + 1][2];   // u[k][0] = u_k[n-1], u[k][1] = u_k[n-2]; u[0] = input history (NB0 <= 3)
  W xh[H0];        // input history of section 0 when NB0 > 3 (xh[j] = x[n-1-j])
  W xe[K][2];      // explicit input histories of sections 1..K-1 (index 0 unused)

  // coefficient record -> registers (rec: this position's record; doubles for W = double, packed floats for float)
  __host__ __device__ __forceinline__ void load_coef(const double* rec) {
    const W* cf = reinterpret_cast<const W*>(rec);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      b0[k] = cf[5 * k + 0];
      c1[k] = cf[5 * k + 1];
      c2[k] = cf[5 * k + 2];
      na1[k] = cf[5 * k + 3];
      na2[k] = cf[5 * k + 4];
    }
    G = cf[5 * K];
    Gf = (float)G;
    if (NB0 > 3) {
#pragma unroll
      for (int j = 3; j < NB0; ++j) ch[j - 3] = cf[5 * K + 1 + (j - 3)];
    }
  }
  __host__ __device__ __forceinline__ void zero_state() {
#pragma unroll
    for (int j = 0; j < H0; ++j) xh[j] = W(0);
#pragma unroll
    for (int k = 0; k <= K; ++k) u[k][0] = u[k][1] = W(0);
#pragma unroll
    for (int k = 0; k < K; ++k) xe[k][0] = xe[k][1] = W(0);
  }

  // The state buffer always holds float64 working-unit values; a float32 tier narrows on load and
  // widens (exactly) on store, so block splitting stays bit-exact in either tier.
  template <class Args>
  __device__ __forceinline__ void load(const AlzTileArgs& a, const Args& ca, long long r, int c_local, bool /*valid*/) {
    load_coef(ca.coef + c_local * ALZ_COEF_STRIDE(K, NB0));   // CTA-uniform address
    const double* st = a.state + r;
    const long long R = a.sstride;
#pragma unroll
    for (int j = 0; j < H0; ++j) xh[j] = (W)__ldcg(st + (long long)j * R);   // .cg: the state may have been written by another CTA of this launch
    u[0][0] = xh[0]; u[0][1] = xh[1];
    xe[0][0] = xe[0][1] = W(0);
    u[1][0] = (W)__ldcg(st + (long long)(H0 + 0) * R);
    u[1][1] = (W)__ldcg(st + (long long)(H0 + 1) * R);
#pragma unroll
    for (int k = 1; k < K; ++k) {
      const int base = ALZ_STATE_BASE(k, NB0);
      xe[k][0] = (W)__ldcg(st + (long long)(base + 0) * R);
      xe[k][1] = (W)__ldcg(st + (long long)(base + 1) * R);
      u[k + 1][0] = (W)__ldcg(st + (long long)(base + 2) * R);
      u[k + 1][1] = (W)__ldcg(st + (long long)(base + 3) * R);
    }
  }

  // Section 0 with a head FIR: reads and shifts the input history xh.
  __host__ __device__ __forceinline__ W head(W in) {
    W t = MONIC ? in : b0[0] * in;
    t = alz_fma(c1[0], xh[0], t);
    t = alz_fma(c2[0], xh[1], t);
#pragma unroll
    for (int j = 3; j < NB0; ++j) t = alz_fma(ch[j - 3], xh[j - 1], t);
#pragma unroll
    for (int j = H0 - 1; j > 0; --j) xh[j] = xh[j - 1];
    xh[0] = in;
    const W y1 = u[1][0], y2 = u[1][1];
    t = alz_fma(na2[0], y2, t);
    const W y = alz_fma(na1[0], y1, t);
    u[1][1] = y1;
    u[1][0] = y;
    return y;
  }

  // One section's arithmetic.  in/in1/in2 = u_{k-1}[n], [n-1], [n-2].
  __host__ __device__ __forceinline__ W section(int k, W in, W in1, W in2, W y1, W y2) const {
    W t = MONIC ? in : b0[k] * in;
    if (NB >= 2 && !((ZMASK >> (2 * k)) & 1)) t = alz_fma(c1[k], in1, t);
    if (NB >= 3 && !((ZMASK >> (2 * k + 1)) & 1)) t = alz_fma(c2[k], in2, t);
    t = alz_fma(na2[k], y2, t);
    return alz_fma(na1[k], y1, t);
  }

  // Steady state: section k reads the history of section k-1's output.
  __host__ __device__ __forceinline__ float step_alias(W xin) { return (float)step_alias_w(xin); }
  __host__ __device__ __forceinline__ float step_explicit(W xin) { return (float)step_explicit_w(xin); }

  __host__ __device__ __forceinline__ W step_alias_w(W xin) {
    W in = xin, in1, in2;
    if (NB0 > 3) {
      in1 = u[1][0]; in2 = u[1][1];       // section 1 reads section 0's OLD output history
      in = head(xin);
    } else {
      in1 = u[0][0]; in2 = u[0][1];
      u[0][1] = in1;
      u[0][0] = in;
    }
#pragma unroll
    for (int k = (NB0 > 3 ? 1 : 0); k < K; ++k) {
      const W y1 = u[k + 1][0], y2 = u[k + 1][1];
      const W y = section(k, in, in1, in2, y1, y2);
      u[k + 1][1] = y1;
      u[k + 1][0] = y;
      in = y; in1 = y1; in2 = y2;
    }
    return MONIC == 1 ? G * in : in;
  }

  // First two samples of a launch: explicit input histories.
  __host__ __device__ __forceinline__ W step_explicit_w(W xin) {
    W in = xin;
    if (NB0 > 3) in = head(xin);
#pragma unroll
    for (int k = (NB0 > 3 ? 1 : 0); k < K; ++k) {
      W in1, in2;
      if (k == 0) { in1 = u[0][0]; in2 = u[0][1]; u[0][1] = in1; u[0][0] = in; }
      else { in1 = xe[k][0]; in2 = xe[k][1]; xe[k][1] = in1; xe[k][0] = in; }
      const W y1 = u[k + 1][0], y2 = u[k + 1][1];
      const W y = section(k, in, in1, in2, y1, y2);
      u[k + 1][1] = y1;
      u[k + 1][0] = y;
      in = y;
    }
    return MONIC == 1 ? G * in : in;
  }

  // float32 sample -> float64 section input (with the input-side gain when MONIC == 2)
  __host__ __device__ __forceinline__ W widen(float x) const { return MONIC == 2 ? (W)(x * Gf) : (W)x; }

  // Filter my row of the tile in place: float32 in, float32 out.  `swz` is the XOR
  // applied to the 16-byte chunk index (0 for the padded cp.async tile, lane & 7 for the
  // TMA 128-byte-swizzled tile).
  // four steady-state samples of group g, in place; xf carries the prefetched next group
  __device__ __forceinline__ void group(float* row, int swz, int g, float4& xf) {
    float* p = row + ((g ^ swz) << 2);
    const float4 xc = xf;
    if (g + 1 < ALZ_TT / 4) xf = *reinterpret_cast<const float4*>(row + (((g + 1) ^ swz) << 2));   // prefetch
    float4 o;
    o.x = step_alias(widen(xc.x));
    o.y = step_alias(widen(xc.y));
    o.z = step_alias(widen(xc.z));
    o.w = step_alias(widen(xc.w));
    *reinterpret_cast<float4*>(p) = o;
  }

  __device__ __forceinline__ void tile(float* row, int swz, int nvalid, long long n_done) {
    if (nvalid == ALZ_TT) {
      if (n_done >= 2) {
        float4 xf = *reinterpret_cast<const float4*>(row + ((0 ^ swz) << 2));
#pragma unroll kAlzGroupUnroll
        for (int g = 0; g < ALZ_TT / 4; ++g) group(row, swz, g, xf);
      } else {   // first tile after a state load: two explicit-history samples, then steady state (kept compact)
        float* p = row + ((0 ^ swz) << 2);
        const float4 xc = *reinterpret_cast<const float4*>(p);
        float4 o;
        o.x = step_explicit(widen(xc.x));
        o.y = step_explicit(widen(xc.y));
        o.z = step_alias(widen(xc.z));
        o.w = step_alias(widen(xc.w));
        *reinterpret_cast<float4*>(p) = o;
        float4 xf = *reinterpret_cast<const float4*>(row + ((1 ^ swz) << 2));
#pragma unroll 1
        for (int g = 1; g < ALZ_TT / 4; ++g) group(row, swz, g, xf);
      }
    } else {
      for (int j = 0; j < nvalid; ++j) {
        float* p = row + ((((j >> 2) ^ swz) << 2) | (j & 3));
        const W xin = widen(*p);
        *p = (n_done + j < 2) ? step_explicit(xin) : step_alias(xin);
      }
    }
  }

  // ParallelFilter (alz_parallel.cuh): this channel's UNROUNDED outputs of one tile are added to acc[] (registers,
  // left-associated over the channels as reference lazy_filters.py:1053-1054); the input row is left untouched.
  // Always called right after load(): the first two samples use the explicit histories.
  template <int J>
  __device__ __forceinline__ void acc_from(const float* xrow, int swz, int nvalid, bool first, W (&acc)[ALZ_TT]) {
    if constexpr (J < ALZ_TT) {
      if (J < nvalid) {
        const W xin = widen(xrow[(((J >> 2) ^ swz) << 2) | (J & 3)]);
        const W y = J < 2 ? step_explicit_w(xin) : step_alias_w(xin);
        acc[J] = first ? y : acc[J] + y;
      }
      acc_from<J + 1>(xrow, swz, nvalid, first, acc);
    }
  }

  __device__ __forceinline__ void store(const AlzTileArgs& a, long long r, long long T) {
    double* st = a.state + r;
    const long long R = a.sstride;
    if (NB0 > 3) {
#pragma unroll
      for (int j = 0; j < H0; ++j) st[(long long)j * R] = (double)xh[j];
    } else {
      st[0] = (double)u[0][0];
      st[R] = (double)u[0][1];
    }
    st[(long long)(H0 + 0) * R] = (double)u[1][0];
    st[(long long)(H0 + 1) * R] = (double)u[1][1];
#pragma unroll
    for (int k = 1; k < K; ++k) {
      const int base = ALZ_STATE_BASE(k, NB0);
      W x1, x2;
      if (T >= 2) { x1 = u[k][0]; x2 = u[k][1]; }   // aliased: section k-1's output history
      else { x1 = xe[k][0]; x2 = xe[k][1]; }
      st[(long long)(base + 0) * R] = (double)x1;
      st[(long long)(base + 1) * R] = (double)x2;
      st[(long long)(base + 2) * R] = (double)u[k + 1][0];
      st[(long long)(base + 3) * R] = (double)u[k + 1][1];
    }
  }
};
