// alz_lane.cuh -- "lane = stream" warp engine: the layout every recurrence kernel runs on.
//
// Why this layout: a DFMA whose three operands are three different register pairs asks
//   the register file for 3 x 64-bit operands per lane; with one operand in a UNIFORM
//   register it asks for two.  Filter
//   coefficients are per-channel constants, so if all 32 lanes of a warp work on the
//   SAME channel the coefficients are warp-uniform: they live in uniform registers
//   (loaded from the kernel-parameter constant bank), cost no vector registers and no
//   register-file bandwidth, and every DFMA of the recurrence has only two register
//   operands (a state value and the running sum).
//
// Work decomposition:
//   * CTA = ONE WARP = (channel c = blockIdx.x, stream group g = blockIdx.y); lane l owns
//     the recurrence of stream s = 32 g + l through channel c, serial in time.  blockIdx.x
//     is the fast grid index, so the C warps that need the same input tile run
//     back to back and share it through L2.
//   * time is cut into tiles of 32 samples.  A tile lives in ONE padded shared buffer
//     [32 rows = lanes][36 floats]:
//       1. cp.async (16 B chunks, .cg) brings 32 input rows x 128 B in, one tile ahead;
//       2. each lane converts and filters ITS OWN row in place (LDS.128 -> 4 x F2F ->
//          4 x cascade step -> STS.128 to the same address);
//       3. the warp writes the buffer out, 4 rows x 128 B per store instruction, every
//          global store a whole 128-byte line of one output row y[s][c][t0:t0+32].
//     Two such buffers alternate: while tile i is filtered in buffer A, tile i+1 lands
//     in buffer B; buffer A is refilled with tile i+2 as soon as it has been written out.
//   * no CTA-wide barrier exists (a CTA is one warp): only __syncwarp.
//
// HBM traffic per input sample: 4 B read (the C re-reads of a tile hit L2) + 4 C B written.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#define ALZ_TT 32          // samples per tile
#define ALZ_PITCH 36       // floats per tile row (32 + 4 pad: conflict-free 16-byte accesses)
#define ALZ_TILE_BYTES (32 * ALZ_PITCH * 4)
#define ALZ_WARP_SMEM (2 * ALZ_TILE_BYTES)

struct AlzTileArgs {
  const float* x;   // [S] rows, stride xs
  float* y;         // [S*C] rows (stream-major, channel-minor), stride ys
  long long S, T, xs, ys;
  long long ysS;    // y stride between consecutive STREAMS (C*ys for the dense [S][C][T] layout)
  long long Stot;   // streams the state buffer was sized for: recurrence index r = c * Stot + s
  double* state;    // state[slot * sstride + r] (float64 working-unit values, in/out)
  long long sstride;   // slot stride of the state buffer (recurrences it was sized for)
  // Time segmentation (TMA engine only; nseg <= 1 = off).  The grid is (channels, groups*nseg);
  // a CTA draws a ticket from its channel's counter, tickets map to (segment, group) segment-major,
  // and segment k of a (channel, group) waits for the flag its segment k-1 raises after storing
  // the state.  Fills the last partial wave of a launch with the next segment's work.
  int nseg;
  int groups;            // stream groups of this launch = ceil(S / 32)
  long long seg_len;     // samples per segment (multiple of 32)
  unsigned* sync;        // [channels of this launch] tickets, then [channels][groups] flags; zeroed per launch
  // TMA engine: 2 / 4 = tiles in groups of that many (all loads issued together, all stores back to
  // back: each output row receives 256 / 512 contiguous bytes at once, better HBM write efficiency,
  // but no prefetch under the compute of the same warp -- for launches that fill the machine);
  // 0 / 1 = one tile at a time with the next one prefetched (latency-bound launches).
  int paired;
  int vec_store;    // TMA engine, tile groups of 4: a group leaves through 32 warp-wide st.global.v4 (one row's 512 B
                    // each) instead of TMA box stores (alz_lane_tma.cuh); y, ys and ysS 16-byte aligned
  int C;            // channels of the whole bank (output row index = s*C + c)
  int vec_in;       // 1: x rows are 16-byte aligned (16 B cp.async), 0: 4 B cp.async
  int vec_out;      // 1: y rows are 16-byte aligned (st.v4), 0: scalar stores
  int vP;           // > 0: VIRTUAL streams (time-parallel evaluation, alz_capi.cu): row v of this launch is chunk v % vP
                    // of real stream v / vP; x / y are reached through 3-D / 4-D tensor maps (TMA engine only, vP % 32 == 0)
  // fused envelope consumer (alz_apply_envelope_f32, TMA engine): instead of storing y, every lane follows its channel
  // output with a one-pole lowpass of |y| or y^2 and keeps every env_decim-th value
  float* env_out;        // [S][C][(env_phase + T) / env_decim] rows, stride env_es (virtual streams: the REAL stream's row)
  long long env_es;
  double* env_state;     // [C * Stot] lowpass states (in/out)
  double env_g, env_R;   // e[n] = g * r[n] + R * e[n-1]
  int env_decim, env_mode;   // mode 0: r = |y|; 1: r = y^2; 2: r = y^2 and sqrt on output (rms)
  int env_phase;         // samples of the current decimation window consumed before this block (0 <= env_phase < env_decim)
  int env_store;         // 0: the envelope values are computed but not stored (only the final lowpass states are wanted)
  int exp;          // ALZ_EXP (profiling experiments, TMA engine; results are garbage): 1 = load only the first
                    // tile group and refilter it, 2 = no tile stores
};

__device__ __forceinline__ void alz_cp_async16(void* smem_dst, const void* gsrc, int src_bytes) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void alz_cp_async4(void* smem_dst, const void* gsrc, int src_bytes) {
  unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4, %2;\n" ::"r"(d), "l"(gsrc), "r"(src_bytes) : "memory");
}
__device__ __forceinline__ void alz_cp_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void alz_cp_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory"); }

__device__ __forceinline__ void alz_st_v4(float* p, float4 v) {
  asm volatile("st.global.v4.f32 [%0], {%1, %2, %3, %4};\n" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

// Bring tile t0 of the 32 input rows of stream group `s0` into `buf` (zero filled beyond S / T).
// xg / xstr: address of row 0 of this stream group and the distance between its rows (real streams: a.x + s0 * xs, xs;
// virtual streams: the 32 rows are consecutive chunks of one real stream, distance = the chunk length).
__device__ __forceinline__ void alz_issue_tile(const AlzTileArgs& a, float* buf, const float* xg, long long xstr, long long s0,
                                               long long t0, int lane, bool lean) {
  const int sub = lane >> 3, col = (lane & 7) << 2;
  if (lean) {   // full tile, full group, aligned: 8 unpredicated 16-byte copies per lane
    const float* src = xg + sub * xstr + t0 + col;
    float* dst = buf + sub * ALZ_PITCH + col;
#pragma unroll
    for (int it = 0; it < 8; ++it) {
      alz_cp_async16(dst, src, 16);
      src += 4 * xstr;
      dst += 4 * ALZ_PITCH;
    }
  } else if (a.vec_in) {
#pragma unroll 1
    for (int it = 0; it < 8; ++it) {
      const int row = it * 4 + sub;
      const long long left = a.T - (t0 + col);
      int n = left >= 4 ? 4 : (left > 0 ? (int)left : 0);
      if (s0 + row >= a.S) n = 0;
      const float* src = n ? xg + row * xstr + t0 + col : a.x;
      alz_cp_async16(buf + row * ALZ_PITCH + col, src, n * 4);
    }
  } else {
#pragma unroll 1
    for (int row = 0; row < 32; ++row) {
      const bool in = (t0 + lane) < a.T && (s0 + row) < a.S;
      const float* src = in ? xg + row * xstr + t0 + lane : a.x;
      alz_cp_async4(buf + row * ALZ_PITCH + lane, src, in ? 4 : 0);
    }
  }
}

// Core concept:
//   struct Core {
//     __device__ void load(const AlzTileArgs&, const CoreArgs&, long long r /* = c*Stot + s */, int c_local, bool valid);
//     __device__ void tile(float* row, int swz, int nvalid, long long n_done);
//         // row[0..nvalid) holds float32 inputs; overwrite them with float32 outputs.
//         // n_done = samples already processed in this launch (warp-uniform).
//     __device__ void store(const AlzTileArgs&, long long r, long long T);
//   };
//   CoreArgs::channel(pos): bank channel handled by grid position pos = blockIdx.x.
template <class Core, class CoreArgs>
__device__ __forceinline__ void alz_run_warp(const AlzTileArgs& a, const CoreArgs& ca, float* smem) {
  const int lane = threadIdx.x;
  const int c_local = blockIdx.x;              // CTA-uniform: coefficients go to uniform registers
  const int c = ca.channel(c_local);           // the plan orders positions so that precision tiers interleave
  const long long s0 = (long long)blockIdx.y * 32;
  const long long s = s0 + lane;
  const bool valid = s < a.S;
  const long long r = (long long)c * a.Stot + (valid ? s : a.S - 1);   // stream-fastest: coalesced state access

  Core core;
  core.load(a, ca, r, c_local, valid);

  const long long ntiles = (a.T + ALZ_TT - 1) / ALZ_TT;
  const long long nfull = a.T / ALZ_TT;
  const bool full_group = s0 + 32 <= a.S;
  const bool lean_in = a.vec_in && full_group;
  const bool lean_out = a.vec_out && full_group;
  const int sub = lane >> 3, col = (lane & 7) << 2;
  float* const myrow0 = smem + lane * ALZ_PITCH;
  // rows of this stream group in x and y (virtual streams: consecutive chunks of ONE real stream, vP % 32 == 0)
  const float* const xg = a.vP > 0 ? a.x + (s0 / a.vP) * a.xs + (s0 % a.vP) * a.T : a.x + s0 * a.xs;
  const long long xstr = a.vP > 0 ? a.T : a.xs;
  float* const yg = (a.vP > 0 ? a.y + (s0 / a.vP) * a.ysS + (s0 % a.vP) * a.T : a.y + s0 * a.ysS) + c * a.ys;
  const long long ystr = a.vP > 0 ? a.T : a.ysS;
  const long long ystep = 4ll * ystr;

  // prologue: tiles 0 and 1 in flight
  alz_issue_tile(a, smem, xg, xstr, s0, 0, lane, lean_in && nfull > 0);
  alz_cp_commit();
  if (ntiles > 1) alz_issue_tile(a, smem + 32 * ALZ_PITCH, xg, xstr, s0, ALZ_TT, lane, lean_in && nfull > 1);
  alz_cp_commit();

  for (long long i = 0; i < ntiles; ++i) {
    const long long t0 = i * ALZ_TT;
    float* const buf = smem + (i & 1) * (32 * ALZ_PITCH);
    alz_cp_wait<1>();   // every iteration commits exactly one group, so tile i has landed
    __syncwarp();
    const int nvalid = i < nfull ? ALZ_TT : (int)(a.T - t0);
    core.tile(myrow0 + (i & 1) * (32 * ALZ_PITCH), 0, nvalid, t0);
    __syncwarp();

    if (a.y == nullptr) {
      // ALZ_EXP & 2 / zero-state pass of the time-parallel evaluation: only the final states are wanted
    } else if (lean_out && i < nfull) {
      float* dst = yg + sub * ystr + t0 + col;
      const float* src = buf + sub * ALZ_PITCH + col;
#pragma unroll
      for (int it = 0; it < 8; ++it) {
        alz_st_v4(dst, *reinterpret_cast<const float4*>(src));
        dst += ystep;
        src += 4 * ALZ_PITCH;
      }
    } else {
#pragma unroll 1
      for (int it = 0; it < 8; ++it) {
        const int row = it * 4 + sub;
        if (s0 + row < a.S && col < nvalid) {
          const float4 v = *reinterpret_cast<const float4*>(buf + row * ALZ_PITCH + col);
          float* dst = yg + row * ystr + t0 + col;
          if (a.vec_out && col + 4 <= nvalid) {
            alz_st_v4(dst, v);
          } else {
            dst[0] = v.x;
            if (col + 1 < nvalid) dst[1] = v.y;
            if (col + 2 < nvalid) dst[2] = v.z;
            if (col + 3 < nvalid) dst[3] = v.w;
          }
        }
      }
    }
    __syncwarp();   // the buffer has been read by every lane: refill it with tile i+2
    if (i + 2 < ntiles) alz_issue_tile(a, buf, xg, xstr, s0, t0 + 2 * ALZ_TT, lane, lean_in && i + 2 < nfull);
    alz_cp_commit();
  }
  alz_cp_wait<0>();
  if (valid) core.store(a, r, a.T);
}
