// alz_lane_tma.cuh -- the "lane = stream" engine with TMA tile movement (sm_90a).
//
// Same decomposition as alz_lane.cuh (CTA = warp = (channel, 32 streams), tiles of 32
// samples filtered in place), but the tile is moved by the Tensor Memory Accelerator:
//   * load : ONE cp.async.bulk.tensor.2d per tile (box 32 samples x 32 streams of x[S][T]),
//            completion on an mbarrier (complete_tx), issued by lane 0;
//   * store: ONE cp.async.bulk.tensor.4d per tile (box 32 samples x 1 channel x 32 streams of
//            y[S][C][T]) straight from the same shared buffer; or, for tile groups of 4 (AlzTileArgs::vec_store),
//            32 warp-wide st.global.v4 per group, each one row's 512 contiguous bytes.
// The shared tile is dense [32 rows][128 B] with the hardware 128-byte swizzle (16-byte chunk
// index XOR row & 7), so the per-lane row accesses (LDS.128 / STS.128, lane = row) are bank
// conflict free without padding, and ragged edges (S % 32, T % 32) are handled by the TMA's
// out-of-bounds zero fill / store clipping: no predicated copy loops, no address arithmetic
// in the warp, ~150 instructions per tile less than the cp.async engine.
// Requires 16-byte aligned base pointers and row strides (else the cp.async engine is used).
#pragma once
#include <cuda.h>
#include "alz_lane.cuh"

#define ALZ_TMA_TILE_BYTES 4096                      // 32 rows x 128 B
#define ALZ_TMA_MAX_GROUP 4                          // tiles moved together (AlzTileArgs::paired)
#define ALZ_TMA_SMEM_FOR(ng) (((ng) < 2 ? 2 : (ng)) * ALZ_TMA_TILE_BYTES + 8 * ALZ_TMA_MAX_GROUP)   // tiles + mbarriers
#define ALZ_TMA_SMEM ALZ_TMA_SMEM_FOR(2)

__device__ __forceinline__ unsigned alz_smem_u32(const void* p) { return (unsigned)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void alz_mbar_init(unsigned mbar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(mbar), "r"(count) : "memory");
}
__device__ __forceinline__ void alz_mbar_expect_tx(unsigned mbar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(mbar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void alz_mbar_wait(unsigned mbar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "ALZ_WAIT:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra ALZ_DONE;\n"
      "bra ALZ_WAIT;\n"
      "ALZ_DONE:\n"
      "}\n" ::"r"(mbar), "r"(parity) : "memory");
}
__device__ __forceinline__ void alz_tma_load_2d(unsigned dst, const CUtensorMap* map, int c0, int c1, unsigned mbar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n"
               ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(mbar) : "memory");
}
__device__ __forceinline__ void alz_tma_store_3d(const CUtensorMap* map, int c0, int c1, int c2, unsigned src) {
  asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%1, %2, %3}], [%4];\n"
               ::"l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(src) : "memory");
}
__device__ __forceinline__ void alz_tma_store_2d(const CUtensorMap* map, int c0, int c1, unsigned src) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%1, %2}], [%3];\n"
               ::"l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(src) : "memory");
}
// L2 cache policies for the bank's tile traffic (createpolicy), handed to the TMA as .L2::cache_hint operands.
__device__ __forceinline__ unsigned long long alz_l2_evict_first() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;\n" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ unsigned long long alz_l2_evict_last() {
  unsigned long long pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;\n" : "=l"(pol));
  return pol;
}
__device__ __forceinline__ void alz_tma_load_3d(unsigned dst, const CUtensorMap* map, int c0, int c1, int c2, unsigned mbar,
                                                unsigned long long pol) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
               " [%0], [%1, {%2, %3, %4}], [%5], %6;\n"
               ::"r"(dst), "l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(mbar), "l"(pol) : "memory");
}
__device__ __forceinline__ void alz_tma_store_4d(const CUtensorMap* map, int c0, int c1, int c2, int c3, unsigned src,
                                                 unsigned long long pol) {
  asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%1, %2, %3, %4}], [%5], %6;\n"
               ::"l"(reinterpret_cast<unsigned long long>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(src), "l"(pol) : "memory");
}
__device__ __forceinline__ void alz_bulk_commit() { asm volatile("cp.async.bulk.commit_group;\n" ::: "memory"); }
__device__ __forceinline__ void alz_bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;\n" ::: "memory"); }
__device__ __forceinline__ void alz_bulk_wait0() { asm volatile("cp.async.bulk.wait_group 0;\n" ::: "memory"); }
__device__ __forceinline__ void alz_fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void alz_st_v4_hint(float* p, float4 v, unsigned long long pol) {
  asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1, %2, %3, %4}, %5;\n"
               ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// Consumers of a filtered tile.  AlzStoreY (default): the tile goes to y[S][C][T] by TMA.  AlzEnvelopePost: the tile is
// consumed in place -- rectifier / squarer, float64 one-pole lowpass (reference lazy_analysis.py:440-520: envelope.abs /
// .squared / .rms = lowpass(cutoff)(abs(sig)) ...), decimation -- and only every env_decim-th envelope value leaves the SM:
// the 256 B per input sample of the bank's output shrink to 256 / env_decim.
struct AlzStoreY {
  static constexpr bool active = false;
};
struct AlzEnvelopePost {
  static constexpr bool active = true;
  double env;
  float* out;          // next output slot of this lane's (stream, channel) row
  double* st;
  int left;            // samples until the next kept value
  // Sample t of this launch's row is sample pos = env_phase + tbeg + t of the caller's decimation grid; a value is kept
  // when pos % env_decim == env_decim - 1, at output index pos / env_decim.  Virtual streams (time-parallel evaluation):
  // `row` is the real stream and `chunk` the lane's chunk of it (the warp's TMA coordinates): its samples start chunk
  // chunk lengths (a.T each) into the real stream's grid.  32-bit arithmetic: fewer than 2^31 samples (TMA coordinates).
  __device__ __forceinline__ void load(const AlzTileArgs& a, int c, long long row, unsigned chunk, long long r, long long tbeg) {
    st = a.env_state + r;
    env = __ldcg(st);
    const unsigned pos = (unsigned)a.env_phase + (unsigned)tbeg + chunk * (unsigned)a.T;
    const unsigned q = pos / (unsigned)a.env_decim;
    out = a.env_out + (row * a.C + c) * a.env_es + q;
    // no-store mode: the countdown never reaches zero within a launch (< 2^31 samples), so the tile loop stays as is
    left = a.env_store ? a.env_decim - (int)(pos - q * (unsigned)a.env_decim) : 0x7fffffff;
  }
  __device__ __forceinline__ void tile(const AlzTileArgs& a, const float* row, int swz, int nvalid, bool valid) {
    for (int j = 0; j < nvalid; ++j) {
      const float y = row[(((j >> 2) ^ swz) << 2) | (j & 3)];
      const double r = a.env_mode == 0 ? (double)fabsf(y) : (double)y * (double)y;
      env = fma(a.env_R, env, a.env_g * r);
      if (--left == 0) {
        if (valid) *out =(float)(a.env_mode == 2 ? sqrt(env) : env);
        ++out;
        left = a.env_decim;
      }
    }
  }
  __device__ __forceinline__ void store() { *st = env; }
};

// VEC: the vector store path is compiled in, and taken where a.vec_store says so.  Instantiations that never run tile
// groups of 4 by default leave it out: its code costs the head-FIR instantiations, which spill, more spill traffic.
template <class Core, class Post = AlzStoreY, bool VEC = false, class CoreArgs>
__device__ __forceinline__ void alz_run_warp_tma(const AlzTileArgs& a, const CoreArgs& ca, const CUtensorMap* tmx,
                                                 const CUtensorMap* tmy, unsigned char* smem) {
  const int lane = threadIdx.x;
  const int c_local = blockIdx.x;              // CTA-uniform: coefficients go to uniform registers
  const int c = ca.channel(c_local);           // the plan orders positions so that precision tiers interleave
  int group = blockIdx.y, seg = 0;
  long long tbeg = 0, tlen = a.T;
  unsigned* flag = nullptr;
  if (a.nseg > 1) {
    // Ticket order = start order within the channel, so the CTA that owns the previous segment
    // of my (channel, group) is already running or done: the wait below cannot deadlock.
    unsigned ticket = 0;
    if (lane == 0) ticket = atomicAdd(a.sync + c_local, 1u);
    ticket = __shfl_sync(0xffffffffu, ticket, 0);
    seg = (int)(ticket / (unsigned)a.groups);
    group = (int)(ticket - (unsigned)seg * (unsigned)a.groups);
    tbeg = (long long)seg * a.seg_len;
    tlen = a.T - tbeg < a.seg_len ? a.T - tbeg : a.seg_len;
    flag = a.sync + gridDim.x + (size_t)c_local * a.groups + group;
    if (seg > 0) {
      unsigned done;
      do {
        asm volatile("ld.acquire.gpu.global.u32 %0, [%1];\n" : "=r"(done) : "l"(flag) : "memory");
      } while (done < (unsigned)seg);
    }
  }
  const long long s0 = (long long)group * 32;
  const long long s = s0 + lane;
  const bool valid = s < a.S;
  const long long r = (long long)c * a.Stot + (valid ? s : a.S - 1);   // stream-fastest: coalesced state access
  // TMA coordinates of this stream group, computed once (ONE code path in the tile loop: x is always a 3-D map, y a 4-D
  // map).  Real streams: x (t, stream, 0), y (t, channel, stream, 0).  Virtual streams (time-parallel evaluation): row v
  // is chunk v % vP of real stream v / vP: x (t, chunk, stream), y (t, chunk, channel, stream).
  int ld1 = (int)s0, ld2 = 0, st1 = c, st2 = (int)s0, st3 = 0;
  if (a.vP > 0) {
    ld2 = (int)(s0 / a.vP);
    ld1 = (int)(s0 - (long long)ld2 * a.vP);
    st1 = ld1; st2 = c; st3 = ld2;
  }

  const int NG = a.paired < 2 ? 1 : a.paired;   // tiles per group (1 = one tile at a time with a prefetch)
  const int nbuf = NG < 2 ? 2 : NG;
  const unsigned tile0 = alz_smem_u32(smem);
  const unsigned mbar0 = tile0 + nbuf * ALZ_TMA_TILE_BYTES;
  if (lane == 0) {
    for (int j = 0; j < nbuf; ++j) alz_mbar_init(mbar0 + 8 * j, 1);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  __syncwarp();

  Core core;
  core.load(a, ca, r, c_local, valid);
  Post post;
  if constexpr (Post::active) {
    if (a.vP > 0) post.load(a, c, ld2, (unsigned)(ld1 + lane), r, tbeg);   // lanes past S only feed the unused state
    else post.load(a, c, valid ? s : a.S - 1, 0u, r, tbeg);
  }

  const int ntiles = (int)((tlen + ALZ_TT - 1) / ALZ_TT);
  const int nfull = (int)(tlen / ALZ_TT);
  const int tb = (int)tbeg;
  const int swz = lane & 7;
  float* const myrow = reinterpret_cast<float*>(smem) + lane * 32;
  const bool tail_by_lanes = (a.T & 3) != 0 && nfull < ntiles;   // see below: the TMA clips at 16-byte granularity
  int last_buf = 0;

  // NG == 1: one tile at a time, the next one prefetched into the other buffer (latency-bound launches).
  // NG >= 2: tiles go in groups of NG (a power of two): all loads are issued together once the previous
  // group's stores have been read out of shared memory, the tiles are filtered as they land, and all
  // stores are issued back to back, so each output row receives NG * 128 contiguous bytes at (nearly)
  // the same time (HBM write efficiency grows with the piece length,
  // profiles/r01_microbench_hbm_write.txt).  The load of the next group is exposed to this warp; the
  // other resident warps hide it.
  const int lg = NG >= 4 ? 2 : (NG >= 2 ? 1 : 0);
  // L2 policy: every channel's warp of this stream group reads the same input tiles, at times that drift apart, while
  // the output stream (64 x the input bytes for a 64-channel bank) is never read again.  Output tiles are stored
  // evict-first and input tiles loaded evict-last, so the L2 gives up output lines first and a late reader still finds
  // its tile there instead of fetching it from HBM again (DESIGN.md section 3: measured on the H100).
  const bool vec = VEC && !Post::active && a.vec_store;   // host: tile groups of 4 only
  unsigned long long st_pol = 0, ld_pol = 0;
  if (lane == 0 || vec) st_pol = alz_l2_evict_first();
  if (lane == 0) ld_pol = alz_l2_evict_last();
  if (lane == 0 && NG == 1) {   // tile 0 in flight
    alz_mbar_expect_tx(mbar0, ALZ_TMA_TILE_BYTES);
    alz_tma_load_3d(tile0, tmx, tb, ld1, ld2, mbar0, ld_pol);
  }
  for (int i = 0; i < ntiles; ++i) {
    const int j = NG == 1 ? (i & 1) : (i & (NG - 1));   // buffer of tile i
    const int t0 = i * ALZ_TT;
    const bool skip_load = (a.exp & 1) && i >= NG;
    if (lane == 0 && !skip_load) {
      if (NG == 1) {
        if (i + 1 < ntiles) {
          // The other buffer was the source of the TMA store of tile i-1: wait until the store has
          // finished READING it (it was issued a whole barrier-wait ago, so this normally does not block).
          if (i >= 1) alz_bulk_wait_read0();
          alz_mbar_expect_tx(mbar0 + 8 * (j ^ 1), ALZ_TMA_TILE_BYTES);
          alz_tma_load_3d(tile0 + (j ^ 1) * ALZ_TMA_TILE_BYTES, tmx, tb + t0 + ALZ_TT, ld1, ld2, mbar0 + 8 * (j ^ 1), ld_pol);
        }
      } else if (j == 0) {
        if (i > 0 && !vec) alz_bulk_wait_read0();   // vector stores: the buffers were read out before the last __syncwarp
        const int n = ntiles - i < NG ? ntiles - i : NG;
        for (int jj = 0; jj < n; ++jj) {
          alz_mbar_expect_tx(mbar0 + 8 * jj, ALZ_TMA_TILE_BYTES);
          alz_tma_load_3d(tile0 + jj * ALZ_TMA_TILE_BYTES, tmx, tb + t0 + jj * ALZ_TT, ld1, ld2, mbar0 + 8 * jj, ld_pol);
        }
      }
    }
    if (!((a.exp & 1) && i >= (NG == 1 ? 2 : NG)))
      alz_mbar_wait(mbar0 + 8 * j, (NG == 1 ? (i >> 1) : (i >> lg)) & 1);   // tile i has landed (async proxy writes visible after the wait)
    const int nvalid = i < nfull ? ALZ_TT : (int)(tlen - t0);
    core.tile(myrow + j * (ALZ_TMA_TILE_BYTES / 4), swz, nvalid, t0);
    if constexpr (Post::active) post.tile(a, myrow + j * (ALZ_TMA_TILE_BYTES / 4), swz, nvalid, valid);
    alz_fence_async_smem();                          // my generic-proxy writes -> visible to the TMA store
    __syncwarp();
    const bool last = i + 1 == ntiles;
    if (vec) {
      if (!(a.exp & 2) && (j == NG - 1 || last)) {
        // The group's tiles 0..j leave row by row: one instruction writes row r's (j + 1) x 128 B, lane l carrying
        // 16-byte chunk l & 7 of tile l >> 3 (the 128-byte swizzle undone on the read).  A 512-byte piece is four
        // whole lines of one row, which HBM takes at the rate of a sequential fill (DESIGN.md section 3) where a
        // TMA box of 32 rows x 128 B does not.  Same clipping as the TMA store: rows past S, samples past the
        // segment, and the ragged last tile of a row length that is no multiple of 4 (stored after the loop).
        const int jt = lane >> 3, k = lane & 7;
        const int ncol = jt < j ? ALZ_TT : (jt == j && !(tail_by_lanes && last) ? nvalid : 0);
        if (4 * k < ncol) {
          const long long rows = a.S - s0 < 32 ? a.S - s0 : 32;
          float* dst = a.y + (a.vP > 0 ? ld2 * a.ysS + (long long)ld1 * a.T : s0 * a.ysS) + (long long)c * a.ys + tb + t0 -
                       (j - jt) * ALZ_TT + 4 * k;
          const long long ystr = a.vP > 0 ? a.T : a.ysS;   // virtual streams: the group's rows are consecutive chunks
          const unsigned char* src = smem + jt * ALZ_TMA_TILE_BYTES;
#pragma unroll 8
          for (int rr = 0; rr < rows; ++rr) {
            alz_st_v4_hint(dst, *reinterpret_cast<const float4*>(src + ((k ^ (rr & 7)) << 4)), st_pol);
            dst += ystr;
            src += 128;
          }
        }
        __syncwarp();   // every lane has read the group out: its buffers may be refilled
      }
    } else if (lane == 0 && !(a.exp & 2) && !Post::active) {
      if (NG == 1) {
        if (!(tail_by_lanes && last)) alz_tma_store_4d(tmy, tb + t0, st1, st2, st3, tile0 + j * ALZ_TMA_TILE_BYTES, st_pol);   // ragged last tile: stored after the loop
        alz_bulk_commit();
      } else if (j == NG - 1 || last) {
        for (int jj = 0; jj <= j; ++jj)
          if (!(tail_by_lanes && last && jj == j))
            alz_tma_store_4d(tmy, tb + t0 - (j - jj) * ALZ_TT, st1, st2, st3, tile0 + jj * ALZ_TMA_TILE_BYTES, st_pol);
        alz_bulk_commit();
      }
    }
    last_buf = j;
  }
  if (tail_by_lanes && valid && !Post::active) {
    // The TMA clips a box at 16-byte granularity: when n_samples is not a multiple of 4 the ragged
    // last tile is written by the lanes themselves (plain stores of the valid samples only).
    const int i = ntiles - 1, t0 = i * ALZ_TT, nvalid = (int)(tlen - t0);
    const float* src = myrow + last_buf * (ALZ_TMA_TILE_BYTES / 4);
    float* dst = a.y + s * a.ysS + (long long)c * a.ys + tbeg + t0;
    for (int j = 0; j < nvalid; ++j) dst[j] = src[(((j >> 2) ^ swz) << 2) | (j & 3)];
  }
  if (lane == 0 && !vec) alz_bulk_wait0();           // all output tiles are globally written before exit
  if (valid) core.store(a, r, tlen);
  if constexpr (Post::active) { if (valid) post.store(); }
  if (flag != nullptr && seg + 1 < a.nseg) {         // hand the state to the next segment
    __threadfence();
    __syncwarp();
    if (lane == 0) asm volatile("st.release.gpu.global.u32 [%0], %1;\n" ::"l"(flag), "r"((unsigned)(seg + 1)) : "memory");
  }
}
