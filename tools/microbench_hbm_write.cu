// Micro-benchmark: what is the H100's achievable HBM bandwidth for a WRITE-dominated
// stream (the filterbank writes 256 B for every 4 B it reads), as opposed to the
// read+write copy that MEASURED_PEAKS.json's hbm_gbs is defined on?
//   fill_seq      : grid-stride 16-byte stores over one contiguous 16 GiB buffer
//   fill_rows<L>  : the kernel's pattern: each warp owns 32 rows (row stride 64 KiB) and
//                   advances all of them L bytes at a time (L = 128, 256, 512), 16-byte
//                   stores, whole 128-byte lines
//   copy          : read + write (same bytes each way), for the copy-peak cross-check
//   read          : pure read (sum reduction)
//   bank_*        : the bank's own store stream: y[S][C][T] at S = 4096, C = 64, T = 16384, one-warp CTAs that each own
//                   (channel, 32 streams) -- 32 rows 4 MB apart -- with the bank's 16 KB of tile buffers (13 CTAs per
//                   SM), writing every row in 512-byte pieces (groups of 4 tiles) with an evict-first L2 hint:
//     bank_tma      (a): the group leaves as 4 TMA box stores (cp.async.bulk.tensor.4d, 32 rows x 128 B each), one
//                        commit, and cp.async.bulk.wait_group.read 0 before the buffers are written again;
//     bank_vec      (b): the group leaves as 32 st.global.v4 instructions, one per row (lane l: tile l >> 3, 16-byte
//                        chunk l & 7, the 128-byte swizzle undone on the shared-memory read);
//     *_rd     (a') (b'): the same, with the bank's input stream: every group first reads its 4 input tiles (32 rows
//                        x 512 B of x[S][T], 268 MB, evict-last), which the 64 channel CTAs of a stream group share in L2
// Each variant is timed with CUDA events over several repetitions on >= 8 GiB, far
// beyond the 50 MB L2.
#include <cstdio>
#include <cstdlib>
#include <cuda.h>
#include <cuda_runtime.h>
#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s line %d\n", cudaGetErrorString(e), __LINE__); exit(1);} } while (0)

template <int MODE>  // 0 default, 1 .cs, 2 .wt
__device__ __forceinline__ void st16(float4* p, float4 v) {
  if (MODE == 0) *p = v;
  else if (MODE == 1) asm volatile("st.global.cs.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
  else asm volatile("st.global.wt.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}

template <int MODE>
__global__ void fill_seq(float4* p, size_t n16, float v) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  const float4 val = make_float4(v, v, v, v);
  for (; i < n16; i += stride) st16<MODE>(p + i, val);
}

// rows of `row_floats` floats; warp w owns rows [32w, 32w+32); per step it writes L bytes of each row
template <int L, int MODE>
__global__ void fill_rows(float* p, long long nrows, long long row_floats, float v) {
  const int lane = threadIdx.x & 31;
  const long long warp = ((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const long long r0 = warp * 32;
  if (r0 >= nrows) return;
  constexpr int LANES_PER_ROW = L / 16;         // lanes covering one L-byte segment
  constexpr int ROWS_PER_INSTR = 32 / LANES_PER_ROW;
  const int sub = lane / LANES_PER_ROW, col = (lane % LANES_PER_ROW) * 4;
  const float4 val = make_float4(v, v, v, v);
  for (long long t0 = 0; t0 < row_floats; t0 += L / 4) {
#pragma unroll
    for (int it = 0; it < 32 / ROWS_PER_INSTR; ++it) {
      const long long row = r0 + it * ROWS_PER_INSTR + sub;
      st16<MODE>(reinterpret_cast<float4*>(p + row * row_floats + t0 + col), val);
    }
  }
}

__global__ void copy_k(const float4* __restrict__ a, float4* __restrict__ b, size_t n16) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n16; i += stride) b[i] = a[i];
}
__global__ void read_k(const float4* __restrict__ a, float* out, size_t n16) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  float s = 0.f;
  for (; i < n16; i += stride) { float4 v = a[i]; s += v.x + v.y + v.z + v.w; }
  if (s == 123.456f) out[0] = s;
}

// ---- the bank's store geometry ------------------------------------------------------------------------------------
static const int kS = 4096, kC = 64, kT = 16384, kGroupTiles = 4;
static const size_t kBankSmem = kGroupTiles * 4096 + 32;   // the bank kernel's tiles + mbarriers (13 CTAs per SM)

__device__ __forceinline__ unsigned long long pol_evict_first() {
  unsigned long long p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ unsigned long long pol_evict_last() {
  unsigned long long p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}

// MODE 0: TMA box stores (a); 1: warp-wide vector stores (b).  READ: the group's input tiles are read first.
template <int MODE, bool READ>
__global__ void __launch_bounds__(32) bank_fill(const __grid_constant__ CUtensorMap tmy, float* y, const float* x, float* sink) {
  extern __shared__ __align__(1024) unsigned char smem[];
  const int lane = threadIdx.x, c = blockIdx.x;
  const long long s0 = (long long)blockIdx.y * 32;
  const unsigned long long st_pol = pol_evict_first(), ld_pol = pol_evict_last();
  const unsigned tile0 = (unsigned)__cvta_generic_to_shared(smem);
  float acc = 0.f;
  for (int t0 = 0; t0 < kT; t0 += 32 * kGroupTiles) {
    if (MODE == 0 && t0 > 0 && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
    __syncwarp();
    if (READ) {   // one row's 512 B of the group per instruction, as the TMA loads of the bank bring them
#pragma unroll 4
      for (int r = 0; r < 32; ++r) {
        const float* p = x + (s0 + r) * kT + t0 + lane * 4;
        float4 v;
        asm volatile("ld.global.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                     : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(ld_pol));
        acc += v.x + v.y + v.z + v.w;
      }
    }
    // the filtered tiles: each lane writes its own row of every tile (STS.128, swizzled as the bank does)
    for (int j = 0; j < kGroupTiles; ++j)
#pragma unroll
      for (int k = 0; k < 8; ++k)
        *reinterpret_cast<float4*>(smem + j * 4096 + lane * 128 + ((k ^ (lane & 7)) << 4)) = make_float4(acc, t0, j, k);
    if (MODE == 0) {
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      __syncwarp();
      if (lane == 0) {
        for (int j = 0; j < kGroupTiles; ++j)
          asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group.L2::cache_hint [%0, {%1, %2, %3, %4}], [%5], %6;"
                       ::"l"(&tmy), "r"(t0 + 32 * j), "r"(c), "r"((int)s0), "r"(0), "r"(tile0 + 4096 * j), "l"(st_pol) : "memory");
        asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      }
    } else {
      __syncwarp();
      const int j = lane >> 3, k = lane & 7;
      float* dst = y + (s0 * kC + c) * (long long)kT + t0 + j * 32 + k * 4;
#pragma unroll 8
      for (int r = 0; r < 32; ++r) {
        const float4 v = *reinterpret_cast<const float4*>(smem + j * 4096 + r * 128 + ((k ^ (r & 7)) << 4));
        asm volatile("st.global.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
                     ::"l"(dst + (long long)r * kC * kT), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(st_pol) : "memory");
      }
    }
  }
  if (MODE == 0 && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  if (acc == 123.456f) sink[0] = acc;
}

typedef CUresult (*encode_fn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                              const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                              CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int main() {
  const size_t bytes = 16ull << 30;
  float* buf; CK(cudaMalloc(&buf, bytes));
  float* buf2; CK(cudaMalloc(&buf2, bytes / 2));
  float* d_out; CK(cudaMalloc(&d_out, 4));
  CK(cudaMemset(buf, 0, bytes));
  cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
  cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
  const int nsm = p.multiProcessorCount;
#define TIME(name, bytes_moved, ...) do { \
    __VA_ARGS__; CK(cudaDeviceSynchronize()); float best = 1e30f; \
    for (int r = 0; r < 4; ++r) { CK(cudaEventRecord(e0)); __VA_ARGS__; CK(cudaEventRecord(e1)); CK(cudaDeviceSynchronize()); \
      float ms; CK(cudaEventElapsedTime(&ms, e0, e1)); if (ms < best) best = ms; } \
    CK(cudaGetLastError()); \
    printf("%-34s %8.3f ms  %8.1f GB/s\n", name, best, (double)(bytes_moved) / best / 1e6); } while (0)
  const size_t n16 = bytes / 16;
  TIME("cudaMemset 16 GiB", bytes, CK(cudaMemsetAsync(buf, 1, bytes)));
  TIME("fill_seq default", bytes, (fill_seq<0><<<nsm * 16, 512>>>((float4*)buf, n16, 1.f)));
  TIME("fill_seq .cs", bytes, (fill_seq<1><<<nsm * 16, 512>>>((float4*)buf, n16, 1.f)));
  TIME("fill_seq .wt", bytes, (fill_seq<2><<<nsm * 16, 512>>>((float4*)buf, n16, 1.f)));
  // the kernel's geometry: 262144 rows of 16384 floats = 16 GiB
  const long long nrows = 262144, rowf = 16384;
  const int blocks = (int)(nrows / 32 / 4);
  TIME("fill_rows L=128 default", bytes, (fill_rows<128, 0><<<blocks, 128>>>(buf, nrows, rowf, 2.f)));
  TIME("fill_rows L=128 .cs", bytes, (fill_rows<128, 1><<<blocks, 128>>>(buf, nrows, rowf, 2.f)));
  TIME("fill_rows L=256 .cs", bytes, (fill_rows<256, 1><<<blocks, 128>>>(buf, nrows, rowf, 2.f)));
  TIME("fill_rows L=512 .cs", bytes, (fill_rows<512, 1><<<blocks, 128>>>(buf, nrows, rowf, 2.f)));
  TIME("fill_rows L=512 default", bytes, (fill_rows<512, 0><<<blocks, 128>>>(buf, nrows, rowf, 2.f)));
  TIME("copy 8 GiB -> 8 GiB (r+w bytes)", bytes, (copy_k<<<nsm * 16, 512>>>((const float4*)buf, (float4*)buf2, n16 / 2)));
  TIME("cudaMemcpy D2D 8 GiB (r+w bytes)", bytes, CK(cudaMemcpyAsync(buf2, buf, bytes / 2, cudaMemcpyDeviceToDevice)));
  TIME("read 16 GiB", bytes, (read_k<<<nsm * 16, 512>>>((const float4*)buf, d_out, n16)));

  // the bank's store stream (see the top of the file)
  CK(cudaFree(buf)); CK(cudaFree(buf2));
  const size_t ybytes = (size_t)kS * kC * kT * 4, xbytes = (size_t)kS * kT * 4;
  float *y, *x;
  CK(cudaMalloc(&y, ybytes)); CK(cudaMalloc(&x, xbytes));
  CK(cudaMemset(y, 0, ybytes)); CK(cudaMemset(x, 0, xbytes));
  void* fn = nullptr; cudaDriverEntryPointQueryResult q;
  CK(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &q));
  if (q != cudaDriverEntryPointSuccess || !fn) { printf("no cuTensorMapEncodeTiled\n"); return 1; }
  CUtensorMap tmy;   // y as (T, C, S, 1), boxes of 32 samples x 1 channel x 32 streams: the bank kernel's output map
  const cuuint64_t dims[4] = {(cuuint64_t)kT, (cuuint64_t)kC, (cuuint64_t)kS, 1};
  const cuuint64_t strides[3] = {(cuuint64_t)kT * 4, (cuuint64_t)kC * kT * 4, (cuuint64_t)kC * kT * 4};
  const cuuint32_t box[4] = {32, 1, 32, 1}, estr[4] = {1, 1, 1, 1};
  if (((encode_fn)fn)(&tmy, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, y, dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                      CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS) {
    printf("tensor map encode failed\n"); return 1;
  }
  const void* kerns[4] = {(const void*)bank_fill<0, false>, (const void*)bank_fill<1, false>, (const void*)bank_fill<0, true>,
                          (const void*)bank_fill<1, true>};
  const char* names[4] = {"bank_tma (a)", "bank_vec (b)", "bank_tma_rd (a')", "bank_vec_rd (b')"};
  for (int v = 0; v < 4; ++v) {
    int per_sm = 0;
    CK(cudaFuncSetAttribute(kerns[v], cudaFuncAttributePreferredSharedMemoryCarveout, cudaSharedmemCarveoutMaxShared));
    CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kerns[v], 32, kBankSmem));
    char label[96];
    snprintf(label, sizeof label, "%s %d/SM", names[v], per_sm);
    void* args[4] = {(void*)&tmy, (void*)&y, (void*)&x, (void*)&d_out};
    TIME(label, ybytes, CK(cudaLaunchKernel(kerns[v], dim3(kC, kS / 32), dim3(32), args, kBankSmem, 0)));
  }
  return 0;
}
