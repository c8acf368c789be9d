// Micro-benchmark: what is the H100's achievable HBM bandwidth for a WRITE-dominated
// stream (the filterbank writes 256 B for every 4 B it reads), as opposed to the
// read+write copy that MEASURED_PEAKS.json's hbm_gbs is defined on?
//   fill_seq      : grid-stride 16-byte stores over one contiguous 16 GiB buffer
//   fill_rows<L>  : the kernel's pattern: each warp owns 32 rows (row stride 64 KiB) and
//                   advances all of them L bytes at a time (L = 128, 256, 512), 16-byte
//                   stores, whole 128-byte lines
//   copy          : read + write (same bytes each way), for the copy-peak cross-check
//   read          : pure read (sum reduction)
// Each variant is timed with CUDA events over several repetitions on >= 8 GiB, far
// beyond the 50 MB L2.
#include <cstdio>
#include <cstdlib>
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
  return 0;
}
