// store_bench.cu -- micro-benchmark of write-only access patterns on one GPU (experiment
// aid for the fill kernel; not part of the product).  Build+run on the GPU box:
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o store_bench scripts/store_bench.cu && ./store_bench
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>
#include <vector>

#define CK(x) do { cudaError_t e = (x); if (e != cudaSuccess) { printf("CUDA error %s at %d\n", cudaGetErrorString(e), __LINE__); return 1; } } while (0)

template <int ST> __device__ __forceinline__ void st16(void* p, uint4 v) {
  if (ST == 0) asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  else if (ST == 1) asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
  else asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// contiguous range per CTA
template <int ST, int U> __global__ void k_range(uint4* dst, uint64_t n, uint32_t salt) {
  uint64_t lo = n * blockIdx.x / gridDim.x, hi = n * (blockIdx.x + 1ull) / gridDim.x;
  uint4 v = make_uint4(salt, threadIdx.x, blockIdx.x, 7);
  uint64_t i = lo + threadIdx.x;
  for (; i + (U - 1) * blockDim.x < hi; i += U * blockDim.x) {
#pragma unroll
    for (int k = 0; k < U; ++k) st16<ST>(dst + i + k * blockDim.x, v);
  }
  for (; i < hi; i += blockDim.x) st16<ST>(dst + i, v);
}
// grid-stride (interleaved tiles)
template <int ST, int U> __global__ void k_stride(uint4* dst, uint64_t n, uint32_t salt) {
  uint4 v = make_uint4(salt, threadIdx.x, blockIdx.x, 7);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (; i + (U - 1) * stride < n; i += U * stride) {
#pragma unroll
    for (int k = 0; k < U; ++k) st16<ST>(dst + i + k * stride, v);
  }
  for (; i < n; i += stride) st16<ST>(dst + i, v);
}
// interleaved tiles of TILE uint4 per CTA visit, consecutive inside the tile
template <int ST, int TILE> __global__ void k_tile(uint4* dst, uint64_t n, uint32_t salt) {
  uint4 v = make_uint4(salt, threadIdx.x, blockIdx.x, 7);
  for (uint64_t t = (uint64_t)blockIdx.x * TILE; t < n; t += (uint64_t)gridDim.x * TILE) {
#pragma unroll
    for (int k = 0; k < TILE; k += 256) {
      uint64_t i = t + k + threadIdx.x;
      if (i < n) st16<ST>(dst + i, v);
    }
  }
}
// each thread writes 2 consecutive uint4 (32 B)
template <int ST> __global__ void k_pair(uint4* dst, uint64_t n, uint32_t salt) {
  uint4 v = make_uint4(salt, threadIdx.x, blockIdx.x, 7);
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x * 2;
  for (uint64_t i = ((uint64_t)blockIdx.x * blockDim.x + threadIdx.x) * 2; i + 1 < n; i += stride) {
    st16<ST>(dst + i, v);
    st16<ST>(dst + i + 1, v);
  }
}

template <typename F> float time_it(F launch, cudaStream_t s, int reps, int sets) {
  cudaGraph_t g; cudaGraphExec_t ge;
  cudaStreamBeginCapture(s, cudaStreamCaptureModeRelaxed);
  for (int r = 0; r < reps; ++r) for (int k = 0; k < sets; ++k) launch(k);
  cudaStreamEndCapture(s, &g);
  cudaGraphInstantiate(&ge, g, 0);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (int i = 0; i < 3; ++i) cudaGraphLaunch(ge, s);
  cudaStreamSynchronize(s);
  cudaEventRecord(a, s);
  const int iters = 20;
  for (int i = 0; i < iters; ++i) cudaGraphLaunch(ge, s);
  cudaEventRecord(b, s);
  cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  return ms / (iters * reps * sets);
}

int main() {
  int sms = 0;
  CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
  const uint64_t small = 38535168, total = 4 * small;
  uint4* buf; CK(cudaMalloc(&buf, total));
  cudaStream_t s; CK(cudaStreamCreate(&s));
  struct Case { const char* name; uint64_t bytes; int sets; };
  Case cases[2] = {{"38.5MB x4 sets", small, 4}, {"154MB", total, 1}};
  for (auto& c : cases) {
    const uint64_t n = c.bytes / 16;
    printf("== %s\n", c.name);
    float ms = time_it([&](int k) { cudaMemsetAsync((char*)buf + (c.sets > 1 ? k * small : 0), 0, c.bytes, s); }, s, 4, c.sets);
    printf("%-40s %8.2f us %8.0f GB/s\n", "cudaMemsetAsync", ms * 1e3, c.bytes / ms / 1e6);
    int grids[] = {sms * 2, sms * 4, sms * 6, sms * 8, sms * 16, sms * 32};
    for (int g : grids) {
      char nm[64];
#define RUN(label, kern) { ms = time_it([&](int k) { kern<<<g, 256, 0, s>>>(buf + (c.sets > 1 ? k * (small / 16) : 0), n, k); }, s, 4, c.sets); \
        snprintf(nm, sizeof nm, "%s grid=%d", label, g); printf("%-40s %8.2f us %8.0f GB/s\n", nm, ms * 1e3, c.bytes / ms / 1e6); }
      RUN("range cs u2", (k_range<0, 2>));
      RUN("range plain u2", (k_range<1, 2>));
      RUN("stride cs u1", (k_stride<0, 1>));
      RUN("stride cs u4", (k_stride<0, 4>));
      RUN("stride plain u4", (k_stride<1, 4>));
      RUN("stride noalloc u4", (k_stride<2, 4>));
      RUN("tile1024 cs", (k_tile<0, 1024>));
      RUN("tile4096 cs", (k_tile<0, 4096>));
      RUN("pair cs", (k_pair<0>));
    }
  }
  return 0;
}
