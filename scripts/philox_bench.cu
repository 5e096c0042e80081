// philox_bench.cu -- how fast can an SM run Philox4x32-10?  (experiment aid, not product)
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o philox_bench scripts/philox_bench.cu && ./philox_bench
#include <cuda_runtime.h>
#include <cstdio>
#include <cstdint>

struct RK { uint32_t k[20]; };
static int g_sms = 0;        // SMs of the device (main)
static double g_clock_hz = 0;  // its maximum SM clock

template <int MODE>
__device__ __forceinline__ void round1(uint32_t& c0, uint32_t& c1, uint32_t& c2, uint32_t& c3, uint32_t k0, uint32_t k1) {
  uint32_t hi0, lo0, hi1, lo1;
  if (MODE == 0) {  // 32x32->64 (IMAD.WIDE)
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    hi0 = p0 >> 32; lo0 = (uint32_t)p0; hi1 = p1 >> 32; lo1 = (uint32_t)p1;
  } else {          // separate hi / lo multiplies
    hi0 = __umulhi(0xD2511F53u, c0); lo0 = 0xD2511F53u * c0;
    hi1 = __umulhi(0xCD9E8D57u, c2); lo1 = 0xCD9E8D57u * c2;
  }
  const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
  c1 = lo1; c3 = lo0; c0 = n0; c2 = n2;
}

template <int MODE, int ILP, int STORE>
__global__ void __launch_bounds__(256) k_philox(uint4* out, uint32_t iters, const RK rk) {
  uint32_t c[ILP][4];
#pragma unroll
  for (int i = 0; i < ILP; ++i) { c[i][0] = threadIdx.x + i * 977; c[i][1] = blockIdx.x; c[i][2] = 3 * i; c[i][3] = 7; }
  uint4 acc = make_uint4(0, 0, 0, 0);
  uint4* dst = out + (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (uint32_t it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < ILP; ++i) { c[i][0] += it; }
#pragma unroll
    for (int r = 0; r < 10; ++r) {
#pragma unroll
      for (int i = 0; i < ILP; ++i) round1<MODE>(c[i][0], c[i][1], c[i][2], c[i][3], rk.k[2 * r], rk.k[2 * r + 1]);
    }
    if (STORE) {
#pragma unroll
      for (int i = 0; i < ILP; ++i) {
        uint4 v = make_uint4(__float_as_uint(__uint_as_float(0x3F800000u | (c[i][0] >> 9)) - 1.0f), __float_as_uint(__uint_as_float(0x3F800000u | (c[i][1] >> 9)) - 1.0f),
                             __float_as_uint(__uint_as_float(0x3F800000u | (c[i][2] >> 9)) - 1.0f), __float_as_uint(__uint_as_float(0x3F800000u | (c[i][3] >> 9)) - 1.0f));
        asm volatile("st.global.cs.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(dst + ((size_t)it * ILP + i) * stride), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
      }
    } else {
#pragma unroll
      for (int i = 0; i < ILP; ++i) { acc.x ^= c[i][0]; acc.y ^= c[i][1]; acc.z ^= c[i][2]; acc.w ^= c[i][3]; }
    }
  }
  if (!STORE && acc.x == 0x12345678u) *dst = acc;
}

template <int MODE, int ILP, int STORE>
void run(const char* name, uint4* buf, int ctas_per_sm, uint32_t iters) {
  RK rk; for (int i = 0; i < 20; ++i) rk.k[i] = 0x9E3779B9u * (i + 1);
  const int grid = g_sms * ctas_per_sm;
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  k_philox<MODE, ILP, STORE><<<grid, 256>>>(buf, iters, rk);
  cudaDeviceSynchronize();
  cudaEventRecord(a);
  k_philox<MODE, ILP, STORE><<<grid, 256>>>(buf, iters, rk);
  cudaEventRecord(b); cudaEventSynchronize(b);
  float ms; cudaEventElapsedTime(&ms, a, b);
  const double calls = (double)grid * 256 * iters * ILP;        // thread-calls
  const double warp_calls_per_smsp = calls / 32 / (g_sms * 4.0);
  const double cycles = ms * 1e-3 * g_clock_hz;
  printf("%-44s ctas/sm=%d  %8.3f ms  %6.1f cycles/warp-call/SMSP  -> %6.0f GB/s of 16 B groups%s\n", name, ctas_per_sm, ms,
         cycles / warp_calls_per_smsp, calls * 16 / (ms * 1e-3) / 1e9, STORE ? " (stored)" : "");
}

int main() {
  int clock_khz = 0;
  cudaDeviceGetAttribute(&g_sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceGetAttribute(&clock_khz, cudaDevAttrClockRate, 0);
  g_clock_hz = clock_khz * 1e3;
  uint4* buf; cudaMalloc(&buf, (size_t)1 << 30);
  for (int cps : {2, 4, 6, 8}) {
    run<0, 1, 0>("imad.wide ilp1 compute only", buf, cps, 2000);
    run<0, 2, 0>("imad.wide ilp2 compute only", buf, cps, 1000);
    run<0, 4, 0>("imad.wide ilp4 compute only", buf, cps, 500);
    run<1, 2, 0>("mulhi+mullo ilp2 compute only", buf, cps, 1000);
    run<1, 4, 0>("mulhi+mullo ilp4 compute only", buf, cps, 500);
  }
  // with stores: grid*256*iters*ILP*16 bytes <= 1 GiB
  for (int cps : {3, 4, 6, 8}) {
    run<0, 2, 1>("imad.wide ilp2 + fp32 convert + store", buf, cps, 80);
    run<0, 4, 1>("imad.wide ilp4 + fp32 convert + store", buf, cps, 40);
  }
  return 0;
}
