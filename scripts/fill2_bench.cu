// fill2_bench.cu -- experiment aid (not product): candidate structures for the homogeneous
// fill launch (C2: 64 x FP32[3,224,224]; C3: 1 x FP16[128,3,224,224]) inside the
// Philox4x32-10 contract of client_b200/csrc/philox.cuh, and the launch mechanics around
// them (plain stream, programmatic dependent launch, graph chains, two streams).
//
//   nvcc -O3 -std=c++17 -lineinfo -gencode arch=compute_90a,code=sm_90a -o fill2_bench scripts/fill2_bench.cu
//   ./fill2_bench               (prints one line per variant x mechanism)
//
// Every variant is checked bit for bit against a host restatement of the contract before
// it is timed.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#define CK(x)                                                                      \
  do {                                                                             \
    cudaError_t e_ = (x);                                                          \
    if (e_ != cudaSuccess) {                                                       \
      printf("CUDA error %s at %s:%d\n", cudaGetErrorString(e_), __FILE__, __LINE__); \
      exit(1);                                                                     \
    }                                                                              \
  } while (0)

constexpr uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
constexpr int kMaxJobs = 64;

struct RK { uint32_t k[20]; };
struct JobTab {            // kernel parameter (constant bank): no global load before the first store
  uint64_t dst[kMaxJobs];
  uint64_t stream[kMaxJobs];
};
struct Launch {
  RK rk;
  uint64_t epoch;
  uint32_t njobs;
  uint32_t rows_per_job;    // rows of 256 groups (4 KiB)
  uint32_t ctas_per_job;    // job-split kernels
  uint32_t total_rows;
  uint32_t magic;           // floor(2^32 / rows_per_job) + 1
};

// ---------------------------------------------------------------- host restatement
static void philox_host(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)M0 * c0, p1 = (uint64_t)M1 * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1; c3 = (uint32_t)p0; c0 = n0; c2 = n2;
    k0 += W0; k1 += W1;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
static uint32_t host_f32(uint32_t w) {
  const uint32_t b = 0x3F800000u | (w >> 9);
  float f; memcpy(&f, &b, 4); f -= 1.0f;
  uint32_t o; memcpy(&o, &f, 4);
  return o;
}
static uint16_t host_f16_1(uint32_t x16) {  // (x16 >> 6) * 2^-10 as a half
  uint32_t m = x16 >> 6;
  if (m == 0) return 0;
  int p = 31 - __builtin_clz(m);
  return (uint16_t)(((p + 5) << 10) | ((m << (10 - p)) & 0x3FFu));
}
static uint32_t host_f16(uint32_t w) { return host_f16_1(w & 0xFFFFu) | ((uint32_t)host_f16_1(w >> 16) << 16); }

// ---------------------------------------------------------------- device pieces
__device__ __forceinline__ void st_cs_v4(void* p, uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(a), "r"(b), "r"(c), "r"(d) : "memory");
}
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

struct JobConst { uint32_t X, Y, Z, E; };
// Rounds 0 and 1 of Philox4x32-10 for counter (g, 0, s_lo, s_hi): everything that depends
// only on the stream is folded into four words (two of the twenty multiplies disappear).
__device__ __forceinline__ JobConst job_const(uint32_t s_lo, uint32_t s_hi, const RK& rk) {
  const uint64_t p1 = (uint64_t)M1 * s_lo;
  const uint32_t A = (uint32_t)(p1 >> 32), B = (uint32_t)p1;
  const uint32_t C0 = A ^ rk.k[0];                 // ^ g_hi (= 0)
  const uint64_t p0b = (uint64_t)M0 * C0;
  JobConst c;
  c.X = s_hi ^ rk.k[1];
  c.Y = B ^ rk.k[2];
  c.Z = (uint32_t)(p0b >> 32) ^ rk.k[3];
  c.E = (uint32_t)p0b;
  return c;
}
// p0 = M0 * g (64-bit), supplied by the caller (multiply or running sum)
__device__ __forceinline__ void philox_tail(uint64_t p0, const JobConst& jc, const RK& rk, uint32_t& o0, uint32_t& o1, uint32_t& o2, uint32_t& o3) {
  uint32_t c2 = (uint32_t)(p0 >> 32) ^ jc.X;
  const uint64_t p1b = (uint64_t)M1 * c2;
  uint32_t c0 = (uint32_t)(p1b >> 32) ^ jc.Y;
  uint32_t c1 = (uint32_t)p1b;
  c2 = (uint32_t)p0 ^ jc.Z;
  uint32_t c3 = jc.E;
#pragma unroll
  for (int r = 2; r < 10; ++r) {
    const uint64_t q0 = (uint64_t)M0 * c0, q1 = (uint64_t)M1 * c2;
    const uint32_t n0 = (uint32_t)(q1 >> 32) ^ c1 ^ rk.k[2 * r];
    const uint32_t n2 = (uint32_t)(q0 >> 32) ^ c3 ^ rk.k[2 * r + 1];
    c1 = (uint32_t)q1; c3 = (uint32_t)q0; c0 = n0; c2 = n2;
  }
  o0 = c0; o1 = c1; o2 = c2; o3 = c3;
}
__device__ __forceinline__ void philox_full(uint32_t g, uint32_t s_lo, uint32_t s_hi, const RK& rk, uint32_t& o0, uint32_t& o1, uint32_t& o2, uint32_t& o3) {
  uint32_t c0 = g, c1 = 0, c2 = s_lo, c3 = s_hi;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t q0 = (uint64_t)M0 * c0, q1 = (uint64_t)M1 * c2;
    const uint32_t n0 = (uint32_t)(q1 >> 32) ^ c1 ^ rk.k[2 * r];
    const uint32_t n2 = (uint32_t)(q0 >> 32) ^ c3 ^ rk.k[2 * r + 1];
    c1 = (uint32_t)q1; c3 = (uint32_t)q0; c0 = n0; c2 = n2;
  }
  o0 = c0; o1 = c1; o2 = c2; o3 = c3;
}

template <int DT>  // 0: fp32 unit interval, 1: fp16 unit interval
__device__ __forceinline__ uint32_t conv(uint32_t w) {
  if (DT == 0) {
    return __float_as_uint(__uint_as_float(__funnelshift_r(w, 0x7Fu, 9)) - 1.0f);
  } else {
    const uint32_t one_plus = 0x3C003C00u | ((w >> 6) & 0x03FF03FFu);
    uint32_t r;
    asm("sub.f16x2 %0, %1, %2;" : "=r"(r) : "r"(one_plus), "r"(0x3C003C00u));
    return r;
  }
}

// ---- KB: job-split rows.  CTA b: job b / cpj, part b % cpj; its rows part, part + cpj, ...
// Constants hoisted once per CTA.  ADD: p0 by running 64-bit sum instead of a multiply.
__device__ uint64_t g_dev_epoch = 7;
__constant__ uint64_t c_epoch[4] = {7, 7, 7, 7};
template <int DT, int THREADS, int U, int MINB, bool ADD, bool PDL, int MODE = 0>
__global__ void __launch_bounds__(THREADS, MINB) k_jobsplit(const __grid_constant__ JobTab tab, const __grid_constant__ Launch L) {
  uint64_t epoch = L.epoch;
  if (MODE & 2) epoch = epoch - 7 + *reinterpret_cast<volatile uint64_t*>(&g_dev_epoch);
  if (MODE & 4) epoch = epoch - 7 + c_epoch[1];
  if (MODE & 8) {
    uint64_t v;
    asm volatile("ld.global.nc.L1::evict_last.u64 %0, [%1];" : "=l"(v) : "l"(&g_dev_epoch));
    epoch = epoch - 7 + v;
  }
  if (PDL) pdl_launch_dependents();
  if (MODE & 16) epoch = epoch - 7 + *reinterpret_cast<volatile uint64_t*>(&g_dev_epoch);  // load AFTER the signal
  const uint32_t j = blockIdx.x / L.ctas_per_job;
  const uint32_t part = blockIdx.x - j * L.ctas_per_job;
  const uint64_t stream = tab.stream[j] + epoch;
  const JobConst jc = job_const((uint32_t)stream, (uint32_t)(stream >> 32), L.rk);
  const uint32_t groups = L.rows_per_job * 256u;      // groups of this job (tail rows handled by bound)
  const uint32_t stride = L.ctas_per_job * THREADS;   // groups between a thread's consecutive iterations
  uint32_t g = part * THREADS + threadIdx.x;
  uint8_t* p = reinterpret_cast<uint8_t*>(tab.dst[j]) + (uint64_t)g * 16u;
  uint64_t pstride = (uint64_t)stride * 16u;
  asm volatile("" : "+l"(pstride));  // opaque: pointer steps are IADD3 pairs on the alu pipe, not IMAD.WIDE
  uint64_t p0 = (uint64_t)M0 * g;
  const uint64_t p0step = (uint64_t)M0 * stride;
  for (; g + (U - 1) * stride < groups; g += U * stride) {
    uint32_t o[U][4];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      uint64_t q;
      if (ADD) { q = p0; p0 += p0step; } else { q = (uint64_t)M0 * (g + k * stride); }
      philox_tail(q, jc, L.rk, o[k][0], o[k][1], o[k][2], o[k][3]);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      st_cs_v4(p, conv<DT>(o[k][0]), conv<DT>(o[k][1]), conv<DT>(o[k][2]), conv<DT>(o[k][3]));
      p += pstride;
    }
  }
  for (; g < groups; g += stride) {
    uint32_t o0, o1, o2, o3;
    philox_tail((uint64_t)M0 * g, jc, L.rk, o0, o1, o2, o3);
    st_cs_v4(p, conv<DT>(o0), conv<DT>(o1), conv<DT>(o2), conv<DT>(o3));
    p += pstride;
  }
  if (MODE & 1) asm volatile("griddepcontrol.wait;" ::: "memory");
}

// ---- KA: global rows.  Row r = blockIdx.x + it * gridDim.x of the launch (all jobs back to
// back), one group per thread per row, U rows in flight; the job of a row is CTA-uniform.
template <int DT, int THREADS, int U, int MINB, bool HOIST, bool PDL>
__global__ void __launch_bounds__(THREADS, MINB) k_rows(const __grid_constant__ JobTab tab, const __grid_constant__ Launch L) {
  if (PDL) pdl_launch_dependents();
  constexpr uint32_t RPB = THREADS / 256u == 0 ? 1 : THREADS / 256u;  // THREADS is 256 here
  (void)RPB;
  const uint32_t G = gridDim.x;
  uint32_t r = blockIdx.x;
  auto one = [&](uint32_t row, uint32_t& a, uint32_t& b, uint32_t& c, uint32_t& d, uint8_t*& addr) {
    const uint32_t j = __umulhi(row, L.magic);
    const uint32_t lr = row - j * L.rows_per_job;
    const uint32_t g = lr * 256u + threadIdx.x;
    const uint64_t stream = tab.stream[j] + L.epoch;
    if (HOIST) {
      const JobConst jc = job_const((uint32_t)stream, (uint32_t)(stream >> 32), L.rk);
      philox_tail((uint64_t)M0 * g, jc, L.rk, a, b, c, d);
    } else {
      philox_full(g, (uint32_t)stream, (uint32_t)(stream >> 32), L.rk, a, b, c, d);
    }
    addr = reinterpret_cast<uint8_t*>(tab.dst[j]) + (uint64_t)g * 16u;
  };
  for (; r + (U - 1) * G < L.total_rows; r += U * G) {
    uint32_t o[U][4];
    uint8_t* a[U];
#pragma unroll
    for (int k = 0; k < U; ++k) one(r + k * G, o[k][0], o[k][1], o[k][2], o[k][3], a[k]);
#pragma unroll
    for (int k = 0; k < U; ++k) st_cs_v4(a[k], conv<DT>(o[k][0]), conv<DT>(o[k][1]), conv<DT>(o[k][2]), conv<DT>(o[k][3]));
  }
  for (; r < L.total_rows; r += G) {
    uint32_t o0, o1, o2, o3;
    uint8_t* a;
    one(r, o0, o1, o2, o3, a);
    st_cs_v4(a, conv<DT>(o0), conv<DT>(o1), conv<DT>(o2), conv<DT>(o3));
  }
}

// ---- KC: contiguous range per CTA inside its job (job-split, but each part is one block of
// consecutive rows instead of interleaved rows)
template <int DT, int THREADS, int U, int MINB, bool PDL>
__global__ void __launch_bounds__(THREADS, MINB) k_jobrange(const __grid_constant__ JobTab tab, const __grid_constant__ Launch L) {
  if (PDL) pdl_launch_dependents();
  const uint32_t j = blockIdx.x / L.ctas_per_job;
  const uint32_t part = blockIdx.x - j * L.ctas_per_job;
  const uint64_t stream = tab.stream[j] + L.epoch;
  const JobConst jc = job_const((uint32_t)stream, (uint32_t)(stream >> 32), L.rk);
  const uint32_t groups = L.rows_per_job * 256u;
  const uint32_t lo = (uint32_t)(((uint64_t)groups * part) / L.ctas_per_job);
  const uint32_t hi = (uint32_t)(((uint64_t)groups * (part + 1)) / L.ctas_per_job);
  uint32_t g = lo + threadIdx.x;
  uint8_t* p = reinterpret_cast<uint8_t*>(tab.dst[j]) + (uint64_t)g * 16u;
  for (; g + (U - 1) * THREADS < hi; g += U * THREADS) {
    uint32_t o[U][4];
#pragma unroll
    for (int k = 0; k < U; ++k) philox_tail((uint64_t)M0 * (g + k * THREADS), jc, L.rk, o[k][0], o[k][1], o[k][2], o[k][3]);
#pragma unroll
    for (int k = 0; k < U; ++k) {
      st_cs_v4(p, conv<DT>(o[k][0]), conv<DT>(o[k][1]), conv<DT>(o[k][2]), conv<DT>(o[k][3]));
      p += THREADS * 16;
    }
  }
  for (; g < hi; g += THREADS) {
    uint32_t o0, o1, o2, o3;
    philox_tail((uint64_t)M0 * g, jc, L.rk, o0, o1, o2, o3);
    st_cs_v4(p, conv<DT>(o0), conv<DT>(o1), conv<DT>(o2), conv<DT>(o3));
    p += THREADS * 16;
  }
}

// pure-store twin of k_jobsplit (what the same access pattern reaches with no arithmetic)
template <int THREADS, int U, bool PDL>
__global__ void __launch_bounds__(THREADS) k_store_only(const __grid_constant__ JobTab tab, const __grid_constant__ Launch L) {
  if (PDL) pdl_launch_dependents();
  const uint32_t j = blockIdx.x / L.ctas_per_job;
  const uint32_t part = blockIdx.x - j * L.ctas_per_job;
  const uint32_t groups = L.rows_per_job * 256u;
  const uint32_t stride = L.ctas_per_job * THREADS;
  uint32_t g = part * THREADS + threadIdx.x;
  uint8_t* p = reinterpret_cast<uint8_t*>(tab.dst[j]) + (uint64_t)g * 16u;
  const uint32_t v = (uint32_t)L.epoch;
  for (; g < groups; g += stride) {
    st_cs_v4(p, v, g, v, g);
    p += (uint64_t)stride * 16u;
  }
}

// ---------------------------------------------------------------- harness
typedef void (*KernelFn)(const JobTab, const Launch);
struct Variant {
  std::string name;
  KernelFn fn, fn_pdl;
  int threads;
  int dt;          // 0 fp32, 1 fp16, -1 store only
  int mode;        // 0 job-split grid (njobs * cpj), 1 global rows (grid = sms * per_sm)
  int per_sm;      // target CTAs per SM
};

static int g_sms = 0;  // set from the device in main
static double g_peak_gbs = 0;  // the device's theoretical DRAM bandwidth (memory clock x bus width, DDR), set in main
static uint8_t* g_buf = nullptr;
static const uint64_t kSlot = 602112, kSet = 64 * kSlot;
static RK g_rk;
static const uint64_t kSeed = 0x1234ABCD5678EF01ull;

static void make_launch(bool c3, int set, const Variant& v, JobTab& tab, Launch& L, int& grid) {
  memset(&tab, 0, sizeof(tab));
  L.rk = g_rk;
  L.epoch = 7;
  if (c3) {
    L.njobs = 1;
    tab.dst[0] = (uint64_t)(g_buf + set * kSet);
    tab.stream[0] = 1000 + set;
    L.rows_per_job = (uint32_t)(kSet / 4096);
  } else {
    L.njobs = 64;
    for (int k = 0; k < 64; ++k) {
      tab.dst[k] = (uint64_t)(g_buf + set * kSet + k * kSlot);
      tab.stream[k] = (uint64_t)k + 100 * set;
    }
    L.rows_per_job = (uint32_t)(kSlot / 4096);
  }
  L.total_rows = L.njobs * L.rows_per_job;
  L.magic = (uint32_t)((1ull << 32) / L.rows_per_job) + 1;
  const int target = g_sms * v.per_sm;
  if (v.mode == 0) {
    int cpj = target / (int)L.njobs;
    if (cpj < 1) cpj = 1;
    L.ctas_per_job = cpj;
    grid = cpj * L.njobs;
  } else {
    L.ctas_per_job = 1;
    grid = target;
  }
}

static bool verify(bool c3, int dt, int set) {
  std::vector<uint8_t> host(kSet);
  CK(cudaMemcpy(host.data(), g_buf + set * kSet, kSet, cudaMemcpyDeviceToHost));
  const uint32_t k0 = (uint32_t)kSeed, k1 = (uint32_t)(kSeed >> 32);
  const int njobs = c3 ? 1 : 64;
  const uint64_t jbytes = c3 ? kSet : kSlot;
  uint64_t bad = 0;
  for (int j = 0; j < njobs; ++j) {
    const uint64_t stream = (c3 ? 1000 + set : (uint64_t)j + 100 * set) + 7;
    const uint32_t* got = reinterpret_cast<const uint32_t*>(host.data() + j * jbytes);
    for (uint64_t g = 0; g < jbytes / 16; ++g) {
      uint32_t w[4];
      philox_host((uint32_t)g, 0, (uint32_t)stream, (uint32_t)(stream >> 32), k0, k1, w);
      for (int i = 0; i < 4; ++i) {
        const uint32_t e = dt == 0 ? host_f32(w[i]) : host_f16(w[i]);
        if (got[g * 4 + i] != e) {
          if (bad < 3) printf("   mismatch job %d group %llu word %d: got %08x want %08x\n", j, (unsigned long long)g, i, got[g * 4 + i], e);
          ++bad;
        }
      }
    }
  }
  return bad == 0;
}

static void launch_one(const Variant& v, bool pdl, const JobTab& tab, const Launch& L, int grid, cudaStream_t s) {
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3(grid);
  cfg.blockDim = dim3(v.threads);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  if (pdl) {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
  }
  CK(cudaLaunchKernelEx(&cfg, pdl ? v.fn_pdl : v.fn, tab, L));
}

// mechanisms: 0 plain stream, 1 PDL stream, 2 graph chain, 3 graph chain with PDL edges, 4 two streams
static double time_variant(const Variant& v, bool c3, int mech, int launches) {
  cudaStream_t s[2];
  CK(cudaStreamCreateWithFlags(&s[0], cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&s[1], cudaStreamNonBlocking));
  JobTab tab[4];
  Launch L[4];
  int grid[4];
  for (int i = 0; i < 4; ++i) make_launch(c3, i, v, tab[i], L[i], grid[i]);
  cudaEvent_t a, b, j1;
  CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b)); CK(cudaEventCreateWithFlags(&j1, cudaEventDisableTiming));
  float ms = 0;
  const bool pdl = (mech == 1 || mech == 3);
  if (mech == 2 || mech == 3) {
    cudaGraph_t g; cudaGraphExec_t ge;
    const int per_graph = 16;
    cudaError_t e = cudaStreamBeginCapture(s[0], cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
      for (int i = 0; i < per_graph; ++i) launch_one(v, pdl, tab[i & 3], L[i & 3], grid[i & 3], s[0]);
      e = cudaStreamEndCapture(s[0], &g);
    }
    if (e != cudaSuccess) { printf("   capture failed: %s\n", cudaGetErrorString(e)); cudaGetLastError(); return -1; }
    e = cudaGraphInstantiate(&ge, g, 0);
    if (e != cudaSuccess) { printf("   instantiate failed: %s\n", cudaGetErrorString(e)); cudaGetLastError(); return -1; }
    for (int i = 0; i < 3; ++i) CK(cudaGraphLaunch(ge, s[0]));
    CK(cudaStreamSynchronize(s[0]));
    const int reps = launches / per_graph;
    CK(cudaEventRecord(a, s[0]));
    for (int i = 0; i < reps; ++i) CK(cudaGraphLaunch(ge, s[0]));
    CK(cudaEventRecord(b, s[0]));
    CK(cudaEventSynchronize(b));
    CK(cudaEventElapsedTime(&ms, a, b));
    ms /= reps * per_graph;
    cudaGraphExecDestroy(ge); cudaGraphDestroy(g);
  } else if (mech == 4) {
    for (int i = 0; i < 8; ++i) launch_one(v, false, tab[i & 3], L[i & 3], grid[i & 3], s[i & 1]);
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(a, s[0]));
    CK(cudaStreamWaitEvent(s[1], a, 0));
    for (int i = 0; i < launches; ++i) launch_one(v, false, tab[i & 3], L[i & 3], grid[i & 3], s[i & 1]);
    CK(cudaEventRecord(j1, s[1]));
    CK(cudaStreamWaitEvent(s[0], j1, 0));
    CK(cudaEventRecord(b, s[0]));
    CK(cudaEventSynchronize(b));
    CK(cudaEventElapsedTime(&ms, a, b));
    ms /= launches;
  } else {
    for (int i = 0; i < 8; ++i) launch_one(v, pdl, tab[i & 3], L[i & 3], grid[i & 3], s[0]);
    CK(cudaStreamSynchronize(s[0]));
    CK(cudaEventRecord(a, s[0]));
    for (int i = 0; i < launches; ++i) launch_one(v, pdl, tab[i & 3], L[i & 3], grid[i & 3], s[0]);
    CK(cudaEventRecord(b, s[0]));
    CK(cudaEventSynchronize(b));
    CK(cudaEventElapsedTime(&ms, a, b));
    ms /= launches;
  }
  CK(cudaDeviceSynchronize());
  cudaEventDestroy(a); cudaEventDestroy(b); cudaEventDestroy(j1);
  cudaStreamDestroy(s[0]); cudaStreamDestroy(s[1]);
  return ms * 1e3;  // us per launch
}

#define V_JS(DT, T, U, MB, ADD, PSM) \
  Variant{std::string("jobsplit " #T "t u" #U " minb" #MB) + (ADD ? " add" : " mul") + " cap" #PSM, k_jobsplit<DT, T, U, MB, ADD, false>, k_jobsplit<DT, T, U, MB, ADD, true>, T, DT, 0, PSM}
#define V_JSM(DT, T, U, MB, PSM, MODE) \
  Variant{std::string("jobsplit " #T "t u" #U " minb" #MB " cap" #PSM " mode" #MODE " (1=wait at end, 2=epoch ld.volatile, 4=epoch __constant__, 8=epoch ld.nc evict_last, 16=epoch ld.volatile after the signal)"), k_jobsplit<DT, T, U, MB, false, false, MODE>, k_jobsplit<DT, T, U, MB, false, true, MODE>, T, DT, 0, PSM}
#define V_ROWS(DT, T, U, MB, H, PSM) \
  Variant{std::string("rows     " #T "t u" #U " minb" #MB) + (H ? " hoist" : " full ") + " cap" #PSM, k_rows<DT, T, U, MB, H, false>, k_rows<DT, T, U, MB, H, true>, T, DT, 1, PSM}
#define V_JR(DT, T, U, MB, PSM) \
  Variant{"jobrange " #T "t u" #U " minb" #MB " cap" #PSM, k_jobrange<DT, T, U, MB, false>, k_jobrange<DT, T, U, MB, true>, T, DT, 0, PSM}

template <int DT>
static std::vector<Variant> variants() {
  std::vector<Variant> v;
  v.push_back(V_JS(DT, 256, 2, 4, false, 4));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 1));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 2));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 3));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 17));
  v.push_back(V_JSM(DT, 256, 4, 4, 4, 17));
  v.push_back(V_JSM(DT, 128, 2, 4, 4, 17));
  v.push_back(V_JSM(DT, 128, 2, 8, 8, 17));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 5));
  v.push_back(V_JSM(DT, 256, 2, 4, 4, 9));
  v.push_back(V_JSM(DT, 256, 2, 3, 3, 3));
  v.push_back(V_JSM(DT, 256, 2, 2, 2, 3));
  v.push_back(V_JSM(DT, 128, 2, 4, 4, 3));
  v.push_back(V_JSM(DT, 128, 2, 6, 6, 3));
  if (getenv("FILL2_SHORT")) return v;
  v.push_back(V_JS(DT, 256, 2, 6, false, 4));
  v.push_back(V_JS(DT, 256, 2, 6, false, 6));
  v.push_back(V_JS(DT, 256, 3, 4, false, 4));
  v.push_back(V_JS(DT, 256, 4, 4, false, 4));
  v.push_back(V_JS(DT, 256, 4, 4, true, 4));
  v.push_back(V_JS(DT, 256, 2, 6, true, 6));
  v.push_back(V_JS(DT, 256, 2, 8, false, 8));
  v.push_back(V_JS(DT, 128, 4, 8, false, 8));
  v.push_back(V_JS(DT, 128, 2, 12, false, 12));
  v.push_back(V_JS(DT, 512, 2, 2, false, 2));
  v.push_back(V_JS(DT, 512, 2, 3, false, 3));
  v.push_back(V_ROWS(DT, 256, 2, 4, true, 4));
  v.push_back(V_ROWS(DT, 256, 4, 4, true, 4));
  v.push_back(V_ROWS(DT, 256, 2, 6, true, 6));
  v.push_back(V_ROWS(DT, 256, 4, 4, false, 4));
  v.push_back(V_JR(DT, 256, 2, 4, 4));
  v.push_back(V_JR(DT, 256, 4, 4, 4));
  v.push_back(V_JR(DT, 256, 2, 6, 6));
  return v;
}

int main(int argc, char** argv) {
  int dev = 0;
  CK(cudaSetDevice(dev));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, dev));
  g_sms = prop.multiProcessorCount;
  int mem_khz = 0, bus_bits = 0;
  CK(cudaDeviceGetAttribute(&mem_khz, cudaDevAttrMemoryClockRate, dev));
  CK(cudaDeviceGetAttribute(&bus_bits, cudaDevAttrGlobalMemoryBusWidth, dev));
  g_peak_gbs = 2.0 * mem_khz * 1e3 * (bus_bits / 8) / 1e9;
  printf("# %s, %d SMs, theoretical DRAM bandwidth %.0f GB/s (frac below is of this)\n", prop.name, g_sms, g_peak_gbs);
  CK(cudaMalloc(&g_buf, 4 * kSet));
  uint32_t k0 = (uint32_t)kSeed, k1 = (uint32_t)(kSeed >> 32);
  for (int r = 0; r < 10; ++r) { g_rk.k[2 * r] = k0; g_rk.k[2 * r + 1] = k1; k0 += W0; k1 += W1; }
  const int launches = argc > 1 ? atoi(argv[1]) : 640;
  const char* mech_name[5] = {"stream", "pdl", "graph", "graph+pdl", "2streams"};

  // pure-store twins
  {
    Variant so{"store only 256t cap4", k_store_only<256, 1, false>, k_store_only<256, 1, true>, 256, -1, 0, 4};
    for (int c3 = 0; c3 < 2; ++c3)
      for (int m = 0; m < 5; ++m) {
        const double us = time_variant(so, c3, m, launches);
        printf("%-44s %-3s %-10s %7.2f us  %6.0f GB/s\n", so.name.c_str(), c3 ? "C3" : "C2", mech_name[m], us, kSet / us / 1e3);
      }
    // memset reference
    cudaEvent_t a, b; CK(cudaEventCreate(&a)); CK(cudaEventCreate(&b));
    for (int i = 0; i < 8; ++i) CK(cudaMemsetAsync(g_buf + (i & 3) * kSet, 0, kSet, 0));
    CK(cudaDeviceSynchronize());
    CK(cudaEventRecord(a, 0));
    for (int i = 0; i < launches; ++i) CK(cudaMemsetAsync(g_buf + (i & 3) * kSet, 0, kSet, 0));
    CK(cudaEventRecord(b, 0)); CK(cudaEventSynchronize(b));
    float ms; CK(cudaEventElapsedTime(&ms, a, b));
    printf("%-44s %-3s %-10s %7.2f us  %6.0f GB/s\n", "cudaMemsetAsync", "-", "stream", ms * 1e3 / launches, kSet / (ms * 1e3 / launches) / 1e3);
  }

  for (int dt = 0; dt < 2; ++dt) {
    const bool c3 = dt == 1;  // fp32 -> C2 shape (64 tensors), fp16 -> C3 shape (one tensor)
    std::vector<Variant> vs = dt == 0 ? variants<0>() : variants<1>();
    for (auto& v : vs) {
      int regs = 0, occ = 0;
      cudaFuncAttributes fa;
      CK(cudaFuncGetAttributes(&fa, (const void*)v.fn));
      regs = fa.numRegs;
      CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, (const void*)v.fn, v.threads, 0));
      // correctness: write set 0 with this variant, compare all of it with the host restatement
      CK(cudaMemset(g_buf, 0xEE, kSet));
      JobTab tab; Launch L; int grid;
      make_launch(c3, 0, v, tab, L, grid);
      launch_one(v, false, tab, L, grid, 0);
      CK(cudaDeviceSynchronize());
      const bool ok = verify(c3, dt, 0);
      printf("%-44s %-3s regs=%d occ=%d grid=%d %s\n", v.name.c_str(), c3 ? "C3" : "C2", regs, occ, grid, ok ? "bit-exact" : "MISMATCH");
      if (!ok) continue;
      for (int m = 0; m < 5; ++m) {
        const double us = time_variant(v, c3, m, launches);
        if (us > 0) printf("    %-10s %7.2f us  %6.0f GB/s  frac %.3f\n", mech_name[m], us, kSet / us / 1e3, kSet / us / 1e3 / g_peak_gbs);
      }
      fflush(stdout);
    }
  }
  return 0;
}
