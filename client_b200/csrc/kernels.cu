// kernels.cu -- the sm_90a kernels of the tritonclient hot path:
//   fill_kernel              synthetic input fill  (Philox4x32-10 -> dtype -> 16 B st.global)
//   pack_image_chw_tma_kernel uint8 HWC -> fp16/fp32/bf16 CHW, source tiles staged in
//                            shared memory by TMA bulk copies (cp.async.bulk + mbarrier)
//   pack_image_generic_kernel fallback for shapes/alignments the TMA path cannot take
//   cast_kernel              contiguous dtype conversion (numpy astype semantics)
//   pack_strided_kernel      ndarray.tobytes() of a strided source
//   concat_kernel            b"".join of N tensors (wire body / region packing)
//   check_kernel(+finalize)  on-device output validation / checksums
// All of them are HBM-bound byte/integer work: no tensor cores, the design rules are
// coalesced 16-byte accesses, enough bytes in flight, grids sized from the SM count.
#include "kernels.cuh"
#include "philox.cuh"

namespace tb200 {

// =============================================================================
// small device helpers
// =============================================================================
__device__ __forceinline__ void st_cs_v4(void* p, const U32x4& v) {
  asm volatile("st.global.cs.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(p), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ void st_cs_v2(void* p, uint32_t a, uint32_t b) {
  asm volatile("st.global.cs.v2.u32 [%0], {%1, %2};" ::"l"(p), "r"(a), "r"(b) : "memory");
}
__device__ __forceinline__ uint4 ld_nc_v4(const void* p) {
  uint4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.u32 {%0, %1, %2, %3}, [%4];"
               : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
               : "l"(p));
  return r;
}
__device__ __forceinline__ uint32_t word_of(const U32x4& v, uint32_t i) {
  return i == 0 ? v.x : (i == 1 ? v.y : (i == 2 ? v.z : v.w));
}
// first n (<16) bytes of v, byte by byte (unaligned destinations and tails)
__device__ __forceinline__ void store_bytes(uint8_t* p, const U32x4& v, uint32_t n) {
  for (uint32_t i = 0; i < n; ++i) {
    p[i] = static_cast<uint8_t>(word_of(v, i >> 2) >> (8 * (i & 3)));
  }
}

// bytes [from, to) of v
__device__ __forceinline__ void store_byte_range(uint8_t* p, const U32x4& v, uint32_t from, uint32_t to) {
  for (uint32_t i = from; i < to; ++i) {
    p[i] = static_cast<uint8_t>(word_of(v, i >> 2) >> (8 * (i & 3)));
  }
}
// the 16 bytes at byte offset `off` (1..15) of the 32-byte concatenation a | b
__device__ __forceinline__ U32x4 funnel16(const U32x4& a, const U32x4& b, uint32_t off) {
  const uint32_t q = off >> 2, r = (off & 3) * 8;
  uint32_t w[5];
#pragma unroll
  for (uint32_t k = 0; k < 5; ++k) {
    const uint32_t i = q + k;  // <= 7
    w[k] = i < 4 ? word_of(a, i) : word_of(b, i - 4);
  }
  U32x4 o;
  o.x = __funnelshift_r(w[0], w[1], r);
  o.y = __funnelshift_r(w[1], w[2], r);
  o.z = __funnelshift_r(w[2], w[3], r);
  o.w = __funnelshift_r(w[3], w[4], r);
  return o;
}

// largest j in [0, n) with prefix[j] <= tile (prefix has n+1 entries, prefix[n] > tile)
__device__ __forceinline__ uint32_t find_job(const uint32_t* __restrict__ prefix, uint32_t n,
                                             uint32_t tile) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(prefix + mid) <= tile) lo = mid; else hi = mid;
  }
  return lo;
}

// =============================================================================
// Kernel 1: fill
// =============================================================================
// largest j in [0, n) with prefix[j] <= g (64-bit prefix)
__device__ __forceinline__ uint32_t find_job64(const uint64_t* __restrict__ prefix, uint32_t n, uint64_t g) {
  uint32_t lo = 0, hi = n;
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (__ldg(prefix + mid) <= g) lo = mid; else hi = mid;
  }
  return lo;
}

// Groups [g0, g0 + count) of one job; the first `full` of them can be written with one
// aligned 16-byte store, the rest (at most the job's last, partial group or an unaligned
// destination) byte-wise.  UNROLL independent Philox chains per thread per iteration;
// every store instruction of a warp covers 512 contiguous bytes.
template <uint32_t DT, int THREADS, int UNROLL, int ROUNDS>
__device__ __forceinline__ void fill_segment_random(uint8_t* __restrict__ dst, uint64_t nbytes,
                                                    uint64_t g0, uint32_t count, uint32_t full,
                                                    const FillParams& p, uint32_t s_lo, uint32_t s_hi,
                                                    const RoundKeys& rk) {
  uint32_t i = threadIdx.x;
  for (; i + (UNROLL - 1) * THREADS < full; i += UNROLL * THREADS) {
    U32x4 o[UNROLL];
#pragma unroll
    for (int k = 0; k < UNROLL; ++k) {
      const uint64_t g = g0 + i + k * THREADS;
      const U32x4 r = philox4x32_10_rk<ROUNDS>(static_cast<uint32_t>(g), static_cast<uint32_t>(g >> 32), s_lo, s_hi, rk);
      if constexpr (DT == kBytes) o[k] = fill_group_bytes(r, g, static_cast<uint32_t>(p.irange));
      else o[k] = fill_group(DT, r, p);
    }
#pragma unroll
    for (int k = 0; k < UNROLL; ++k) st_cs_v4(dst + (g0 + i + k * THREADS) * 16, o[k]);
  }
  for (; i < count; i += THREADS) {
    const uint64_t g = g0 + i;
    const U32x4 r = philox4x32_10_rk<ROUNDS>(static_cast<uint32_t>(g), static_cast<uint32_t>(g >> 32), s_lo, s_hi, rk);
    U32x4 o;
    if constexpr (DT == kBytes) o = fill_group_bytes(r, g, static_cast<uint32_t>(p.irange));
    else o = fill_group(DT, r, p);
    if (i < full) {
      st_cs_v4(dst + g * 16, o);
    } else {
      const uint64_t left = nbytes - g * 16;
      store_bytes(dst + g * 16, o, left >= 16 ? 16u : static_cast<uint32_t>(left));
    }
  }
}

// Destinations that are not 16-byte aligned (tensors behind a protobuf tag + length inside a
// gRPC message image, odd offsets in a region): the thread of group g writes the ALIGNED
// 16-byte cell that holds the end of group g-1 and the start of group g with one store,
// generating both groups (Philox is counter based; twice the arithmetic, but full-width
// stores instead of 16 single bytes -- these tensors are small and often sit in pinned host
// memory, where a byte store is a PCIe transaction).  Cells that reach outside the tensor
// (first, last, spill-over of the last group) are written byte-wise.  Lives in its own
// kernel (fill_unaligned_kernel, launched only when a launch has such jobs), dtype
// dispatched at run time: the aligned kernel's register budget is not touched.
template <int THREADS, int ROUNDS>
__device__ __forceinline__ void fill_segment_unaligned(const tb200_fill_job& jb, uint64_t g0, uint32_t count, uint64_t stream,
                                                    const RoundKeys& rk) {
  uint8_t* dst = reinterpret_cast<uint8_t*>(jb.dst);
  const uint64_t nbytes = jb.nbytes;
  const uint32_t k = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(dst) & 15);  // 1..15
  const uint64_t last_group = (nbytes + 15) / 16 - 1;
  FillParams p;
  p.lo_f = static_cast<float>(jb.lo);
  p.span_f = static_cast<float>(jb.span);
  p.lo_d = jb.lo;
  p.span_d = jb.span;
  p.ilo = jb.ilo;
  p.irange = jb.irange;
  p.unit = (jb.span == 0.0) ? 1u : 0u;
  const uint32_t s_lo = static_cast<uint32_t>(stream), s_hi = static_cast<uint32_t>(stream >> 32);
  const uint32_t const_word = jb.mode == TB200_FILL_BYTE ? (static_cast<uint32_t>(jb.ilo) & 0xFFu) * 0x01010101u : 0u;
  auto group = [&](uint64_t g) -> U32x4 {
    if (jb.mode != TB200_FILL_RANDOM) return U32x4{const_word, const_word, const_word, const_word};
    const U32x4 r = philox4x32_10_rk<ROUNDS>(static_cast<uint32_t>(g), static_cast<uint32_t>(g >> 32), s_lo, s_hi, rk);
    if (jb.dtype == kBytes) return fill_group_bytes(r, g, static_cast<uint32_t>(jb.irange));
    return fill_group(jb.dtype, r, p);
  };
  for (uint32_t i = threadIdx.x; i < count; i += THREADS) {
    const uint64_t g = g0 + i;
    uint8_t* at = dst + g * 16;  // group g starts here; its cell starts k bytes earlier
    const U32x4 cur = group(g);
    const uint64_t left = nbytes - g * 16;  // bytes of this group and everything after it
    if (g != 0) {
      const U32x4 prev = group(g - 1);
      if (left >= 16 - k) {
        st_cs_v4(at - k, funnel16(prev, cur, 16 - k));
      } else {
        store_byte_range(at - 16, prev, 16 - k, 16);
        store_byte_range(at, cur, 0, static_cast<uint32_t>(left));
      }
    } else {
      store_byte_range(at, cur, 0, left < 16 - k ? static_cast<uint32_t>(left) : 16 - k);
    }
    if (g == last_group && left > 16 - k) {  // what of the last group lies in the next cell
      store_byte_range(at, cur, 16 - k, left < 16 ? static_cast<uint32_t>(left) : 16u);
    }
  }
}

template <int THREADS>
__device__ __forceinline__ void fill_segment_const(uint8_t* __restrict__ dst, uint64_t nbytes,
                                                   uint64_t g0, uint32_t count, uint32_t full,
                                                   uint32_t word) {
  const U32x4 o{word, word, word, word};
  for (uint32_t i = threadIdx.x; i < count; i += THREADS) {
    const uint64_t g = g0 + i;
    if (i < full) {
      st_cs_v4(dst + g * 16, o);
    } else {
      const uint64_t left = nbytes - g * 16;
      store_bytes(dst + g * 16, o, left >= 16 ? 16u : static_cast<uint32_t>(left));
    }
  }
}

// The launch's groups (all jobs back to back) are split evenly over the CTAs: CTA b owns
// [T*b/P, T*(b+1)/P) and walks across job boundaries, so the load is balanced to one
// group for any mix of tensor sizes and every CTA is resident from the start.
template <int THREADS, int UNROLL, int MINB, int ROUNDS>
__global__ void __launch_bounds__(THREADS, MINB) fill_kernel(const FillLaunch L) {
  uint64_t epoch = L.epoch;
  if (L.dev_epoch != nullptr) epoch += *L.dev_epoch;

  uint64_t lo = (L.total_groups * blockIdx.x) / gridDim.x;
  const uint64_t hi = (L.total_groups * (blockIdx.x + 1ull)) / gridDim.x;
  uint32_t j = 0;
  if (lo < hi) {
    j = L.uniform_groups != 0 ? static_cast<uint32_t>(lo / L.uniform_groups) : find_job64(L.group_prefix, L.njobs, lo);
  }
  while (lo < hi) {
    const uint64_t job_begin = L.uniform_groups != 0 ? L.uniform_groups * j : __ldg(L.group_prefix + j);
    const uint64_t job_end = L.uniform_groups != 0 ? job_begin + L.uniform_groups : __ldg(L.group_prefix + j + 1);
    if (job_end <= lo) {  // empty job
      ++j;
      continue;
    }
    const uint64_t seg_hi = hi < job_end ? hi : job_end;
    const tb200_fill_job jb = L.jobs[j];
    uint8_t* dst = reinterpret_cast<uint8_t*>(jb.dst);
    const uint64_t g0 = lo - job_begin;
    const uint32_t count = static_cast<uint32_t>(seg_hi - lo);
    uint32_t full = 0;
    if ((reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
      const uint64_t whole = jb.nbytes / 16;
      if (whole > g0) full = (whole - g0) < count ? static_cast<uint32_t>(whole - g0) : count;
    } else {  // fill_unaligned_kernel's job
      lo = seg_hi;
      ++j;
      continue;
    }
    if (jb.mode != TB200_FILL_RANDOM) {
      uint32_t word = 0;
      if (jb.mode == TB200_FILL_BYTE) word = (static_cast<uint32_t>(jb.ilo) & 0xFFu) * 0x01010101u;
      fill_segment_const<THREADS>(dst, jb.nbytes, g0, count, full, word);
    } else {
      FillParams p;
      p.lo_f = static_cast<float>(jb.lo);
      p.span_f = static_cast<float>(jb.span);
      p.lo_d = jb.lo;
      p.span_d = jb.span;
      p.ilo = jb.ilo;
      p.irange = jb.irange;
      p.unit = (jb.span == 0.0) ? 1u : 0u;
      const uint64_t stream = jb.stream + epoch;
      const uint32_t s_lo = static_cast<uint32_t>(stream);
      const uint32_t s_hi = static_cast<uint32_t>(stream >> 32);
#define TB200_FILL_CASE(DT) \
  fill_segment_random<DT, THREADS, UNROLL, ROUNDS>(dst, jb.nbytes, g0, count, full, p, s_lo, s_hi, L.rk); break
      switch (jb.dtype) {
        case kF32: TB200_FILL_CASE(kF32);
        case kF16: TB200_FILL_CASE(kF16);
        case kBF16: TB200_FILL_CASE(kBF16);
        case kF64: TB200_FILL_CASE(kF64);
        case kI64: case kU64: TB200_FILL_CASE(kI64);
        case kI32: case kU32: TB200_FILL_CASE(kI32);
        case kI16: case kU16: TB200_FILL_CASE(kI16);
        case kI8: case kU8: TB200_FILL_CASE(kI8);
        case kBytes: TB200_FILL_CASE(kBytes);
        default: TB200_FILL_CASE(kBool);
      }
#undef TB200_FILL_CASE
    }
    lo = seg_hi;
    ++j;
  }

  // graph replays: the last CTA to finish advances the device epoch, so the next replay
  // generates fresh data without any host involvement (every CTA read the epoch above)
  if (L.bump != 0 && threadIdx.x == 0) {
    __threadfence();
    const unsigned int prev = atomicInc(L.done_counter, gridDim.x - 1);
    if (prev == gridDim.x - 1) *L.dev_epoch += L.bump;
  }
}

// The jobs fill_kernel leaves out: destinations that are not 16-byte aligned.  Same split of
// the launch's groups over the CTAs.  Runs BEFORE fill_kernel on the stream (it reads the
// device epoch that fill_kernel's last CTA advances).
template <int THREADS, int ROUNDS>
__global__ void __launch_bounds__(THREADS) fill_unaligned_kernel(const FillLaunch L) {
  uint64_t epoch = L.epoch;
  if (L.dev_epoch != nullptr) epoch += *L.dev_epoch;
  uint64_t lo = (L.total_groups * blockIdx.x) / gridDim.x;
  const uint64_t hi = (L.total_groups * (blockIdx.x + 1ull)) / gridDim.x;
  uint32_t j = 0;
  if (lo < hi) {
    j = L.uniform_groups != 0 ? static_cast<uint32_t>(lo / L.uniform_groups) : find_job64(L.group_prefix, L.njobs, lo);
  }
  while (lo < hi) {
    const uint64_t job_begin = L.uniform_groups != 0 ? L.uniform_groups * j : __ldg(L.group_prefix + j);
    const uint64_t job_end = L.uniform_groups != 0 ? job_begin + L.uniform_groups : __ldg(L.group_prefix + j + 1);
    if (job_end <= lo) {
      ++j;
      continue;
    }
    const uint64_t seg_hi = hi < job_end ? hi : job_end;
    const tb200_fill_job jb = L.jobs[j];
    if ((jb.dst & 15) != 0) {
      fill_segment_unaligned<THREADS, ROUNDS>(jb, lo - job_begin, static_cast<uint32_t>(seg_hi - lo), jb.stream + epoch, L.rk);
    }
    lo = seg_hi;
    ++j;
  }
}

// Homogeneous launches (every tensor the same size, dtype and range -- the perf_analyzer
// case: N slots of one model input): groups of ALL tensors form one index space that the
// grid walks with a grid stride, so at any moment the chip writes one dense moving window
// (scripts/store_bench.cu compares it with one contiguous range per CTA).  Per group only (dst, stream) of its tensor are
// looked up; the dtype parameters are hoisted out of the loop.
template <uint32_t DT, int THREADS, int UNROLL, int ROUNDS>
__global__ void __launch_bounds__(THREADS) fill_stride_kernel(const FillLaunch L) {
  uint64_t epoch = L.epoch;
  if (L.dev_epoch != nullptr) epoch += *L.dev_epoch;
  const tb200_fill_job j0 = L.jobs[0];
  FillParams p;
  p.lo_f = static_cast<float>(j0.lo);
  p.span_f = static_cast<float>(j0.span);
  p.lo_d = j0.lo;
  p.span_d = j0.span;
  p.ilo = j0.ilo;
  p.irange = j0.irange;
  p.unit = (j0.span == 0.0) ? 1u : 0u;
  const uint64_t gpj = L.uniform_groups;
  const uint64_t total = L.total_groups;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * THREADS;

  auto one = [&](uint64_t g, U32x4& out, uint8_t*& addr) {
    const uint64_t j = __umul64hi(g, L.div_magic);  // g / gpj (exact: g * gpj < 2^64)
    const uint64_t lg = g - j * gpj;
    const tb200_fill_job* jb = L.jobs + j;
    const uint64_t dst = __ldg(&jb->dst);
    const uint64_t stream = __ldg(&jb->stream) + epoch;
    const U32x4 r = philox4x32_10_rk<ROUNDS>(static_cast<uint32_t>(lg), static_cast<uint32_t>(lg >> 32),
                                              static_cast<uint32_t>(stream), static_cast<uint32_t>(stream >> 32), L.rk);
    out = fill_group(DT, r, p);
    addr = reinterpret_cast<uint8_t*>(dst) + lg * 16;
  };

  uint64_t g = static_cast<uint64_t>(blockIdx.x) * THREADS + threadIdx.x;
  for (; g + (UNROLL - 1) * stride < total; g += UNROLL * stride) {
    U32x4 o[UNROLL];
    uint8_t* a[UNROLL];
#pragma unroll
    for (int k = 0; k < UNROLL; ++k) one(g + k * stride, o[k], a[k]);
#pragma unroll
    for (int k = 0; k < UNROLL; ++k) st_cs_v4(a[k], o[k]);
  }
  for (; g < total; g += stride) {
    U32x4 o;
    uint8_t* a;
    one(g, o, a);
    st_cs_v4(a, o);
  }
  if (L.bump != 0 && threadIdx.x == 0) {
    __threadfence();
    const unsigned int prev = atomicInc(L.done_counter, gridDim.x - 1);
    if (prev == gridDim.x - 1) *L.dev_epoch += L.bump;
  }
}

template <int THREADS, int UNROLL, int ROUNDS>
static cudaError_t launch_fill_stride(const FillLaunch& l, uint32_t dtype, int sm_count, cudaStream_t s, int ctas_per_sm) {
  uint64_t grid = static_cast<uint64_t>(sm_count) * ctas_per_sm;
  const uint64_t max_useful = (l.total_groups + THREADS - 1) / THREADS;
  if (grid > max_useful) grid = max_useful;
  if (grid == 0) grid = 1;
  const uint32_t g = static_cast<uint32_t>(grid);
#define TB200_STRIDE_CASE(DT) fill_stride_kernel<DT, THREADS, UNROLL, ROUNDS><<<g, THREADS, 0, s>>>(l); break
  switch (dtype) {
    case kF32: TB200_STRIDE_CASE(kF32);
    case kF16: TB200_STRIDE_CASE(kF16);
    case kBF16: TB200_STRIDE_CASE(kBF16);
    case kF64: TB200_STRIDE_CASE(kF64);
    case kI64: case kU64: TB200_STRIDE_CASE(kI64);
    case kI32: case kU32: TB200_STRIDE_CASE(kI32);
    case kI16: case kU16: TB200_STRIDE_CASE(kI16);
    case kI8: case kU8: TB200_STRIDE_CASE(kI8);
    default: TB200_STRIDE_CASE(kBool);
  }
#undef TB200_STRIDE_CASE
  return cudaGetLastError();
}

// ---- the homogeneous launch (BASELINE C2: 64 x FP32[3,224,224]; C3: 1 x FP16[128,3,224,224]) ----
// What the general kernel above pays for and this one does not:
//   * the (dst, stream) table and every parameter sit in the constant bank: a CTA's first
//     Philox call is ~100 cycles after it starts, nothing is loaded from global memory
//     (only the device epoch of graph replays, one L2 hit);
//   * dtype and range are compile-time / constant-bank values, ~30 registers per thread;
//   * the stream-dependent multiplies of rounds 0 and 1 are folded once per CTA and job
//     (philox_stream_const): 18 IMAD.WIDE per 16 bytes instead of 20, and the store address
//     advances by 64-bit adds on the alu pipe instead of a 21st IMAD.WIDE;
//   * consecutive launches overlap: the kernel releases its dependents at once
//     (griddepcontrol.launch_dependents) and a successor launched with the programmatic-
//     serialization attribute starts on the SM slots this grid leaves free, so ramp and tail
//     of back-to-back fills hide behind each other (scripts/fill2_bench.cu times a graph chain
//     with and without; bench.py reports both as roofline.launches_serialised).  Before it
//     exits every CTA waits for the grid it overlapped with (griddepcontrol.wait), so "this
//     launch completed" still implies "every earlier launch of the stream completed".
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait_primary() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

// groups g = first, first + stride, ... < end of one tensor; U independent Philox chains per thread
// PLAIN: unit-interval floats / raw-bit integers (the default data of the generator): the range
// test of fill_group folds away at compile time instead of costing a predicated FFMA per word
template <uint32_t DT, int U, bool PLAIN>
__device__ __forceinline__ void fill_run(uint8_t* __restrict__ dst, uint32_t first, uint32_t stride, uint32_t end,
                                         const PhiloxStreamConst& sc, const FillUniform& L) {
  FillParams prm = L.p;
  if (PLAIN) {
    prm.unit = 1u;
    prm.irange = 0;
  } else {
    prm.unit = 0u;
    if (prm.irange == 0) prm.irange = 1;  // never taken: integer launches with irange == 0 are PLAIN
  }
  uint32_t g = first;
  uint8_t* p = dst + static_cast<uint64_t>(g) * 16u;
  uint64_t pstep = static_cast<uint64_t>(stride) * 16u;
  asm volatile("" : "+l"(pstep));  // opaque: the pointer advances by IADD3 pairs, not IMAD.WIDE
  for (; g + (U - 1) * stride < end; g += U * stride) {
    U32x4 o[U];
#pragma unroll
    for (int k = 0; k < U; ++k) {
      const U32x4 r = philox4x32_10_hoisted<10>(static_cast<uint64_t>(kPhiloxM0) * (g + k * stride), sc, L.rk);
      o[k] = fill_group(DT, r, prm);
    }
#pragma unroll
    for (int k = 0; k < U; ++k) {
      st_cs_v4(p, o[k]);
      p += pstep;
    }
  }
  for (; g < end; g += stride) {
    const U32x4 r = philox4x32_10_hoisted<10>(static_cast<uint64_t>(kPhiloxM0) * g, sc, L.rk);
    st_cs_v4(p, fill_group(DT, r, prm));
    p += pstep;
  }
}

constexpr int kFillUniThreads = 256;
template <uint32_t DT, int CAP, int THREADS, int U, bool PLAIN>
__global__ void __launch_bounds__(THREADS, 4) fill_uniform_kernel(const __grid_constant__ FillTab<CAP> tab, const __grid_constant__ FillUniform L) {
  // Release the dependents first: the instruction waits for the thread's outstanding loads, and
  // the epoch load behind it would delay every successor by its latency (scripts/fill2_bench.cu
  // modes 3 / 17).  Reading the epoch afterwards is
  // safe: the device epoch is only written by a plain kernel behind the chain (the last node of
  // a graph, tb200_graph_end), which starts after the chain's last fill completed, and that
  // implies -- by the griddepcontrol.wait below -- that every fill of the chain completed.
  pdl_launch_dependents();
  uint64_t epoch = L.epoch;
  if (L.dev_epoch != nullptr) epoch += *L.dev_epoch;
  if (L.ctas_per_job != 0) {
    const uint32_t j = blockIdx.x / L.ctas_per_job;
    const uint32_t part = blockIdx.x - j * L.ctas_per_job;
    const uint64_t stream = tab.stream[j] + epoch;
    const PhiloxStreamConst sc = philox_stream_const(static_cast<uint32_t>(stream), static_cast<uint32_t>(stream >> 32), L.rk);
    fill_run<DT, U, PLAIN>(reinterpret_cast<uint8_t*>(tab.dst[j]), part * THREADS + threadIdx.x, L.ctas_per_job * THREADS,
                    L.groups_per_job, sc, L);
  } else {
    uint64_t lo = (L.total_groups * blockIdx.x) / gridDim.x;
    const uint64_t hi = (L.total_groups * (blockIdx.x + 1ull)) / gridDim.x;
    uint32_t j = static_cast<uint32_t>(lo / L.groups_per_job);
    uint32_t g0 = static_cast<uint32_t>(lo - static_cast<uint64_t>(j) * L.groups_per_job);
    while (lo < hi) {
      const uint64_t left = hi - lo;
      const uint32_t room = L.groups_per_job - g0;
      const uint32_t n = left < room ? static_cast<uint32_t>(left) : room;
      const uint64_t stream = tab.stream[j] + epoch;
      const PhiloxStreamConst sc = philox_stream_const(static_cast<uint32_t>(stream), static_cast<uint32_t>(stream >> 32), L.rk);
      fill_run<DT, U, PLAIN>(reinterpret_cast<uint8_t*>(tab.dst[j]), g0 + threadIdx.x, THREADS, g0 + n, sc, L);
      lo += n;
      ++j;
      g0 = 0;
    }
  }
  pdl_wait_primary();
}

void plan_fill_uniform(FillUniform* u, int sm_count) {
  constexpr uint32_t kThreads = kFillUniThreads, kU = 2;
  // CTAs of one grid: 4 per SM, half of what fits -- the other slots take the CTAs of the next
  // launch, whose start-up then hides behind this grid's arithmetic
  const uint32_t target = static_cast<uint32_t>(sm_count) * 4u;
  u->ctas_per_job = 0;
  const uint32_t cpj = u->njobs <= target ? target / u->njobs : 0;
  // interleaved rows when the split fills the chip evenly and every part has whole iterations
  if (cpj != 0 && static_cast<uint64_t>(u->njobs) * cpj * 100 >= static_cast<uint64_t>(target) * 93 &&
      u->groups_per_job / cpj >= kThreads * kU * 2) {
    u->ctas_per_job = cpj;
    u->grid = u->njobs * cpj;
    return;
  }
  uint64_t grid = u->total_groups / (kThreads * kU);
  if (grid > target) grid = target;
  if (grid == 0) grid = 1;
  u->grid = static_cast<uint32_t>(grid);
}

template <uint32_t DT, int CAP>
static cudaError_t launch_fill_uniform_t(const FillUniform& u, const tb200_fill_job* host_jobs, cudaStream_t s, bool pdl) {
  FillTab<CAP> tab;
  for (uint32_t i = 0; i < u.njobs; ++i) {
    tab.dst[i] = host_jobs[i].dst;
    tab.stream[i] = host_jobs[i].stream;
  }
  for (uint32_t i = u.njobs; i < static_cast<uint32_t>(CAP); ++i) tab.dst[i] = tab.stream[i] = 0;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(u.grid);
  cfg.blockDim = dim3(kFillUniThreads);
  cfg.stream = s;
  cudaLaunchAttribute at[1];
  if (pdl) {
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at;
    cfg.numAttrs = 1;
  }
  const bool is_float = DT == kF32 || DT == kF16 || DT == kBF16 || DT == kF64;
  const bool plain = DT == kBool || (is_float ? u.p.unit != 0 : u.p.irange == 0);
  if (plain) return cudaLaunchKernelEx(&cfg, fill_uniform_kernel<DT, CAP, kFillUniThreads, 2, true>, tab, u);
  return cudaLaunchKernelEx(&cfg, fill_uniform_kernel<DT, CAP, kFillUniThreads, 2, false>, tab, u);
}

cudaError_t launch_fill_uniform(const FillUniform& u, const tb200_fill_job* host_jobs, uint32_t dtype, cudaStream_t s, bool pdl) {
  if (u.njobs == 0 || u.njobs > static_cast<uint32_t>(kFillTabLarge)) return cudaErrorInvalidValue;
#define TB200_UNI_CASE(DT)                                                                              \
  return u.njobs <= static_cast<uint32_t>(kFillTabSmall) ? launch_fill_uniform_t<DT, kFillTabSmall>(u, host_jobs, s, pdl) \
                                                         : launch_fill_uniform_t<DT, kFillTabLarge>(u, host_jobs, s, pdl)
  switch (dtype) {
    case kF32: TB200_UNI_CASE(kF32);
    case kF16: TB200_UNI_CASE(kF16);
    case kBF16: TB200_UNI_CASE(kBF16);
    case kF64: TB200_UNI_CASE(kF64);
    case kI64: case kU64: TB200_UNI_CASE(kI64);
    case kI32: case kU32: TB200_UNI_CASE(kI32);
    case kI16: case kU16: TB200_UNI_CASE(kI16);
    case kI8: case kU8: TB200_UNI_CASE(kI8);
    case kBool: TB200_UNI_CASE(kBool);
    default: return cudaErrorInvalidValue;
  }
#undef TB200_UNI_CASE
}

static int g_fill_variant = 0;
void set_fill_variant(int v) { g_fill_variant = v; }

template <int THREADS, int UNROLL, int MINB, int ROUNDS>
static cudaError_t launch_fill_t(const FillLaunch& l, int sm_count, cudaStream_t s, int ctas_per_sm) {
  static int occ = 0;
  if (occ == 0) {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, fill_kernel<THREADS, UNROLL, MINB, ROUNDS>, THREADS, 0) != cudaSuccess || n < 1) n = 1;
    occ = n;
  }
  int per_sm = (ctas_per_sm > 0 && ctas_per_sm < occ) ? ctas_per_sm : occ;
  uint64_t grid = static_cast<uint64_t>(sm_count) * per_sm;
  // no point in CTAs with less than one iteration of work
  const uint64_t max_useful = (l.total_groups + THREADS * UNROLL - 1) / (THREADS * UNROLL);
  if (grid > max_useful) grid = max_useful;
  if (grid == 0) grid = 1;
  fill_kernel<THREADS, UNROLL, MINB, ROUNDS><<<static_cast<uint32_t>(grid), THREADS, 0, s>>>(l);
  return cudaGetLastError();
}

cudaError_t launch_fill(const FillLaunch& l, int sm_count, cudaStream_t s) {
  if (l.total_groups == 0 && l.bump == 0) return cudaSuccess;
  if (l.unaligned_jobs != 0) {
    uint64_t grid = static_cast<uint64_t>(sm_count) * 4;
    const uint64_t max_useful = (l.total_groups + 255) / 256;
    if (grid > max_useful) grid = max_useful;
    fill_unaligned_kernel<256, 10><<<static_cast<uint32_t>(grid), 256, 0, s>>>(l);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return e;
    if (l.unaligned_jobs == l.njobs && l.bump == 0) return cudaSuccess;  // nothing left for the aligned kernel
  }
  const int v = g_fill_variant;
  // Default policy (scripts/fill_sweep.py times the alternatives): the kernel is issue-bound
  // at 10 Philox rounds, so the cheapest indexing wins: many small equal tensors (wire-mode
  // slots, a few KB each) take the grid-stride kernel (no per-CTA tensor walk), everything
  // else the balanced contiguous ranges.
  const bool small_homogeneous = l.homogeneous && l.total_groups != 0 && l.uniform_groups * 16 <= 32768;
  if (v == 0) {
    if (small_homogeneous) return launch_fill_stride<256, 4, 10>(l, l.dtype0, sm_count, s, 4);
    return launch_fill_t<256, 3, 1, 10>(l, sm_count, s, 0);
  }
  if (l.homogeneous && l.total_groups != 0 && v < 100) {
    switch (v) {
      case 20: return launch_fill_stride<256, 1, 10>(l, l.dtype0, sm_count, s, 8);
      case 21: return launch_fill_stride<256, 2, 10>(l, l.dtype0, sm_count, s, 6);
      case 22: return launch_fill_stride<256, 2, 10>(l, l.dtype0, sm_count, s, 16);
      case 24: return launch_fill_stride<256, 4, 10>(l, l.dtype0, sm_count, s, 4);
      case 28: return launch_fill_stride<256, 2, 1>(l, l.dtype0, sm_count, s, 6);   // NOT the contract: ceiling
      default: break;
    }
  }
  switch (v >= 100 ? v - 100 : v) {
    // experiment matrix (scripts/fill_sweep.py): threads, unroll, min CTAs/SM, rounds
    case 1: return launch_fill_t<256, 2, 1, 10>(l, sm_count, s, 0);
    case 2: return launch_fill_t<256, 4, 1, 10>(l, sm_count, s, 0);
    case 6: return launch_fill_t<512, 2, 1, 10>(l, sm_count, s, 0);
    case 9: return launch_fill_t<256, 2, 1, 7>(l, sm_count, s, 0);   // NOT the contract: sensitivity only
    case 10: return launch_fill_t<256, 2, 1, 1>(l, sm_count, s, 0);  // NOT the contract: store ceiling
    default: return launch_fill_t<256, 3, 1, 10>(l, sm_count, s, 0);
  }
}

// =============================================================================
// Kernel 2a: uint8 HWC -> CHW cast+pack, TMA-staged
// =============================================================================
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count)
               : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  uint32_t done;
  uint32_t spins = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(addr), "r"(parity)
        : "memory");
    // a copy that never lands is a bug: fail the launch instead of hanging the GPU
    if (!done && ++spins > (1u << 26)) __trap();
  } while (!done);
}
// TMA bulk copy global -> shared, completion signalled on the mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
      ::"r"(smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}

constexpr int kPackThreads = 128;
constexpr int kPackStages = 4;

template <uint32_t DST>
struct PackTraits {
  static constexpr int kElem = (DST == kF32) ? 4 : 2;
  static constexpr int kPxPerThread = 16 / kElem;  // one 16-byte store per channel
  static constexpr int kTilePx = kPackThreads * kPxPerThread;
};

template <uint32_t DST, int C, uint32_t SCALING>
__global__ void __launch_bounds__(kPackThreads)
pack_image_chw_tma_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                          uint32_t hw, uint32_t tiles_per_image, uint32_t total_tiles) {
  using T = PackTraits<DST>;
  constexpr int PPT = T::kPxPerThread;
  constexpr int TILE_PX = T::kTilePx;
  constexpr int TILE_B = TILE_PX * C;  // 3072 (fp16,c=3) / 1536 (fp32,c=3): multiples of 16
  constexpr int NB = PPT * C;          // source bytes per thread
  constexpr int NW = (NB + 3) / 4;

  __shared__ __align__(128) uint8_t stage[kPackStages][TILE_B];
  __shared__ __align__(8) uint64_t full[kPackStages];

  const uint32_t tid = threadIdx.x;
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < kPackStages; ++s) mbar_init(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const uint32_t my_count =
      (total_tiles > blockIdx.x) ? (total_tiles - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;

  auto issue = [&](uint32_t i) {
    const uint32_t tile = blockIdx.x + i * gridDim.x;
    const uint32_t img = tile / tiles_per_image;
    const uint32_t px0 = (tile - img * tiles_per_image) * TILE_PX;
    const uint32_t npx = min(static_cast<uint32_t>(TILE_PX), hw - px0);
    const uint32_t bytes = npx * C;  // multiple of 16 (launcher checks hw*C % 16 == 0)
    const uint32_t s = i % kPackStages;
    mbar_expect_tx(&full[s], bytes);
    bulk_g2s(stage[s], src + (static_cast<uint64_t>(img) * hw + px0) * C, bytes, &full[s]);
  };

  if (tid == 0) {
    const uint32_t pre = my_count < kPackStages ? my_count : kPackStages;
    for (uint32_t i = 0; i < pre; ++i) issue(i);
  }

  for (uint32_t i = 0; i < my_count; ++i) {
    const uint32_t s = i % kPackStages;
    mbar_wait(&full[s], (i / kPackStages) & 1u);

    const uint32_t tile = blockIdx.x + i * gridDim.x;
    const uint32_t img = tile / tiles_per_image;
    const uint32_t px0 = (tile - img * tiles_per_image) * TILE_PX;
    const uint32_t npx = min(static_cast<uint32_t>(TILE_PX), hw - px0);
    const bool active = tid * PPT < npx;  // npx is a multiple of PPT

    uint32_t wv[NW];
    if (active) {
      const uint8_t* sp = stage[s] + tid * NB;
      if constexpr (NB % 8 == 0) {
#pragma unroll
        for (int k = 0; k < NB / 8; ++k) {
          const uint2 v = *reinterpret_cast<const uint2*>(sp + 8 * k);
          wv[2 * k] = v.x;
          wv[2 * k + 1] = v.y;
        }
      } else {
#pragma unroll
        for (int k = 0; k < NW; ++k) wv[k] = *reinterpret_cast<const uint32_t*>(sp + 4 * k);
      }
    }
    __syncthreads();  // every thread has consumed stage s: it may be refilled
    if (tid == 0 && i + kPackStages < my_count) issue(i + kPackStages);

    if (!active) continue;
    const uint64_t plane0 = (static_cast<uint64_t>(img) * C) * hw + px0 + tid * PPT;
#pragma unroll
    for (int ch = 0; ch < C; ++ch) {
      uint8_t* out = dst + (plane0 + static_cast<uint64_t>(ch) * hw) * T::kElem;
      if constexpr (DST == kF32) {
        uint32_t of[PPT];
#pragma unroll
        for (int j = 0; j < PPT; ++j) {
          const int kb = j * C + ch;
          const uint32_t b = (wv[kb >> 2] >> (8 * (kb & 3))) & 0xFFu;
          of[j] = f32_bits(scale_pixel_f32(b, SCALING, C, ch));
        }
        st_cs_v4(out, U32x4{of[0], of[1], of[2], of[3]});
      } else if constexpr (DST == kF16) {
        // Packed fp16 path, two pixels per instruction where possible.  Exact for all 256
        // pixel values (enumerated in tests/test_kernels_gpu.py and tests/test_host_emul.py):
        //   NONE / VGG : half(1024 + p) is built by byte permutation, one HADD2 subtracts
        //                1024 (+ mean) exactly
        //   INCEPTION  : q = fl32(p * fl32(1/127.5)) via one FFMA on the magic float
        //                2^23 + p, cvt.rn.f16x2 rounds the pair like numpy's fl16(x / 127.5)
        //                (the product rounds to the same half as the true quotient for
        //                every p), HSUB2 subtracts 1 exactly
        uint32_t pair[PPT / 2];
#pragma unroll
        for (int j = 0; j < PPT; j += 2) {
          const int ka = j * C + ch, kb = (j + 1) * C + ch;
          const uint32_t wa = wv[ka >> 2], wb = wv[kb >> 2];
          if constexpr (SCALING == 1) {
            constexpr float r = 1.0f / 127.5f;
            constexpr float c0 = -8388608.0f * r;  // exact: power-of-two scaling of r
            const float ma = __uint_as_float(__byte_perm(wa, 0x4B000000u, (ka & 3) | 0x7650));
            const float mb = __uint_as_float(__byte_perm(wb, 0x4B000000u, (kb & 3) | 0x7650));
            const __half2 q = __floats2half2_rn(__fmaf_rn(ma, r, c0), __fmaf_rn(mb, r, c0));
            const __half2 y = __hsub2(q, __float2half2_rn(1.0f));
            pair[j / 2] = *reinterpret_cast<const uint32_t*>(&y);
          } else {
            // byte0 <- pixel a, byte2 <- pixel b, then or in the exponent of 1024
            const uint32_t t = __byte_perm(wa, wb, (ka & 3) | ((4 + (kb & 3)) << 8));
            const uint32_t m2 = (t & 0x00FF00FFu) | 0x64006400u;
            const float bias = (SCALING == 2) ? 1024.0f + vgg_mean(C, ch) : 1024.0f;
            const __half2 y = __hsub2(*reinterpret_cast<const __half2*>(&m2), __float2half2_rn(bias));
            pair[j / 2] = *reinterpret_cast<const uint32_t*>(&y);
          }
        }
        st_cs_v4(out, U32x4{pair[0], pair[1], pair[2], pair[3]});
      } else {
        uint32_t h[PPT];
#pragma unroll
        for (int j = 0; j < PPT; ++j) {
          const int kb = j * C + ch;
          const uint32_t b = (wv[kb >> 2] >> (8 * (kb & 3))) & 0xFFu;
          h[j] = f32_to_bf16_trunc(scale_pixel_f32(b, SCALING, C, ch));
        }
        U32x4 o;
        o.x = h[0] | (h[1] << 16);
        o.y = h[2] | (h[3] << 16);
        o.z = h[4] | (h[5] << 16);
        o.w = h[6] | (h[7] << 16);
        st_cs_v4(out, o);
      }
    }
  }
}

// ---- fallback: any shape / alignment / layout, one destination element per thread
__global__ void __launch_bounds__(256)
pack_image_generic_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src,
                          uint32_t dst_dtype, uint32_t layout, uint32_t scaling, uint32_t c,
                          uint64_t hw, uint64_t total) {
  for (uint64_t idx = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; idx < total;
       idx += static_cast<uint64_t>(gridDim.x) * blockDim.x) {
    uint32_t ch;
    uint64_t sidx;
    if (layout == TB200_NCHW) {
      const uint64_t chw = c * hw;
      const uint64_t img = idx / chw;
      const uint64_t rem = idx - img * chw;
      ch = static_cast<uint32_t>(rem / hw);
      const uint64_t p = rem - ch * hw;
      sidx = (img * hw + p) * c + ch;
    } else {
      ch = static_cast<uint32_t>(idx % c);
      sidx = idx;
    }
    const uint32_t b = src[sidx];
    if (dst_dtype == kF32) {
      reinterpret_cast<float*>(dst)[idx] = scale_pixel_f32(b, scaling, c, ch);
    } else if (dst_dtype == kF16) {
      reinterpret_cast<uint16_t*>(dst)[idx] = scale_pixel_f16(b, scaling, c, ch);
    } else {
      reinterpret_cast<uint16_t*>(dst)[idx] =
          f32_to_bf16_trunc(scale_pixel_f32(b, scaling, c, ch));
    }
  }
}

// ---- resize + pack: one CTA per 32 x tile_h output tile --------------------------------
// Phase A resamples the source rows the tile needs horizontally into shared memory
// (8-bit, exactly Pillow's intermediate image), phase B resamples those vertically and
// applies astype / scaling / layout on the way out.
constexpr int kResizeBits = 22;  // Pillow: PRECISION_BITS = 32 - 8 - 2
// The triangle filter's coefficients are >= 0 and a pixel's taps sum to 2^22 +- taps/2
// (resample.h), so 0 < acc and (acc >> 22) <= 255: Pillow's clip8 never clips and is left out.
__device__ __forceinline__ uint32_t resize_round8(int32_t acc) { return static_cast<uint32_t>(acc) >> kResizeBits; }

// N-tap dot product of bytes at stride `step` with int32 coefficients, N a compile-time bound
template <int N>
__device__ __forceinline__ int32_t resize_dot(const uint8_t* px, int step, const int32_t* k) {
  int32_t acc = 1 << (kResizeBits - 1);
#pragma unroll
  for (int t = 0; t < N; ++t) acc += static_cast<int32_t>(px[t * step]) * k[t];
  return acc;
}
// one output element: astype + scaling of an 8-bit pixel, by destination type
template <uint32_t DST, uint32_t SCALING, int C>
__device__ __forceinline__ void resize_store(void* dst, size_t idx, uint32_t px, int ch) {
  if constexpr (DST == kF32) static_cast<float*>(dst)[idx] = scale_pixel_f32(px, SCALING, C, ch);
  else if constexpr (DST == kF16) static_cast<uint16_t*>(dst)[idx] = scale_pixel_f16(px, SCALING, C, ch);
  else if constexpr (DST == kBF16) static_cast<uint16_t*>(dst)[idx] = f32_to_bf16_trunc(scale_pixel_f32(px, SCALING, C, ch));
  else static_cast<uint8_t*>(dst)[idx] = static_cast<uint8_t>(px);
}

// what every phase of a tile needs to know
struct ResizeTile {
  uint8_t* raw;            // staged source rows [rows][raw_stride], each at its 16-byte granule
  uint8_t* tmp;            // horizontally resampled 8-bit rows [rows][32*C]
  const uint8_t* shift_s;  // a row's offset inside its first granule
  uint64_t* bar;           // completes when every row is staged
  int2 hb;                 // lane l: (first source column, taps) of output column x0 + l; (c0, 0) right of the image
  int c0, rows;
  uint32_t raw_stride;
};

// phase A with N unrolled taps: a warp per staged row; lane l owns the (column, channel) pairs l, 32 + l, ...
// (C of them: neighbouring lanes read neighbouring bytes) and keeps their taps in registers.  Taps past a
// pair's own count carry a zero coefficient -- the bytes they read lie inside the shared memory block (the
// staged rows are followed by the 8-bit image) and do not matter; a pair right of the image produces 0.
template <int N, int C>
__device__ __forceinline__ void resize_phase_a(const ResizeTile& t, const int32_t* __restrict__ hcoeffs, int hk) {
  constexpr int P = 32 * C;
  const int lane = threadIdx.x & 31;
  int32_t kr[C][N];
  int off[C];
#pragma unroll
  for (int g = 0; g < C; ++g) {
    const int pair = g * 32 + lane;
    const int xl = pair / C;
    const int bx = __shfl_sync(0xFFFFFFFFu, t.hb.x, xl), by = __shfl_sync(0xFFFFFFFFu, t.hb.y, xl);
    off[g] = (bx - t.c0) * C + (pair - xl * C);
    const int32_t* k = hcoeffs + xl * hk;
#pragma unroll
    for (int i = 0; i < N; ++i) kr[g][i] = i < by ? __ldg(k + i) : 0;
  }
  mbar_wait(t.bar, 0);  // the coefficient loads above overlap the row copies
#pragma unroll 2
  for (int row = threadIdx.x >> 5; row < t.rows; row += 8) {
    const uint8_t* line = t.raw + static_cast<uint32_t>(row) * t.raw_stride + t.shift_s[row];
    uint8_t* out = t.tmp + row * P + lane;
#pragma unroll
    for (int g = 0; g < C; ++g) {
      int32_t acc = 1 << (kResizeBits - 1);
#pragma unroll
      for (int i = 0; i < N; ++i) acc += static_cast<int32_t>(line[off[g] + i * C]) * kr[g][i];
      out[g * 32] = static_cast<uint8_t>(resize_round8(acc));
    }
  }
}

// any tap count: the same mapping, coefficients read through the cache
template <int C>
__device__ __forceinline__ void resize_phase_a_any(const ResizeTile& t, const int32_t* __restrict__ hcoeffs, int hk) {
  constexpr int P = 32 * C;
  const int lane = threadIdx.x & 31;
  mbar_wait(t.bar, 0);
  for (int g = 0; g < C; ++g) {
    const int pair = g * 32 + lane;
    const int xl = pair / C;
    const int bx = __shfl_sync(0xFFFFFFFFu, t.hb.x, xl), by = __shfl_sync(0xFFFFFFFFu, t.hb.y, xl);
    const int off = (bx - t.c0) * C + (pair - xl * C);
    const int32_t* k = hcoeffs + xl * hk;
    for (int row = threadIdx.x >> 5; row < t.rows; row += 8) {
      const uint8_t* line = t.raw + static_cast<uint32_t>(row) * t.raw_stride + t.shift_s[row] + off;
      int32_t acc = 1 << (kResizeBits - 1);
      for (int i = 0; i < by; ++i) acc += static_cast<int32_t>(line[i * C]) * __ldg(k + i);
      t.tmp[row * P + pair] = static_cast<uint8_t>(resize_round8(acc));
    }
  }
}

// phase B with N unrolled taps: a warp per output row, a lane per output column.  Rows with fewer taps
// use zero coefficients (the table is zero-padded) on rows of the 8-bit image past their own -- the block
// has `vk` slack rows for that.  voff: lane l holds the byte offset of output row l's first tap row.
template <int N, uint32_t DST, uint32_t SCALING, int C>
__device__ __forceinline__ void resize_phase_b(const uint8_t* tmp, const int32_t* vk_s, int vk, int voff, int out_rows, bool live,
                                               void* dst, size_t base, size_t row_stride, size_t ch_stride) {
  constexpr int P = 32 * C;
  const uint8_t* colbase = tmp + (threadIdx.x & 31) * C;
#pragma unroll 2
  for (int yl = threadIdx.x >> 5; yl < out_rows; yl += 8, base += 8 * row_stride) {
    const uint8_t* col = colbase + __shfl_sync(0xFFFFFFFFu, voff, yl);
    const int32_t* k = vk_s + yl * vk;
    int32_t kr[N];
#pragma unroll
    for (int i = 0; i < N; ++i) kr[i] = k[i];
    if (live) {
#pragma unroll
      for (int ch = 0; ch < C; ++ch) {
        int32_t acc = 1 << (kResizeBits - 1);
#pragma unroll
        for (int i = 0; i < N; ++i) acc += static_cast<int32_t>(col[ch + i * P]) * kr[i];
        resize_store<DST, SCALING, C>(dst, base + ch * ch_stride, resize_round8(acc), ch);
      }
    }
  }
}

// shared memory: mbarrier (16 B) | raw source block [max_rows][raw_stride] | horizontally resampled
// [max_rows + vk][32*C] | the tile's vertical coefficients (tile_h*vk int32) | per-row alignment shifts
template <int C, uint32_t DST, uint32_t SCALING>
__global__ void __launch_bounds__(256, 5) resize_pack_kernel(const __grid_constant__ ResizePack p) {
  extern __shared__ __align__(16) uint8_t rp_smem[];
  constexpr int P = 32 * C;  // (column, channel) pairs of a tile
  const int lane = threadIdx.x & 31;
  const int x0 = blockIdx.x * 32;
  const int xe = min(x0 + 32, p.dw) - 1;
  const int y0 = blockIdx.y * p.tile_h;  // tile_h <= 32: a lane per output row as well
  const int y1 = min(y0 + p.tile_h, p.dh) - 1;
  const int img = blockIdx.z;
  // every warp loads the tile's bounds, one column and one row per lane
  int2 hb = x0 + lane <= xe ? p.hbounds[x0 + lane] : make_int2(0, 0);
  const int2 vb = y0 + lane <= y1 ? p.vbounds[y0 + lane] : make_int2(0, 0);
  const int c0 = __shfl_sync(0xFFFFFFFFu, hb.x, 0);
  const int span = __shfl_sync(0xFFFFFFFFu, hb.x + hb.y, xe - x0) - c0;  // source columns the tile reads
  const int r0 = __shfl_sync(0xFFFFFFFFu, vb.x, 0);
  const int rows = __shfl_sync(0xFFFFFFFFu, vb.x + vb.y, y1 - y0) - r0;
  const int nmaxh = __reduce_max_sync(0xFFFFFFFFu, hb.y);
  const int nmaxv = __reduce_max_sync(0xFFFFFFFFu, vb.y);
  if (x0 + lane > xe) hb.x = c0;
  const int voff = (vb.x - r0) * P;

  ResizeTile t;
  t.bar = reinterpret_cast<uint64_t*>(rp_smem);
  t.raw = rp_smem + 16;
  t.tmp = t.raw + static_cast<size_t>(p.max_rows) * p.raw_stride;
  int32_t* vk_s = reinterpret_cast<int32_t*>(t.tmp + ((static_cast<size_t>(p.max_rows + p.vk) * P + 15) & ~static_cast<size_t>(15)));
  uint8_t* shift_s = reinterpret_cast<uint8_t*>(vk_s + p.tile_h * p.vk);
  t.shift_s = shift_s;
  t.hb = hb; t.c0 = c0; t.rows = rows; t.raw_stride = p.raw_stride;

  if (threadIdx.x == 0) {
    mbar_init(t.bar, static_cast<uint32_t>(rows));  // one arrival per staged row
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  // phase 0: one TMA bulk copy per source row, issued by one thread each: the 16-byte granules that cover
  // the row's bytes -- row starts are arbitrary byte addresses; the row's offset inside its first granule
  // goes to shift_s.  Nothing waits here.
  {
    const uint8_t* img_src = p.src + static_cast<size_t>(img) * p.sh * p.sw * C + static_cast<size_t>(c0) * C;
    const uint8_t* src_end = p.src + static_cast<size_t>(p.n) * p.sh * p.sw * C;
    const uint32_t pitch = static_cast<uint32_t>(p.sw) * C;
    // rows dealt round the warps (thread (lane, warp) takes row lane * 8 + warp): the copies of a warp's lanes are
    // issued one after the other, eight warps get the block under way sooner than two
    for (int row = lane * 8 + (threadIdx.x >> 5); row < rows; row += 256) {
      const uint8_t* g = img_src + static_cast<size_t>(static_cast<uint32_t>(r0 + row) * pitch);  // an image is < 4 GiB
      const uint32_t shift = static_cast<uint32_t>(reinterpret_cast<uintptr_t>(g) & 15u);
      const uint8_t* ga = g - shift;
      const uint32_t bytes = (shift + static_cast<uint32_t>(span) * C + 15u) & ~15u;
      uint8_t* srow = t.raw + static_cast<size_t>(row) * p.raw_stride;
      shift_s[row] = static_cast<uint8_t>(shift);
      if (ga >= p.src && ga + bytes <= src_end) {
        mbar_expect_tx(t.bar, bytes);
        bulk_g2s(srow, ga, bytes, t.bar);
      } else {  // the granules of the first / last row of the whole source may leave the buffer: bytes, guarded
        for (uint32_t i = 0; i < bytes; ++i) srow[i] = (ga + i >= p.src && ga + i < src_end) ? ga[i] : uint8_t{0};
        asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(t.bar)) : "memory");
      }
    }
    const int32_t* vc = p.vcoeffs + static_cast<size_t>(y0) * p.vk;
    const int vlive = (y1 - y0 + 1) * p.vk;
#pragma unroll 1
    for (int i = threadIdx.x; i < vlive; i += 256) vk_s[i] = __ldg(vc + i);  // read after the barrier below
  }

  // phase A: horizontal pass into 8-bit rows (Pillow's intermediate image)
  {
    const int32_t* hc = p.hcoeffs + static_cast<size_t>(x0) * p.hk;
    switch (nmaxh) {
      case 0: case 1: case 2: case 3: resize_phase_a<3, C>(t, hc, p.hk); break;
      case 4: resize_phase_a<4, C>(t, hc, p.hk); break;
      case 5: resize_phase_a<5, C>(t, hc, p.hk); break;
      case 6: resize_phase_a<6, C>(t, hc, p.hk); break;
      default: resize_phase_a_any<C>(t, hc, p.hk); break;
    }
  }
  __syncthreads();

  // phase B: vertical pass + astype / scaling / layout
  const bool live = x0 + lane <= xe;
  const size_t hw = static_cast<size_t>(p.dh) * p.dw;
  const bool nchw = p.layout == TB200_NCHW;
  const size_t ch_stride = nchw ? hw : 1;
  const size_t row_stride = nchw ? static_cast<size_t>(p.dw) : static_cast<size_t>(p.dw) * C;
  const size_t base = (nchw ? static_cast<size_t>(img) * C * hw + (x0 + lane) : (static_cast<size_t>(img) * hw + (x0 + lane)) * C) +
                      static_cast<size_t>(y0 + (threadIdx.x >> 5)) * row_stride;
  const int out_rows = y1 - y0 + 1;
  switch (nmaxv) {
    case 1: resize_phase_b<1, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    case 2: resize_phase_b<2, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    case 3: resize_phase_b<3, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    case 4: resize_phase_b<4, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    case 5: resize_phase_b<5, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    case 6: resize_phase_b<6, DST, SCALING, C>(t.tmp, vk_s, p.vk, voff, out_rows, live, p.dst, base, row_stride, ch_stride); break;
    default: {
      const uint8_t* colbase = t.tmp + lane * C;
      size_t bs = base;
      for (int yl = threadIdx.x >> 5; yl < out_rows; yl += 8, bs += 8 * row_stride) {
        const uint8_t* col = colbase + __shfl_sync(0xFFFFFFFFu, voff, yl);
        const int taps = __shfl_sync(0xFFFFFFFFu, vb.y, yl);
        const int32_t* k = vk_s + yl * p.vk;
        if (!live) continue;
        for (int ch = 0; ch < C; ++ch) {
          int32_t acc = 1 << (kResizeBits - 1);
          for (int i = 0; i < taps; ++i) acc += static_cast<int32_t>(col[ch + i * P]) * k[i];
          resize_store<DST, SCALING, C>(p.dst, bs + ch * ch_stride, resize_round8(acc), ch);
        }
      }
    }
  }
}

template <int C, uint32_t DST>
static cudaError_t launch_resize_scaling(const ResizePack& p, dim3 grid, cudaStream_t s) {
  cudaError_t e = cudaSuccess;
  switch (p.scaling) {
    case TB200_SCALE_NONE:
      e = cudaFuncSetAttribute(resize_pack_kernel<C, DST, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e == cudaSuccess) resize_pack_kernel<C, DST, 0><<<grid, 256, p.smem_bytes, s>>>(p);
      break;
    case TB200_SCALE_INCEPTION:
      e = cudaFuncSetAttribute(resize_pack_kernel<C, DST, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e == cudaSuccess) resize_pack_kernel<C, DST, 1><<<grid, 256, p.smem_bytes, s>>>(p);
      break;
    default:
      e = cudaFuncSetAttribute(resize_pack_kernel<C, DST, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
      if (e == cudaSuccess) resize_pack_kernel<C, DST, 2><<<grid, 256, p.smem_bytes, s>>>(p);
      break;
  }
  return e != cudaSuccess ? e : cudaGetLastError();
}

template <int C>
static cudaError_t launch_resize_dtype(const ResizePack& p, dim3 grid, cudaStream_t s) {
  switch (p.dst_dtype) {
    case kF32: return launch_resize_scaling<C, kF32>(p, grid, s);
    case kF16: return launch_resize_scaling<C, kF16>(p, grid, s);
    case kBF16: return launch_resize_scaling<C, kBF16>(p, grid, s);
    default: return launch_resize_scaling<C, kU8>(p, grid, s);
  }
}

cudaError_t launch_resize_pack(const ResizePack& p, cudaStream_t s) {
  dim3 grid((p.dw + 31) / 32, (p.dh + p.tile_h - 1) / p.tile_h, p.n);
  return p.c == 1 ? launch_resize_dtype<1>(p, grid, s) : launch_resize_dtype<3>(p, grid, s);
}

template <uint32_t DST, int C>
static cudaError_t launch_pack_tma(const ImagePack& p, int sm_count, cudaStream_t s) {
  using T = PackTraits<DST>;
  const uint32_t hw = static_cast<uint32_t>(p.h) * static_cast<uint32_t>(p.w);
  const uint32_t tpi = (hw + T::kTilePx - 1) / T::kTilePx;
  const uint64_t total64 = static_cast<uint64_t>(tpi) * static_cast<uint64_t>(p.n);
  if (total64 > 0xFFFFFFFFull) return cudaErrorInvalidValue;
  const uint32_t total = static_cast<uint32_t>(total64);
  uint32_t grid = static_cast<uint32_t>(sm_count) * 12u;
  if (grid > total) grid = total;
  uint8_t* d = static_cast<uint8_t*>(p.dst);
  switch (p.scaling) {
    case TB200_SCALE_NONE:
      pack_image_chw_tma_kernel<DST, C, 0><<<grid, kPackThreads, 0, s>>>(d, p.src, hw, tpi, total);
      break;
    case TB200_SCALE_INCEPTION:
      pack_image_chw_tma_kernel<DST, C, 1><<<grid, kPackThreads, 0, s>>>(d, p.src, hw, tpi, total);
      break;
    default:
      pack_image_chw_tma_kernel<DST, C, 2><<<grid, kPackThreads, 0, s>>>(d, p.src, hw, tpi, total);
      break;
  }
  return cudaGetLastError();
}

cudaError_t launch_pack_image(const ImagePack& p, int sm_count, cudaStream_t s, int* launches) {
  if (p.n <= 0 || p.h <= 0 || p.w <= 0 || p.c <= 0) return cudaErrorInvalidValue;
  if (p.dst_dtype != kF16 && p.dst_dtype != kF32 && p.dst_dtype != kBF16) return cudaErrorInvalidValue;
  if (p.scaling > TB200_SCALE_VGG) return cudaErrorInvalidValue;
  if (p.scaling == TB200_SCALE_VGG && p.c != 1 && p.c != 3) return cudaErrorInvalidValue;
  *launches = 1;
  const uint64_t hw = static_cast<uint64_t>(p.h) * p.w;
  const int ppt = (p.dst_dtype == kF32) ? 4 : 8;
  const bool tma_ok = p.layout == TB200_NCHW && (p.c == 3 || p.c == 1) &&
                      (reinterpret_cast<uintptr_t>(p.src) & 15) == 0 &&
                      (reinterpret_cast<uintptr_t>(p.dst) & 15) == 0 &&
                      (hw * p.c) % 16 == 0 && hw % ppt == 0 && hw < (1ull << 31);
  if (tma_ok) {
    if (p.c == 3) {
      if (p.dst_dtype == kF16) return launch_pack_tma<kF16, 3>(p, sm_count, s);
      if (p.dst_dtype == kF32) return launch_pack_tma<kF32, 3>(p, sm_count, s);
      return launch_pack_tma<kBF16, 3>(p, sm_count, s);
    }
    if (p.dst_dtype == kF16) return launch_pack_tma<kF16, 1>(p, sm_count, s);
    if (p.dst_dtype == kF32) return launch_pack_tma<kF32, 1>(p, sm_count, s);
    return launch_pack_tma<kBF16, 1>(p, sm_count, s);
  }
  const uint64_t total = hw * p.c * p.n;
  uint64_t blocks = (total + 255) / 256;
  const uint64_t cap = static_cast<uint64_t>(sm_count) * 16;
  if (blocks > cap) blocks = cap;
  pack_image_generic_kernel<<<static_cast<uint32_t>(blocks), 256, 0, s>>>(
      static_cast<uint8_t*>(p.dst), p.src, p.dst_dtype, p.layout, p.scaling,
      static_cast<uint32_t>(p.c), hw, total);
  return cudaGetLastError();
}

// =============================================================================
// Kernel 2b: contiguous cast (numpy astype semantics)
// =============================================================================
struct HalfBits { uint16_t v; };
struct Bf16Bits { uint16_t v; };
struct BoolByte { uint8_t v; };

template <uint32_t DT> struct CType;
template <> struct CType<kBool> { using type = BoolByte; };
template <> struct CType<kU8> { using type = uint8_t; };
template <> struct CType<kI8> { using type = int8_t; };
template <> struct CType<kU16> { using type = uint16_t; };
template <> struct CType<kI16> { using type = int16_t; };
template <> struct CType<kU32> { using type = uint32_t; };
template <> struct CType<kI32> { using type = int32_t; };
template <> struct CType<kU64> { using type = uint64_t; };
template <> struct CType<kI64> { using type = int64_t; };
template <> struct CType<kF16> { using type = HalfBits; };
template <> struct CType<kBF16> { using type = Bf16Bits; };
template <> struct CType<kF32> { using type = float; };
template <> struct CType<kF64> { using type = double; };

// source -> "wide" value that represents it exactly
__device__ __forceinline__ int64_t widen(BoolByte x) { return x.v != 0; }
__device__ __forceinline__ int64_t widen(uint8_t x) { return x; }
__device__ __forceinline__ int64_t widen(int8_t x) { return x; }
__device__ __forceinline__ int64_t widen(uint16_t x) { return x; }
__device__ __forceinline__ int64_t widen(int16_t x) { return x; }
__device__ __forceinline__ int64_t widen(uint32_t x) { return x; }
__device__ __forceinline__ int64_t widen(int32_t x) { return x; }
__device__ __forceinline__ int64_t widen(int64_t x) { return x; }
__device__ __forceinline__ float widen(HalfBits x) { return f16_bits_to_f32(x.v); }
__device__ __forceinline__ float widen(Bf16Bits x) { return bits_f32(static_cast<uint32_t>(x.v) << 16); }
__device__ __forceinline__ float widen(float x) { return x; }
__device__ __forceinline__ double widen(double x) { return x; }

template <typename D> struct Narrow;
template <> struct Narrow<HalfBits> {
  // only reached from <=16-bit integers (exact in fp32) and from fp32
  __device__ static HalfBits from(int64_t v) { return HalfBits{f32_to_f16_bits(static_cast<float>(v))}; }
  __device__ static HalfBits from(float v) { return HalfBits{f32_to_f16_bits(v)}; }
  __device__ static HalfBits from(double v) { return HalfBits{__half_as_ushort(__double2half(v))}; }
};
template <> struct Narrow<Bf16Bits> {
  __device__ static Bf16Bits from(int64_t v) { return Bf16Bits{f32_to_bf16_trunc(static_cast<float>(v))}; }
  __device__ static Bf16Bits from(float v) { return Bf16Bits{f32_to_bf16_trunc(v)}; }
  __device__ static Bf16Bits from(double v) { return Bf16Bits{f32_to_bf16_trunc(static_cast<float>(v))}; }
};
template <> struct Narrow<float> {
  __device__ static float from(int64_t v) { return __ll2float_rn(v); }
  __device__ static float from(float v) { return v; }
  __device__ static float from(double v) { return __double2float_rn(v); }
};
template <> struct Narrow<double> {
  __device__ static double from(int64_t v) { return __ll2double_rn(v); }
  __device__ static double from(float v) { return static_cast<double>(v); }
  __device__ static double from(double v) { return v; }
};
template <> struct Narrow<int32_t> {
  __device__ static int32_t from(int64_t v) { return static_cast<int32_t>(v); }  // wraps like numpy
  __device__ static int32_t from(float v) { return static_cast<int32_t>(v); }
  __device__ static int32_t from(double v) { return static_cast<int32_t>(v); }
};
template <> struct Narrow<int64_t> {
  __device__ static int64_t from(int64_t v) { return v; }
  __device__ static int64_t from(float v) { return static_cast<int64_t>(v); }
  __device__ static int64_t from(double v) { return static_cast<int64_t>(v); }
};

template <int BYTES> struct VecOf;
template <> struct VecOf<16> { using type = uint4; };
template <> struct VecOf<8> { using type = uint2; };
template <> struct VecOf<4> { using type = uint32_t; };
template <> struct VecOf<2> { using type = uint16_t; };
template <> struct VecOf<1> { using type = uint8_t; };

template <uint32_t SRC, uint32_t DST>
__global__ void __launch_bounds__(256)
cast_kernel(void* __restrict__ dst_v, const void* __restrict__ src_v, uint64_t nelem, int vec_ok) {
  using S = typename CType<SRC>::type;
  using D = typename CType<DST>::type;
  constexpr int SS = sizeof(S), DS = sizeof(D);
  constexpr int E = 16 / (SS > DS ? SS : DS);  // elements per thread-iteration
  using VS = typename VecOf<E * SS>::type;
  using VD = typename VecOf<E * DS>::type;
  const S* src = static_cast<const S*>(src_v);
  D* dst = static_cast<D*>(dst_v);
  const uint64_t nvec = vec_ok ? nelem / E : 0;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; v < nvec; v += stride) {
    union { VS vec; S e[E]; } in;
    union { VD vec; D e[E]; } out;
    in.vec = reinterpret_cast<const VS*>(src)[v];
#pragma unroll
    for (int k = 0; k < E; ++k) out.e[k] = Narrow<D>::from(widen(in.e[k]));
    reinterpret_cast<VD*>(dst)[v] = out.vec;
  }
  // scalar tail (and the whole tensor when the pointers are not vector aligned)
  for (uint64_t i = nvec * E + blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; i < nelem;
       i += stride) {
    dst[i] = Narrow<D>::from(widen(src[i]));
  }
}

template <uint32_t SRC, uint32_t DST>
static cudaError_t launch_cast_t(void* dst, const void* src, uint64_t nelem, int sm_count, cudaStream_t s) {
  using S = typename CType<SRC>::type;
  using D = typename CType<DST>::type;
  constexpr int E = 16 / (sizeof(S) > sizeof(D) ? sizeof(S) : sizeof(D));
  const int vec_ok = (reinterpret_cast<uintptr_t>(src) % (E * sizeof(S)) == 0) &&
                     (reinterpret_cast<uintptr_t>(dst) % (E * sizeof(D)) == 0);
  uint64_t blocks = (nelem / E + 255) / 256 + 1;
  const uint64_t cap = static_cast<uint64_t>(sm_count) * 16;
  if (blocks > cap) blocks = cap;
  cast_kernel<SRC, DST><<<static_cast<uint32_t>(blocks), 256, 0, s>>>(dst, src, nelem, vec_ok);
  return cudaGetLastError();
}

#define TB200_CAST_PAIRS(X)                                                        \
  X(kBool, kF16) X(kBool, kF32) X(kU8, kF16) X(kU8, kF32) X(kU8, kBF16)            \
  X(kI8, kF16) X(kI8, kF32) X(kU16, kF16) X(kU16, kF32) X(kI16, kF16) X(kI16, kF32) \
  X(kI32, kF32) X(kI32, kF64) X(kI32, kI64) X(kU32, kF32) X(kU32, kI64)            \
  X(kI64, kI32) X(kI64, kF32) X(kI64, kF64)                                        \
  X(kF16, kF32) X(kBF16, kF32) X(kF32, kF16) X(kF32, kBF16) X(kF32, kF64)          \
  X(kF64, kF32) X(kF64, kF16)

bool cast_supported(uint32_t src_dtype, uint32_t dst_dtype) {
  if (src_dtype == dst_dtype) return src_dtype != kBytes && tb200_dtype_size(src_dtype) != 0;
#define X(S, D) if (src_dtype == S && dst_dtype == D) return true;
  TB200_CAST_PAIRS(X)
#undef X
  return false;
}

__global__ void __launch_bounds__(256)
copy_bytes_kernel(uint8_t* __restrict__ dst, const uint8_t* __restrict__ src, uint64_t nbytes, int vec_ok) {
  const uint64_t nvec = vec_ok ? nbytes / 16 : 0;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  const uint64_t t = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x;
  for (uint64_t v = t; v < nvec; v += stride) {
    const uint4 x = ld_nc_v4(src + v * 16);
    st_cs_v4(dst + v * 16, U32x4{x.x, x.y, x.z, x.w});
  }
  for (uint64_t i = nvec * 16 + t; i < nbytes; i += stride) dst[i] = src[i];
}

cudaError_t launch_cast(void* dst, uint32_t dst_dtype, const void* src, uint32_t src_dtype,
                        uint64_t nelem, int sm_count, cudaStream_t s) {
  if (nelem == 0) return cudaSuccess;
  if (src_dtype == dst_dtype) {
    const uint64_t nbytes = nelem * tb200_dtype_size(src_dtype);
    const int vec_ok = ((reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst)) & 15) == 0;
    uint64_t blocks = (nbytes / 16 + 255) / 256 + 1;
    const uint64_t cap = static_cast<uint64_t>(sm_count) * 16;
    if (blocks > cap) blocks = cap;
    copy_bytes_kernel<<<static_cast<uint32_t>(blocks), 256, 0, s>>>(
        static_cast<uint8_t*>(dst), static_cast<const uint8_t*>(src), nbytes, vec_ok);
    return cudaGetLastError();
  }
#define X(S, D) if (src_dtype == S && dst_dtype == D) return launch_cast_t<S, D>(dst, src, nelem, sm_count, s);
  TB200_CAST_PAIRS(X)
#undef X
  return cudaErrorInvalidValue;
}

// =============================================================================
// Kernel 2c: strided -> contiguous (ndarray.tobytes() of a non-contiguous array)
// =============================================================================
template <int ES> struct ElemOf;
template <> struct ElemOf<1> { using type = uint8_t; };
template <> struct ElemOf<2> { using type = uint16_t; };
template <> struct ElemOf<4> { using type = uint32_t; };
template <> struct ElemOf<8> { using type = uint64_t; };

template <int ES>
__global__ void __launch_bounds__(256) pack_strided_kernel(const StridedPack P, int vec_ok) {
  using ET = typename ElemOf<ES>::type;
  constexpr int E = 16 / ES;
  const uint8_t* src = static_cast<const uint8_t*>(P.src);
  uint8_t* dst = static_cast<uint8_t*>(P.dst);
  const uint64_t nchunk = (P.nelem + E - 1) / E;
  const uint64_t stride = static_cast<uint64_t>(gridDim.x) * blockDim.x;
  for (uint64_t v = blockIdx.x * static_cast<uint64_t>(blockDim.x) + threadIdx.x; v < nchunk; v += stride) {
    const uint64_t first = v * E;
    // mixed-radix decomposition of the first element, then odometer increments
    int64_t idx[TB200_MAX_DIMS];
    int64_t off = 0;
    uint64_t rem = first;
#pragma unroll
    for (int d = TB200_MAX_DIMS - 1; d >= 0; --d) {
      idx[d] = 0;
      if (d < P.ndim) {
        const uint64_t ext = static_cast<uint64_t>(P.shape[d]);
        const uint64_t q = rem / ext;
        idx[d] = static_cast<int64_t>(rem - q * ext);
        rem = q;
        off += idx[d] * P.strides[d];
      }
    }
    union { uint4 vec; ET e[E]; } out;
    out.vec = make_uint4(0, 0, 0, 0);
    const int count = (P.nelem - first) < static_cast<uint64_t>(E) ? static_cast<int>(P.nelem - first) : E;
#pragma unroll
    for (int k = 0; k < E; ++k) {
      if (k < count) {
        out.e[k] = *reinterpret_cast<const ET*>(src + off);
        // advance the odometer by one element
        bool carry = true;
#pragma unroll
        for (int d = TB200_MAX_DIMS - 1; d >= 0; --d) {
          if (d < P.ndim && carry) {
            idx[d] += 1;
            off += P.strides[d];
            if (idx[d] == P.shape[d]) {
              off -= P.strides[d] * P.shape[d];
              idx[d] = 0;
            } else {
              carry = false;
            }
          }
        }
      }
    }
    if (count == E && vec_ok) {
      st_cs_v4(dst + first * ES, U32x4{out.vec.x, out.vec.y, out.vec.z, out.vec.w});
    } else {
      for (int k = 0; k < count; ++k) reinterpret_cast<ET*>(dst)[first + k] = out.e[k];
    }
  }
}

cudaError_t launch_pack_strided(const StridedPack& p, int sm_count, cudaStream_t s) {
  if (p.nelem == 0) return cudaSuccess;
  const int vec_ok = (reinterpret_cast<uintptr_t>(p.dst) & 15) == 0;
  const uint64_t e = 16 / p.elem_size;
  uint64_t blocks = ((p.nelem + e - 1) / e + 255) / 256;
  const uint64_t cap = static_cast<uint64_t>(sm_count) * 16;
  if (blocks > cap) blocks = cap;
  const uint32_t g = static_cast<uint32_t>(blocks);
  switch (p.elem_size) {
    case 1: pack_strided_kernel<1><<<g, 256, 0, s>>>(p, vec_ok); break;
    case 2: pack_strided_kernel<2><<<g, 256, 0, s>>>(p, vec_ok); break;
    case 4: pack_strided_kernel<4><<<g, 256, 0, s>>>(p, vec_ok); break;
    case 8: pack_strided_kernel<8><<<g, 256, 0, s>>>(p, vec_ok); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

// =============================================================================
// Kernel 2d: concat (N copies in one launch)
// =============================================================================
__global__ void __launch_bounds__(256) concat_kernel(const CopyLaunch L) {
  for (uint32_t tile = blockIdx.x; tile < L.total_tiles; tile += gridDim.x) {
    const uint32_t j = find_job(L.tile_prefix, L.njobs, tile);
    const uint32_t lt = tile - __ldg(L.tile_prefix + j);
    const tb200_copy_job jb = L.jobs[j];
    const uint8_t* src = reinterpret_cast<const uint8_t*>(jb.src);
    uint8_t* dst = reinterpret_cast<uint8_t*>(jb.dst);
    const uint64_t begin = static_cast<uint64_t>(lt) * kCopyTileBytes;
    const uint64_t end = (begin + kCopyTileBytes < jb.nbytes) ? begin + kCopyTileBytes : jb.nbytes;
    if (((jb.src | jb.dst) & 15) == 0) {
      const uint64_t nvec = (end - begin) / 16;
      for (uint64_t v = threadIdx.x; v < nvec; v += blockDim.x) {
        const uint4 x = ld_nc_v4(src + begin + v * 16);
        st_cs_v4(dst + begin + v * 16, U32x4{x.x, x.y, x.z, x.w});
      }
      for (uint64_t i = begin + nvec * 16 + threadIdx.x; i < end; i += blockDim.x) dst[i] = src[i];
    } else {
      for (uint64_t i = begin + threadIdx.x; i < end; i += blockDim.x) dst[i] = src[i];
    }
  }
}

cudaError_t launch_concat(const CopyLaunch& l, int sm_count, cudaStream_t s) {
  if (l.total_tiles == 0) return cudaSuccess;
  uint32_t grid = static_cast<uint32_t>(sm_count) * 8u;
  if (grid > l.total_tiles) grid = l.total_tiles;
  concat_kernel<<<grid, 256, 0, s>>>(l);
  return cudaGetLastError();
}

// =============================================================================
// Kernel 3: check
// =============================================================================
__device__ __forceinline__ uint32_t load_word(const uint8_t* p, uint64_t off, uint64_t nbytes, bool aligned4) {
  // little-endian u32 at byte `off`, zero-extended past nbytes
  if (aligned4 && off + 4 <= nbytes) return *reinterpret_cast<const uint32_t*>(p + off);
  uint32_t w = 0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    if (off + k < nbytes) w |= static_cast<uint32_t>(p[off + k]) << (8 * k);
  }
  return w;
}
__device__ __forceinline__ uint32_t differing_bytes(uint32_t x, uint32_t y) {
  const uint32_t d = x ^ y;
  return ((d & 0xFFu) != 0) + ((d & 0xFF00u) != 0) + ((d & 0xFF0000u) != 0) + ((d & 0xFF000000u) != 0);
}
__device__ __forceinline__ uint32_t f32_order_key(uint32_t b) {
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

struct CheckLocal {
  unsigned long long mism = 0, sum = 0, best = 0;
  uint32_t x = 0;
};
__device__ __forceinline__ void check_word(CheckLocal& acc, uint32_t kind, uint32_t wa, uint32_t wb,
                                           uint32_t wc, uint32_t wd, uint64_t word_index) {
  acc.sum += wa;
  acc.x ^= wa;
  if (kind == TB200_CHECK_EQUAL) {
    acc.mism += differing_bytes(wa, wb);
  } else if (kind == TB200_CHECK_ADDSUB) {
    acc.mism += (wa != wc + wd) + (wb != wc - wd);
  } else if (kind == TB200_CHECK_TOP1) {
    const uint32_t absb = wa & 0x7FFFFFFFu;
    if (absb >= 0x7F800000u) acc.mism += 1;
    if (absb <= 0x7F800000u) {  // not NaN; -0.0 compares equal to +0.0
      const unsigned long long cand =
          (static_cast<unsigned long long>(f32_order_key(absb == 0 ? 0u : wa)) << 32) |
          (0xFFFFFFFFull - (word_index & 0xFFFFFFFFull));
      if (cand > acc.best) acc.best = cand;
    }
  }
}

__global__ void __launch_bounds__(256) check_kernel(const CheckLaunch L) {
  const uint32_t j = blockIdx.y;
  const tb200_check_job jb = L.jobs[j];
  const uint64_t begin = static_cast<uint64_t>(blockIdx.x) * kCheckChunkBytes;
  if (begin >= jb.nbytes && !(jb.nbytes == 0 && blockIdx.x == 0)) return;
  const uint64_t end = (jb.nbytes == 0) ? begin : ((begin + kCheckChunkBytes < jb.nbytes) ? begin + kCheckChunkBytes : jb.nbytes);
  const uint8_t* a = reinterpret_cast<const uint8_t*>(jb.a);
  const uint8_t* b = reinterpret_cast<const uint8_t*>(jb.b);
  const uint8_t* c = reinterpret_cast<const uint8_t*>(jb.c);
  const uint8_t* d = reinterpret_cast<const uint8_t*>(jb.d);
  const uint32_t kind = jb.kind;
  const bool need_b = kind == TB200_CHECK_EQUAL || kind == TB200_CHECK_ADDSUB;
  const bool need_cd = kind == TB200_CHECK_ADDSUB;

  CheckLocal acc;
  uint64_t mask = jb.a;
  if (need_b) mask |= jb.b;
  if (need_cd) mask |= jb.c | jb.d;
  const uint64_t nvec = ((mask & 15) == 0) ? (end - begin) / 16 : 0;
  for (uint64_t v = threadIdx.x; v < nvec; v += blockDim.x) {
    const uint64_t off = begin + v * 16;
    const uint4 va = ld_nc_v4(a + off);
    uint4 vb = make_uint4(0, 0, 0, 0), vc = vb, vd = vb;
    if (need_b) vb = ld_nc_v4(b + off);
    if (need_cd) {
      vc = ld_nc_v4(c + off);
      vd = ld_nc_v4(d + off);
    }
    const uint64_t w0 = off / 4;
    check_word(acc, kind, va.x, vb.x, vc.x, vd.x, w0);
    check_word(acc, kind, va.y, vb.y, vc.y, vd.y, w0 + 1);
    check_word(acc, kind, va.z, vb.z, vc.z, vd.z, w0 + 2);
    check_word(acc, kind, va.w, vb.w, vc.w, vd.w, w0 + 3);
  }
  // remaining words (unaligned buffers take this path for the whole chunk)
  const bool al4 = (mask & 3) == 0;
  const uint64_t tail0 = begin + nvec * 16;  // chunk starts are multiples of 1 MiB
  const uint64_t nwords = (end - tail0 + 3) / 4;
  for (uint64_t w = threadIdx.x; w < nwords; w += blockDim.x) {
    const uint64_t off = tail0 + w * 4;
    const uint32_t wa = load_word(a, off, jb.nbytes, al4);
    const uint32_t wb = need_b ? load_word(b, off, jb.nbytes, al4) : 0;
    const uint32_t wc = need_cd ? load_word(c, off, jb.nbytes, al4) : 0;
    const uint32_t wd = need_cd ? load_word(d, off, jb.nbytes, al4) : 0;
    check_word(acc, kind, wa, wb, wc, wd, off / 4);
  }

  // block reduction: warp shuffles, then the warp leaders through shared memory
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    acc.mism += __shfl_xor_sync(0xFFFFFFFFu, acc.mism, o);
    acc.sum += __shfl_xor_sync(0xFFFFFFFFu, acc.sum, o);
    acc.x ^= __shfl_xor_sync(0xFFFFFFFFu, acc.x, o);
    const unsigned long long ob = __shfl_xor_sync(0xFFFFFFFFu, acc.best, o);
    if (ob > acc.best) acc.best = ob;
  }
  __shared__ unsigned long long s_m[8], s_s[8], s_b[8];
  __shared__ uint32_t s_x[8];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane == 0) {
    s_m[warp] = acc.mism; s_s[warp] = acc.sum; s_b[warp] = acc.best; s_x[warp] = acc.x;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  unsigned long long m = 0, sm = 0, bst = 0;
  uint32_t x = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    m += s_m[k]; sm += s_s[k]; x ^= s_x[k];
    if (s_b[k] > bst) bst = s_b[k];
  }
  const uint32_t nchunks = static_cast<uint32_t>((jb.nbytes + kCheckChunkBytes - 1) / kCheckChunkBytes);
  if (nchunks > 1) {
    // several CTAs share the job: combine through the accumulator, the last one finalizes
    // and leaves the accumulator zeroed for the next launch
    CheckAccum* ac = L.accum + j;
    if (m) atomicAdd(&ac->mismatches, m);
    atomicAdd(&ac->sum, sm);
    atomicXor(&ac->xor32, x);
    if (bst) atomicMax(&ac->best, bst);
    __threadfence();
    if (atomicInc(&ac->done, nchunks - 1) != nchunks - 1) return;
    __threadfence();
    m = atomicExch(&ac->mismatches, 0ull);
    sm = atomicExch(&ac->sum, 0ull);
    bst = atomicExch(&ac->best, 0ull);
    x = atomicExch(&ac->xor32, 0u);
  }
  tb200_check_result r;
  r.mismatches = m;
  r.sum = sm;
  r.xor32 = x;
  r.pad = 0;
  if (bst == 0) {
    r.argmax = 0xFFFFFFFFu;
    r.max_value = 0.0f;
  } else {
    const uint32_t key = static_cast<uint32_t>(bst >> 32);
    const uint32_t bits = (key & 0x80000000u) ? (key & 0x7FFFFFFFu) : ~key;
    r.argmax = 0xFFFFFFFFu - static_cast<uint32_t>(bst & 0xFFFFFFFFull);
    r.max_value = bits_f32(bits);
  }
  L.results[j] = r;
  __threadfence_system();  // results may live in mapped host memory
}

cudaError_t launch_check(const CheckLaunch& l, cudaStream_t s) {
  if (l.njobs == 0) return cudaSuccess;
  dim3 grid(l.max_chunks == 0 ? 1 : l.max_chunks, l.njobs);
  check_kernel<<<grid, 256, 0, s>>>(l);
  return cudaGetLastError();
}

// ---- top-k ---------------------------------------------------------------------------
// One CTA per vector; pass r selects the best element strictly after pass r-1's pick in the
// total order (value desc, index asc): composite = order_key(value) << 32 | ~index, larger
// is better, NaN has key 0.  k passes over a vector that sits in L1/L2 after the first.
__device__ __forceinline__ float topk_load(const void* src, uint32_t dtype, uint32_t i) {
  if (dtype == TB200_FP32) return static_cast<const float*>(src)[i];
  const uint16_t h = static_cast<const uint16_t*>(src)[i];
  if (dtype == TB200_FP16) return f16_bits_to_f32(h);
  return __uint_as_float(static_cast<uint32_t>(h) << 16);  // BF16
}
__device__ __forceinline__ unsigned long long topk_composite(float v, uint32_t i) {
  uint32_t key = 0;
  if (v == v) key = f32_order_key(v == 0.0f ? 0u : __float_as_uint(v));
  return (static_cast<unsigned long long>(key) << 32) | (0xFFFFFFFFu - i);
}

__global__ void __launch_bounds__(256) topk_kernel(const tb200_topk_job* __restrict__ jobs, uint32_t k,
                                                   tb200_topk_entry* __restrict__ out) {
  __shared__ unsigned long long warp_best[8];
  __shared__ unsigned long long picked;
  const tb200_topk_job job = jobs[blockIdx.x];
  const void* src = reinterpret_cast<const void*>(job.src);
  const uint32_t n = static_cast<uint32_t>(job.count);
  tb200_topk_entry* dst = out + static_cast<size_t>(blockIdx.x) * k;
  unsigned long long prev = ~0ull;
  for (uint32_t r = 0; r < k; ++r) {
    unsigned long long best = 0;
    if (prev != 0) {
      for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const unsigned long long c = topk_composite(topk_load(src, job.dtype, i), i);
        if (c < prev && c > best) best = c;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const unsigned long long o = __shfl_xor_sync(0xFFFFFFFFu, best, off);
      best = o > best ? o : best;
    }
    if ((threadIdx.x & 31) == 0) warp_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long b = warp_best[0];
      for (int w = 1; w < 8; ++w) b = warp_best[w] > b ? warp_best[w] : b;
      picked = b;
      tb200_topk_entry e;
      if (b != 0) {
        e.index = 0xFFFFFFFFu - static_cast<uint32_t>(b);
        e.value = topk_load(src, job.dtype, e.index);
      } else {
        e.index = 0xFFFFFFFFu;
        e.value = 0.0f;
      }
      dst[r] = e;
    }
    __syncthreads();
    prev = picked;  // rewritten only after the next pass's barrier
  }
  if (threadIdx.x == 0) __threadfence_system();  // out may live in mapped host memory
}

cudaError_t launch_topk(const tb200_topk_job* jobs, uint32_t njobs, uint32_t k, tb200_topk_entry* out, cudaStream_t s) {
  if (njobs == 0) return cudaSuccess;
  topk_kernel<<<njobs, 256, 0, s>>>(jobs, k, out);
  return cudaGetLastError();
}

// =============================================================================
// BYTES decode: the <u32 length><payload> chain of serialize_byte_tensor, on the device
// =============================================================================
// Reference: deserialize_bytes_tensor (PY/utils/__init__.py:264-291) and the BYTES branch of
// cuda_shared_memory.get_contents_as_numpy (:306-323) walk the chain on the host after copying
// the whole region.  The walk is a chain of dependent loads -- the offset of element i+1 is
// known only after the length of element i -- so one CTA stages the stream through shared
// memory in 32 KiB windows (coalesced 16-byte loads by all threads) and one thread follows the
// chain inside the window (a shared-memory load per element instead of an L2 round trip);
// strings longer than the window are skipped over without being staged.  The walk records
// where every payload starts in the source and the prefix sums of the payload lengths; a
// second, fully parallel kernel packs the payloads back to back.  Only offsets[count + 1] and
// the packed payload bytes have to cross PCIe, not the region.
constexpr uint32_t kBytesWindow = 32768;

__global__ void __launch_bounds__(256) bytes_scan_kernel(const uint8_t* __restrict__ src, uint64_t src_bytes, uint64_t count,
                                                          uint64_t* __restrict__ src_off, uint32_t* __restrict__ offsets,
                                                          uint64_t* __restrict__ status) {
  __shared__ __align__(16) uint8_t win[kBytesWindow + 16];
  __shared__ uint64_t s_pos, s_done, s_total;
  __shared__ uint32_t s_err;
  if (threadIdx.x == 0) {
    s_pos = 0;
    s_done = 0;
    s_total = 0;
    s_err = 0;
    offsets[0] = 0;
  }
  __syncthreads();
  const uintptr_t base_addr = reinterpret_cast<uintptr_t>(src);
  while (true) {
    const uint64_t pos = s_pos, done = s_done;
    if (done >= count || s_err != 0 || pos >= src_bytes) break;
    // window: starts at the 16-byte aligned address at or below src + pos (for pos = 0 and an
    // unaligned src that is up to 15 bytes before the tensor, inside the same 16-byte cell of
    // the allocation)
    const uint64_t lead = (base_addr + pos) & 15;
    const int64_t w0 = static_cast<int64_t>(pos) - static_cast<int64_t>(lead);  // stream offset of the window's first byte
    const uint8_t* wsrc = reinterpret_cast<const uint8_t*>((base_addr + pos) & ~static_cast<uintptr_t>(15));
    const uint64_t avail = src_bytes - pos + lead;
    const uint32_t wbytes = static_cast<uint32_t>(avail < kBytesWindow ? avail : kBytesWindow);
    for (uint32_t i = threadIdx.x * 16; i < wbytes; i += blockDim.x * 16) {
      if (i + 16 <= wbytes) {
        *reinterpret_cast<uint4*>(win + i) = ld_nc_v4(wsrc + i);
      } else {
        for (uint32_t b = i; b < wbytes; ++b) win[b] = wsrc[b];
      }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      uint64_t p = pos, n = done, total = s_total;
      const int64_t wend = w0 + wbytes;  // stream offset one past the window
      while (n < count) {
        if (p + 4 > src_bytes) {
          s_err = 1;  // truncated: no room for a length word
          break;
        }
        if (static_cast<int64_t>(p + 4) > wend) break;  // header not (fully) staged: next window
        const uint32_t o = static_cast<uint32_t>(static_cast<int64_t>(p) - w0);
        const uint32_t len = static_cast<uint32_t>(win[o]) | (static_cast<uint32_t>(win[o + 1]) << 8) |
                             (static_cast<uint32_t>(win[o + 2]) << 16) | (static_cast<uint32_t>(win[o + 3]) << 24);
        if (len > src_bytes - (p + 4)) {
          s_err = 2;  // payload runs past the end of the source
          break;
        }
        if (total + len > 0xFFFFFFFFull) {
          s_err = 3;  // offsets are 32-bit, as in numpy's per-element view of the packed buffer
          break;
        }
        src_off[n] = p + 4;
        total += len;
        ++n;
        offsets[n] = static_cast<uint32_t>(total);
        p += 4ull + len;
      }
      s_pos = p;
      s_done = n;
      s_total = total;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    status[0] = s_done;
    status[1] = s_pos;
    status[2] = s_total;
    status[3] = s_err != 0 ? s_err : (s_done < count ? 1u : 0u);
    __threadfence_system();
  }
}

// one warp per element (grid-stride): payload bytes to packed + offsets[i]
__global__ void __launch_bounds__(256) bytes_gather_kernel(const uint8_t* __restrict__ src, const uint64_t* __restrict__ src_off,
                                                            const uint32_t* __restrict__ offsets, const uint64_t* __restrict__ status,
                                                            uint8_t* __restrict__ packed, uint64_t packed_capacity) {
  const uint64_t n = status[0];
  if (status[3] != 0 || status[2] > packed_capacity) return;
  const uint32_t lane = threadIdx.x & 31;
  const uint64_t warps = static_cast<uint64_t>(gridDim.x) * (blockDim.x >> 5);
  for (uint64_t i = static_cast<uint64_t>(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5); i < n; i += warps) {
    const uint8_t* from = src + src_off[i];
    uint8_t* to = packed + offsets[i];
    const uint32_t len = offsets[i + 1] - offsets[i];
    for (uint32_t b = lane; b < len; b += 32) to[b] = from[b];
  }
}

cudaError_t launch_bytes_decode(const uint8_t* src, uint64_t src_bytes, uint64_t count, uint64_t* src_off, uint32_t* offsets,
                                uint8_t* packed, uint64_t packed_capacity, uint64_t* status, int sm_count, cudaStream_t s) {
  bytes_scan_kernel<<<1, 256, 0, s>>>(src, src_bytes, count, src_off, offsets, status);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || count == 0) return e;
  uint64_t grid = (count + 7) / 8;
  if (grid > static_cast<uint64_t>(sm_count) * 8) grid = static_cast<uint64_t>(sm_count) * 8;
  bytes_gather_kernel<<<static_cast<uint32_t>(grid), 256, 0, s>>>(src, src_off, offsets, status, packed, packed_capacity);
  return cudaGetLastError();
}

__global__ void epoch_bump_kernel(uint64_t* e, uint64_t delta) { *e += delta; }
cudaError_t launch_epoch_bump(uint64_t* dev_epoch, uint64_t delta, cudaStream_t s) {
  epoch_bump_kernel<<<1, 1, 0, s>>>(dev_epoch, delta);
  return cudaGetLastError();
}

}  // namespace tb200
