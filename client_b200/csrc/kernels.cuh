// kernels.cuh -- launch interface between runtime.cu (contexts, regions, ABI)
// and kernels.cu (the sm_90a kernels).  Internal; the public surface is
// include/tb200.h.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tb200.h"
#include "philox.cuh"

namespace tb200 {

// ---- fill ---------------------------------------------------------------------
struct FillLaunch {
  const tb200_fill_job* jobs;    // device
  const uint64_t* group_prefix;  // device, njobs+1 entries (16-byte groups before job j); unused when uniform
  uint64_t* dev_epoch;           // device or nullptr: added to every stream id
  unsigned int* done_counter;    // device: CTAs finished (wraps), used when bump != 0
  uint64_t seed;
  uint64_t epoch;
  uint64_t bump;                 // != 0: the last CTA adds this to *dev_epoch
  uint64_t total_groups;
  uint64_t uniform_groups;       // >0: every job has exactly this many groups
  uint64_t div_magic;            // floor(2^64 / uniform_groups) + 1 (homogeneous launches)
  uint32_t njobs;
  uint32_t dtype0;               // dtype of job 0 (the dtype of a homogeneous launch)
  uint32_t homogeneous;          // 1: uniform sizes, one dtype/range, random mode, every tensor a
                                 //    16-byte-aligned multiple of 16 bytes -> grid-stride kernel
  uint32_t unaligned_jobs;       // jobs whose dst is not 16-byte aligned (fill_unaligned_kernel's share)
  RoundKeys rk;                  // Philox key schedule of `seed`
};
cudaError_t launch_fill(const FillLaunch& l, int sm_count, cudaStream_t s);

// Homogeneous launches (N tensors of one size, dtype and range, 16-byte aligned -- the N slots
// of one model input, BASELINE configs C2 / C3): the (dst, stream) pairs travel in the kernel
// parameters (constant bank: no table upload, no global load before the first store), the
// dtype is a template parameter and the stream-dependent part of Philox is hoisted per CTA.
constexpr int kFillTabSmall = 64, kFillTabLarge = 256;
template <int CAP>
struct FillTab {
  uint64_t dst[CAP];
  uint64_t stream[CAP];
};
struct FillUniform {
  RoundKeys rk;               // Philox key schedule of the seed
  FillParams p;               // range of the dtype
  const uint64_t* dev_epoch;  // device or nullptr: added to every stream id
  uint64_t epoch;
  uint64_t total_groups;      // njobs * groups_per_job
  uint32_t njobs;
  uint32_t groups_per_job;    // < 2^31
  uint32_t ctas_per_job;      // > 0: CTA b owns rows (b % cpj) + k * cpj of job b / cpj (interleaved rows of
                              //      256 groups); 0: CTA b owns groups [T*b/G, T*(b+1)/G) of the launch
  uint32_t grid;
};
// pdl: launch with the programmatic-stream-serialization attribute (the kernel may start while
// the previous kernel of the stream drains; only set when the two write disjoint memory)
cudaError_t launch_fill_uniform(const FillUniform& u, const tb200_fill_job* host_jobs, uint32_t dtype, cudaStream_t s, bool pdl);
// fills u.ctas_per_job / u.grid for a launch of u.njobs x u.groups_per_job groups
void plan_fill_uniform(FillUniform* u, int sm_count);
// tuning knob for experiments (scripts/fill_sweep.py); 0 = default configuration
void set_fill_variant(int v);

// ---- pack / cast ----------------------------------------------------------------
struct ImagePack {
  void* dst;
  const uint8_t* src;
  uint32_t dst_dtype;  // FP16 / FP32 / BF16
  uint32_t layout;     // TB200_NCHW / TB200_NHWC
  uint32_t scaling;
  int n, h, w, c;
};
// returns cudaErrorInvalidValue for unsupported combinations
cudaError_t launch_pack_image(const ImagePack& p, int sm_count, cudaStream_t s,
                              int* launches);

// resize + cast + scaling + layout (Pillow BILINEAR semantics); tables live on the device
struct ResizePack {
  void* dst;
  const uint8_t* src;
  const int2* hbounds;    // [dst_w] (first source column, taps)
  const int32_t* hcoeffs; // [dst_w * hk]
  const int2* vbounds;    // [dst_h] (first source row, taps)
  const int32_t* vcoeffs; // [dst_h * vk]
  uint32_t dst_dtype, layout, scaling;
  int n, sh, sw, c, dh, dw, hk, vk;
  int tile_h;             // output rows per CTA (1..32)
  int max_rows;           // source rows the tallest tile needs
  uint32_t raw_stride;    // bytes per staged source row (widest tile's span * c in whole 16-byte granules)
  uint32_t smem_bytes;    // see resize_pack_kernel
};
cudaError_t launch_resize_pack(const ResizePack& p, cudaStream_t s);

cudaError_t launch_cast(void* dst, uint32_t dst_dtype, const void* src,
                        uint32_t src_dtype, uint64_t nelem, int sm_count,
                        cudaStream_t s);
bool cast_supported(uint32_t src_dtype, uint32_t dst_dtype);

struct StridedPack {
  void* dst;
  const void* src;
  uint32_t elem_size;
  int ndim;
  int64_t shape[TB200_MAX_DIMS];
  int64_t strides[TB200_MAX_DIMS];  // bytes
  uint64_t nelem;
};
cudaError_t launch_pack_strided(const StridedPack& p, int sm_count, cudaStream_t s);

constexpr uint32_t kCopyTileBytes = 16384;
struct CopyLaunch {
  const tb200_copy_job* jobs;   // device
  const uint32_t* tile_prefix;  // device, njobs+1
  uint32_t njobs;
  uint32_t total_tiles;
};
cudaError_t launch_concat(const CopyLaunch& l, int sm_count, cudaStream_t s);

// ---- check ----------------------------------------------------------------------
struct CheckAccum {  // device scratch, one per job; all-zero between launches (self-cleaning)
  unsigned long long mismatches;
  unsigned long long sum;
  unsigned long long best;  // (orderable fp32 key << 32) | (0xFFFFFFFF - index)
  unsigned int xor32;
  unsigned int done;        // chunks of the job finished so far (wraps to 0)
};
constexpr uint32_t kCheckChunkBytes = 1u << 20;  // one CTA per MiB of a job
struct CheckLaunch {
  const tb200_check_job* jobs;  // device
  CheckAccum* accum;            // device, njobs entries
  tb200_check_result* results;  // device or mapped host
  uint32_t njobs;
  uint32_t max_chunks;          // grid.x
};
cudaError_t launch_check(const CheckLaunch& l, cudaStream_t s);

// ---- deflate (deflate.cu) ---------------------------------------------------------
struct DeflateChunkMeta {
  unsigned long long offset;  // of the chunk's bytes in the stream body (set by the finalize kernel)
  uint32_t out_bytes, in_bytes;
  uint32_t adler_a, adler_b;  // Adler-32 piece sums (a from 0)
  uint32_t crc_raw0;          // CRC-32 register over the chunk from init 0, no final xor
  uint32_t pad;
};
cudaError_t launch_deflate(const uint8_t* src, uint64_t nbytes, uint32_t format, uint8_t* scratch, DeflateChunkMeta* meta, uint8_t* dst,
                           uint64_t* out_size, cudaStream_t s);

cudaError_t launch_topk(const tb200_topk_job* jobs, uint32_t njobs, uint32_t k, tb200_topk_entry* out, cudaStream_t s);

// serialised BYTES tensor -> offsets[count + 1] + packed payloads; src_off: device scratch, count entries
cudaError_t launch_bytes_decode(const uint8_t* src, uint64_t src_bytes, uint64_t count, uint64_t* src_off, uint32_t* offsets,
                                uint8_t* packed, uint64_t packed_capacity, uint64_t* status, int sm_count, cudaStream_t s);

cudaError_t launch_epoch_bump(uint64_t* dev_epoch, uint64_t delta, cudaStream_t s);

}  // namespace tb200
