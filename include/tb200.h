/*
 * tb200.h -- C ABI of libtb200.so, the GPU-native data plane behind the
 * tritonclient-compatible Python package `client_b200`.
 *
 * Every entry point is plain C: pointers, sizes, opaque handles.  No torch,
 * numpy or Python types cross this boundary.  The Python drop-in modules
 * (client_b200/utils/cuda_shared_memory, client_b200/perf) bind it with
 * ctypes; INTEGRATION.md shows the stub a tritonclient maintainer would add.
 *
 * Conventions
 *   - every function returns 0 on success and a negative tb200_status on
 *     failure; tb200_last_error() returns the message of the calling thread's
 *     last failure (the Python layer turns it into CudaSharedMemoryException /
 *     InferenceServerException with the reference's message texts).
 *   - all device work of a context is issued on that context's stream; calls
 *     whose name ends in _async return before the work completed.
 *   - the library never falls back to host code for device work: without a
 *     usable CUDA device the calls fail with TB200_ERR_CUDA.
 *
 * Each block cites the reference interface it replaces
 * (paths relative to the reference root, PY = src/python/library/tritonclient).
 */
#ifndef TB200_H_
#define TB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TB200_ABI_VERSION 1

typedef enum tb200_status {
  TB200_OK = 0,
  TB200_ERR_INVALID = -1,  /* bad argument */
  TB200_ERR_CUDA = -2,     /* CUDA runtime/driver failure (message has it) */
  TB200_ERR_RANGE = -3,    /* offset/size outside the region */
  TB200_ERR_NOMEM = -4,
  TB200_ERR_STATE = -5,    /* call not valid in the object's current state */
  TB200_ERR_IO = -6        /* socket / transport failure (load generator) */
} tb200_status;

/* Triton/KServe datatypes. Names and element sizes follow
 * PY/utils/__init__.py:148-205 (np_to_triton_dtype / triton_to_np_dtype) and
 * PY/utils/_dlpack.py:170-216.  BYTES is variable length and never reaches a
 * kernel as an element type. */
typedef enum tb200_dtype {
  TB200_INVALID = 0,
  TB200_BOOL = 1,
  TB200_UINT8 = 2,
  TB200_UINT16 = 3,
  TB200_UINT32 = 4,
  TB200_UINT64 = 5,
  TB200_INT8 = 6,
  TB200_INT16 = 7,
  TB200_INT32 = 8,
  TB200_INT64 = 9,
  TB200_FP16 = 10,
  TB200_FP32 = 11,
  TB200_FP64 = 12,
  TB200_BYTES = 13,
  TB200_BF16 = 14
} tb200_dtype;

/* size in bytes of one element, 0 for BYTES/invalid */
uint32_t tb200_dtype_size(uint32_t dtype);
/* "FP32" -> TB200_FP32 ; unknown -> TB200_INVALID */
uint32_t tb200_dtype_from_name(const char* triton_name);
const char* tb200_dtype_name(uint32_t dtype);

int tb200_abi_version(void);
const char* tb200_last_error(void);
/* number of visible CUDA devices (0 and TB200_ERR_CUDA when there is none) */
int tb200_device_count(int* count);

/* ------------------------------------------------------------------------
 * Context: one device + one stream + scratch (job tables, pinned staging).
 * Replaces the module-global per-device stream cache of
 * PY/utils/cuda_shared_memory/__init__.py:57-70 and _utils.py:103-121.
 * ---------------------------------------------------------------------- */
typedef struct tb200_ctx tb200_ctx;

int tb200_ctx_create(int device_id, tb200_ctx** out);
int tb200_ctx_destroy(tb200_ctx* ctx);
/* use an externally owned cudaStream_t (e.g. torch's current stream) */
int tb200_ctx_set_stream(tb200_ctx* ctx, void* cuda_stream);
void* tb200_ctx_stream(tb200_ctx* ctx);
int tb200_ctx_device(tb200_ctx* ctx);
int tb200_ctx_sync(tb200_ctx* ctx);
/* fork: subsequent launches go to a side stream ordered after everything issued so
 * far; join: the main stream waits for it.  Inside a graph capture this builds two
 * parallel branches (e.g. fill the inputs while the outputs are validated). */
int tb200_ctx_fork(tb200_ctx* ctx);            /* launches now go to the side stream   */
int tb200_ctx_select(tb200_ctx* ctx, int side); /* while forked: 0 = main, 1 = side      */
int tb200_ctx_join(tb200_ctx* ctx);
/* kernels launched by this context since creation (bench.py gpu_launches) */
uint64_t tb200_ctx_launch_count(tb200_ctx* ctx);
int tb200_ctx_sm_count(tb200_ctx* ctx);

/* CUDA-event stopwatch on the context's stream (bench.py times kernels with
 * these because torch.cuda.Event only sees torch's own stream). */
typedef struct tb200_timer tb200_timer;
int tb200_timer_create(tb200_ctx* ctx, tb200_timer** out);
int tb200_timer_start(tb200_timer* t);
int tb200_timer_stop(tb200_timer* t);
/* blocks until the stop event completed; milliseconds between start/stop */
int tb200_timer_elapsed_ms(tb200_timer* t, float* ms);
int tb200_timer_destroy(tb200_timer* t);

/* ------------------------------------------------------------------------
 * CUDA-IPC regions.
 * Replaces PY/utils/cuda_shared_memory/__init__.py:
 *   create_shared_memory_region :107-149   -> tb200_region_create
 *   get_raw_handle              :152-170   -> tb200_region_ipc_handle
 *   set_shared_memory_region    :173-239   -> tb200_region_write_host(+_gather)
 *   get_contents_as_numpy       :242-325   -> tb200_region_read_host
 *   set_..._from_dlpack         :328-388   -> tb200_region_write_ptr
 *   destroy_shared_memory_region:414-429 / _utils.py:88-100 (cudaFree in
 *   __del__)                               -> tb200_region_destroy
 * and, for the server side of the loop (the process that receives the
 * register call of PY/http/_client.py:1129-1175), tb200_region_open.
 * ---------------------------------------------------------------------- */
typedef struct tb200_region tb200_region;

#define TB200_IPC_HANDLE_BYTES 64

int tb200_region_create(const char* name, uint64_t byte_size, int device_id,
                        tb200_region** out);
/* map a region exported by another process (cudaIpcOpenMemHandle) */
int tb200_region_open(const uint8_t ipc_handle[TB200_IPC_HANDLE_BYTES],
                      uint64_t byte_size, int device_id, tb200_region** out);
int tb200_region_destroy(tb200_region* r);
int tb200_region_ipc_handle(const tb200_region* r,
                            uint8_t out[TB200_IPC_HANDLE_BYTES]);
uint64_t tb200_region_base(const tb200_region* r); /* device address */
uint64_t tb200_region_size(const tb200_region* r);
int tb200_region_device(const tb200_region* r);
const char* tb200_region_name(const tb200_region* r);

/* host -> region: multi-threaded pinned staging + async H2D, returns after the
 * bytes are visible on the device (same blocking contract as the reference's
 * cudaMemcpyAsync + cudaStreamSynchronize at :222-231). */
int tb200_region_write_host(tb200_ctx* ctx, tb200_region* r, uint64_t offset,
                            const void* src, uint64_t nbytes);
/* N host chunks packed back to back from `offset` (the per-array loop of
 * :203-230) with one synchronisation at the end */
int tb200_region_write_host_gather(tb200_ctx* ctx, tb200_region* r,
                                   uint64_t offset, int nchunks,
                                   const void* const* srcs,
                                   const uint64_t* sizes);
/* region -> host, only the requested bytes (the reference copies the whole
 * region, :266-276) */
int tb200_region_read_host(tb200_ctx* ctx, const tb200_region* r,
                           uint64_t offset, void* dst, uint64_t nbytes);
/* any UVA pointer (device, pinned, pageable) -> region, cudaMemcpyDefault */
int tb200_region_write_ptr(tb200_ctx* ctx, tb200_region* r, uint64_t offset,
                           const void* src, uint64_t nbytes);

/* pinned, device-mapped host memory: the staging the HTTP binary body and the
 * gRPC raw_input_contents are emitted into by the kernels below. */
int tb200_host_alloc(uint64_t nbytes, void** host_ptr, void** device_ptr);
int tb200_host_free(void* host_ptr);
/* plain device memory for sources / scratch owned by the caller */
int tb200_device_alloc(int device_id, uint64_t nbytes, void** device_ptr);
int tb200_device_free(int device_id, void* device_ptr);
int tb200_memcpy_h2d_async(tb200_ctx* ctx, void* dst, const void* src,
                           uint64_t nbytes);
int tb200_memcpy_d2h_async(tb200_ctx* ctx, void* dst, const void* src,
                           uint64_t nbytes);

/* ------------------------------------------------------------------------
 * Kernel 1: synthetic-input fill (Philox4x32-10, one coalesced 16-byte store
 * per lane per call).  perf_analyzer's random / zero input generation is NOT
 * in the reference (SURVEY.md F1); the contract is defined in DESIGN.md and
 * restated on the CPU in oracle/ (parity with perf_analyzer values: unpinned).
 *
 * Tensor bytes are cut into 16-byte groups; group g of a job is
 *   philox4x32_10(ctr = {g.lo, g.hi, stream.lo, stream.hi}, key = seed)
 * mapped to elements by dtype (DESIGN.md "fill contract").
 * ---------------------------------------------------------------------- */
typedef enum tb200_fill_mode {
  TB200_FILL_RANDOM = 0, /* uniform: floats in [lo, lo+span), ints in
                            [ilo, ilo+irange) or raw bits when irange == 0;
                            dtype TB200_BYTES: fixed-length random strings in the
                            serialised <u32 length><chars> form of
                            PY/utils/__init__.py:208-261, irange = string length,
                            nbytes = count * (4 + length), chars from 0-9A-Za-z */
  TB200_FILL_ZERO = 1,
  TB200_FILL_BYTE = 2    /* every byte = (uint8_t)ilo */
} tb200_fill_mode;

typedef struct tb200_fill_job {
  uint64_t dst;     /* device (or mapped-host) address of the tensor bytes   */
  uint64_t nbytes;  /* tensor byte size                                      */
  uint64_t stream;  /* Philox stream id: (request, input) -> distinct data   */
  uint32_t dtype;   /* tb200_dtype                                           */
  uint32_t mode;    /* tb200_fill_mode                                       */
  double lo;        /* float dtypes: lower bound                             */
  double span;      /* float dtypes: width; 0 -> unit interval [0,1)         */
  int64_t ilo;      /* integer dtypes: lower bound / fill byte               */
  uint64_t irange;  /* integer dtypes: number of values, 0 -> raw bits       */
} tb200_fill_job;   /* 64 bytes */

/* One launch covers all jobs (one job = one input tensor of one concurrency
 * slot). `stream_epoch` is added to every job's stream id; when
 * `device_epoch` is non-NULL the kernel adds *device_epoch as well (used by
 * captured graphs so that every replay produces fresh data). */
int tb200_fill_async(tb200_ctx* ctx, const tb200_fill_job* jobs, int njobs,
                     uint64_t seed, uint64_t stream_epoch);

/* ------------------------------------------------------------------------
 * Kernel 2: cast + layout pack.
 *  - tb200_pack_image_async: uint8 HWC images -> {FP16,FP32,BF16} CHW (or HWC)
 *    with NONE / INCEPTION / VGG scaling; restates the numpy arithmetic of
 *    src/python/examples/image_client.py:154-193 (preprocess).  Source tiles
 *    are staged in shared memory with TMA bulk copies (cp.async.bulk).
 *  - tb200_cast_async: contiguous element-wise dtype conversion with numpy
 *    astype semantics; FP32->BF16 truncates like serialize_bf16_tensor
 *    (PY/utils/__init__.py:294-335).
 *  - tb200_pack_strided_async: ndarray.tobytes() of a strided source
 *    (PY/http/_infer_input.py:212, PY/grpc/_infer_input.py:173).
 *  - tb200_concat_async: b"".join of N tensors into one wire body
 *    (PY/http/_utils.py:141-151) or into one region
 *    (PY/utils/cuda_shared_memory/__init__.py:203-230).
 * ---------------------------------------------------------------------- */
typedef enum tb200_scaling {
  TB200_SCALE_NONE = 0,
  TB200_SCALE_INCEPTION = 1, /* (x / 127.5) - 1 */
  TB200_SCALE_VGG = 2        /* x - (123, 117, 104)   (c == 1: x - 128) */
} tb200_scaling;

typedef enum tb200_layout { TB200_NCHW = 0, TB200_NHWC = 1 } tb200_layout;

int tb200_pack_image_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype,
                           uint32_t dst_layout, const void* src_u8_nhwc,
                           int n, int h, int w, int c, uint32_t scaling);

/* The whole image_client.preprocess (src/python/examples/image_client.py:154-193) in one
 * launch: Image.resize((dst_w, dst_h), Image.BILINEAR) -> astype -> scaling -> layout.
 * The resize restates Pillow's separable antialiased triangle filter bit for bit
 * (horizontal pass first, 8-bit intermediate, 22-bit fixed-point coefficients normalised
 * in double precision on the host; oracle/image.py pins it against Pillow itself).
 * src: n uint8 images [src_h, src_w, c] (c = 1 or 3; decoded RGB / L pixels);
 * dst_dtype FP32 | FP16 | BF16, or UINT8 with TB200_SCALE_NONE for the bare resize.
 * Limits: src_h <= 100 * src_w (Pillow switches the pass order beyond), and the source
 * rows one 32-pixel-wide output tile needs must fit into shared memory. */
int tb200_resize_pack_image_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype,
                                  uint32_t dst_layout, const void* src_u8_nhwc, int n,
                                  int src_h, int src_w, int c, int dst_h, int dst_w,
                                  uint32_t scaling);

int tb200_cast_async(tb200_ctx* ctx, void* dst, uint32_t dst_dtype,
                     const void* src, uint32_t src_dtype, uint64_t nelem);

#define TB200_MAX_DIMS 8
/* dst is C-contiguous; src_strides are in BYTES (numpy convention) and may be
 * negative or zero */
int tb200_pack_strided_async(tb200_ctx* ctx, void* dst, const void* src,
                             uint32_t elem_size, int ndim,
                             const int64_t* shape, const int64_t* src_strides);

typedef struct tb200_copy_job {
  uint64_t dst;
  uint64_t src;
  uint64_t nbytes;
} tb200_copy_job;
int tb200_concat_async(tb200_ctx* ctx, const tb200_copy_job* jobs, int njobs);

/* ------------------------------------------------------------------------
 * Kernel 3: on-device output unpack / validation.  Replaces the whole-region
 * D2H + numpy compare of the examples
 * (src/python/examples/simple_http_cudashm_client.py:164-195,
 *  PY/utils/cuda_shared_memory/__init__.py:266-304).
 * Every job produces one tb200_check_result; the array is written to
 * `results` (device or mapped-host memory).
 * ---------------------------------------------------------------------- */
typedef enum tb200_check_kind {
  TB200_CHECK_SUM = 0,     /* checksum only                                  */
  TB200_CHECK_EQUAL = 1,   /* a[i] == b[i] bytewise                          */
  TB200_CHECK_ADDSUB = 2,  /* int32: a == c + d and b == c - d               */
  TB200_CHECK_TOP1 = 3     /* fp32 vector: checksum, argmax, non-finite count */
} tb200_check_kind;

typedef struct tb200_check_job {
  uint64_t a;      /* primary buffer (the output tensor; ADDSUB: OUTPUT0)    */
  uint64_t b;      /* EQUAL: expected bytes ; ADDSUB: OUTPUT1                */
  uint64_t c;      /* ADDSUB: INPUT0                                         */
  uint64_t d;      /* ADDSUB: INPUT1                                         */
  uint64_t nbytes; /* bytes of `a`                                           */
  uint32_t kind;
  uint32_t pad;
} tb200_check_job; /* 48 bytes */

typedef struct tb200_check_result {
  uint64_t mismatches; /* EQUAL / ADDSUB: elements (bytes for EQUAL) that
                          differ; TOP1: count of non-finite values           */
  uint64_t sum;        /* sum of the little-endian u32 words of `a` mod 2^64
                          (trailing bytes zero-extended)                      */
  uint32_t xor32;      /* xor of the same words                              */
  uint32_t argmax;     /* TOP1: index of the maximum (lowest index on ties)  */
  float max_value;     /* TOP1                                               */
  uint32_t pad;
} tb200_check_result;  /* 32 bytes */

int tb200_check_async(tb200_ctx* ctx, const tb200_check_job* jobs, int njobs,
                      tb200_check_result* results);

/* ------------------------------------------------------------------------
 * Kernel 3b: classification of outputs that stay in shared memory.  The server refuses
 * `classification` on a shared-memory output ("shared memory can't be set on
 * classification output", PY/http/_requested_output.py:84-85), so the examples'
 * top-k post-processing (src/python/examples/image_client.py:196-216) would need the
 * whole tensor on the host; here only k (value, index) pairs per tensor leave the device.
 * Order: value descending, lower index first on ties, -0.0 == +0.0, NaN after every
 * number (numpy.argsort(-x, kind="stable")).  Entries past `count` get index 0xFFFFFFFF.
 * ---------------------------------------------------------------------- */
typedef struct tb200_topk_job {
  uint64_t src;    /* device address of the vector                          */
  uint64_t count;  /* elements (< 2^32 - 1)                                 */
  uint32_t dtype;  /* TB200_FP32 | TB200_FP16 | TB200_BF16                  */
  uint32_t pad;
} tb200_topk_job;  /* 24 bytes */

typedef struct tb200_topk_entry {
  float value;
  uint32_t index;
} tb200_topk_entry;

/* out: njobs * k entries, job-major (device or mapped-host memory); 1 <= k <= 1024 */
int tb200_topk_async(tb200_ctx* ctx, const tb200_topk_job* jobs, int njobs, int k,
                     tb200_topk_entry* out);

/* Response side, BYTES tensors on the device: walk the <u32 LE length><payload> chain of a
 * serialised BYTES tensor of `count` elements -- what deserialize_bytes_tensor
 * (PY/utils/__init__.py:264-291) and the BYTES branch of cuda_shared_memory.get_contents_as_numpy
 * (PY/utils/cuda_shared_memory/__init__.py:306-323) do on the host after copying the whole region --
 * and write  offsets[count + 1]  (prefix sums of the payload lengths, offsets[0] = 0) and the
 * payloads packed back to back into `packed`.  offsets / packed / status may be device or mapped
 * host memory.  status[0] = elements decoded, [1] = bytes of `src` consumed, [2] = packed bytes,
 * [3] = 0 ok | 1 truncated (fewer than `count` elements fit) | 2 a payload runs past src_bytes |
 * 3 more than 4 GiB of payload; nothing is packed when status[3] != 0 or status[2] > packed_capacity. */
int tb200_bytes_decode_async(tb200_ctx* ctx, const void* src, uint64_t src_bytes, uint64_t count,
                             uint32_t* offsets, void* packed, uint64_t packed_capacity, uint64_t* status);

/* ------------------------------------------------------------------------
 * Kernel 4: request-body compression.  The reference compresses a body with zlib / gzip on
 * the host (PY/http/_client.py:1440-1460, CC/http_client.cc:146-221, `Content-Encoding:
 * deflate | gzip`); a body generated on the device is compressed there: 8 KiB chunks, one
 * fixed-Huffman deflate block each (LZ77 matches inside the chunk), sync-flush between
 * chunks, stored fallback, Adler-32 / CRC-32 combined on the device.  Any zlib / gzip
 * decoder accepts the stream; it is not byte-identical to zlib's own output.
 * `dst` must hold tb200_deflate_bound(nbytes) bytes; *out_size (device or mapped-host
 * memory) receives the stream length when the stream reaches the launch.
 * ---------------------------------------------------------------------- */
typedef enum tb200_deflate_format {
  TB200_DEFLATE_ZLIB = 0, /* "deflate" content encoding: 2-byte header, Adler-32 trailer */
  TB200_DEFLATE_GZIP = 1  /* 10-byte header, CRC-32 + ISIZE trailer                      */
} tb200_deflate_format;

uint64_t tb200_deflate_bound(uint64_t nbytes);
int tb200_deflate_async(tb200_ctx* ctx, void* dst, uint64_t dst_capacity, const void* src,
                        uint64_t nbytes, uint32_t format, uint64_t* out_size);

/* ------------------------------------------------------------------------
 * Issue loop building blocks: capture any sequence of the *_async calls above
 * into a CUDA graph and replay it per measurement step / concurrency slot.
 * The concurrency loop itself (the absent perf_analyzer ConcurrencyManager /
 * ConcurrencyWorker, SURVEY.md row P) is restated natively in loadgen.h.
 * ---------------------------------------------------------------------- */
typedef struct tb200_graph tb200_graph;
int tb200_graph_begin(tb200_ctx* ctx);
int tb200_graph_end(tb200_ctx* ctx, tb200_graph** out);
int tb200_graph_launch(tb200_ctx* ctx, tb200_graph* g);
int tb200_graph_destroy(tb200_graph* g);
/* device-resident epoch counter added to Philox stream ids inside graphs */
int tb200_ctx_epoch_set(tb200_ctx* ctx, uint64_t value);
int tb200_ctx_epoch_bump_async(tb200_ctx* ctx, uint64_t delta);
/* fill variant that adds the context's device epoch to every stream id (graph
 * friendly); when bump != 0 the kernel itself advances the device epoch by `bump`
 * after its last CTA finished, so each replay produces fresh data */
int tb200_fill_epoch_async(tb200_ctx* ctx, const tb200_fill_job* jobs,
                           int njobs, uint64_t seed, uint64_t bump);

/* One closed-loop step in a single call: generate the inputs of `nfill` jobs, validate
 * `ncheck` outputs, wait for both.  The results land in `results` (mapped host memory);
 * the job tables are copied host->device from the pinned ring inside the call. */
int tb200_step_sync(tb200_ctx* ctx, const tb200_fill_job* fill_jobs, int nfill, uint64_t seed,
                    uint64_t stream_epoch, const tb200_check_job* check_jobs, int ncheck,
                    tb200_check_result* results);

/* The same step without the wait: tb200_step_submit returns once both launches are queued (the
 * fill on the context's stream, the validation on its side stream) and hands out a ticket;
 * tb200_step_wait(ticket) returns when that step's inputs are generated and its results are
 * visible in `results`.  Up to TB200_STEP_DEPTH steps may be in flight, so the host forms the job
 * tables of step i+1 while the device runs step i (steps in flight must not share slots or
 * result entries); submitting a step whose ring entry is still unwaited waits for it first.
 * This is the load generator's pipelined pass and bench.py's e2e loop. */
#define TB200_STEP_DEPTH 8
int tb200_step_submit(tb200_ctx* ctx, const tb200_fill_job* fill_jobs, int nfill, uint64_t seed,
                      uint64_t stream_epoch, const tb200_check_job* check_jobs, int ncheck,
                      tb200_check_result* results, uint64_t* ticket);
int tb200_step_wait(tb200_ctx* ctx, uint64_t ticket);

/* knobs: "fill_variant" (experiment matrix of scripts/fill_sweep.py, 0 = default policy);
 * "step_parallel_min_mb": tb200_step_sync runs check and fill as parallel branches only
 * when the fill writes at least this many MiB (default 0 = always) */
int tb200_tune(const char* key, int value);

/* write > L2-size bytes so the next timed kernel starts with a cold L2 */
int tb200_l2_flush_async(tb200_ctx* ctx);

#ifdef __cplusplus
}
#endif
#endif /* TB200_H_ */
