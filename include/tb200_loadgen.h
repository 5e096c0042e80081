/*
 * tb200_loadgen.h -- C ABI of the native closed-loop load generator in libtb200.so.
 *
 * What it restates: perf_analyzer's ConcurrencyManager / ConcurrencyWorker loop --
 * NOT part of the reference (SURVEY.md F1, section 8a row P); its only traces there are
 * the friend hooks in src/c++/library/common.h:42-47,358-360,462-464.  The per-request
 * timestamps and the cumulative statistics follow the reference's C++ client types
 * RequestTimers (src/c++/library/common.h:568-648) and InferStat (:93-114, folded by
 * UpdateInferStat, src/c++/library/common.cc:56-106).
 *
 * Shape: `concurrency` keep-alive HTTP/1.1 connections, one per slot, each with one request
 * in flight (closed loop), served by a few epoll-driven transport threads.  A request is a
 * pre-formed byte string per concurrency slot (with shared memory it only names regions,
 * golden "A" of SURVEY.md 9.4).  One device thread serves all slots: slots whose responses
 * came back are validated (tb200_check_async) and regenerated (tb200_fill_async) as parallel
 * branches of ONE pass, then handed back to the transport threads in one batch -- the
 * transport threads never touch tensor bytes and no thread is woken per request.  Several
 * passes can be in flight (pipeline_depth): the issue loop the reference leaves to Python
 * futures and queues (grpc/_client.py:1574-1741, grpc/_infer_stream.py:108-168).
 */
#ifndef TB200_LOADGEN_H_
#define TB200_LOADGEN_H_

#include "tb200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct tb200_loadgen tb200_loadgen;

typedef struct tb200_loadgen_config {
  const char* host;              /* numeric IPv4 address, e.g. "127.0.0.1" */
  int port;
  int concurrency;               /* requests in flight = connections = slots */
  const uint8_t* const* requests; /* [concurrency] complete HTTP requests (headers + body) */
  const uint64_t* request_sizes;  /* [concurrency] */
  /* optional binary tails sent right after requests[s] and NOT copied: they point into
   * pinned staging that the fill kernel rewrites before every send (HTTP binary-tensor
   * body in --shared-memory none mode); NULL when the request is self-contained */
  const uint8_t* const* tails;
  const uint64_t* tail_sizes;
  /* device side (all optional: ctx == NULL -> transport only) */
  tb200_ctx* ctx;
  const tb200_fill_job* fill_jobs;   /* [concurrency * fill_jobs_per_slot], slot-major */
  int fill_jobs_per_slot;
  uint64_t seed;
  int regenerate;                    /* 1: refill a slot's inputs before every request */
  const tb200_check_job* check_jobs; /* [concurrency * check_jobs_per_slot] */
  int check_jobs_per_slot;
  tb200_check_result* results;       /* device-visible (mapped host), same count as check_jobs */
  /* the device thread waits up to this long for further returned slots before a pass
   * (ends early once every slot in flight is back); 0 = take what is there.  Worth ~150
   * when client and server are time-sliced CUDA contexts (no MPS): each GPU hand-over
   * between the processes costs ~100 us, so passes should be few and full */
  uint32_t device_window_us;
  /* 0: requests[] are complete HTTP/1.1 requests.  1: unary gRPC calls over cleartext HTTP/2
   * (what grpcio does under PY/grpc/_client.py:1445-1572): requests[s] holds the serialised
   * ModelInferRequest WITHOUT its raw_input_contents, tails[s] the remaining message bytes
   * (field-7 tag + length + tensor, per input) in pinned staging; one stream per request,
   * messages up to the peer's stream window (64 KiB by default);
   * 2 = the same messages on ONE long-lived ModelStreamInfer stream per connection (reference
   * grpc/_client.py start_stream / async_stream_infer): a request completes at the response
   * that does not carry triton_final_response = false, or at a response with an error message;
   * the time to the first response is reported */
  uint32_t protocol;
  const char* grpc_path; /* NULL -> "/inference.GRPCInferenceService/ModelInfer" */
  /* wire mode look-ahead: tails[s] is the first of `lookahead` staging images, `tail_stride`
   * bytes apart, each tail_sizes[s] long; fill_jobs_per_slot then covers all of them.  The
   * transport sends image 0, 1, ... with consecutive requests and hands the slot back to the
   * device thread only after the last one, so every request carries freshly generated tensors
   * while the device is visited once per `lookahead` requests.  0 or 1 = off. */
  uint32_t lookahead;
  uint64_t tail_stride;
  /* shared-memory look-ahead: requests[] holds `requests_per_slot` (= lookahead) pre-formed requests
   * per slot, slot-major, one per staging image (they name different region offsets); check and
   * fill jobs per slot cover all images.  0 or 1 = one request per slot. */
  uint32_t requests_per_slot;
  /* device passes in flight.  0 / 1: the device thread runs one pass at a time (validate the
   * returned slots || generate their next inputs, wait, hand the slots back).  N > 1: up to N
   * passes are in flight (tb200_step_submit / tb200_step_wait): the thread forms the next pass
   * while the device runs the previous ones, consecutive generations overlap on the device, and
   * slots go back to their connections in pass order.  At most TB200_STEP_DEPTH / 2. */
  uint32_t pipeline_depth;
  /* replayed inputs (perf --input-data FILE|DIR).  0 entries = off: the fill jobs generate the inputs.
   * Otherwise `replay_entries` user-supplied entries sit in a device pool and every device pass copies
   * the next entry of each returned slot into its inputs (tb200_concat_async / tb200_step_submit_copy):
   * copy_jobs[concurrency * copy_jobs_per_slot] are laid out like fill_jobs (slot-major, then staging
   * image, then input) and point at entry 0; job j of a slot reads entry e at
   * src + e * copy_src_stride[j].  check_b_stride[k] (one per check job of a slot) does the same for
   * the expected bytes `b` of an EQUAL check; 0 leaves check k as it is.  Request r of slot s carries
   * entry tb200_loadgen_replay_entry(s, r, lookahead, !regenerate, replay_entries), and its response is
   * checked against the same entry. */
  uint64_t replay_entries;
  const tb200_copy_job* copy_jobs;
  int copy_jobs_per_slot;
  const uint64_t* copy_src_stride;  /* [copy_jobs_per_slot] */
  const uint64_t* check_b_stride;   /* [check_jobs_per_slot], may be NULL */
} tb200_loadgen_config;

/* The entry rule of replayed inputs: (slot + r) mod entries, r = request mod lookahead when the
 * inputs are written once (`once` != 0, i.e. regenerate == 0); request r of a slot is image g of its
 * generation k when r = k * lookahead + g. */
uint64_t tb200_loadgen_replay_entry(uint64_t slot, uint64_t request, uint32_t lookahead, int once, uint64_t entries);

typedef struct tb200_loadgen_stats {
  /* InferStat (reference common.h:93-114) over the window */
  uint64_t completed_request_count;
  uint64_t failed_request_count;
  uint64_t cumulative_total_request_time_ns; /* REQUEST_START -> REQUEST_END */
  uint64_t cumulative_send_time_ns;          /* SEND_START -> SEND_END       */
  uint64_t cumulative_receive_time_ns;       /* RECV_START -> RECV_END       */
  /* latency distribution over the window (ns) */
  uint64_t p50_ns, p90_ns, p95_ns, p99_ns, min_ns, max_ns;
  double window_seconds;
  /* device thread */
  uint64_t device_batches;    /* fill(+check) passes                                  */
  uint64_t device_slots;      /* slots served by them (device_slots / device_batches = */
                              /* requests covered per launch)                          */
  uint64_t nonfinite_outputs; /* from TOP1 checks                                      */
  uint64_t check_mismatches;  /* from EQUAL / ADDSUB checks                            */
  /* protocol 2 (one ModelStreamInfer stream per connection): responses received for the    */
  /* completed requests (tokens of a decoupled model) and REQUEST_START -> first response   */
  uint64_t response_count;
  uint64_t first_response_p50_ns, first_response_p99_ns;
} tb200_loadgen_stats;

int tb200_loadgen_create(const tb200_loadgen_config* cfg, tb200_loadgen** out);
int tb200_loadgen_start(tb200_loadgen* lg);
/* sleep `seconds`, then report and reset the statistics gathered meanwhile */
int tb200_loadgen_window(tb200_loadgen* lg, double seconds, tb200_loadgen_stats* out);
/* count-window helper (perf_analyzer's --measurement-mode count_windows): block until `count`
 * requests finished (completed + failed) since the last tb200_loadgen_window call, or the
 * timeout; *reached = how many had.  Follow it with tb200_loadgen_window(lg, 0, &stats). */
int tb200_loadgen_wait_count(tb200_loadgen* lg, uint64_t count, double timeout_seconds, uint64_t* reached);
int tb200_loadgen_stop(tb200_loadgen* lg);
int tb200_loadgen_destroy(tb200_loadgen* lg);

/* A canned-response HTTP server for measuring the generator itself (every POST gets
 * `200` + the given body; GET /v2/health/* gets 200).  Test/bench tooling: it does not
 * open shared memory.  Returns the bound port through *port (pass 0 to pick one). */
typedef struct tb200_stub_server tb200_stub_server;
int tb200_stub_server_start(const char* host, int* port, const char* response_body,
                            tb200_stub_server** out);
int tb200_stub_server_stop(tb200_stub_server* s);
/* the same for gRPC: every unary call is answered with `response` (a serialised protobuf
 * message, e.g. ModelInferResponse) and grpc-status 0 */
typedef struct tb200_grpc_stub_server tb200_grpc_stub_server;
int tb200_grpc_stub_server_start(const char* host, int* port, const uint8_t* response,
                                 uint64_t response_bytes, tb200_grpc_stub_server** out);
/* Stream mode of the same stub (ModelStreamInfer): every request message on a stream is answered
 * with `responses_per_request - 1` copies of `response` and one `final_response` (serialised
 * ModelStreamInferResponse messages; the caller marks the last one triton_final_response = true). */
int tb200_grpc_stub_server_start_streaming(const char* host, int* port, const uint8_t* response,
                                           uint64_t response_bytes, const uint8_t* final_response,
                                           uint64_t final_bytes, int responses_per_request,
                                           tb200_grpc_stub_server** out);
int tb200_grpc_stub_server_stop(tb200_grpc_stub_server* s);

/* A gRPC echo server on the event-loop core the native model server uses (csrc/grpc_server.h):
 * every unary call of inference.GRPCInferenceService is answered with its own request message
 * (a ModelInferRequest parses as a ModelInferResponse: the fields line up), every message on a
 * ModelStreamInfer stream with ModelStreamInferResponse{infer_response = that message}.  Test
 * tooling: exercises HPACK decoding, message reassembly and flow control in both directions
 * against real gRPC clients without a GPU. */
typedef struct tb200_grpc_echo_server tb200_grpc_echo_server;
int tb200_grpc_echo_server_start(const char* host, int* port, tb200_grpc_echo_server** out);
int tb200_grpc_echo_server_stop(tb200_grpc_echo_server* s);

/* A native KServe-v2 stand-in server for loopback load runs over CUDA shared memory
 * (csrc/mock_server.cu; tooling -- the reference has no server, SURVEY.md F6).  It opens
 * the client's cudaIpcMemHandle_t from the register call (protocol of
 * src/python/library/tritonclient/http/_client.py:1153-1207), so it must live in ANOTHER
 * process than the client, and runs models `densenet_onnx` / `simple` as CUDA kernels
 * on the mapped regions. */
typedef struct tb200_mock_server tb200_mock_server;
int tb200_mock_server_start(const char* host, int* port, int device_id, tb200_mock_server** out);
/* ... and with a gRPC port beside the HTTP one (csrc/grpc_server.h + the generated message
 * classes): health / metadata / config / repository index / CUDA shared memory RPCs, ModelInfer
 * and ModelStreamInfer for `densenet_onnx`, `simple` (shared memory or tensors in the message),
 * `bert_large` (2 x INT64[1,384] -> FP32[1,384], BASELINE configs[3]) and the decoupled
 * `llama3_8b` (INT32[1,n] prompt -> max_tokens token responses, configs[4]); tensors that travel
 * in messages are staged in pinned, device-mapped slabs (16 KiB of inputs per request). */
int tb200_mock_server_start2(const char* host, int* port, int* grpc_port, int device_id, tb200_mock_server** out);
uint64_t tb200_mock_server_requests(tb200_mock_server* s);
uint64_t tb200_mock_server_batches(tb200_mock_server* s); /* kernel launches that served them */
int tb200_mock_server_stop(tb200_mock_server* s);

#ifdef __cplusplus
}
#endif
#endif /* TB200_LOADGEN_H_ */
