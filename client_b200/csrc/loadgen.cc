// loadgen.cc -- native closed-loop load generator (C ABI: include/tb200_loadgen.h).
//
// Restates perf_analyzer's ConcurrencyManager / ConcurrencyWorker behaviour (not in the
// reference, SURVEY.md F1) with the reference C++ client's RequestTimers / InferStat
// bookkeeping (src/c++/library/common.h:568-648, :93-114; common.cc:56-106).  Transport
// is plain HTTP/1.1 over POSIX sockets: the reference's libcurl path
// (src/c++/library/http_client.cc:1767-1830) cannot be built here and is not needed to
// send a pre-formed request and read a Content-Length response.
//
// Threads: a few epoll-driven transport threads, each owning the keep-alive connections of
// a share of the slots (slot s <-> connection s, thread s % T), plus one device thread.
// A request is one non-blocking sendmsg of the pre-formed bytes (+ the borrowed tail); the
// hand-over between transport and device thread is batched (one eventfd write per thread
// and pass), so the host cost per request is a send, a recv and no thread wake-up.
#include <arpa/inet.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <poll.h>
#include <fcntl.h>
#include <sys/epoll.h>
#include <sys/eventfd.h>
#include <sys/socket.h>
#include <sys/uio.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "../../include/tb200_loadgen.h"
#include "../cpp/pb.h"
#include "grpc_server.h"
#include "h2.h"
#include "h2_stub_server.h"
#include "http_server.h"

namespace {

uint64_t now_ns() {
  return static_cast<uint64_t>(std::chrono::duration_cast<std::chrono::nanoseconds>(
                                   std::chrono::steady_clock::now().time_since_epoch())
                                   .count());
}

int connect_to(const char* host, int port) {
  int fd = socket(AF_INET, SOCK_STREAM, 0);
  if (fd < 0) return -1;
  sockaddr_in addr{};
  addr.sin_family = AF_INET;
  addr.sin_port = htons(static_cast<uint16_t>(port));
  if (inet_pton(AF_INET, host, &addr.sin_addr) != 1 ||
      connect(fd, reinterpret_cast<sockaddr*>(&addr), sizeof(addr)) != 0) {
    close(fd);
    return -1;
  }
  int one = 1;
  setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
  return fd;
}

// case-insensitive search of "content-length:" in the header block
long content_length(const char* hdr, size_t len) {
  static const char key[] = "content-length:";
  for (size_t i = 0; i + sizeof(key) - 1 <= len; ++i) {
    size_t k = 0;
    while (k < sizeof(key) - 1 && (hdr[i + k] | 0x20) == key[k]) ++k;
    if (k == sizeof(key) - 1 && (i == 0 || hdr[i - 1] == '\n')) return strtol(hdr + i + k, nullptr, 10);
  }
  return 0;
}

struct SlotQueue {
  std::mutex mu;
  std::condition_variable cv;
  std::deque<int> q;
  void push(int s) {
    {
      std::lock_guard<std::mutex> lk(mu);
      q.push_back(s);
    }
    cv.notify_one();
  }
  // -1 on timeout
  int pop(int timeout_ms) {
    std::unique_lock<std::mutex> lk(mu);
    if (!cv.wait_for(lk, std::chrono::milliseconds(timeout_ms), [&] { return !q.empty(); })) return -1;
    int s = q.front();
    q.pop_front();
    return s;
  }
  // -1 on timeout
  int pop_ns(uint64_t ns) {
    std::unique_lock<std::mutex> lk(mu);
    if (!cv.wait_for(lk, std::chrono::nanoseconds(ns), [&] { return !q.empty(); })) return -1;
    int s = q.front();
    q.pop_front();
    return s;
  }
  size_t drain(std::vector<int>& out) {
    std::lock_guard<std::mutex> lk(mu);
    const size_t n = q.size();
    out.insert(out.end(), q.begin(), q.end());
    q.clear();
    return n;
  }
};

struct WorkerStats {
  std::mutex mu;
  std::vector<uint64_t> latencies;  // REQUEST_START -> REQUEST_END
  std::vector<uint64_t> first_ns;   // stream mode: REQUEST_START -> first response of the request
  uint64_t completed = 0, failed = 0, total_ns = 0, send_ns = 0, recv_ns = 0, responses = 0;
};

// one keep-alive connection = one concurrency slot
struct Conn {
  int fd = -1;
  int slot = 0;
  std::vector<iovec> tx;   // what is left of the request being sent
  size_t tx_idx = 0;
  std::vector<uint8_t> txbuf;  // gRPC: frame headers + message prefix + protobuf head of this request
  bool want_out = false;   // EPOLLOUT armed
  bool in_flight = false;
  int attempts = 0;
  std::vector<char> buf;   // response bytes so far
  size_t header_end = 0;
  long body = 0;
  uint64_t t_start = 0, t_send_end = 0, t_recv_start = 0;
  // gRPC over cleartext HTTP/2 (h2.h)
  uint32_t next_stream = 1, cur_stream = 0;
  int64_t conn_window = tb200::h2::kDefaultWindow;      // what the peer lets us send on the connection
  uint32_t peer_stream_window = tb200::h2::kDefaultWindow;
  uint32_t peer_max_frame = tb200::h2::kDefaultMaxFrame;
  uint64_t recv_consumed = 0;
  bool got_data = false, waiting_window = false, goaway = false;
  std::string ctrl;        // control frames (acks, window updates) waiting for a frame boundary
  // stream mode (ModelStreamInfer): one long-lived stream per connection, a request = one message on it
  bool stream_open = false;
  int64_t stream_window = 0;        // what the peer lets us send on the stream
  uint64_t stream_recv_consumed = 0;
  std::string rx_msg;               // response messages being reassembled from DATA frames
  uint64_t t_first = 0;             // first response of the request in flight
  uint32_t responses = 0;
  uint32_t image = 0;               // look-ahead: which of the slot's staging images goes out next
};

struct Transport {
  int epfd = -1, evfd = -1;
  std::mutex mu;
  std::vector<int> ready;   // slots released by the device thread (guarded by mu)
  std::vector<Conn> conns;  // the slots this thread owns
  WorkerStats stats;
};

}  // namespace

struct tb200_loadgen {
  std::string host;
  int port = 0;
  int concurrency = 0;
  std::vector<std::vector<uint8_t>> requests;
  std::vector<const uint8_t*> tails;  // borrowed (pinned staging), may be empty
  std::vector<uint64_t> tail_sizes;
  uint32_t lookahead = 1;             // staging images per slot
  uint32_t rps = 1;                   // pre-formed requests per slot (shared-memory look-ahead: one per image)
  uint64_t tail_stride = 0;
  bool passthrough = false;           // no device work per request: workers keep their slot
  bool grpc = false;                  // requests[] are ModelInferRequest bytes sent as unary gRPC calls
  bool grpc_stream = false;           // ... or as messages of one ModelStreamInfer stream per connection
  std::string grpc_headers;           // HEADERS payload shared by all requests
  tb200_ctx* ctx = nullptr;
  std::vector<tb200_fill_job> fill_jobs;
  int fill_per_slot = 0;
  uint64_t seed = 0;
  bool regenerate = false;
  uint64_t device_window_ns = 0;
  uint32_t pipeline_depth = 1;        // device passes in flight (tb200_step_submit / tb200_step_wait)
  tb200_check_result* own_results = nullptr;  // depth > 1: one result block per pass in flight (mapped host)
  void* own_results_host = nullptr;
  std::vector<tb200_check_job> check_jobs;
  int check_per_slot = 0;
  tb200_check_result* results = nullptr;

  std::atomic<bool> stop{false};
  bool started = false;
  SlotQueue returned;                          // transport threads -> device thread
  std::vector<std::unique_ptr<Transport>> transports;
  std::vector<std::thread> threads;
  // device thread counters (guarded by dev_mu)
  std::mutex dev_mu;
  uint64_t device_batches = 0, device_slots = 0, nonfinite = 0, mismatches = 0, epoch = 0;
  std::string error;
  uint64_t window_start_ns = 0;
  // replayed inputs (cfg.replay_entries != 0): copy and check templates point at entry 0.  Kept
  // behind every other member, so the members the transport and device threads share keep the
  // layout they have in a run without replay.
  uint64_t replay_entries = 0;
  std::vector<tb200_copy_job> copy_jobs;
  int copy_per_slot = 0;
  std::vector<uint64_t> copy_stride, check_b_stride;
  std::vector<uint64_t> replay_gen;  // per slot: the generation its inputs hold (device thread only)
};

namespace {

constexpr uint32_t kEvTag = 0xFFFFFFFFu;

// replayed inputs: the entry image g of slot s's current generation carries
uint64_t replay_entry_of(const tb200_loadgen* lg, int s, int g) {
  return tb200_loadgen_replay_entry(static_cast<uint64_t>(s), lg->replay_gen[static_cast<size_t>(s)] * lg->lookahead + static_cast<uint64_t>(g),
                                    lg->lookahead, lg->regenerate ? 0 : 1, lg->replay_entries);
}

// the check jobs of slot s; a replay check's expected bytes are the entry its request carried
void append_checks(const tb200_loadgen* lg, int s, std::vector<tb200_check_job>& out) {
  const tb200_check_job* first = lg->check_jobs.data() + static_cast<size_t>(s) * lg->check_per_slot;
  if (lg->check_b_stride.empty()) {  // no replay check: the slot's jobs as they are
    out.insert(out.end(), first, first + lg->check_per_slot);
    return;
  }
  const int per_image = lg->check_per_slot / static_cast<int>(lg->lookahead);
  for (int k = 0; k < lg->check_per_slot; ++k) {
    tb200_check_job job = first[k];
    if (lg->check_b_stride[static_cast<size_t>(k)] != 0) {
      job.b += replay_entry_of(lg, s, k / per_image) * lg->check_b_stride[static_cast<size_t>(k)];
    }
    out.push_back(job);
  }
}

// the copies that write the entries of slot s's current generation into its inputs
void append_copies(const tb200_loadgen* lg, int s, std::vector<tb200_copy_job>& out) {
  const int per_image = lg->copy_per_slot / static_cast<int>(lg->lookahead);
  for (int j = 0; j < lg->copy_per_slot; ++j) {
    tb200_copy_job job = lg->copy_jobs[static_cast<size_t>(s) * lg->copy_per_slot + j];
    job.src += replay_entry_of(lg, s, j / per_image) * lg->copy_stride[static_cast<size_t>(j)];
    out.push_back(job);
  }
}

void h2_flush_ctrl(Conn& c);

void conn_close(Transport* t, Conn& c) {
  c.ctrl.clear();
  if (c.fd >= 0) {
    epoll_ctl(t->epfd, EPOLL_CTL_DEL, c.fd, nullptr);
    close(c.fd);
  }
  c.fd = -1;
  c.want_out = false;
}

bool conn_open(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index) {
  c.fd = connect_to(lg->host.c_str(), lg->port);
  if (c.fd < 0) return false;
  fcntl(c.fd, F_SETFL, fcntl(c.fd, F_GETFL, 0) | O_NONBLOCK);
  epoll_event ev{};
  ev.events = EPOLLIN;
  ev.data.u32 = index;
  epoll_ctl(t->epfd, EPOLL_CTL_ADD, c.fd, &ev);
  if (lg->grpc) {  // fresh HTTP/2 connection state; requests may follow the preface at once
    c.next_stream = 1;
    c.cur_stream = 0;
    c.conn_window = tb200::h2::kDefaultWindow;
    c.peer_stream_window = tb200::h2::kDefaultWindow;
    c.peer_max_frame = tb200::h2::kDefaultMaxFrame;
    c.recv_consumed = 0;
    c.waiting_window = c.goaway = false;
    c.stream_open = false;
    c.stream_window = 0;
    c.stream_recv_consumed = 0;
    c.rx_msg.clear();
    c.buf.clear();
    c.ctrl = tb200::h2::client_preface();
    h2_flush_ctrl(c);
  }
  return true;
}

void conn_arm(Transport* t, Conn& c, uint32_t index, bool want_out) {
  if (c.want_out == want_out) return;
  epoll_event ev{};
  ev.events = EPOLLIN | (want_out ? EPOLLOUT : 0);
  ev.data.u32 = index;
  epoll_ctl(t->epfd, EPOLL_CTL_MOD, c.fd, &ev);
  c.want_out = want_out;
}

void request_done(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index, bool ok, uint64_t t_end);

// queued HTTP/2 control frames go out only between requests' frames
void h2_flush_ctrl(Conn& c) {
  if (c.ctrl.empty() || c.want_out || c.fd < 0) return;
  size_t off = 0;
  while (off < c.ctrl.size()) {
    const ssize_t k = send(c.fd, c.ctrl.data() + off, c.ctrl.size() - off, MSG_NOSIGNAL | MSG_DONTWAIT);
    if (k > 0) {
      off += static_cast<size_t>(k);
    } else if (k < 0 && errno == EINTR) {
      continue;
    } else if (k < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) {
      pollfd pfd{c.fd, POLLOUT, 0};
      if (poll(&pfd, 1, 100) <= 0) break;
    } else {
      break;
    }
  }
  c.ctrl.erase(0, off);
}

// push the rest of c.tx; false on a dead connection
bool conn_send(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index) {
  (void)lg;
  while (c.tx_idx < c.tx.size()) {
    msghdr msg{};
    msg.msg_iov = &c.tx[c.tx_idx];
    msg.msg_iovlen = std::min<size_t>(c.tx.size() - c.tx_idx, 64);
    const ssize_t k = sendmsg(c.fd, &msg, MSG_NOSIGNAL | MSG_DONTWAIT);
    if (k < 0) {
      if (errno == EINTR) continue;
      if (errno == EAGAIN || errno == EWOULDBLOCK) {
        conn_arm(t, c, index, true);
        return true;
      }
      return false;
    }
    size_t left = static_cast<size_t>(k);
    while (c.tx_idx < c.tx.size() && left >= c.tx[c.tx_idx].iov_len) {
      left -= c.tx[c.tx_idx].iov_len;
      ++c.tx_idx;
    }
    if (c.tx_idx < c.tx.size() && left > 0) {
      c.tx[c.tx_idx].iov_base = static_cast<char*>(c.tx[c.tx_idx].iov_base) + left;
      c.tx[c.tx_idx].iov_len -= left;
    }
  }
  c.t_send_end = now_ns();
  conn_arm(t, c, index, false);
  h2_flush_ctrl(c);
  return true;
}

// Lay out one unary gRPC call on a fresh stream: HEADERS, then DATA frames over
// prefix(5) | protobuf head | borrowed tail, cut at the peer's maximum frame size.
// Returns 0 ok, 1 must wait for connection window, -1 cannot be sent at all.
int grpc_build(tb200_loadgen* lg, Conn& c) {
  namespace h2 = tb200::h2;
  const std::vector<uint8_t>& head = lg->requests[static_cast<size_t>(c.slot) * lg->rps + (lg->rps > 1 ? c.image : 0)];
  const uint8_t* tail = lg->tails.empty() ? nullptr : lg->tails[c.slot] + static_cast<uint64_t>(c.image) * lg->tail_stride;
  const size_t tail_size = lg->tails.empty() ? 0 : static_cast<size_t>(lg->tail_sizes[c.slot]);
  const size_t message = head.size() + tail_size;
  const size_t payload = 5 + message;
  if (payload > c.peer_stream_window || payload > 0x7FFFFFFFu) return -1;
  if (static_cast<int64_t>(payload) > c.conn_window) return 1;
  const bool open_stream = !lg->grpc_stream || !c.stream_open;
  if (lg->grpc_stream && c.stream_open && static_cast<int64_t>(payload) > c.stream_window) return 1;
  if (open_stream) {
    c.cur_stream = c.next_stream;
    c.next_stream += 2;
    c.stream_window = c.peer_stream_window;
    c.stream_open = lg->grpc_stream;
    c.stream_recv_consumed = 0;  // receive credit is per stream
  }
  c.got_data = false;
  c.t_first = 0;
  c.responses = 0;
  const size_t maxf = c.peer_max_frame;
  const size_t nframes = (payload + maxf - 1) / maxf;
  const size_t hdr_bytes = open_stream ? 9 + lg->grpc_headers.size() : 0;
  // txbuf: [HEADERS frame (a new stream only)][prefix + head][DATA frame headers ...]
  c.txbuf.resize(hdr_bytes + 5 + head.size() + 9 * nframes);
  uint8_t* w = c.txbuf.data();
  if (open_stream) {
    h2::put_frame_header(w, static_cast<uint32_t>(lg->grpc_headers.size()), h2::HEADERS, h2::kEndHeaders, c.cur_stream);
    memcpy(w + 9, lg->grpc_headers.data(), lg->grpc_headers.size());
  }
  uint8_t* body = w + hdr_bytes;
  h2::put_grpc_prefix(body, static_cast<uint32_t>(message));
  memcpy(body + 5, head.data(), head.size());
  const size_t in_buf = 5 + head.size();
  uint8_t* fh = body + in_buf;
  c.tx.clear();
  c.tx_idx = 0;
  if (open_stream) c.tx.push_back(iovec{w, hdr_bytes});
  size_t off = 0;
  for (size_t f = 0; f < nframes; ++f) {
    const size_t chunk = std::min(maxf, payload - off);
    const bool last = off + chunk == payload && !lg->grpc_stream;  // a stream stays open between requests
    h2::put_frame_header(fh + 9 * f, static_cast<uint32_t>(chunk), h2::DATA, last ? h2::kEndStream : 0, c.cur_stream);
    c.tx.push_back(iovec{fh + 9 * f, 9});
    size_t o = off, left = chunk;
    if (o < in_buf) {
      const size_t n = std::min(left, in_buf - o);
      c.tx.push_back(iovec{body + o, n});
      o += n;
      left -= n;
    }
    if (left > 0) c.tx.push_back(iovec{const_cast<uint8_t*>(tail) + (o - in_buf), left});
    off += chunk;
  }
  c.conn_window -= static_cast<int64_t>(payload);
  c.stream_window -= static_cast<int64_t>(payload);
  return 0;
}

// One ModelStreamInferResponse (grpc_service.proto: 1 error_message, 2 infer_response; in the latter
// 4 parameters map<string, InferParameter{1 bool_param}>): *error when error_message is set, *final
// unless the response carries triton_final_response = false (the rule of the Python engine,
// perf/loadgen.py, and of perf_analyzer for decoupled models).
void parse_stream_response(const uint8_t* p, size_t n, bool* error, bool* final) {
  namespace pb = tb200::pb;
  *error = false;
  *final = true;
  pb::Reader r(p, n);
  uint32_t field = 0, wt = 0;
  while (r.tag(&field, &wt)) {
    const uint8_t* d = nullptr;
    size_t len = 0;
    if (wt != pb::kBytes || !r.bytes(&d, &len)) {
      r.skip(wt);
      continue;
    }
    if (field == 1 && len != 0) *error = true;
    if (field != 2) continue;
    pb::Reader resp(d, len);
    uint32_t f2 = 0, w2 = 0;
    while (resp.tag(&f2, &w2)) {
      const uint8_t* e = nullptr;
      size_t elen = 0;
      if (w2 != pb::kBytes || !resp.bytes(&e, &elen)) {
        resp.skip(w2);
        continue;
      }
      if (f2 != 4) continue;
      pb::Reader entry(e, elen);
      uint32_t f3 = 0, w3 = 0;
      bool is_final_key = false, value = false, has_value = false;
      while (entry.tag(&f3, &w3)) {
        const uint8_t* v = nullptr;
        size_t vlen = 0;
        if (w3 != pb::kBytes || !entry.bytes(&v, &vlen)) {
          entry.skip(w3);
          continue;
        }
        if (f3 == 1) {
          is_final_key = vlen == 21 && memcmp(v, "triton_final_response", 21) == 0;
        } else if (f3 == 2) {
          pb::Reader param(v, vlen);
          uint32_t f4 = 0, w4 = 0;
          while (param.tag(&f4, &w4)) {
            if (f4 == 1 && w4 == pb::kVarint) {
              value = param.varint() != 0;
              has_value = true;
            } else {
              param.skip(w4);
            }
          }
        }
      }
      if (is_final_key && has_value) *final = value;
    }
  }
  if (!r.ok) *error = true;
}

void request_start(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index, bool retry) {
  if (!retry) c.attempts = 0;
  for (;;) {
    if (c.fd < 0 && !conn_open(lg, t, c, index)) break;
    c.in_flight = true;
    c.header_end = 0;
    c.t_recv_start = 0;
    c.t_start = now_ns();  // REQUEST_START == SEND_START (the request is pre-formed)
    c.t_send_end = c.t_start;
    if (lg->grpc) {
      const int rc = grpc_build(lg, c);
      if (rc > 0) {  // resumes when the peer's WINDOW_UPDATE arrives
        c.waiting_window = true;
        return;
      }
      if (rc < 0) break;
    } else {
      c.buf.clear();
      c.tx.clear();
      c.tx_idx = 0;
      const std::vector<uint8_t>& req = lg->requests[static_cast<size_t>(c.slot) * lg->rps + (lg->rps > 1 ? c.image : 0)];
      c.tx.push_back(iovec{const_cast<uint8_t*>(req.data()), req.size()});
      if (!lg->tails.empty() && lg->tail_sizes[c.slot] != 0) {
        c.tx.push_back(iovec{const_cast<uint8_t*>(lg->tails[c.slot]) + static_cast<uint64_t>(c.image) * lg->tail_stride,
                             static_cast<size_t>(lg->tail_sizes[c.slot])});
      }
    }
    if (conn_send(lg, t, c, index)) return;
    conn_close(t, c);  // keep-alive connection the server dropped: reconnect once
    if (++c.attempts >= 2) break;
  }
  std::this_thread::sleep_for(std::chrono::milliseconds(1));  // unreachable server: fail slowly, do not spin
  request_done(lg, t, c, index, false, now_ns());
}

void request_done(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index, bool ok, uint64_t t_end) {
  c.in_flight = false;
  {
    std::lock_guard<std::mutex> lk(t->stats.mu);
    if (ok) {
      t->stats.completed += 1;
      t->stats.total_ns += t_end - c.t_start;
      t->stats.send_ns += c.t_send_end - c.t_start;
      t->stats.recv_ns += t_end - c.t_recv_start;
      t->stats.latencies.push_back(t_end - c.t_start);
      if (lg->grpc_stream) {
        t->stats.responses += c.responses;
        t->stats.first_ns.push_back((c.t_first != 0 ? c.t_first : t_end) - c.t_start);
      }
    } else {
      t->stats.failed += 1;
    }
  }
  // look-ahead: the slot's next staging image is ready to go, no device work needed until the
  // last one is used (without per-request device work the images are simply cycled)
  bool more_images = false;
  if (ok && lg->lookahead > 1) {
    c.image = (c.image + 1) % lg->lookahead;
    more_images = c.image != 0;
  } else if (!ok) {
    c.image = 0;
  }
  if (lg->passthrough || more_images) {
    if (lg->stop.load(std::memory_order_relaxed)) return;
    if (ok) {
      request_start(lg, t, c, index, false);
    } else {
      // do not recurse on a dead server: retry from the event loop
      {
        std::lock_guard<std::mutex> lk(t->mu);
        t->ready.push_back(c.slot);
      }
      const uint64_t one = 1;
      if (write(t->evfd, &one, sizeof(one)) < 0) return;
    }
  } else {
    lg->returned.push(c.slot);
  }
}

void conn_readable(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index) {
  char tmp[16384];
  for (;;) {
    const ssize_t k = recv(c.fd, tmp, sizeof(tmp), MSG_DONTWAIT);
    if (k < 0) {
      if (errno == EINTR) continue;
      if (errno == EAGAIN || errno == EWOULDBLOCK) return;
    }
    if (k <= 0) {  // dropped
      conn_close(t, c);
      if (!c.in_flight) return;
      if (++c.attempts < 2 && !lg->stop.load(std::memory_order_relaxed)) request_start(lg, t, c, index, true);
      else request_done(lg, t, c, index, false, now_ns());
      return;
    }
    if (!c.in_flight) continue;  // stray bytes
    if (c.t_recv_start == 0) c.t_recv_start = now_ns();
    const size_t old = c.buf.size();
    c.buf.insert(c.buf.end(), tmp, tmp + k);
    if (c.header_end == 0) {
      for (size_t i = old > 3 ? old - 3 : 0; i + 3 < c.buf.size(); ++i) {
        if (c.buf[i] == '\r' && c.buf[i + 1] == '\n' && c.buf[i + 2] == '\r' && c.buf[i + 3] == '\n') {
          c.header_end = i + 4;
          c.body = content_length(c.buf.data(), c.header_end);
          break;
        }
      }
      if (c.header_end == 0 && c.buf.size() > (1u << 20)) {
        conn_close(t, c);
        request_done(lg, t, c, index, false, now_ns());
        return;
      }
    }
    if (c.header_end != 0 && c.buf.size() >= c.header_end + static_cast<size_t>(c.body)) {
      const uint64_t t_end = now_ns();
      int status = 0;
      if (c.buf.size() > 12 && memcmp(c.buf.data(), "HTTP/1.", 7) == 0) status = atoi(c.buf.data() + 9);
      request_done(lg, t, c, index, status == 200, t_end);
      return;  // one response per request; level-triggered epoll reports anything left
    }
  }
}

// HTTP/2 frames of a gRPC connection: acknowledgements, flow control, end of the call
void grpc_readable(tb200_loadgen* lg, Transport* t, Conn& c, uint32_t index) {
  namespace h2 = tb200::h2;
  char tmp[16384];
  bool closed = false;
  for (;;) {
    const ssize_t k = recv(c.fd, tmp, sizeof(tmp), MSG_DONTWAIT);
    if (k > 0) {
      if (c.in_flight && c.t_recv_start == 0 && c.tx_idx >= c.tx.size()) c.t_recv_start = now_ns();
      c.buf.insert(c.buf.end(), tmp, tmp + k);
      if (static_cast<size_t>(k) < sizeof(tmp)) break;
      continue;
    }
    if (k < 0 && errno == EINTR) continue;
    if (k < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) break;
    closed = true;
    break;
  }
  size_t pos = 0;
  bool finished = false, ok = false;
  while (!finished) {
    h2::FrameView f;
    const size_t n = h2::parse_frame(reinterpret_cast<const uint8_t*>(c.buf.data()) + pos, c.buf.size() - pos, &f);
    if (n == 0) break;
    pos += n;
    switch (f.type) {
      case h2::SETTINGS:
        if (!(f.flags & h2::kAck)) {
          for (uint32_t o = 0; o + 6 <= f.length; o += 6) {
            const uint16_t id = static_cast<uint16_t>((f.payload[o] << 8) | f.payload[o + 1]);
            const uint32_t v = h2::get_u32(f.payload + o + 2);
            if (id == h2::kSettingsInitialWindow) {
              c.stream_window += static_cast<int64_t>(v) - static_cast<int64_t>(c.peer_stream_window);
              c.peer_stream_window = v;
            }
            else if (id == h2::kSettingsMaxFrame && v >= h2::kDefaultMaxFrame) c.peer_max_frame = std::min<uint32_t>(v, 1u << 20);
          }
          c.ctrl += h2::frame(h2::SETTINGS, h2::kAck, 0, "");
        }
        break;
      case h2::PING:
        if (!(f.flags & h2::kAck) && f.length == 8) c.ctrl += h2::frame(h2::PING, h2::kAck, 0, std::string(reinterpret_cast<const char*>(f.payload), 8));
        break;
      case h2::WINDOW_UPDATE:
        if (f.length == 4 && f.stream == 0) c.conn_window += h2::get_u32(f.payload) & 0x7FFFFFFFu;
        else if (f.length == 4 && f.stream == c.cur_stream) c.stream_window += h2::get_u32(f.payload) & 0x7FFFFFFFu;
        break;
      case h2::DATA:
        c.recv_consumed += f.length;
        if (lg->grpc_stream) {
          if (f.stream != c.cur_stream) break;
          c.stream_recv_consumed += f.length;
          c.rx_msg.append(reinterpret_cast<const char*>(f.payload), f.length);
          size_t off = 0;
          while (c.rx_msg.size() - off >= 5) {
            const uint8_t* h = reinterpret_cast<const uint8_t*>(c.rx_msg.data()) + off;
            const size_t len = h2::get_u32(h + 1);
            if (c.rx_msg.size() - off - 5 < len) break;
            if (c.in_flight && !finished) {
              bool error = false, final = true;
              parse_stream_response(h + 5, len, &error, &final);
              c.responses += 1;
              if (c.t_first == 0) c.t_first = now_ns();
              if (error || final) {
                finished = true;
                ok = !error;
              }
            }
            off += 5 + len;
          }
          if (off) c.rx_msg.erase(0, off);
          if (f.flags & h2::kEndStream) {  // the server ended the stream: start over on a new connection
            c.goaway = true;
            if (c.in_flight && !finished) finished = true;
          }
          break;
        }
        if (f.stream == c.cur_stream && c.in_flight) {
          // unary calls return stream-level credit too: a response larger than the stream window
          // we advertise (h2::kOurStreamWindow) would otherwise stall the server for good
          if (!(f.flags & h2::kEndStream)) c.stream_recv_consumed += f.length;
          if (f.length >= 5) c.got_data = true;
          if (f.flags & h2::kEndStream) {
            finished = true;
            ok = c.got_data;
          }
        }
        break;
      case h2::HEADERS:
        if (lg->grpc_stream) {
          if (f.stream == c.cur_stream && (f.flags & h2::kEndStream)) {  // trailers: the stream is over
            c.goaway = true;
            if (c.in_flight) finished = true;
          }
          break;
        }
        if (f.stream == c.cur_stream && c.in_flight && (f.flags & h2::kEndStream)) {
          finished = true;  // trailers; an error arrives as a trailers-only response without DATA
          ok = c.got_data;
        }
        break;
      case h2::RST_STREAM:
        if (f.stream == c.cur_stream && lg->grpc_stream) c.goaway = true;
        if (f.stream == c.cur_stream && c.in_flight) finished = true;
        break;
      case h2::GOAWAY:
        c.goaway = true;
        break;
      default:
        break;
    }
  }
  if (pos) c.buf.erase(c.buf.begin(), c.buf.begin() + static_cast<long>(pos));
  if (c.stream_recv_consumed >= (tb200::h2::kOurStreamWindow / 2) && c.fd >= 0 && !c.goaway) {
    c.ctrl += h2::window_update(c.cur_stream, static_cast<uint32_t>(c.stream_recv_consumed));
    c.stream_recv_consumed = 0;
  }
  if (c.recv_consumed >= (1u << 28)) {  // give the connection window back long before it runs out
    c.ctrl += h2::window_update(0, static_cast<uint32_t>(c.recv_consumed));
    c.recv_consumed = 0;
  }
  h2_flush_ctrl(c);
  if (finished) {
    const uint64_t t_end = now_ns();
    if (c.t_recv_start == 0) c.t_recv_start = t_end;
    if (c.goaway) conn_close(t, c);
    request_done(lg, t, c, index, ok, t_end);
    return;
  }
  if (c.goaway && !c.in_flight && c.fd >= 0) {  // nothing pending on a connection the server is done with
    conn_close(t, c);
    return;
  }
  if (closed) {
    conn_close(t, c);
    if (!c.in_flight) return;
    c.waiting_window = false;
    if (++c.attempts < 2 && !lg->stop.load(std::memory_order_relaxed)) request_start(lg, t, c, index, true);
    else request_done(lg, t, c, index, false, now_ns());
    return;
  }
  if (c.waiting_window && c.in_flight) {  // a WINDOW_UPDATE may have made room
    const int rc = grpc_build(lg, c);
    if (rc == 0) {
      c.waiting_window = false;
      if (!conn_send(lg, t, c, index)) {
        conn_close(t, c);
        request_done(lg, t, c, index, false, now_ns());
      }
    } else if (rc < 0) {
      c.waiting_window = false;
      request_done(lg, t, c, index, false, now_ns());
    }
  }
}

void transport_main(tb200_loadgen* lg, Transport* t) {
  if (lg->passthrough) {
    for (uint32_t i = 0; i < t->conns.size(); ++i) request_start(lg, t, t->conns[i], i, false);
  }
  std::vector<int> ready;
  epoll_event events[64];
  uint64_t drain_deadline = 0;
  for (;;) {
    if (lg->stop.load(std::memory_order_relaxed)) {
      // stopping: issue nothing new, but let the requests in flight complete (the server is
      // still reading the regions they name) -- for at most two seconds
      bool busy = false;
      for (const Conn& c : t->conns) busy = busy || c.in_flight;
      if (drain_deadline == 0) drain_deadline = now_ns() + 2000000000ull;
      if (!busy || now_ns() > drain_deadline) break;
    }
    const int n = epoll_wait(t->epfd, events, 64, 50);
    for (int e = 0; e < n; ++e) {
      const uint32_t tag = events[e].data.u32;
      if (tag == kEvTag) {
        uint64_t count;
        if (read(t->evfd, &count, sizeof(count)) < 0) continue;
        {
          std::lock_guard<std::mutex> lk(t->mu);
          ready.swap(t->ready);
        }
        for (int slot : ready) {
          if (lg->stop.load(std::memory_order_relaxed)) break;
          const uint32_t i = static_cast<uint32_t>(slot / static_cast<int>(lg->transports.size()));
          request_start(lg, t, t->conns[i], i, false);
        }
        ready.clear();
        continue;
      }
      Conn& c = t->conns[tag];
      if (c.fd < 0) continue;
      if ((events[e].events & EPOLLOUT) && c.in_flight && !conn_send(lg, t, c, tag)) {
        conn_close(t, c);
        if (++c.attempts < 2) request_start(lg, t, c, tag, true);
        else request_done(lg, t, c, tag, false, now_ns());
        continue;
      }
      if (events[e].events & (EPOLLIN | EPOLLERR | EPOLLHUP)) {
        if (lg->grpc) grpc_readable(lg, t, c, tag);
        else conn_readable(lg, t, c, tag);
      }
    }
  }
  for (Conn& c : t->conns) conn_close(t, c);
}

// hand slots to the transport threads that own them: one eventfd write per thread
void release_slots(tb200_loadgen* lg, const std::vector<int>& slots) {
  const int T = static_cast<int>(lg->transports.size());
  // one lock and one wake-up per transport thread, not per slot
  static thread_local std::vector<std::vector<int>> per;
  per.resize(static_cast<size_t>(T));
  for (auto& v : per) v.clear();
  for (int s : slots) per[static_cast<size_t>(s % T)].push_back(s);
  const uint64_t one = 1;
  for (int i = 0; i < T; ++i) {
    if (per[static_cast<size_t>(i)].empty()) continue;
    Transport* t = lg->transports[static_cast<size_t>(i)].get();
    {
      std::lock_guard<std::mutex> lk(t->mu);
      t->ready.insert(t->ready.end(), per[static_cast<size_t>(i)].begin(), per[static_cast<size_t>(i)].end());
    }
    if (write(t->evfd, &one, sizeof(one)) < 0) continue;
  }
}

// The issue loop with several passes in flight (cfg.pipeline_depth > 1).  A pass = the slots whose
// responses came back: their outputs are validated and their next inputs generated
// (tb200_step_submit: fill on the context's stream, validation on its side stream, events behind
// both).  The thread forms pass i+1 -- collects returned slots, builds the job lists, copies the
// tables, launches -- while the device runs pass i, and retires passes in order (tb200_step_wait,
// read the results, hand the slots back to their transport threads).  Passes in flight own
// disjoint slots, so consecutive fills overlap on the device as well (fill_uniform_kernel's
// programmatic dependent launch).  This is where the reference's clients hand every request
// through a Python future / queue (grpc/_client.py:1574-1741, grpc/_infer_stream.py:108-168).
void device_main_pipelined(tb200_loadgen* lg) {
  struct Pass {
    std::vector<int> batch;
    std::vector<tb200_check_job> checks;
    tb200_check_result* results = nullptr;       // device address of the pass's result block
    const tb200_check_result* results_host = nullptr;  // the same block as the host reads it
    uint64_t ticket = 0;
    int rc = TB200_OK;
  };
  const uint32_t depth = lg->pipeline_depth;
  const size_t max_checks = static_cast<size_t>(lg->concurrency) * static_cast<size_t>(std::max(lg->check_per_slot, 0));
  std::deque<Pass> inflight;
  std::vector<Pass> pool(depth);  // reused vectors, one per ring position
  uint64_t seq = 0;
  std::vector<tb200_fill_job> fills;
  std::vector<tb200_copy_job> copies;
  const bool do_check = lg->check_per_slot > 0;
  const bool do_fill = lg->regenerate && lg->fill_per_slot > 0;
  const bool do_copy = lg->regenerate && lg->replay_entries > 0;

  auto retire = [&](Pass& p) {
    uint64_t bad = 0, mism = 0;
    int rc = p.rc;
    if (rc == TB200_OK) rc = tb200_step_wait(lg->ctx, p.ticket);
    if (rc != TB200_OK) {
      std::lock_guard<std::mutex> lk(lg->dev_mu);
      if (lg->error.empty()) lg->error = tb200_last_error();
    } else {
      for (size_t k = 0; k < p.checks.size(); ++k) {
        if (p.checks[k].kind == TB200_CHECK_TOP1) bad += p.results_host[k].mismatches;
        else if (p.checks[k].kind != TB200_CHECK_SUM) mism += p.results_host[k].mismatches;
      }
    }
    {
      std::lock_guard<std::mutex> lk(lg->dev_mu);
      lg->device_batches += 1;
      lg->device_slots += p.batch.size();
      lg->nonfinite += bad;
      lg->mismatches += mism;
    }
    release_slots(lg, p.batch);
  };

  // A pass costs the host ~15 us of launches and table copies whatever its size, so while passes
  // are in flight a new one is only worth forming once enough slots are back (an eighth of the
  // concurrency); fewer than that wait for the oldest pass to retire and accumulate meanwhile.
  // With nothing in flight whatever is back goes out at once (latency at low concurrency).
  const size_t min_batch = std::max<size_t>(1, static_cast<size_t>(lg->concurrency) / 8);
  std::vector<int> batch;
  while (!lg->stop.load(std::memory_order_relaxed)) {
    if (inflight.empty() && batch.empty()) {
      const int first = lg->returned.pop(50);
      if (first < 0) continue;
      batch.push_back(first);
    }
    lg->returned.drain(batch);
    if (inflight.empty() && lg->device_window_ns != 0) {  // accumulation window, see device_main
      const uint64_t t0 = now_ns();
      while (batch.size() < static_cast<size_t>(lg->concurrency)) {
        const uint64_t el = now_ns() - t0;
        if (el >= lg->device_window_ns) break;
        const int s = lg->returned.pop_ns(lg->device_window_ns - el);
        if (s < 0) break;
        batch.push_back(s);
        lg->returned.drain(batch);
      }
    }
    const bool submit = !batch.empty() && (inflight.empty() || (inflight.size() < depth && batch.size() >= min_batch));
    if (submit) {
      Pass p = std::move(pool[seq % depth]);
      p.batch.clear();
      p.batch.swap(batch);
      p.checks.clear();
      fills.clear();
      copies.clear();
      if (do_check) {
        for (int s : p.batch) append_checks(lg, s, p.checks);
      }
      if (do_copy) {
        for (int s : p.batch) {
          lg->replay_gen[static_cast<size_t>(s)] += 1;
          append_copies(lg, s, copies);
        }
      }
      if (do_fill) {
        for (int s : p.batch) {
          for (int k = 0; k < lg->fill_per_slot; ++k) fills.push_back(lg->fill_jobs[s * lg->fill_per_slot + k]);
        }
        lg->epoch += 1ull << 20;  // fresh Philox streams for every generation
      }
      p.results = lg->own_results + (seq % depth) * max_checks;
      p.results_host = static_cast<const tb200_check_result*>(lg->own_results_host) + (seq % depth) * max_checks;
      if (do_copy) {
        p.rc = tb200_step_submit_copy(lg->ctx, copies.data(), static_cast<int>(copies.size()), p.checks.data(),
                                      static_cast<int>(p.checks.size()), p.results, &p.ticket);
      } else {
        p.rc = tb200_step_submit(lg->ctx, fills.data(), static_cast<int>(fills.size()), lg->seed, lg->epoch, p.checks.data(),
                                 static_cast<int>(p.checks.size()), p.results, &p.ticket);
      }
      ++seq;
      inflight.push_back(std::move(p));
      if (inflight.size() < depth) continue;  // room for another pass: look for returned slots first
    }
    if (!inflight.empty()) {  // too little came back, or the pipeline is full: retire the oldest pass
      retire(inflight.front());
      pool[(seq - inflight.size()) % depth] = std::move(inflight.front());
      inflight.pop_front();
    }
  }
  while (!inflight.empty()) {
    retire(inflight.front());
    inflight.pop_front();
  }
}

// validate + regenerate the slots that came back, one launch each, then release them
void device_main(tb200_loadgen* lg) {
  if (lg->pipeline_depth > 1 && lg->ctx != nullptr) {
    device_main_pipelined(lg);
    return;
  }
  std::vector<int> batch;
  std::vector<tb200_fill_job> fills;
  std::vector<tb200_check_job> checks;
  std::vector<tb200_copy_job> copies;
  while (!lg->stop.load(std::memory_order_relaxed)) {
    batch.clear();
    const int first = lg->returned.pop(50);
    if (first < 0) continue;
    batch.push_back(first);
    lg->returned.drain(batch);
    // Accumulation window (cfg.device_window_us): without MPS client and server are two CUDA
    // contexts time-sliced on one GPU and every hand-over costs ~100 us, so a pass should then
    // cover the slots that are about to return anyway.  Ends at once when all are back.
    const uint64_t window_ns = lg->device_window_ns;
    if (window_ns != 0 && lg->ctx != nullptr) {
      const uint64_t t0 = now_ns();
      while (batch.size() < static_cast<size_t>(lg->concurrency)) {
        const uint64_t el = now_ns() - t0;
        if (el >= window_ns) break;
        const int s = lg->returned.pop_ns(window_ns - el);
        if (s < 0) break;
        batch.push_back(s);
        lg->returned.drain(batch);
      }
    }
    if (lg->ctx != nullptr) {
      uint64_t bad = 0, mism = 0;
      const bool do_check = lg->check_per_slot > 0;
      const bool do_fill = lg->regenerate && lg->fill_per_slot > 0;
      const bool do_copy = lg->regenerate && lg->replay_entries > 0;
      checks.clear();
      fills.clear();
      copies.clear();
      if (do_check) {
        for (int s : batch) append_checks(lg, s, checks);
      }
      if (do_copy) {
        for (int s : batch) {
          lg->replay_gen[static_cast<size_t>(s)] += 1;
          append_copies(lg, s, copies);
        }
      }
      if (do_fill) {
        for (int s : batch) {
          for (int k = 0; k < lg->fill_per_slot; ++k) fills.push_back(lg->fill_jobs[s * lg->fill_per_slot + k]);
        }
        lg->epoch += 1ull << 20;  // fresh Philox streams for every generation
      }
      // validation of the returned outputs + generation of the next inputs: parallel branches
      // under one sync (tb200_step_sync).  TB200_LOADGEN_DEVICE_MODE (experiments only):
      // 1 = check, sync, fill, sync; 2 = one stream, one sync
      static const int mode = getenv("TB200_LOADGEN_DEVICE_MODE") ? atoi(getenv("TB200_LOADGEN_DEVICE_MODE")) : 0;
      int rc = TB200_OK;
      if (do_copy) {  // replayed entries: validate, copy the next entries, one sync
        if (do_check) rc = tb200_check_async(lg->ctx, checks.data(), static_cast<int>(checks.size()), lg->results);
        if (rc == TB200_OK) rc = tb200_concat_async(lg->ctx, copies.data(), static_cast<int>(copies.size()));
        if (rc == TB200_OK) rc = tb200_ctx_sync(lg->ctx);
      } else if (do_fill && mode == 0) {
        rc = tb200_step_sync(lg->ctx, fills.data(), static_cast<int>(fills.size()), lg->seed, lg->epoch,
                             checks.data(), static_cast<int>(checks.size()), lg->results);
      } else {
        if (do_check) {
          rc = tb200_check_async(lg->ctx, checks.data(), static_cast<int>(checks.size()), lg->results);
          if (rc == TB200_OK && (mode == 1 || !do_fill)) rc = tb200_ctx_sync(lg->ctx);
        }
        if (rc == TB200_OK && do_fill) {
          rc = tb200_fill_async(lg->ctx, fills.data(), static_cast<int>(fills.size()), lg->seed, lg->epoch);
          if (rc == TB200_OK) rc = tb200_ctx_sync(lg->ctx);
        }
      }
      if (rc != TB200_OK) {
        std::lock_guard<std::mutex> lk(lg->dev_mu);
        lg->error = tb200_last_error();
      } else {
        for (size_t k = 0; k < checks.size(); ++k) {
          if (checks[k].kind == TB200_CHECK_TOP1) bad += lg->results[k].mismatches;
          else if (checks[k].kind != TB200_CHECK_SUM) mism += lg->results[k].mismatches;
        }
      }
      std::lock_guard<std::mutex> lk(lg->dev_mu);
      lg->device_batches += 1;
      lg->device_slots += batch.size();
      lg->nonfinite += bad;
      lg->mismatches += mism;
    }
    release_slots(lg, batch);
  }
}

}  // namespace

namespace tb200 {
void set_last_error(const char* msg);  // runtime.cu: feeds tb200_last_error()
}

namespace {
int lg_fail(int code, const char* msg) {
  tb200::set_last_error(msg);
  return code;
}
}  // namespace

extern "C" {

int tb200_loadgen_create(const tb200_loadgen_config* cfg, tb200_loadgen** out) {
  if (cfg == nullptr || out == nullptr || cfg->host == nullptr || cfg->concurrency <= 0 ||
      cfg->requests == nullptr || cfg->request_sizes == nullptr) {
    return lg_fail(TB200_ERR_INVALID, "bad load generator configuration");
  }
  tb200_loadgen* lg = new tb200_loadgen();
  lg->host = cfg->host;
  lg->port = cfg->port;
  lg->concurrency = cfg->concurrency;
  lg->rps = cfg->requests_per_slot > 1 ? cfg->requests_per_slot : 1;
  const size_t nreq = static_cast<size_t>(cfg->concurrency) * lg->rps;
  lg->requests.resize(nreq);
  for (size_t s = 0; s < nreq; ++s) {
    lg->requests[s].assign(cfg->requests[s], cfg->requests[s] + cfg->request_sizes[s]);
  }
  lg->ctx = cfg->ctx;
  lg->seed = cfg->seed;
  lg->regenerate = cfg->regenerate != 0;
  lg->device_window_ns = 1000ull * cfg->device_window_us;
  lg->lookahead = cfg->lookahead > 1 ? cfg->lookahead : 1;
  lg->tail_stride = cfg->tail_stride;
  if (lg->lookahead > 1 && (cfg->tails == nullptr || cfg->tail_stride == 0) && lg->rps != lg->lookahead) {
    delete lg;
    return lg_fail(TB200_ERR_INVALID, "lookahead needs tails with a tail_stride, or one request per image (requests_per_slot)");
  }
  if (lg->rps > 1 && lg->rps != lg->lookahead) {
    delete lg;
    return lg_fail(TB200_ERR_INVALID, "requests_per_slot must equal lookahead");
  }
  lg->grpc = cfg->protocol == 1 || cfg->protocol == 2;
  lg->grpc_stream = cfg->protocol == 2;
  if (cfg->protocol > 2) {
    delete lg;
    return lg_fail(TB200_ERR_INVALID, "unknown load generator protocol");
  }
  if (lg->grpc) {
    lg->grpc_headers = tb200::h2::grpc_request_headers(lg->host + ":" + std::to_string(lg->port),
                                                       cfg->grpc_path ? cfg->grpc_path
                                                                      : (lg->grpc_stream ? "/inference.GRPCInferenceService/ModelStreamInfer"
                                                                                         : "/inference.GRPCInferenceService/ModelInfer"));
  }
  if (cfg->ctx != nullptr && cfg->replay_entries > 0) {
    const int L = static_cast<int>(lg->lookahead);
    if (cfg->copy_jobs == nullptr || cfg->copy_jobs_per_slot <= 0 || cfg->copy_src_stride == nullptr ||
        cfg->copy_jobs_per_slot % L != 0 || (cfg->check_jobs_per_slot > 0 && cfg->check_jobs_per_slot % L != 0)) {
      delete lg;
      return lg_fail(TB200_ERR_INVALID, "replayed inputs need copy jobs (and check jobs) for every staging image of a slot");
    }
    lg->replay_entries = cfg->replay_entries;
    lg->copy_per_slot = cfg->copy_jobs_per_slot;
    lg->copy_jobs.assign(cfg->copy_jobs, cfg->copy_jobs + static_cast<size_t>(cfg->concurrency) * cfg->copy_jobs_per_slot);
    lg->copy_stride.assign(cfg->copy_src_stride, cfg->copy_src_stride + cfg->copy_jobs_per_slot);
    if (cfg->check_b_stride != nullptr && cfg->check_jobs_per_slot > 0) {
      lg->check_b_stride.assign(cfg->check_b_stride, cfg->check_b_stride + cfg->check_jobs_per_slot);
    }
    lg->replay_gen.assign(static_cast<size_t>(cfg->concurrency), 0);
  } else if (cfg->ctx != nullptr && cfg->fill_jobs != nullptr && cfg->fill_jobs_per_slot > 0) {
    lg->fill_per_slot = cfg->fill_jobs_per_slot;
    lg->fill_jobs.assign(cfg->fill_jobs, cfg->fill_jobs + static_cast<size_t>(cfg->concurrency) * cfg->fill_jobs_per_slot);
  }
  if (cfg->ctx != nullptr && cfg->check_jobs != nullptr && cfg->check_jobs_per_slot > 0 && cfg->results != nullptr) {
    lg->check_per_slot = cfg->check_jobs_per_slot;
    lg->check_jobs.assign(cfg->check_jobs, cfg->check_jobs + static_cast<size_t>(cfg->concurrency) * cfg->check_jobs_per_slot);
    lg->results = cfg->results;
  }
  if (cfg->tails != nullptr && cfg->tail_sizes != nullptr) {
    lg->tails.assign(cfg->tails, cfg->tails + cfg->concurrency);
    lg->tail_sizes.assign(cfg->tail_sizes, cfg->tail_sizes + cfg->concurrency);
  }
  lg->passthrough = lg->ctx == nullptr || (lg->check_per_slot == 0 && !(lg->regenerate && (lg->fill_per_slot > 0 || lg->replay_entries > 0)));
  lg->pipeline_depth = cfg->pipeline_depth == 0 ? 1u : std::min<uint32_t>(cfg->pipeline_depth, TB200_STEP_DEPTH / 2);
  if (getenv("TB200_LOADGEN_DEVICE_MODE") != nullptr) lg->pipeline_depth = 1;  // the experiment modes are synchronous
  if (lg->pipeline_depth > 1 && !lg->passthrough) {
    // every pass in flight writes its own block of results
    const uint64_t per_pass = static_cast<uint64_t>(cfg->concurrency) * static_cast<uint64_t>(std::max(lg->check_per_slot, 1));
    void* h = nullptr;
    void* d = nullptr;
    if (tb200_host_alloc(per_pass * lg->pipeline_depth * sizeof(tb200_check_result), &h, &d) != TB200_OK) {
      delete lg;
      return lg_fail(TB200_ERR_CUDA, tb200_last_error());
    }
    lg->own_results_host = h;
    lg->own_results = static_cast<tb200_check_result*>(d);
  }
  *out = lg;
  return TB200_OK;
}

uint64_t tb200_loadgen_replay_entry(uint64_t slot, uint64_t request, uint32_t lookahead, int once, uint64_t entries) {
  if (entries == 0) return 0;
  const uint64_t r = once ? request % (lookahead > 1 ? lookahead : 1) : request;
  return (slot % entries + r % entries) % entries;
}

int tb200_loadgen_start(tb200_loadgen* lg) {
  if (lg == nullptr || lg->started) return lg_fail(TB200_ERR_STATE, "load generator already started");
  // initial generation of every slot: one launch
  if (lg->ctx != nullptr && lg->replay_entries > 0) {
    std::vector<tb200_copy_job> copies;
    for (int s = 0; s < lg->concurrency; ++s) {
      lg->replay_gen[static_cast<size_t>(s)] = 0;
      append_copies(lg, s, copies);
    }
    if (tb200_concat_async(lg->ctx, copies.data(), static_cast<int>(copies.size())) != 0 || tb200_ctx_sync(lg->ctx) != 0) {
      return lg_fail(TB200_ERR_CUDA, tb200_last_error());
    }
  } else if (lg->ctx != nullptr && lg->fill_per_slot > 0) {
    if (tb200_fill_async(lg->ctx, lg->fill_jobs.data(), static_cast<int>(lg->fill_jobs.size()), lg->seed, 0) != 0 ||
        tb200_ctx_sync(lg->ctx) != 0) {
      return lg_fail(TB200_ERR_CUDA, tb200_last_error());
    }
  }
  lg->started = true;
  lg->window_start_ns = now_ns();
  // transport threads: ~8 connections each, at most 32 threads (and half the host's cores)
  const int hw = static_cast<int>(std::max(2u, std::thread::hardware_concurrency()));
  const int T = std::max(1, std::min({(lg->concurrency + 7) / 8, 32, hw / 2}));
  lg->transports.clear();
  for (int i = 0; i < T; ++i) {
    std::unique_ptr<Transport> t(new Transport());
    t->epfd = epoll_create1(0);
    t->evfd = eventfd(0, EFD_NONBLOCK);
    if (t->epfd < 0 || t->evfd < 0) return lg_fail(TB200_ERR_IO, "epoll / eventfd setup failed");
    epoll_event ev{};
    ev.events = EPOLLIN;
    ev.data.u32 = kEvTag;
    epoll_ctl(t->epfd, EPOLL_CTL_ADD, t->evfd, &ev);
    lg->transports.push_back(std::move(t));
  }
  for (int s = 0; s < lg->concurrency; ++s) {  // slot s -> thread s % T, connection s / T
    Conn c;
    c.slot = s;
    c.buf.reserve(4096);
    lg->transports[static_cast<size_t>(s % T)]->conns.push_back(std::move(c));
  }
  if (!lg->passthrough) {
    std::vector<int> all(static_cast<size_t>(lg->concurrency));
    for (int s = 0; s < lg->concurrency; ++s) all[static_cast<size_t>(s)] = s;
    release_slots(lg, all);
    lg->threads.emplace_back(device_main, lg);
  }
  for (auto& t : lg->transports) lg->threads.emplace_back(transport_main, lg, t.get());
  return TB200_OK;
}

int tb200_loadgen_window(tb200_loadgen* lg, double seconds, tb200_loadgen_stats* out) {
  if (lg == nullptr || out == nullptr || !lg->started) return lg_fail(TB200_ERR_STATE, "load generator not running");
  if (seconds > 0) std::this_thread::sleep_for(std::chrono::duration<double>(seconds));
  memset(out, 0, sizeof(*out));
  std::vector<uint64_t> lat, first;
  for (auto& tr : lg->transports) {
    WorkerStats& st = tr->stats;
    std::lock_guard<std::mutex> lk(st.mu);
    out->completed_request_count += st.completed;
    out->failed_request_count += st.failed;
    out->cumulative_total_request_time_ns += st.total_ns;
    out->cumulative_send_time_ns += st.send_ns;
    out->cumulative_receive_time_ns += st.recv_ns;
    lat.insert(lat.end(), st.latencies.begin(), st.latencies.end());
    st.latencies.clear();
    first.insert(first.end(), st.first_ns.begin(), st.first_ns.end());
    st.first_ns.clear();
    out->response_count += st.responses;
    st.completed = st.failed = st.total_ns = st.send_ns = st.recv_ns = st.responses = 0;
  }
  const uint64_t t = now_ns();
  out->window_seconds = static_cast<double>(t - lg->window_start_ns) * 1e-9;
  lg->window_start_ns = t;
  if (!lat.empty()) {
    std::sort(lat.begin(), lat.end());
    auto pct = [&](double p) { return lat[std::min(lat.size() - 1, static_cast<size_t>(p * (lat.size() - 1) + 0.5))]; };
    out->p50_ns = pct(0.50);
    out->p90_ns = pct(0.90);
    out->p95_ns = pct(0.95);
    out->p99_ns = pct(0.99);
    out->min_ns = lat.front();
    out->max_ns = lat.back();
  }
  if (!first.empty()) {
    std::sort(first.begin(), first.end());
    auto pct = [&](double p) { return first[std::min(first.size() - 1, static_cast<size_t>(p * (first.size() - 1) + 0.5))]; };
    out->first_response_p50_ns = pct(0.50);
    out->first_response_p99_ns = pct(0.99);
  }
  {
    std::lock_guard<std::mutex> lk(lg->dev_mu);
    out->device_batches = lg->device_batches;
    out->device_slots = lg->device_slots;
    out->nonfinite_outputs = lg->nonfinite;
    out->check_mismatches = lg->mismatches;
    lg->device_batches = lg->device_slots = lg->nonfinite = lg->mismatches = 0;
    if (!lg->error.empty()) return lg_fail(TB200_ERR_CUDA, lg->error.c_str());
  }
  return TB200_OK;
}

int tb200_loadgen_wait_count(tb200_loadgen* lg, uint64_t count, double timeout_seconds, uint64_t* reached) {
  if (lg == nullptr || !lg->started) return lg_fail(TB200_ERR_STATE, "load generator not running");
  const uint64_t deadline = now_ns() + static_cast<uint64_t>(std::max(0.0, timeout_seconds) * 1e9);
  uint64_t total = 0;
  for (;;) {
    total = 0;
    for (auto& tr : lg->transports) {
      std::lock_guard<std::mutex> lk(tr->stats.mu);
      total += tr->stats.completed + tr->stats.failed;
    }
    if (total >= count || now_ns() >= deadline) break;
    {
      std::lock_guard<std::mutex> lk(lg->dev_mu);
      if (!lg->error.empty()) break;
    }
    std::this_thread::sleep_for(std::chrono::microseconds(100));
  }
  if (reached != nullptr) *reached = total;
  return TB200_OK;
}

int tb200_loadgen_stop(tb200_loadgen* lg) {
  if (lg == nullptr) return TB200_OK;
  lg->stop.store(true);
  for (std::thread& t : lg->threads) {
    if (t.joinable()) t.join();
  }
  lg->threads.clear();
  for (auto& t : lg->transports) {
    if (t->evfd >= 0) close(t->evfd);
    if (t->epfd >= 0) close(t->epfd);
  }
  lg->transports.clear();
  lg->stop.store(false);
  lg->started = false;
  return TB200_OK;
}

int tb200_loadgen_destroy(tb200_loadgen* lg) {
  if (lg == nullptr) return TB200_OK;
  tb200_loadgen_stop(lg);
  if (lg->own_results_host != nullptr) tb200_host_free(lg->own_results_host);
  delete lg;
  return TB200_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------
// canned-response server (tooling for measuring the generator)
// ---------------------------------------------------------------------------------------
struct tb200_stub_server {
  tb200::EpollHttpServer http;
  std::string response;
};

extern "C" {

int tb200_stub_server_start(const char* host, int* port, const char* response_body, tb200_stub_server** out) {
  if (host == nullptr || port == nullptr || out == nullptr) return lg_fail(TB200_ERR_INVALID, "NULL argument");
  tb200_stub_server* s = new tb200_stub_server();
  s->response = tb200::EpollHttpServer::Response(200, response_body ? response_body : "{}");
  const int hw = static_cast<int>(std::max(2u, std::thread::hardware_concurrency()));
  const std::string* canned = &s->response;
  if (!s->http.Start(host, port, std::min(16, hw / 2), [canned](uint64_t, const tb200::HttpRequest&, std::string* resp) {
        *resp = *canned;
        return true;
      })) {
    delete s;
    return lg_fail(TB200_ERR_IO, "cannot bind the stub server");
  }
  *out = s;
  return TB200_OK;
}

int tb200_stub_server_stop(tb200_stub_server* s) {
  if (s == nullptr) return TB200_OK;
  s->http.Stop();
  delete s;
  return TB200_OK;
}

int tb200_grpc_stub_server_start(const char* host, int* port, const uint8_t* response, uint64_t response_bytes,
                                 tb200_grpc_stub_server** out);
int tb200_grpc_stub_server_start_streaming(const char* host, int* port, const uint8_t* response, uint64_t response_bytes,
                                           const uint8_t* final_response, uint64_t final_bytes, int responses_per_request,
                                           tb200_grpc_stub_server** out);
int tb200_grpc_stub_server_stop(tb200_grpc_stub_server* s);

}  // extern "C"

struct tb200_grpc_stub_server {
  tb200::H2StubServer h2;
};
struct tb200_grpc_echo_server {
  tb200::EpollGrpcServer server;
};

extern "C" {

int tb200_grpc_stub_server_start(const char* host, int* port, const uint8_t* response, uint64_t response_bytes,
                                 tb200_grpc_stub_server** out) {
  if (host == nullptr || port == nullptr || out == nullptr || (response == nullptr && response_bytes != 0)) {
    return lg_fail(TB200_ERR_INVALID, "NULL argument");
  }
  tb200_grpc_stub_server* s = new tb200_grpc_stub_server();
  const int hw = static_cast<int>(std::max(2u, std::thread::hardware_concurrency()));
  if (!s->h2.Start(host, port, std::min(16, hw / 2), std::string(reinterpret_cast<const char*>(response), response_bytes))) {
    delete s;
    return lg_fail(TB200_ERR_IO, "cannot bind the gRPC stub server");
  }
  *out = s;
  return TB200_OK;
}

int tb200_grpc_stub_server_start_streaming(const char* host, int* port, const uint8_t* response, uint64_t response_bytes,
                                           const uint8_t* final_response, uint64_t final_bytes, int responses_per_request,
                                           tb200_grpc_stub_server** out) {
  if (host == nullptr || port == nullptr || out == nullptr || (response == nullptr && response_bytes != 0) ||
      (final_response == nullptr && final_bytes != 0) || responses_per_request < 1) {
    return lg_fail(TB200_ERR_INVALID, "NULL argument / responses_per_request < 1");
  }
  tb200_grpc_stub_server* s = new tb200_grpc_stub_server();
  const int hw = static_cast<int>(std::max(2u, std::thread::hardware_concurrency()));
  if (!s->h2.StartStreaming(host, port, std::min(16, hw / 2), std::string(reinterpret_cast<const char*>(response), response_bytes),
                            std::string(reinterpret_cast<const char*>(final_response), final_bytes), responses_per_request)) {
    delete s;
    return lg_fail(TB200_ERR_IO, "cannot bind the gRPC stub server");
  }
  *out = s;
  return TB200_OK;
}

int tb200_grpc_echo_server_start(const char* host, int* port, tb200_grpc_echo_server** out) {
  if (host == nullptr || port == nullptr || out == nullptr) return lg_fail(TB200_ERR_INVALID, "NULL argument");
  tb200_grpc_echo_server* s = new tb200_grpc_echo_server();
  auto handler = [](uint64_t, const std::string& path, std::string&& message, bool is_message, bool half_close, tb200::GrpcReply* reply) {
    const bool stream = path.size() >= 16 && path.compare(path.size() - 16, 16, "ModelStreamInfer") == 0;
    if (path.find("/inference.GRPCInferenceService/") != 0) {
      reply->status = 12;  // UNIMPLEMENTED
      reply->status_message = "unknown service in " + path;
      return true;
    }
    if (is_message) {
      if (stream) {  // ModelStreamInferResponse{infer_response = the request bytes}
        std::string wrapped;
        tb200::pb::put_bytes(&wrapped, 2, message);
        reply->messages.push_back(std::move(wrapped));
      } else {
        reply->messages.push_back(std::move(message));
      }
    }
    reply->finish = stream ? half_close : true;
    return true;
  };
  if (!s->server.Start(host, port, 4, handler)) {
    delete s;
    return lg_fail(TB200_ERR_IO, "cannot bind the gRPC echo server");
  }
  *out = s;
  return TB200_OK;
}

int tb200_grpc_echo_server_stop(tb200_grpc_echo_server* s) {
  if (s == nullptr) return TB200_OK;
  s->server.Stop();
  delete s;
  return TB200_OK;
}

int tb200_grpc_stub_server_stop(tb200_grpc_stub_server* s) {
  if (s == nullptr) return TB200_OK;
  s->h2.Stop();
  delete s;
  return TB200_OK;
}

}  // extern "C"
