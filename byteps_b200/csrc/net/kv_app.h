// Key-value push/pull apps on top of Customer/Van.
//
// Parity: KVWorker<char>/KVServer<char> (/root/reference/3rdparty/ps-lite/include/ps/kv_app.h:68-796)
// and SimpleApp (include/ps/simple_app.h:33-196).  BytePS only ever sends ONE
// key per message to ONE server, so the general key-slicing machinery of
// ps-lite collapses to: pick the server from the key range, send, count the
// single response.  Values are byte arrays (SArray<char>); zero-copy on send,
// and pulled data is written straight into the caller's buffer.
#pragma once
#include <atomic>
#include <chrono>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <unordered_map>
#include "core/env.h"
#include <unordered_set>

#include "core/log.h"
#include "net/van.h"

namespace bps {
namespace net {

struct KVMeta {
  int cmd = 0;
  int head = 0;            // init push: number of pushers expected for this key (0 = server default)
  bool push = false;
  bool pull = false;
  int sender = kEmpty;
  int timestamp = kEmpty;
  int customer_id = 0;
  uint64_t key = 0;
  uint64_t val_len = 0;
  // destination shm window announced by a colocated worker's pull request
  std::string shm_name;
  bool want_ref = false;      // pull request: the requester accepts a reference to the server's store
  uint64_t shm_offset = 0;
  uint64_t shm_len = 0;
};

struct KVPairs {
  uint64_t key = 0;
  SArray<char> vals;
  int len = 0;
};

class SimpleApp {
 public:
  using Handle = std::function<void(const Message& msg, SimpleApp* app)>;
  SimpleApp(int app_id, int customer_id, Postoffice* po) : po_(po) {
    obj_.reset(new Customer(app_id, customer_id, [this](const Message& m) { Process(m); }, po));
  }
  virtual ~SimpleApp() { obj_.reset(); }
  int Request(int head, const std::string& body, int recv_id) {
    Message msg;
    msg.meta.head = head;
    msg.meta.body = body;
    int ts = obj_->NewRequest(recv_id);
    msg.meta.timestamp = ts;
    msg.meta.request = true;
    msg.meta.simple_app = true;
    msg.meta.app_id = obj_->app_id();
    msg.meta.customer_id = obj_->customer_id();
    for (int r : po_->GetNodeIDs(recv_id)) {
      msg.meta.recver = r;
      msg.meta.msg_sig = 0;
      po_->van()->Send(msg);
    }
    return ts;
  }
  void Wait(int ts) { obj_->WaitRequest(ts); }

  void Response(const Message& req, const std::string& body = "") {
    Message msg;
    msg.meta.head = req.meta.head;
    msg.meta.body = body;
    msg.meta.timestamp = req.meta.timestamp;
    msg.meta.request = false;
    msg.meta.simple_app = true;
    msg.meta.app_id = obj_->app_id();
    msg.meta.customer_id = req.meta.customer_id;
    msg.meta.recver = req.meta.sender;
    po_->van()->Send(msg);
  }
  void set_request_handle(Handle h) { request_handle_ = std::move(h); }
  void set_response_handle(Handle h) { response_handle_ = std::move(h); }
  Customer* customer() { return obj_.get(); }

 protected:
  SimpleApp(Postoffice* po) : po_(po) {}
  virtual void Process(const Message& msg) {
    if (msg.meta.request) {
      if (request_handle_) request_handle_(msg, this);
    } else if (response_handle_) {
      response_handle_(msg, this);
    }
  }
  Postoffice* po_;
  std::unique_ptr<Customer> obj_;
  Handle request_handle_, response_handle_;
};

constexpr int kPullWantsRef = 0x52454631;   // Meta::head of a pull request: "a reference to your store is fine"

class KVWorker : public SimpleApp {
 public:
  using Callback = std::function<void()>;
  KVWorker(int app_id, int customer_id, Postoffice* po) : SimpleApp(po) {
    obj_.reset(new Customer(app_id, customer_id, [this](const Message& m) { Process(m); }, po));
  }
  ~KVWorker() override { obj_.reset(); }

  // server_rank: which server owns the key (the caller hashes, like BytePSGlobal::EncodeDefaultKey)
  int ZPush(int server_rank, uint64_t key, const SArray<char>& vals, int cmd = 0, Callback cb = nullptr,
            int head = 0) {
    int ts = obj_->NewRequest(Postoffice::ServerRankToID(server_rank));
    AddCallback(ts, std::move(cb));
    Message msg = MakeRequest(ts, server_rank, key, cmd, true, false);
    msg.meta.val_len = vals.size();
    msg.meta.head = head;
    msg.add_data(vals);
    po_->van()->Send(msg);
    return ts;
  }

  // the response payload is copied (or, for colocated IPC, already written) into `dst`
  // `ts_out` (optional) receives the timestamp BEFORE the request leaves: a callback that needs it (pulled_len) may
  // run on the customer thread before this function has returned to the caller.
  // want_ref: a colocated server may answer with a REFERENCE to its own (shared-memory) store instead of copying
  // the value into `dst`; the caller then takes it with take_pull_ref(ts) - e.g. to DMA it to a GPU straight
  // from there.  Only meaningful with BYTEPS_ENABLE_IPC=1.
  int ZPull(int server_rank, uint64_t key, char* dst, size_t len, int cmd = 0, Callback cb = nullptr,
            int* ts_out = nullptr, bool want_ref = false) {
    int ts = obj_->NewRequest(Postoffice::ServerRankToID(server_rank));
    if (ts_out) *ts_out = ts;
    AddCallback(ts, std::move(cb));
    {
      std::lock_guard<std::mutex> g(mu_);
      pull_dst_[ts] = {dst, len};
      if (ts_out) want_len_.insert(ts);     // only callers that ask for the length get an entry (compressed pulls)
    }
    Message msg = MakeRequest(ts, server_rank, key, cmd, false, true);
    msg.meta.val_len = len;
    // shared-memory names only mean something to a server on this host
    const bool colocated = po_->cfg().enable_ipc && po_->van()->IsColocated(Postoffice::ServerRankToID(server_rank));
    if (want_ref && colocated) msg.meta.head = kPullWantsRef;
    // the transport reads the response payload straight into dst (no intermediate buffer, no memcpy)
    po_->van()->ExpectPullResponse(obj_->app_id(), obj_->customer_id(), ts, dst, len);
    if (colocated) {
      std::string name;
      uint64_t off;
      if (ShmRegistry::get().lookup(dst, len, &name, &off)) {
        msg.meta.shm_name = name;
        msg.meta.shm_offset = off;
        msg.meta.shm_len = len;
      }
    }
    po_->van()->Send(msg);
    return ts;
  }

  void Wait(int ts) { obj_->WaitRequest(ts); }
  // (pointer, length, base and length of the whole mapped region) of a pull answered by reference; pointer is null
  // when the value was delivered into the destination buffer as usual.  Take-and-remove.
  struct PullRef {
    char* ptr = nullptr;
    size_t len = 0;
    char* region = nullptr;
    size_t region_len = 0;
  };
  PullRef take_pull_ref(int ts) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = pull_ref_.find(ts);
    if (it == pull_ref_.end()) return PullRef{};
    PullRef r = it->second;
    pull_ref_.erase(it);
    return r;
  }
  // bytes the pull with timestamp `ts` delivered.  Take-and-remove: one entry per pull response would otherwise
  // stay in the map for the life of the job (one per partition per step).
  size_t pulled_len(int ts) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = pulled_len_.find(ts);
    if (it == pulled_len_.end()) return 0;
    const size_t n = it->second;
    pulled_len_.erase(it);
    return n;
  }

 private:
  Message MakeRequest(int ts, int server_rank, uint64_t key, int cmd, bool push, bool pull) {
    Message msg;
    msg.meta.app_id = obj_->app_id();
    msg.meta.customer_id = obj_->customer_id();
    msg.meta.request = true;
    msg.meta.push = push;
    msg.meta.pull = pull;
    msg.meta.cmd = cmd;
    msg.meta.timestamp = ts;
    msg.meta.key = key;
    msg.meta.recver = Postoffice::ServerRankToID(server_rank);
    return msg;
  }
  void AddCallback(int ts, Callback cb) {
    if (!cb) return;
    std::lock_guard<std::mutex> g(mu_);
    callbacks_[ts] = std::move(cb);
  }
  void Process(const Message& msg) override {
    if (msg.meta.simple_app) {
      SimpleApp::Process(msg);
      return;
    }
    int ts = msg.meta.timestamp;
    if (msg.meta.pull) {
      po_->van()->CancelRecvBuffer(obj_->app_id(), obj_->customer_id(), ts);   // unused slot (IPC / size mismatch)
      std::pair<char*, size_t> dst{nullptr, 0};
      {
        std::lock_guard<std::mutex> g(mu_);
        auto it = pull_dst_.find(ts);
        if (it != pull_dst_.end()) {
          dst = it->second;
          pull_dst_.erase(it);
        }
      }
      size_t got = 0;
      if (msg.data.empty() && !msg.meta.shm_name.empty()) {
        // answered by reference: the value sits in the server's shared-memory store
        const size_t rlen = (size_t)(msg.meta.shm_offset + msg.meta.shm_len);
        char* base = (char*)ShmRegistry::get().open(msg.meta.shm_name, rlen);
        if (base) {
          got = (size_t)msg.meta.shm_len;
          std::lock_guard<std::mutex> g(mu_);
          pull_ref_[ts] = PullRef{base + msg.meta.shm_offset, got, base, ShmRegistry::get().region_len(msg.meta.shm_name)};
        } else {
          BPS_LOG(ERROR) << "cannot map the server store " << msg.meta.shm_name;
        }
      } else if (!msg.data.empty() && dst.first) {
        got = std::min(dst.second, msg.data[0].size());
        if (msg.data[0].data() != dst.first) memcpy(dst.first, msg.data[0].data(), got);
      } else if (msg.data.empty()) {
        got = (size_t)msg.meta.val_len;   // colocated IPC: the server wrote into our shm window
      }
      std::lock_guard<std::mutex> g(mu_);
      if (want_len_.erase(ts)) pulled_len_[ts] = got;
    }
    Callback cb;
    {
      std::lock_guard<std::mutex> g(mu_);
      auto it = callbacks_.find(ts);
      if (it != callbacks_.end()) {
        cb = std::move(it->second);
        callbacks_.erase(it);
      }
    }
    if (cb) cb();
  }
  std::mutex mu_;
  std::unordered_map<int, Callback> callbacks_;
  std::unordered_map<int, std::pair<char*, size_t>> pull_dst_;
  std::unordered_map<int, size_t> pulled_len_;
  std::unordered_set<int> want_len_;
  std::unordered_map<int, PullRef> pull_ref_;
};

// BYTEPS_SERVER_PROFILE=1: how the pull responses left this server (printed when the server stops)
struct IpcStats {
  std::atomic<uint64_t> shm_responses{0}, shm_bytes{0}, shm_ns{0}, payload_responses{0}, payload_bytes{0};
  std::atomic<uint64_t> ref_responses{0}, ref_bytes{0};
  static IpcStats& get() {
    static IpcStats s;
    return s;
  }
};

// Parallel copy into a colocated worker's window: chunks of 256 KB over an OpenMP team.
inline void ipc_copy(char* dst, const char* src, size_t n) {
  static const int threads = (int)std::max<long long>(
      1, env_int("BYTEPS_IPC_COPY_NUM_THREADS", std::thread::hardware_concurrency() >= 64 ? 8 : 4));
  const size_t chunk = 256 << 10;
  if (threads <= 1 || n < 2 * chunk) {
    memcpy(dst, src, n);
    return;
  }
  const long nchunks = (long)((n + chunk - 1) / chunk);
#pragma omp parallel for num_threads(threads) schedule(static)
  for (long c = 0; c < nchunks; ++c) {
    const size_t off = (size_t)c * chunk;
    memcpy(dst + off, src + off, off + chunk <= n ? chunk : n - off);
  }
}

class KVServer : public SimpleApp {
 public:
  using ReqHandle = std::function<void(const KVMeta& req_meta, const KVPairs& req_data, KVServer* server)>;
  KVServer(int app_id, Postoffice* po) : SimpleApp(po) {
    obj_.reset(new Customer(app_id, app_id, [this](const Message& m) { Process(m); }, po));
  }
  ~KVServer() override { obj_.reset(); }
  void set_kv_request_handle(ReqHandle h) { handle_ = std::move(h); }

  void Response(const KVMeta& req, const KVPairs& res = KVPairs()) {
    Message msg;
    msg.meta.app_id = obj_->app_id();
    msg.meta.customer_id = req.customer_id;
    msg.meta.request = false;
    msg.meta.push = req.push;
    msg.meta.pull = req.pull;
    msg.meta.cmd = req.cmd;
    msg.meta.timestamp = req.timestamp;
    msg.meta.recver = req.sender;
    msg.meta.key = res.key ? res.key : req.key;
    if (!res.vals.empty()) {
      msg.meta.val_len = res.vals.size();
      bool via_shm = false;
      if (req.want_ref && po_->cfg().enable_ipc) {
        // the requester can read my store where it is (it lives in shared memory): no copy at all
        std::string name;
        uint64_t off;
        if (ShmRegistry::get().lookup(res.vals.data(), res.vals.size(), &name, &off)) {
          msg.meta.shm_name = name;
          msg.meta.shm_offset = off;
          msg.meta.shm_len = res.vals.size();
          via_shm = true;
          IpcStats::get().ref_responses++;
          IpcStats::get().ref_bytes += res.vals.size();
        }
      }
      if (!via_shm && !req.shm_name.empty() && po_->cfg().enable_ipc) {
        // colocated worker announced its destination window: write there, send only the meta
        void* base = ShmRegistry::get().open(req.shm_name, (size_t)(req.shm_offset + req.shm_len));
        if (base && res.vals.size() <= req.shm_len) {
          // the reference hands this copy to BYTEPS_IPC_COPY_NUM_THREADS async copy threads
          // (rdma_transport.h:577-644); one memcpy of a 4 MB partition per response was THE bottleneck of the
          // colocated CPU-server path
          const auto t0 = std::chrono::steady_clock::now();
          ipc_copy((char*)base + req.shm_offset, res.vals.data(), res.vals.size());
          via_shm = true;
          auto& st = IpcStats::get();
          st.shm_responses++;
          st.shm_bytes += res.vals.size();
          st.shm_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                           std::chrono::steady_clock::now() - t0).count();
        }
      }
      if (!via_shm) {
        msg.add_data(res.vals);
        IpcStats::get().payload_responses++;
        IpcStats::get().payload_bytes += res.vals.size();
      }
    }
    po_->van()->Send(msg);
  }

 private:
  void Process(const Message& msg) override {
    if (msg.meta.simple_app) {
      SimpleApp::Process(msg);
      return;
    }
    KVMeta meta;
    meta.cmd = msg.meta.cmd;
    meta.head = msg.meta.head > 0 ? msg.meta.head : 0;
    meta.push = msg.meta.push;
    meta.pull = msg.meta.pull;
    meta.sender = msg.meta.sender;
    meta.timestamp = msg.meta.timestamp;
    meta.customer_id = msg.meta.customer_id;
    meta.key = msg.meta.key;
    meta.val_len = msg.meta.val_len;
    meta.shm_name = msg.meta.shm_name;
    meta.want_ref = msg.meta.pull && msg.meta.head == kPullWantsRef;
    meta.shm_offset = msg.meta.shm_offset;
    meta.shm_len = msg.meta.shm_len;
    KVPairs data;
    data.key = msg.meta.key;
    if (!msg.data.empty()) {
      data.vals = msg.data[0];
      data.len = (int)msg.data[0].size();
    }
    BPS_CHECK(handle_) << "KVServer: no request handle set";
    handle_(meta, data, this);
  }
  ReqHandle handle_;
};

}  // namespace net
}  // namespace bps
