#include "server/server.h"

#include <map>

#include "core/numa.h"
#include "core/trace.h"

#include <unistd.h>

#include <chrono>
#include <thread>

#include <algorithm>
#include <cstdlib>
#include <cstring>

#include "core/env.h"
#include "core/log.h"
#include "cpu/half.h"

namespace bps {
namespace server {

// ------------------------------------------------------------------ queue
bool PriorityQueue::Before(const EngineMessage& a, const EngineMessage& b) {
  // true when a should be served before b.  Keys that have seen fewer pushes in
  // this round go first (reference queue.h:88-94); all messages of one key share
  // the same count, so per-key arrival order is always preserved.
  if (schedule_) {
    uint64_t pa = push_cnt_[a.key], pb = push_cnt_[b.key];
    if (pa != pb) return pa < pb;
  }
  return a.id < b.id;
}

void PriorityQueue::Push(EngineMessage m) {
  {
    std::lock_guard<std::mutex> g(mu_);
    if (schedule_ && (m.op == COPY_FIRST || m.op == SUM_RECV)) ++push_cnt_[m.key];
    heap_.push_back(std::move(m));
  }
  cv_.notify_one();
}

void PriorityQueue::WaitAndPop(EngineMessage* m) {
  std::unique_lock<std::mutex> lk(mu_);
  cv_.wait(lk, [this] { return !heap_.empty(); });
  // priorities move while messages wait, so select at pop time (queues are short)
  size_t best = 0;
  for (size_t i = 1; i < heap_.size(); ++i)
    if (Before(heap_[i], heap_[best])) best = i;
  *m = std::move(heap_[best]);
  heap_.erase(heap_.begin() + best);
}

void PriorityQueue::ClearCounter(uint64_t key) {
  if (!schedule_) return;
  std::lock_guard<std::mutex> g(mu_);
  push_cnt_[key] = 0;
}

size_t PriorityQueue::size() {
  std::lock_guard<std::mutex> g(mu_);
  return heap_.size();
}

// ------------------------------------------------------------------ config
ServerConfig ServerConfig::from_env() {
  ServerConfig c;
  // the reference's default is 4 engine threads (server.cc:412-456); hosts that carry 8 GPUs have the cores to
  // merge more keys at once (128 hardware threads: 8 engine threads x 4 summation threads per server)
  const long long cores = (long long)std::thread::hardware_concurrency();
  c.engine_threads = (int)env_int("BYTEPS_SERVER_ENGINE_THREAD", std::max<long long>(4, std::min<long long>(16, cores / 16)));
  c.enable_schedule = env_bool("BYTEPS_SERVER_ENABLE_SCHEDULE", false);
  c.engine_blocking = env_bool("BYTEPS_SERVER_ENGINE_BLOCKING", false);
  c.sync_mode = !env_bool("BYTEPS_ENABLE_ASYNC", false);
  c.pushers_per_key = (int)env_int("BYTEPS_SERVER_PUSHERS_PER_KEY", 0);
  c.log_keys = env_bool("PS_KEY_LOG", false);
  if (env_bool("BYTEPS_SERVER_DEBUG", false)) c.debug_key = env_int("BYTEPS_SERVER_DEBUG_KEY", 0);
  return c;
}

static char* page_alloc(size_t n) {
  void* p = nullptr;
  size_t sz = round_up(n ? n : 1, 4096);
  if (posix_memalign(&p, 4096, sz) != 0) return nullptr;
  memset(p, 0, sz);
  return (char*)p;
}

// ------------------------------------------------------------------ server
SumServer::SumServer(net::Postoffice* po, const ServerConfig& cfg, int app_id)
    : po_(po), cfg_(cfg),
      // threads of ONE summation: 1 on small hosts (the engine threads already use the cores), 4 from 64 hardware
      // threads up (one thread merging a 4 MB partition dominated the colocated path)
      reducer_((int)env_int("BYTEPS_SERVER_OMP_THREADS", std::thread::hardware_concurrency() >= 64 ? 4 : 1)) {
  pushers_ = cfg.pushers_per_key > 0 ? cfg.pushers_per_key : po->num_workers();
  inline_bytes_ = (size_t)std::max<long long>(0, env_int("BYTEPS_SERVER_INLINE_BYTES", 16384));
  profile_ = env_bool("BYTEPS_SERVER_PROFILE", false);
  if (po->cfg().enable_ipc && env_bool("BYTEPS_SHM_REAP_STALE", false)) {
    // a server / worker that was killed leaves its shared-memory objects behind; they are named by pid.  Opt-in:
    // "pid not found" only proves death when every process that shares this /dev/shm also shares the pid namespace
    const int reaped = net::ShmRegistry::reap_stale();
    if (reaped) BPS_LOG(INFO) << "removed " << reaped << " shared-memory objects of dead byteps processes";
  }
  int nt = std::max(1, cfg.engine_threads);
  acc_load_.assign(nt, 0);
  for (int i = 0; i < nt; ++i) queues_.emplace_back(new PriorityQueue(cfg.enable_schedule));
  // BYTEPS_NUMA_AWARE=1 on a multi-socket host: engine thread i lives on node i % nodes, a key's summation runs on
  // a thread of the node its store was placed on (ThreadOf)
  const int nodes = numa_aware() ? numa_num_nodes() : 1;
  thread_node_.assign(nt, -1);
  if (nodes > 1 && nt >= nodes)
    for (int i = 0; i < nt; ++i) thread_node_[i] = i % nodes;
  for (int i = 0; i < nt; ++i)
    threads_.emplace_back([this, i] {
      int node;
      {
        std::lock_guard<std::mutex> g(load_mu_);
        node = thread_node_[i];
      }
      if (node >= 0 && !numa_pin_thread_to_node(node)) {
        std::lock_guard<std::mutex> g(load_mu_);      // ThreadOf reads the table under the same lock
        thread_node_[i] = -1;
      }
      EngineLoop(i);
    });
  kv_.reset(new net::KVServer(app_id, po));
  kv_->set_kv_request_handle(
      [this](const net::KVMeta& m, const net::KVPairs& d, net::KVServer* s) { Handle(m, d, s); });
  BPS_LOG(INFO) << "byteps_b200 server: " << nt << " engine threads, " << pushers_ << " pushers per key, "
                << (cfg.sync_mode ? "sync" : "async") << " mode";
}

SumServer::~SumServer() { Stop(); }

void SumServer::Stop() {
  if (stopped_) return;
  stopped_ = true;
  if (env_bool("BYTEPS_SERVER_PROFILE", false)) {
    auto& ipc = net::IpcStats::get();
    BPS_LOG_AT(L_WARNING) << "server profile: pushes " << n_push_ << " (by reference " << n_push_ref_ << ", "
                          << push_ref_bytes_ / 1e6 << " MB; as payload " << push_payload_bytes_ / 1e6 << " MB), merge "
                          << merge_ns_ / 1e6 << " ms over " << merge_bytes_ / 1e6 << " MB on "
                          << threads_.size() << " engine threads x " << reducer_.num_threads() << " summation threads; pull responses "
                          << "into shared windows " << ipc.shm_responses << " (" << ipc.shm_bytes / 1e6 << " MB, "
                          << ipc.shm_ns / 1e6 << " ms of copying), by reference " << ipc.ref_responses << " ("
                          << ipc.ref_bytes / 1e6 << " MB, no copy), as payload " << ipc.payload_responses << " ("
                          << ipc.payload_bytes / 1e6 << " MB); rounds " << rounds_ << ": pusher skew avg "
                          << (rounds_ ? skew_us_ / rounds_ : 0) << " us (max " << skew_max_us_
                          << "), last push -> pulls answered avg " << (rounds_ ? serve_us_ / rounds_ : 0) << " us (max "
                          << serve_max_us_ << "), pulls already parked at that point " << parked_at_publish_
                          << "; NUMA: stores bound " << numa_bound_ << ", refused " << numa_refused_;
  }
  kv_.reset();   // stop receiving first
  for (auto& q : queues_) {
    EngineMessage m;
    m.id = msg_id_++;
    m.op = TERMINATE;
    q->Push(std::move(m));
  }
  for (auto& t : threads_)
    if (t.joinable()) t.join();
  std::lock_guard<std::mutex> g(map_mu_);
  for (auto& kv : states_) {
    if (!kv.second->shm_names[0].empty()) {
      for (int b = 0; b < 2; ++b) net::ShmRegistry::get().release(kv.second->shm_names[b]);
      continue;
    }
    free(kv.second->store2[0]);
    if (kv.second->store2[1] != kv.second->store2[0]) free(kv.second->store2[1]);
  }
  states_.clear();
}

size_t SumServer::num_keys() {
  std::lock_guard<std::mutex> g(map_mu_);
  return states_.size();
}

SumServer::KeyState* SumServer::GetState(uint64_t key) {
  std::lock_guard<std::mutex> g(map_mu_);
  auto& p = states_[key];
  if (!p) p.reset(new KeyState());
  return p.get();
}

// keys are pinned to the least-loaded engine thread the first time their size is known
int SumServer::ThreadOf(KeyState* st, size_t len) {
  if (st->tid >= 0) return st->tid;
  std::lock_guard<std::mutex> g(load_mu_);
  int best = -1;
  if (st->numa_node >= 0)      // least-loaded engine thread on the node of the key's store, if there is one
    for (size_t i = 0; i < acc_load_.size(); ++i)
      if (thread_node_[i] == st->numa_node && (best < 0 || acc_load_[i] < acc_load_[best])) best = (int)i;
  if (best < 0) {
    best = 0;
    for (size_t i = 1; i < acc_load_.size(); ++i)
      if (acc_load_[i] < acc_load_[best]) best = (int)i;
  }
  acc_load_[best] += len;
  st->tid = best;
  return best;
}

void SumServer::SendPush(const net::KVMeta& req) { kv_->Response(req); }

void SumServer::SendPull(KeyState* st, uint64_t key, const net::KVMeta& req) {
  net::KVPairs res;
  res.key = key;
  const char* src = st->merged ? st->merged : st->store2[st->rd];
  size_t len = st->merged ? st->merged_len : st->len;
  // zero-copy view over the store (response caches of the reference collapse to this)
  res.vals = net::SArray<char>(const_cast<char*>(src), len, false);
  res.len = (int)len;
  kv_->Response(req, res);
  ++n_pull_;
}

static double first_value(const void* p, int dtype) {
  switch (dtype) {
    case F32: return *(const float*)p;
    case F64: return *(const double*)p;
    case F16: return f16_to_f32(*(const uint16_t*)p);
    case BF16: return bf16_to_f32(*(const uint16_t*)p);
    case I32: return *(const int32_t*)p;
    case I64: return (double)*(const int64_t*)p;
    case U8: return *(const uint8_t*)p;
    case I8: return *(const int8_t*)p;
  }
  return 0;
}

void SumServer::Debug(const char* stage, uint64_t key, const void* dst, const void* src, size_t len, int dtype) {
  if (cfg_.debug_key < 0 || (uint64_t)cfg_.debug_key != key) return;
  BPS_LOG_AT(L_WARNING) << "server stage: " << stage << "\tkey: " << key << "\tdst: " << (dst ? first_value(dst, dtype) : 0)
                        << "\tsrc: " << (src ? first_value(src, dtype) : 0) << "\tlen: " << len;
}

void SumServer::Handle(const net::KVMeta& req, const net::KVPairs& data, net::KVServer*) {
  int rtype, dtype;
  command_decode(req.cmd, &rtype, &dtype);
  const uint64_t key = req.key;
  KeyState* st = GetState(key);
  if (cfg_.log_keys) {
    BPS_LOG_AT(L_WARNING) << (req.push ? "push" : "pull") << " key=" << key << "\t sender=" << req.sender
                          << "\t size=" << data.vals.size();
  }
  std::unique_lock<std::mutex> lk(st->mu);
  if (st->pushers == 0) st->pushers = (req.push && numa_head_pushers(req.head) > 0) ? numa_head_pushers(req.head) : pushers_;
  const int pushers = st->pushers;

  // ---- compressor registration (payload = serialized kwargs)
  if (rtype == kCompressedPushPull) {
    if (!st->compressor) {
      BPS_CHECK(st->inited) << "compressed push for key " << key << " before its init push";
      std::string content(data.vals.data(), data.vals.size());
      Kwargs kw = kwargs_deserialize(content);
      st->compressor = CompressorRegistry::create(kw, st->len, st->dtype, /*server_side=*/true);
      BPS_CHECK(st->compressor != nullptr) << "kwargs name no compressor";
      st->comp_out.resize(st->compressor->max_compressed_bytes() + 64);
      st->decomp.resize(st->len);
      if (cfg_.log_keys) BPS_LOG_AT(L_WARNING) << "register compressor for key=" << key;
    }
    st->comp_reqs.push_back(req);
    if ((int)st->comp_reqs.size() < pushers) return;
    for (auto& r : st->comp_reqs) SendPush(r);
    st->comp_reqs.clear();
    return;
  }

  if (req.push) {
    ++n_push_;
    const size_t len = data.vals.size();
    const char* recved = data.vals.data();
    if (!req.shm_name.empty()) {
      ++n_push_ref_;
      push_ref_bytes_ += len;
    } else {
      push_payload_bytes_ += len;
    }
    if (!st->inited) {
      // ---- init push: global barrier + store allocation
      st->init_reqs.push_back(req);
      if ((int)st->init_reqs.size() < pushers) return;
      st->store_cap = align_payload(len, dtype);
      if (numa_aware()) {
        // the node most pushers asked for (their GPUs' node); ties go to the lower node
        std::map<int, int> votes;
        for (auto& r : st->init_reqs)
          if (numa_head_node(r.head) >= 0) ++votes[numa_head_node(r.head)];
        int most = 0;
        for (auto& v : votes)
          if (v.second > most) {
            most = v.second;
            st->numa_node = v.first;
          }
      }
      if (po_->cfg().enable_ipc && cfg_.sync_mode) {
        // colocated workers may read the merged value where it is (pull by reference, kv_app.h): the store lives in
        // POSIX shared memory, one object per buffer
        for (int b = 0; b < 2; ++b) {
          st->shm_names[b] = "BytePS_SrvStore_" + std::to_string((long)getpid()) + "_" + std::to_string(key) + "_" +
                             std::to_string(b);
          st->store2[b] = (char*)net::ShmRegistry::get().create(st->shm_names[b], round_up(st->store_cap, 4096));
          if (st->store2[b]) {
            // bind BEFORE the first touch: the memset below then faults the pages in on the right node
            if (st->numa_node >= 0) ++(numa_bind_memory(st->store2[b], round_up(st->store_cap, 4096), st->numa_node) ? numa_bound_ : numa_refused_);
            memset(st->store2[b], 0, st->store_cap);
          }
        }
      } else {
        st->store2[0] = page_alloc(st->store_cap);
        st->store2[1] = cfg_.sync_mode ? page_alloc(st->store_cap) : st->store2[0];
        if (st->numa_node >= 0)     // already touched by page_alloc: mbind migrates the pages
          for (int b = 0; b < (cfg_.sync_mode ? 2 : 1); ++b)
            if (st->store2[b]) ++(numa_bind_memory(st->store2[b], round_up(st->store_cap, 4096), st->numa_node) ? numa_bound_ : numa_refused_);
      }
      BPS_CHECK(st->store2[0] != nullptr && st->store2[1] != nullptr);
      if (!cfg_.sync_mode) st->wr = 0;
      st->len = len;
      st->dtype = dtype;
      st->inited = true;
      reducer_.copy(st->store2[st->rd], recved, len);
      for (auto& r : st->init_reqs) SendPush(r);
      st->init_reqs.clear();
      return;
    }
    // a key's size is fixed by its init push: a shorter payload would be an out-of-bounds read in the reducer,
    // a longer one silently truncated (workers re-key a tensor whose size changes, comm/ps.py)
    if (!st->compressor)
      BPS_CHECK_EQ(len, st->len) << "push of " << len << " bytes for key " << key << " initialised with " << st->len
                                 << " bytes (sender " << req.sender << ")";
    const int tid = ThreadOf(st, st->len);
    if (!cfg_.sync_mode) {
      // ---- async: accumulate straight into the store, never block pulls
      if (st->compressor) st->compressor->decompress_add(recved, len, st->store2[0]);
      else reducer_.sum(st->store2[0], recved, st->len, st->dtype);
      SendPush(req);
      return;
    }
    const bool first = st->round_reqs.empty();
    if (profile_) {
      const int64_t now = now_us();
      if (first) st->t_first_push = now;
      st->t_last_push = now;
    }
    // small keys are merged right here: summing a few KB costs less than the two thread hand-offs through an engine
    // queue (a key's size never changes, so it always takes the same path)
    const bool inline_merge = cfg_.engine_blocking || st->len <= inline_bytes_;
    if (inline_merge) {
      if (st->compressor) {
        if (first) st->compressor->decompress(recved, len, st->store2[st->wr]);
        else st->compressor->decompress_add(recved, len, st->store2[st->wr]);
      } else if (first) {
        reducer_.copy(st->store2[st->wr], recved, st->len);
      } else {
        reducer_.sum(st->store2[st->wr], recved, st->len, st->dtype);
      }
    } else {
      EngineMessage m;
      m.id = msg_id_++;
      m.op = first ? COPY_FIRST : SUM_RECV;
      m.key = key;
      m.dtype = st->dtype;
      m.src = data.vals;
      m.len = len;
      m.req = req;
      queues_[tid]->Push(std::move(m));
    }
    st->round_reqs.push_back(req);
    SendPush(req);
    if ((int)st->round_reqs.size() == pushers) {
      st->round_reqs.clear();
      if (inline_merge) {
        Publish(st, key);
      } else {
        EngineMessage m;
        m.id = msg_id_++;
        m.op = ALL_RECV;
        m.key = key;
        m.dtype = st->dtype;
        queues_[tid]->Push(std::move(m));
        queues_[tid]->ClearCounter(key);
      }
    }
    return;
  }

  // ---- pull
  BPS_CHECK(st->inited) << "pull for key " << key << " before it was initialised";
  if (!cfg_.sync_mode) {
    st->merged = nullptr;
    SendPull(st, key, req);
    return;
  }
  if (st->push_finished && !st->seen_sender.count(req.sender)) {
    SendPull(st, key, req);
    st->seen_sender.insert(req.sender);
    if (++st->pull_cnt == (size_t)pushers) {
      st->push_finished = false;
      st->pull_cnt = 0;
      st->seen_sender.clear();
    }
  } else {
    st->parked_pulls.push_back(req);   // answered when ALL_RECV runs
  }
}

void SumServer::EngineLoop(int tid) {
  auto& q = *queues_[tid];
  while (true) {
    EngineMessage m;
    q.WaitAndPop(&m);
    if (m.op == TERMINATE) break;
    KeyState* st = GetState(m.key);
    if (m.op == COPY_FIRST || m.op == SUM_RECV) {
      const char* src = m.src.data();
      // the store is only touched by this engine thread between rounds; the
      // handler thread never writes it in sync mode, so no lock is held here
      if (st->compressor) {
        // straight into the store: the first push of a round is decompressed in place of a copy, later ones are
        // accumulated (sparse payloads touch k entries instead of three passes over the partition)
        BPS_CHECK_LE(m.len, st->store_cap + 64);
        if (m.op == COPY_FIRST) st->compressor->decompress(src, m.len, st->store2[st->wr]);
        else st->compressor->decompress_add(src, m.len, st->store2[st->wr]);
        continue;
      }
      if (m.op == COPY_FIRST) {
        if (st->pushers >= 2 && !st->compressor && cfg_.debug_key < 0 && m.len == st->len) {
          // zero-copy: the payload (receive buffer or the worker's shm window) stays alive in `held_first`
          st->held_first = m.src;
          st->holding = true;
        } else {
          Debug("ENGINE_COPY_MERGED_TO_STORE_BEFORE", m.key, st->store2[st->wr], src, st->len, st->dtype);
          reducer_.copy(st->store2[st->wr], src, st->len);
          Debug("ENGINE_COPY_MERGED_TO_STORE_AFTER", m.key, st->store2[st->wr], src, st->len, st->dtype);
        }
      } else if (st->holding) {
        const auto t0 = std::chrono::steady_clock::now();
        BPS_CHECK_GE(reducer_.sum(st->store2[st->wr], st->held_first.data(), src, st->len, st->dtype), 0);
        merge_ns_ += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                         std::chrono::steady_clock::now() - t0).count();
        merge_bytes_ += st->len;
        st->held_first = net::SArray<char>();
        st->holding = false;
      } else {
        Debug("ENGINE_SUM_RECV_BEFORE", m.key, st->store2[st->wr], src, st->len, st->dtype);
        BPS_CHECK_GE(reducer_.sum(st->store2[st->wr], src, st->len, st->dtype), 0);
        Debug("ENGINE_SUM_RECV_AFTER", m.key, st->store2[st->wr], src, st->len, st->dtype);
      }
    } else if (m.op == ALL_RECV) {
      if (st->holding) {     // not reached with >= 2 pushers; keeps the store right if a round ends early
        reducer_.copy(st->store2[st->wr], st->held_first.data(), st->len);
        st->held_first = net::SArray<char>();
        st->holding = false;
      }
      std::unique_lock<std::mutex> lk(st->mu);
      Publish(st, m.key);
    }
  }
}

// The round's merged buffer becomes readable: flip buffers, (re)compress, flush parked pulls.
void SumServer::Publish(KeyState* st, uint64_t key) {
  st->rd = st->wr;
  if (cfg_.sync_mode) st->wr ^= 1;
  if (st->compressor) {
    st->merged_len = st->compressor->compress(st->store2[st->rd], st->comp_out.data());
    st->merged = st->comp_out.data();
  } else {
    st->merged = st->store2[st->rd];
    st->merged_len = st->len;
  }
  st->push_finished = true;
  std::vector<net::KVMeta> parked;
  parked.swap(st->parked_pulls);
  const size_t n_parked = parked.size();
  for (auto& p : parked) {
    if (st->push_finished && !st->seen_sender.count(p.sender)) {
      SendPull(st, key, p);
      st->seen_sender.insert(p.sender);
      if (++st->pull_cnt == (size_t)st->pushers) {
        st->push_finished = false;
        st->pull_cnt = 0;
        st->seen_sender.clear();
      }
    } else {
      st->parked_pulls.push_back(p);
    }
  }
  if (profile_ && st->t_first_push && st->len > inline_bytes_) {
    // where a round's latency goes: waiting for the slowest pusher vs queueing + summation + answering here
    const int64_t now = now_us();
    const uint64_t skew = (uint64_t)(st->t_last_push - st->t_first_push), serve = (uint64_t)(now - st->t_last_push);
    ++rounds_;
    skew_us_ += skew;
    serve_us_ += serve;
    parked_at_publish_ += n_parked;
    uint64_t m = serve_max_us_.load();
    while (serve > m && !serve_max_us_.compare_exchange_weak(m, serve)) {}
    m = skew_max_us_.load();
    while (skew > m && !skew_max_us_.compare_exchange_weak(m, skew)) {}
  }
}

}  // namespace server
}  // namespace bps
