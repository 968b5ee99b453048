// Intra-box control signalling between the GPU processes of one worker.
//
// Parity: BytePSCommSocket (/root/reference/byteps/common/communicator.cc:28-276):
// Unix-domain DATAGRAM sockets `<dir>/socket_<suffix>_<rank>`, 16-byte messages
// {src, signal, key}, the root runs a listen thread that turns *_READY signals
// into ReadyTable increments, and the root can broadcast DO_* commands that the
// other ranks receive in order.  In the reference this protocol gates every
// NCCL call; on the H100 data path readiness is detected by flags in peer
// device memory instead (common.cuh barrier_peers, the ring kernel's per-slot
// generations), and launch order is enforced on the device (ring scheduler
// warp) or by BYTEPS_STRICT_ORDER.  The protocol is used where the data really
// lives in host memory: core/host_reduce.{h,cc} reduces the CPU tensors of the
// local ranks of a box through shared-memory slots with exactly these signals
// (REDUCE_READY -> root sums -> DO_BROADCAST -> BCAST_READY) before the box's
// root talks to the servers.
#pragma once
#include <atomic>
#include <condition_variable>
#include <cstdint>
#include <deque>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

#include "core/ready_table.h"

namespace bps {

enum LocalSignal : int {
  SIG_REDUCE_READY = 0,
  SIG_PCIE_REDUCE_READY,
  SIG_BCAST_READY,
  SIG_PUSH_READY,
  SIG_DO_REDUCE,
  SIG_DO_BROADCAST,
  SIG_DO_GROUP,
  SIG_DO_COPYH2D,
  SIG_COUNT
};

struct LocalMsg {
  int32_t src;
  int32_t signal;
  uint64_t key;
};
static_assert(sizeof(LocalMsg) == 16, "wire format is 16 bytes");

class LocalComm {
 public:
  // members: local ranks taking part; root = highest rank (like the reference)
  // start_listening = false: the root's listener thread is started by start() - after set_tables(), so no early
  // *_READY datagram can arrive before its table is in place
  LocalComm(int local_rank, const std::vector<int>& members, const std::string& dir, const std::string& suffix,
            bool start_listening = true);
  void start();
  ~LocalComm();
  int rank() const { return rank_; }
  int root() const { return root_; }
  bool is_root() const { return rank_ == root_; }
  // non-root -> root
  bool send_to_root(int signal, uint64_t key);
  // root -> all other members
  bool broadcast(int signal, uint64_t key);
  // blocking receive of the next command from the root (non-root); false on timeout/close
  bool recv_from_root(LocalMsg* out, int timeout_ms);
  // root: *_READY signals bump these tables (may be null)
  void set_tables(ReadyTable* reduce, ReadyTable* pcie, ReadyTable* bcast, ReadyTable* push);
  // root: optional hook for every received message
  void set_listener(std::function<void(const LocalMsg&)> fn) { listener_ = std::move(fn); }
  uint64_t received() const { return received_; }

 private:
  std::string path_of(int r) const;
  void listen_loop();
  int rank_, root_;
  std::vector<int> members_;
  std::string dir_, suffix_;
  int fd_ = -1;
  std::thread listener_thread_;
  std::atomic<bool> stop_{false};
  std::mutex tables_mu_;
  ReadyTable* tables_[4] = {nullptr, nullptr, nullptr, nullptr};
  std::function<void(const LocalMsg&)> listener_;
  std::atomic<uint64_t> received_{0};
};

}  // namespace bps
