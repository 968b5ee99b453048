// ShmVan: a socket-free transport for jobs whose nodes all live on ONE host (an 8xH100 box running scheduler,
// servers and workers side by side).  It plays the role ps-lite's RDMAVan + IPCTransport play between hosts
// (/root/reference/3rdparty/ps-lite/src/rdma_van.h:26-975, rdma_transport.h:513-712): one-sided writes into
// memory the receiver registered up front, completion by polling, no kernel on the data path - with POSIX
// shared memory standing in for registered NIC memory.
//
//   * every node owns a RECEIVE QUEUE in shm ("/bps_shmvan_<port>"): a bounded multi-producer ring of 8 KB
//     slots.  A sender claims a slot with one CAS, writes header + packed meta (+ small payloads inline) and
//     publishes it with a release store of the slot's sequence number ("write with immediate").
//   * the receiver's van thread polls the ring (spin, then FUTEX_WAIT on a doorbell word in the same region:
//     the completion-queue thread of the verbs van).
//   * payloads that do not fit a slot travel through a per-(sender, receiver) ARENA, a second shm segment the
//     receiver maps on first use (the memory-region cache); space is returned with a consumed counter.  A
//     payload that already lives in a registered window (ShmRegistry: the worker's staging buffers) is passed
//     by name + offset, zero copy, exactly like the colocated-IPC path of the TCP van.
//   * pull responses are copied from the arena straight into the buffer the requester registered with
//     ExpectPullResponse (one copy end to end).
//
// Selected with DMLC_PS_VAN_TYPE=shm.  The node "port" is only an identity here (the scheduler's is
// DMLC_PS_ROOT_PORT); nothing listens on a socket.
#pragma once

#include <atomic>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <unordered_map>

#include "net/van.h"

namespace bps {
namespace net {

class ShmVan : public Van {
 public:
  explicit ShmVan(Postoffice* po) : Van(po) {}
  ~ShmVan() override;

  static constexpr uint32_t kSlotBytes = 8192;
  static constexpr uint32_t kSlots = 512;          // power of two
  static constexpr uint32_t kMaxBlobs = 8;

  struct Slot;
  struct QueueHeader;
  struct ArenaHeader;

 protected:
  int Bind(Node& node, int max_retry) override;
  void Connect(const Node& node) override;
  int SendMsg(Message& msg) override;
  int RecvMsg(Message* msg) override;
  void StopTransport() override;
  bool IsColocated(int) override { return true; }     // this van only exists between processes of one host

 private:
  struct Mapping {           // one mmap'd shm object
    std::string name;
    char* base = nullptr;
    size_t len = 0;
    bool owner = false;
  };
  struct Peer {              // send side of one connection
    Mapping queue;           // the peer's receive queue
    Mapping arena;           // my arena towards that peer (I own it)
    uint64_t arena_head = 0; // bytes ever allocated (only this van writes to the arena)
    std::mutex mu;           // serialises arena allocation + slot publication per peer (keeps per-key order)
    int port = 0;
  };
  static bool MapObject(const std::string& name, size_t len, bool create, Mapping* out);
  static void Unmap(Mapping* m, bool unlink);
  char* ArenaAlloc(Peer* p, size_t n, uint64_t* off);
  Mapping* PeerArena(const std::string& name, size_t len);
  void Ring(QueueHeader* q);

  Mapping my_queue_;
  uint64_t head_ = 0;                                     // consumer cursor (van thread only)
  std::mutex peers_mu_;
  std::unordered_map<int, std::shared_ptr<Peer>> peers_;  // node id -> connection
  std::mutex arenas_mu_;
  std::map<std::string, Mapping> peer_arenas_;            // arenas of peers sending to me (receive side)
  std::atomic<bool> closed_{true};
  size_t arena_bytes_ = 32u << 20;
};

}  // namespace net
}  // namespace bps
