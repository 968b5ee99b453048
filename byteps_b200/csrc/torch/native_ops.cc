// Native torch adapter: push_pull on at::Tensor without Python on the per-partition path.
//
// Parity: /root/reference/byteps/torch/ops.cc:54-135 (DoPushPull / StartTask / PollHandle /
// WaitAndClear), adapter.cc:23-79 (TorchTensor), ready_event.cc:43-115 (pooled CUDA events),
// handle_manager.cc:22-52 - without TH/THC.  What differs underneath:
//
//   * declare -> partition (Registry) -> priority/credit queue (ScheduledQueue) -> ONE fused
//     pack + exchange + unpack kernel per batch of partitions (kernels/pushpull.cu) instead of
//     12 stage queues and NCCL groups;
//   * readiness is cudaStreamWaitEvent on the communication stream (no host thread polls
//     cudaEventQuery), completion is an event the caller's stream waits on in synchronize();
//   * a flush window batches what was enqueued since the last launch: small tensors (ResNet-50
//     has 161, most of them a few KB) share one launch, in (priority desc, key asc) order
//     inside the byte-credit window - BytePSScheduledQueue's contract.
#include <ATen/cuda/CUDAContext.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <cuda_runtime_api.h>
#include <torch/extension.h>

#include <array>
#include <cstring>
#include <deque>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "core/handle_manager.h"
#include "core/registry.h"
#include "core/scheduler.h"
#include "core/types.h"
#include "kernels/pushpull.cuh"

namespace py = pybind11;
using namespace bps;

namespace {

void cuda_check(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

int wire_of(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return WIRE_F32;
    case at::kBFloat16: return WIRE_BF16;
    case at::kHalf: return WIRE_F16;
    default: return -1;
  }
}
int core_dtype_of(at::ScalarType t) {
  switch (t) {
    case at::kFloat: return F32;
    case at::kBFloat16: return BF16;
    case at::kHalf: return F16;
    default: return -1;
  }
}
size_t wire_bytes(int w) { return w == WIRE_F32 ? 4 : 2; }

struct Part {                 // one partition waiting for a launch
  uint64_t key;
  const char* src;
  char* dst;
  size_t numel;
  size_t nbytes;
  int handle;
  int dtype;                  // WireDType of the user tensor
  bool average;
};

struct HandleState {
  at::Tensor input, output;   // keep the storage alive until the exchange has run
  uint32_t pending = 0;       // partitions not launched yet
  cudaEvent_t done = nullptr; // recorded on the communication stream after the last launch
};

class NativeSymmOps {
 public:
  NativeSymmOps(const std::vector<uintptr_t>& data, const std::vector<uintptr_t>& sig, uintptr_t mc, uintptr_t epoch,
                int rank, int world, size_t arena_bytes, uintptr_t comm_stream, int device, size_t partition_bytes,
                size_t group_bytes, size_t one_shot_bytes, size_t flush_bytes, uint64_t credit_bytes, int blocks,
                int threads, bool nvls, int wire_override)
      : world_(world), arena_bytes_(arena_bytes), comm_((cudaStream_t)comm_stream), device_(device),
        partition_bytes_(partition_bytes), group_bytes_(group_bytes), one_shot_bytes_(one_shot_bytes),
        flush_bytes_(flush_bytes), blocks_(blocks), threads_(threads), nvls_(nvls), wire_override_(wire_override),
        queue_(REDUCE, true, credit_bytes) {
    if ((int)data.size() != world || (int)sig.size() != world || world < 1 || world > kMaxRanks)
      throw std::runtime_error("NativeSymmOps: need `world` data and signal pointers");
    memset(&pv_, 0, sizeof(pv_));
    for (int r = 0; r < world; ++r) {
      pv_.data[r] = (char*)data[r];
      pv_.sig[r] = (uint32_t*)sig[r];
    }
    pv_.mc_data = (char*)mc;
    pv_.epoch = (uint32_t*)epoch;
    pv_.rank = rank;
    pv_.world = world;
    c10::cuda::CUDAGuard guard(device_);
    for (auto& s : seg_ring_) {
      cuda_check(cudaMallocHost((void**)&s.host, kSegRows * sizeof(SegDesc)), "cudaMallocHost");
      cuda_check(cudaMalloc((void**)&s.dev, kSegRows * sizeof(SegDesc)), "cudaMalloc");
      cuda_check(cudaEventCreateWithFlags(&s.copied, cudaEventDisableTiming), "cudaEventCreate");
      s.used = false;
    }
    cuda_check(cudaEventCreateWithFlags(&ready_, cudaEventDisableTiming), "cudaEventCreate");
  }

  ~NativeSymmOps() {
    cudaStreamSynchronize(comm_);
    for (auto& s : seg_ring_) {
      if (s.host) cudaFreeHost(s.host);
      if (s.dev) cudaFree(s.dev);
      if (s.copied) cudaEventDestroy(s.copied);
    }
    if (ready_) cudaEventDestroy(ready_);
    for (auto e : event_pool_) cudaEventDestroy(e);
  }

  uint32_t declare(const std::string& name) { return registry_.declare(name); }

  // Returns the handle.  Nothing is launched before a flush point: flush_bytes of pending
  // partitions, an explicit flush(), or poll()/synchronize() of a pending handle.
  int push_pull_async(const at::Tensor& t, const at::Tensor& out, bool average, const std::string& name, int priority,
                      int version) {
    (void)version;
    if (!t.is_cuda() || !out.is_cuda() || !t.is_contiguous() || !out.is_contiguous())
      throw std::invalid_argument("native push_pull needs contiguous CUDA tensors");
    const int w = wire_of(t.scalar_type());
    if (w < 0 || out.scalar_type() != t.scalar_type() || out.numel() != t.numel())
      throw std::invalid_argument("native push_pull supports float32 / bfloat16 / float16 of equal shape");
    std::lock_guard<std::mutex> g(mu_);
    const size_t es = t.element_size();
    const size_t nbytes = (size_t)t.numel() * es;
    Plan& plan = plans_[name];
    if (plan.nbytes != nbytes || plan.dtype != w) {
      registry_.declare(name);
      auto ctx = registry_.context(name);
      ctx->initialized = false;
      registry_.init_tensor(ctx, nbytes, core_dtype_of(t.scalar_type()), partition_bytes_, 4096);
      plan.nbytes = nbytes;
      plan.dtype = w;
      plan.keys = ctx->keys;
      plan.parts = ctx->parts;
    }
    const int h = handles_.allocate();
    HandleState& st = states_[h];
    st.input = t;
    st.output = out;
    st.pending = (uint32_t)plan.parts.size();
    const char* sp = (const char*)t.data_ptr();
    char* dp = (char*)out.data_ptr();
    for (size_t i = 0; i < plan.parts.size(); ++i) {
      const Partition& p = plan.parts[i];
      Part part{plan.keys[i], sp + p.offset, dp + p.offset, p.len / es, p.len, h, w, average};
      parts_[part.key].push_back(part);
      auto task = std::make_shared<Task>();
      task->key = part.key;
      task->priority = priority;
      task->len = p.len;
      queue_.add(task);
    }
    pending_bytes_ += nbytes;
    if (plan.parts.empty()) finish_empty(h);
    if (flush_bytes_ && pending_bytes_ >= flush_bytes_) flush_locked();
    return h;
  }

  // Entry point of the python engine: takes the user's name (the "byteps." prefix is added here),
  // returns -1 instead of raising when the tensors are not something this adapter moves (CPU tensors,
  // integer dtypes, empty tensors, an output of another dtype or size).  eager: launch right away when the
  // tensor is at least one partition long (it overlaps with whatever the caller enqueues next).
  int try_push_pull_async(const at::Tensor& t, const at::Tensor& out, bool average, const std::string& name,
                          int priority, int version, bool eager) {
    if (!t.is_cuda() || !out.is_cuda() || t.numel() == 0 || wire_of(t.scalar_type()) < 0 ||
        out.scalar_type() != t.scalar_type() || out.numel() != t.numel() || !t.is_contiguous() || !out.is_contiguous())
      return -1;
    const int h = push_pull_async(t, out, average, "byteps." + name, priority, version);
    bytes_total_ += (size_t)t.numel() * t.element_size();
    if (eager && (size_t)t.numel() * t.element_size() >= partition_bytes_) flush();
    return h;
  }

  // bytes enqueued since the last call (telemetry)
  size_t take_bytes() {
    std::lock_guard<std::mutex> g(mu_);
    const size_t b = bytes_total_;
    bytes_total_ = 0;
    return b;
  }

  void flush() {
    std::lock_guard<std::mutex> g(mu_);
    flush_locked();
  }

  bool poll(int h) {
    std::lock_guard<std::mutex> g(mu_);
    auto it = states_.find(h);
    if (it == states_.end()) return true;
    // never flushes: flush points must be the same on every rank, and polling is not
    if (it->second.pending > 0) return false;
    if (it->second.done == nullptr) return true;
    cudaError_t e = cudaEventQuery(it->second.done);
    if (e == cudaSuccess) return true;
    if (e != cudaErrorNotReady) cuda_check(e, "cudaEventQuery");
    return false;
  }

  // Makes the caller's current stream wait for the exchange (or blocks the host) and returns
  // the output tensor; the handle is released.
  at::Tensor synchronize(int h, bool block_host) {
    std::unique_lock<std::mutex> g(mu_);
    auto it = states_.find(h);
    if (it == states_.end()) throw std::invalid_argument("unknown or already synchronised handle");
    if (it->second.pending > 0) flush_locked();
    HandleState st = std::move(it->second);
    states_.erase(it);
    handles_.mark_done(h, Status::OK());
    handles_.wait_and_release(h, 0);
    g.unlock();
    if (st.done != nullptr) {
      if (block_host) {
        py::gil_scoped_release nogil;
        cuda_check(cudaEventSynchronize(st.done), "cudaEventSynchronize");
      } else {
        cudaStream_t cur = at::cuda::getCurrentCUDAStream(device_).stream();
        if (cur != last_wait_stream_ || st.done != last_wait_event_) {   // handles of one launch share an event
          cuda_check(cudaStreamWaitEvent(cur, st.done, 0), "cudaStreamWaitEvent");
          last_wait_stream_ = cur;
          last_wait_event_ = st.done;
        }
      }
    }
    return st.output;
  }

  size_t outstanding() {
    std::lock_guard<std::mutex> g(mu_);
    return states_.size();
  }
  size_t launches() const { return launches_; }

  // The CPU-server hierarchical path (comm/ps.py) stages its windows through the same allocator.
  size_t alloc_stage(size_t nbytes, bool end_barrier) {
    std::lock_guard<std::mutex> g(mu_);
    return alloc_stage_locked(nbytes, end_barrier);
  }

 private:
  static constexpr int kSegRows = 2048;
  struct Plan {
    size_t nbytes = 0;
    int dtype = -1;
    std::vector<uint64_t> keys;
    std::vector<Partition> parts;
  };
  struct SegSlot {
    SegDesc* host = nullptr;
    SegDesc* dev = nullptr;
    cudaEvent_t copied = nullptr;
    bool used = false;
  };

  void finish_empty(int h) { states_[h].pending = 0; }

  cudaEvent_t new_event() {
    // events are recycled once every handle that referenced them is gone; a small ring is enough
    // because launches complete in stream order
    if (event_pool_.size() < 256) {
      cudaEvent_t e;
      cuda_check(cudaEventCreateWithFlags(&e, cudaEventDisableTiming), "cudaEventCreate");
      event_pool_.push_back(e);
      return e;
    }
    cudaEvent_t e = event_pool_[event_cursor_ % event_pool_.size()];
    ++event_cursor_;
    return e;
  }

  // Bump allocation over the staging ring.  A one-shot launch skips its end barrier (one NVLink
  // round trip less): peers may still be reading my window when my kernel exits.  That is safe as
  // long as the NEXT launch uses a different window - any rank that starts launch k+2 has passed
  // launch k+1's start barrier, i.e. every rank finished launch k.  If the ring wrapped onto the
  // window of a launch that had no end barrier, a barrier-only kernel fences it first.
  size_t alloc_stage_locked(size_t nbytes, bool end_barrier) {
    if (nbytes > arena_bytes_) throw std::runtime_error("push_pull batch exceeds BYTEPS_ARENA_BYTES");
    if (stage_cursor_ + nbytes > arena_bytes_) stage_cursor_ = 0;
    const size_t off = stage_cursor_;
    stage_cursor_ = (off + nbytes + 255) / 256 * 256;
    if (have_prev_ && !prev_end_barrier_ && off < prev_hi_ && prev_lo_ < off + nbytes) {
      cuda_check(launch_barrier(pv_, 1, 0, comm_), "barrier");
      ++launches_;
    }
    have_prev_ = true;
    prev_lo_ = off;
    prev_hi_ = off + nbytes;
    prev_end_barrier_ = end_barrier;
    return off;
  }

  void flush_locked() {
    if (queue_.pending() == 0) return;
    c10::cuda::CUDAGuard guard(device_);
    // one readiness edge per flush window: everything enqueued so far was produced on this stream
    cudaStream_t cur = at::cuda::getCurrentCUDAStream(device_).stream();
    cuda_check(cudaEventRecord(ready_, cur), "cudaEventRecord");
    cuda_check(cudaStreamWaitEvent(comm_, ready_, 0), "cudaStreamWaitEvent");
    std::vector<Part> batch;
    size_t batch_bytes = 0;
    int sig_dtype = -1;
    bool sig_avg = false;
    while (true) {
      TaskPtr task = queue_.get();
      if (!task) {
        if (!batch.empty()) {
          launch(batch);
          batch.clear();
          batch_bytes = 0;
          continue;   // credits came back: try again
        }
        break;
      }
      auto& fifo = parts_[task->key];
      Part part = fifo.front();
      fifo.pop_front();
      if (fifo.empty()) parts_.erase(task->key);
      if (!batch.empty() && (part.dtype != sig_dtype || part.average != sig_avg ||
                             batch_bytes + part.nbytes > group_bytes_ || (int)batch.size() >= kSegRows)) {
        launch(batch);
        batch.clear();
        batch_bytes = 0;
      }
      sig_dtype = part.dtype;
      sig_avg = part.average;
      batch.push_back(part);
      batch_bytes += part.nbytes;
    }
    pending_bytes_ = 0;
  }

  void launch(const std::vector<Part>& batch) {
    const int dtype = batch[0].dtype;
    const int wire = (dtype == WIRE_F32 && wire_override_ >= 0) ? wire_override_ : dtype;
    SegSlot& slot = seg_ring_[seg_cursor_++ % seg_ring_.size()];
    if (slot.used) cuda_check(cudaEventSynchronize(slot.copied), "cudaEventSynchronize");
    size_t start = 0;
    for (size_t i = 0; i < batch.size(); ++i) {
      slot.host[i] = SegDesc{batch[i].src, batch[i].dst, (int64_t)start, (int64_t)batch[i].numel};
      start += (batch[i].numel + 7) / 8 * 8;
    }
    const size_t total = start;
    const size_t nbytes = total * wire_bytes(wire);
    const bool one_shot = nbytes <= one_shot_bytes_ && world_ > 1;
    const bool end_barrier = !one_shot;
    const size_t off = alloc_stage_locked(nbytes, end_barrier);
    cuda_check(cudaMemcpyAsync(slot.dev, slot.host, batch.size() * sizeof(SegDesc), cudaMemcpyHostToDevice, comm_),
               "cudaMemcpyAsync");
    cuda_check(cudaEventRecord(slot.copied, comm_), "cudaEventRecord");
    slot.used = true;
    const float scale = batch[0].average ? 1.0f / (float)world_ : 1.0f;
    const size_t shard = one_shot ? nbytes : (nbytes + world_ - 1) / world_;
    LaunchCfg cfg;
    cfg.threads = threads_;
    if (blocks_ > 0) {
      cfg.blocks = blocks_;
    } else {
      const size_t tile = (size_t)threads_ * 32;
      size_t need = (shard + tile - 1) / tile;
      cfg.blocks = (int)std::max<size_t>(1, std::min<size_t>(need, 64));
    }
    cfg.channel = 0;
    cfg.use_nvls = (nvls_ && !one_shot) ? 1 : 0;
    cfg.one_shot = one_shot ? 1 : 0;
    cfg.end_barrier = end_barrier ? 1 : 0;
    cuda_check(launch_pushpull_packed(pv_, dtype, wire, slot.dev, (int)batch.size(), off, total, scale, cfg, comm_),
               "pushpull_packed");
    ++launches_;
    cudaEvent_t ev = new_event();
    cuda_check(cudaEventRecord(ev, comm_), "cudaEventRecord");
    for (const Part& p : batch) {
      queue_.report_finish(p.nbytes);
      auto it = states_.find(p.handle);
      if (it != states_.end()) {
        if (it->second.pending > 0) --it->second.pending;
        it->second.done = ev;
      }
    }
  }

  PeerView pv_;
  int world_;
  size_t arena_bytes_;
  cudaStream_t comm_;
  int device_;
  size_t partition_bytes_, group_bytes_, one_shot_bytes_, flush_bytes_;
  int blocks_, threads_;
  bool nvls_;
  int wire_override_;
  std::mutex mu_;
  Registry registry_;
  ScheduledQueue queue_;
  HandleManager handles_;
  std::unordered_map<std::string, Plan> plans_;
  std::unordered_map<uint64_t, std::deque<Part>> parts_;
  std::unordered_map<int, HandleState> states_;
  std::array<SegSlot, 8> seg_ring_;
  size_t seg_cursor_ = 0;
  cudaEvent_t ready_ = nullptr;
  std::vector<cudaEvent_t> event_pool_;
  size_t event_cursor_ = 0;
  size_t stage_cursor_ = 0;
  bool have_prev_ = false, prev_end_barrier_ = true;
  size_t prev_lo_ = 0, prev_hi_ = 0;
  size_t pending_bytes_ = 0;
  size_t launches_ = 0;
  size_t bytes_total_ = 0;
  cudaStream_t last_wait_stream_ = nullptr;
  cudaEvent_t last_wait_event_ = nullptr;
};

}  // namespace

PYBIND11_MODULE(_torch_ops, m) {
  m.doc() = "byteps_b200 native torch adapter (push_pull on at::Tensor)";
  py::class_<NativeSymmOps>(m, "NativeSymmOps")
      .def(py::init<const std::vector<uintptr_t>&, const std::vector<uintptr_t>&, uintptr_t, uintptr_t, int, int, size_t,
                    uintptr_t, int, size_t, size_t, size_t, size_t, uint64_t, int, int, bool, int>(),
           py::arg("data"), py::arg("sig"), py::arg("mc"), py::arg("epoch"), py::arg("rank"), py::arg("world"),
           py::arg("arena_bytes"), py::arg("comm_stream"), py::arg("device"), py::arg("partition_bytes"),
           py::arg("group_bytes"), py::arg("one_shot_bytes"), py::arg("flush_bytes"), py::arg("credit_bytes"),
           py::arg("blocks"), py::arg("threads"), py::arg("nvls"), py::arg("wire_override"))
      .def("declare", &NativeSymmOps::declare)
      .def("push_pull_async", &NativeSymmOps::push_pull_async, py::arg("tensor"), py::arg("output"), py::arg("average"),
           py::arg("name"), py::arg("priority") = 0, py::arg("version") = 0)
      .def("try_push_pull_async", &NativeSymmOps::try_push_pull_async, py::arg("tensor"), py::arg("output"),
           py::arg("average"), py::arg("name"), py::arg("priority") = 0, py::arg("version") = 0,
           py::arg("eager") = true)
      .def("take_bytes", &NativeSymmOps::take_bytes)
      .def("flush", &NativeSymmOps::flush)
      .def("poll", &NativeSymmOps::poll)
      .def("synchronize", &NativeSymmOps::synchronize, py::arg("handle"), py::arg("block_host") = false)
      .def("outstanding", &NativeSymmOps::outstanding)
      .def("alloc_stage", &NativeSymmOps::alloc_stage)
      .def_property_readonly("launches", &NativeSymmOps::launches);
}
