// Persistent descriptor-ring exchange kernel (sm_90a).
//
// The reference moves every <=4 MB partition with its own NCCL calls, issued in groups of 4+4 by a
// host thread that pops a priority queue with byte credits and tells the other ranks what it
// picked over Unix datagrams (/root/reference/byteps/common/scheduled_queue.cc:82-163,
// core_loops.cc:271-360, communicator.cc:185-196).  Here ONE launch per step consumes a
// device-visible ring of bucket/partition descriptors:
//
//   * readiness   - a gradient window becomes ready when the producing stream runs `ring_mark`
//                   (or the ring kernel marks its own descriptors at entry); the mark is a
//                   release-store of the slot's next generation into EVERY rank's signal pad, so
//                   "all 8 ranks have this gradient" is a poll of local memory;
//   * order       - static (table order) by default, like the reference without
//                   BYTEPS_SCHEDULING_CREDIT; with scheduling on, a scheduler warp on rank 0 picks
//                   the globally-ready descriptor with the highest priority (ties: lowest key)
//                   that fits the byte-credit window and publishes the decision sequence to all
//                   ranks (the reference's root -> DO_REDUCE broadcast);
//   * exchange    - every worker CTA reduces its tiles of "my shard" out of all peers
//                   (multimem.ld_reduce in the switch, or 16-byte P2P loads), applies the epilogue
//                   (scale | SGD | Adam on fp32 master weights) and multicasts the result
//                   (multimem.st / P2P stores), then moves on to the next descriptor WITHOUT any
//                   cross-rank barrier: nothing in descriptor i+1 depends on remote progress of
//                   descriptor i;
//   * completion  - the last CTA of a rank to finish a slot publishes its generation to every
//                   peer; a slot is complete locally when all peers have published.  The kernel
//                   leaves only when every slot of the launch is complete on every rank, so
//                   stream order after the launch means "all gradients / parameters are in place".
//
// Generations are per-slot counters kept in device memory (peer_view.h::RingState), so a captured
// CUDA graph can replay the launch and its marks forever without host involvement.
#include "kernels/pushpull_ring.cuh"

#include "kernels/common.cuh"
#include "kernels/pushpull_dev.cuh"

namespace bps {

namespace {

constexpr int kRingThreads = 512;
constexpr int kRingUnrollNvls = 4;      // units in flight per thread on the multimem path (plain all-reduce)

__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_release_sys64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.add.acq_rel.gpu.global.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}
__device__ __forceinline__ void nanosleep(unsigned ns) { asm volatile("nanosleep.u32 %0;" ::"r"(ns)); }

__device__ __forceinline__ uint32_t* ready_flag(const PeerView& pv, int owner, uint32_t slot, int src) {
  return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(pv.sig[owner]) + kRingReadyOff) + slot * kMaxRanks + src;
}
__device__ __forceinline__ uint32_t* done_flag(const PeerView& pv, int owner, uint32_t slot, int src) {
  return reinterpret_cast<uint32_t*>(reinterpret_cast<char*>(pv.sig[owner]) + kRingDoneOff) + slot * kMaxRanks + src;
}
__device__ __forceinline__ unsigned long long* order_entry(const PeerView& pv, int owner, int pos) {
  return reinterpret_cast<unsigned long long*>(reinterpret_cast<char*>(pv.sig[owner]) + kRingOrderOff) + pos;
}

__device__ __forceinline__ void ring_timeout(const PeerView& pv, const char* what, int a, int b) {
  printf("byteps_b200: rank %d block %d timed out in the descriptor ring waiting for %s (%d, %d)\n", pv.rank,
         (int)blockIdx.x, what, a, b);
  __trap();
}

// Publish this rank's next generation of `slot` to every rank (including itself).  One thread.
__device__ __forceinline__ void publish_ready(const PeerView& pv, RingState* rs, uint32_t slot) {
  const uint32_t gen = rs->marked[slot] + 1;
  rs->marked[slot] = gen;
  fence_sys();   // everything the producing stream wrote is performed before the flag (release pattern)
  for (int p = 0; p < pv.world; ++p) st_relaxed_sys(ready_flag(pv, p, slot, pv.rank), gen);
}

// true when every rank has published generation `want` (or later) of `slot`
__device__ __forceinline__ bool all_ready(const PeerView& pv, uint32_t slot, uint32_t want) {
  for (int p = 0; p < pv.world; ++p)
    if ((int32_t)(ld_acquire_sys(ready_flag(pv, pv.rank, slot, p)) - want) < 0) return false;
  return true;
}

// ------------------------------------------------------------------------------------------------
// one descriptor, worker CTA `id.cta` of `id.ncta`
// One descriptor, worker CTA `id.cta` of `id.ncta`.  The kernel is specialised on (wire dtype,
// epilogue kind): with all nine combinations in one kernel the union of their live ranges spilled
// kilobytes per thread.  A launch therefore takes descriptors of ONE class; a step with bf16 and
// fp32 buckets is two launches.
template <class W, int KIND>
__device__ __forceinline__ void process_desc(const PeerView& pv, const RingDesc& d, bool nvls, CtaId id) {
  constexpr int E = W::kPerVec;
  size_t s0, s1;
  shard_units_of<E>(d.groups, pv.world, pv.rank, &s0, &s1);
  if constexpr (KIND != RING_ALLREDUCE) {
    if (d.hp->skip) return;     // a step skipped by dynamic loss scaling: no update, nothing written
  }
  const int rot = rot_of(pv);
  const size_t goff = d.grad_off, poff = d.param_off;
  if constexpr (KIND == RING_ALLREDUCE) {
    EpiScale epi{d.scale};
    if (nvls)
      reduce_phase_nvls<W, kRingUnrollNvls>(pv, goff, s0, s1, epi,
                                            [&](const float* f, size_t unit) { sink_peers<W, E>(pv, goff, unit, f, true); },
                                            id);
    else
      reduce_phase<W, kUnroll>(pv, goff, s0, s1, false, rot, epi,
                               [&](const float* f, size_t unit) { sink_peers<W, E>(pv, goff, unit, f, false); }, id);
  } else if constexpr (KIND == RING_SGD) {
    EpiSGD epi{d.master, d.state0, s0 * E, d.scale, *d.hp};
    reduce_phase<W, kUnrollOpt>(pv, goff, s0, s1, nvls, rot, epi,
                                [&](const float* f, size_t unit) { sink_peers<W, E>(pv, poff, unit, f, nvls); }, id);
  } else {
    EpiAdam epi{d.master, d.state0, d.state1, s0 * E, d.scale, *d.hp};
    reduce_phase<W, kUnrollOpt>(pv, goff, s0, s1, nvls, rot, epi,
                                [&](const float* f, size_t unit) { sink_peers<W, E>(pv, poff, unit, f, nvls); }, id);
  }
}

// The scheduling root (rank 0, last CTA): picks among the globally ready descriptors by
// (priority desc, table position asc) under a byte-credit window - BytePSScheduledQueue::getTask -
// and publishes the decision sequence to every rank.
__device__ void scheduler_loop(const PeerView& pv, RingState* rs, const RingDesc* descs, int n, uint32_t launch,
                               unsigned long long credit) {
  __shared__ uint32_t taken[kRingSlots / 32];
  const int lane = threadIdx.x & 31;
  if (threadIdx.x >= 32) return;
  for (int i = lane; i < kRingSlots / 32; i += 32) taken[i] = 0;
  __syncwarp();
  unsigned long long decided_bytes = 0;
  int decided = 0;
  SpinWatch watch;
  while (decided < n) {
    unsigned long long best = 0;   // (priority + 2^31) << 32 | (2^31 - position): larger is better, 0 = none
    for (int i = lane; i < n; i += 32) {
      if ((taken[i >> 5] >> (i & 31)) & 1u) continue;
      const uint32_t slot = descs[i].slot;
      if (!all_ready(pv, slot, rs->expected[slot])) continue;
      const unsigned long long key =
          ((unsigned long long)((uint32_t)descs[i].priority ^ 0x80000000u) << 32) | ((1u << 31) - (uint32_t)i);
      if (key > best) best = key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
      if (other > best) best = other;
    }
    bool issued = false;
    if (best != 0) {
      const int i = (int)((1u << 31) - (uint32_t)(best & 0xffffffffull));
      const unsigned long long done = *(volatile unsigned long long*)&rs->done_bytes;
      const unsigned long long inflight = decided_bytes - done;
      if (credit == 0 || inflight == 0 || inflight + descs[i].bytes <= credit) {
        if (lane < pv.world)
          st_release_sys64(order_entry(pv, lane, decided), ((unsigned long long)launch << 32) | (uint32_t)i);
        if (lane == 0) taken[i >> 5] |= 1u << (i & 31);
        __syncwarp();
        decided_bytes += descs[i].bytes;
        ++decided;
        issued = true;
        watch.reset();
      }
    }
    if (!issued) {
      nanosleep(200);
      if (watch.expired(pv)) ring_timeout(pv, "a ready descriptor (scheduler)", decided, n);
    }
  }
}

template <class W, int KIND>
__global__ void __launch_bounds__(kRingThreads, 1)
    pushpull_ring_kernel(PeerView pv, const RingDesc* __restrict__ descs, int n, int nvls, int sched, int self_mark,
                         unsigned long long credit, int solo) {
  RingState* rs = ring_state_of(pv.epoch);
  const int nworkers = sched ? (int)gridDim.x - 1 : (int)gridDim.x;
  const uint32_t launch = rs->launch_id + 1;
  __shared__ uint32_t s_last;

  if (sched && (int)blockIdx.x == nworkers) {
    // ------------------------------------------------------------------ scheduler CTA
    if (pv.rank == 0) scheduler_loop(pv, rs, descs, n, launch, credit);
  } else {
    // ------------------------------------------------------------------ worker CTAs
    if (self_mark && blockIdx.x == 0) {
      // the launch itself is ordered after the producers (stream order): mark every descriptor now
      for (int i = threadIdx.x; i < n; i += blockDim.x) publish_ready(pv, rs, descs[i].slot);
    }
    // No CTA-wide synchronisation on the per-descriptor path: every warp finds out on its own which
    // descriptor is next and that it is ready (local polls), does its share of the tiles and ARRIVES on a
    // named barrier; only warp 0 waits on that barrier, fences the CTA's remote stores (one NVLink round trip)
    // and reports the CTA done - while the other fifteen warps are already loading the next descriptor.
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    for (int seq = 0; seq < n; ++seq) {
      // ---- which descriptor, and is it ready everywhere?
      int i = seq;
      if (sched) {
        if (lane == 0) {
          SpinWatch watch;
          const unsigned long long* e = order_entry(pv, pv.rank, seq);
          unsigned long long v;
          while ((uint32_t)((v = ld_acquire_sys64(e)) >> 32) != launch) {
            nanosleep(100);
            if (watch.expired(pv)) ring_timeout(pv, "the scheduler's decision", seq, n);
          }
          i = (int)(uint32_t)v;
        }
        i = __shfl_sync(0xffffffffu, i, 0);
      }
      const RingDesc& d = descs[i];
      const uint32_t slot = d.slot;
      if (lane < pv.world) {
        // with scheduling on the root has already seen every rank's flag; acquiring them here
        // as well keeps the data dependency explicit (and costs one local load per peer)
        const uint32_t want = rs->expected[slot];
        const uint32_t* f = ready_flag(pv, pv.rank, slot, lane);
        SpinWatch watch;
        while ((int32_t)(ld_acquire_sys(f) - want) < 0) {
          nanosleep(64);
          if (watch.expired(pv)) ring_timeout(pv, "a peer's gradient (slot, peer)", (int)slot, lane);
        }
      }
      __syncwarp();
      if (blockIdx.x == 0 && threadIdx.x == 0) {
        rs->t_start[slot] = globaltimer_ns();
        rs->order_pos[slot] = (uint32_t)seq;
      }
      // rotate the tile -> CTA map so small descriptors do not always land on the first CTAs
      const int vcta = ((int)blockIdx.x + seq * 5) % nworkers;
      const CtaId id(vcta, nworkers);
      process_desc<W, KIND>(pv, d, nvls != 0, id);
      // ---- completion: last CTA of this rank publishes the slot's generation to every peer
      const int bar_id = 1 + (seq & 7);
      if (warp != 0) {
        named_bar_arrive(bar_id, kRingThreads);
      } else {
        named_bar_sync(bar_id, kRingThreads);      // all sixteen warps have issued their stores
        if (lane == 0) {
          fence_sys();   // this CTA's peer stores / multimem stores are performed before it counts as arrived
          const uint32_t prev = atom_add_acq_rel_gpu(&rs->arrive[slot], 1u);
          if (prev == (uint32_t)nworkers - 1) {
            rs->arrive[slot] = 0;
            const uint32_t gen = rs->expected[slot];
            fence_sys();
            for (int p = 0; p < pv.world; ++p) st_relaxed_sys(done_flag(pv, p, slot, pv.rank), gen);
            rs->t_end[slot] = globaltimer_ns();
            atomicAdd(&rs->done_bytes, (unsigned long long)d.bytes);
          }
        }
        __syncwarp();
      }
      // the eight barrier ids are reused round robin: never let a warp run a whole cycle ahead of warp 0
      if ((seq & 7) == 7) __syncthreads();
    }
    __syncthreads();
    // ---- leave only when every slot is complete on every rank: peers have finished reading my
    // gradient windows and writing my result windows
    // (solo: profiling only - one rank runs alone under ncu, the peers' flags were published beforehand)
    if (blockIdx.x == 0 && !solo) {
      for (int k = threadIdx.x; k < n * pv.world; k += blockDim.x) {
        const int i = k / pv.world, p = k - i * pv.world;
        const uint32_t slot = descs[i].slot;
        const uint32_t want = rs->expected[slot];
        const uint32_t* f = done_flag(pv, pv.rank, slot, p);
        SpinWatch watch;
        while ((int32_t)(ld_acquire_sys(f) - want) < 0) {
          nanosleep(64);
          if (watch.expired(pv)) ring_timeout(pv, "a peer to finish (slot, peer)", (int)slot, p);
        }
      }
    }
  }
  // ---- the last CTA out advances the generations for the next launch
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    s_last = atom_add_acq_rel_gpu(&rs->exit_count, 1u) == gridDim.x - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (s_last) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) rs->expected[descs[i].slot] += 1;
    if (threadIdx.x == 0) {
      rs->launch_id = launch;
      rs->exit_count = 0;
      rs->done_bytes = 0;
    }
  }
}

__global__ void ring_mark_kernel(PeerView pv, RingSlotList slots) {
  RingState* rs = ring_state_of(pv.epoch);
  if ((int)threadIdx.x < slots.n) publish_ready(pv, rs, slots.slot[threadIdx.x]);
}

__global__ void ring_stamp_kernel(PeerView pv, int idx) {
  ring_state_of(pv.epoch)->stamps[idx] = globaltimer_ns();
}

}  // namespace

cudaError_t launch_pushpull_ring(const PeerView& pv, int wire, int kind, const RingDesc* descs, int n, int blocks,
                                 int use_nvls, int sched, int self_mark, unsigned long long credit_bytes,
                                 cudaStream_t stream, int solo) {
  if (n < 1 || n > kRingSlots || blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  const int grid = blocks + (sched ? 1 : 0);
#define BPS_RING(W, K)                                                                                              \
  pushpull_ring_kernel<W, K><<<grid, kRingThreads, 0, stream>>>(pv, descs, n, use_nvls, sched, self_mark,           \
                                                                credit_bytes, solo);                               \
  return cudaGetLastError();
#define BPS_RING_KINDS(W)                                \
  if (kind == RING_ALLREDUCE) { BPS_RING(W, RING_ALLREDUCE) } \
  if (kind == RING_SGD) { BPS_RING(W, RING_SGD) }             \
  if (kind == RING_ADAM) { BPS_RING(W, RING_ADAM) }
  if (wire == WIRE_F32) { BPS_RING_KINDS(TagF32) }
  if (wire == WIRE_BF16) { BPS_RING_KINDS(TagBF16) }
  if (wire == WIRE_F16) { BPS_RING_KINDS(TagF16) }
#undef BPS_RING_KINDS
#undef BPS_RING
  return cudaErrorInvalidValue;
}

cudaError_t launch_ring_mark(const PeerView& pv, const uint32_t* slots, int n, cudaStream_t stream) {
  if (n < 1) return cudaSuccess;
  for (int base = 0; base < n; base += kRingMarkBatch) {
    RingSlotList l;
    l.n = n - base < kRingMarkBatch ? n - base : kRingMarkBatch;
    for (int i = 0; i < l.n; ++i) {
      if (slots[base + i] >= (uint32_t)kRingSlots) return cudaErrorInvalidValue;
      l.slot[i] = slots[base + i];
    }
    ring_mark_kernel<<<1, kRingMarkBatch, 0, stream>>>(pv, l);
  }
  return cudaGetLastError();
}

// CUDA loads kernels lazily, and a first-time load may wait for kernels that are running.  A ring
// kernel spins until its producers have run, so everything a producer might launch from this
// module must be resident before the first persistent launch.
cudaError_t ring_preload() {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, ring_mark_kernel);
  if (e != cudaSuccess) return e;
  e = cudaFuncGetAttributes(&a, ring_stamp_kernel);
  if (e != cudaSuccess) return e;
#define BPS_PRELOAD(W)                                                                      \
  if ((e = cudaFuncGetAttributes(&a, pushpull_ring_kernel<W, RING_ALLREDUCE>)) != cudaSuccess) return e; \
  if ((e = cudaFuncGetAttributes(&a, pushpull_ring_kernel<W, RING_SGD>)) != cudaSuccess) return e;       \
  if ((e = cudaFuncGetAttributes(&a, pushpull_ring_kernel<W, RING_ADAM>)) != cudaSuccess) return e;
  BPS_PRELOAD(TagF32)
  BPS_PRELOAD(TagBF16)
  BPS_PRELOAD(TagF16)
#undef BPS_PRELOAD
  return cudaSuccess;
}

cudaError_t launch_ring_stamp(const PeerView& pv, int idx, cudaStream_t stream) {
  if (idx < 0 || idx >= kRingStamps) return cudaErrorInvalidValue;
  ring_stamp_kernel<<<1, 1, 0, stream>>>(pv, idx);
  return cudaGetLastError();
}

}  // namespace bps
