// Host-visible launch API of the fused push-pull kernels (sm_90a).
//
// What the reference does with ncclReduceScatter + ncclAllGather (+ncclReduce/
// ncclBroadcast tails) per <=4 MB partition, a host-side div_ and framework
// cast kernels (/root/reference/byteps/common/core_loops.cc:190-269,
// /root/reference/byteps/torch/ops.cc:78-91, torch/compression.py:47-65) is ONE
// kernel here: gather/cast the user tensors into the symmetric staging window,
// flag-barrier with the peers, reduce my shard straight out of every peer's
// memory over NVLink (P2P loads or one NVLS multimem.ld_reduce), apply the
// epilogue (scale | SGD | Adam on fp32 master weights), push the result into
// every peer (P2P stores or one multimem.st), flag-barrier, scatter/cast back.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"

namespace bps {

// One user tensor inside a packed launch.  `start` is the element offset in the
// flat wire range (multiple of 8), `n` the element count.
struct SegDesc {
  const void* src;   // user input  (dtype U)
  void* dst;         // user output (dtype U); may equal src
  int64_t start;
  int64_t n;
};

enum WireDType : int { WIRE_F32 = 0, WIRE_BF16 = 1, WIRE_F16 = 2 };

enum OptKind : int { OPT_NONE = 0, OPT_SGD = 1, OPT_ADAM = 2 };

// Hyper-parameters live in device memory so a captured CUDA graph sees new
// values (lr schedules, Adam step) on every replay.
struct OptHParams {
  float lr;
  float weight_decay;
  float momentum;
  float dampening;
  float beta1;
  float beta2;
  float eps;
  float bias_c1;     // 1 - beta1^t
  float bias_c2;     // 1 - beta2^t
  int nesterov;
  int adamw;         // decoupled weight decay
  int first_step;    // momentum buffer initialisation (buf = g)
  float grad_scale;  // extra multiplier on the reduced gradient (loss-scale^-1)
  int skip;          // dynamic loss scaling found an overflow: leave the optimizer state as it is
  int adapt;         // LAMB / LARS: scale the update by the trust ratio (0: ratio 1)
  float trust_coefficient;  // LARS: eta of phi = eta * ||w|| / (||g|| + wd * ||w|| + eps)
};

struct LaunchCfg {
  int blocks;        // CTAs (<= kMaxBlocks)
  int threads;       // threads per CTA
  int channel;       // signal-pad channel (0/1)
  int use_nvls;      // multimem path
  int one_shot;      // every rank reduces everything; no all-gather
  int end_barrier;   // 0 only for one-shot with ping-pong staging
};

// ---- in-place exchange on the symmetric arena ---------------------------------
// data at [off, off + n*elem) of every rank's arena is replaced by scale * sum.  The kernels work in
// groups of 8 elements: when n is not a multiple of 8, the elements up to the next multiple of 8
// ([off + n*elem, off + pad8(n)*elem)) are exchanged too and must be free to change.  The same holds
// for launch_pushpull_inplace_tma, launch_reduce_scatter and launch_all_gather.
cudaError_t launch_pushpull_inplace(const PeerView& pv, int wire, size_t off_bytes, size_t nelem, float scale,
                                    const LaunchCfg& cfg, cudaStream_t stream);

// Same contract, but the NVLink traffic is issued by the SM's copy engine: 1-D TMA bulk copies
// (cp.async.bulk, SASS UBLKCP) into an mbarrier-tracked shared-memory ring and bulk stores back out.
// P2P only (multicast addresses need multimem instructions).  stages in [1,4].
cudaError_t launch_pushpull_inplace_tma(const PeerView& pv, int wire, size_t off_bytes, size_t nelem, float scale,
                                        int blocks, int stages, int channel, cudaStream_t stream);

// ---- packed exchange of user tensors -----------------------------------------
// segs: device array (nsegs entries, sorted by start).  user_dtype/wire: WireDType.
// staging window = [stage_off, stage_off + total_elems * wire_size) of the arena.
cudaError_t launch_pushpull_packed(const PeerView& pv, int user_dtype, int wire, const SegDesc* segs, int nsegs,
                                   size_t stage_off, size_t total_elems, float scale, const LaunchCfg& cfg,
                                   cudaStream_t stream);

// ---- fused exchange + optimizer ------------------------------------------------
// Gradients (user tensors, dtype grad_dtype) are packed to the wire dtype,
// reduced on the shard owner, which updates its fp32 master shard / optimizer
// state and writes the new parameters (dtype param_dtype) into EVERY rank's
// parameter window at param_off.  master/state0/state1 are local fp32 arrays
// indexed by (element - shard_begin).
cudaError_t launch_pushpull_fused_opt(const PeerView& pv, int grad_dtype, int wire, int param_dtype, int opt_kind,
                                      const SegDesc* segs, int nsegs, size_t stage_off, size_t param_off,
                                      size_t total_elems, float scale, float* master, float* state0, float* state1,
                                      const OptHParams* hp, const LaunchCfg& cfg, cudaStream_t stream);

// ---- split phases for the CPU-server mode ---------------------------------------
// reduce-scatter only: my shard of the window becomes the local sum (REDUCE stage)
cudaError_t launch_reduce_scatter(const PeerView& pv, int wire, size_t off_bytes, size_t nelem, const LaunchCfg& cfg,
                                  cudaStream_t stream);
// all-gather only: my shard is pushed to every peer (BROADCAST stage), scaled
cudaError_t launch_all_gather(const PeerView& pv, int wire, size_t off_bytes, size_t nelem, float scale,
                              const LaunchCfg& cfg, cudaStream_t stream);

// barrier-only kernel (staging reuse fence, tests)
// TMA-streamed fused optimizer (gradient window already in the arena, wire == grad == param dtype):
// optimizer state moves through a shared-memory ring of `stages` tiles with bulk copies.
cudaError_t launch_pushpull_fused_opt_tma(const PeerView& pv, int wire, int opt_kind, size_t grad_off,
                                          size_t param_off, size_t total_elems, float scale, float* master,
                                          float* state0, float* state1, const OptHParams* hp, int blocks, int stages,
                                          int use_nvls, int channel, cudaStream_t stream);

cudaError_t launch_barrier(const PeerView& pv, int blocks, int channel, cudaStream_t stream);

// shard geometry shared by host and device: units of 8 elements
__host__ __device__ inline void shard_units(size_t total_units, int world, int rank, size_t* begin, size_t* end) {
  size_t per = (total_units + world - 1) / world;
  size_t b = per * (size_t)rank;
  if (b > total_units) b = total_units;
  size_t e = b + per;
  if (e > total_units) e = total_units;
  *begin = b;
  *end = e;
}

}  // namespace bps
