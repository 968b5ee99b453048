// LARS in the fused exchange (sm_90a): three launches per bucket on the communication stream.
//
//   lars_norms_partial  pack the gradients to the wire dtype (when a wire cast is needed), meet the peers, reduce
//                       this rank's shard and sum w^2 and g^2 of every parameter over it, g the averaged unscaled
//                       gradient: the fixed-order segmented warp sums of LAMB, into the same `groups` / `heads`
//                       scratch.  No optimizer state is written.
//   lars_norms          per parameter: this rank's partial sums stored into its slot of every peer's window;
//                       barrier_peers; the ranks' slots summed in rank order give ||w|| and ||g||, and
//                       phi = eta * ||w|| / (||g|| + wd * ||w|| + eps) in float64, rounded once to float.
//   lars_apply          reduce the shard again from the peers' gradient or staging windows (the same reduce code and
//                       tile-to-CTA map as the first launch), v <- momentum * v + lr * phi * (g + wd * w),
//                       w <- w - v, the new parameters pushed into every peer's parameter window; barrier_peers.
// The scratch, the window and the (start, numel) table have LAMB's layout (pushpull_lamb.cuh: LambParam,
// lamb_scratch_bytes, lamb_window_bytes).  No float atomics: runs repeat bit for bit and every rank scales a
// parameter by the same phi.  See DESIGN.md 1.12.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"
#include "kernels/pushpull.cuh"
#include "kernels/pushpull_lamb.cuh"

namespace bps {

// grad_dtype / wire: the (gradient, wire) pairs of launch_pushpull_fused_opt; the parameters have the gradient dtype.
// segs/nsegs/stage_off as there (nsegs = 0: the gradients are in the arena at stage_off).  master: this rank's fp32
// shard, indexed by (element - shard begin).  scratch: lamb_scratch_bytes of this rank's shard.  hp: the group's
// OptHParams (grad_scale, skip).
cudaError_t launch_lars_norms_partial(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                      size_t stage_off, size_t total_elems, float scale, const float* master,
                                      const LambParam* params, int nparams, double* scratch, const OptHParams* hp,
                                      int blocks, int threads, int channel, int use_nvls, cudaStream_t stream);

// blocks: CTAs, the same on every rank (a function of the bucket only).  phi: one float per parameter, local.
// hp: weight_decay, eps, adapt, trust_coefficient, skip.
cudaError_t launch_lars_norms(const PeerView& pv, int wire, size_t total_elems, const LambParam* params, int nparams,
                              const double* scratch, size_t win_off, float* phi, const OptHParams* hp, int blocks,
                              int channel, cudaStream_t stream);

// stage_off: the window lars_norms_partial reduced (gradients, or the staging window of a wire cast).  mom: the
// momentum shard.  blocks and threads must be those of lars_norms_partial.  hp: lr, weight_decay, momentum,
// grad_scale, skip.
cudaError_t launch_lars_apply(const PeerView& pv, int grad_dtype, int wire, size_t stage_off, size_t param_off,
                              size_t total_elems, float scale, float* master, float* mom, const LambParam* params,
                              int nparams, const float* phi, const OptHParams* hp, int blocks, int threads,
                              int channel, int use_nvls, cudaStream_t stream);

// Load every LARS kernel now: a lazy load while a peer spins in a barrier can deadlock (DESIGN.md 1.6).
cudaError_t lars_load_kernels();

}  // namespace bps
