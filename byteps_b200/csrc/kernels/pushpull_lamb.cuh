// LAMB in the fused exchange (sm_90a): three launches per bucket on the communication stream.
//
//   lamb_moments  pack the gradients to the wire dtype (when a wire cast is needed), meet the peers, reduce this
//                 rank's shard, update the Adam moments m and v, form u = m^ / (sqrt(v^) + eps) + wd * w and sum
//                 w^2 and u^2 of every parameter over the shard: one fixed-order segmented warp sum per 32 wire
//                 units, kept in `groups` (the segment that begins at a warp's first unit) and `heads` (a segment
//                 that begins at a parameter's first unit inside a warp).
//   lamb_norms    per parameter: this rank's partial sums (the warp sums in unit order, then a fixed tree over the
//                 CTA, all float64), stored into this rank's slot of every peer's window; barrier_peers; the ranks'
//                 slots summed in rank order give ||w||^2 and ||u||^2, and the trust ratio phi of the parameter.
//   lamb_apply    w <- w - lr * phi * u (u formed again from w, m and v, with the same instructions), and the new
//                 parameters pushed into every peer's parameter window; barrier_peers.
// No float atomics anywhere: every rank computes phi from the same float64 values in the same order, so the ranks
// that share a parameter scale it by the same bits, and runs repeat bit for bit.  See DESIGN.md 1.11.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"
#include "kernels/pushpull.cuh"

namespace bps {

// One parameter of a bucket: `n` elements from element `start` (a multiple of 8) of the bucket's flat layout.
// The parameter's padding, [start + n, start + pad8(n)), belongs to no norm.
struct LambParam {
  int64_t start;
  int64_t n;
};

// Bytes of the float64 scratch lamb_moments leaves for lamb_norms: `groups` (one (w^2, u^2) pair per 32 wire units
// of the shard) followed by `heads` (one pair per parameter).  A wire unit has 4 or 8 elements.
inline size_t lamb_scratch_bytes(size_t shard_elems, int nparams) {
  return ((shard_elems / 4 + 31) / 32 + 1 + (size_t)nparams) * 16;
}

// Bytes of one bucket's window in the arena: a (w^2, u^2) float64 pair per (parameter, source rank).
inline size_t lamb_window_bytes(int nparams, int world) { return (size_t)nparams * world * 16; }

// grad_dtype / wire / param_dtype: the (gradient, wire) pairs of launch_pushpull_fused_opt; the parameters have the
// gradient dtype.  segs/nsegs/stage_off as there (nsegs = 0: the gradients are in the arena at stage_off).
// master/m1/m2: this rank's fp32 shard state, indexed by (element - shard begin).  scratch: lamb_scratch_bytes of
// this rank's shard; phi: one float per parameter, local.  hp: the group's OptHParams (bias corrections, adapt).
cudaError_t launch_lamb_moments(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                size_t stage_off, size_t total_elems, float scale, float* master, float* m1, float* m2,
                                const LambParam* params, int nparams, double* scratch, const OptHParams* hp,
                                int blocks, int threads, int channel, int use_nvls, cudaStream_t stream);

// blocks: CTAs, the same on every rank (a function of the bucket only).
cudaError_t launch_lamb_norms(const PeerView& pv, int wire, size_t total_elems, const LambParam* params, int nparams,
                              const double* scratch, size_t win_off, float* phi, const OptHParams* hp, int blocks,
                              int channel, cudaStream_t stream);

cudaError_t launch_lamb_apply(const PeerView& pv, int grad_dtype, int wire, size_t param_off, size_t total_elems,
                              float* master, const float* m1, const float* m2, const LambParam* params, int nparams,
                              const float* phi, const OptHParams* hp, int blocks, int threads, int channel,
                              int use_nvls, cudaStream_t stream);

// Load every LAMB kernel now: a lazy load while a peer spins in a barrier can deadlock (DESIGN.md 1.6).
cudaError_t lamb_load_kernels();

}  // namespace bps
