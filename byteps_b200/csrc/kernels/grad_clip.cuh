// Global gradient-norm clipping in the fused exchange (sm_90a), as torch.nn.utils.clip_grad_norm_ with the 2-norm.
//
//   clip_norm_partial  one launch per bucket: pack the gradients to the wire dtype (when a wire cast is needed), meet
//                      the peers, reduce this rank's shard with the reduce code and tile-to-CTA map of the fused
//                      kernels, form g = reduced * (scale * grad_scale) in fp32 as the epilogues do and add g^2 in
//                      float64 over the parameters' elements (padding counts in no norm).  Per CTA: per-thread sums
//                      in unit order, then a fixed tree; one float64 per CTA into the bucket's scratch row.  A closing
//                      barrier: the staging window is shared by all buckets, so no peer may repack it for the next
//                      bucket while this rank still reads the current one.  It writes no optimizer state, no
//                      parameter and no window other than the staging pack, and ignores OptHParams::skip, so a step
//                      that dynamic loss scaling skips still yields its (non-finite) norm.
//   clip_norm_update   one launch per step, one block: the scratch summed in (bucket, CTA) order in float64, this
//                      rank's total stored into its slot of every peer's [parity][rank] window, barrier_peers, the
//                      slots summed in rank order; N = sqrt(sum) is written to grad_norm and
//                      coef = min(1, max_norm / (N + 1e-6)) is formed in float64 and rounded once; every group's
//                      OptHParams::grad_scale is multiplied by coef.  Every rank sums the same float64 values in
//                      the same order, so every rank scales by the same bits.
// The fused epilogues multiply the reduced gradient by scale * grad_scale before anything else, so folding coef into
// grad_scale is torch's order (clip, then step) for every fused kind and engine.  See DESIGN.md 1.13.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"
#include "kernels/pushpull.cuh"
#include "kernels/pushpull_lamb.cuh"

namespace bps {

// Bytes of the [parity][source rank] float64 window of clip_norm_update.
constexpr size_t kClipWindowBytes = 2 * kMaxRanks * sizeof(double);

// grad_dtype / wire: the (gradient, wire) pairs of launch_pushpull_fused_opt.  segs/nsegs/stage_off as there
// (nsegs = 0: the gradients are in the arena at stage_off).  params: the bucket's (start, numel) table.  row: the
// bucket's scratch row, `blocks` float64 written.  hp: the group's OptHParams (grad_scale).  blocks and threads must
// be the same on every rank (a function of the bucket only).
cudaError_t launch_clip_norm_partial(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                     size_t stage_off, size_t total_elems, float scale, const LambParam* params,
                                     int nparams, double* row, const OptHParams* hp, int blocks, int threads,
                                     int channel, int use_nvls, cudaStream_t stream);

// scratch: nrows rows of row_len float64 (entries no CTA wrote must be zero).  win_off: kClipWindowBytes in the arena.
// grad_norm: one float, local.  hp: the groups' OptHParams blocks, contiguous.
cudaError_t launch_clip_norm_update(const PeerView& pv, int channel, size_t win_off, const double* scratch, int nrows,
                                    int row_len, double max_norm, float* grad_norm, OptHParams* hp, int ngroups,
                                    cudaStream_t stream);

// Load both kernels now: a lazy load while a peer spins in a barrier can deadlock (DESIGN.md 1.6).
cudaError_t clip_load_kernels();

}  // namespace bps
