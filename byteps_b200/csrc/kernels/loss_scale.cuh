// Dynamic loss scaling for the fused optimizer (sm_90a), decided on the device.
//
// Two launches per step on the communication stream, before the fused exchanges of the step:
//   loss_scale_check   one wave of blocks over this rank's gradient windows: does any element overflow (inf or
//                      NaN) once it is rounded to its wire dtype?  ORs an integer flag into LossScaleState::found.
//   loss_scale_update  one block: publishes the flag into every peer's slot of a small window in the arena, meets
//                      the peers (barrier_peers), ORs the W flags in rank order, updates the scale with the rule
//                      of torch._amp_update_scale_, counts applied steps per param group and writes grad_scale,
//                      skip, first_step and the Adam bias corrections into the OptHParams block of every group.
// The epilogues (EpiSGD / EpiAdam) leave the optimizer state untouched when OptHParams::skip is set.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"
#include "kernels/pushpull.cuh"

namespace bps {

// One gradient window of this rank: `n` elements (a multiple of 8) of dtype `grad` at byte offset `off` of the
// local arena, sent as dtype `wire`.
struct LossScaleCheckEntry {
  uint64_t off;
  uint64_t n;
  int32_t grad;
  int32_t wire;
  int32_t pad[2];
};

// What counts as an overflow.  GradScaler checks the gradients after the all-reduce and after unscaling; here the
// check runs on each rank's values before the exchange, so it must also rule out a finite local value whose rank
// sum, or that sum times 1/S, overflows.  An element counts when its value rounded to the wire dtype is inf, NaN, or
// larger in magnitude than kLossScaleSumLimit / world * min(1, S).  The exchange sums the peers' values in fp32
// registers (and an NVLS in-switch reduction of a bf16 or fp32 wire returns bf16 or fp32), so no sum of `world`
// checked values can overflow: 3.38e38 leaves room below bf16's largest value, 3.3895e38, for the fp32 rounding of
// the partial sums.  The bound lies far above every 16-bit wire's range, so for those it only adds the case S < 1.
// An fp16 sum reduced in the switch is returned in fp16, where finite values could sum to inf: the bucket layer
// does not use the in-switch reduction for fp16 wires in this mode.
constexpr float kLossScaleSumLimit = 3.38e38f;

// Scaler state in device memory (40 bytes).  The growth / backoff parameters live here too, so a loaded
// checkpoint reaches a step that was captured into a CUDA graph earlier.  They are float64, the precision in
// which torch._amp_update_scale_ multiplies the float scale by them.
struct LossScaleState {
  double growth;        // growth_factor
  double backoff;       // backoff_factor
  float scale;          // S: the loss of the coming step is multiplied by it
  int32_t interval;     // growth_interval
  int32_t tracker;      // clean steps since the last change of S (GradScaler's _growth_tracker)
  int32_t skipped;      // steps skipped so far
  uint32_t found;       // this rank's local overflow flag: set by the check, consumed by the update
  int32_t pad;
};

// Bytes of the agreement window in the arena: [parity][source rank] flags.
constexpr size_t kLossScaleWindowBytes = 2 * kMaxRanks * sizeof(uint32_t);

// max_vectors: 16-byte vectors of the largest window (sizes the grid)
cudaError_t launch_loss_scale_check(const PeerView& pv, const LossScaleCheckEntry* table, int nentries,
                                    size_t max_vectors, LossScaleState* state, cudaStream_t stream);

// steps: applied-step count per param group (int32); betas: (beta1, beta2) per group in float64 (Adam only);
// hp: the groups' OptHParams blocks, contiguous.
cudaError_t launch_loss_scale_update(const PeerView& pv, int channel, size_t win_off, LossScaleState* state,
                                     int32_t* steps, const double* betas, OptHParams* hp, int ngroups, int adam,
                                     cudaStream_t stream);

cudaError_t loss_scale_load_kernels();

}  // namespace bps
