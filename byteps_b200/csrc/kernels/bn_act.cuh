// Training-mode batch norm fused with the residual add and ReLU that follow it in the ResNet blocks, over NHWC
// activations viewed as M = N*H*W rows x C channels (C a multiple of 8).  Activations are fp32, bf16 or fp16
// (dtype: WIRE_F32 / WIRE_BF16 / WIRE_F16); mean, invstd, running statistics, weight, bias and their gradients are
// fp32.  Four passes:
//
//   fwd_stats    per-channel mean and biased variance: row-chunk (count, mean, M2) partials merged with Chan's
//                formula in a fixed order by the last block of each channel group; writes save_mean / save_invstd
//                and updates the running statistics (unbiased variance) when they are given
//   fwd_apply    y = act((x - mean) * invstd * weight + bias [+ residual]); with ReLU also a 1-bit mask of
//                y > 0, one byte per 8 channels of a row (bit k = channel 8j + k)
//   bwd_reduce   g = dy * mask; dbias = sum g, dweight = invstd * sum g * (x - mean)
//   bwd_apply    dx = weight * invstd * (g - dbias / M - xhat * dweight / M); dres = g when there is a residual
//
// Every reduction has a fixed shape and order and uses no float atomics, so results are bit-identical from run to
// run.  The two reduction passes need a workspace of bn_act_workspace_floats() floats and bn_act_counters() zeroed
// uint32 counters (left zeroed again on exit); a workspace must not be shared by two launches that can be in
// flight at the same time.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "kernels/peer_view.h"

namespace bps {

size_t bn_act_workspace_floats(size_t M, int C);
int bn_act_counters(int C);

cudaError_t launch_bn_act_fwd_stats(const void* x, int dtype, size_t M, int C, float eps, float momentum,
                                    float* running_mean, float* running_var, float* save_mean, float* save_invstd,
                                    float* ws, uint32_t* counters, cudaStream_t s);
cudaError_t launch_bn_act_fwd_apply(const void* x, const void* residual, int dtype, size_t M, int C, const float* mean,
                                    const float* invstd, const float* weight, const float* bias, int relu, void* y,
                                    uint8_t* mask, cudaStream_t s);
cudaError_t launch_bn_act_bwd_reduce(const void* dy, const void* x, const uint8_t* mask, int dtype, size_t M, int C,
                                     const float* mean, const float* invstd, float* dweight, float* dbias, float* ws,
                                     uint32_t* counters, cudaStream_t s);
// total: device pointer to the row count the statistics were formed over (synchronised batch norm: all ranks'
// rows, written by launch_bn_sync_stats); nullptr divides by M.
cudaError_t launch_bn_act_bwd_apply(const void* dy, const void* x, const uint8_t* mask, int dtype, size_t M, int C,
                                    const float* mean, const float* invstd, const float* weight, const float* dweight,
                                    const float* dbias, void* dx, void* dresidual, cudaStream_t s,
                                    const float* total = nullptr);

// ---- single-launch passes ------------------------------------------------------------------------------------
//
//   fwd   fwd_stats then fwd_apply in one launch: same outputs, save_mean / save_invstd and the running statistics
//   bwd   bwd_reduce then bwd_apply (dividing by M) in one launch: same outputs, dweight and dbias.  With a residual it
//         may take a second gradient dy2 of the output (the gradient of a second consumer, such as a ResNet block's
//         skip path): it then computes what the two-pass kernels compute for dy + dy2 summed as torch's add does
//         (in fp32, rounded once to the activation dtype), without that sum ever being stored
//
// Each is one cooperative launch of exactly one wave; a grid barrier separates the reduction from the apply.  A block
// holds its whole chunk in its share of shared memory when it fits; otherwise a ring of a few row-steps streams the
// rest of the chunk through shared memory with asynchronous copies, and the held rows get the space the ring leaves
// (at most `cap` bytes of them when cap >= 0; cap = 0 streams every row twice), so the apply reads most of its input
// from on chip or L2 instead of HBM.  Results do not depend on how many rows are held.  bn_act_fused_plan tells
// whether the pass can run at (M, C, dtype) on the current device (false: use the two-pass kernels; the launchers
// then return cudaErrorNotSupported) and fills in its workspace: ws_floats floats and `counters` zeroed uint32
// counters, per launch as for the two-pass kernels, except that the counters are left non-zero.
struct BnFusedPlan {
  size_t ws_floats;
  int counters;
  size_t rows_per_chunk;   // rows of a block's chunk (the last chunk may have fewer)
  int held_rows;           // rows of a chunk held in shared memory from the reduction to the apply
  size_t held_bytes;       // shared memory of the held rows per block
  int ring_depth;          // row-steps of the streaming ring (0: the whole chunk is held)
  size_t smem_bytes;       // dynamic shared memory per block: held rows and ring
  size_t bytes_moved;      // bytes a launch with (relu, residual, dy2) reads and writes, re-reads of streamed rows included
  int wave_blocks;         // blocks in one wave on this device: the grid is at most this large
};
// residual selects the backward's layout too (a residual backward needs more shared memory per ring slot).
// pool_h, pool_w > 0: the pooled passes below over images of pool_h x pool_w (M a multiple of pool_h * pool_w; relu
// and no residual), whose bytes_moved counts the pooled tensors, the halo rows and their re-reads.
bool bn_act_fused_plan(int bwd, int dtype, size_t M, int C, long long cap, int relu, int residual, int dy2,
                       BnFusedPlan* plan, int pool_h = 0, int pool_w = 0);
cudaError_t launch_bn_act_fwd(const void* x, const void* residual, int dtype, size_t M, int C, float eps,
                              float momentum, float* running_mean, float* running_var, float* save_mean,
                              float* save_invstd, const float* weight, const float* bias, int relu, void* y,
                              uint8_t* mask, float* ws, uint32_t* counters, long long cap, cudaStream_t s);
// dy2: nullptr, or a second gradient laid out as dy (needs dresidual)
cudaError_t launch_bn_act_bwd(const void* dy, const void* dy2, const void* x, const uint8_t* mask, int dtype, size_t M,
                              int C, const float* mean, const float* invstd, const float* weight, float* dweight,
                              float* dbias, void* dx, void* dresidual, float* ws, uint32_t* counters, long long cap,
                              cudaStream_t s);

// ---- pooled single-launch passes: ReLU, then a max pool of kernel 3, stride 2, padding 1 (ResNet's stem) -------
//
// Over N NHWC images of H x W x C; the pooled output is N x OH x OW x C with OH = (H - 1) / 2 + 1 and likewise OW.
//   fwd_pool   launch_bn_act_fwd's statistics, bit for bit; writes the pooled output (what torch's max_pool2d of y
//              gives) and, per pooled row and 8 channels, one uint32 of 4-bit window codes (N * OH * OW * C / 8
//              words) instead of y and the mask
//   bwd_pool   for the gradients g1 and g2 (nullptr: none) of the pooled output: dx, dweight and dbias of
//              launch_bn_act_bwd fed what torch's add of g1 and g2, max-pool backward and ReLU mask produce, bit for
//              bit, without that gradient ever being stored
// Plans, workspaces and cap as for the single-launch passes (bn_act_fused_plan with pool_h = H, pool_w = W).
cudaError_t launch_bn_act_fwd_pool(const void* x, int dtype, int N, int H, int W, int C, float eps, float momentum,
                                   float* running_mean, float* running_var, float* save_mean, float* save_invstd,
                                   const float* weight, const float* bias, void* pooled, uint32_t* code, float* ws,
                                   uint32_t* counters, long long cap, cudaStream_t s);
cudaError_t launch_bn_act_bwd_pool(const void* g1, const void* g2, const uint32_t* code, const void* x, int dtype,
                                   int N, int H, int W, int C, const float* mean, const float* invstd,
                                   const float* weight, float* dweight, float* dbias, void* dx, float* ws,
                                   uint32_t* counters, long long cap, cudaStream_t s);

// ---- synchronised batch norm (torch.nn.SyncBatchNorm semantics) over peer-mapped memory --------------------
//
//   fwd_stats_local   fwd_stats in local-partials mode: this rank's per-channel mean and M2 over its M >= 1 rows
//   sync_stats        pushes (M_r, mean, M2) into every peer's window, meets the peers (barrier_peers on
//                     `channel`), merges the W partials in rank order with Chan's formula; writes mean, invstd
//                     (biased variance), the running statistics (unbiased variance) and the total count N.  Every
//                     rank performs the same operations in the same order, so all ranks get the same bits.  N must
//                     be at least 2.
//   sync_grad         the same exchange for bwd_reduce's local (dbias, dweight) = (sum g, invstd * sum g (x - mean));
//                     writes their sums over the ranks in rank order, which bwd_apply reads together with N.
//
// The window at pv.data[r] + win_off holds bn_sync_window_floats(world, cmax) floats (16-byte aligned) on every
// rank; C <= cmax.  Launches on one rank must come from one stream, in the same order on every
// rank, and every kernel a rank may launch must be loaded (bn_act_load_kernels) before the first one, since a
// module load while a peer's kernel spins can deadlock.  The grids are at most 8 blocks of 64 threads.
size_t bn_sync_window_floats(int world, int cmax);
cudaError_t bn_act_load_kernels();
cudaError_t launch_bn_act_fwd_stats_local(const void* x, int dtype, size_t M, int C, float* local_mean,
                                          float* local_m2, float* ws, uint32_t* counters, cudaStream_t s);
cudaError_t launch_bn_sync_stats(const PeerView& pv, int channel, size_t win_off, int cmax, int C,
                                 const float* local_mean, const float* local_m2, float count, float eps,
                                 float momentum, float* running_mean, float* running_var, float* save_mean,
                                 float* save_invstd, float* total, cudaStream_t s);
cudaError_t launch_bn_sync_grad(const PeerView& pv, int channel, size_t win_off, int cmax, int C, const float* dbias,
                                const float* dweight, float* sum_dbias, float* sum_dweight, cudaStream_t s);

}  // namespace bps
