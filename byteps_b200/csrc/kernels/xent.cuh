// Softmax cross-entropy over logits viewed as M rows x V classes (one launch per direction).  Logits and dlogits are
// fp32, bf16 or fp16 (dtype: WIRE_F32 / WIRE_BF16 / WIRE_F16), contiguous, with 16-byte aligned bases; V is
// arbitrary, so a row may start anywhere in a 16-byte line and the kernels peel a scalar head and tail around the
// row's 16-byte vectors.  Targets are int64 [M].  All arithmetic is fp32; offsets are 64-bit.
//
//   fwd   per row: lse = max + log(sum exp(x - max)) from one pass (running max and sum), loss = lse - x[target].
//         A row whose target is ignore_index is not read: loss 0, lse 0.  A target outside [0, V) that is not
//         ignore_index is never read either: its loss is NaN (and so is the reduced loss).  Writes lse[M] and
//         loss_rows[M], *count = the rows that are not ignored (int64), and *out = sum of loss_rows, divided by
//         *count when `mean` (NaN when no row counts).  The sum runs in a fixed order: each block adds its rows in
//         row order, the last block of every 16 adds theirs in block order and the last of those adds the runs, so
//         results are bit-identical from run to run.  It needs xent_workspace_floats(M) floats of workspace and
//         xent_counters(M) zeroed uint32 counters (left zeroed again on exit), not shared by two launches that can
//         be in flight at the same time.
//   bwd   dlogits[i, j] = g_i * (exp(x[i, j] - lse[i]) - [j == target[i]]) in the logits dtype, with g_i read on the
//         device: grad[i] (mode XENT_NONE), grad[0] (XENT_SUM) or grad[0] / *count (XENT_MEAN).  Ignored rows get
//         zeros; rows with a target outside [0, V) get NaN.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bps {

enum XentMode : int { XENT_NONE = 0, XENT_SUM = 1, XENT_MEAN = 2 };

size_t xent_workspace_floats(size_t M);
int xent_counters(size_t M);

cudaError_t launch_xent_fwd(const void* logits, const int64_t* target, int dtype, size_t M, int V,
                            int64_t ignore_index, bool mean, float* lse, float* loss_rows, float* out, int64_t* count,
                            float* ws, uint32_t* counters, cudaStream_t s);
cudaError_t launch_xent_bwd(const void* logits, const int64_t* target, int dtype, size_t M, int V,
                            int64_t ignore_index, const float* lse, const float* grad, int mode, const int64_t* count,
                            void* dlogits, cudaStream_t s);

}  // namespace bps
