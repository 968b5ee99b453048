// Dropout, residual add and LayerNorm of the BERT encoder fused into one launch per direction, over activations
// viewed as M rows x H columns (normalised over a row; H a multiple of 8, 8 <= H <= 2048).  Activations are fp32,
// bf16 or fp16 (dtype: WIRE_F32 / WIRE_BF16 / WIRE_F16); gamma, beta and their gradients are fp32 or the activation
// dtype (wdtype); mean and rstd are fp32.  Every pointer is 16-byte aligned and every row contiguous.
//
//   fwd   z = residual + dropout(y), rounded to the activation dtype; out = (z - mean) * rstd * gamma + beta with the
//         row's mean and rstd = 1 / sqrt(var + eps) formed in two steps from the held row (the mean, then the sum of
//         squared deviations).  Writes out, mean and rstd, z when z != nullptr, and the 1-bit keep mask when
//         mask != nullptr (dropout on): one byte per 8 elements of a row, bit k = element 8j + k.  residual may be
//         nullptr.
//   bwd   g = dout * gamma, xhat = (z - mean) * rstd, dz = rstd * (g - mean_H(g) - xhat * mean_H(g * xhat));
//         writes dres = dz and dy = dz * mask * scale, each when its pointer is given (mask nullptr: dy = dz * scale),
//         and dgamma = sum dout * xhat, dbeta = sum dout over the rows.
//
// Dropout keeps element i = row * H + col when word i % 4 of Philox4x32-10 (key = seed, counter = (i / 4, offset),
// 64 bits each, low word first) is below `keep` (= (1 - p) * 2^32), and scales kept values by `scale` (1 / (1 - p)).
// seed points to the device pair {seed, offset}, so the bits do not depend on the launch geometry and a captured
// launch reads whatever pair the step drew before it.
//
// A group of 16 to 128 threads owns a row and holds it in registers; each block walks a contiguous chunk of rows and
// the grid is one resident wave (sized with the occupancy API).  bwd sums each block's dgamma / dbeta partials in a
// fixed order, then the last block of every 16 sums theirs and the last of those writes the result, so results are
// bit-identical from run to run; it needs a workspace of ln_workspace_floats(M, H) floats and ln_counters(M, H)
// zeroed uint32 counters (left zeroed again on exit), which must not be shared by two launches that can be in flight
// at the same time.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bps {

constexpr int kLnMaxH = 2048;

size_t ln_workspace_floats(size_t M, int H);
int ln_counters(size_t M, int H);

cudaError_t launch_ln_fwd(const void* y, const void* residual, int dtype, int wdtype, size_t M, int H, float eps,
                          const void* gamma, const void* beta, const int64_t* seed, uint32_t keep, float scale,
                          void* z, void* out, float* mean, float* rstd, uint8_t* mask, cudaStream_t s);
cudaError_t launch_ln_bwd(const void* dout, const void* z, const uint8_t* mask, int dtype, int wdtype, size_t M, int H,
                          float scale, const float* mean, const float* rstd, const void* gamma, void* dres, void* dy,
                          void* dgamma, void* dbeta, float* ws, uint32_t* counters, cudaStream_t s);

}  // namespace bps
