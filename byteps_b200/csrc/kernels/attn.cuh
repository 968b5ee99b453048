// Self-attention of the BERT encoder, softmax(Q K^T / sqrt(64) + mask) -> dropout(p) -> @ V, fused into one launch
// forward and two backward, reading Q, K and V in place from the qkv projection's output.
//
// Layouts (B batch, S sequence, H heads, head dimension D = 64, E = 64 H; bf16 or fp16 by dtype = WIRE_BF16 /
// WIRE_F16):
//   qkv   [B, S, 3, H, 64] contiguous: row (b, s) has stride 3E, Q at column h * 64, K at E + h * 64, V at 2E + h * 64
//   out   [B, S, H, 64] = [B, S, E] contiguous, the context the output projection reads
//   dout  like out;  dqkv like qkv (every element written once)
//   lse   fp32 [B, H, S]: the natural log-sum-exp of each query row's scaled, masked scores (+inf for a row whose keys
//         are all masked, whose output and gradients are then zero)
//   delta fp32 [B, H, S] workspace of the backward: rowsum(dout * out)
//   mask  nullptr, or one additive value per key: element (b, k) at mask[b * mask_bstride + k] (mask_bstride 0
//         broadcasts one row over the batch) of kind ATTN_MASK_F32 / BF16 / F16 (added to the score) or
//         ATTN_MASK_BOOL (uint8: nonzero attends, zero adds -inf)
//
// Dropout keeps element i = ((b H + h) S + q) S + k of the attention matrix when word i % 4 of Philox4x32-10 (key =
// seed, counter = (i / 4, offset), 64 bits each, low word first) is below `keep` (= (1 - p) * 2^32), the scheme of
// the LayerNorm kernels (ln.cuh); kept probabilities are scaled by `scale` (1 / (1 - p)).  seed points to the device
// pair {seed, offset}; nullptr means no dropout.  The backward regenerates the bits.
//
// Every pointer but mask, lse and delta is 16-byte aligned.  Sums run in a fixed order and nothing is accumulated
// with atomics, so results are bit-identical from run to run.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bps {

constexpr int kAttnHeadDim = 64;
constexpr int kAttnMaxSeq = 512;

enum AttnMaskKind { ATTN_MASK_F32 = 0, ATTN_MASK_BF16 = 1, ATTN_MASK_F16 = 2, ATTN_MASK_BOOL = 3 };

cudaError_t launch_attn_fwd(const void* qkv, int dtype, int B, int S, int H, int D, const void* mask, int mask_kind,
                            int64_t mask_bstride, const int64_t* seed, uint32_t keep, float scale, void* out,
                            float* lse, cudaStream_t s);
// launch 1 (one CTA per 64-query tile) writes delta and dQ; launch 2 (one CTA per 64-key tile) writes dK and dV
cudaError_t launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype, int B,
                            int S, int H, int D, const void* mask, int mask_kind, int64_t mask_bstride,
                            const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                            cudaStream_t s);

}  // namespace bps
