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
//
// Packed variable-length form (attn_varlen.cu): N sequences concatenated into one stream of T tokens, attention
// never crossing a sequence boundary.
//   qkv   [T, 3, H, 64], out / dout [T, E], dqkv like qkv, lse / delta fp32 [H, T]
//   cu_seqlens  device int32 [N + 1]: sequence n is tokens [cu[n], cu[n + 1]); zero-length sequences are allowed, so
//         a caller can pad the array to a fixed capacity by repeating its last value
//   max_seqlen  host bound on every length, in [1, 512]; the grid is (ceil(max_seqlen / 64), H, N), fixed for a
//         given capacity, so a launch captures into a CUDA graph and cu_seqlens may change between replays
// Tokens outside every sequence (before cu[0], or from cu[N] on) get a zero context, lse = +inf and zero d(qkv).  A
// sequence longer than max_seqlen gets NaN in its context, lse and d(qkv) rows.  Offsets are clamped into [0, T)
// before any address is formed from them, so no cu_seqlens makes an access leave the buffers; for offsets out of
// order the results are unspecified.
// Dropout keeps element (head h, query token t, key token u of sequence n) when word i % 4 of the Philox block with
// counter (i / 4, offset) is below `keep`, where i = (h T + t) * 512 + (u - cu[n]): the padded numbering with the
// batch row replaced by the token and the key stride fixed at the longest supported sequence.
//
// Causal mask (causal = true, attn_causal.cu): query q attends to key k only when k <= q, in the padded form with
// q and k the positions in the batch row and in the packed form the positions within the sequence (t - cu[n] and
// u - cu[n]).  A key-padding mask still applies on top: a query row whose allowed keys are all masked gets a zero
// context, lse = +inf and zero gradients, as above.  The dropout numbering is the one above, so an element a causal
// call keeps is one the bidirectional call with the same (seed, offset) keeps.  Forward and the dQ launch of query
// tile x visit key tiles 0 .. x only and the dK / dV launch of key tile y query tiles y .. last, masking the diagonal
// tile element by element; everything else above holds unchanged, and it is still one launch forward and two
// backward.
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
                            float* lse, cudaStream_t s, bool causal = false);
// launch 1 (one CTA per 64-query tile) writes delta and dQ; launch 2 (one CTA per 64-key tile) writes dK and dV
cudaError_t launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype, int B,
                            int S, int H, int D, const void* mask, int mask_kind, int64_t mask_bstride,
                            const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                            cudaStream_t s, bool causal = false);

cudaError_t launch_attn_varlen_fwd(const void* qkv, int dtype, int T, int N, int H, int D, int max_seqlen,
                                   const int* cu_seqlens, const int64_t* seed, uint32_t keep, float scale, void* out,
                                   float* lse, cudaStream_t s, bool causal = false);
cudaError_t launch_attn_varlen_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype,
                                   int T, int N, int H, int D, int max_seqlen, const int* cu_seqlens,
                                   const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                                   cudaStream_t s, bool causal = false);

}  // namespace bps
