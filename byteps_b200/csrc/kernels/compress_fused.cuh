// Host-visible API of the fused GPU compressors (compress_fused.cu).
//
// Payload windows: every rank owns, inside the symmetric arena, `world` slots of `slot_bytes`;
// rank r writes its payload into its own slot r locally, `launch_payload_push` copies it into slot
// r of every peer and ends in the cross-rank flag barrier, and the consuming kernels read the
// local slots only.  Windows are double buffered by the caller (step parity), so no trailing
// barrier is needed.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"

namespace bps {

constexpr int kFusedMaxBlocks = 132 * 8;          // also the size of the per-block partial arrays
constexpr int kTopkScratchBytes = 4096 * 4 + 64 + 32768 * 4;

// ---- onebit (+ nesterov momentum, + vanilla error feedback with the lr ratio) -------------------
// producer: p = g [+ mu * (mu*mom + g)] [+ ratio * err]; p_out (may alias err, may be null) = p;
// words[ceil(n/32)] = sign bits (1 = negative, first element in the most significant bit) followed
// by one float: mean|p| (use_scale) or 1.  parts: kFusedMaxBlocks floats, counter: one zeroed u32.
cudaError_t launch_onebit_pre(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                              float* p_out, size_t n, uint32_t* words, int use_scale, float* parts, uint32_t* counter,
                              cudaStream_t s);
// consumer pass A over the `world` local slots:
//   s = sum_p D(payload_p);   err (if given, holding p) <- p - D(C(p))
//   two-stage (c2_out != null): c2_out = s [+ err2]; scale2_out = mean|c2| (or 1)
//   one-stage (c2_out == null): out = mult * s  (user dtype)
cudaError_t launch_onebit_sum(const void* slots, size_t slot_bytes, int world, int me, size_t n, float* err,
                              const float* err2, float* c2_out, void* out, int dtype, float mult, int use_scale2,
                              float* parts, uint32_t* counter, float* scale2_out, cudaStream_t s);
// consumer pass B (two-stage): out = mult * sign(c2) * scale2; err2 (if given) = c2 - sign(c2) * scale2
cudaError_t launch_onebit_out(const float* c2, size_t n, const float* scale2, float* err2, void* out, int dtype,
                              float mult, cudaStream_t s);

// ---- payload push + barrier ------------------------------------------------------------------------
cudaError_t launch_payload_push(const PeerView& pv, size_t win_off, size_t slot_bytes, size_t bytes, int blocks,
                                int channel, cudaStream_t s);

// ---- top-k ------------------------------------------------------------------------------------------
// producer: p -> p_out (fp32, required; may alias err) and the first radix histogram in `scratch`
// (kTopkScratchBytes of device memory)
cudaError_t launch_topk_pre(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                            float* p_out, size_t n, uint32_t k, void* scratch, cudaStream_t s);
// remaining radix levels (first_level = 1 after launch_topk_pre, 0 for a plain fp32 tensor) + compaction:
// pairs[k] = {index, value}; the kept entries of x are zeroed when zero_kept (the error-feedback update)
cudaError_t launch_topk_finish(float* x, size_t n, uint32_t k, int first_level, uint32_t* pairs, int zero_kept,
                               void* scratch, cudaStream_t s);
// dst[idx] += val for one payload (unique indices)
cudaError_t launch_sparse_add_pairs(const uint32_t* pairs, uint32_t k, size_t n, float* dst, cudaStream_t s);
// out = 0; out[idx] = mult * val   (user dtype)
cudaError_t launch_scatter_pairs(const uint32_t* pairs, uint32_t k, size_t n, void* out, int dtype, float mult,
                                 cudaStream_t s);
cudaError_t launch_cast_scale4(const float* in, size_t n, void* out, int dtype, float mult, cudaStream_t s);

// ---- random-k -----------------------------------------------------------------------------------------
// idx[k] = the next k draws of xorshift128+ (state: 2 x u64 in device memory, advanced by k), computed in
// parallel with the jump matrices T^(2^j), j < 32 (32 x 128 rows x 2 u64, from the host)
cudaError_t launch_randomk_draw(uint64_t* state, const uint64_t* jump, uint32_t k, size_t n, uint32_t* idx,
                                cudaStream_t s);
// vals[j] = p[idx[j]]; momentum advanced, err = p with the drawn entries zeroed (when given)
cudaError_t launch_randomk_pre(const void* g, int dtype, float* mom, float mu, float* err, float ratio, size_t n,
                               const uint32_t* idx, uint32_t k, float* vals, cudaStream_t s);
// out[j] = sum over the local slots (k floats each), fixed order
cudaError_t launch_dense_sum_slots(const void* slots, size_t slot_bytes, int world, uint32_t k, float* out,
                                   cudaStream_t s);

// ---- dithering ------------------------------------------------------------------------------------------
// sum[i] = sum over the local slots of D(levels, scale) (payload format of compress.cu::dither_quantize)
cudaError_t launch_dither_sum_slots(const void* slots, size_t slot_bytes, int world, size_t n, int s_levels,
                                    int partition, float* sum, cudaStream_t s);

}  // namespace bps
