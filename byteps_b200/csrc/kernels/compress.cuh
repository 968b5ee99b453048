// GPU gradient compression with fused error feedback, exchanged over NVLink.
//
// The reference compresses on the CPU (scalar / omp-simd loops) after a D2H copy
// and exchanges through the server (/root/reference/byteps/common/compressor/impl/*.cc,
// core_loops.cc:498-536,620-648, server.cc:92-118).  Here the compressors are
// device kernels, the payloads sit in the symmetric arena, and ONE kernel per
// compressor does "flag barrier -> read every peer's payload over NVLink ->
// decompress + sum".  Because every rank ends up holding every (tiny) payload,
// the reference's second, server-side compression of the sum is reproduced
// locally and redundantly instead of with another round trip.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels/peer_view.h"

namespace bps {

// user dtype codes follow WireDType (0 f32, 1 bf16, 2 f16)

// corrected = g + ratio*err (fp32, written to `corrected`); acc[0] = sum|corrected|, acc[1] = sum corrected^2,
// acc[2] = max|corrected|, computed with a fixed reduction order (bit-reproducible on every rank).
// acc must hold kEfAccFloats floats (results + per-block partials).  err may be null (ratio ignored).
constexpr int kEfAccFloats = 4 + 3 * 132 * 8;
cudaError_t launch_ef_correct(const void* g, int dtype, const float* err, float ratio, float* corrected, size_t n,
                              float* acc, cudaStream_t s);

// ---- onebit: payload = [ceil(n/32) words, 1 = negative, MSB first][float scale]
cudaError_t launch_onebit_pack(const float* corrected, size_t n, const float* acc, int use_scale, uint32_t* words,
                               float* err_out, cudaStream_t s);
// sum[i] = sum_p (+-scale_p) over all peers' payloads at arena offset `off`; barriers at both ends
cudaError_t launch_onebit_exchange_sum(const PeerView& pv, size_t off, size_t n, float* sum, int blocks, int channel,
                                       cudaStream_t s);
// out[i] = mult * (+-scale) from a local payload
cudaError_t launch_onebit_unpack(const uint32_t* words, size_t n, void* out, int dtype, float mult, cudaStream_t s);

// ---- top-k: payload = k x {uint32 index, float value}
// scratch: >= 1024 uint32.  Selects the k largest |corrected|; err_out (may be null) = corrected with the
// selected entries zeroed.
cudaError_t launch_topk_select(const float* corrected, size_t n, uint32_t k, uint32_t* pairs, float* err_out,
                               uint32_t* scratch, cudaStream_t s);
// sum must be zeroed; scatter-adds every peer's k pairs (payload at arena offset off); barriers at both ends
cudaError_t launch_sparse_exchange_sum(const PeerView& pv, size_t off, uint32_t k, size_t n, float* sum, int blocks,
                                       int channel, cudaStream_t s);
// sum[idx] += val for ONE payload (indices unique): launched once per peer between two barrier kernels, this
// gives a rank-independent summation order (the atomic variant above does not)
cudaError_t launch_sparse_add(const uint32_t* pairs, uint32_t k, size_t n, float* sum, cudaStream_t s);
// out (zeroed by this call) [idx] = mult * val
cudaError_t launch_sparse_scatter(const uint32_t* pairs, uint32_t k, size_t n, void* out, int dtype, float mult,
                                  cudaStream_t s);

// ---- random-k: all ranks draw the SAME indices (xorshift128+ stream identical to the CPU compressor)
// state: 2 x uint64 in device memory, advanced by the kernel
cudaError_t launch_randomk_indices(uint64_t* state, uint32_t k, size_t n, uint32_t* idx, cudaStream_t s);
// vals[j] = corrected[idx[j]]; err_out = corrected with idx zeroed
cudaError_t launch_randomk_gather(const float* corrected, const uint32_t* idx, uint32_t k, size_t n, float* vals,
                                  float* err_out, cudaStream_t s);
// dense sum of the k values of every peer (payload = k floats at off) -> vals_sum; barriers at both ends
cudaError_t launch_dense_exchange_sum(const PeerView& pv, size_t off, uint32_t k, float* vals_sum, int blocks,
                                      int channel, cudaStream_t s);
// out (zeroed by this call) [idx[j]] = mult * vals[j]   (later duplicates win, like the reference)
cudaError_t launch_index_scatter(const uint32_t* idx, const float* vals, uint32_t k, size_t n, void* out, int dtype,
                                 float mult, cudaStream_t s);

// ---- dithering (GPU contract: counter-based RNG, dense int8 levels)
// payload = [n int8 signed levels][float scale]; normalize 0 = max, 1 = l2; partition 0 = linear (s levels),
// 1 = natural (powers of two up to 2^(s-1))
cudaError_t launch_dither_quantize(const float* corrected, size_t n, const float* acc, int s_levels, int partition,
                                   int normalize, uint64_t seed, uint64_t step, int8_t* levels, float* scale_out,
                                   float* err_out, cudaStream_t s);
cudaError_t launch_dither_exchange_sum(const PeerView& pv, size_t off, size_t n, int s_levels, int partition,
                                       float* sum, int blocks, int channel, cudaStream_t s);
cudaError_t launch_dither_unpack(const int8_t* levels, const float* scale, size_t n, int s_levels, int partition,
                                 void* out, int dtype, float mult, cudaStream_t s);

// out = mult * in (fp32 -> user dtype)
cudaError_t launch_cast_scale(const float* in, size_t n, void* out, int dtype, float mult, cudaStream_t s);

// momentum (nesterov): m = mu*m + g ; g += mu*m   (g in user dtype, m fp32)
cudaError_t launch_nesterov(void* g, int dtype, float* m, float mu, size_t n, cudaStream_t s);

}  // namespace bps
