// Element-wise stages of the GPU gradient compressors.
//
// The reference compresses on the CPU after a D2H copy and exchanges through the server
// (byteps/common/compressor/impl/*.cc, server.cc:92-118).  Here the payloads are exchanged through
// the symmetric arena by the kernels of compress_fused.cu (launch_payload_push, then a sum over the
// local slots).  This file holds the stages those kernels do not fuse: the error-feedback
// correction (with bit-reproducible norms), the dithering quantiser and unpacker, the random-k
// scatter and the cast to the user dtype.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bps {

// user dtype codes follow WireDType (0 f32, 1 bf16, 2 f16)

// corrected = g (+ nesterov momentum) + ratio*err (fp32, written to `corrected`); acc[0] = sum|corrected|,
// acc[1] = sum corrected^2, acc[2] = max|corrected|, computed with a fixed reduction order (bit-reproducible on
// every rank).  Momentum (mom non-null, fp32): m = mu*m + g ; corrected = g + mu*m, so g is only read.
// acc must hold kEfAccFloats floats (results + per-block partials).  err may be null (ratio ignored).
constexpr int kEfAccFloats = 4 + 3 * 132 * 8;
cudaError_t launch_ef_correct(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                              float* corrected, size_t n, float* acc, cudaStream_t s);

// ---- random-k
// out (zeroed by this call) [idx[j]] = mult * vals[j]   (later duplicates win, like the reference)
cudaError_t launch_index_scatter(const uint32_t* idx, const float* vals, uint32_t k, size_t n, void* out, int dtype,
                                 float mult, cudaStream_t s);

// ---- dithering (GPU contract: counter-based RNG, dense int8 levels)
// payload = [n int8 signed levels][float scale]; normalize 0 = max, 1 = l2; partition 0 = linear (s levels),
// 1 = natural (powers of two up to 2^(s-1))
cudaError_t launch_dither_quantize(const float* corrected, size_t n, const float* acc, int s_levels, int partition,
                                   int normalize, uint64_t seed, uint64_t step, int8_t* levels, float* scale_out,
                                   float* err_out, cudaStream_t s);
cudaError_t launch_dither_unpack(const int8_t* levels, const float* scale, size_t n, int s_levels, int partition,
                                 void* out, int dtype, float mult, cudaStream_t s);

// out = mult * in (fp32 -> user dtype)
cudaError_t launch_cast_scale(const float* in, size_t n, void* out, int dtype, float mult, cudaStream_t s);

}  // namespace bps
