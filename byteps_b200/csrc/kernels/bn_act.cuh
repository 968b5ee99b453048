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
cudaError_t launch_bn_act_bwd_apply(const void* dy, const void* x, const uint8_t* mask, int dtype, size_t M, int C,
                                    const float* mean, const float* invstd, const float* weight, const float* dweight,
                                    const float* dbias, void* dx, void* dresidual, cudaStream_t s);

}  // namespace bps
