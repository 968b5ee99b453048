// ResNet's stem convolution, y = conv(x, w) with 3 input channels, 64 output channels, a 7x7 kernel, stride 2 and
// padding 3, on bf16 NHWC tensors, and its weight gradient.  The image needs no gradient, so there is no dgrad.
//
//   x   [N, H, W, 3] bf16, any 2-byte aligned address (rows of an odd W are not 16-byte aligned)
//   y   [N, OH, OW, 64] bf16 with OH = (H - 1) / 2 + 1, OW = (W - 1) / 2 + 1, 16-byte aligned
//   w   64 x 3 x 7 x 7 bf16, channels_last (co, kh, kw, c) when w_cl, else contiguous (co, c, kh, kw)
//
// fwd    one persistent launch; each output element is one fp32 mma accumulation over its 147 products, rounded once.
// wgrad  two launches: a persistent grid in which CTA b sums the pixels of its contiguous range of output-row
//        segments into partial b of ws (fp32 [P, 64, 147], (co, kh, kw, c)); then dW = the partials summed in the
//        order b = 0 .. P - 1, rounded once, written in w's layout.  dy is [N, OH, OW, 64], 16-byte aligned.
//        P = stem_conv_wgrad_partials(N, H, W) on the current device.  No atomics: results repeat bit for bit.
// Offsets are 64-bit; nothing is read on the host, so both capture into a CUDA graph.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace bps {

int stem_conv_wgrad_partials(int64_t N, int64_t H, int64_t W);
cudaError_t launch_stem_conv_fwd(const void* x, const void* w, bool w_cl, void* y, int64_t N, int64_t H, int64_t W,
                                 cudaStream_t s);
cudaError_t launch_stem_conv_wgrad(const void* x, const void* dy, float* ws, int partials, void* dw, bool w_cl,
                                   int64_t N, int64_t H, int64_t W, cudaStream_t s);

}  // namespace bps
