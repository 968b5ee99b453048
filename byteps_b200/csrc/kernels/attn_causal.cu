// The causal instantiations of the padded (attn_kernels.cuh) and packed (attn_varlen_kernels.cuh) attention kernels,
// launched by launch_attn_{fwd,bwd} and launch_attn_varlen_{fwd,bwd} with causal = true.  A translation unit of their
// own, so attn.cu and attn_varlen.cu keep only the bidirectional kernels.
#include "kernels/attn_kernels.cuh"
#include "kernels/attn_varlen_kernels.cuh"

namespace bps {

cudaError_t attn_causal_fwd(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return fwd<true>(a, grid, bf, drop, s);
}
cudaError_t attn_causal_bwd_dq(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return bwd_dq<true>(a, grid, bf, drop, s);
}
cudaError_t attn_causal_bwd_dkv(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return bwd_dkv<true>(a, grid, bf, drop, s);
}

cudaError_t attn_varlen_causal_fwd(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return fwd<true>(a, grid, bf, drop, s);
}
cudaError_t attn_varlen_causal_bwd_dq(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return bwd_dq<true>(a, grid, bf, drop, s);
}
cudaError_t attn_varlen_causal_bwd_dkv(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  return bwd_dkv<true>(a, grid, bf, drop, s);
}

}  // namespace bps
