// Fused self-attention over packed variable-length sequences (see attn.cuh): the launchers, and the bidirectional
// instantiations of the kernels of attn_varlen_kernels.cuh.  The causal ones live in attn_causal.cu.
#include "kernels/attn_varlen_kernels.cuh"

namespace bps {

namespace {

bool aligned4(const void* p) { return ((uintptr_t)p & 3u) == 0; }

bool bad_args(int dtype, int T, int N, int H, int D, int max_seqlen, const int* cu) {
  return (dtype != WIRE_BF16 && dtype != WIRE_F16) || D != kAttnHeadDim || max_seqlen < 1 ||
         max_seqlen > kAttnMaxSeq || N < 1 || N > 65535 || H < 1 || H > 65535 || T < 1 || cu == nullptr ||
         !aligned4(cu);
}

VArgs make_args(const void* qkv, int T, int N, int H, int max_seqlen, const int* cu, const int64_t* seed,
                uint32_t keep, float scale) {
  VArgs a{};
  a.qkv = (const uint16_t*)qkv;
  a.cu = cu;
  a.seed = seed;
  a.T = T;
  a.H = H;
  a.N = N;
  a.max_seqlen = max_seqlen;
  a.keep = keep;
  a.scale = scale;
  return a;
}

dim3 grid_of(int N, int H, int max_seqlen) { return dim3((max_seqlen + kTile - 1) / kTile, H, N); }

}  // namespace

cudaError_t launch_attn_varlen_fwd(const void* qkv, int dtype, int T, int N, int H, int D, int max_seqlen,
                                   const int* cu_seqlens, const int64_t* seed, uint32_t keep, float scale, void* out,
                                   float* lse, cudaStream_t s, bool causal) {
  if (bad_args(dtype, T, N, H, D, max_seqlen, cu_seqlens) || qkv == nullptr || out == nullptr || lse == nullptr ||
      !aligned16(qkv) || !aligned16(out) || !aligned4(lse))
    return cudaErrorInvalidValue;
  VArgs a = make_args(qkv, T, N, H, max_seqlen, cu_seqlens, seed, keep, scale);
  a.o = (uint16_t*)out;
  a.lse = lse;
  const dim3 grid = grid_of(N, H, max_seqlen);
  const bool bf = dtype == WIRE_BF16, drop = seed != nullptr;
  return causal ? attn_varlen_causal_fwd(a, grid, bf, drop, s) : fwd<false>(a, grid, bf, drop, s);
}

cudaError_t launch_attn_varlen_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype,
                                   int T, int N, int H, int D, int max_seqlen, const int* cu_seqlens,
                                   const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                                   cudaStream_t s, bool causal) {
  if (bad_args(dtype, T, N, H, D, max_seqlen, cu_seqlens) || qkv == nullptr || out == nullptr || dout == nullptr ||
      lse == nullptr || delta == nullptr || dqkv == nullptr || !aligned16(qkv) || !aligned16(out) ||
      !aligned16(dout) || !aligned16(dqkv) || !aligned4(lse) || !aligned4(delta))
    return cudaErrorInvalidValue;
  VArgs a = make_args(qkv, T, N, H, max_seqlen, cu_seqlens, seed, keep, scale);
  a.out = (const uint16_t*)out;
  a.dout = (const uint16_t*)dout;
  a.lse = (float*)lse;
  a.delta = delta;
  a.dqkv = (uint16_t*)dqkv;
  const dim3 grid = grid_of(N, H, max_seqlen);
  const bool bf = dtype == WIRE_BF16, drop = seed != nullptr;
  const cudaError_t e =
      causal ? attn_varlen_causal_bwd_dq(a, grid, bf, drop, s) : bwd_dq<false>(a, grid, bf, drop, s);
  if (e != cudaSuccess) return e;
  return causal ? attn_varlen_causal_bwd_dkv(a, grid, bf, drop, s) : bwd_dkv<false>(a, grid, bf, drop, s);
}

}  // namespace bps
