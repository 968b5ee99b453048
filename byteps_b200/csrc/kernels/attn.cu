// Fused self-attention over padded batches (see attn.cuh): the launchers, and the bidirectional instantiations of the
// kernels of attn_kernels.cuh.  The causal ones live in attn_causal.cu.
#include "kernels/attn_kernels.cuh"

namespace bps {

namespace {

bool bad_args(int dtype, int B, int S, int H, int D, const void* mask, int mask_kind, int64_t mask_bstride) {
  return (dtype != WIRE_BF16 && dtype != WIRE_F16) || D != kAttnHeadDim || S < 1 || S > kAttnMaxSeq || B < 1 ||
         B > 65535 || H < 1 || H > 65535 ||
         (mask != nullptr && (mask_kind < ATTN_MASK_F32 || mask_kind > ATTN_MASK_BOOL || mask_bstride < 0));
}

Args make_args(const void* qkv, int S, int H, const void* mask, int mask_kind, int64_t mask_bstride,
               const int64_t* seed, uint32_t keep, float scale) {
  Args a{};
  a.qkv = (const uint16_t*)qkv;
  a.mask = mask;
  a.seed = seed;
  a.mask_bstride = mask_bstride;
  a.S = S;
  a.H = H;
  a.mask_kind = mask_kind;
  a.keep = keep;
  a.scale = scale;
  return a;
}

}  // namespace

cudaError_t launch_attn_fwd(const void* qkv, int dtype, int B, int S, int H, int D, const void* mask, int mask_kind,
                            int64_t mask_bstride, const int64_t* seed, uint32_t keep, float scale, void* out,
                            float* lse, cudaStream_t s, bool causal) {
  if (bad_args(dtype, B, S, H, D, mask, mask_kind, mask_bstride) || qkv == nullptr || out == nullptr ||
      lse == nullptr || !aligned16(qkv) || !aligned16(out))
    return cudaErrorInvalidValue;
  Args a = make_args(qkv, S, H, mask, mask_kind, mask_bstride, seed, keep, scale);
  a.o = (uint16_t*)out;
  a.lse = lse;
  const dim3 grid((S + kTile - 1) / kTile, H, B);
  const bool bf = dtype == WIRE_BF16, drop = seed != nullptr;
  return causal ? attn_causal_fwd(a, grid, bf, drop, s) : fwd<false>(a, grid, bf, drop, s);
}

cudaError_t launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype, int B,
                            int S, int H, int D, const void* mask, int mask_kind, int64_t mask_bstride,
                            const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                            cudaStream_t s, bool causal) {
  if (bad_args(dtype, B, S, H, D, mask, mask_kind, mask_bstride) || qkv == nullptr || out == nullptr ||
      dout == nullptr || lse == nullptr || delta == nullptr || dqkv == nullptr || !aligned16(qkv) ||
      !aligned16(out) || !aligned16(dout) || !aligned16(dqkv))
    return cudaErrorInvalidValue;
  Args a = make_args(qkv, S, H, mask, mask_kind, mask_bstride, seed, keep, scale);
  a.out = (const uint16_t*)out;
  a.dout = (const uint16_t*)dout;
  a.lse = (float*)lse;
  a.delta = delta;
  a.dqkv = (uint16_t*)dqkv;
  const dim3 grid((S + kTile - 1) / kTile, H, B);
  const bool bf = dtype == WIRE_BF16, drop = seed != nullptr;
  const cudaError_t e = causal ? attn_causal_bwd_dq(a, grid, bf, drop, s) : bwd_dq<false>(a, grid, bf, drop, s);
  if (e != cudaSuccess) return e;
  return causal ? attn_causal_bwd_dkv(a, grid, bf, drop, s) : bwd_dkv<false>(a, grid, bf, drop, s);
}

}  // namespace bps
