// Kernels of the padded fused self-attention (see attn.cuh), templated on the causal mask.  attn.cu instantiates the
// bidirectional kernels and attn_causal.cu the causal ones, each set in a translation unit of its own.
//
// Every launch runs 128 threads per CTA over one 64-row tile (queries for fwd and bwd_dq, keys for bwd_dkv) of one
// (head, batch); each warp owns 16 rows of it.  The other operand streams through shared memory in 64-row tiles,
// double-buffered with cp.async (rows past S are zero-filled), and the products run on mma.sync.m16n8k16 with fp32
// accumulators, fragments loaded with ldmatrix from XOR-swizzled tiles.  A 16 x 64 accumulator tile is reused from
// registers as the A operand of the next product after rounding to the activation dtype (P for P V, dS for dS K).
// Scores are kept in the exp2 domain: x = (q . k) * log2(e) / 8 + mask * log2(e).
//
// CAUSAL: key k attends to query q only when k <= q.  Forward and bwd_dq of query tile x visit key tiles 0 .. x, and
// bwd_dkv of key tile y visits query tiles y .. last; only the diagonal tile is masked element by element, its
// scores above the diagonal replaced by -inf.  The query tiles of fwd and bwd_dq run in reverse order of blockIdx.x,
// so the CTAs with the most key tiles start first.
#pragma once
#include "kernels/attn_tile.cuh"

namespace bps {

struct AttnArgs {
  const uint16_t *qkv, *out, *dout;
  const void* mask;
  const int64_t* seed;
  uint16_t *o, *dqkv;
  float *lse, *delta;
  int64_t mask_bstride;
  int S, H, mask_kind;
  uint32_t keep;
  float scale;
};

// the causal forms of fwd / bwd_dq / bwd_dkv below, instantiated in attn_causal.cu
cudaError_t attn_causal_fwd(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);
cudaError_t attn_causal_bwd_dq(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);
cudaError_t attn_causal_bwd_dkv(const AttnArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);

namespace {

using Args = AttnArgs;

constexpr int kFwdSmem = 5 * kTileBytes + 2 * kTile * 4;    // Q, K x 2, V x 2, key mask x 2
constexpr int kDqSmem = 6 * kTileBytes + 2 * kTile * 4;     // Q, dO, K x 2, V x 2, key mask x 2
constexpr int kDkvSmem = 6 * kTileBytes + 4 * kTile * 4;    // K, V, Q x 2, dO x 2, lse x 2, delta x 2

// the mask of key k of batch b times log2(e): -inf past the sequence and for a masked key
__device__ __forceinline__ float mask_l2(const Args& a, int b, int k) {
  if (k >= a.S) return -INFINITY;
  if (a.mask == nullptr) return 0.f;
  const size_t i = (size_t)b * a.mask_bstride + k;
  switch (a.mask_kind) {
    case ATTN_MASK_BOOL: return ((const uint8_t*)a.mask)[i] ? 0.f : -INFINITY;
    case ATTN_MASK_BF16: return __bfloat162float(((const __nv_bfloat16*)a.mask)[i]) * kLog2e;
    case ATTN_MASK_F16: return __half2float(((const __half*)a.mask)[i]) * kLog2e;
    default: return ((const float*)a.mask)[i] * kLog2e;
  }
}

template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* mk = reinterpret_cast<float*>(smem + 5 * kTileBytes);
  const uint32_t sq = smem_u32(smem), sk = sq + kTileBytes, sv = sq + 3 * kTileBytes;
  const int qx = query_tile<CAUSAL>();
  const int S = a.S, H = a.H, E = H * kTile, b = blockIdx.z, h = blockIdx.y, q0 = qx * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E;
  const uint16_t* qg = a.qkv + (size_t)b * S * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const int nk = CAUSAL ? qx + 1 : (S + kTile - 1) / kTile;

  load_tile(sq, qg, ld, q0, S);
  load_tile(sk, kg, ld, 0, S);
  load_tile(sv, vg, ld, 0, S);
  cp_commit();
  if (threadIdx.x < kTile) mk[threadIdx.x] = mask_l2(a, b, threadIdx.x);
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  const uint64_t run_i = ((uint64_t)(b * H + h) * S + q0 + warp * 16 + (lane >> 1)) * S + 32 * (lane & 1);

  float o[8][4], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      load_tile(sk + (buf ^ 1) * kTileBytes, kg, ld, (kt + 1) * kTile, S);
      load_tile(sv + (buf ^ 1) * kTileBytes, vg, ld, (kt + 1) * kTile, S);
      cp_commit();
      if (threadIdx.x < kTile) mk[(buf ^ 1) * kTile + threadIdx.x] = mask_l2(a, b, (kt + 1) * kTile + threadIdx.x);
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    gemm_abt<BF>(s, sq, warp * 16, sk + buf * kTileBytes);
    const float* mrow = mk + buf * kTile;
    const bool diag = CAUSAL && kt == qx;
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[n][j] = fmaf(s[n][j], kScaleLog2, mrow[n * 8 + 2 * t + (j & 1)]);
        if (diag && above_diagonal(warp * 16 + g + 8 * (j >> 1), n * 8 + 2 * t + (j & 1))) s[n][j] = -INFINITY;
        mx[j >> 1] = fmaxf(mx[j >> 1], s[n][j]);
      }
    }
    float mu[2], alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      mu[r] = mx[r] == -INFINITY ? 0.f : mx[r];   // a row masked so far stays all zero
      alpha[r] = exp2f(m[r] - mu[r]);
      m[r] = mx[r];
      l[r] *= alpha[r];
    }
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[n][j] = exp2f(s[n][j] - mu[j >> 1]);
        l[j >> 1] += s[n][j];
        o[n][j] *= alpha[j >> 1];
      }
    }
    if (DROP) {
      uint32_t w[2][2];
      row_keep_bits(key, off, run_i + (uint64_t)kt * kTile, a.keep, w);
#pragma unroll
      for (int n = 0; n < 8; ++n) {
#pragma unroll
        for (int j = 0; j < 4; ++j) s[n][j] = row_kept(w, n, j) ? s[n][j] : 0.f;
      }
    }
    uint32_t pa[4][4];
    to_a<BF>(pa, s);
    gemm_pb<BF>(o, pa, sv + buf * kTileBytes);
    __syncthreads();
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 1);
    l[r] += __shfl_xor_sync(0xffffffffu, l[r], 2);
    const int q = q0 + warp * 16 + g + 8 * r;
    if (q >= S) continue;
    const float inv = l[r] > 0.f ? a.scale / l[r] : 0.f;
    uint16_t* dst = a.o + ((size_t)b * S + q) * E + h * kTile + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(o[n][2 * r] * inv, o[n][2 * r + 1] * inv);
    if (t == 0) a.lse[((size_t)b * H + h) * S + q] = l[r] > 0.f ? (m[r] + log2f(l[r])) * kLn2 : INFINITY;
  }
}

// delta = rowsum(dout * out) and dQ = dS K / 8 of one query tile, with dS = P * (dropout'(dO V^T) - delta)
template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* mk = reinterpret_cast<float*>(smem + 6 * kTileBytes);
  const uint32_t sq = smem_u32(smem), sdo = sq + kTileBytes, sk = sq + 2 * kTileBytes, sv = sq + 4 * kTileBytes;
  const int qx = query_tile<CAUSAL>();
  const int S = a.S, H = a.H, E = H * kTile, b = blockIdx.z, h = blockIdx.y, q0 = qx * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E, bh = (size_t)b * H + h;
  const uint16_t* qg = a.qkv + (size_t)b * S * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const size_t obase = (size_t)b * S * E + h * kTile;
  const int nk = CAUSAL ? qx + 1 : (S + kTile - 1) / kTile;

  load_tile(sq, qg, ld, q0, S);
  load_tile(sdo, a.dout + obase, E, q0, S);
  load_tile(sk, kg, ld, 0, S);
  load_tile(sv, vg, ld, 0, S);
  cp_commit();
  if (threadIdx.x < kTile) mk[threadIdx.x] = mask_l2(a, b, threadIdx.x);
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  const uint64_t run_i = ((uint64_t)bh * S + q0 + warp * 16 + (lane >> 1)) * S + 32 * (lane & 1);

  // delta of row warp * 16 + lane / 2, two lanes per row
  float dsum = 0.f;
  const int qd = q0 + warp * 16 + (lane >> 1);
  if (qd < S) {
    const size_t e = obase + (size_t)qd * E + 32 * (lane & 1);
#pragma unroll
    for (int v = 0; v < 4; ++v) dsum += dot8<BF>(a.out + e + 8 * v, a.dout + e + 8 * v);
  }
  dsum += __shfl_xor_sync(0xffffffffu, dsum, 1);
  if ((lane & 1) == 0 && qd < S) a.delta[bh * S + qd] = dsum;
  float dl[2], lr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + warp * 16 + g + 8 * r;
    dl[r] = __shfl_sync(0xffffffffu, dsum, 2 * (g + 8 * r));
    lr[r] = q < S ? a.lse[bh * S + q] * kLog2e : INFINITY;
  }

  float dq[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) dq[n][0] = dq[n][1] = dq[n][2] = dq[n][3] = 0.f;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      load_tile(sk + (buf ^ 1) * kTileBytes, kg, ld, (kt + 1) * kTile, S);
      load_tile(sv + (buf ^ 1) * kTileBytes, vg, ld, (kt + 1) * kTile, S);
      cp_commit();
      if (threadIdx.x < kTile) mk[(buf ^ 1) * kTile + threadIdx.x] = mask_l2(a, b, (kt + 1) * kTile + threadIdx.x);
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s[n][j] = dp[n][j] = 0.f;
    }
    gemm_abt<BF>(s, sq, warp * 16, sk + buf * kTileBytes);
    gemm_abt<BF>(dp, sdo, warp * 16, sv + buf * kTileBytes);
    uint32_t w[2][2];
    if (DROP) row_keep_bits(key, off, run_i + (uint64_t)kt * kTile, a.keep, w);
    const float* mrow = mk + buf * kTile;
    const bool diag = CAUSAL && kt == qx;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        float x = fmaf(s[n][j], kScaleLog2, mrow[n * 8 + 2 * t + (j & 1)]);
        if (diag && above_diagonal(warp * 16 + g + 8 * (j >> 1), n * 8 + 2 * t + (j & 1))) x = -INFINITY;
        const float p = exp2f(x - lr[j >> 1]);
        const float d = (!DROP || row_kept(w, n, j)) ? dp[n][j] * a.scale : 0.f;
        s[n][j] = p * (d - dl[j >> 1]);
      }
    }
    uint32_t pa[4][4];
    to_a<BF>(pa, s);
    gemm_pb<BF>(dq, pa, sk + buf * kTileBytes);
    __syncthreads();
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + warp * 16 + g + 8 * r;
    if (q >= S) continue;
    uint16_t* dst = a.dqkv + ((size_t)b * S + q) * ld + h * kTile + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(dq[n][2 * r] * 0.125f, dq[n][2 * r + 1] * 0.125f);
  }
}

// dK = dS^T Q / 8 and dV = dropout(P)^T dO of one key tile, over the query tiles in order
template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_bwd_dkv_kernel(Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* ls = reinterpret_cast<float*>(smem + 6 * kTileBytes);   // [2][64] lse * log2(e) of the query tile
  float* dls = ls + 2 * kTile;                                    // [2][64] delta of the query tile
  const uint32_t sk = smem_u32(smem), sv = sk + kTileBytes, sq = sk + 2 * kTileBytes, sdo = sk + 4 * kTileBytes;
  const int S = a.S, H = a.H, E = H * kTile, b = blockIdx.z, h = blockIdx.y, k0 = blockIdx.x * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E, bh = (size_t)b * H + h;
  const uint16_t* qg = a.qkv + (size_t)b * S * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E, *dog = a.dout + (size_t)b * S * E + h * kTile;
  const int nq = (S + kTile - 1) / kTile;
  // the first query tile, staged in buffer qt0 & 1 as the loop expects
  const int qt0 = CAUSAL ? (int)blockIdx.x : 0, b0 = qt0 & 1;

  load_tile(sk, kg, ld, k0, S);
  load_tile(sv, vg, ld, k0, S);
  load_tile(sq + b0 * kTileBytes, qg, ld, qt0 * kTile, S);
  load_tile(sdo + b0 * kTileBytes, dog, E, qt0 * kTile, S);
  cp_commit();
  if (threadIdx.x < kTile) {
    const int q = qt0 * kTile + threadIdx.x;
    ls[b0 * kTile + threadIdx.x] = q < S ? a.lse[bh * S + q] * kLog2e : INFINITY;
    dls[b0 * kTile + threadIdx.x] = q < S ? a.delta[bh * S + q] : 0.f;
  }
  float km[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) km[r] = mask_l2(a, b, k0 + warp * 16 + g + 8 * r);
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  // lane l draws the keys of the warp's 16 for queries l and l + 32 of each tile
  const uint64_t run_i = ((uint64_t)bh * S + lane) * S + k0 + warp * 16;

  float dk[8][4], dv[8][4];
#pragma unroll
  for (int n = 0; n < 8; ++n) {
#pragma unroll
    for (int j = 0; j < 4; ++j) dk[n][j] = dv[n][j] = 0.f;
  }
  for (int qt = qt0; qt < nq; ++qt) {
    const int buf = qt & 1;
    if (qt + 1 < nq) {
      load_tile(sq + (buf ^ 1) * kTileBytes, qg, ld, (qt + 1) * kTile, S);
      load_tile(sdo + (buf ^ 1) * kTileBytes, dog, E, (qt + 1) * kTile, S);
      cp_commit();
      if (threadIdx.x < kTile) {
        const int q = (qt + 1) * kTile + threadIdx.x;
        ls[(buf ^ 1) * kTile + threadIdx.x] = q < S ? a.lse[bh * S + q] * kLog2e : INFINITY;
        dls[(buf ^ 1) * kTile + threadIdx.x] = q < S ? a.delta[bh * S + q] : 0.f;
      }
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    float s[8][4], dp[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) s[n][j] = dp[n][j] = 0.f;
    }
    gemm_abt<BF>(s, sk, warp * 16, sq + buf * kTileBytes);    // S^T: rows keys, columns queries
    gemm_abt<BF>(dp, sv, warp * 16, sdo + buf * kTileBytes);  // (dO V^T)^T
    uint32_t kb = 0;
    if (DROP) {
      const uint64_t i = run_i + (uint64_t)qt * kTile * S;
      kb = keep_run<5>(key, off, i, a.keep) & 0xffffu;
      kb |= keep_run<5>(key, off, i + (uint64_t)32 * S, a.keep) << 16;
    }
    const float* lrow = ls + buf * kTile;
    const float* drow = dls + buf * kTile;
    const bool diag = CAUSAL && qt == qt0;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const int col = n * 8 + 2 * t + c;
        const uint32_t bits = DROP ? __shfl_sync(0xffffffffu, kb, col & 31) >> (16 * (n >> 2)) : 0xffffu;
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int j = 2 * r + c;
          const bool kept = !DROP || ((bits >> (g + 8 * r)) & 1u);
          float x = fmaf(s[n][j], kScaleLog2, km[r]);
          if (diag && above_diagonal(col, warp * 16 + g + 8 * r)) x = -INFINITY;   // key after query
          const float p = exp2f(x - lrow[col]);
          const float d = kept ? dp[n][j] * a.scale : 0.f;
          s[n][j] = p * (d - drow[col]);
          dp[n][j] = kept ? p * a.scale : 0.f;
        }
      }
    }
    uint32_t pa[4][4];
    to_a<BF>(pa, dp);
    gemm_pb<BF>(dv, pa, sdo + buf * kTileBytes);
    to_a<BF>(pa, s);
    gemm_pb<BF>(dk, pa, sq + buf * kTileBytes);
    __syncthreads();
  }

#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int k = k0 + warp * 16 + g + 8 * r;
    if (k >= S) continue;
    uint16_t* dst = a.dqkv + ((size_t)b * S + k) * ld + E + h * kTile + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(dk[n][2 * r] * 0.125f, dk[n][2 * r + 1] * 0.125f);
      *reinterpret_cast<uint32_t*>(dst + E + n * 8) = pack2<BF>(dv[n][2 * r], dv[n][2 * r + 1]);
    }
  }
}

// ---- host side

template <bool CAUSAL>
cudaError_t fwd(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_fwd_kernel, kFwdSmem, CAUSAL)
}
template <bool CAUSAL>
cudaError_t bwd_dq(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_bwd_dq_kernel, kDqSmem, CAUSAL)
}
template <bool CAUSAL>
cudaError_t bwd_dkv(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_bwd_dkv_kernel, kDkvSmem, CAUSAL)
}

}  // namespace

}  // namespace bps
