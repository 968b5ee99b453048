// Kernels of the fused self-attention over packed variable-length sequences (see attn.cuh), templated on the causal
// mask.  attn_varlen.cu instantiates the bidirectional kernels and attn_causal.cu the causal ones.
//
// The kernels are those of attn_kernels.cuh with one (sequence, head) in place of one (batch, head): CTA (x, h, n)
// runs the 64-row tile x of sequence n, whose rows are tokens [cu[n], cu[n + 1]) of the stream.  Keys past the
// sequence's length are masked and its rows past the length read as zero, so a sequence behaves as one padded batch
// row whose length is its own.  Sequence offsets come from device memory and are clamped into [0, T) before any
// address is formed from them.  Under the causal mask the tiles run as in attn_kernels.cuh, with the query and key
// indices taken as positions within the sequence.
#pragma once
#include "kernels/attn_tile.cuh"

namespace bps {

struct AttnVArgs {
  const uint16_t *qkv, *out, *dout;
  const int* cu;
  const int64_t* seed;
  uint16_t *o, *dqkv;
  float *lse, *delta;
  int T, H, N, max_seqlen;
  uint32_t keep;
  float scale;
};

// the causal forms of fwd / bwd_dq / bwd_dkv below, instantiated in attn_causal.cu
cudaError_t attn_varlen_causal_fwd(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);
cudaError_t attn_varlen_causal_bwd_dq(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);
cudaError_t attn_varlen_causal_bwd_dkv(const AttnVArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s);

namespace {

using VArgs = AttnVArgs;

constexpr int kVFwdSmem = 5 * kTileBytes;                   // Q, K x 2, V x 2
constexpr int kVDqSmem = 6 * kTileBytes;                    // Q, dO, K x 2, V x 2
constexpr int kVDkvSmem = 6 * kTileBytes + 4 * kTile * 4;   // K, V, Q x 2, dO x 2, lse x 2, delta x 2

__device__ __forceinline__ int clamp_row(int r, int T) { return min(max(r, 0), T); }

// The token rows of the CTA's sequence, [x, x + y), clamped into [0, T); offsets out of order give an empty one.
__device__ __forceinline__ int2 seq_rows(const VArgs& a) {
  const int lo = clamp_row(a.cu[blockIdx.z], a.T), hi = clamp_row(a.cu[blockIdx.z + 1], a.T);
  return make_int2(lo, max(hi - lo, 0));
}

// Calls f(row, chunk) for the eight 16-byte chunks of a head's 64 columns in rows [r0, r1), spread over the CTAs
// along x.  It covers the rows no tile owns: those outside every sequence, and every row of a sequence longer than
// max_seqlen.
template <class F>
__device__ __forceinline__ void for_rows(int r0, int r1, F f) {
  for (int r = r0 + blockIdx.x * 16 + (threadIdx.x >> 3); r < r1; r += gridDim.x * 16) f(r, threadIdx.x & 7);
}

// Runs fill(r0, r1, nan) on the rows the tiles do not write: the CTAs of sequence 0 and N - 1 own the rows before
// cu[0] and from cu[N] on (zero), and a sequence longer than max_seqlen gets NaN in all its rows.  Returns whether
// the sequence is too long, in which case the CTA has nothing else to do.
template <class F>
__device__ __forceinline__ bool fill_untiled(const VArgs& a, int2 sq, F fill) {
  if (blockIdx.z == 0) fill(0, clamp_row(a.cu[0], a.T), false);
  if (blockIdx.z == a.N - 1) fill(clamp_row(a.cu[a.N], a.T), a.T, false);
  if (sq.y <= a.max_seqlen) return false;
  fill(sq.x, sq.x + sq.y, true);
  return true;
}

template <bool BF>
__device__ __forceinline__ uint4 fill16(bool nan) {
  const uint32_t w = nan ? (BF ? 0x7fc07fc0u : 0x7e007e00u) : 0u;
  return make_uint4(w, w, w, w);
}

template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_varlen_fwd_kernel(VArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sq = smem_u32(smem), sk = sq + kTileBytes, sv = sq + 3 * kTileBytes;
  const int T = a.T, H = a.H, E = H * kTile, h = blockIdx.y, qx = query_tile<CAUSAL>(), q0 = qx * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E;
  uint16_t* og = a.o + h * kTile;
  float* lg = a.lse + (size_t)h * T;
  const int2 rows = seq_rows(a);
  if (fill_untiled(a, rows, [&](int r0, int r1, bool nan) {
        for_rows(r0, r1, [&](int r, int c) {
          *reinterpret_cast<uint4*>(og + (size_t)r * E + c * 8) = fill16<BF>(nan);
          if (c == 0) lg[r] = nan ? NAN : INFINITY;
        });
      }))
    return;
  const int S = rows.y;
  if (q0 >= S) return;
  const uint16_t* qg = a.qkv + (size_t)rows.x * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const int nk = CAUSAL ? qx + 1 : (S + kTile - 1) / kTile;

  load_tile(sq, qg, ld, q0, S);
  load_tile(sk, kg, ld, 0, S);
  load_tile(sv, vg, ld, 0, S);
  cp_commit();
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  const uint64_t run_i =
      ((uint64_t)h * T + rows.x + q0 + warp * 16 + (lane >> 1)) * kAttnMaxSeq + 32 * (lane & 1);

  float o[8][4], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};
#pragma unroll
  for (int n = 0; n < 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) {
      load_tile(sk + (buf ^ 1) * kTileBytes, kg, ld, (kt + 1) * kTile, S);
      load_tile(sv + (buf ^ 1) * kTileBytes, vg, ld, (kt + 1) * kTile, S);
      cp_commit();
      cp_wait<1>();
    } else {
      cp_wait<0>();
    }
    __syncthreads();
    float s[8][4];
#pragma unroll
    for (int n = 0; n < 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    gemm_abt<BF>(s, sq, warp * 16, sk + buf * kTileBytes);
    const int kend = S - kt * kTile;   // keys of this tile inside the sequence
    const bool diag = CAUSAL && kt == qx;
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[n][j] = fmaf(s[n][j], kScaleLog2, n * 8 + 2 * t + (j & 1) < kend ? 0.f : -INFINITY);
        if (diag && above_diagonal(warp * 16 + g + 8 * (j >> 1), n * 8 + 2 * t + (j & 1))) s[n][j] = -INFINITY;
        mx[j >> 1] = fmaxf(mx[j >> 1], s[n][j]);
      }
    }
    float mu[2], alpha[2];
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
      mu[r] = mx[r] == -INFINITY ? 0.f : mx[r];
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
    uint16_t* dst = og + (size_t)(rows.x + q) * E + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(o[n][2 * r] * inv, o[n][2 * r + 1] * inv);
    if (t == 0) lg[rows.x + q] = l[r] > 0.f ? (m[r] + log2f(l[r])) * kLn2 : INFINITY;
  }
}

// delta = rowsum(dout * out) and dQ = dS K / 8 of one query tile, with dS = P * (dropout'(dO V^T) - delta)
template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_varlen_bwd_dq_kernel(VArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  const uint32_t sq = smem_u32(smem), sdo = sq + kTileBytes, sk = sq + 2 * kTileBytes, sv = sq + 4 * kTileBytes;
  const int T = a.T, H = a.H, E = H * kTile, h = blockIdx.y, qx = query_tile<CAUSAL>(), q0 = qx * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E, ht = (size_t)h * T;
  uint16_t* dqg = a.dqkv + h * kTile;
  const int2 rows = seq_rows(a);
  if (fill_untiled(a, rows, [&](int r0, int r1, bool nan) {
        for_rows(r0, r1, [&](int r, int c) {
          *reinterpret_cast<uint4*>(dqg + (size_t)r * ld + c * 8) = fill16<BF>(nan);
        });
      }))
    return;
  const int S = rows.y;
  if (q0 >= S) return;
  const uint16_t* qg = a.qkv + (size_t)rows.x * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const size_t obase = (size_t)rows.x * E + h * kTile, sbase = ht + rows.x;
  const int nk = CAUSAL ? qx + 1 : (S + kTile - 1) / kTile;

  load_tile(sq, qg, ld, q0, S);
  load_tile(sdo, a.dout + obase, E, q0, S);
  load_tile(sk, kg, ld, 0, S);
  load_tile(sv, vg, ld, 0, S);
  cp_commit();
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  const uint64_t run_i = ((uint64_t)sbase + q0 + warp * 16 + (lane >> 1)) * kAttnMaxSeq + 32 * (lane & 1);

  // delta of row warp * 16 + lane / 2, two lanes per row
  float dsum = 0.f;
  const int qd = q0 + warp * 16 + (lane >> 1);
  if (qd < S) {
    const size_t e = obase + (size_t)qd * E + 32 * (lane & 1);
#pragma unroll
    for (int v = 0; v < 4; ++v) dsum += dot8<BF>(a.out + e + 8 * v, a.dout + e + 8 * v);
  }
  dsum += __shfl_xor_sync(0xffffffffu, dsum, 1);
  if ((lane & 1) == 0 && qd < S) a.delta[sbase + qd] = dsum;
  float dl[2], lr[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) {
    const int q = q0 + warp * 16 + g + 8 * r;
    dl[r] = __shfl_sync(0xffffffffu, dsum, 2 * (g + 8 * r));
    lr[r] = q < S ? a.lse[sbase + q] * kLog2e : INFINITY;
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
    const int kend = S - kt * kTile;
    const bool diag = CAUSAL && kt == qx;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float mk = n * 8 + 2 * t + (j & 1) < kend ? 0.f : -INFINITY;
        float x = fmaf(s[n][j], kScaleLog2, mk);
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
    uint16_t* dst = dqg + (size_t)(rows.x + q) * ld + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(dq[n][2 * r] * 0.125f, dq[n][2 * r + 1] * 0.125f);
  }
}

// dK = dS^T Q / 8 and dV = dropout(P)^T dO of one key tile, over the query tiles in order
template <bool BF, bool DROP, bool CAUSAL>
__global__ void __launch_bounds__(kThreads) attn_varlen_bwd_dkv_kernel(VArgs a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* ls = reinterpret_cast<float*>(smem + 6 * kTileBytes);   // [2][64] lse * log2(e) of the query tile
  float* dls = ls + 2 * kTile;                                    // [2][64] delta of the query tile
  const uint32_t sk = smem_u32(smem), sv = sk + kTileBytes, sq = sk + 2 * kTileBytes, sdo = sk + 4 * kTileBytes;
  const int T = a.T, H = a.H, E = H * kTile, h = blockIdx.y, k0 = blockIdx.x * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E;
  uint16_t* dkg = a.dqkv + E + h * kTile;
  const int2 rows = seq_rows(a);
  if (fill_untiled(a, rows, [&](int r0, int r1, bool nan) {
        for_rows(r0, r1, [&](int r, int c) {
          uint16_t* dst = dkg + (size_t)r * ld + c * 8;
          *reinterpret_cast<uint4*>(dst) = fill16<BF>(nan);
          *reinterpret_cast<uint4*>(dst + E) = fill16<BF>(nan);
        });
      }))
    return;
  const int S = rows.y;
  if (k0 >= S) return;
  const size_t sbase = (size_t)h * T + rows.x;
  const uint16_t* qg = a.qkv + (size_t)rows.x * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E, *dog = a.dout + (size_t)rows.x * E + h * kTile;
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
    ls[b0 * kTile + threadIdx.x] = q < S ? a.lse[sbase + q] * kLog2e : INFINITY;
    dls[b0 * kTile + threadIdx.x] = q < S ? a.delta[sbase + q] : 0.f;
  }
  float km[2];
#pragma unroll
  for (int r = 0; r < 2; ++r) km[r] = k0 + warp * 16 + g + 8 * r < S ? 0.f : -INFINITY;
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (DROP) philox_key(a.seed, &key, &off);
  // lane l draws the keys of the warp's 16 for queries l and l + 32 of each tile
  const uint64_t run_i = ((uint64_t)sbase + lane) * kAttnMaxSeq + k0 + warp * 16;

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
        ls[(buf ^ 1) * kTile + threadIdx.x] = q < S ? a.lse[sbase + q] * kLog2e : INFINITY;
        dls[(buf ^ 1) * kTile + threadIdx.x] = q < S ? a.delta[sbase + q] : 0.f;
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
      const uint64_t i = run_i + (uint64_t)qt * kTile * kAttnMaxSeq;
      kb = keep_run<5>(key, off, i, a.keep) & 0xffffu;
      kb |= keep_run<5>(key, off, i + (uint64_t)32 * kAttnMaxSeq, a.keep) << 16;
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
    uint16_t* dst = dkg + (size_t)(rows.x + k) * ld + 2 * t;
#pragma unroll
    for (int n = 0; n < 8; ++n) {
      *reinterpret_cast<uint32_t*>(dst + n * 8) = pack2<BF>(dk[n][2 * r] * 0.125f, dk[n][2 * r + 1] * 0.125f);
      *reinterpret_cast<uint32_t*>(dst + E + n * 8) = pack2<BF>(dv[n][2 * r], dv[n][2 * r + 1]);
    }
  }
}

// ---- host side

template <bool CAUSAL>
cudaError_t fwd(const VArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_varlen_fwd_kernel, kVFwdSmem, CAUSAL)
}
template <bool CAUSAL>
cudaError_t bwd_dq(const VArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_varlen_bwd_dq_kernel, kVDqSmem, CAUSAL)
}
template <bool CAUSAL>
cudaError_t bwd_dkv(const VArgs& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_varlen_bwd_dkv_kernel, kVDkvSmem, CAUSAL)
}

}  // namespace

}  // namespace bps
