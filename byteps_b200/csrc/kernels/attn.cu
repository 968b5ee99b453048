// Fused self-attention of the BERT encoder (see attn.cuh).
//
// Every launch runs 128 threads per CTA over one 64-row tile (queries for fwd and bwd_dq, keys for bwd_dkv) of one
// (head, batch); each warp owns 16 rows of it.  The other operand streams through shared memory in 64-row tiles,
// double-buffered with cp.async (rows past S are zero-filled), and the products run on mma.sync.m16n8k16 with fp32
// accumulators, fragments loaded with ldmatrix from XOR-swizzled tiles.  A 16 x 64 accumulator tile is reused from
// registers as the A operand of the next product after rounding to the activation dtype (P for P V, dS for dS K).
// Scores are kept in the exp2 domain: x = (q . k) * log2(e) / 8 + mask * log2(e).
#include "kernels/attn.cuh"

#include <type_traits>

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kTile = 64;   // rows of a tile, and the head dimension
constexpr int kThreads = 128;
constexpr uint32_t kTileBytes = kTile * kTile * 2;
constexpr float kLog2e = 1.4426950408889634f;
constexpr float kLn2 = 0.6931471805599453f;
constexpr float kScaleLog2 = 0.125f * kLog2e;
constexpr int kMaxDevices = 64;
constexpr int kFwdSmem = 5 * kTileBytes + 2 * kTile * 4;    // Q, K x 2, V x 2, key mask x 2
constexpr int kDqSmem = 6 * kTileBytes + 2 * kTile * 4;     // Q, dO, K x 2, V x 2, key mask x 2
constexpr int kDkvSmem = 6 * kTileBytes + 4 * kTile * 4;    // K, V, Q x 2, dO x 2, lse x 2, delta x 2

struct Args {
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

// byte offset of 16-byte chunk c of row r in a 64 x 64 tile of 16-bit elements; the chunks are XOR-swizzled by the
// row so the 8 rows one ldmatrix phase reads fall in distinct banks
__device__ __forceinline__ uint32_t swz(int r, int c) { return (uint32_t)(r * 128 + ((c ^ (r & 7)) << 4)); }

__device__ __forceinline__ void cp_async16(uint32_t dst, const void* src, bool ok) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(ok ? 16 : 0) : "memory");
}
__device__ __forceinline__ void cp_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// rows r0 .. r0 + 63 of a matrix of 64-element rows `ld` elements apart into the tile at dst; rows >= n read as zero
__device__ __forceinline__ void load_tile(uint32_t dst, const uint16_t* src, size_t ld, int r0, int n) {
#pragma unroll
  for (int i = 0; i < kTile * 8 / kThreads; ++i) {
    const int c = threadIdx.x + i * kThreads, r = c >> 3, ch = c & 7;
    const bool ok = r0 + r < n;
    cp_async16(dst + swz(r, ch), ok ? src + (size_t)(r0 + r) * ld + ch * 8 : src, ok);
  }
}

__device__ __forceinline__ void ldsm4(uint32_t* r, uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(a)
               : "memory");
}
__device__ __forceinline__ void ldsm4t(uint32_t* r, uint32_t a) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(a)
               : "memory");
}

template <bool BF>
__device__ __forceinline__ void mma(float* c, const uint32_t* a, uint32_t b0, uint32_t b1) {
  if constexpr (BF) {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  } else {
    asm("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
        : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
  }
}

template <bool BF>
__device__ __forceinline__ uint32_t pack2(float x, float y) {
  if constexpr (BF) return f2_to_bf16x2(x, y);
  else return f2_to_f16x2(x, y);
}

// Accumulator layout of a warp's 16 x 64 tile c[n][j]: row g + 8 (j >> 1), column 8 n + 2 t + (j & 1), where
// g = lane / 4 and t = lane % 4.

// c += rows r0 .. r0 + 15 of tile A times tile B transposed: c[r][n] += sum_d A[r][d] B[n][d]
template <bool BF>
__device__ __forceinline__ void gemm_abt(float (*c)[4], uint32_t ta, int r0, uint32_t tb) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    uint32_t a[4];
    ldsm4(a, ta + swz(r0 + (lane & 15), 2 * kk + (lane >> 4)));
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm4(b, tb + swz(16 * np + (lane & 7) + ((lane >> 4) << 3), 2 * kk + ((lane >> 3) & 1)));
      mma<BF>(c[2 * np], a, b[0], b[1]);
      mma<BF>(c[2 * np + 1], a, b[2], b[3]);
    }
  }
}

// c += P times tile B: c[r][n] += sum_k P[r][k] B[k][n], P given as the A fragments of its four 16-column steps
template <bool BF>
__device__ __forceinline__ void gemm_pb(float (*c)[4], const uint32_t (*pa)[4], uint32_t tb) {
  const int lane = threadIdx.x & 31;
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
#pragma unroll
    for (int np = 0; np < 4; ++np) {
      uint32_t b[4];
      ldsm4t(b, tb + swz(16 * kk + (lane & 7) + (((lane >> 3) & 1) << 3), 2 * np + (lane >> 4)));
      mma<BF>(c[2 * np], pa[kk], b[0], b[1]);
      mma<BF>(c[2 * np + 1], pa[kk], b[2], b[3]);
    }
  }
}

// an accumulator tile as the A fragments of the next product, rounded to the activation dtype
template <bool BF>
__device__ __forceinline__ void to_a(uint32_t (*pa)[4], const float (*c)[4]) {
#pragma unroll
  for (int kk = 0; kk < 4; ++kk) {
    pa[kk][0] = pack2<BF>(c[2 * kk][0], c[2 * kk][1]);
    pa[kk][1] = pack2<BF>(c[2 * kk][2], c[2 * kk][3]);
    pa[kk][2] = pack2<BF>(c[2 * kk + 1][0], c[2 * kk + 1][1]);
    pa[kk][3] = pack2<BF>(c[2 * kk + 1][2], c[2 * kk + 1][3]);
  }
}

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

__device__ __forceinline__ void philox_key(const int64_t* seed, uint2* key, uint2* off) {
  const uint64_t sd = (uint64_t)seed[0], of = (uint64_t)seed[1];
  *key = make_uint2((uint32_t)sd, (uint32_t)(sd >> 32));
  *off = make_uint2((uint32_t)of, (uint32_t)(of >> 32));
}

// keep bits of the 4 NG - 3 elements from element index i: bit j for element i + j
template <int NG>
__device__ __forceinline__ uint32_t keep_run(uint2 key, uint2 off, uint64_t i, uint32_t keep) {
  uint64_t w = 0;
#pragma unroll
  for (int g = 0; g < NG; ++g) w |= (uint64_t)keep_nibble(key, off, (i >> 2) + g, keep) << (4 * g);
  return (uint32_t)(w >> (i & 3));
}

// Keep bits of a query-row tile: lane l draws keys 32 (l & 1) .. + 31 of row l / 2 of the warp's 16 rows, whose
// dropout element index at key 0 of the tile is i; w[r][hh] receives the run of row g + 8 r, half hh.
__device__ __forceinline__ void row_keep_bits(uint2 key, uint2 off, uint64_t i, uint32_t keep, uint32_t (*w)[2]) {
  const int lane = threadIdx.x & 31, g = lane >> 2;
  const uint32_t run = keep_run<9>(key, off, i, keep);
#pragma unroll
  for (int r = 0; r < 2; ++r) {
#pragma unroll
    for (int hh = 0; hh < 2; ++hh) w[r][hh] = __shfl_sync(0xffffffffu, run, 2 * (g + 8 * r) + hh);
  }
}
__device__ __forceinline__ bool row_kept(const uint32_t (*w)[2], int n, int j) {
  const int t = threadIdx.x & 3;
  return (w[j >> 1][n >> 2] >> ((n & 3) * 8 + 2 * t + (j & 1))) & 1u;
}

template <bool BF, bool DROP>
__global__ void __launch_bounds__(kThreads) attn_fwd_kernel(Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* mk = reinterpret_cast<float*>(smem + 5 * kTileBytes);
  const uint32_t sq = smem_u32(smem), sk = sq + kTileBytes, sv = sq + 3 * kTileBytes;
  const int S = a.S, H = a.H, E = H * kTile, b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E;
  const uint16_t* qg = a.qkv + (size_t)b * S * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const int nk = (S + kTile - 1) / kTile;

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
    float mx[2] = {m[0], m[1]};
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        s[n][j] = fmaf(s[n][j], kScaleLog2, mrow[n * 8 + 2 * t + (j & 1)]);
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

template <bool BF>
__device__ __forceinline__ float dot8(const uint16_t* x, const uint16_t* y) {
  using U = typename std::conditional<BF, TagBF16, TagF16>::type;
  float fx[8], fy[8], s = 0.f;
  U::unpack(ld_stream16(x), fx);
  U::unpack(ld_stream16(y), fy);
#pragma unroll
  for (int i = 0; i < 8; ++i) s = fmaf(fx[i], fy[i], s);
  return s;
}

// delta = rowsum(dout * out) and dQ = dS K / 8 of one query tile, with dS = P * (dropout'(dO V^T) - delta)
template <bool BF, bool DROP>
__global__ void __launch_bounds__(kThreads) attn_bwd_dq_kernel(Args a) {
  extern __shared__ __align__(128) uint8_t smem[];
  float* mk = reinterpret_cast<float*>(smem + 6 * kTileBytes);
  const uint32_t sq = smem_u32(smem), sdo = sq + kTileBytes, sk = sq + 2 * kTileBytes, sv = sq + 4 * kTileBytes;
  const int S = a.S, H = a.H, E = H * kTile, b = blockIdx.z, h = blockIdx.y, q0 = blockIdx.x * kTile;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const size_t ld = 3 * (size_t)E, bh = (size_t)b * H + h;
  const uint16_t* qg = a.qkv + (size_t)b * S * ld + h * kTile;
  const uint16_t *kg = qg + E, *vg = qg + 2 * E;
  const size_t obase = (size_t)b * S * E + h * kTile;
  const int nk = (S + kTile - 1) / kTile;

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
#pragma unroll
    for (int n = 0; n < 8; ++n) {
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float p = exp2f(fmaf(s[n][j], kScaleLog2, mrow[n * 8 + 2 * t + (j & 1)]) - lr[j >> 1]);
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
template <bool BF, bool DROP>
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

  load_tile(sk, kg, ld, k0, S);
  load_tile(sv, vg, ld, k0, S);
  load_tile(sq, qg, ld, 0, S);
  load_tile(sdo, dog, E, 0, S);
  cp_commit();
  if (threadIdx.x < kTile) {
    const int q = threadIdx.x;
    ls[q] = q < S ? a.lse[bh * S + q] * kLog2e : INFINITY;
    dls[q] = q < S ? a.delta[bh * S + q] : 0.f;
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
  for (int qt = 0; qt < nq; ++qt) {
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
          const float p = exp2f(fmaf(s[n][j], kScaleLog2, km[r]) - lrow[col]);
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

int device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

// launches `kernel` with `smem` dynamic bytes, raising its limit above 48 KB once per device
template <class F>
cudaError_t launch(F kernel, int smem, bool* raised, dim3 grid, const Args& a, cudaStream_t s) {
  const int dev = device();
  if (!raised[dev]) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    raised[dev] = true;
  }
  kernel<<<grid, kThreads, smem, s>>>(a);
  return cudaGetLastError();
}

#define ATTN_KERNEL(NAME, BF, DROP, SMEM)              \
  {                                                    \
    static bool raised[kMaxDevices];                   \
    return launch(NAME<BF, DROP>, SMEM, raised, grid, a, s); \
  }
#define ATTN_DISPATCH(NAME, SMEM)                                   \
  if (bf) {                                                         \
    if (drop) ATTN_KERNEL(NAME, true, true, SMEM)                   \
    else ATTN_KERNEL(NAME, true, false, SMEM)                       \
  } else {                                                          \
    if (drop) ATTN_KERNEL(NAME, false, true, SMEM)                  \
    else ATTN_KERNEL(NAME, false, false, SMEM)                      \
  }

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

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

cudaError_t fwd(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_fwd_kernel, kFwdSmem)
}
cudaError_t bwd_dq(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_bwd_dq_kernel, kDqSmem)
}
cudaError_t bwd_dkv(const Args& a, dim3 grid, bool bf, bool drop, cudaStream_t s) {
  ATTN_DISPATCH(attn_bwd_dkv_kernel, kDkvSmem)
}

}  // namespace

cudaError_t launch_attn_fwd(const void* qkv, int dtype, int B, int S, int H, int D, const void* mask, int mask_kind,
                            int64_t mask_bstride, const int64_t* seed, uint32_t keep, float scale, void* out,
                            float* lse, cudaStream_t s) {
  if (bad_args(dtype, B, S, H, D, mask, mask_kind, mask_bstride) || qkv == nullptr || out == nullptr ||
      lse == nullptr || !aligned16(qkv) || !aligned16(out))
    return cudaErrorInvalidValue;
  Args a = make_args(qkv, S, H, mask, mask_kind, mask_bstride, seed, keep, scale);
  a.o = (uint16_t*)out;
  a.lse = lse;
  return fwd(a, dim3((S + kTile - 1) / kTile, H, B), dtype == WIRE_BF16, seed != nullptr, s);
}

cudaError_t launch_attn_bwd(const void* qkv, const void* out, const void* dout, const float* lse, int dtype, int B,
                            int S, int H, int D, const void* mask, int mask_kind, int64_t mask_bstride,
                            const int64_t* seed, uint32_t keep, float scale, float* delta, void* dqkv,
                            cudaStream_t s) {
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
  const cudaError_t e = bwd_dq(a, grid, bf, drop, s);
  if (e != cudaSuccess) return e;
  return bwd_dkv(a, grid, bf, drop, s);
}

}  // namespace bps
