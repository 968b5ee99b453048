// Tile code shared by the padded (attn_kernels.cuh) and packed variable-length (attn_varlen_kernels.cuh) attention
// kernels: cp.async tile loads into XOR-swizzled shared memory, ldmatrix + mma.sync.m16n8k16 products with fp32
// accumulators, the dropout keep bits of a tile, and the host-side launch helpers.  Included by those two headers
// and by the stem convolution (stem_conv.cu), which uses the tile loads and the ldmatrix / mma wrappers.
#pragma once
#include <type_traits>

#include "kernels/attn.cuh"
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

// the query tile of a CTA that walks one query tile over the key tiles: under the causal mask the last tile first,
// so the CTAs with the most key tiles start first
template <bool CAUSAL>
__device__ __forceinline__ int query_tile() {
  return CAUSAL ? (int)(gridDim.x - 1 - blockIdx.x) : (int)blockIdx.x;
}

// whether the score of tile row r and tile column c lies above the diagonal of a diagonal tile (causal mask)
__device__ __forceinline__ bool above_diagonal(int r, int c) { return c > r; }

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

// ---- host side

int device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

// launches `kernel` with `smem` dynamic bytes, raising its limit above 48 KB once per device
template <class F, class A>
cudaError_t launch(F kernel, int smem, bool* raised, dim3 grid, const A& a, cudaStream_t s) {
  const int dev = device();
  if (!raised[dev]) {
    const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    if (e != cudaSuccess) return e;
    raised[dev] = true;
  }
  kernel<<<grid, kThreads, smem, s>>>(a);
  return cudaGetLastError();
}

#define ATTN_KERNEL(NAME, BF, DROP, CAUSAL, SMEM)                    \
  {                                                                   \
    static bool raised[kMaxDevices];                                  \
    return launch(NAME<BF, DROP, CAUSAL>, SMEM, raised, grid, a, s);  \
  }
#define ATTN_DISPATCH(NAME, SMEM, CAUSAL)                           \
  if (bf) {                                                         \
    if (drop) ATTN_KERNEL(NAME, true, true, CAUSAL, SMEM)           \
    else ATTN_KERNEL(NAME, true, false, CAUSAL, SMEM)               \
  } else {                                                          \
    if (drop) ATTN_KERNEL(NAME, false, true, CAUSAL, SMEM)          \
    else ATTN_KERNEL(NAME, false, false, CAUSAL, SMEM)              \
  }

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

}  // namespace

}  // namespace bps
