// FP8 casts with delayed scaling (see fp8.cuh).
//
// fp8_cast works on 128 x 128 tiles.  Block b owns column tile b / R and a contiguous run of row tiles, so its bias
// partials cover 128 columns.  A tile is read in four passes of 32 rows; thread t takes 16 elements (two 16-byte
// loads) of row t / 8, columns 16 (t % 8) onward, and writes their 16 FP8 bytes with one 16-byte store.  For the
// transposed copy it also stores them in a 16 KB shared tile whose 16-byte chunks are XOR-swizzled by row / 16; each
// thread then reads a 16-row x 4-column patch (sixteen 32-bit words, no bank conflicts), transposes it with byte
// permutes and writes four 16-byte rows of the [K, M] copy.  The grid is one resident wave (occupancy API).
//
// An optional elementwise prologue (ACT) turns each loaded value into torch's GELU of it, or into torch's GELU
// gradient of it at the matching element of a second input, rounded to the input dtype as torch stores them; the
// amax, the bias sums and the cast then see exactly the tensor the unfused torch op would have written.
#include "kernels/fp8.cuh"

#include <math.h>

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kT = 256;
constexpr int kW = kT / 32;
constexpr int kTile = 128;       // tile rows and columns
constexpr int kPass = kT / 8;    // tile rows per pass
constexpr int kGroup = 16;       // bias partials summed by the last block of each run of kGroup blocks
constexpr int kMaxDevices = 64;
constexpr uint32_t kInfBits = 0x7f800000u;

struct E4M3 {
  static constexpr float kMax = 448.f;
  __device__ static __forceinline__ uint32_t cvt2(float lo, float hi) {
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
  }
};
struct E5M2 {
  static constexpr float kMax = 57344.f;
  __device__ static __forceinline__ uint32_t cvt2(float lo, float hi) {
    uint16_t r;
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
  }
};

float fmax_of(int fmt) { return fmt == FP8_E5M2 ? E5M2::kMax : E4M3::kMax; }

template <class F>
__device__ __forceinline__ Vec16 pack16(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) w[k] = F::cvt2(f[4 * k], f[4 * k + 1]) | F::cvt2(f[4 * k + 2], f[4 * k + 3]) << 16;
  return Vec16{w[0], w[1], w[2], w[3]};
}

// torch's GELU (erf form) and its gradient, in the order torch's sm_90 kernels evaluate them: every operation is
// pinned with an _rn intrinsic so that contraction cannot change it (torch's gradient contracts 0.5 * (1 + erf)
// into the add, which the __fmaf_rn reproduces); erff and expf are the accurate library functions, as in torch
__device__ __forceinline__ float gelu_f32(float x) {
  constexpr float kAlpha = (float)M_SQRT1_2;
  return __fmul_rn(__fmul_rn(x, 0.5f), __fadd_rn(1.f, erff(__fmul_rn(x, kAlpha))));
}
__device__ __forceinline__ float dgelu_f32(float dy, float x) {
  constexpr float kAlpha = (float)M_SQRT1_2, kBeta = (float)(M_2_SQRTPI * M_SQRT1_2 * 0.5);
  const float pdf = __fmul_rn(expf(__fmul_rn(__fmul_rn(x, -0.5f), x)), kBeta);
  return __fmul_rn(dy, __fmaf_rn(__fadd_rn(1.f, erff(__fmul_rn(x, kAlpha))), 0.5f, __fmul_rn(x, pdf)));
}
__device__ __forceinline__ float round_as(TagBF16, float v) { return __bfloat162float(__float2bfloat16_rn(v)); }
__device__ __forceinline__ float round_as(TagF16, float v) { return __half2float(__float2half_rn(v)); }

// |x| as bits: unsigned order is float order for non-negative values, with inf above every finite value and NaN
// above inf, so a max over them is order-free and says whether the tensor was finite
__device__ __forceinline__ uint32_t abs_bits(float f) { return __float_as_uint(f) & 0x7fffffffu; }

// max of v over the block, returned to thread 0
__device__ __forceinline__ uint32_t block_max(uint32_t v) {
  __shared__ uint32_t sh[kW];
  v = __reduce_max_sync(0xffffffffu, v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  if (threadIdx.x == 0) {
#pragma unroll
    for (int k = 1; k < kW; ++k) v = max(v, sh[k]);
  }
  return v;
}

// max of the G per-block partials, in the last block; returned to thread 0
__device__ __forceinline__ uint32_t grid_max(const uint32_t* part, int G) {
  uint32_t v = 0;
  for (int b = threadIdx.x; b < G; b += kT) v = max(v, __ldcg(part + b));
  return block_max(v);
}

__device__ __forceinline__ float scale_from(const Fp8State* st, float fmax) {
  float h = st->hist[0];
#pragma unroll
  for (int i = 1; i < kFp8History; ++i) h = fmaxf(h, st->hist[i]);
  return fmax / fmaxf(h, 1e-12f);
}

struct AmaxArgs {
  const void* x;
  Fp8State* state;
  uint32_t* ws;
  uint32_t* counters;
  size_t nvec;
  float fmax;
};

template <class U>
__global__ void __launch_bounds__(kT) fp8_amax_kernel(AmaxArgs a) {
  const Vec16* p = reinterpret_cast<const Vec16*>(a.x);
  uint32_t m = 0;
  for (size_t i = (size_t)blockIdx.x * kT + threadIdx.x; i < a.nvec; i += (size_t)gridDim.x * kT) {
    float f[U::kPerVec];
    U::unpack(ld_stream16(p + i), f);
#pragma unroll
    for (int k = 0; k < U::kPerVec; ++k) m = max(m, abs_bits(f[k]));
  }
  m = block_max(m);
  if (threadIdx.x == 0) a.ws[blockIdx.x] = m;
  if (!last_block(a.counters, gridDim.x)) return;
  m = grid_max(a.ws, gridDim.x);
  if (threadIdx.x == 0) {
    const bool finite = m < kInfBits;
    const float amax = __uint_as_float(m);
    Fp8State* st = a.state;
    st->hist[0] = finite ? amax : 0.f;
#pragma unroll
    for (int i = 1; i < kFp8History; ++i) st->hist[i] = 0.f;
    st->count = 0;
    st->scale = finite ? a.fmax / fmaxf(amax, 1e-12f) : NAN;
  }
}

struct CastArgs {
  const void* x;
  Fp8State* state;
  uint8_t *rows, *cols;
  float* inv;
  void* dbias;
  float* ws;
  uint32_t* counters;
  size_t M, rpb;   // rows; row tiles per block
  int K, R;        // columns; blocks per column tile
  const void* aux; // z of FP8_ACT_DGELU, at the offsets of x
};

template <class U, class F, int L, bool BIAS, int ACT>
__global__ void __launch_bounds__(kT) fp8_cast_kernel(CastArgs a) {
  constexpr bool AUX = ACT == FP8_ACT_DGELU;
  constexpr bool ROWS = (L & FP8_ROWS) != 0, COLS = (L & FP8_COLS) != 0;
  __shared__ __align__(16) uint8_t tile[COLS ? kTile * kTile : 16];
  __shared__ float red[BIAS ? kPass * kTile : 1];
  const int tid = threadIdx.x, rr = tid >> 3, ch = tid & 7;
  const int G = gridDim.x, ct = blockIdx.x / a.R, rc = blockIdx.x % a.R;
  const size_t M = a.M, mtiles = (M + kTile - 1) / kTile;
  const size_t t0 = (size_t)rc * a.rpb, t1 = min(mtiles, t0 + a.rpb);
  const int K = a.K, col = ct * kTile + ch * 16;
  const bool colok = col < K;
  const float s = a.state->scale;
  uint32_t amax = 0;
  float cs[16];
#pragma unroll
  for (int k = 0; k < 16; ++k) cs[k] = 0.f;

  for (size_t mt = t0; mt < t1; ++mt) {
    const size_t r0 = mt * kTile;
    Vec16 v[4][2], z[AUX ? 4 : 1][2];
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      const size_t r = r0 + p * kPass + rr;
      if (colok && r < M) {
        const size_t off = (r * (size_t)K + col) * U::kBytes;
        const char* src = reinterpret_cast<const char*>(a.x) + off;
        v[p][0] = ld_stream16(src);
        v[p][1] = ld_stream16(src + 16);
        if (AUX) {
          const char* zs = reinterpret_cast<const char*>(a.aux) + off;
          z[AUX ? p : 0][0] = ld_stream16(zs);
          z[AUX ? p : 0][1] = ld_stream16(zs + 16);
        }
      } else {   // zeros: GELU and its gradient map them to +0, which changes neither the amax nor a sum
        v[p][0] = v[p][1] = Vec16{0, 0, 0, 0};
        if (AUX) z[AUX ? p : 0][0] = z[AUX ? p : 0][1] = Vec16{0, 0, 0, 0};
      }
    }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
      float f[16];
      U::unpack(v[p][0], f);
      U::unpack(v[p][1], f + 8);
      if (ACT == FP8_ACT_GELU) {
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] = round_as(U{}, gelu_f32(f[k]));
      } else if (AUX) {
        float g[16];
        U::unpack(z[AUX ? p : 0][0], g);
        U::unpack(z[AUX ? p : 0][1], g + 8);
#pragma unroll
        for (int k = 0; k < 16; ++k) f[k] = round_as(U{}, dgelu_f32(f[k], g[k]));
      }
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        amax = max(amax, abs_bits(f[k]));
        if (BIAS) cs[k] += f[k];
        f[k] *= s;
      }
      const Vec16 q = pack16<F>(f);
      const int tr = p * kPass + rr;
      const size_t r = r0 + tr;
      if (ROWS && colok && r < M) st_stream16(a.rows + r * (size_t)K + col, q);
      if (COLS) sts16(tile + tr * kTile + ((ch ^ ((tr >> 4) & 7)) * 16), q);
    }
    if (COLS) {
      __syncthreads();
      const int lane = tid & 31, w = tid >> 5, sg = lane & 7, gq = lane >> 3;
      const size_t m = r0 + sg * 16;
      const int k0 = ct * kTile + 4 * (w * 4 + gq);
      if (m < M && k0 < K) {
        uint32_t W[16];
#pragma unroll
        for (int i = 0; i < 16; ++i)
          W[i] = *reinterpret_cast<const uint32_t*>(tile + (sg * 16 + i) * kTile + (w ^ sg) * 16 + gq * 4);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const uint32_t sel = j | (j + 4) << 4;
          uint32_t o[4];
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            const uint32_t lo = __byte_perm(W[4 * q], W[4 * q + 1], sel);
            const uint32_t hi = __byte_perm(W[4 * q + 2], W[4 * q + 3], sel);
            o[q] = __byte_perm(lo, hi, 0x5410);
          }
          st_stream16(a.cols + (size_t)(k0 + j) * M + m, Vec16{o[0], o[1], o[2], o[3]});
        }
      }
      __syncthreads();
    }
  }

  // amax: block partials, then the last block of the grid records it
  uint32_t* amax_part = reinterpret_cast<uint32_t*>(a.ws);
  amax = block_max(amax);
  if (tid == 0) amax_part[blockIdx.x] = amax;
  if (BIAS) {   // the block's column sums: its 32 row threads of each column in order
#pragma unroll
    for (int k = 0; k < 16; ++k) red[rr * kTile + ch * 16 + k] = cs[k];
    __syncthreads();
    if (tid < kTile) {
      float c = red[tid];
#pragma unroll 8
      for (int i = 1; i < kPass; ++i) c += red[i * kTile + tid];
      a.ws[G + (size_t)blockIdx.x * kTile + tid] = c;
    }
  }
  if (last_block(a.counters, G)) {
    const uint32_t m = grid_max(amax_part, G);
    if (tid == 0) {
      Fp8State* st = a.state;
      const bool finite = m < kInfBits;
      *a.inv = finite ? 1.f / s : NAN;
      if (finite) {
        const uint32_t t = st->count;
        st->hist[t % kFp8History] = __uint_as_float(m);
        st->count = t + 1;
        st->scale = scale_from(st, F::kMax);
      }
    }
  }
  if (!BIAS) return;

  // bias: runs of kGroup blocks of a column tile, then the column tile's runs, each summed in block order by the
  // last block to arrive
  const int ngr = (a.R + kGroup - 1) / kGroup, grp = rc / kGroup, gid = ct * ngr + grp;
  const float* bpart = a.ws + G;
  float* gpart = a.ws + G + (size_t)G * kTile;
  if (!last_block(a.counters + 1 + gid, min(kGroup, a.R - grp * kGroup))) return;
  if (tid < kTile) {
    const int b0 = ct * a.R + grp * kGroup, b1 = ct * a.R + min(a.R, (grp + 1) * kGroup);
    float c = __ldcg(bpart + (size_t)b0 * kTile + tid);
    for (int b = b0 + 1; b < b1; ++b) c += __ldcg(bpart + (size_t)b * kTile + tid);
    gpart[(size_t)gid * kTile + tid] = c;
  }
  const int ngroups = (G / a.R) * ngr;
  if (!last_block(a.counters + 1 + ngroups + ct, ngr)) return;
  const int c0 = ct * kTile + tid;
  if (tid < kTile && c0 < K) {
    float c = __ldcg(gpart + (size_t)(ct * ngr) * kTile + tid);
    for (int g = 1; g < ngr; ++g) c += __ldcg(gpart + (size_t)(ct * ngr + g) * kTile + tid);
    U::store1(a.dbias, c0, c);
  }
}

// ---- host side

using CastFn = void (*)(CastArgs);

template <class U, class F, int ACT, bool BIAS>
CastFn cast_kernel_l(int layout) {
  switch (layout) {
    case FP8_ROWS: return fp8_cast_kernel<U, F, FP8_ROWS, BIAS, ACT>;
    case FP8_COLS: return fp8_cast_kernel<U, F, FP8_COLS, BIAS, ACT>;
    case FP8_BOTH: return fp8_cast_kernel<U, F, FP8_BOTH, BIAS, ACT>;
    default: return nullptr;
  }
}

// the forward GELU has no bias gradient to produce, so it is not built with one
template <class U, class F, int ACT>
CastFn cast_kernel_ufa(int layout, bool bias) {
  if constexpr (ACT == FP8_ACT_GELU)
    return bias ? nullptr : cast_kernel_l<U, F, ACT, false>(layout);
  else
    return bias ? cast_kernel_l<U, F, ACT, true>(layout) : cast_kernel_l<U, F, ACT, false>(layout);
}

template <class U, class F>
CastFn cast_kernel_uf(int layout, bool bias, int act) {
  if (act == FP8_ACT_NONE) return cast_kernel_ufa<U, F, FP8_ACT_NONE>(layout, bias);
  if (act == FP8_ACT_GELU) return cast_kernel_ufa<U, F, FP8_ACT_GELU>(layout, bias);
  if (act == FP8_ACT_DGELU) return cast_kernel_ufa<U, F, FP8_ACT_DGELU>(layout, bias);
  return nullptr;
}

template <class U>
CastFn cast_kernel_u(int fmt, int layout, bool bias, int act) {
  if (fmt == FP8_E4M3) return cast_kernel_uf<U, E4M3>(layout, bias, act);
  if (fmt == FP8_E5M2) return cast_kernel_uf<U, E5M2>(layout, bias, act);
  return nullptr;
}

CastFn cast_kernel(int dtype, int fmt, int layout, bool bias, int act) {
  if (dtype == WIRE_BF16) return cast_kernel_u<TagBF16>(fmt, layout, bias, act);
  if (dtype == WIRE_F16) return cast_kernel_u<TagF16>(fmt, layout, bias, act);
  return nullptr;
}

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

bool bad_shape(size_t M, int K) { return M < 16 || K < 16 || M % 16 != 0 || K % 16 != 0; }

int device() {
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) dev = 0;
  return dev;
}

int sm_count() {
  int sms = 132;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device()) != cudaSuccess) sms = 132;
  return sms;
}

// blocks of `kernel` one SM holds, from the occupancy API, cached per device in `cache`
template <class Fn>
int resident(Fn kernel, int* cache) {
  const int dev = device();
  int n = cache[dev];
  if (n == 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kT, 0) != cudaSuccess || n < 1) n = 1;
    cache[dev] = n;
  }
  return n;
}

// each activation is its own instantiation, with its own registers and so its own resident count
int cast_wave(int dtype, int fmt, int layout, bool bias, int act) {
  static int cache[3][2][2][4][2][kMaxDevices];
  const int d = dtype == WIRE_F16 ? 1 : 0;
  return resident(cast_kernel(dtype, fmt, layout, bias, act), cache[act][d][fmt][layout][bias ? 1 : 0]) *
         sm_count();
}

// the wave a cast's grid is planned for.  A bias gradient's fp32 sums follow the grid (row tiles per block, blocks
// per column tile), so a cast with a prologue plans the plain cast's grid and its bias gradient is bit for bit that
// of the plain cast of the activation; the gradient prologue, at half the plain cast's resident blocks, then runs it
// in two waves.  Without a bias gradient every cast fills its own resident wave.
int plan_wave(int dtype, int fmt, int layout, bool bias, int act) {
  return cast_wave(dtype, fmt, layout, bias, bias ? FP8_ACT_NONE : act);
}

int amax_wave(int dtype) {
  static int cache[2][kMaxDevices];
  if (dtype == WIRE_F16) return resident(fp8_amax_kernel<TagF16>, cache[1]) * sm_count();
  return resident(fp8_amax_kernel<TagBF16>, cache[0]) * sm_count();
}

// column tiles, blocks per column tile and row tiles per block of one wave
void cast_grid(size_t M, int K, int wave, int* nct, int* R, size_t* rpb) {
  const size_t mtiles = (M + kTile - 1) / kTile;
  *nct = (K + kTile - 1) / kTile;
  size_t r = (size_t)(wave / *nct);
  if (r < 1) r = 1;
  if (r > mtiles) r = mtiles;
  *rpb = (mtiles + r - 1) / r;
  *R = (int)((mtiles + *rpb - 1) / *rpb);
}

int amax_grid(size_t nvec, int wave) {
  const size_t want = (nvec + kT - 1) / kT;
  return (int)(want < (size_t)wave ? want : (size_t)wave);
}

bool bad_cast_args(int dtype, int fmt, int layout, int act, bool dbias) {
  return (dtype != WIRE_BF16 && dtype != WIRE_F16) || (fmt != FP8_E4M3 && fmt != FP8_E5M2) || layout < FP8_ROWS ||
         layout > FP8_BOTH || act < FP8_ACT_NONE || act > FP8_ACT_DGELU || (act == FP8_ACT_GELU && dbias);
}

}  // namespace

void fp8_cast_workspace(size_t M, int K, int dtype, int fmt, int layout, bool dbias, int act, size_t* floats,
                        int* counters) {
  *floats = 0;
  *counters = 0;
  if (bad_shape(M, K) || bad_cast_args(dtype, fmt, layout, act, dbias)) return;
  int nct, R;
  size_t rpb;
  cast_grid(M, K, plan_wave(dtype, fmt, layout, dbias, act), &nct, &R, &rpb);
  const size_t G = (size_t)nct * R, ngroups = (size_t)nct * ((R + kGroup - 1) / kGroup);
  *floats = G + (dbias ? (G + ngroups) * kTile : 0);
  *counters = 1 + (dbias ? (int)(ngroups + nct) : 0);
}

void fp8_amax_workspace(size_t M, int K, int dtype, size_t* floats, int* counters) {
  *floats = 0;
  *counters = 0;
  if (bad_shape(M, K) || (dtype != WIRE_BF16 && dtype != WIRE_F16)) return;
  *floats = (size_t)amax_grid(M * (size_t)K / 8, amax_wave(dtype));
  *counters = 1;
}

cudaError_t launch_fp8_amax(const void* x, int dtype, size_t M, int K, int fmt, Fp8State* state, float* ws,
                            uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, K) || x == nullptr || !aligned16(x) || state == nullptr || ws == nullptr || counters == nullptr ||
      (fmt != FP8_E4M3 && fmt != FP8_E5M2))
    return cudaErrorInvalidValue;
  AmaxArgs a{x, state, reinterpret_cast<uint32_t*>(ws), counters, M * (size_t)K / 8, fmax_of(fmt)};
  const int grid = amax_grid(a.nvec, amax_wave(dtype));
  if (dtype == WIRE_BF16)
    fp8_amax_kernel<TagBF16><<<grid, kT, 0, s>>>(a);
  else if (dtype == WIRE_F16)
    fp8_amax_kernel<TagF16><<<grid, kT, 0, s>>>(a);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_fp8_cast(const void* x, int dtype, size_t M, int K, int fmt, int layout, Fp8State* state,
                            void* out_rows, void* out_cols, float* inv, void* dbias, float* ws, uint32_t* counters,
                            cudaStream_t s, int act, const void* aux) {
  if (bad_shape(M, K) || bad_cast_args(dtype, fmt, layout, act, dbias != nullptr) || x == nullptr ||
      !aligned16(x) || state == nullptr || inv == nullptr || ws == nullptr || counters == nullptr ||
      (act == FP8_ACT_DGELU ? aux == nullptr || !aligned16(aux) : aux != nullptr) ||
      ((layout & FP8_ROWS) && (out_rows == nullptr || !aligned16(out_rows))) ||
      ((layout & FP8_COLS) && (out_cols == nullptr || !aligned16(out_cols))))
    return cudaErrorInvalidValue;
  const bool bias = dbias != nullptr;
  int nct, R;
  size_t rpb;
  cast_grid(M, K, plan_wave(dtype, fmt, layout, bias, act), &nct, &R, &rpb);
  CastArgs a{x, state, (uint8_t*)out_rows, (uint8_t*)out_cols, inv, dbias, ws, counters, M, rpb, K, R, aux};
  cast_kernel(dtype, fmt, layout, bias, act)<<<nct * R, kT, 0, s>>>(a);
  return cudaGetLastError();
}

}  // namespace bps
