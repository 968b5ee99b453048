// Fused dropout + residual add + LayerNorm (see ln.cuh).
//
// A thread owns up to NU "units" of a row: 8 consecutive elements, i.e. one 16-byte vector for 16-bit activations
// (two for fp32) and one mask byte.  The TPR threads of a row group take units l, l + TPR, ... so a warp's loads are
// contiguous; groups of up to 32 threads reduce with shuffles, wider ones add their warps' sums in shared memory
// behind a named barrier of the group.  Every group of a block runs the same number of row steps (idle at the end of
// a chunk), so the shuffles of a warp shared by two groups always meet.
#include "kernels/ln.cuh"

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kT = 256;
constexpr int kCh = 8;          // elements per unit
constexpr int kGroup = 16;      // block partials summed by the last block of each run of kGroup blocks
constexpr int kMaxDevices = 64;
// Register budgets: fwd holds a row slice (16 floats); bwd holds xhat and g of it plus the thread's dgamma / dbeta
// partials (64 floats).
constexpr int kFwdBlocksPerSM = 4;
constexpr int kBwdBlocksPerSM = 2;

template <class U>
struct Io {
  static constexpr int kVecs = kCh / U::kPerVec;
  __device__ static __forceinline__ void load(const void* base, size_t unit, float* f) {
    const Vec16* p = reinterpret_cast<const Vec16*>(base) + unit * kVecs;
#pragma unroll
    for (int v = 0; v < kVecs; ++v) U::unpack(ld_stream16(p + v), f + v * U::kPerVec);
  }
  // parameters: read by every row, so cached
  __device__ static __forceinline__ void load_cached(const void* base, int unit, float* f) {
    const uint4* p = reinterpret_cast<const uint4*>(base) + (size_t)unit * kVecs;
#pragma unroll
    for (int v = 0; v < kVecs; ++v) {
      const uint4 q = __ldg(p + v);
      U::unpack(Vec16{q.x, q.y, q.z, q.w}, f + v * U::kPerVec);
    }
  }
  __device__ static __forceinline__ void store(void* base, size_t unit, const float* f) {
    Vec16* p = reinterpret_cast<Vec16*>(base) + unit * kVecs;
#pragma unroll
    for (int v = 0; v < kVecs; ++v) st_stream16(p + v, U::pack(f + v * U::kPerVec));
  }
  __device__ static __forceinline__ void round(float* f) {
#pragma unroll
    for (int v = 0; v < kVecs; ++v) U::unpack(U::pack(f + v * U::kPerVec), f + v * U::kPerVec);
  }
};

// Sum of the K values over the TPR threads of row group `grp`, returned to all of them.  Wider groups go through
// sh[K][TPR / 32]; callers alternate between two such buffers, so a buffer is written again only after every thread
// of the group has passed the barrier of the reduction in between.
template <int TPR, int K>
__device__ __forceinline__ void row_sum(float* v, float (*sh)[TPR > 32 ? TPR / 32 : 1], int grp) {
#pragma unroll
  for (int o = (TPR < 32 ? TPR : 32) / 2; o > 0; o >>= 1) {
#pragma unroll
    for (int k = 0; k < K; ++k) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
  }
  if constexpr (TPR > 32) {
    const int w = (threadIdx.x % TPR) / 32;
    if ((threadIdx.x & 31) == 0) {
#pragma unroll
      for (int k = 0; k < K; ++k) sh[k][w] = v[k];
    }
    named_bar_sync(1 + grp, TPR);
#pragma unroll
    for (int k = 0; k < K; ++k) {
      float s = sh[k][0];
#pragma unroll
      for (int i = 1; i < TPR / 32; ++i) s += sh[k][i];
      v[k] = s;
    }
  }
}

struct FwdArgs {
  const void *y, *res, *gamma, *beta;
  const int64_t* seed;
  void *z, *out;
  float *mean, *rstd;
  uint8_t* mask;
  size_t M, rpc;
  int H;
  float eps, scale;
  uint32_t keep;
};

template <class U, class W, int NU, int TPR>
__global__ void __launch_bounds__(kT, kFwdBlocksPerSM) ln_fwd_kernel(FwdArgs a) {
  constexpr int RPB = kT / TPR, NW = TPR > 32 ? TPR / 32 : 1;
  __shared__ float sh[RPB][2][1][NW];
  const int units = a.H / kCh, grp = threadIdx.x / TPR, l = threadIdx.x % TPR;
  const size_t r0 = (size_t)blockIdx.x * a.rpc, r1 = min(a.M, r0 + a.rpc);
  const bool drop = a.mask != nullptr;
  uint2 key = make_uint2(0, 0), off = make_uint2(0, 0);
  if (drop) {
    const uint64_t sd = (uint64_t)a.seed[0], of = (uint64_t)a.seed[1];
    key = make_uint2((uint32_t)sd, (uint32_t)(sd >> 32));
    off = make_uint2((uint32_t)of, (uint32_t)(of >> 32));
  }
  for (size_t base = r0; base < r1; base += RPB) {
    const size_t row = base + grp;
    const bool active = row < r1;
    float v[NU][kCh];
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = k * TPR + l;
#pragma unroll
      for (int j = 0; j < kCh; ++j) v[k][j] = 0.f;
      if (active && u < units) {
        const size_t gu = row * units + u;
        Io<U>::load(a.y, gu, v[k]);
        if (drop) {
          const uint32_t bits = keep_bits(key, off, row * (size_t)a.H + (size_t)u * kCh, a.keep);
#pragma unroll
          for (int j = 0; j < kCh; ++j) v[k][j] = (bits >> j) & 1u ? v[k][j] * a.scale : 0.f;
          a.mask[gu] = (uint8_t)bits;
        }
        if (a.res != nullptr) {
          float r[kCh];
          Io<U>::load(a.res, gu, r);
#pragma unroll
          for (int j = 0; j < kCh; ++j) v[k][j] += r[j];
        }
        if (drop || a.res != nullptr) {
          Io<U>::round(v[k]);   // the statistics and the backward both see the stored z
          if (a.z != nullptr) Io<U>::store(a.z, gu, v[k]);
        }
      }
#pragma unroll
      for (int j = 0; j < kCh; ++j) s += v[k][j];
    }
    row_sum<TPR, 1>(&s, sh[grp][0], grp);
    const float mean = s / (float)a.H;
    float q = 0.f;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      if (k * TPR + l < units) {
#pragma unroll
        for (int j = 0; j < kCh; ++j) {
          const float d = v[k][j] - mean;
          q = fmaf(d, d, q);
        }
      }
    }
    row_sum<TPR, 1>(&q, sh[grp][1], grp);
    const float rstd = 1.f / sqrtf(q / (float)a.H + a.eps);
    if (!active) continue;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = k * TPR + l;
      if (u < units) {
        float g[kCh], b[kCh];
        Io<W>::load_cached(a.gamma, u, g);
        Io<W>::load_cached(a.beta, u, b);
#pragma unroll
        for (int j = 0; j < kCh; ++j) v[k][j] = fmaf((v[k][j] - mean) * rstd, g[j], b[j]);
        Io<U>::store(a.out, row * units + u, v[k]);
      }
    }
    if (l == 0) {
      a.mean[row] = mean;
      a.rstd[row] = rstd;
    }
  }
}

struct BwdArgs {
  const void *dout, *z, *gamma;
  const uint8_t* mask;
  const float *mean, *rstd;
  void *dres, *dy, *dgamma, *dbeta;
  float* ws;
  uint32_t* counters;
  size_t M, rpc;
  int H;
  float scale;
};

template <class U, class W, int NU, int TPR>
__global__ void __launch_bounds__(kT, kBwdBlocksPerSM) ln_bwd_kernel(BwdArgs a) {
  constexpr int RPB = kT / TPR, NW = TPR > 32 ? TPR / 32 : 1;
  __shared__ float sh[RPB][2][2][NW];
  __shared__ float red[RPB * 2 * NU * kCh * TPR];   // the groups' dgamma / dbeta partials, 2H floats per group
  const int H = a.H, units = H / kCh, grp = threadIdx.x / TPR, l = threadIdx.x % TPR;
  const size_t r0 = (size_t)blockIdx.x * a.rpc, r1 = min(a.M, r0 + a.rpc);
  float dg[NU][kCh], db[NU][kCh];
#pragma unroll
  for (int k = 0; k < NU; ++k) {
#pragma unroll
    for (int j = 0; j < kCh; ++j) dg[k][j] = db[k][j] = 0.f;
  }
  int step = 0;
  for (size_t base = r0; base < r1; base += RPB, ++step) {
    const size_t row = base + grp;
    const bool active = row < r1;
    const float mean = active ? a.mean[row] : 0.f, rstd = active ? a.rstd[row] : 0.f;
    float xh[NU][kCh], g[NU][kCh];
    float sums[2] = {0.f, 0.f};   // sum g, sum g * xhat
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = k * TPR + l;
#pragma unroll
      for (int j = 0; j < kCh; ++j) xh[k][j] = g[k][j] = 0.f;
      if (active && u < units) {
        const size_t gu = row * units + u;
        float d[kCh], w[kCh];
        Io<U>::load(a.z, gu, xh[k]);
        Io<U>::load(a.dout, gu, d);
        Io<W>::load_cached(a.gamma, u, w);
#pragma unroll
        for (int j = 0; j < kCh; ++j) {
          xh[k][j] = (xh[k][j] - mean) * rstd;
          g[k][j] = d[j] * w[j];
          dg[k][j] = fmaf(d[j], xh[k][j], dg[k][j]);
          db[k][j] += d[j];
          sums[0] += g[k][j];
          sums[1] = fmaf(g[k][j], xh[k][j], sums[1]);
        }
      }
    }
    row_sum<TPR, 2>(sums, sh[grp][step & 1], grp);
    if (!active) continue;
    const float ma = sums[0] / (float)H, mb = sums[1] / (float)H;
#pragma unroll
    for (int k = 0; k < NU; ++k) {
      const int u = k * TPR + l;
      if (u < units) {
        const size_t gu = row * units + u;
        float dz[kCh];
#pragma unroll
        for (int j = 0; j < kCh; ++j) dz[j] = rstd * (g[k][j] - ma - xh[k][j] * mb);
        if (a.dres != nullptr) Io<U>::store(a.dres, gu, dz);
        if (a.dy != nullptr) {
          const uint32_t bits = a.mask != nullptr ? a.mask[gu] : 0xffu;
#pragma unroll
          for (int j = 0; j < kCh; ++j) dz[j] = (bits >> j) & 1u ? dz[j] * a.scale : 0.f;
          Io<U>::store(a.dy, gu, dz);
        }
      }
    }
  }

  // the block's partials: the groups' sums added in group order
  const int H2 = 2 * H;
#pragma unroll
  for (int k = 0; k < NU; ++k) {
    const int u = k * TPR + l;
    if (u < units) {
#pragma unroll
      for (int j = 0; j < kCh; ++j) {
        red[grp * H2 + u * kCh + j] = dg[k][j];
        red[grp * H2 + H + u * kCh + j] = db[k][j];
      }
    }
  }
  __syncthreads();
  float* part = a.ws + (size_t)blockIdx.x * H2;
  for (int c = threadIdx.x; c < H2; c += kT) {
    float s = red[c];
#pragma unroll 4
    for (int i = 1; i < RPB; ++i) s += red[i * H2 + c];
    part[c] = s;
  }

  // runs of kGroup blocks, then the runs, each summed in block order by the last block to arrive
  const int G = gridDim.x, runs = (G + kGroup - 1) / kGroup, run = blockIdx.x / kGroup;
  if (!last_block(a.counters + run, min(kGroup, G - run * kGroup))) return;
  float* run_part = a.ws + (size_t)(G + run) * H2;
  for (int c = threadIdx.x; c < H2; c += kT) {
    const int b0 = run * kGroup, b1 = min(G, b0 + kGroup);
    float s = __ldcg(a.ws + (size_t)b0 * H2 + c);
    for (int b = b0 + 1; b < b1; ++b) s += __ldcg(a.ws + (size_t)b * H2 + c);
    run_part[c] = s;
  }
  if (!last_block(a.counters + runs, runs)) return;
  for (int c = threadIdx.x; c < H2; c += kT) {
    float s = __ldcg(a.ws + (size_t)G * H2 + c);
    for (int r = 1; r < runs; ++r) s += __ldcg(a.ws + (size_t)(G + r) * H2 + c);
    if (c < H)
      W::store1(a.dgamma, c, s);
    else
      W::store1(a.dbeta, c - H, s);
  }
}

// ---- host side

// (activation, parameter) element types and the row layout (units per thread, threads per row) of width H
#define LN_DISPATCH(dtype, wdtype, H, STMT)                                                  \
  switch ((dtype) * 3 + (wdtype)) {                                                          \
    case WIRE_F32 * 3 + WIRE_F32: { using U = TagF32; using W = TagF32; LN_LAYOUT(H, STMT) } \
    case WIRE_BF16 * 3 + WIRE_F32: { using U = TagBF16; using W = TagF32; LN_LAYOUT(H, STMT) } \
    case WIRE_BF16 * 3 + WIRE_BF16: { using U = TagBF16; using W = TagBF16; LN_LAYOUT(H, STMT) } \
    case WIRE_F16 * 3 + WIRE_F32: { using U = TagF16; using W = TagF32; LN_LAYOUT(H, STMT) } \
    case WIRE_F16 * 3 + WIRE_F16: { using U = TagF16; using W = TagF16; LN_LAYOUT(H, STMT) } \
    default: return cudaErrorInvalidValue;                                                   \
  }
#define LN_LAYOUT(H, STMT)                                                  \
  if ((H) <= 128) { constexpr int NU = 1, TPR = 16; STMT; }                 \
  else if ((H) <= 256) { constexpr int NU = 1, TPR = 32; STMT; }            \
  else if ((H) <= 512) { constexpr int NU = 2, TPR = 32; STMT; }            \
  else if ((H) <= 1024) { constexpr int NU = 2, TPR = 64; STMT; }           \
  else { constexpr int NU = 2, TPR = 128; STMT; }                           \
  break;

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

bool bad_shape(size_t M, int H) { return M < 1 || H < kCh || H > kLnMaxH || H % kCh != 0; }

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
template <class F>
int resident(F kernel, int* cache) {
  const int dev = device();
  int n = cache[dev];
  if (n == 0) {
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, kT, 0) != cudaSuccess || n < 1) n = 1;
    cache[dev] = n;
  }
  return n;
}

template <class U, class W, int NU, int TPR>
int fwd_wave() {
  static int cache[kMaxDevices];
  return resident(ln_fwd_kernel<U, W, NU, TPR>, cache) * sm_count();
}

template <class U, class W, int NU, int TPR>
int bwd_wave() {
  static int cache[kMaxDevices];
  return resident(ln_bwd_kernel<U, W, NU, TPR>, cache) * sm_count();
}

// Contiguous chunks of rows (a multiple of the block's rpb rows per step), at most one per block of a wave.
void chunks(size_t M, size_t rpb, int wave, size_t* rpc, int* grid) {
  size_t want = (M + rpb - 1) / rpb;
  if (want > (size_t)wave) want = (size_t)wave;
  size_t r = (M + want - 1) / want;
  r = (r + rpb - 1) / rpb * rpb;
  *rpc = r;
  *grid = (int)((M + r - 1) / r);
}

// The most blocks a bwd launch at (M, H) takes, over the parameter dtypes: the workspace fits all of them.
int bwd_blocks(size_t M, int H) {
  int most = 0;
  for (int dt = WIRE_F32; dt <= WIRE_F16; ++dt) {
    for (int wt : {(int)WIRE_F32, dt}) {
      int grid = 0;
      auto pick = [&]() -> cudaError_t {
        LN_DISPATCH(dt, wt, H, ({
          size_t rpc;
          chunks(M, kT / TPR, bwd_wave<U, W, NU, TPR>(), &rpc, &grid);
        }));
        return cudaSuccess;
      };
      pick();
      if (grid > most) most = grid;
    }
  }
  return most;
}

}  // namespace

size_t ln_workspace_floats(size_t M, int H) {
  if (bad_shape(M, H)) return 0;
  const size_t G = (size_t)bwd_blocks(M, H);
  return (G + (G + kGroup - 1) / kGroup) * 2 * (size_t)H;
}

int ln_counters(size_t M, int H) {
  if (bad_shape(M, H)) return 0;
  return (bwd_blocks(M, H) + kGroup - 1) / kGroup + 1;
}

cudaError_t launch_ln_fwd(const void* y, const void* residual, int dtype, int wdtype, size_t M, int H, float eps,
                          const void* gamma, const void* beta, const int64_t* seed, uint32_t keep, float scale,
                          void* z, void* out, float* mean, float* rstd, uint8_t* mask, cudaStream_t s) {
  if (bad_shape(M, H) || !aligned16(y) || !aligned16(residual) || !aligned16(z) || !aligned16(out) ||
      !aligned16(gamma) || !aligned16(beta) || gamma == nullptr || beta == nullptr || out == nullptr ||
      mean == nullptr || rstd == nullptr || (mask != nullptr && seed == nullptr))
    return cudaErrorInvalidValue;
  FwdArgs a{y, residual, gamma, beta, seed, z, out, mean, rstd, mask, M, 0, H, eps, scale, keep};
  LN_DISPATCH(dtype, wdtype, H, ({
    int grid;
    chunks(M, kT / TPR, fwd_wave<U, W, NU, TPR>(), &a.rpc, &grid);
    ln_fwd_kernel<U, W, NU, TPR><<<grid, kT, 0, s>>>(a);
  }));
  return cudaGetLastError();
}

cudaError_t launch_ln_bwd(const void* dout, const void* z, const uint8_t* mask, int dtype, int wdtype, size_t M, int H,
                          float scale, const float* mean, const float* rstd, const void* gamma, void* dres, void* dy,
                          void* dgamma, void* dbeta, float* ws, uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, H) || !aligned16(dout) || !aligned16(z) || !aligned16(gamma) || !aligned16(dres) ||
      !aligned16(dy) || dout == nullptr || z == nullptr || gamma == nullptr || mean == nullptr || rstd == nullptr ||
      dgamma == nullptr || dbeta == nullptr || ws == nullptr || counters == nullptr)
    return cudaErrorInvalidValue;
  BwdArgs a{dout, z, gamma, mask, mean, rstd, dres, dy, dgamma, dbeta, ws, counters, M, 0, H, scale};
  LN_DISPATCH(dtype, wdtype, H, ({
    int grid;
    chunks(M, kT / TPR, bwd_wave<U, W, NU, TPR>(), &a.rpc, &grid);
    ln_bwd_kernel<U, W, NU, TPR><<<grid, kT, 0, s>>>(a);
  }));
  return cudaGetLastError();
}

}  // namespace bps
