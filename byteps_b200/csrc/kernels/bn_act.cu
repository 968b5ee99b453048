// Fused NHWC batch norm + residual add + ReLU (see bn_act.cuh).
//
// All four passes share one thread layout.  A thread owns a "unit": 8 consecutive channels of a row, i.e. one
// 16-byte vector for 16-bit activations (two for fp32) and one mask byte.  A block of kT threads covers CB units
// of one channel group (CB a power of two <= 32; blockIdx.y selects the group) times RL = kT / CB rows, and
// blockIdx.x walks the rows.  A thread therefore keeps the same channels for the whole launch: their parameters
// live in registers, and a warp touches 512 contiguous bytes of a 16-bit row when C >= 256.
#include "kernels/bn_act.cuh"

#include <mutex>

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kT = 256;
constexpr int kCh = 8;                  // channels per unit
constexpr int kMaxCB = 32;              // units per block row of an elementwise pass
// Units per block row of a reduction pass.  Narrow channel groups leave few chunk partials per channel, and the
// finalize gives each channel kT / (CB * kCh) threads, so its sums stay short.  8 units are a full 128-byte line
// of a 16-bit row, which no two blocks then share; that pays once C >= 256 leaves at least 4 groups.  Narrower C
// keeps 4-unit groups: with 1 or 2 groups the finalize's per-thread sums would be too long.
int red_cb(int C) { return C >= 256 ? 8 : 4; }
// Every pass is sized to one full wave: kBlocksPerSM resident blocks on every SM (the register budget
// __launch_bounds__ enforces), each walking its rows with 16-byte loads of several rows in flight.  A second,
// partial wave would leave most SMs idle for its whole duration.
constexpr int kBlocksPerSM = 3;
constexpr int kBwdApplyBlocksPerSM = 2;   // its per-channel coefficients and two rows in flight need ~90 registers
constexpr int kMinRows = 4;             // fewest rows a thread of a reduction pass walks

struct Geo {
  int shift;   // log2(CB)
  int ncb;     // channel groups (gridDim.y)
  int rl;      // rows per block step (RL)
};

Geo geo(int C, int max_cb) {
  const int units = C / kCh;
  int shift = 0;
  while ((2 << shift) <= units && (2 << shift) <= max_cb) ++shift;
  return Geo{shift, (units + (1 << shift) - 1) >> shift, kT >> shift};
}

// Rows per chunk of a reduction pass (a multiple of RL) and the chunk count (gridDim.x).
int wave_blocks(int per_sm = kBlocksPerSM) {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    sms = 132;
  return sms * per_sm;
}

void chunks(size_t M, const Geo& g, size_t* rpc, int* nchunks) {
  const size_t want = (size_t)(wave_blocks() / g.ncb > 0 ? wave_blocks() / g.ncb : 1);
  size_t r = (M + want - 1) / want;
  if (r < (size_t)g.rl * kMinRows) r = (size_t)g.rl * kMinRows;
  r = (r + g.rl - 1) / g.rl * g.rl;
  *rpc = r;
  *nchunks = (int)((M + r - 1) / r);
}

template <class U>
struct Unit {
  static constexpr int kVecs = kCh / U::kPerVec;
  __device__ static __forceinline__ void load(const void* base, size_t unit, float* f) {
    const Vec16* p = reinterpret_cast<const Vec16*>(base) + unit * kVecs;
#pragma unroll
    for (int v = 0; v < kVecs; ++v) U::unpack(ld_stream16(p + v), f + v * U::kPerVec);
  }
  __device__ static __forceinline__ void store(void* base, size_t unit, const float* f) {
    Vec16* p = reinterpret_cast<Vec16*>(base) + unit * kVecs;
#pragma unroll
    for (int v = 0; v < kVecs; ++v) st_stream16(p + v, U::pack(f + v * U::kPerVec));
  }
  // rounds f to the activation dtype, as storing and reloading it would
  __device__ static __forceinline__ void round(float* f) {
#pragma unroll
    for (int v = 0; v < kVecs; ++v) U::unpack(U::pack(f + v * U::kPerVec), f + v * U::kPerVec);
  }
};

__device__ __forceinline__ void welford_push(float& n, float* mean, float* m2, const float* f) {
  n += 1.f;
  const float inv = __frcp_rn(n);
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    const float d = f[k] - mean[k];
    mean[k] = fmaf(d, inv, mean[k]);
    m2[k] = fmaf(d, f[k] - mean[k], m2[k]);
  }
}

// Chan's merge of (nb, mean_b, m2_b) into (n, mean, m2); the count is shared by the K channels.
template <int K>
__device__ __forceinline__ void chan_merge(float& n, float* mean, float* m2, float nb, const float* mb,
                                           const float* m2b) {
  if (nb == 0.f) return;
  if (n == 0.f) {
    n = nb;
#pragma unroll
    for (int k = 0; k < K; ++k) {
      mean[k] = mb[k];
      m2[k] = m2b[k];
    }
    return;
  }
  const float nn = n + nb, fb = nb / nn, w = n * fb;
#pragma unroll
  for (int k = 0; k < K; ++k) {
    const float d = mb[k] - mean[k];
    mean[k] = fmaf(d, fb, mean[k]);
    m2[k] = m2[k] + m2b[k] + d * d * w;
  }
  n = nn;
}

// Fixed-order tree over the `lanes` threads of a column: thread t = lane * cols + col (t == threadIdx.x,
// lanes * cols == kT); the result is in lane 0.  At level s lane L < s takes lane L + s, i.e. thread t + s * cols.
// The levels with s * cols >= 32 pair threads of different warps and go through shared memory, where the senders
// t in [s * cols, 2 s * cols) need only kT / 2 slots; the rest pair threads of warp 0 and use shuffles.
template <int K>
__device__ __forceinline__ void tree_welford(float& n, float* mean, float* m2, int lane, int cols, int lanes) {
  __shared__ float sh[2 * K + 1][kT / 2];
  const int t = threadIdx.x;
  int s = lanes >> 1;
  for (; s * cols >= 32; s >>= 1) {
    __syncthreads();
    if (lane >= s && lane < 2 * s) {
      const int p = t - s * cols;
      sh[0][p] = n;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        sh[1 + k][p] = mean[k];
        sh[1 + K + k][p] = m2[k];
      }
    }
    __syncthreads();
    if (lane < s) {
      float mb[K], m2b[K];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        mb[k] = sh[1 + k][t];
        m2b[k] = sh[1 + K + k][t];
      }
      chan_merge<K>(n, mean, m2, sh[0][t], mb, m2b);
    }
  }
  if (t < 32) {
    for (; s >= 1; s >>= 1) {
      const int d = s * cols;
      const float nb = __shfl_down_sync(0xffffffffu, n, d);
      float mb[K], m2b[K];
#pragma unroll
      for (int k = 0; k < K; ++k) {
        mb[k] = __shfl_down_sync(0xffffffffu, mean[k], d);
        m2b[k] = __shfl_down_sync(0xffffffffu, m2[k], d);
      }
      if (lane < s) chan_merge<K>(n, mean, m2, nb, mb, m2b);
    }
  }
}

// The same tree as tree_welford, adding two K-vectors.
template <int K>
__device__ __forceinline__ void tree_sum2(float* a, float* b, int lane, int cols, int lanes) {
  __shared__ float sh[2 * K][kT / 2];
  const int t = threadIdx.x;
  int s = lanes >> 1;
  for (; s * cols >= 32; s >>= 1) {
    __syncthreads();
    if (lane >= s && lane < 2 * s) {
      const int p = t - s * cols;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        sh[k][p] = a[k];
        sh[K + k][p] = b[k];
      }
    }
    __syncthreads();
    if (lane < s) {
#pragma unroll
      for (int k = 0; k < K; ++k) {
        a[k] += sh[k][t];
        b[k] += sh[K + k][t];
      }
    }
  }
  if (t < 32) {
    for (; s >= 1; s >>= 1) {
      const int d = s * cols;
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float ab = __shfl_down_sync(0xffffffffu, a[k], d), bb = __shfl_down_sync(0xffffffffu, b[k], d);
        if (lane < s) {
          a[k] += ab;
          b[k] += bb;
        }
      }
    }
  }
}

constexpr int kMaxRedCh = 8 * kCh;   // channels of a reduction-layout channel group (red_cb <= 8 units)

// Finalize layout of the last block of a channel group: nc = CB * kCh channels, tpc = kT / nc threads per channel
// (thread t: channel t % nc, lane t / nc).  Each lane sums a fixed stride of the G chunk partials, then a fixed
// tree adds the lanes; every lane of the channel gets the result.
struct Fin {
  int nc, tpc, cl, sub;
  __device__ Fin(int CB) : nc(CB * kCh), tpc(kT / (CB * kCh)), cl(threadIdx.x % (CB * kCh)),
                           sub(threadIdx.x / (CB * kCh)) {}
  __device__ float all_sum(float v) const {
    __shared__ float out[kMaxRedCh];
    float dummy = 0.f;
    tree_sum2<1>(&v, &dummy, sub, nc, tpc);
    __syncthreads();
    if (sub == 0) out[cl] = v;
    __syncthreads();
    return out[cl];
  }
};

// Merge of the G chunk partials (chunk g: rpc rows, the last M - (G - 1) rpc) of channel c with Chan's formula for
// G parts: mean = sum n_g mean_g / M, M2 = sum (M2_g + n_g (mean_g - mean)^2), two fixed-order sums.  ws holds the
// chunk means, then the chunk M2s, G x C each.  Every thread of the block must call it; lanes of c >= C get 0.
__device__ __forceinline__ void merge_stats(const Fin& fin, const float* ws, int G, size_t M, int C, int c,
                                            size_t rpc, float* fmean, float* fm2) {
  const float* ws_mean = ws;
  const float* ws_m2 = ws + (size_t)G * C;
  const bool live = c < C;
  const float rpcf = (float)rpc, last_n = (float)(M - (size_t)(G - 1) * rpc);
  float a = 0.f;
  if (live) {
#pragma unroll 8
    for (int g = fin.sub; g < G; g += fin.tpc) a += (g == G - 1 ? last_n : rpcf) * __ldcg(ws_mean + (size_t)g * C + c);
  }
  const float mean = fin.all_sum(a) / (float)M;
  a = 0.f;
  if (live) {
#pragma unroll 8
    for (int g = fin.sub; g < G; g += fin.tpc) {
      const float d = __ldcg(ws_mean + (size_t)g * C + c) - mean;
      a += __ldcg(ws_m2 + (size_t)g * C + c) + (g == G - 1 ? last_n : rpcf) * d * d;
    }
  }
  *fmean = mean;
  *fm2 = fin.all_sum(a);
}

// kLocal: local-partials mode of synchronised batch norm - save_mean / save_invstd receive this rank's mean and
// M2 over its M rows (M >= 1), and the running statistics are left to bn_sync_kernel.
template <class U, bool kLocal>
__global__ void __launch_bounds__(kT, kBlocksPerSM) bn_act_fwd_stats_kernel(const void* __restrict__ x, size_t M, int C, int shift,
                                                             size_t rpc, float eps, float momentum, float* run_mean,
                                                             float* run_var, float* save_mean, float* save_invstd,
                                                             float* ws, uint32_t* counters) {
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  const size_t r0 = (size_t)blockIdx.x * rpc, r1 = min(M, r0 + rpc);
  float n = 0.f, mean[kCh], m2[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) mean[k] = m2[k] = 0.f;
  if (u < units) {
    size_t r = r0 + lane;
    for (; r + 3 * RL < r1; r += 4 * RL) {
      float f[4][kCh];
#pragma unroll
      for (int j = 0; j < 4; ++j) Unit<U>::load(x, (r + j * RL) * units + u, f[j]);
#pragma unroll
      for (int j = 0; j < 4; ++j) welford_push(n, mean, m2, f[j]);
    }
    for (; r < r1; r += RL) {
      float f[kCh];
      Unit<U>::load(x, r * units + u, f);
      welford_push(n, mean, m2, f);
    }
  }
  tree_welford<kCh>(n, mean, m2, lane, CB, RL);
  const int G = gridDim.x;
  float* ws_mean = ws;
  float* ws_m2 = ws + (size_t)G * C;
  if (lane == 0 && u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      ws_mean[(size_t)blockIdx.x * C + u * kCh + k] = mean[k];
      ws_m2[(size_t)blockIdx.x * C + u * kCh + k] = m2[k];
    }
  }
  if (!last_block(counters + blockIdx.y)) return;

  // The last chunk of this channel group to finish merges the group's G partials.
  const Fin fin(CB);
  const int c = blockIdx.y * fin.nc + fin.cl;
  const bool live = c < C;
  float fmean, fm2;
  merge_stats(fin, ws, G, M, C, c, rpc, &fmean, &fm2);
  if constexpr (kLocal) {
    if (fin.sub == 0 && live) {
      save_mean[c] = fmean;
      save_invstd[c] = fm2;
    }
  } else if (fin.sub == 0 && live) {
    const float invstd = 1.f / sqrtf(fm2 / (float)M + eps);
    save_mean[c] = fmean;
    save_invstd[c] = invstd;
    if (run_mean != nullptr) {
      run_mean[c] = momentum * fmean + (1.f - momentum) * run_mean[c];
      run_var[c] = momentum * (fm2 / (float)(M - 1)) + (1.f - momentum) * run_var[c];
    }
  }
}

// The normalised, scaled and shifted value of x = f before the residual and the activation; every apply forms it so.
__device__ __forceinline__ float bn_value(float f, float mu, float sc, float sh) { return fmaf(f - mu, sc, sh); }

template <class U, bool kRelu, bool kRes>
__device__ __forceinline__ void fwd_row(size_t i, const float* mu, const float* sc, const float* sh, void* y,
                                        uint8_t* mask, const float* f, const float* q) {
  float o[kCh];
  uint32_t bits = 0;
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    float v = bn_value(f[k], mu[k], sc[k], sh[k]);
    if constexpr (kRes) v += q[k];
    if constexpr (kRelu) {
      bits |= (v > 0.f ? 1u : 0u) << k;
      v = v <= 0.f ? 0.f : v;   // NaN propagates, as in torch.relu
    }
    o[k] = v;
  }
  Unit<U>::store(y, i, o);
  if constexpr (kRelu) mask[i] = (uint8_t)bits;
}

template <class U, bool kRelu, bool kRes>
__global__ void __launch_bounds__(kT, kBlocksPerSM) bn_act_fwd_apply_kernel(const void* __restrict__ x, const void* __restrict__ res,
                                                             size_t M, int C, int shift, const float* mean,
                                                             const float* invstd, const float* weight,
                                                             const float* bias, void* y, uint8_t* mask) {
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  if (u >= units) return;
  float mu[kCh], sc[kCh], sh[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    const int c = u * kCh + k;
    mu[k] = mean[c];
    sc[k] = weight[c] * invstd[c];
    sh[k] = bias[c];
  }
  const size_t step = (size_t)gridDim.x * RL;
  for (size_t r = (size_t)blockIdx.x * RL + lane; r < M; r += 2 * step) {
    const size_t i0 = r * units + u, i1 = (r + step) * units + u;
    const bool two = r + step < M;
    float f0[kCh], f1[kCh], q0[kCh], q1[kCh];
    Unit<U>::load(x, i0, f0);
    if constexpr (kRes) Unit<U>::load(res, i0, q0);
    if (two) {
      Unit<U>::load(x, i1, f1);
      if constexpr (kRes) Unit<U>::load(res, i1, q1);
    }
    fwd_row<U, kRelu, kRes>(i0, mu, sc, sh, y, mask, f0, q0);
    if (two) fwd_row<U, kRelu, kRes>(i1, mu, sc, sh, y, mask, f1, q1);
  }
}

template <bool kRelu>
__device__ __forceinline__ void mask_grad(float* d, uint32_t bits) {
  if constexpr (kRelu) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) d[k] = (bits >> k) & 1u ? d[k] : 0.f;
  }
}

template <class U, bool kRelu>
__global__ void __launch_bounds__(kT, kBlocksPerSM) bn_act_bwd_reduce_kernel(const void* __restrict__ dy, const void* __restrict__ x,
                                                              const uint8_t* __restrict__ mask, size_t M, int C,
                                                              int shift, size_t rpc, const float* mean,
                                                              const float* invstd, float* dweight, float* dbias,
                                                              float* ws, uint32_t* counters) {
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  const size_t r0 = (size_t)blockIdx.x * rpc, r1 = min(M, r0 + rpc);
  float sg[kCh], sgx[kCh], mu[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) sg[k] = sgx[k] = 0.f;
  if (u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) mu[k] = mean[u * kCh + k];
    size_t r = r0 + lane;
    for (; r + 3 * RL < r1; r += 4 * RL) {
      float d[4][kCh], f[4][kCh];
      uint32_t bits[4];
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const size_t i = (r + j * RL) * units + u;
        Unit<U>::load(dy, i, d[j]);
        Unit<U>::load(x, i, f[j]);
        if constexpr (kRelu) bits[j] = __ldcs(mask + i);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mask_grad<kRelu>(d[j], bits[j]);
#pragma unroll
        for (int k = 0; k < kCh; ++k) {
          sg[k] += d[j][k];
          sgx[k] = fmaf(d[j][k], f[j][k] - mu[k], sgx[k]);
        }
      }
    }
    for (; r < r1; r += RL) {
      const size_t i = r * units + u;
      float d[kCh], f[kCh];
      Unit<U>::load(dy, i, d);
      Unit<U>::load(x, i, f);
      if constexpr (kRelu) mask_grad<kRelu>(d, __ldcs(mask + i));
#pragma unroll
      for (int k = 0; k < kCh; ++k) {
        sg[k] += d[k];
        sgx[k] = fmaf(d[k], f[k] - mu[k], sgx[k]);
      }
    }
  }
  tree_sum2<kCh>(sg, sgx, lane, CB, RL);
  const int G = gridDim.x;
  float* ws_g = ws;
  float* ws_gx = ws + (size_t)G * C;
  if (lane == 0 && u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      ws_g[(size_t)blockIdx.x * C + u * kCh + k] = sg[k];
      ws_gx[(size_t)blockIdx.x * C + u * kCh + k] = sgx[k];
    }
  }
  if (!last_block(counters + blockIdx.y)) return;

  const Fin fin(CB);
  const int c = blockIdx.y * fin.nc + fin.cl;
  float a = 0.f, b = 0.f;
  if (c < C) {
#pragma unroll 8
    for (int g = fin.sub; g < G; g += fin.tpc) {
      a += __ldcg(ws_g + (size_t)g * C + c);
      b += __ldcg(ws_gx + (size_t)g * C + c);
    }
  }
  tree_sum2<1>(&a, &b, fin.sub, fin.nc, fin.tpc);
  if (fin.sub == 0 && c < C) {
    dbias[c] = a;
    dweight[c] = b * invstd[c];
  }
}

template <class U, bool kRelu, bool kRes>
__device__ __forceinline__ void bwd_row(size_t i, const float* mu, const float* A, const float* D, const float* E,
                                        void* dx, void* dres, float* d, const float* f, uint32_t bits) {
  mask_grad<kRelu>(d, bits);
  float o[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) o[k] = fmaf(A[k], d[k], fmaf(D[k], f[k] - mu[k], E[k]));
  Unit<U>::store(dx, i, o);
  if constexpr (kRes) Unit<U>::store(dres, i, d);
}

// kTotal: divide by *total, the row count of all ranks (synchronised batch norm), instead of M.
template <class U, bool kRelu, bool kRes, bool kTotal>
__global__ void __launch_bounds__(kT, kBwdApplyBlocksPerSM) bn_act_bwd_apply_kernel(const void* __restrict__ dy, const void* __restrict__ x,
                                                             const uint8_t* __restrict__ mask, size_t M, int C,
                                                             int shift, const float* mean, const float* invstd,
                                                             const float* weight, const float* dweight,
                                                             const float* dbias, void* dx, void* dres,
                                                             const float* total) {
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  if (u >= units) return;
  // dx = A * g + D * (x - mean) + E with A = w * invstd, D = -A * invstd * dweight / N, E = -A * dbias / N, where
  // N is the row count of the statistics
  float mu[kCh], A[kCh], D[kCh], E[kCh];
  const float invM = 1.f / (kTotal ? *total : (float)M);
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    const int c = u * kCh + k;
    mu[k] = mean[c];
    A[k] = weight[c] * invstd[c];
    D[k] = -A[k] * invstd[c] * (dweight[c] * invM);
    E[k] = -A[k] * (dbias[c] * invM);
  }
  const size_t step = (size_t)gridDim.x * RL;
  for (size_t r = (size_t)blockIdx.x * RL + lane; r < M; r += 2 * step) {
    const size_t i0 = r * units + u, i1 = (r + step) * units + u;
    const bool two = r + step < M;
    float d0[kCh], d1[kCh], f0[kCh], f1[kCh];
    uint32_t b0 = 0, b1 = 0;
    Unit<U>::load(dy, i0, d0);
    Unit<U>::load(x, i0, f0);
    if constexpr (kRelu) b0 = __ldcs(mask + i0);
    if (two) {
      Unit<U>::load(dy, i1, d1);
      Unit<U>::load(x, i1, f1);
      if constexpr (kRelu) b1 = __ldcs(mask + i1);
    }
    bwd_row<U, kRelu, kRes>(i0, mu, A, D, E, dx, dres, d0, f0, b0);
    if (two) bwd_row<U, kRelu, kRes>(i1, mu, A, D, E, dx, dres, d1, f1, b1);
  }
}

// ---- single-launch passes: reduction, grid barrier, merge and apply in one cooperative launch ----------------
//
// The grid is exactly one wave of kResBlocksPerSM blocks per SM, laid out as the reduction passes: channel group
// blockIdx.y, chunk blockIdx.x of rpc rows, thread (col, lane) on rows lane, lane + RL, ... of the chunk.  The first
// `held` rows of a chunk (a multiple of RL, or the whole chunk) are copied into shared memory in phase 1 and applied
// from there in phase 2; the rest are read from global memory in both phases, the second time in reverse order so
// that what phase 1 read last, the part most likely still in L2, is read first.  Between the phases every block of a
// channel group waits for the group's partials and merges them itself, in the same fixed order, so all of the group's
// blocks get the same bits without a second barrier.
//
// Streamed rows pass through a ring of kStages[bwd] block row-steps in shared memory behind the held rows, fed by
// cp.async: one commit group per row-step, and a thread only ever reads the slots it filled itself, so the ring needs
// no block synchronisation.  Phase 1 pushes a thread's rows in row order (held rows first, as they come first in the
// chunk), so the statistics do not depend on how many rows are held.
//
// Shared memory of a block: held / RL held row-steps, then the ring (fused_layout).
constexpr int kResBlocksPerSM = 2;
constexpr int kFwdStages = 4;
constexpr int kBwdStages = 2;

// The carve-up of a block's dynamic shared memory, in Vec16: `step` per held row-step and `slot` per ring slot.  A
// row-step is kT threads x one unit (kT * V Vec16, V Vec16 per unit), the thread's part at t * V; a block of kT mask
// words (kT / 4 Vec16) holds, at word t, the aligned 4-byte word with the thread's mask byte (mask_copy).
//   forward              held step: x                   slot: x (with a residual, phase 2 pairs slots: x, residual)
//   backward             held step: dy, x, mask words   slot: dy, x, mask words
//   backward, residual   held step: dz, x               slot: dy, dy2, x, mask words (phase 2 uses its dz, x part)
//   backward, pooled     held step: dyi, x              slot: x (dyi is formed from the pooled gradients)
// The pooled forward uses the forward's layout.  The residual backward passes every row through the ring in phase 1,
// so it always has one.  The kernels index shared memory and fused_plan sizes it from this one function.
struct Layout {
  int step, slot;
  bool ring_always;
};
__host__ __device__ constexpr Layout fused_layout(bool bwd, bool res, int V, bool pool = false) {
  return !bwd ? Layout{kT * V, kT * V, false}
         : pool ? Layout{2 * kT * V, kT * V, false}
         : !res ? Layout{2 * kT * V + kT / 4, 2 * kT * V + kT / 4, false}
                : Layout{2 * kT * V, 3 * kT * V + kT / 4, true};
}

__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void cp_async16(void* smem, const void* g) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem, const void* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

// Copies the aligned 4-byte word holding mask byte i to *w; mask_byte extracts the byte again.  A word reaching
// outside the n mask bytes (at most the first and the last) is assembled from the byte alone.
__device__ __forceinline__ void mask_copy(uint32_t* w, const uint8_t* mask, size_t i, size_t n) {
  const uintptr_t a = (uintptr_t)(mask + i), a0 = a & ~(uintptr_t)3;
  if (a0 >= (uintptr_t)mask && a0 + 4 <= (uintptr_t)(mask + n))
    cp_async4(w, reinterpret_cast<const void*>(a0));
  else
    *w = (uint32_t)mask[i] << (8 * (a & 3));
}
__device__ __forceinline__ uint32_t mask_byte(uint32_t w, const uint8_t* mask, size_t i) {
  return (w >> (8 * (((uintptr_t)mask + i) & 3))) & 0xffu;
}

// Runs use(k, slot) for k = 0 .. n - 1 with the copies of step k, started by issue(k, slot), complete: D steps in
// flight, step k in ring slot k % D.  The groups of steps 0 .. D - 1 are the last D the thread committed
// (ring_fill); groups committed before them complete first.
template <int D, class Issue, class Use>
__device__ __forceinline__ void ring_drain(int n, Issue issue, Use use) {
  for (int k = 0; k < n; ++k) {
    cp_async_wait<D - 1>();
    const int slot = k % D;
    use(k, slot);
    if (k + D < n) issue(k + D, slot);
    cp_async_commit();
  }
}
template <int D, class Issue>
__device__ __forceinline__ void ring_fill(int n, Issue issue) {
#pragma unroll 1
  for (int k = 0; k < D; ++k) {
    if (k < n) issue(k, k);
    cp_async_commit();
  }
}

// One-shot barrier of the gridDim.x blocks of a channel group on a zeroed counter.  Only cooperative launches use
// it, so every block is resident and the wait ends; the time limit turns a broken launch into an error, not a hang.
__device__ __forceinline__ void group_barrier(uint32_t* counter) {
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    atomicAdd(counter, 1u);
    const long long t0 = clock64();
    while (ld_acquire_gpu(counter) < gridDim.x) {
      if (clock64() - t0 > kBarrierSpinLimit) {
        printf("byteps_b200: bn_act block (%d, %d) timed out at its grid barrier\n", (int)blockIdx.x, (int)blockIdx.y);
        __trap();
      }
    }
  }
  __syncthreads();
}

template <class U>
__device__ __forceinline__ void hold_load(const Vec16* h, float* f) {
#pragma unroll
  for (int v = 0; v < Unit<U>::kVecs; ++v) U::unpack(lds16(h + v), f + v * U::kPerVec);
}
template <class U>
__device__ __forceinline__ void hold_copy(Vec16* h, const void* base, size_t unit) {
  const Vec16* p = reinterpret_cast<const Vec16*>(base) + unit * Unit<U>::kVecs;
#pragma unroll
  for (int v = 0; v < Unit<U>::kVecs; ++v) cp_async16(h + v, p + v);
}

// ---- the pooled variant: ReLU then max pool (kernel 3, stride 2, padding 1) of the stem
//
// Rows are the pixels (n, h, w) of N images of H x W; the pooled rows (n, oh, ow) of OH x OW, OH = (H - 1) / 2 + 1,
// are ordered the same way, so their window centres (n, 2 oh, 2 ow) increase with the pooled row.  Per unit and
// pooled row the forward writes one 32-bit code word, 4 bits per channel (bits 4k .. 4k + 3: channel 8j + k): the
// window position kh * 3 + kw of the channel's maximum, or kPoolDead when that maximum carries no gradient.
constexpr uint32_t kPoolDead = 0xf;

struct PoolShape {
  int H, W, OH, OW;
  size_t hw, ohw;
  __host__ __device__ PoolShape(int h, int w)
      : H(h), W(w), OH((h - 1) / 2 + 1), OW((w - 1) / 2 + 1), hw((size_t)h * w),
        ohw((size_t)((h - 1) / 2 + 1) * ((w - 1) / 2 + 1)) {}
  // pooled rows whose window centre is a row before r
  __host__ __device__ size_t pooled_before(size_t r) const {
    const size_t n = r / hw;
    const int rem = (int)(r - n * hw), h = rem / W, w = rem - h * W;
    return n * ohw + (size_t)((h + 1) / 2) * OW + (h % 2 == 0 ? (w + 1) / 2 : 0);
  }
  __host__ __device__ void pooled_at(size_t j, size_t* n, int* oh, int* ow) const { split2(j, ohw, OW, n, oh, ow); }
  __host__ __device__ void split(size_t r, size_t* n, int* h, int* w) const { split2(r, hw, W, n, h, w); }
  // i = (n * plane + a) * width + b; 32-bit divisions where i fits, as it does at any practical size
  __host__ __device__ static void split2(size_t i, size_t plane, int width, size_t* n, int* a, int* b) {
    if ((i | plane) <= 0xffffffffu) {
      const uint32_t n32 = (uint32_t)i / (uint32_t)plane, rem = (uint32_t)i - n32 * (uint32_t)plane;
      *n = n32;
      *a = (int)(rem / (uint32_t)width);
      *b = (int)(rem - (uint32_t)*a * (uint32_t)width);
    } else {
      *n = i / plane;
      const int rem = (int)(i - *n * plane);
      *a = rem / width;
      *b = rem - *a * width;
    }
  }
};

// Dynamic shared memory: x of `held` block rows, then the ring (see above).
//
// kPool (with kRelu, without kRes): the rows are images of IH x IW, and phase 2 writes the max pool of y to y (pooled
// rows) and the window codes to pool_code instead of y and the mask; phase 1 is the same as without it.
template <class U, bool kRelu, bool kRes, bool kPool>
__global__ void __launch_bounds__(kT, kResBlocksPerSM) bn_act_fwd_fused_kernel(
    const void* __restrict__ x, const void* __restrict__ res, size_t M, int C, int shift, size_t rpc, int held,
    float eps, float momentum, float* run_mean, float* run_var, float* save_mean, float* save_invstd,
    const float* weight, const float* bias, void* y, uint8_t* mask, float* ws, uint32_t* counters, int IH, int IW,
    uint32_t* pool_code) {
  static_assert(!kPool || (kRelu && !kRes), "the pooled forward is ReLU without a residual");
  extern __shared__ Vec16 hold[];
  constexpr int V = Unit<U>::kVecs, SV = kT * V;   // SV: Vec16 of one row-step
  constexpr Layout L = fused_layout(false, kRes, V);
  __shared__ float s_mu[kMaxRedCh], s_sc[kMaxRedCh];
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  const size_t r0 = (size_t)blockIdx.x * rpc, r1 = min(M, r0 + rpc);
  const int rows = (int)(r1 - r0), nh = min(held, rows);
  // this thread's held and streamed rows (row-steps), their first units and the units between two of them
  const int hn = lane < nh ? (nh - 1 - lane) / RL + 1 : 0;
  const int sn = lane < rows - nh ? (rows - nh - 1 - lane) / RL + 1 : 0;
  const size_t i_h = (r0 + lane) * units + u, i_s = i_h + (size_t)nh * units, ustep = (size_t)RL * units;
  static_assert(L.step == SV && L.slot == SV, "the forward indexes held steps and ring slots of one row-step");
  Vec16* hx = hold + threadIdx.x * V;                                      // held step k at hx + k * SV
  Vec16* ring = hold + (size_t)(held / RL) * L.step + threadIdx.x * V;     // ring slot j at ring + j * SV

  // phase 1: Welford over the thread's rows in row order, the held ones copied to shared memory on the way
  float n = 0.f, mean[kCh], m2[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) mean[k] = m2[k] = 0.f;
  if (u < units) {
    for (int k = 0; k < hn; ++k) hold_copy<U>(hx + (size_t)k * SV, x, i_h + k * ustep);
    cp_async_commit();
    auto issue = [&](int k, int slot) { hold_copy<U>(ring + slot * SV, x, i_s + k * ustep); };
    ring_fill<kFwdStages>(sn, issue);
    cp_async_wait<kFwdStages>();
    for (int k = 0; k < hn; ++k) {
      float f[kCh];
      hold_load<U>(hx + (size_t)k * SV, f);
      welford_push(n, mean, m2, f);
    }
    ring_drain<kFwdStages>(sn, issue, [&](int, int slot) {
      float f[kCh];
      hold_load<U>(ring + slot * SV, f);
      welford_push(n, mean, m2, f);
    });
  }
  tree_welford<kCh>(n, mean, m2, lane, CB, RL);
  const int G = gridDim.x;
  if (lane == 0 && u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      ws[(size_t)blockIdx.x * C + u * kCh + k] = mean[k];
      ws[((size_t)G + blockIdx.x) * C + u * kCh + k] = m2[k];
    }
  }
  group_barrier(counters + blockIdx.y);

  const Fin fin(CB);
  const int c = blockIdx.y * fin.nc + fin.cl;
  float fmean, fm2;
  merge_stats(fin, ws, G, M, C, c, rpc, &fmean, &fm2);
  if (fin.sub == 0 && c < C) {
    const float invstd = 1.f / sqrtf(fm2 / (float)M + eps);
    s_mu[fin.cl] = fmean;
    s_sc[fin.cl] = weight[c] * invstd;
    if (blockIdx.x == 0) {
      save_mean[c] = fmean;
      save_invstd[c] = invstd;
      if (run_mean != nullptr) {
        run_mean[c] = momentum * fmean + (1.f - momentum) * run_mean[c];
        run_var[c] = momentum * (fm2 / (float)(M - 1)) + (1.f - momentum) * run_var[c];
      }
    }
  }
  __syncthreads();
  if (u >= units) return;

  // phase 2: streamed rows, last read first, then the held rows.  The ring carries x of the streamed rows and, with
  // a residual, the residual of every row, in pairs of slots.  A block holding its whole chunk has no ring and reads
  // the residual directly.
  float mu[kCh], sc[kCh], sh[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    mu[k] = s_mu[col * kCh + k];
    sc[k] = s_sc[col * kCh + k];
    sh[k] = bias[u * kCh + k];
  }
  if constexpr (kPool) {
    // The block's pooled outputs: those whose window centre (n, 2 oh, 2 ow) lies in the chunk, a contiguous range
    // [p0, p1) of the pooled rows, walked in order so that the image lines a step reads are read again by the next
    // steps while still in L1 / L2.  A window row the block holds comes from shared memory (held row r0 + i of
    // column col sits at ((i * CB + col) * V), any other, halo rows of the neighbouring chunks included, from global
    // memory: x is read-only, so no synchronisation is needed.  y is formed as fwd_row forms it and rounded to the
    // activation dtype; the maximum is picked as torch's NHWC max pool does (window scanned row-major, strict >, a
    // NaN always taken).  The code of a channel is the winner's window position, or kPoolDead when the winner's
    // ReLU mask bit would be 0 (y <= 0 before the ReLU), where the stock chain's gradient ends.
    const PoolShape ps(IH, IW);
    const size_t p0 = ps.pooled_before(r0), p1 = ps.pooled_before(r1);
    for (size_t j = p0 + lane; j < p1; j += RL) {
      size_t n;
      int oh, ow;
      ps.pooled_at(j, &n, &oh, &ow);
      float best[kCh];
      uint32_t code = 0, live = 0;
#pragma unroll
      for (int k = 0; k < kCh; ++k) best[k] = -INFINITY;
      // QB window positions at a time, their loads in flight together (generic loads: shared or global memory)
      constexpr int QB = V == 1 ? 9 : 3;
#pragma unroll
      for (int q0 = 0; q0 < 9; q0 += QB) {
        Vec16 raw[QB][V];
#pragma unroll
        for (int q = q0; q < q0 + QB; ++q) {
          const int h = 2 * oh - 1 + q / 3, w = 2 * ow - 1 + q % 3;
          if (h < 0 || h >= IH || w < 0 || w >= IW) continue;
          const size_t r = n * ps.hw + (size_t)h * IW + w;
          const uint4* src = r - r0 < (size_t)nh ? reinterpret_cast<const uint4*>(hold + ((r - r0) * CB + col) * V)
                                                : reinterpret_cast<const uint4*>(x) + (r * units + u) * V;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            const uint4 t = src[v];
            raw[q - q0][v] = Vec16{t.x, t.y, t.z, t.w};
          }
        }
#pragma unroll
        for (int q = q0; q < q0 + QB; ++q) {
          const int h = 2 * oh - 1 + q / 3, w = 2 * ow - 1 + q % 3;
          if (h < 0 || h >= IH || w < 0 || w >= IW) continue;
          float f[kCh], v[kCh], o[kCh];
#pragma unroll
          for (int e = 0; e < V; ++e) U::unpack(raw[q - q0][e], f + e * U::kPerVec);
#pragma unroll
          for (int k = 0; k < kCh; ++k) {
            v[k] = bn_value(f[k], mu[k], sc[k], sh[k]);
            o[k] = v[k] <= 0.f ? 0.f : v[k];   // as fwd_row's ReLU
          }
          Unit<U>::round(o);
#pragma unroll
          for (int k = 0; k < kCh; ++k) {
            if (o[k] > best[k] || isnan(o[k])) {
              best[k] = o[k];
              code = (code & ~(0xfu << (4 * k))) | (uint32_t)q << (4 * k);
              live = (live & ~(1u << k)) | (v[k] > 0.f ? 1u : 0u) << k;
            }
          }
        }
      }
#pragma unroll
      for (int k = 0; k < kCh; ++k)
        if (!((live >> k) & 1u)) code |= kPoolDead << (4 * k);
      Unit<U>::store(y, j * units + u, best);
      pool_code[j * units + u] = code;
    }
    return;
  }
  constexpr int W = kRes ? 2 : 1, D2 = kFwdStages / W;
  const int n2 = sn + (kRes && (size_t)held < rpc ? hn : 0);
  auto unit2 = [&](int k) { return k < sn ? i_s + (size_t)(sn - 1 - k) * ustep : i_h + (size_t)(k - sn) * ustep; };
  auto issue2 = [&](int k, int slot) {
    const size_t i = unit2(k);
    if (k < sn) hold_copy<U>(ring + slot * W * SV, x, i);
    if constexpr (kRes) hold_copy<U>(ring + (slot * W + 1) * SV, res, i);
  };
  ring_fill<D2>(n2, issue2);
  ring_drain<D2>(n2, issue2, [&](int k, int slot) {
    float f[kCh], q[kCh];
    hold_load<U>(k < sn ? ring + slot * W * SV : hx + (size_t)(k - sn) * SV, f);
    if constexpr (kRes) hold_load<U>(ring + (slot * W + 1) * SV, q);
    fwd_row<U, kRelu, kRes>(unit2(k), mu, sc, sh, y, mask, f, q);
  });
  for (int k = n2 - sn; k < hn; k += 2) {   // the held rows the ring did not carry
    const size_t i0 = i_h + k * ustep, i1 = i0 + ustep;
    const bool two = k + 1 < hn;
    float f0[kCh], f1[kCh], q0[kCh], q1[kCh];
    if constexpr (kRes) {
      Unit<U>::load(res, i0, q0);
      if (two) Unit<U>::load(res, i1, q1);
    }
    hold_load<U>(hx + (size_t)k * SV, f0);
    fwd_row<U, kRelu, kRes>(i0, mu, sc, sh, y, mask, f0, q0);
    if (two) {
      hold_load<U>(hx + (size_t)(k + 1) * SV, f1);
      fwd_row<U, kRelu, kRes>(i1, mu, sc, sh, y, mask, f1, q1);
    }
  }
}

// Between the phases of a single-launch backward: the block's sums of g and g * (x - mean) (sg, sgx of the thread)
// are reduced, the channel group's blocks meet at the grid barrier, each merges the G partials in the same fixed
// order and derives bwd_apply's coefficients dx = A * g + D * (x - mean) + E of the thread's channels; block 0 writes
// dweight and dbias.  Returns false for a thread without a unit (u >= units), which has nothing left to do.
__device__ __forceinline__ bool bwd_coefficients(float* sg, float* sgx, int lane, int col, int CB, int RL, int u,
                                                 int units, size_t M, int C, const float* invstd, const float* weight,
                                                 float* dweight, float* dbias, float* ws, uint32_t* counters, float* A,
                                                 float* D, float* E) {
  __shared__ float s_A[kMaxRedCh], s_D[kMaxRedCh], s_E[kMaxRedCh];
  tree_sum2<kCh>(sg, sgx, lane, CB, RL);
  const int G = gridDim.x;
  if (lane == 0 && u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      ws[(size_t)blockIdx.x * C + u * kCh + k] = sg[k];
      ws[((size_t)G + blockIdx.x) * C + u * kCh + k] = sgx[k];
    }
  }
  group_barrier(counters + blockIdx.y);

  const Fin fin(CB);
  const int c = blockIdx.y * fin.nc + fin.cl;
  float a = 0.f, b = 0.f;
  if (c < C) {
#pragma unroll 8
    for (int g = fin.sub; g < G; g += fin.tpc) {
      a += __ldcg(ws + (size_t)g * C + c);
      b += __ldcg(ws + ((size_t)G + g) * C + c);
    }
  }
  tree_sum2<1>(&a, &b, fin.sub, fin.nc, fin.tpc);
  if (fin.sub == 0 && c < C) {
    // the coefficients of bwd_apply, from the same sums
    const float is = invstd[c], db = a, dw = b * is, invM = 1.f / (float)M;
    const float a_ = weight[c] * is;
    s_A[fin.cl] = a_;
    s_D[fin.cl] = -a_ * is * (dw * invM);
    s_E[fin.cl] = -a_ * (db * invM);
    if (blockIdx.x == 0) {
      dbias[c] = db;
      dweight[c] = dw;
    }
  }
  __syncthreads();
  if (u >= units) return false;
#pragma unroll
  for (int k = 0; k < kCh; ++k) {
    A[k] = s_A[col * kCh + k];
    D[k] = s_D[col * kCh + k];
    E[k] = s_E[col * kCh + k];
  }
  return true;
}

// Dynamic shared memory: `held` block rows, then the ring (fused_layout).
//
// Without a residual, phase 1 copies dy, x and the mask word of the held rows to shared memory and streams the
// rest through the ring; phase 2 applies the held rows from there and streams the others again.
//
// With a residual (kRes), phase 1 passes every row through the ring in row order and forms the gradient at the
// junction, dz = round(dy + dy2) * mask (dy2: the optional second gradient, summed in fp32 and rounded once to the
// activation dtype as torch's add does).  It writes dz to dres for every row, and a held row keeps dz and x in shared
// memory.  Phase 2 reads dz back from dres, with x, for the streamed rows: a re-read of two tensors instead of dy,
// dy2 and the mask.
template <class U, bool kRelu, bool kRes>
__global__ void __launch_bounds__(kT, kResBlocksPerSM) bn_act_bwd_fused_kernel(
    const void* __restrict__ dy, const void* __restrict__ dy2, const void* __restrict__ x,
    const uint8_t* __restrict__ mask, size_t M, int C, int shift, size_t rpc, int held, const float* mean,
    const float* invstd, const float* weight, float* dweight, float* dbias, void* dx, void* dres, float* ws,
    uint32_t* counters) {
  extern __shared__ Vec16 hold[];
  // SV: Vec16 of one row-step of dy or x; MW: offset of the mask words in a non-residual held step or ring slot
  constexpr int V = Unit<U>::kVecs, SV = kT * V, MW = 2 * SV;
  constexpr Layout L = fused_layout(true, kRes, V);
  static_assert(kRes || (L.step == MW + kT / 4 && L.slot == L.step), "dy, x, mask words");
  static_assert(!kRes || (L.step == 2 * SV && L.slot == 3 * SV + kT / 4), "dz, x | dy, dy2, x, mask words");
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  const size_t r0 = (size_t)blockIdx.x * rpc, r1 = min(M, r0 + rpc);
  const int rows = (int)(r1 - r0), nh = min(held, rows);
  const int hn = lane < nh ? (nh - 1 - lane) / RL + 1 : 0;
  const int sn = lane < rows - nh ? (rows - nh - 1 - lane) / RL + 1 : 0;
  float A[kCh], D[kCh], E[kCh];
  // row-step k of the thread (held ones first) is unit i_h + k * ustep; the streamed ones start at i_s
  const size_t i_h = (r0 + lane) * units + u, i_s = i_h + (size_t)nh * units, ustep = (size_t)RL * units;
  const size_t nm = M * units;
  const int t = threadIdx.x;
  const size_t hs = (size_t)(held / RL);
  Vec16* hst = hold + t * V;               // the thread's part of held step k at hst + k * L.step
  Vec16* ring = hold + hs * L.step + t * V;   // of ring slot j at ring + j * L.slot
  // the thread's mask word in a step or slot whose mask words start `off` Vec16 into it (p: the thread's part)
  auto word = [&](Vec16* p, int off) { return reinterpret_cast<uint32_t*>(p - t * V + off) + t; };
  auto issue_at = [&](int j, size_t i) {   // non-residual ring slot: dy, x, mask word
    Vec16* s = ring + j * L.slot;
    hold_copy<U>(s, dy, i);
    hold_copy<U>(s + SV, x, i);
    if constexpr (kRelu) mask_copy(word(s, MW), mask, i, nm);
  };

  // phase 1: the thread's rows in row order
  float sg[kCh], sgx[kCh], mu[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) sg[k] = sgx[k] = 0.f;
  auto push = [&](const float* d, const float* f) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      sg[k] += d[k];
      sgx[k] = fmaf(d[k], f[k] - mu[k], sgx[k]);
    }
  };
  if (u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) mu[k] = mean[u * kCh + k];
    if constexpr (kRes) {
      // ring slot: dy, dy2, x, then the mask words at 3 * SV
      auto issue = [&](int k, int slot) {
        const size_t i = i_h + k * ustep;
        Vec16* s = ring + slot * L.slot;
        hold_copy<U>(s, dy, i);
        if (dy2 != nullptr) hold_copy<U>(s + SV, dy2, i);
        hold_copy<U>(s + 2 * SV, x, i);
        if constexpr (kRelu) mask_copy(word(s, 3 * SV), mask, i, nm);
      };
      const int n1 = hn + sn;
      ring_fill<kBwdStages>(n1, issue);
      ring_drain<kBwdStages>(n1, issue, [&](int k, int slot) {
        const size_t i = i_h + k * ustep;
        Vec16* s = ring + slot * L.slot;
        float d[kCh], f[kCh];
        hold_load<U>(s, d);
        if (dy2 != nullptr) {
          float e[kCh];
          hold_load<U>(s + SV, e);
#pragma unroll
          for (int c = 0; c < kCh; ++c) d[c] += e[c];
        }
        if constexpr (kRelu) mask_grad<kRelu>(d, mask_byte(*word(s, 3 * SV), mask, i));
        Vec16 z[V], xv[V];
#pragma unroll
        for (int v = 0; v < V; ++v) {
          z[v] = U::pack(d + v * U::kPerVec);   // the rounding of torch's add; exact when there is no dy2
          U::unpack(z[v], d + v * U::kPerVec);
          st_stream16(reinterpret_cast<Vec16*>(dres) + i * V + v, z[v]);
          xv[v] = lds16(s + 2 * SV + v);
          U::unpack(xv[v], f + v * U::kPerVec);
        }
        push(d, f);
        if (k < hn) {
          Vec16* h = hst + (size_t)k * L.step;
#pragma unroll
          for (int v = 0; v < V; ++v) {
            sts16(h + v, z[v]);
            sts16(h + SV + v, xv[v]);
          }
        }
      });
    } else {
      // held rows copied to shared memory on the way
      for (int k = 0; k < hn; ++k) {
        const size_t i = i_h + k * ustep;
        Vec16* h = hst + (size_t)k * L.step;
        hold_copy<U>(h, dy, i);
        hold_copy<U>(h + SV, x, i);
        if constexpr (kRelu) mask_copy(word(h, MW), mask, i, nm);
      }
      cp_async_commit();
      auto issue = [&](int k, int slot) { issue_at(slot, i_s + k * ustep); };
      ring_fill<kBwdStages>(sn, issue);
      cp_async_wait<kBwdStages>();
      auto push_smem = [&](Vec16* p, size_t i) {
        float d[kCh], f[kCh];
        hold_load<U>(p, d);
        hold_load<U>(p + SV, f);
        if constexpr (kRelu) mask_grad<kRelu>(d, mask_byte(*word(p, MW), mask, i));
        push(d, f);
      };
      for (int k = 0; k < hn; ++k) push_smem(hst + (size_t)k * L.step, i_h + k * ustep);
      ring_drain<kBwdStages>(sn, issue, [&](int k, int slot) { push_smem(ring + slot * L.slot, i_s + k * ustep); });
    }
  }
  if (!bwd_coefficients(sg, sgx, lane, col, CB, RL, u, units, M, C, invstd, weight, dweight, dbias, ws, counters, A,
                        D, E))
    return;
  // phase 2: streamed rows through the ring, last read first, then the held rows.  With a residual a slot carries
  // dz (read back from dres) and x, and the held rows hold dz: the mask is already applied.
  auto unit2 = [&](int k) { return i_s + (size_t)(sn - 1 - k) * ustep; };
  auto issue2 = [&](int k, int slot) {
    if constexpr (kRes) {
      // This thread stored dres at unit i itself in phase 1, before group_barrier, with a store that does not
      // allocate in L1; the copy below is issued after it in program order, to the same address, and reads through
      // L2 (cp.async.cg), so it returns what the thread stored.  No other thread writes this unit.
      const size_t i = unit2(k);
      Vec16* s = ring + slot * L.slot;
      hold_copy<U>(s, dres, i);
      hold_copy<U>(s + SV, x, i);
    } else {
      issue_at(slot, unit2(k));
    }
  };
  auto apply = [&](Vec16* p, size_t i) {
    float d[kCh], f[kCh];
    hold_load<U>(p, d);
    hold_load<U>(p + SV, f);
    if constexpr (kRes)
      bwd_row<U, false, false>(i, mu, A, D, E, dx, nullptr, d, f, 0u);
    else
      bwd_row<U, kRelu, false>(i, mu, A, D, E, dx, nullptr, d, f, kRelu ? mask_byte(*word(p, MW), mask, i) : 0u);
  };
  ring_fill<kBwdStages>(sn, issue2);
  ring_drain<kBwdStages>(sn, issue2, [&](int k, int slot) { apply(ring + slot * L.slot, unit2(k)); });
  for (int k = 0; k < hn; ++k) apply(hst + (size_t)k * L.step, i_h + k * ustep);
}

// The pooled backward (ReLU, no residual), in the chunking and row order of bn_act_bwd_fused_kernel.  The gradient
// reaching row (n, h, w) of y is
//   dyi = round(sum of g over the 1, 2 or 4 windows covering the row whose code names its position, in ascending
//               (oh, ow) order, in fp32 from 0),   g = round(g1 + g2) of the window (g1 when g2 is nullptr),
// which is what torch's add of the two pooled gradients, its NHWC max-pool backward and the ReLU mask give: a window
// whose maximum carries no gradient is dead, and so is every window naming a row the ReLU zeroed.  Phase 1 forms dyi
// from the pooled tensors (a quarter of the rows, mostly in L2) and keeps dyi and x of the held rows in shared memory;
// phase 2 forms dyi again for the streamed rows, whose x comes through the ring.
template <class U>
__global__ void __launch_bounds__(kT, kResBlocksPerSM) bn_act_bwd_pool_kernel(
    const void* __restrict__ g1, const void* __restrict__ g2, const uint32_t* __restrict__ pool_code,
    const void* __restrict__ x, size_t M, int C, int shift, size_t rpc, int held, int H, int W, const float* mean,
    const float* invstd, const float* weight, float* dweight, float* dbias, void* dx, float* ws, uint32_t* counters) {
  extern __shared__ Vec16 hold[];
  constexpr int V = Unit<U>::kVecs, SV = kT * V;
  constexpr Layout L = fused_layout(true, false, V, true);
  static_assert(L.step == 2 * SV && L.slot == SV, "held step: dyi, x; ring slot: x");
  const int units = C / kCh, CB = 1 << shift, RL = kT >> shift;
  const int col = threadIdx.x & (CB - 1), lane = threadIdx.x >> shift;
  const int u = blockIdx.y * CB + col;
  const size_t r0 = (size_t)blockIdx.x * rpc, r1 = min(M, r0 + rpc);
  const int rows = (int)(r1 - r0), nh = min(held, rows);
  const int hn = lane < nh ? (nh - 1 - lane) / RL + 1 : 0;
  const int sn = lane < rows - nh ? (rows - nh - 1 - lane) / RL + 1 : 0;
  Vec16* hst = hold + threadIdx.x * V;                                   // held step k at hst + k * L.step
  Vec16* ring = hold + (size_t)(held / RL) * L.step + threadIdx.x * V;   // ring slot j at ring + j * L.slot
  const PoolShape ps(H, W);
  // dyi of row (n, h, w), unit u.  The covering windows are among (h / 2 + a, w / 2 + b), a, b in {0, 1}, taken in
  // that (ascending) order; their codes are loaded together, then the gradients of the windows that name the row.
  const size_t jrow = (size_t)ps.OW * units;
  auto grad = [&](size_t r, float* d) {
    size_t n;
    int h, w;
    ps.split(r, &n, &h, &w);
    const int oh = h >> 1, ow = w >> 1;
    const bool h2 = (h & 1) && oh + 1 < ps.OH, w2 = (w & 1) && ow + 1 < ps.OW;
    const size_t j0 = (n * ps.ohw + (size_t)oh * ps.OW + ow) * units + u;
    uint32_t cw[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const bool ok = (q & 2 ? h2 : true) && (q & 1 ? w2 : true);
      cw[q] = ok ? __ldg(pool_code + j0 + (q & 2 ? jrow : 0) + (q & 1 ? units : 0)) : 0xffffffffu;
    }
    uint32_t hit[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t pos = (uint32_t)((h - 2 * (oh + (q >> 1)) + 1) * 3 + (w - 2 * (ow + (q & 1)) + 1));
      hit[q] = 0;
#pragma unroll
      for (int k = 0; k < kCh; ++k) hit[q] |= (((cw[q] >> (4 * k)) & 0xfu) == pos ? 1u : 0u) << k;
    }
#pragma unroll
    for (int k = 0; k < kCh; ++k) d[k] = 0.f;
    constexpr int QB = V == 1 ? 4 : 2;   // windows whose gradient loads are in flight together
#pragma unroll
    for (int q0 = 0; q0 < 4; q0 += QB) {
      Vec16 a[QB][V], b[QB][V];
#pragma unroll
      for (int q = q0; q < q0 + QB; ++q) {
        if (hit[q] == 0) continue;
        const size_t j = j0 + (q & 2 ? jrow : 0) + (q & 1 ? units : 0);
        const uint4* p1 = reinterpret_cast<const uint4*>(g1) + j * V;
        const uint4* p2 = reinterpret_cast<const uint4*>(g2) + j * V;
#pragma unroll
        for (int v = 0; v < V; ++v) {
          const uint4 t = __ldg(p1 + v);
          a[q - q0][v] = Vec16{t.x, t.y, t.z, t.w};
          if (g2 != nullptr) {
            const uint4 e = __ldg(p2 + v);
            b[q - q0][v] = Vec16{e.x, e.y, e.z, e.w};
          }
        }
      }
#pragma unroll
      for (int q = q0; q < q0 + QB; ++q) {
        if (hit[q] == 0) continue;
        float g[kCh];
#pragma unroll
        for (int v = 0; v < V; ++v) U::unpack(a[q - q0][v], g + v * U::kPerVec);
        if (g2 != nullptr) {
          float e[kCh];
#pragma unroll
          for (int v = 0; v < V; ++v) U::unpack(b[q - q0][v], e + v * U::kPerVec);
#pragma unroll
          for (int k = 0; k < kCh; ++k) g[k] += e[k];
          Unit<U>::round(g);   // torch's add at the junction
        }
#pragma unroll
        for (int k = 0; k < kCh; ++k)
          if ((hit[q] >> k) & 1u) d[k] += g[k];
      }
    }
    Unit<U>::round(d);
  };

  // phase 1: the thread's rows in row order, x of the held ones copied to shared memory, their dyi stored beside it
  float sg[kCh], sgx[kCh], mu[kCh];
#pragma unroll
  for (int k = 0; k < kCh; ++k) sg[k] = sgx[k] = 0.f;
  auto push = [&](const float* d, const float* f) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) {
      sg[k] += d[k];
      sgx[k] = fmaf(d[k], f[k] - mu[k], sgx[k]);
    }
  };
  const size_t row_h = r0 + lane, row_s = r0 + nh + lane;   // the thread's first held and first streamed row
  if (u < units) {
#pragma unroll
    for (int k = 0; k < kCh; ++k) mu[k] = mean[u * kCh + k];
    for (int k = 0; k < hn; ++k) hold_copy<U>(hst + (size_t)k * L.step + SV, x, (row_h + (size_t)k * RL) * units + u);
    cp_async_commit();
    auto issue = [&](int k, int slot) { hold_copy<U>(ring + slot * L.slot, x, (row_s + (size_t)k * RL) * units + u); };
    ring_fill<kBwdStages>(sn, issue);
    cp_async_wait<kBwdStages>();
    for (int k = 0; k < hn; ++k) {
      Vec16* p = hst + (size_t)k * L.step;
      float d[kCh], f[kCh];
      grad(row_h + (size_t)k * RL, d);
      hold_load<U>(p + SV, f);
      push(d, f);
#pragma unroll
      for (int v = 0; v < V; ++v) sts16(p + v, U::pack(d + v * U::kPerVec));
    }
    ring_drain<kBwdStages>(sn, issue, [&](int k, int slot) {
      float d[kCh], f[kCh];
      grad(row_s + (size_t)k * RL, d);
      hold_load<U>(ring + slot * L.slot, f);
      push(d, f);
    });
  }
  float A[kCh], D[kCh], E[kCh];
  if (!bwd_coefficients(sg, sgx, lane, col, CB, RL, u, units, M, C, invstd, weight, dweight, dbias, ws, counters, A,
                        D, E))
    return;

  // phase 2: streamed rows through the ring, last read first, then the held rows
  auto row2 = [&](int k) { return row_s + (size_t)(sn - 1 - k) * RL; };
  auto issue2 = [&](int k, int slot) { hold_copy<U>(ring + slot * L.slot, x, row2(k) * units + u); };
  ring_fill<kBwdStages>(sn, issue2);
  ring_drain<kBwdStages>(sn, issue2, [&](int k, int slot) {
    const size_t r = row2(k);
    float d[kCh], f[kCh];
    grad(r, d);
    hold_load<U>(ring + slot * L.slot, f);
    bwd_row<U, false, false>(r * units + u, mu, A, D, E, dx, nullptr, d, f, 0u);
  });
  for (int k = 0; k < hn; ++k) {
    Vec16* p = hst + (size_t)k * L.step;
    float d[kCh], f[kCh];
    hold_load<U>(p, d);
    hold_load<U>(p + SV, f);
    bwd_row<U, false, false>((row_h + (size_t)k * RL) * units + u, mu, A, D, E, dx, nullptr, d, f, 0u);
  }
}

// ---- synchronised batch norm: the cross-rank step between the local reduction and the apply pass -------------
//
// Window of one rank (float offsets from its base): slot (parity p, source rank r) at (p * W + r) * slot, with
// slot = kSyncPad + 2 * cmax floats: [counts: one 16-byte vector per block][a: cmax][b: cmax].  Block k owns the
// channel steps k, k + gridDim.x, ... of kSyncStep channels.  gridDim.x is min(steps, kMaxSyncBlocks), so step j
// is always owned by block j % kMaxSyncBlocks whatever C is, and a window area is only ever written by blocks
// with one blockIdx.x, under that block's barrier generation.
//
// Slot reuse.  A block works in the slots of parity g & 1, g being its barrier generation in device memory
// (epoch[channel][block]); every rank runs the same sequence of sync launches, so the counterparts of a block on
// all ranks are at the same generation when they meet.  The block of participation j on rank A writes A's slot in
// every peer's window before barrier j, and reads its own window after it.  A peer block can be at most one
// participation ahead: to pass barrier j + 1 it needs this block at j + 1, which this rank's stream starts only
// after participation j has finished.  So a peer writing participation j + 1 (parity flipped) can overlap this
// block's reads of participation j, but nothing writes parity j & 1 again until those reads are done.
constexpr int kSyncT = 64;                       // threads of a sync block; a thread owns 4 channels
constexpr int kSyncStep = kSyncT * 4;            // channels per block step
constexpr int kMaxSyncBlocks = 8;
constexpr int kSyncPad = 4 * kMaxSyncBlocks;     // floats of the count vectors at the head of a slot

__device__ __forceinline__ Vec16 ld_vec4(const float* p) { return *reinterpret_cast<const Vec16*>(p); }
__device__ __forceinline__ void unpack4(const Vec16& v, float* f) { TagF32::unpack(v, f); }

// kStats: push (M_r, mean, M2), merge in rank order with Chan's formula and write mean, invstd, the running
// statistics and the total count.  Otherwise: push (dbias, dweight) partials and write their rank-ordered sums.
template <bool kStats>
__global__ void __launch_bounds__(kSyncT) bn_sync_kernel(PeerView pv, int channel, size_t win_off, int cmax, int C,
                                                         const float* __restrict__ a_in,
                                                         const float* __restrict__ b_in, float count, float eps,
                                                         float momentum, float* run_mean, float* run_var,
                                                         float* out_a, float* out_b, float* total) {
  const int W = pv.world, me = pv.rank;
  const size_t slot = kSyncPad + 2 * (size_t)cmax;
  const size_t par = pv.epoch[channel * kMaxBlocks + blockIdx.x] & 1u;
  const size_t mine = (par * W + me) * slot;
  for (int c = (blockIdx.x * kSyncT + threadIdx.x) * 4; c < C; c += gridDim.x * kSyncStep) {
    const Vec16 va = ld_vec4(a_in + c), vb = ld_vec4(b_in + c);
    for (int p = 0; p < W; ++p) {
      float* dst = reinterpret_cast<float*>(pv.data[p] + win_off) + mine + kSyncPad;
      st_peer16(dst + c, va);
      st_peer16(dst + cmax + c, vb);
    }
  }
  if (kStats && threadIdx.x < W) {
    float* dst = reinterpret_cast<float*>(pv.data[threadIdx.x] + win_off) + mine + 4 * blockIdx.x;
    st_peer16(dst, Vec16{__float_as_uint(count), 0u, 0u, 0u});
  }
  barrier_peers(pv, channel);

  const float* win = reinterpret_cast<const float*>(pv.data[me] + win_off) + par * W * slot;
  for (int c = (blockIdx.x * kSyncT + threadIdx.x) * 4; c < C; c += gridDim.x * kSyncStep) {
    float n = 0.f, a[4] = {0.f, 0.f, 0.f, 0.f}, b[4] = {0.f, 0.f, 0.f, 0.f};
    for (int r = 0; r < W; ++r) {
      const float* s = win + r * slot;
      float ra[4], rb[4];
      unpack4(ld_peer16(s + kSyncPad + c), ra);
      unpack4(ld_peer16(s + kSyncPad + cmax + c), rb);
      if constexpr (kStats) {
        chan_merge<4>(n, a, b, __uint_as_float(ld_peer16(s + 4 * blockIdx.x).x), ra, rb);
      } else {
#pragma unroll
        for (int k = 0; k < 4; ++k) {
          a[k] += ra[k];
          b[k] += rb[k];
        }
      }
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      if constexpr (kStats) {
        out_a[c + k] = a[k];
        out_b[c + k] = 1.f / sqrtf(b[k] / n + eps);
        if (run_mean != nullptr) {
          run_mean[c + k] = momentum * a[k] + (1.f - momentum) * run_mean[c + k];
          run_var[c + k] = momentum * (b[k] / (n - 1.f)) + (1.f - momentum) * run_var[c + k];
        }
      } else {
        out_a[c + k] = a[k];
        out_b[c + k] = b[k];
      }
    }
    if (kStats && c == 0) *total = n;
  }
}

#define BN_DISPATCH_U(dtype, STMT)              \
  switch (dtype) {                              \
    case WIRE_F32: { using U = TagF32; STMT; } break;   \
    case WIRE_BF16: { using U = TagBF16; STMT; } break; \
    case WIRE_F16: { using U = TagF16; STMT; } break;   \
    default: return cudaErrorInvalidValue;      \
  }
#define BN_DISPATCH_B(flag, NAME, STMT) \
  if (flag) {                           \
    constexpr bool NAME = true;         \
    STMT;                               \
  } else {                              \
    constexpr bool NAME = false;        \
    STMT;                               \
  }

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

bool bad_shape(size_t M, int C) { return M < 1 || C < kCh || C % kCh != 0; }

int apply_grid(size_t M, const Geo& g, int per_sm) {
  const size_t want = (size_t)(wave_blocks(per_sm) / g.ncb > 0 ? wave_blocks(per_sm) / g.ncb : 1);
  const size_t most = (M + 2 * (size_t)g.rl - 1) / (2 * (size_t)g.rl);
  return (int)(most < want ? (most < 1 ? 1 : most) : want);
}

// ---- single-launch host side
constexpr int kMaxDevices = 64;

int dtype_index(int dtype) { return dtype == WIRE_F32 ? 0 : dtype == WIRE_BF16 ? 1 : dtype == WIRE_F16 ? 2 : -1; }

using FusedFwd = void (*)(const void*, const void*, size_t, int, int, size_t, int, float, float, float*, float*,
                          float*, float*, const float*, const float*, void*, uint8_t*, float*, uint32_t*, int, int,
                          uint32_t*);
using FusedBwd = void (*)(const void*, const void*, const void*, const uint8_t*, size_t, int, int, size_t, int,
                          const float*, const float*, const float*, float*, float*, void*, void*, float*, uint32_t*);
using FusedBwdPool = void (*)(const void*, const void*, const uint32_t*, const void*, size_t, int, int, size_t, int,
                              int, int, const float*, const float*, const float*, float*, float*, void*, float*,
                              uint32_t*);

// Per device: the SM count and, per pass (forward, backward, pooled backward) and dtype, the dynamic shared memory a
// block may hold when kResBlocksPerSM blocks share an SM (0: the single-launch pass cannot run on this device).
struct FusedDev {
  int sms = 0;
  size_t dyn[3][3] = {};
};

// Opts every variant of (direction, dtype) in to `*dyn` bytes of dynamic shared memory, first lowering *dyn by the
// largest static shared memory of the variants; leaves *dyn = 0 unless each variant then fits kResBlocksPerSM blocks
// per SM.
template <class K>
void opt_in(const K* kernels, int n, size_t share, size_t* dyn) {
  size_t stat = 0;
  for (int i = 0; i < n; ++i) {
    cudaFuncAttributes a;
    if (cudaFuncGetAttributes(&a, (const void*)kernels[i]) != cudaSuccess) return;
    stat = a.sharedSizeBytes > stat ? a.sharedSizeBytes : stat;
  }
  if (share <= stat) return;
  const size_t d = (share - stat) & ~(size_t)15;
  for (int i = 0; i < n; ++i) {
    int nb = 0;
    if (cudaFuncSetAttribute((const void*)kernels[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)d) !=
            cudaSuccess ||
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&nb, kernels[i], kT, d) != cudaSuccess || nb < kResBlocksPerSM)
      return;
  }
  *dyn = d;
}

template <class U>
void opt_in_u(size_t share, size_t* fwd, size_t* bwd, size_t* bwd_pool) {
  const FusedFwd f[5] = {bn_act_fwd_fused_kernel<U, false, false, false>,
                         bn_act_fwd_fused_kernel<U, false, true, false>,
                         bn_act_fwd_fused_kernel<U, true, false, false>,
                         bn_act_fwd_fused_kernel<U, true, true, false>,
                         bn_act_fwd_fused_kernel<U, true, false, true>};   // the pooled forward
  const FusedBwd b[4] = {bn_act_bwd_fused_kernel<U, false, false>, bn_act_bwd_fused_kernel<U, false, true>,
                            bn_act_bwd_fused_kernel<U, true, false>, bn_act_bwd_fused_kernel<U, true, true>};
  const FusedBwdPool bp[1] = {bn_act_bwd_pool_kernel<U>};
  opt_in(f, 5, share, fwd);
  opt_in(b, 4, share, bwd);
  opt_in(bp, 1, share, bwd_pool);
}

const FusedDev* fused_dev() {
  static std::mutex mu;
  static FusedDev devs[kMaxDevices];
  static bool done[kMaxDevices] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= kMaxDevices) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  FusedDev& d = devs[dev];
  if (!done[dev]) {
    done[dev] = true;
    int coop = 0, sms = 0, per_sm = 0, reserved = 0;
    if (cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev) != cudaSuccess || !coop ||
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&per_sm, cudaDevAttrMaxSharedMemoryPerMultiprocessor, dev) != cudaSuccess ||
        cudaDeviceGetAttribute(&reserved, cudaDevAttrReservedSharedMemoryPerBlock, dev) != cudaSuccess)
      return &d;
    const size_t share = (size_t)per_sm / kResBlocksPerSM - (size_t)reserved;
    opt_in_u<TagF32>(share, &d.dyn[0][0], &d.dyn[1][0], &d.dyn[2][0]);
    opt_in_u<TagBF16>(share, &d.dyn[0][1], &d.dyn[1][1], &d.dyn[2][1]);
    opt_in_u<TagF16>(share, &d.dyn[0][2], &d.dyn[1][2], &d.dyn[2][2]);
    d.sms = sms;
  }
  return &d;
}

struct FusedPlan {
  Geo g;
  size_t rpc;   // rows per chunk, a multiple of RL
  int G;        // chunks (gridDim.x)
  int held;     // rows of a chunk held in shared memory: a multiple of RL, or rpc
  int depth;    // ring row-steps: 0 when the whole chunk is held
  size_t held_bytes, smem;   // shared memory of the held rows; all dynamic shared memory per block
};

// The whole chunk is held when it fits (with the ring the layout always needs); otherwise the ring of kFwdStages /
// kBwdStages row-steps comes first and the held rows get what is left (at most `cap` bytes of them when cap >= 0).
// res selects the backward's residual layout, pool the pooled backward's (fused_layout).  The chunking depends on
// neither, so the pooled kernels reduce in the same order as the others at the same (M, C).
bool fused_plan(int bwd, int dtype, size_t M, int C, long long cap, bool res, FusedPlan* p, bool pool = false) {
  const int dt = dtype_index(dtype);
  const FusedDev* d = fused_dev();
  const int pass = bwd ? (pool ? 2 : 1) : 0;
  if (dt < 0 || bad_shape(M, C) || d == nullptr || d->dyn[pass][dt] == 0) return false;
  const Geo g = geo(C, red_cb(C));
  const int blocks = d->sms * kResBlocksPerSM;
  if (g.ncb > blocks) return false;
  const size_t want = (size_t)(blocks / g.ncb), rl = (size_t)g.rl;
  size_t rpc = (M + want - 1) / want;
  rpc = (rpc < rl ? rl : (rpc + rl - 1) / rl * rl);
  const Layout L = fused_layout(bwd != 0, bwd && res, dtype == WIRE_F32 ? 2 : 1, bwd && pool);
  const size_t dyn = d->dyn[pass][dt], capb = cap >= 0 ? (size_t)cap : dyn;
  const size_t step = 16 * (size_t)L.step, stages = bwd ? kBwdStages : kFwdStages;   // bytes of a held row-step
  size_t held = rpc;
  int depth = 0;
  if (L.ring_always || rpc / rl * step > (dyn < capb ? dyn : capb)) {
    depth = (int)stages;
    const size_t ring = stages * 16 * (size_t)L.slot;
    if (ring > dyn) return false;
    const size_t budget = dyn - ring < capb ? dyn - ring : capb;
    held = budget / step * rl;
    held = held < rpc ? held : rpc;
  }
  const size_t hb = held / rl * step;
  *p = FusedPlan{g, rpc, (int)((M + rpc - 1) / rpc), (int)held, depth, hb, hb + (size_t)depth * 16 * L.slot};
  return true;
}

// Bytes a launch moves between HBM (or L2) and the SMs: every row once, and the rows a block does not hold again in
// phase 2 (x forward; dy, x and the mask backward, or dz and x with a residual), plus the residual or the second
// gradient (dy2) read, the outputs and the mask written.
size_t fused_bytes(const FusedPlan& p, int bwd, int dtype, size_t M, int C, bool relu, bool res, bool dy2) {
  const size_t last = M - (size_t)(p.G - 1) * p.rpc;
  const size_t held = (size_t)(p.G - 1) * ((size_t)p.held < p.rpc ? p.held : p.rpc) +
                      ((size_t)p.held < last ? p.held : last);
  const size_t e = (size_t)C * (dtype == WIRE_F32 ? 4 : 2), m = relu ? (size_t)C / kCh : 0;   // per row
  if (bwd) return M * (3 * e + m) + (res ? M * e : 0) + (dy2 ? M * e : 0) + (M - held) * (res ? 2 * e : 2 * e + m);
  return M * (2 * e + m) + (res ? M * e : 0) + (M - held) * e;
}

// The same for the pooled passes over N images of H x W (M = N H W rows, P pooled rows of C channels; the pooled
// gradients g1 (and g2) and the codes, 4 bits a channel, are the pooled tensors).  Forward: x once, then in phase 2
// every row a block's windows span that it does not hold (its streamed rows and the halo rows of the neighbouring
// chunks), the pooled output and the codes written.  Backward: x and the pooled tensors once in phase 1, then x of
// the streamed rows and the pooled tensors again for them in phase 2 (counted as that share of the pooled tensors),
// dx written.  Re-reads of a row or pooled row within one phase of one block (the overlapping windows) are not counted.
size_t pool_bytes(const FusedPlan& p, int bwd, int dtype, size_t M, int C, int H, int W, bool dy2) {
  const PoolShape ps(H, W);
  const size_t e = (size_t)C * (dtype == WIRE_F32 ? 4 : 2), P = M / ps.hw * ps.ohw, pc = (size_t)C / 2;
  size_t held = 0, span = 0;
  for (int g = 0; g < p.G; ++g) {
    const size_t r0 = (size_t)g * p.rpc, r1 = r0 + p.rpc < M ? r0 + p.rpc : M;
    const size_t h = (size_t)p.held < r1 - r0 ? (size_t)p.held : r1 - r0;
    held += h;
    const size_t p0 = ps.pooled_before(r0), p1 = ps.pooled_before(r1);
    if (p0 == p1) continue;
    size_t n;
    int oh, ow;
    ps.pooled_at(p0, &n, &oh, &ow);
    const size_t c0 = n * ps.hw + (size_t)(2 * oh) * W + 2 * ow;
    ps.pooled_at(p1 - 1, &n, &oh, &ow);
    const size_t c1 = n * ps.hw + (size_t)(2 * oh) * W + 2 * ow;
    const size_t lo = c0 > (size_t)W + 1 ? c0 - W - 1 : 0, hi = c1 + W + 2 < M ? c1 + W + 2 : M;
    const size_t a = lo > r0 ? lo : r0, b = hi < r0 + h ? hi : r0 + h;   // held rows inside the span
    span += (hi - lo) - (b > a ? b - a : 0);
  }
  if (!bwd) return M * e + span * e + P * (e + pc);
  const size_t pooled = P * ((dy2 ? 2 : 1) * e + pc);
  return 2 * M * e + pooled + (M - held) * e + (size_t)((double)pooled * (double)(M - held) / (double)M);
}

template <class... P, class... A>
cudaError_t launch_coop(void (*kernel)(P...), const FusedPlan& p, cudaStream_t s, A... args) {
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(p.G, p.g.ncb);
  cfg.blockDim = dim3(kT);
  cfg.dynamicSmemBytes = p.smem;
  cfg.stream = s;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

}  // namespace

size_t bn_act_workspace_floats(size_t M, int C) {
  size_t rpc;
  int G;
  chunks(M, geo(C, red_cb(C)), &rpc, &G);
  return 2 * (size_t)G * (size_t)C;
}

int bn_act_counters(int C) { return geo(C, red_cb(C)).ncb; }

cudaError_t launch_bn_act_fwd_stats(const void* x, int dtype, size_t M, int C, float eps, float momentum,
                                    float* running_mean, float* running_var, float* save_mean, float* save_invstd,
                                    float* ws, uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, C) || M < 2 || !aligned16(x) || (running_mean == nullptr) != (running_var == nullptr))
    return cudaErrorInvalidValue;
  const Geo g = geo(C, red_cb(C));
  size_t rpc;
  int G;
  chunks(M, g, &rpc, &G);
  const dim3 grid(G, g.ncb);
  BN_DISPATCH_U(dtype, (bn_act_fwd_stats_kernel<U, false><<<grid, kT, 0, s>>>(x, M, C, g.shift, rpc, eps, momentum,
                                                                        running_mean, running_var, save_mean,
                                                                        save_invstd, ws, counters)));
  return cudaGetLastError();
}

cudaError_t launch_bn_act_fwd_apply(const void* x, const void* residual, int dtype, size_t M, int C, const float* mean,
                                    const float* invstd, const float* weight, const float* bias, int relu, void* y,
                                    uint8_t* mask, cudaStream_t s) {
  if (bad_shape(M, C) || !aligned16(x) || !aligned16(residual) || !aligned16(y) || (relu && mask == nullptr))
    return cudaErrorInvalidValue;
  const Geo g = geo(C, kMaxCB);
  const dim3 grid(apply_grid(M, g, kBlocksPerSM), g.ncb);
  BN_DISPATCH_U(dtype, BN_DISPATCH_B(relu, kRelu, BN_DISPATCH_B(residual != nullptr, kRes, (
      bn_act_fwd_apply_kernel<U, kRelu, kRes><<<grid, kT, 0, s>>>(x, residual, M, C, g.shift, mean, invstd, weight,
                                                                  bias, y, mask)))));
  return cudaGetLastError();
}

cudaError_t launch_bn_act_bwd_reduce(const void* dy, const void* x, const uint8_t* mask, int dtype, size_t M, int C,
                                     const float* mean, const float* invstd, float* dweight, float* dbias, float* ws,
                                     uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, C) || !aligned16(dy) || !aligned16(x)) return cudaErrorInvalidValue;
  const Geo g = geo(C, red_cb(C));
  size_t rpc;
  int G;
  chunks(M, g, &rpc, &G);
  const dim3 grid(G, g.ncb);
  BN_DISPATCH_U(dtype, BN_DISPATCH_B(mask != nullptr, kRelu, (
      bn_act_bwd_reduce_kernel<U, kRelu><<<grid, kT, 0, s>>>(dy, x, mask, M, C, g.shift, rpc, mean, invstd, dweight,
                                                             dbias, ws, counters))));
  return cudaGetLastError();
}

cudaError_t launch_bn_act_bwd_apply(const void* dy, const void* x, const uint8_t* mask, int dtype, size_t M, int C,
                                    const float* mean, const float* invstd, const float* weight, const float* dweight,
                                    const float* dbias, void* dx, void* dresidual, cudaStream_t s,
                                    const float* total) {
  if (bad_shape(M, C) || !aligned16(dy) || !aligned16(x) || !aligned16(dx) || !aligned16(dresidual))
    return cudaErrorInvalidValue;
  const Geo g = geo(C, kMaxCB);
  const dim3 grid(apply_grid(M, g, kBwdApplyBlocksPerSM), g.ncb);
  BN_DISPATCH_U(dtype, BN_DISPATCH_B(mask != nullptr, kRelu, BN_DISPATCH_B(dresidual != nullptr, kRes,
      BN_DISPATCH_B(total != nullptr, kTotal, (bn_act_bwd_apply_kernel<U, kRelu, kRes, kTotal><<<grid, kT, 0, s>>>(
          dy, x, mask, M, C, g.shift, mean, invstd, weight, dweight, dbias, dx, dresidual, total))))));
  return cudaGetLastError();
}

cudaError_t launch_bn_act_fwd_stats_local(const void* x, int dtype, size_t M, int C, float* local_mean,
                                          float* local_m2, float* ws, uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, C) || !aligned16(x)) return cudaErrorInvalidValue;
  const Geo g = geo(C, red_cb(C));
  size_t rpc;
  int G;
  chunks(M, g, &rpc, &G);
  const dim3 grid(G, g.ncb);
  BN_DISPATCH_U(dtype, (bn_act_fwd_stats_kernel<U, true><<<grid, kT, 0, s>>>(x, M, C, g.shift, rpc, 0.f, 0.f,
                                                                             nullptr, nullptr, local_mean, local_m2,
                                                                             ws, counters)));
  return cudaGetLastError();
}

bool bn_act_fused_plan(int bwd, int dtype, size_t M, int C, long long cap, int relu, int residual, int dy2,
                       BnFusedPlan* out, int pool_h, int pool_w) {
  const bool pool = pool_h > 0 || pool_w > 0;
  if (pool && (pool_h < 1 || pool_w < 1 || M % ((size_t)pool_h * pool_w) != 0 || !relu || residual)) return false;
  FusedPlan p;
  if (!fused_plan(bwd, dtype, M, C, cap, residual != 0, &p, pool)) return false;
  *out = BnFusedPlan{2 * (size_t)p.G * (size_t)C, p.g.ncb, p.rpc, p.held, p.held_bytes, p.depth, p.smem,
                     pool ? pool_bytes(p, bwd, dtype, M, C, pool_h, pool_w, bwd && dy2)
                          : fused_bytes(p, bwd, dtype, M, C, relu != 0, residual != 0, bwd && residual && dy2),
                     fused_dev()->sms * kResBlocksPerSM};
  return true;
}

cudaError_t launch_bn_act_fwd(const void* x, const void* residual, int dtype, size_t M, int C, float eps,
                              float momentum, float* running_mean, float* running_var, float* save_mean,
                              float* save_invstd, const float* weight, const float* bias, int relu, void* y,
                              uint8_t* mask, float* ws, uint32_t* counters, long long cap, cudaStream_t s) {
  FusedPlan p;
  if (bad_shape(M, C) || M < 2 || !aligned16(x) || !aligned16(residual) || !aligned16(y) ||
      (relu && mask == nullptr) || (running_mean == nullptr) != (running_var == nullptr))
    return cudaErrorInvalidValue;
  if (!fused_plan(0, dtype, M, C, cap, residual != nullptr, &p)) return cudaErrorNotSupported;
  cudaError_t e = cudaSuccess;
  BN_DISPATCH_U(dtype, BN_DISPATCH_B(relu, kRelu, BN_DISPATCH_B(residual != nullptr, kRes, (
      e = launch_coop(bn_act_fwd_fused_kernel<U, kRelu, kRes, false>, p, s, x, residual, M, C, p.g.shift, p.rpc,
                      p.held, eps, momentum, running_mean, running_var, save_mean, save_invstd, weight, bias, y, mask,
                      ws, counters, 0, 0, (uint32_t*)nullptr)))));
  return e;
}

cudaError_t launch_bn_act_fwd_pool(const void* x, int dtype, int N, int H, int W, int C, float eps, float momentum,
                                   float* running_mean, float* running_var, float* save_mean, float* save_invstd,
                                   const float* weight, const float* bias, void* pooled, uint32_t* code, float* ws,
                                   uint32_t* counters, long long cap, cudaStream_t s) {
  FusedPlan p;
  const size_t M = (size_t)N * H * W;
  if (N < 1 || H < 1 || W < 1 || bad_shape(M, C) || M < 2 || !aligned16(x) || !aligned16(pooled) ||
      pooled == nullptr || code == nullptr || (running_mean == nullptr) != (running_var == nullptr))
    return cudaErrorInvalidValue;
  if (!fused_plan(0, dtype, M, C, cap, false, &p)) return cudaErrorNotSupported;
  cudaError_t e = cudaSuccess;
  BN_DISPATCH_U(dtype, (
      e = launch_coop(bn_act_fwd_fused_kernel<U, true, false, true>, p, s, x, (const void*)nullptr, M, C, p.g.shift,
                      p.rpc, p.held, eps, momentum, running_mean, running_var, save_mean, save_invstd, weight, bias,
                      pooled, (uint8_t*)nullptr, ws, counters, H, W, code)));
  return e;
}

cudaError_t launch_bn_act_bwd_pool(const void* g1, const void* g2, const uint32_t* code, const void* x, int dtype,
                                   int N, int H, int W, int C, const float* mean, const float* invstd,
                                   const float* weight, float* dweight, float* dbias, void* dx, float* ws,
                                   uint32_t* counters, long long cap, cudaStream_t s) {
  FusedPlan p;
  const size_t M = (size_t)N * H * W;
  if (N < 1 || H < 1 || W < 1 || bad_shape(M, C) || g1 == nullptr || code == nullptr || !aligned16(g1) ||
      !aligned16(g2) || !aligned16(x) || !aligned16(dx))
    return cudaErrorInvalidValue;
  if (!fused_plan(1, dtype, M, C, cap, false, &p, true)) return cudaErrorNotSupported;
  cudaError_t e = cudaSuccess;
  BN_DISPATCH_U(dtype, (
      e = launch_coop(bn_act_bwd_pool_kernel<U>, p, s, g1, g2, code, x, M, C, p.g.shift, p.rpc, p.held, H, W, mean,
                      invstd, weight, dweight, dbias, dx, ws, counters)));
  return e;
}

cudaError_t launch_bn_act_bwd(const void* dy, const void* dy2, const void* x, const uint8_t* mask, int dtype, size_t M,
                              int C, const float* mean, const float* invstd, const float* weight, float* dweight,
                              float* dbias, void* dx, void* dresidual, float* ws, uint32_t* counters, long long cap,
                              cudaStream_t s) {
  FusedPlan p;
  if (bad_shape(M, C) || !aligned16(dy) || !aligned16(dy2) || !aligned16(x) || !aligned16(dx) ||
      !aligned16(dresidual) || (dy2 != nullptr && dresidual == nullptr))
    return cudaErrorInvalidValue;
  if (!fused_plan(1, dtype, M, C, cap, dresidual != nullptr, &p)) return cudaErrorNotSupported;
  cudaError_t e = cudaSuccess;
  BN_DISPATCH_U(dtype, BN_DISPATCH_B(mask != nullptr, kRelu, BN_DISPATCH_B(dresidual != nullptr, kRes, (
      e = launch_coop(bn_act_bwd_fused_kernel<U, kRelu, kRes>, p, s, dy, dy2, x, mask, M, C, p.g.shift, p.rpc,
                      p.held, mean, invstd, weight, dweight, dbias, dx, dresidual, ws, counters)))));
  return e;
}

size_t bn_sync_window_floats(int world, int cmax) { return 2 * (size_t)world * (kSyncPad + 2 * (size_t)cmax); }

namespace {
cudaError_t check_sync(const PeerView& pv, int channel, const void* window, int cmax, int C, const float* a,
                       const float* b) {
  if (pv.world < 1 || pv.world > kMaxRanks || channel < 0 || channel > 1 || C < kCh || C % kCh != 0 || C > cmax ||
      cmax % kCh != 0 || !aligned16(window) || !aligned16(a) || !aligned16(b))
    return cudaErrorInvalidValue;
  return cudaSuccess;
}
int sync_grid(int C) {
  const int steps = (C + kSyncStep - 1) / kSyncStep;
  return steps < kMaxSyncBlocks ? steps : kMaxSyncBlocks;
}
}  // namespace

cudaError_t launch_bn_sync_stats(const PeerView& pv, int channel, size_t win_off, int cmax, int C,
                                 const float* local_mean, const float* local_m2, float count, float eps,
                                 float momentum, float* running_mean, float* running_var, float* save_mean,
                                 float* save_invstd, float* total, cudaStream_t s) {
  if (check_sync(pv, channel, pv.data[pv.rank] + win_off, cmax, C, local_mean, local_m2) != cudaSuccess ||
      !(count >= 1.f) || (running_mean == nullptr) != (running_var == nullptr) || total == nullptr)
    return cudaErrorInvalidValue;
  bn_sync_kernel<true><<<sync_grid(C), kSyncT, 0, s>>>(pv, channel, win_off, cmax, C, local_mean, local_m2, count,
                                                       eps, momentum, running_mean, running_var, save_mean,
                                                       save_invstd, total);
  return cudaGetLastError();
}

cudaError_t launch_bn_sync_grad(const PeerView& pv, int channel, size_t win_off, int cmax, int C, const float* dbias,
                                const float* dweight, float* sum_dbias, float* sum_dweight, cudaStream_t s) {
  if (check_sync(pv, channel, pv.data[pv.rank] + win_off, cmax, C, dbias, dweight) != cudaSuccess)
    return cudaErrorInvalidValue;
  bn_sync_kernel<false><<<sync_grid(C), kSyncT, 0, s>>>(pv, channel, win_off, cmax, C, dbias, dweight, 0.f, 0.f,
                                                        0.f, nullptr, nullptr, sum_dbias, sum_dweight, nullptr);
  return cudaGetLastError();
}

namespace {
template <class K>
cudaError_t load1(K* kernel) {
  cudaFuncAttributes a;
  return cudaFuncGetAttributes(&a, (const void*)kernel);
}
template <class U>
cudaError_t load_u() {
  cudaError_t e = cudaSuccess;
  auto keep = [&e](cudaError_t x) { if (e == cudaSuccess) e = x; };
  keep(load1(bn_act_fwd_stats_kernel<U, false>));
  keep(load1(bn_act_fwd_stats_kernel<U, true>));
  keep(load1(bn_act_fwd_apply_kernel<U, false, false>));
  keep(load1(bn_act_fwd_apply_kernel<U, false, true>));
  keep(load1(bn_act_fwd_apply_kernel<U, true, false>));
  keep(load1(bn_act_fwd_apply_kernel<U, true, true>));
  keep(load1(bn_act_bwd_reduce_kernel<U, false>));
  keep(load1(bn_act_bwd_reduce_kernel<U, true>));
  keep(load1(bn_act_bwd_apply_kernel<U, false, false, false>));
  keep(load1(bn_act_bwd_apply_kernel<U, false, true, false>));
  keep(load1(bn_act_bwd_apply_kernel<U, true, false, false>));
  keep(load1(bn_act_bwd_apply_kernel<U, true, true, false>));
  keep(load1(bn_act_bwd_apply_kernel<U, false, false, true>));
  keep(load1(bn_act_bwd_apply_kernel<U, false, true, true>));
  keep(load1(bn_act_bwd_apply_kernel<U, true, false, true>));
  keep(load1(bn_act_bwd_apply_kernel<U, true, true, true>));
  return e;
}
}  // namespace

cudaError_t bn_act_load_kernels() {
  cudaError_t e = load_u<TagF32>();
  if (e == cudaSuccess) e = load_u<TagBF16>();
  if (e == cudaSuccess) e = load_u<TagF16>();
  if (e == cudaSuccess) e = load1(bn_sync_kernel<true>);
  if (e == cudaSuccess) e = load1(bn_sync_kernel<false>);
  if (e == cudaSuccess && fused_dev() == nullptr) e = cudaErrorInvalidDevice;
  return e;
}

}  // namespace bps
