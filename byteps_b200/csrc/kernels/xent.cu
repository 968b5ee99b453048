// Softmax cross-entropy forward and backward (see xent.cuh).
//
// A block of kT threads takes one row at a time and walks a contiguous chunk of rows; the grid is one resident wave
// (sized with the occupancy API).  A row is split at its first 16-byte boundary: the head elements before it and the
// tail elements after the last whole vector are read one at a time by the first threads of the block, and the
// vectors in between are strided over all threads, kUnroll loads in flight per thread.
#include "kernels/xent.cuh"

#include <math.h>

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kT = 256;
constexpr int kW = kT / 32;
constexpr int kUnroll = 4;
constexpr int kGroup = 16;      // block partials summed by the last block of each run of kGroup blocks
constexpr int kMaxDevices = 64;
constexpr float kLog2e = 1.4426950408889634f;

// head / vector / tail split of a row that starts at p (element-aligned inside a 16-byte aligned allocation)
template <class U>
struct Split {
  static constexpr int E = U::kPerVec;
  int head, nvec, tail;
  __device__ __forceinline__ Split(const void* p, int V) {
    const int mis = (int)(((uintptr_t)p & 15u) / U::kBytes);
    head = min(V, (E - mis) % E);
    nvec = (V - head) / E;
    tail = V - head - nvec * E;
  }
};

// factor that carries a sum of exp(x - m) over to exp(x - M), M >= m (1 when nothing changes, so -inf stays exact)
__device__ __forceinline__ float rescale(float m, float M) { return m == M ? 1.f : exp2f((m - M) * kLog2e); }

// running (max, sum exp(x - max)) over N more values
template <int N>
__device__ __forceinline__ void online(float& m, float& s, const float* f) {
  float mx = f[0];
#pragma unroll
  for (int k = 1; k < N; ++k) mx = fmaxf(mx, f[k]);
  const float M = fmaxf(m, mx);
  const float ref = M == -INFINITY ? 0.f : M;   // a row of -inf so far adds exp(-inf) = 0, not NaN
  float acc = 0.f;
#pragma unroll
  for (int k = 0; k < N; ++k) acc += exp2f((f[k] - ref) * kLog2e);
  s = fmaf(s, rescale(m, M), acc);
  m = M;
}

__device__ __forceinline__ void merge(float& m, float& s, float m2, float s2) {
  const float M = fmaxf(m, m2);
  s = s * rescale(m, M) + s2 * rescale(m2, M);
  m = M;
}

__device__ __forceinline__ bool in_range(int64_t t, int V) { return t >= 0 && t < (int64_t)V; }

struct FwdArgs {
  const void* x;
  const int64_t* target;
  float *lse, *loss, *out, *ws;
  int64_t* count;
  uint32_t* counters;
  size_t M, rpc;
  int64_t ignore;
  int V;
  bool mean;
};

template <class U>
__global__ void __launch_bounds__(kT) xent_fwd_kernel(FwdArgs a) {
  constexpr int E = U::kPerVec;
  __shared__ float sh[2][2][kW];   // per-warp (max, sum), alternating by row so a row's writes never meet the last
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const size_t r0 = (size_t)blockIdx.x * a.rpc, r1 = min(a.M, r0 + a.rpc);
  float bsum = 0.f;      // thread 0: the block's losses in row order
  uint32_t bcnt = 0;
  int par = 0;
  for (size_t row = r0; row < r1; ++row) {
    const int64_t t = a.target[row];
    if (t == a.ignore || !in_range(t, a.V)) {   // not read
      if (tid == 0) {
        a.lse[row] = t == a.ignore ? 0.f : NAN;
        a.loss[row] = t == a.ignore ? 0.f : NAN;
        if (t != a.ignore) {
          bsum += NAN;
          ++bcnt;
        }
      }
      continue;
    }
    const char* base = reinterpret_cast<const char*>(a.x) + row * (size_t)a.V * U::kBytes;
    const Split<U> sp(base, a.V);
    float m = -INFINITY, s = 0.f;
    if (tid < sp.head) {
      const float f = U::load1(base, tid);
      online<1>(m, s, &f);
    }
    if (tid < sp.tail) {
      const float f = U::load1(base, (size_t)(sp.head + sp.nvec * E + tid));
      online<1>(m, s, &f);
    }
    const Vec16* vp = reinterpret_cast<const Vec16*>(base + (size_t)sp.head * U::kBytes);
    int i = tid;
    for (; i + (kUnroll - 1) * kT < sp.nvec; i += kUnroll * kT) {
      Vec16 v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) v[u] = ld_stream16(vp + i + u * kT);
      float f[kUnroll * E];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) U::unpack(v[u], f + u * E);
      online<kUnroll * E>(m, s, f);
    }
    for (; i < sp.nvec; i += kT) {
      float f[E];
      U::unpack(ld_stream16(vp + i), f);
      online<E>(m, s, f);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
      merge(m, s, m2, s2);
    }
    if (lane == 0) {
      sh[par][0][w] = m;
      sh[par][1][w] = s;
    }
    __syncthreads();
    if (tid == 0) {
      m = sh[par][0][0];
      s = sh[par][1][0];
#pragma unroll
      for (int k = 1; k < kW; ++k) merge(m, s, sh[par][0][k], sh[par][1][k]);
      const float lse = m + logf(s);
      const float loss = lse - U::load1(base, (size_t)t);
      a.lse[row] = lse;
      a.loss[row] = loss;
      bsum += loss;
      ++bcnt;
    }
    par ^= 1;
  }

  // block partials, then runs of kGroup blocks, then the runs, each summed in block order by the last to arrive
  const int G = gridDim.x, runs = (G + kGroup - 1) / kGroup, run = blockIdx.x / kGroup;
  float* sums = a.ws;
  uint32_t* cnts = reinterpret_cast<uint32_t*>(a.ws + G + runs);
  if (tid == 0) {
    sums[blockIdx.x] = bsum;
    cnts[blockIdx.x] = bcnt;
  }
  if (!last_block(a.counters + run, min(kGroup, G - run * kGroup))) return;
  if (tid == 0) {
    const int b0 = run * kGroup, b1 = min(G, b0 + kGroup);
    float s = __ldcg(sums + b0);
    uint32_t c = __ldcg(cnts + b0);
    for (int b = b0 + 1; b < b1; ++b) {
      s += __ldcg(sums + b);
      c += __ldcg(cnts + b);
    }
    sums[G + run] = s;
    cnts[G + run] = c;
  }
  if (!last_block(a.counters + runs, runs)) return;
  if (tid == 0) {
    float s = __ldcg(sums + G);
    uint64_t c = __ldcg(cnts + G);
    for (int r = 1; r < runs; ++r) {
      s += __ldcg(sums + G + r);
      c += __ldcg(cnts + G + r);
    }
    *a.count = (int64_t)c;
    *a.out = a.mean ? s / (float)c : s;
  }
}

struct BwdArgs {
  const void* x;
  const int64_t* target;
  const float *lse, *grad;
  const int64_t* count;
  void* dx;
  size_t M, rpc;
  int64_t ignore;
  int V, mode;
};

template <class U>
__global__ void __launch_bounds__(kT) xent_bwd_kernel(BwdArgs a) {
  constexpr int E = U::kPerVec;
  const int tid = threadIdx.x;
  const size_t r0 = (size_t)blockIdx.x * a.rpc, r1 = min(a.M, r0 + a.rpc);
  float g = 0.f;
  if (a.mode == XENT_SUM) g = a.grad[0];
  if (a.mode == XENT_MEAN) g = a.grad[0] / (float)*a.count;
  for (size_t row = r0; row < r1; ++row) {
    const int64_t t = a.target[row];
    const size_t off = row * (size_t)a.V * U::kBytes;
    const char* base = reinterpret_cast<const char*>(a.x) + off;
    char* dbase = reinterpret_cast<char*>(a.dx) + off;
    const Split<U> sp(base, a.V);
    const Vec16* vp = reinterpret_cast<const Vec16*>(base + (size_t)sp.head * U::kBytes);
    Vec16* dp = reinterpret_cast<Vec16*>(dbase + (size_t)sp.head * U::kBytes);
    const int tl = sp.head + sp.nvec * E;   // first tail element
    if (t == a.ignore || !in_range(t, a.V)) {   // not read: zeros, or NaN for a target outside [0, V)
      float f[E];
#pragma unroll
      for (int k = 0; k < E; ++k) f[k] = t == a.ignore ? 0.f : NAN;
      if (tid < sp.head) U::store1(dbase, tid, f[0]);
      if (tid < sp.tail) U::store1(dbase, (size_t)(tl + tid), f[0]);
      const Vec16 q = U::pack(f);
      for (int i = tid; i < sp.nvec; i += kT) st_stream16(dp + i, q);
      continue;
    }
    const float gr = a.mode == XENT_NONE ? a.grad[row] : g;
    const float l = a.lse[row];
    const int jt = (int)t;
    auto d = [&](float x, int j) { return gr * (exp2f((x - l) * kLog2e) - (j == jt ? 1.f : 0.f)); };
    if (tid < sp.head) U::store1(dbase, tid, d(U::load1(base, tid), tid));
    if (tid < sp.tail) U::store1(dbase, (size_t)(tl + tid), d(U::load1(base, (size_t)(tl + tid)), tl + tid));
    int i = tid;
    for (; i + (kUnroll - 1) * kT < sp.nvec; i += kUnroll * kT) {
      Vec16 v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) v[u] = ld_stream16(vp + i + u * kT);
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        float f[E];
        U::unpack(v[u], f);
        const int j0 = sp.head + (i + u * kT) * E;
#pragma unroll
        for (int k = 0; k < E; ++k) f[k] = d(f[k], j0 + k);
        st_stream16(dp + i + u * kT, U::pack(f));
      }
    }
    for (; i < sp.nvec; i += kT) {
      float f[E];
      U::unpack(ld_stream16(vp + i), f);
      const int j0 = sp.head + i * E;
#pragma unroll
      for (int k = 0; k < E; ++k) f[k] = d(f[k], j0 + k);
      st_stream16(dp + i, U::pack(f));
    }
  }
}

// ---- host side

#define XENT_DISPATCH(dtype, STMT)                 \
  switch (dtype) {                                 \
    case WIRE_F32: { using U = TagF32; STMT; break; }   \
    case WIRE_BF16: { using U = TagBF16; STMT; break; } \
    case WIRE_F16: { using U = TagF16; STMT; break; }   \
    default: return cudaErrorInvalidValue;         \
  }

bool aligned16(const void* p) { return ((uintptr_t)p & 15u) == 0; }

bool bad_shape(size_t M, int V) { return M < 1 || V < 1; }

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

template <class U>
int fwd_wave() {
  static int cache[kMaxDevices];
  return resident(xent_fwd_kernel<U>, cache) * sm_count();
}

template <class U>
int bwd_wave() {
  static int cache[kMaxDevices];
  return resident(xent_bwd_kernel<U>, cache) * sm_count();
}

// contiguous chunks of rows, at most one per block of a wave
void chunks(size_t M, int wave, size_t* rpc, int* grid) {
  const size_t want = M < (size_t)wave ? M : (size_t)wave;
  *rpc = (M + want - 1) / want;
  *grid = (int)((M + *rpc - 1) / *rpc);
}

// the most blocks a fwd launch over M rows takes, over the dtypes: the workspace fits all of them
int fwd_blocks(size_t M) {
  int most = 0;
  for (int dt = WIRE_F32; dt <= WIRE_F16; ++dt) {
    int grid = 0;
    auto pick = [&]() -> cudaError_t {
      XENT_DISPATCH(dt, ({
        size_t rpc;
        chunks(M, fwd_wave<U>(), &rpc, &grid);
      }));
      return cudaSuccess;
    };
    pick();
    if (grid > most) most = grid;
  }
  return most;
}

}  // namespace

size_t xent_workspace_floats(size_t M) {
  if (M < 1) return 0;
  const size_t G = (size_t)fwd_blocks(M);
  return 2 * (G + (G + kGroup - 1) / kGroup);
}

int xent_counters(size_t M) {
  if (M < 1) return 0;
  return (fwd_blocks(M) + kGroup - 1) / kGroup + 1;
}

cudaError_t launch_xent_fwd(const void* logits, const int64_t* target, int dtype, size_t M, int V,
                            int64_t ignore_index, bool mean, float* lse, float* loss_rows, float* out, int64_t* count,
                            float* ws, uint32_t* counters, cudaStream_t s) {
  if (bad_shape(M, V) || logits == nullptr || !aligned16(logits) || target == nullptr || lse == nullptr ||
      loss_rows == nullptr || out == nullptr || count == nullptr || ws == nullptr || counters == nullptr)
    return cudaErrorInvalidValue;
  FwdArgs a{logits, target, lse, loss_rows, out, ws, count, counters, M, 0, ignore_index, V, mean};
  XENT_DISPATCH(dtype, ({
    int grid;
    chunks(M, fwd_wave<U>(), &a.rpc, &grid);
    xent_fwd_kernel<U><<<grid, kT, 0, s>>>(a);
  }));
  return cudaGetLastError();
}

cudaError_t launch_xent_bwd(const void* logits, const int64_t* target, int dtype, size_t M, int V,
                            int64_t ignore_index, const float* lse, const float* grad, int mode, const int64_t* count,
                            void* dlogits, cudaStream_t s) {
  if (bad_shape(M, V) || logits == nullptr || !aligned16(logits) || dlogits == nullptr || !aligned16(dlogits) ||
      target == nullptr || lse == nullptr || grad == nullptr || mode < XENT_NONE || mode > XENT_MEAN ||
      (mode == XENT_MEAN && count == nullptr))
    return cudaErrorInvalidValue;
  BwdArgs a{logits, target, lse, grad, count, dlogits, M, 0, ignore_index, V, mode};
  XENT_DISPATCH(dtype, ({
    int grid;
    chunks(M, bwd_wave<U>(), &a.rpc, &grid);
    xent_bwd_kernel<U><<<grid, kT, 0, s>>>(a);
  }));
  return cudaGetLastError();
}

}  // namespace bps
