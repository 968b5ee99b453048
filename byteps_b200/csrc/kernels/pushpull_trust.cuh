// Device pieces shared by the trust-ratio optimizers of the fused exchange, LAMB (pushpull_lamb.cu) and LARS
// (pushpull_lars.cu): the parameter cursor over a bucket's (start, numel) table, the reduction of one wire unit of
// this rank's shard, the fixed-order segmented warp sums of a pair of per-parameter squares, and the exchange of
// those float64 partial sums through the bucket's window with the rank-order sum that forms each ratio.
// Everything has internal linkage (one copy per translation unit), like pushpull_dev.cuh.
#pragma once
#include "kernels/pushpull_dev.cuh"
#include "kernels/pushpull_lamb.cuh"

namespace bps {

namespace {

constexpr int kNormThreads = 256;
constexpr unsigned kFull = 0xffffffffu;

// The parameter that holds flat element e: the last one whose start is <= e (its padding included).  Each thread
// visits its units in increasing order, so after one binary search the cursor only moves forward.
struct ParamCursor {
  const LambParam* params;
  int n;
  int i;
  __device__ __forceinline__ void init(const LambParam* p, int np, int64_t e) {
    params = p;
    n = np;
    int lo = 0, hi = np - 1;
    while (lo < hi) {
      const int mid = (lo + hi + 1) >> 1;
      if (__ldg(&params[mid].start) <= e) lo = mid;
      else hi = mid - 1;
    }
    i = lo;
  }
  __device__ __forceinline__ void seek(int64_t e) {
    while (i + 1 < n && __ldg(&params[i + 1].start) <= e) ++i;
  }
  // init on the first call of a thread (`inited` false), seek afterwards; the parameter index of e
  __device__ __forceinline__ int at(const LambParam* p, int np, int64_t e, bool& inited) {
    if (!inited) {
      init(p, np, e);
      inited = true;
    } else {
      seek(e);
    }
    return i;
  }
};

// The sum over the peers of wire unit `unit` of the window at `off` (the gradients, or the staging window of a wire
// cast), in g: the peer loads of reduce_units_p2p in the order `rot` sets.  Every lane of the warp calls it; lanes with
// !valid get zeros.  (The NVLS path is one multimem.ld_reduce per unit, W::mm_reduce, in the kernels themselves.)
template <class W>
__device__ __forceinline__ void reduce_unit_p2p(const PeerView& pv, size_t off, size_t unit, bool valid, int rot,
                                                float (&g)[W::kPerVec]) {
  const size_t idx[1] = {unit};
  const bool vld[1] = {valid};
  float acc[1][W::kPerVec];
  reduce_units_p2p<W, 1>(pv, off, idx, vld, rot, acc);
#pragma unroll
  for (int k = 0; k < W::kPerVec; ++k) g[k] = acc[0][k];
}

// Segmented suffix sums of the float64 lvalues (A, B) over the warp's 32 units: a parameter's units are contiguous,
// so after the five steps the first lane of each segment holds the segment's sum, added in a fixed order.  That lane
// stores it in GROUPS[(UNIT - S0) / 32] (the segment that begins at the warp's first unit) or HEADS[PID] (one that
// begins at a parameter's first unit inside the warp).  Every lane of the warp runs it; PID is -1 on the invalid
// lanes, the warp's last ones.  A macro rather than an inline function: inlined as a function, nvcc schedules LAMB's
// first kernel differently, and LAMB's kernels keep the instructions they had before LARS shared this code.
#define BPS_STORE_SEGMENT_SUMS(A, B, PID, VALID, LANE, UNIT, S0, GROUPS, HEADS)                \
  do {                                                                                          \
    _Pragma("unroll") for (int off_ = 1; off_ < 32; off_ <<= 1) {                               \
      const double oa_ = __shfl_down_sync(kFull, A, off_);                                      \
      const double ob_ = __shfl_down_sync(kFull, B, off_);                                      \
      const int op_ = __shfl_down_sync(kFull, PID, off_);                                       \
      if ((LANE) + off_ < 32 && op_ == (PID)) {                                                 \
        A += oa_;                                                                               \
        B += ob_;                                                                               \
      }                                                                                         \
    }                                                                                           \
    const int prev_ = __shfl_up_sync(kFull, PID, 1);                                            \
    if ((VALID) && ((LANE) == 0 || prev_ != (PID)))                                             \
      ((LANE) == 0 ? (GROUPS)[((UNIT) - (S0)) / 32] : (HEADS)[PID]) = make_double2(A, B);       \
  } while (0)

// The norms launch of a bucket, kNormThreads threads per CTA.  Per parameter (one CTA each, strided): this rank's
// partial sums (the warp sums of BPS_STORE_SEGMENT_SUMS in unit order, then a fixed tree over the CTA, all float64),
// stored into this rank's slot of every peer's window at win_off; barrier_peers; the ranks' slots summed in rank
// order, and phi[p] = ratio(sum a, sum b, p).  A skipped step stores no slot and no ratio but meets the barrier.
template <int E, class Ratio>
__device__ __forceinline__ void exchange_norms(const PeerView& pv, size_t total_groups, const LambParam* params,
                                               int nparams, const double* scratch, size_t win_off, float* phi,
                                               bool skip, int channel, Ratio&& ratio) {
  __shared__ double2 red[kNormThreads];
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  const double2* heads = reinterpret_cast<const double2*>(scratch);
  const double2* groups = heads + nparams;
  for (int p = blockIdx.x; p < nparams; p += gridDim.x) {
    const int64_t st = params[p].start;
    const size_t ua = (size_t)st / E, ub = (size_t)(st + (params[p].n + 7) / 8 * 8) / E;
    const size_t a = ua > s0 ? ua : s0, b = ub < s1 ? ub : s1;
    double2 acc = make_double2(0.0, 0.0);
    if (!skip && a < b) {
      // the warp segments of the parameter in this shard: those that begin a 32-unit group, in unit order per
      // thread, and the one that begins at the parameter's first unit inside a group
      const size_t g0 = (a - s0 + 31) / 32, g1 = (b - s0 + 31) / 32;
      for (size_t gi = g0 + threadIdx.x; gi < g1; gi += blockDim.x) {
        acc.x += groups[gi].x;
        acc.y += groups[gi].y;
      }
      if (threadIdx.x == 0 && a == ua && ((a - s0) & 31)) {
        acc.x += heads[p].x;
        acc.y += heads[p].y;
      }
    }
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = kNormThreads / 2; s > 0; s >>= 1) {
      if (threadIdx.x < s) {
        red[threadIdx.x].x += red[threadIdx.x + s].x;
        red[threadIdx.x].y += red[threadIdx.x + s].y;
      }
      __syncthreads();
    }
    if (!skip && threadIdx.x < pv.world)
      reinterpret_cast<double2*>(pv.data[threadIdx.x] + win_off)[(size_t)p * pv.world + pv.rank] = red[0];
    __syncthreads();
  }
  barrier_peers(pv, channel);   // the peers' CTA of this index has stored the same parameters' slots
  if (skip) return;
  const volatile double* win = reinterpret_cast<const volatile double*>(pv.data[pv.rank] + win_off);
  for (int p = blockIdx.x + threadIdx.x * gridDim.x; p < nparams; p += gridDim.x * blockDim.x) {
    double as = 0.0, bs = 0.0;
    for (int r = 0; r < pv.world; ++r) {
      as += win[((size_t)p * pv.world + r) * 2];
      bs += win[((size_t)p * pv.world + r) * 2 + 1];
    }
    phi[p] = ratio(as, bs);
  }
}

inline bool bad_geometry(int blocks, int threads) {
  return blocks < 1 || blocks > kMaxBlocks || threads < 32 || threads > 512 || (threads & 31);
}

// exactly the (gradient, wire) pairs of launch_pushpull_fused_opt; the parameters have the gradient dtype
template <class F>
cudaError_t dispatch_pair(int grad_dtype, int wire, F&& f) {
  if (grad_dtype == WIRE_F32 && wire == WIRE_F32) return f(TagF32{}, TagF32{});
  if (grad_dtype == WIRE_F32 && wire == WIRE_BF16) return f(TagF32{}, TagBF16{});
  if (grad_dtype == WIRE_F32 && wire == WIRE_F16) return f(TagF32{}, TagF16{});
  if (grad_dtype == WIRE_BF16 && wire == WIRE_BF16) return f(TagBF16{}, TagBF16{});
  if (grad_dtype == WIRE_F16 && wire == WIRE_F16) return f(TagF16{}, TagF16{});
  return cudaErrorInvalidValue;
}

}  // namespace

}  // namespace bps
