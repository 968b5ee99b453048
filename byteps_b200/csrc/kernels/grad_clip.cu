// Global gradient-norm clipping in the fused exchange: the norm pass of a bucket and the per-step update (see
// grad_clip.cuh).  The pack phase and the peer reduction are those of the fused kernels (pushpull_dev.cuh); the
// parameter cursor and the reduction of one wire unit are the trust-ratio optimizers' (pushpull_trust.cuh).
#include <math.h>

#include "kernels/common.cuh"
#include "kernels/grad_clip.cuh"
#include "kernels/pushpull_dev.cuh"
#include "kernels/pushpull_trust.cuh"

namespace bps {

namespace {

constexpr int kClipMaxThreads = 512;
constexpr int kClipUpdateThreads = 128;

// Sum of red[0, n) in shared memory in a fixed order for any n <= blockDim.x: pairs at distance 1, 2, 4, ...
// Every thread calls it; the result is in red[0].
__device__ __forceinline__ void tree_sum(double* red, int n) {
  for (int s = 1; s < n; s <<= 1) {
    __syncthreads();
    const int i = threadIdx.x;
    if ((i & (2 * s - 1)) == 0 && i + s < n) red[i] += red[i + s];
  }
  __syncthreads();
}

template <class G, class W>
__global__ void __launch_bounds__(kClipMaxThreads, 1) clip_norm_partial_kernel(
    PeerView pv, const SegDesc* segs, int nsegs, size_t stage_off, size_t total_groups, float scale,
    const LambParam* params, int nparams, double* row, const OptHParams* hpp, int nvls, int channel) {
  constexpr int E = W::kPerVec;
  __shared__ double red[kClipMaxThreads];
  pack_phase<G, W, kUnrollOpt>(pv, segs, nsegs, stage_off, total_groups);
  barrier_peers(pv, channel);
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  const float gs = scale * hpp->grad_scale;       // as the epilogues form it; skip is ignored on purpose
  const int rot = rot_of(pv);
  ParamCursor cur;
  bool inited = false;
  double acc = 0.0;
  for_owned_tiles<1>(s0, s1, [&](size_t t) {
    const size_t unit = t + threadIdx.x;
    const bool valid = unit < s1;       // the invalid lanes of a tile are its last ones
    float g[E];
    if (nvls) {
      if (valid) W::unpack(W::mm_reduce(pv.mc_data + stage_off + unit * 16), g);
    } else {
      reduce_unit_p2p<W>(pv, stage_off, unit, valid, rot, g);
    }
    if (valid) {
      const int64_t e = (int64_t)(unit * E);
      const int pid = cur.at(params, nparams, e, inited);
      const int64_t end = __ldg(&params[pid].start) + __ldg(&params[pid].n);
#pragma unroll
      for (int k = 0; k < E; ++k) {
        const float gk = __fmul_rn(g[k], gs);
        if (e + k < end) acc = fma((double)gk, (double)gk, acc);     // padding counts in no norm
      }
    }
  });
  red[threadIdx.x] = acc;
  tree_sum(red, blockDim.x);
  if (threadIdx.x == 0) row[blockIdx.x] = red[0];
  // the staging window is shared by all buckets: once every CTA of this launch has met its peers here, no peer
  // reads this rank's staging any more, and the next pack may overwrite it
  barrier_peers(pv, channel);
}

// The window of rank r: float64 totals [parity][source rank] at win_off.  As loss_scale_update's flags (see
// loss_scale.cu): the block works in parity g & 1 of its barrier generation g; a peer can be at most one
// participation ahead, so it writes the other parity while this block reads, and nothing writes parity g & 1 again
// before the reads are done.
__global__ void __launch_bounds__(kClipUpdateThreads) clip_norm_update_kernel(PeerView pv, int channel, size_t win_off,
                                                                              const double* scratch, int nrows,
                                                                              int row_len, double max_norm,
                                                                              float* grad_norm, OptHParams* hp,
                                                                              int ngroups) {
  __shared__ double rows[kClipUpdateThreads];
  const int W = pv.world, me = pv.rank;
  const uint32_t par = pv.epoch[channel * kMaxBlocks + blockIdx.x] & 1u;
  // each bucket's row in CTA order (one thread per bucket), then the buckets in bucket order (thread 0)
  double total = 0.0;
  for (int b0 = 0; b0 < nrows; b0 += blockDim.x) {
    const int b = b0 + threadIdx.x;
    double s = 0.0;
    if (b < nrows)
      for (int c = 0; c < row_len; ++c) s += scratch[(size_t)b * row_len + c];
    rows[threadIdx.x] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      const int n = nrows - b0 < (int)blockDim.x ? nrows - b0 : (int)blockDim.x;
      for (int i = 0; i < n; ++i) total += rows[i];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) rows[0] = total;
  __syncthreads();
  total = rows[0];
  if (threadIdx.x < W) {
    double* dst = reinterpret_cast<double*>(pv.data[threadIdx.x] + win_off) + par * kMaxRanks + me;
    asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(dst), "d"(total) : "memory");
  }
  barrier_peers(pv, channel);
  if (threadIdx.x != 0) return;
  const volatile double* win = reinterpret_cast<const volatile double*>(pv.data[me] + win_off) + par * kMaxRanks;
  double sum = 0.0;
  for (int r = 0; r < W; ++r) sum += win[r];
  const double n = sqrt(sum);
  *grad_norm = (float)n;
  // torch: clamp(max_norm / (N + 1e-6), max=1); a NaN norm gives a NaN coefficient, as torch's clamp does
  const double c = max_norm / (n + 1e-6);
  const float coef = (float)(c > 1.0 ? 1.0 : c);
  for (int g = 0; g < ngroups; ++g) hp[g].grad_scale = __fmul_rn(hp[g].grad_scale, coef);
}

}  // namespace

cudaError_t launch_clip_norm_partial(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                     size_t stage_off, size_t total_elems, float scale, const LambParam* params,
                                     int nparams, double* row, const OptHParams* hp, int blocks, int threads,
                                     int channel, int use_nvls, cudaStream_t stream) {
  if (bad_geometry(blocks, threads) || (stage_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      row == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  return dispatch_pair(grad_dtype, wire, [&](auto g, auto w) {
    using G = decltype(g);
    using W = decltype(w);
    clip_norm_partial_kernel<G, W><<<blocks, threads, 0, stream>>>(pv, segs, nsegs, stage_off, total_elems / 8,
                                                                   scale, params, nparams, row, hp, use_nvls,
                                                                   channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_clip_norm_update(const PeerView& pv, int channel, size_t win_off, const double* scratch, int nrows,
                                    int row_len, double max_norm, float* grad_norm, OptHParams* hp, int ngroups,
                                    cudaStream_t stream) {
  if (pv.world < 1 || pv.world > kMaxRanks || channel < 0 || channel > 1 || (win_off & 15) || scratch == nullptr ||
      nrows < 1 || row_len < 1 || !(max_norm > 0.0) || !isfinite(max_norm) || grad_norm == nullptr || hp == nullptr ||
      ngroups < 1)
    return cudaErrorInvalidValue;
  // one block, always block 0: barrier_peers pairs CTAs by index, so every rank meets in the same CTA
  clip_norm_update_kernel<<<1, kClipUpdateThreads, 0, stream>>>(pv, channel, win_off, scratch, nrows, row_len,
                                                                max_norm, grad_norm, hp, ngroups);
  return cudaGetLastError();
}

cudaError_t clip_load_kernels() {
  cudaFuncAttributes a;
  cudaError_t e = cudaSuccess;
  auto load = [&](const void* k) {
    if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, k);
  };
  for (int gd : {WIRE_F32, WIRE_BF16, WIRE_F16})
    for (int wd : {WIRE_F32, WIRE_BF16, WIRE_F16})
      dispatch_pair(gd, wd, [&](auto g, auto w) {
        using G = decltype(g);
        using W = decltype(w);
        load((const void*)clip_norm_partial_kernel<G, W>);
        return cudaSuccess;
      });
  load((const void*)clip_norm_update_kernel);
  return e;
}

}  // namespace bps
