// LARS in the fused exchange: the three kernels of a bucket (see pushpull_lars.cuh for the sequence).
//
// The pack phase, the peer reduction and the all-gather sink are those of the fused SGD kernel (pushpull_dev.cuh);
// the parameter cursor, the segmented warp sums and the norm exchange are LAMB's (pushpull_trust.cuh).  Grids depend
// on the bucket only, so barrier_peers pairs the same CTA index on every rank, a rank with an empty shard included.
#include "kernels/pushpull_lars.cuh"

#include "kernels/common.cuh"
#include "kernels/pushpull_dev.cuh"
#include "kernels/pushpull_trust.cuh"

namespace bps {

namespace {

// (512, 1): without the minimum-blocks hint ptxas picks 64 registers for the bf16 wire and spills
template <class G, class W>
__global__ void __launch_bounds__(512, 1) lars_norms_partial_kernel(PeerView pv, const SegDesc* segs, int nsegs,
                                                                 size_t stage_off, size_t total_groups, float scale,
                                                                 const float* master, const LambParam* params,
                                                                 int nparams, double* scratch, const OptHParams* hpp,
                                                                 int nvls, int channel) {
  constexpr int E = W::kPerVec;
  pack_phase<G, W, kUnrollOpt>(pv, segs, nsegs, stage_off, total_groups);
  barrier_peers(pv, channel);
  const OptHParams hp = *hpp;
  if (hp.skip) return;          // a step skipped by dynamic loss scaling: nothing written
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  double2* heads = reinterpret_cast<double2*>(scratch);
  double2* groups = heads + nparams;
  const float gs = scale * hp.grad_scale;
  const int lane = threadIdx.x & 31;
  const int rot = rot_of(pv);
  ParamCursor cur;
  bool inited = false;
  for_owned_tiles<1>(s0, s1, [&](size_t t) {
    const size_t unit = t + threadIdx.x;
    const bool valid = unit < s1;       // the invalid lanes of a tile are its last ones
    float w[E], g[E];
    if (valid) ldf<E>(master + (unit - s0) * E, w);
    if (nvls) {
      if (valid) W::unpack(W::mm_reduce(pv.mc_data + stage_off + unit * 16), g);
    } else {
      reduce_unit_p2p<W>(pv, stage_off, unit, valid, rot, g);
    }
    double w2 = 0.0, g2 = 0.0;
    int pid = -1;
    if (valid) {
      const int64_t e = (int64_t)(unit * E);
      pid = cur.at(params, nparams, e, inited);
      const int64_t end = __ldg(&params[pid].start) + __ldg(&params[pid].n);
#pragma unroll
      for (int k = 0; k < E; ++k) {
        const float gk = __fmul_rn(g[k], gs);     // as lars_apply forms it
        if (e + k < end) {      // padding counts in no norm
          w2 = fma((double)w[k], (double)w[k], w2);
          g2 = fma((double)gk, (double)gk, g2);
        }
      }
    }
    BPS_STORE_SEGMENT_SUMS(w2, g2, pid, valid, lane, unit, s0, groups, heads);
  });
}

template <int E>
__global__ void __launch_bounds__(kNormThreads) lars_norms_kernel(PeerView pv, size_t total_groups,
                                                                  const LambParam* params, int nparams,
                                                                  const double* scratch, size_t win_off, float* phi,
                                                                  const OptHParams* hpp, int channel) {
  exchange_norms<E>(pv, total_groups, params, nparams, scratch, win_off, phi, hpp->skip != 0, channel,
                    [&](double ws, double gs) {
                      if (!hpp->adapt || !(ws > 0.0) || !(gs > 0.0)) return 1.f;
                      const double wn = sqrt(ws);
                      const double den = sqrt(gs) + (double)hpp->weight_decay * wn + (double)hpp->eps;
                      return (float)((double)hpp->trust_coefficient * wn / den);
                    });
}

template <class W, class P>
__global__ void __launch_bounds__(512) lars_apply_kernel(PeerView pv, size_t stage_off, size_t param_off,
                                                         size_t total_groups, float scale, float* master, float* mom,
                                                         const LambParam* params, int nparams, const float* phi,
                                                         const OptHParams* hpp, int nvls, int channel) {
  constexpr int E = W::kPerVec;
  const OptHParams hp = *hpp;
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  if (hp.skip) s1 = s0;
  const float gs = scale * hp.grad_scale;
  const int rot = rot_of(pv);
  ParamCursor cur;
  bool inited = false;
  for_owned_tiles<1>(s0, s1, [&](size_t t) {
    const size_t unit = t + threadIdx.x;
    if (unit >= s1) return;
    const size_t li = (unit - s0) * E;
    float w[E], v[E], g[E];
    ldf<E>(master + li, w);
    ldf<E>(mom + li, v);
    if (nvls) W::unpack(W::mm_reduce(pv.mc_data + stage_off + unit * 16), g);
    else reduce_unit_p2p<W>(pv, stage_off, unit, true, rot, g);
    const float lr_phi = hp.lr * __ldg(&phi[cur.at(params, nparams, (int64_t)(unit * E), inited)]);
#pragma unroll
    for (int k = 0; k < E; ++k) {
      const float d = __fmaf_rn(hp.weight_decay, w[k], __fmul_rn(g[k], gs));
      v[k] = __fmaf_rn(lr_phi, d, __fmul_rn(hp.momentum, v[k]));
      w[k] = __fsub_rn(w[k], v[k]);
    }
    stf<E>(master + li, w);
    stf<E>(mom + li, v);
    sink_peers<P, E>(pv, param_off, unit, w, nvls != 0);
  });
  barrier_peers(pv, channel);
}

}  // namespace

cudaError_t launch_lars_norms_partial(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                      size_t stage_off, size_t total_elems, float scale, const float* master,
                                      const LambParam* params, int nparams, double* scratch, const OptHParams* hp,
                                      int blocks, int threads, int channel, int use_nvls, cudaStream_t stream) {
  if (bad_geometry(blocks, threads) || (stage_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      scratch == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  return dispatch_pair(grad_dtype, wire, [&](auto g, auto w) {
    using G = decltype(g);
    using W = decltype(w);
    lars_norms_partial_kernel<G, W><<<blocks, threads, 0, stream>>>(pv, segs, nsegs, stage_off, total_elems / 8,
                                                                    scale, master, params, nparams, scratch, hp,
                                                                    use_nvls, channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_lars_norms(const PeerView& pv, int wire, size_t total_elems, const LambParam* params, int nparams,
                              const double* scratch, size_t win_off, float* phi, const OptHParams* hp, int blocks,
                              int channel, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks || (win_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      scratch == nullptr || phi == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  if (wire == WIRE_F32)
    lars_norms_kernel<4><<<blocks, kNormThreads, 0, stream>>>(pv, total_elems / 8, params, nparams, scratch, win_off,
                                                              phi, hp, channel);
  else if (wire == WIRE_BF16 || wire == WIRE_F16)
    lars_norms_kernel<8><<<blocks, kNormThreads, 0, stream>>>(pv, total_elems / 8, params, nparams, scratch, win_off,
                                                              phi, hp, channel);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_lars_apply(const PeerView& pv, int grad_dtype, int wire, size_t stage_off, size_t param_off,
                              size_t total_elems, float scale, float* master, float* mom, const LambParam* params,
                              int nparams, const float* phi, const OptHParams* hp, int blocks, int threads,
                              int channel, int use_nvls, cudaStream_t stream) {
  if (bad_geometry(blocks, threads) || (stage_off & 15) || (param_off & 15) || (total_elems & 7) || nparams < 1 ||
      params == nullptr || phi == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  return dispatch_pair(grad_dtype, wire, [&](auto g, auto w) {
    using G = decltype(g);
    using W = decltype(w);
    lars_apply_kernel<W, G><<<blocks, threads, 0, stream>>>(pv, stage_off, param_off, total_elems / 8, scale, master,
                                                            mom, params, nparams, phi, hp, use_nvls, channel);
    return cudaGetLastError();
  });
}

cudaError_t lars_load_kernels() {
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
        load((const void*)lars_norms_partial_kernel<G, W>);
        load((const void*)lars_apply_kernel<W, G>);
        return cudaSuccess;
      });
  load((const void*)lars_norms_kernel<4>);
  load((const void*)lars_norms_kernel<8>);
  return e;
}

}  // namespace bps
