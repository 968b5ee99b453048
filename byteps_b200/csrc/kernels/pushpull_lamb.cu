// LAMB in the fused exchange: the three kernels of a bucket (see pushpull_lamb.cuh for the sequence).
//
// The shard geometry, the pack phase, the peer reduction and the all-gather sink are those of the fused Adam kernel
// (pushpull_dev.cuh); the parameter cursor, the segmented warp sums and the norm exchange are shared with LARS
// (pushpull_trust.cuh).  Grids depend on the bucket only: lamb_moments and lamb_apply take the bucket's CTA count,
// lamb_norms one CTA per parameter up to its cap, so barrier_peers pairs the same CTA index on every rank, a rank
// with an empty shard included.
#include "kernels/pushpull_lamb.cuh"

#include "kernels/common.cuh"
#include "kernels/pushpull_dev.cuh"
#include "kernels/pushpull_trust.cuh"

namespace bps {

namespace {

// u of one element from the updated moments and the master before the update.  lamb_moments (for the norm) and
// lamb_apply (for the step) both call this with the same inputs; the rounding steps are spelled out so the two
// agree bit for bit whatever the compiler contracts elsewhere.  MUFU sqrt and divide as in EpiAdam.
__device__ __forceinline__ float lamb_u(float w, float m, float v, float inv_c1, float inv_c2, const OptHParams& hp) {
  const float den = __fadd_rn(sqrt_approx(__fmul_rn(v, inv_c2)), hp.eps);
  return __fmaf_rn(hp.weight_decay, w, __fdividef(__fmul_rn(m, inv_c1), den));
}

template <class G, class W>
__global__ void __launch_bounds__(512) lamb_moments_kernel(PeerView pv, const SegDesc* segs, int nsegs,
                                                           size_t stage_off, size_t total_groups, float scale,
                                                           float* master, float* m1, float* m2,
                                                           const LambParam* params, int nparams, double* scratch,
                                                           const OptHParams* hpp, int nvls, int channel) {
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
  const float inv_c1 = 1.f / hp.bias_c1;
  const float inv_c2 = 1.f / hp.bias_c2;
  const int lane = threadIdx.x & 31;
  const int rot = rot_of(pv);
  ParamCursor cur;
  bool inited = false;
  for_owned_tiles<1>(s0, s1, [&](size_t t) {
    const size_t unit = t + threadIdx.x;
    const bool valid = unit < s1;       // the invalid lanes of a tile are its last ones
    const size_t li = (unit - s0) * E;
    float w[E], m[E], v[E], g[E];
    if (valid) {
      ldf<E>(master + li, w);
      ldf<E>(m1 + li, m);
      ldf<E>(m2 + li, v);
    }
    if (nvls) {
      if (valid) W::unpack(W::mm_reduce(pv.mc_data + stage_off + unit * 16), g);
    } else {
      reduce_unit_p2p<W>(pv, stage_off, unit, valid, rot, g);
    }
    double w2 = 0.0, u2 = 0.0;
    int pid = -1;
    if (valid) {
      const int64_t e = (int64_t)(unit * E);
      pid = cur.at(params, nparams, e, inited);
      const int64_t end = __ldg(&params[pid].start) + __ldg(&params[pid].n);
#pragma unroll
      for (int k = 0; k < E; ++k) {
        const float gk = g[k] * gs;
        m[k] = hp.beta1 * m[k] + (1.f - hp.beta1) * gk;
        v[k] = hp.beta2 * v[k] + (1.f - hp.beta2) * gk * gk;
        const float u = lamb_u(w[k], m[k], v[k], inv_c1, inv_c2, hp);
        if (e + k < end) {      // padding counts in no norm
          w2 = fma((double)w[k], (double)w[k], w2);
          u2 = fma((double)u, (double)u, u2);
        }
      }
      stf<E>(m1 + li, m);
      stf<E>(m2 + li, v);
    }
    BPS_STORE_SEGMENT_SUMS(w2, u2, pid, valid, lane, unit, s0, groups, heads);
  });
}

template <int E>
__global__ void __launch_bounds__(kNormThreads) lamb_norms_kernel(PeerView pv, size_t total_groups,
                                                                  const LambParam* params, int nparams,
                                                                  const double* scratch, size_t win_off, float* phi,
                                                                  const OptHParams* hpp, int channel) {
  exchange_norms<E>(pv, total_groups, params, nparams, scratch, win_off, phi, hpp->skip != 0, channel,
                    [&](double ws, double us) {
                      return (hpp->adapt && ws > 0.0 && us > 0.0) ? (float)(sqrt(ws) / sqrt(us)) : 1.f;
                    });
}

template <class W, class P>
__global__ void __launch_bounds__(512) lamb_apply_kernel(PeerView pv, size_t param_off, size_t total_groups,
                                                         float* master, const float* m1, const float* m2,
                                                         const LambParam* params, int nparams, const float* phi,
                                                         const OptHParams* hpp, int nvls, int channel) {
  constexpr int E = W::kPerVec;
  const OptHParams hp = *hpp;
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  if (hp.skip) s1 = s0;
  const float inv_c1 = 1.f / hp.bias_c1;
  const float inv_c2 = 1.f / hp.bias_c2;
  ParamCursor cur;
  bool inited = false;
  for_owned_tiles<1>(s0, s1, [&](size_t t) {
    const size_t unit = t + threadIdx.x;
    if (unit >= s1) return;
    const size_t li = (unit - s0) * E;
    float w[E], m[E], v[E];
    ldf<E>(master + li, w);
    ldf<E>(m1 + li, m);
    ldf<E>(m2 + li, v);
    const int64_t e = (int64_t)(unit * E);
    const float lr_phi = hp.lr * __ldg(&phi[cur.at(params, nparams, e, inited)]);
#pragma unroll
    for (int k = 0; k < E; ++k) w[k] = __fmaf_rn(-lr_phi, lamb_u(w[k], m[k], v[k], inv_c1, inv_c2, hp), w[k]);
    stf<E>(master + li, w);
    sink_peers<P, E>(pv, param_off, unit, w, nvls != 0);
  });
  barrier_peers(pv, channel);
}

}  // namespace

cudaError_t launch_lamb_moments(const PeerView& pv, int grad_dtype, int wire, const SegDesc* segs, int nsegs,
                                size_t stage_off, size_t total_elems, float scale, float* master, float* m1, float* m2,
                                const LambParam* params, int nparams, double* scratch, const OptHParams* hp,
                                int blocks, int threads, int channel, int use_nvls, cudaStream_t stream) {
  if (bad_geometry(blocks, threads) || (stage_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      scratch == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  return dispatch_pair(grad_dtype, wire, [&](auto g, auto w) {
    using G = decltype(g);
    using W = decltype(w);
    lamb_moments_kernel<G, W><<<blocks, threads, 0, stream>>>(pv, segs, nsegs, stage_off, total_elems / 8, scale,
                                                              master, m1, m2, params, nparams, scratch, hp, use_nvls,
                                                              channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_lamb_norms(const PeerView& pv, int wire, size_t total_elems, const LambParam* params, int nparams,
                              const double* scratch, size_t win_off, float* phi, const OptHParams* hp, int blocks,
                              int channel, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks || (win_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      scratch == nullptr || phi == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  if (wire == WIRE_F32)
    lamb_norms_kernel<4><<<blocks, kNormThreads, 0, stream>>>(pv, total_elems / 8, params, nparams, scratch, win_off,
                                                              phi, hp, channel);
  else if (wire == WIRE_BF16 || wire == WIRE_F16)
    lamb_norms_kernel<8><<<blocks, kNormThreads, 0, stream>>>(pv, total_elems / 8, params, nparams, scratch, win_off,
                                                              phi, hp, channel);
  else
    return cudaErrorInvalidValue;
  return cudaGetLastError();
}

cudaError_t launch_lamb_apply(const PeerView& pv, int grad_dtype, int wire, size_t param_off, size_t total_elems,
                              float* master, const float* m1, const float* m2, const LambParam* params, int nparams,
                              const float* phi, const OptHParams* hp, int blocks, int threads, int channel,
                              int use_nvls, cudaStream_t stream) {
  if (bad_geometry(blocks, threads) || (param_off & 15) || (total_elems & 7) || nparams < 1 || params == nullptr ||
      phi == nullptr || hp == nullptr)
    return cudaErrorInvalidValue;
  return dispatch_pair(grad_dtype, wire, [&](auto g, auto w) {
    using G = decltype(g);
    using W = decltype(w);
    lamb_apply_kernel<W, G><<<blocks, threads, 0, stream>>>(pv, param_off, total_elems / 8, master, m1, m2, params,
                                                            nparams, phi, hp, use_nvls, channel);
    return cudaGetLastError();
  });
}

cudaError_t lamb_load_kernels() {
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
        load((const void*)lamb_moments_kernel<G, W>);
        load((const void*)lamb_apply_kernel<W, G>);
        return cudaSuccess;
      });
  load((const void*)lamb_norms_kernel<4>);
  load((const void*)lamb_norms_kernel<8>);
  return e;
}

}  // namespace bps
