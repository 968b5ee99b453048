// Fused push-pull kernels for sm_90a (see pushpull.cuh for the contract).
//
// Geometry.  A wire UNIT is one 16-byte vector of the wire dtype W: E = 8
// elements for bf16/fp16, E = 4 for fp32.  Consecutive lanes touch consecutive
// units, so every NVLink access is a fully used 32-byte sector pair (an earlier
// revision used 8-element units for fp32, i.e. 16-byte accesses at a 32-byte
// stride, and ran at half the bandwidth).  Shards are cut in groups of 8
// elements so host and device agree independently of W: rank r owns the
// contiguous range of groups [r*per, (r+1)*per).  Inside a shard, tiles of
// (blockDim * UNROLL) units are dealt round-robin to the CTAs; the same
// (shard-local tile -> blockIdx) map is used on every rank and in every phase,
// so the CTA that packs a tile on rank A is the peer-barrier partner of the CTA
// that reduces it on rank B.  That lets every cross-rank dependency be a
// per-CTA flag barrier; no grid-wide sync exists anywhere.
#include "kernels/pushpull.cuh"

#include "kernels/common.cuh"
#include "kernels/pushpull_dev.cuh"

namespace bps {

namespace {

// ---------------------------------------------------------------- kernels
// mode: 0 = reduce-scatter + all-gather, 1 = reduce-scatter only, 2 = all-gather only
template <class W>
__global__ void __launch_bounds__(512) pushpull_inplace_kernel(PeerView pv, size_t off, size_t total_groups,
                                                               float scale, int mode, int nvls, int channel) {
  constexpr int E = W::kPerVec;
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  barrier_peers(pv, channel);
  if (mode == 2) {
    const char* mine = pv.data[pv.rank] + off;
    for_owned_tiles<kUnroll>(s0, s1, [&](size_t t) {
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) {
        size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
        if (unit < s1) {
          float f[E];
          W::unpack(ld_stream16(mine + unit * 16), f);
#pragma unroll
          for (int k = 0; k < E; ++k) f[k] *= scale;
          sink_peers<W, E>(pv, off, unit, f, nvls != 0);
        }
      }
    });
  } else {
    EpiScale epi{scale};
    if (mode == 0) {
      reduce_phase<W, kUnroll>(pv, off, s0, s1, nvls != 0, rot_of(pv), epi,
                               [&](const float* f, size_t unit) { sink_peers<W, E>(pv, off, unit, f, nvls != 0); });
    } else {
      char* mine = pv.data[pv.rank] + off;
      reduce_phase<W, kUnroll>(pv, off, s0, s1, nvls != 0, rot_of(pv), epi,
                               [&](const float* f, size_t unit) { st_stream16(mine + unit * 16, W::pack(f)); });
    }
  }
  barrier_peers(pv, channel);
}

template <class U, class W>
__global__ void __launch_bounds__(512) pushpull_packed_kernel(PeerView pv, const SegDesc* segs, int nsegs,
                                                              size_t stage_off, size_t total_groups, float scale,
                                                              int nvls, int one_shot, int end_barrier, int channel) {
  constexpr int E = W::kPerVec;
  pack_phase<U, W, kUnroll>(pv, segs, nsegs, stage_off, total_groups);
  barrier_peers(pv, channel);
  EpiScale epi{scale};
  if (one_shot) {
    // every rank reduces every unit and scatters straight into the user tensors.
    // Shard r is summed in the peer order its owner uses in two-shot mode (rotation r + 1),
    // so the results are bit-identical on all ranks and in both modes.
    SegCursor cur;
    bool inited = false;
    for (int r = 0; r < pv.world; ++r) {
      size_t s0, s1;
      shard_units_of<E>(total_groups, pv.world, r, &s0, &s1);
      const int rot = r + 1 == pv.world ? 0 : r + 1;
      reduce_phase<W, kUnroll>(pv, stage_off, s0, s1, nvls != 0, rot, epi, [&](const float* f, size_t unit) {
        int64_t e = (int64_t)unit * E;
        if (!inited) {
          cur.init(segs, nsegs, e);
          inited = true;
        }
        // round through the wire dtype so one-shot and two-shot agree bit for bit
        float g[E];
        W::unpack(W::pack(f), g);
        scatter_elems<U, E>(cur, e, g);
      });
    }
    if (end_barrier) barrier_peers(pv, channel);
  } else {
    size_t s0, s1;
    shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
    reduce_phase<W, kUnroll>(pv, stage_off, s0, s1, nvls != 0, rot_of(pv), epi,
                             [&](const float* f, size_t unit) { sink_peers<W, E>(pv, stage_off, unit, f, nvls != 0); });
    barrier_peers(pv, channel);
    unpack_phase<U, W, kUnroll>(pv, segs, nsegs, stage_off, total_groups);
  }
}

template <class G, class W, class P, class Epi>
__global__ void __launch_bounds__(512) pushpull_fused_opt_kernel(PeerView pv, const SegDesc* segs, int nsegs,
                                                                 size_t stage_off, size_t param_off,
                                                                 size_t total_groups, Epi epi_proto,
                                                                 const OptHParams* hp, int nvls, int channel) {
  constexpr int E = W::kPerVec;
  pack_phase<G, W, kUnrollOpt>(pv, segs, nsegs, stage_off, total_groups);
  barrier_peers(pv, channel);
  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  Epi epi = epi_proto;
  epi.shard_begin = s0 * E;
  epi.hp = *hp;
  if (epi.hp.skip) s1 = s0;     // a step skipped by dynamic loss scaling: no update, nothing written
  reduce_phase<W, kUnrollOpt>(pv, stage_off, s0, s1, nvls != 0, rot_of(pv), epi,
                           [&](const float* f, size_t unit) { sink_peers<P, E>(pv, param_off, unit, f, nvls != 0); });
  barrier_peers(pv, channel);
}

// ---- TMA-streamed variant of the fused optimizer kernel ---------------------------------------
// The LSU kernel above holds the gradient AND the fp32 optimizer state of a unit in registers
// (100-113 registers, one 512-thread CTA per SM, ~40 KB of loads in flight per SM).  Here the state streams (master weights, momentum / Adam
// moments - contiguous fp32 arrays of this rank's shard) move through a shared-memory ring with
// 1-D bulk copies: a producer thread prefetches `stages` tiles ahead (cp.async.bulk + mbarrier
// complete_tx), consumers read the state from shared memory, update it in place and one thread
// writes the tile back with bulk stores.  Only the gradient reduction (multimem.ld_reduce or
// P2P loads, issued BEFORE the wait on the state) and the parameter all-gather (multimem.st /
// P2P stores) use registers, so the bytes in flight are bounded by shared memory, not by the
// register file.  Requires the gradient window in the arena (no pack phase) and W == P.
constexpr int kOptTileUnits = 256;               // wire units per tile = consumer threads
constexpr int kOptThreads = kOptTileUnits + 32;  // + producer warp
constexpr int kOptMaxStages = 8;

struct OptSmem {
  uint64_t full[kOptMaxStages];
  uint64_t empty[kOptMaxStages];
};

template <int E>
__device__ __forceinline__ void lds_f(const unsigned char* p, float* f) {
#pragma unroll
  for (int k = 0; k < E; k += 4) {
    Vec16 v = lds16(p + k * 4);
    f[k] = __uint_as_float(v.x); f[k + 1] = __uint_as_float(v.y);
    f[k + 2] = __uint_as_float(v.z); f[k + 3] = __uint_as_float(v.w);
  }
}
template <int E>
__device__ __forceinline__ void sts_f(unsigned char* p, const float* f) {
#pragma unroll
  for (int k = 0; k < E; k += 4)
    sts16(p + k * 4, Vec16{__float_as_uint(f[k]), __float_as_uint(f[k + 1]), __float_as_uint(f[k + 2]),
                           __float_as_uint(f[k + 3])});
}

template <class W, class Epi>
__global__ void __launch_bounds__(kOptThreads, 2) pushpull_fused_opt_tma_kernel(PeerView pv, size_t grad_off,
                                                                             size_t param_off, size_t total_groups,
                                                                             Epi epi_proto, const OptHParams* hp,
                                                                             int nvls, int stages, int channel) {
  constexpr int E = W::kPerVec;
  constexpr uint32_t kUnitBytes = E * 4;                       // fp32 state of one wire unit, one stream
  constexpr size_t kStreamBytes = (size_t)kOptTileUnits * kUnitBytes;
  constexpr size_t kStageBytes = Epi::kStreams * kStreamBytes;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  OptSmem* sm = reinterpret_cast<OptSmem*>(smem_raw);
  unsigned char* ring = smem_raw + 128;                        // [stage][stream][kStreamBytes]

  size_t s0, s1;
  shard_units_of<E>(total_groups, pv.world, pv.rank, &s0, &s1);
  Epi epi = epi_proto;
  epi.shard_begin = s0 * E;
  epi.hp = *hp;
  if (epi.hp.skip) s1 = s0;     // a step skipped by dynamic loss scaling: no tile, nothing written
  const int nstreams = epi.active_streams();
  const bool is_producer = (threadIdx.x >> 5) == (kOptTileUnits >> 5);

  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], 1);
    }
    mbar_fence_init();
  }
  barrier_peers(pv, channel);   // includes __syncthreads: mbarriers initialised, every peer's gradients are ready
  fence_proxy_async();

  const size_t first = s0 + (size_t)blockIdx.x * kOptTileUnits;
  const size_t stride = (size_t)gridDim.x * kOptTileUnits;

  if (is_producer) {
    if ((threadIdx.x & 31) == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (size_t t = first; t < s1; t += stride) {
        const uint32_t units = (uint32_t)((s1 - t) < (size_t)kOptTileUnits ? (s1 - t) : (size_t)kOptTileUnits);
        const uint32_t bytes = units * kUnitBytes;
        mbar_wait(&sm->empty[s], phase ^ 1);                   // slot written back (first pass falls through)
        mbar_arrive_expect_tx(&sm->full[s], bytes * nstreams);
        unsigned char* dst = ring + (size_t)s * kStageBytes;
        const size_t li = (t - s0) * E;                        // shard-local element index
        for (int i = 0; i < nstreams; ++i)
          bulk_g2s(dst + (size_t)i * kStreamBytes, epi.stream(i) + li, bytes, &sm->full[s]);
        if (++s == stages) {
          s = 0;
          phase ^= 1;
        }
      }
    }
  } else {
    const int rot = rot_of(pv);
    int s = 0, prev_s = -1;
    uint32_t phase = 0;
    // One load per unit (in-switch reduction, or a single rank): the NEXT tile's gradient vector is
    // requested before the current tile is processed, so its latency hides behind the update math.
    const bool single_load = nvls != 0 || pv.world == 1;
    auto grad_raw = [&](size_t tile) {
      Vec16 v{0u, 0u, 0u, 0u};
      const size_t u = tile + threadIdx.x;
      if (tile < s1 && u < s1)
        v = nvls ? W::mm_reduce(pv.mc_data + grad_off + u * 16) : ld_stream16(pv.data[0] + grad_off + u * 16);
      return v;
    };
    Vec16 g_next{0u, 0u, 0u, 0u};
    if (single_load) g_next = grad_raw(first);
    for (size_t t = first; t < s1; t += stride) {
      const uint32_t units = (uint32_t)((s1 - t) < (size_t)kOptTileUnits ? (s1 - t) : (size_t)kOptTileUnits);
      const size_t unit = t + threadIdx.x;
      const bool valid = threadIdx.x < units;
      float acc[E];
      if (single_load) {
        const Vec16 g_cur = g_next;
        g_next = grad_raw(t + stride);
        W::unpack(g_cur, acc);
      } else {
        // several peers: 16-byte loads from every rank, summed in fp32 (NVLink-bound, no prefetch)
        const size_t idx[1] = {unit};
        const bool vld[1] = {valid};
        float a1[1][E];
        reduce_units_p2p<W, 1>(pv, grad_off, idx, vld, rot, a1);
#pragma unroll
        for (int k = 0; k < E; ++k) acc[k] = a1[0][k];
      }
      unsigned char* slot = ring + (size_t)s * kStageBytes;
      mbar_wait(&sm->full[s], phase);                          // state tile has landed
      if (valid) {
        typename Epi::template State<E> st;
        for (int i = 0; i < nstreams; ++i)
          lds_f<E>(slot + (size_t)i * kStreamBytes + threadIdx.x * kUnitBytes, epi.template field<E>(st, i));
        epi.template update<E>(acc, st);
        for (int i = 0; i < nstreams; ++i)
          sts_f<E>(slot + (size_t)i * kStreamBytes + threadIdx.x * kUnitBytes, epi.template field<E>(st, i));
        sink_peers<W, E>(pv, param_off, unit, acc, nvls != 0);   // new parameters to every replica
      }
      fence_proxy_async_smem();                                // generic-proxy writes -> visible to the bulk stores
      named_bar_sync(1, kOptTileUnits);
      if (threadIdx.x == 0) {
        const uint32_t bytes = units * kUnitBytes;
        const size_t li = (t - s0) * E;
        for (int i = 0; i < nstreams; ++i) bulk_s2g(epi.stream(i) + li, slot + (size_t)i * kStreamBytes, bytes);
        bulk_commit();
        if (prev_s >= 0) {
          bulk_wait_read<1>();                                 // the previous tile's stores have read their slot
          mbar_arrive(&sm->empty[prev_s]);
        }
        prev_s = s;
      }
      if (++s == stages) {
        s = 0;
        phase ^= 1;
      }
    }
    if (threadIdx.x == 0) {
      bulk_wait<0>();                                          // all state write-backs of this CTA are complete
      fence_proxy_async();
    }
  }
  barrier_peers(pv, channel);
}

__global__ void barrier_only_kernel(PeerView pv, int channel) { barrier_peers(pv, channel); }

// ---------------------------------------------------------------- dispatch helpers
inline size_t groups_of(size_t nelem) { return (nelem + 7) / 8; }

template <class F>
cudaError_t dispatch_wire(int wire, F&& f) {
  switch (wire) {
    case WIRE_F32: return f(TagF32{});
    case WIRE_BF16: return f(TagBF16{});
    case WIRE_F16: return f(TagF16{});
    default: return cudaErrorInvalidValue;
  }
}

}  // namespace

cudaError_t launch_pushpull_inplace(const PeerView& pv, int wire, size_t off, size_t nelem, float scale,
                                    const LaunchCfg& cfg, cudaStream_t stream) {
  if (cfg.blocks < 1 || cfg.blocks > kMaxBlocks || (off & 15)) return cudaErrorInvalidValue;
  return dispatch_wire(wire, [&](auto w) {
    using W = decltype(w);
    pushpull_inplace_kernel<W><<<cfg.blocks, cfg.threads, 0, stream>>>(pv, off, groups_of(nelem), scale, 0,
                                                                       cfg.use_nvls, cfg.channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_reduce_scatter(const PeerView& pv, int wire, size_t off, size_t nelem, const LaunchCfg& cfg,
                                  cudaStream_t stream) {
  if (cfg.blocks < 1 || cfg.blocks > kMaxBlocks || (off & 15)) return cudaErrorInvalidValue;
  return dispatch_wire(wire, [&](auto w) {
    using W = decltype(w);
    pushpull_inplace_kernel<W><<<cfg.blocks, cfg.threads, 0, stream>>>(pv, off, groups_of(nelem), 1.0f, 1,
                                                                       cfg.use_nvls, cfg.channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_all_gather(const PeerView& pv, int wire, size_t off, size_t nelem, float scale,
                              const LaunchCfg& cfg, cudaStream_t stream) {
  if (cfg.blocks < 1 || cfg.blocks > kMaxBlocks || (off & 15)) return cudaErrorInvalidValue;
  return dispatch_wire(wire, [&](auto w) {
    using W = decltype(w);
    pushpull_inplace_kernel<W><<<cfg.blocks, cfg.threads, 0, stream>>>(pv, off, groups_of(nelem), scale, 2,
                                                                       cfg.use_nvls, cfg.channel);
    return cudaGetLastError();
  });
}

cudaError_t launch_pushpull_packed(const PeerView& pv, int user_dtype, int wire, const SegDesc* segs, int nsegs,
                                   size_t stage_off, size_t total_elems, float scale, const LaunchCfg& cfg,
                                   cudaStream_t stream) {
  if (cfg.blocks < 1 || cfg.blocks > kMaxBlocks || (stage_off & 15) || (total_elems & 7)) return cudaErrorInvalidValue;
  const size_t groups = total_elems / 8;
#define BPS_PACKED(U, W)                                                                                             \
  pushpull_packed_kernel<U, W><<<cfg.blocks, cfg.threads, 0, stream>>>(pv, segs, nsegs, stage_off, groups, scale,    \
                                                                       cfg.use_nvls, cfg.one_shot, cfg.end_barrier,  \
                                                                       cfg.channel);                                 \
  return cudaGetLastError();
  if (user_dtype == WIRE_F32 && wire == WIRE_F32) { BPS_PACKED(TagF32, TagF32) }
  if (user_dtype == WIRE_F32 && wire == WIRE_BF16) { BPS_PACKED(TagF32, TagBF16) }
  if (user_dtype == WIRE_F32 && wire == WIRE_F16) { BPS_PACKED(TagF32, TagF16) }
  if (user_dtype == WIRE_BF16 && wire == WIRE_BF16) { BPS_PACKED(TagBF16, TagBF16) }
  if (user_dtype == WIRE_F16 && wire == WIRE_F16) { BPS_PACKED(TagF16, TagF16) }
  if (user_dtype == WIRE_BF16 && wire == WIRE_F32) { BPS_PACKED(TagBF16, TagF32) }
  if (user_dtype == WIRE_F16 && wire == WIRE_F32) { BPS_PACKED(TagF16, TagF32) }
#undef BPS_PACKED
  return cudaErrorInvalidValue;
}

cudaError_t launch_pushpull_fused_opt(const PeerView& pv, int grad_dtype, int wire, int param_dtype, int opt_kind,
                                      const SegDesc* segs, int nsegs, size_t stage_off, size_t param_off,
                                      size_t total_elems, float scale, float* master, float* state0, float* state1,
                                      const OptHParams* hp, const LaunchCfg& cfg, cudaStream_t stream) {
  if (cfg.blocks < 1 || cfg.blocks > kMaxBlocks || (stage_off & 15) || (param_off & 15) || (total_elems & 7))
    return cudaErrorInvalidValue;
  const size_t groups = total_elems / 8;
#define BPS_FUSED(G, W, P)                                                                                           \
  if (opt_kind == OPT_SGD) {                                                                                         \
    EpiSGD e{master, state0, 0, scale, OptHParams{}};                                                                \
    pushpull_fused_opt_kernel<G, W, P, EpiSGD><<<cfg.blocks, cfg.threads, 0, stream>>>(                              \
        pv, segs, nsegs, stage_off, param_off, groups, e, hp, cfg.use_nvls, cfg.channel);                            \
  } else if (opt_kind == OPT_ADAM) {                                                                                 \
    EpiAdam e{master, state0, state1, 0, scale, OptHParams{}};                                                       \
    pushpull_fused_opt_kernel<G, W, P, EpiAdam><<<cfg.blocks, cfg.threads, 0, stream>>>(                             \
        pv, segs, nsegs, stage_off, param_off, groups, e, hp, cfg.use_nvls, cfg.channel);                            \
  } else {                                                                                                           \
    return cudaErrorInvalidValue;                                                                                    \
  }                                                                                                                  \
  return cudaGetLastError();
  // exactly the (gradient, wire) pairs the bucket layer produces: fp32 gradients on an fp32, bf16 or fp16 wire,
  // 16-bit gradients on their own dtype; parameters always have the gradient dtype
  if (grad_dtype == WIRE_BF16 && wire == WIRE_BF16 && param_dtype == WIRE_BF16) { BPS_FUSED(TagBF16, TagBF16, TagBF16) }
  if (grad_dtype == WIRE_F32 && wire == WIRE_F32 && param_dtype == WIRE_F32) { BPS_FUSED(TagF32, TagF32, TagF32) }
  if (grad_dtype == WIRE_F32 && wire == WIRE_BF16 && param_dtype == WIRE_F32) { BPS_FUSED(TagF32, TagBF16, TagF32) }
  if (grad_dtype == WIRE_F32 && wire == WIRE_F16 && param_dtype == WIRE_F32) { BPS_FUSED(TagF32, TagF16, TagF32) }
  if (grad_dtype == WIRE_F16 && wire == WIRE_F16 && param_dtype == WIRE_F16) { BPS_FUSED(TagF16, TagF16, TagF16) }
#undef BPS_FUSED
  return cudaErrorInvalidValue;
}

namespace {
template <class W, class Epi>
cudaError_t launch_opt_tma(const PeerView& pv, const Epi& e, size_t grad_off, size_t param_off, size_t groups,
                           const OptHParams* hp, int blocks, int stages, int use_nvls, int channel,
                           cudaStream_t stream) {
  const size_t smem = 128 + (size_t)stages * Epi::kStreams * kOptTileUnits * W::kPerVec * 4;
  if (smem > 227 * 1024) return cudaErrorInvalidValue;
  cudaError_t err = cudaFuncSetAttribute(pushpull_fused_opt_tma_kernel<W, Epi>,
                                         cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (err != cudaSuccess) return err;
  pushpull_fused_opt_tma_kernel<W, Epi><<<blocks, kOptThreads, smem, stream>>>(pv, grad_off, param_off, groups, e, hp,
                                                                               use_nvls, stages, channel);
  return cudaGetLastError();
}
}  // namespace

cudaError_t launch_pushpull_fused_opt_tma(const PeerView& pv, int wire, int opt_kind, size_t grad_off,
                                          size_t param_off, size_t total_elems, float scale, float* master,
                                          float* state0, float* state1, const OptHParams* hp, int blocks, int stages,
                                          int use_nvls, int channel, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks || (grad_off & 15) || (param_off & 15) || (total_elems & 7) || stages < 2 ||
      stages > kOptMaxStages || (opt_kind != OPT_SGD && opt_kind != OPT_ADAM))
    return cudaErrorInvalidValue;
  const size_t groups = total_elems / 8;
  return dispatch_wire(wire, [&](auto w) {
    using W = decltype(w);
    if (opt_kind == OPT_SGD) {
      EpiSGD e{master, state0, 0, scale, OptHParams{}};
      return launch_opt_tma<W, EpiSGD>(pv, e, grad_off, param_off, groups, hp, blocks, stages, use_nvls, channel,
                                       stream);
    }
    EpiAdam e{master, state0, state1, 0, scale, OptHParams{}};
    return launch_opt_tma<W, EpiAdam>(pv, e, grad_off, param_off, groups, hp, blocks, stages, use_nvls, channel,
                                      stream);
  });
}

cudaError_t launch_barrier(const PeerView& pv, int blocks, int channel, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  barrier_only_kernel<<<blocks, 32, 0, stream>>>(pv, channel);
  return cudaGetLastError();
}

}  // namespace bps
