// Device-side building blocks shared by the push-pull kernels (pushpull.cu, pushpull_ring.cu):
// element packing, segment cursors, the peer reduction, the all-gather sink, the optimizer
// epilogues and the tile loops.  Everything has internal linkage (one copy per translation unit).
#pragma once
#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"

namespace bps {

namespace {

constexpr int kPeerChunk = 8;  // peers handled per statically-unrolled pass
constexpr int kUnroll = 2;     // units per thread per tile (16 x 16 B loads in flight with 8 peers)
constexpr int kUnrollOpt = 1;  // fused optimizer epilogues hold master/moment registers too

// ---------------------------------------------------------------- E elements of type T <-> floats
// bytes = E * sizeof(T): 8 (4 x 16-bit), 16, or 32 (8 x fp32)
template <class T, int E>
struct Elems {
  static constexpr int kBytes = E * T::kBytes;
  __device__ static __forceinline__ void load(const char* p, float* f) {
    if constexpr (kBytes == 16) {
      Vec16 v = ld_stream16(p);
      T::unpack(v, f);
    } else if constexpr (kBytes == 32) {
      Vec16 a = ld_stream16(p), b = ld_stream16(p + 16);
      T::unpack(a, f);
      T::unpack(b, f + T::kPerVec);
    } else {  // 8 bytes: four 16-bit values
      uint32_t x, y;
      asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(x), "=r"(y) : "l"(p) : "memory");
      Vec16 v{x, y, 0u, 0u};
      float t[8];
      T::unpack(v, t);
      f[0] = t[0]; f[1] = t[1]; f[2] = t[2]; f[3] = t[3];
    }
  }
  __device__ static __forceinline__ void store(char* p, const float* f) {
    if constexpr (kBytes == 16) {
      st_stream16(p, T::pack(f));
    } else if constexpr (kBytes == 32) {
      st_stream16(p, T::pack(f));
      st_stream16(p + 16, T::pack(f + T::kPerVec));
    } else {
      float t[8] = {f[0], f[1], f[2], f[3], 0.f, 0.f, 0.f, 0.f};
      Vec16 v = T::pack(t);
      asm volatile("st.global.L1::no_allocate.v2.u32 [%0], {%1,%2};" ::"l"(p), "r"(v.x), "r"(v.y) : "memory");
    }
  }
};

// ---------------------------------------------------------------- segment cursor
struct SegCursor {
  const SegDesc* segs;
  int nsegs;
  int i;
  __device__ __forceinline__ void init(const SegDesc* s, int n, int64_t e) {
    segs = s;
    nsegs = n;
    int lo = 0, hi = n - 1;
    while (lo < hi) {  // last seg with start <= e
      int mid = (lo + hi + 1) >> 1;
      if (__ldg(&segs[mid].start) <= e) lo = mid;
      else hi = mid - 1;
    }
    i = lo;
  }
  __device__ __forceinline__ void seek(int64_t e) {
    while (i + 1 < nsegs && __ldg(&segs[i + 1].start) <= e) ++i;
  }
};

// gather E elements starting at flat element e from the user tensors (zero padded)
template <class U, int E>
__device__ __forceinline__ void gather_elems(SegCursor& c, int64_t e, float* f) {
  c.seek(e);
  const int64_t start = __ldg(&c.segs[c.i].start);
  const int64_t n = __ldg(&c.segs[c.i].n);
  const char* src = (const char*)__ldg((const unsigned long long*)&c.segs[c.i].src);
  const int64_t local = e - start;
  if (local + E <= n && ((reinterpret_cast<uintptr_t>(src) & 15) == 0)) {
    Elems<U, E>::load(src + local * U::kBytes, f);
  } else {
#pragma unroll
    for (int k = 0; k < E; ++k) f[k] = (local + k < n && local + k >= 0) ? U::load1(src, local + k) : 0.f;
  }
}

template <class U, int E>
__device__ __forceinline__ void scatter_elems(SegCursor& c, int64_t e, const float* f) {
  c.seek(e);
  const int64_t start = __ldg(&c.segs[c.i].start);
  const int64_t n = __ldg(&c.segs[c.i].n);
  char* dst = (char*)__ldg((const unsigned long long*)&c.segs[c.i].dst);
  const int64_t local = e - start;
  if (local + E <= n && ((reinterpret_cast<uintptr_t>(dst) & 15) == 0)) {
    Elems<U, E>::store(dst + local * U::kBytes, f);
  } else {
#pragma unroll
    for (int k = 0; k < E; ++k)
      if (local + k < n && local + k >= 0) U::store1(dst, local + k, f[k]);
  }
}

// ---------------------------------------------------------------- reduce over peers
template <class W, int UNROLL>
__device__ __forceinline__ void reduce_units_p2p(const PeerView& pv, size_t off, const size_t (&idx)[UNROLL],
                                                 const bool (&valid)[UNROLL], int rot,
                                                 float (&acc)[UNROLL][W::kPerVec]) {
  constexpr int E = W::kPerVec;
#pragma unroll
  for (int u = 0; u < UNROLL; ++u)
#pragma unroll
    for (int k = 0; k < E; ++k) acc[u][k] = 0.f;
  for (int base = 0; base < pv.world; base += kPeerChunk) {
    Vec16 v[UNROLL][kPeerChunk];
#pragma unroll
    for (int j = 0; j < kPeerChunk; ++j) {
      if (base + j < pv.world) {
        int p = base + j + rot;
        if (p >= pv.world) p -= pv.world;
        const char* src = pv.data[p] + off;
#pragma unroll
        for (int u = 0; u < UNROLL; ++u)
          if (valid[u]) v[u][j] = ld_stream16(src + idx[u] * 16);
      }
    }
#pragma unroll
    for (int j = 0; j < kPeerChunk; ++j) {
      if (base + j < pv.world) {
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
          if (valid[u]) {
            float f[E];
            W::unpack(v[u][j], f);
#pragma unroll
            for (int k = 0; k < E; ++k) acc[u][k] += f[k];
          }
        }
      }
    }
  }
}

// write the E results of wire unit `unit` into the window (dtype P) of every rank
template <class P, int E>
__device__ __forceinline__ void sink_peers(const PeerView& pv, size_t off, size_t unit, const float* f, bool nvls) {
  constexpr int kBytes = Elems<P, E>::kBytes;
  const size_t boff = off + unit * kBytes;
  if (nvls && kBytes >= 16) {
    mm_st16(pv.mc_data + boff, P::pack(f));
    if constexpr (kBytes == 32) mm_st16(pv.mc_data + boff + 16, P::pack(f + P::kPerVec));
  } else {
    for (int base = 0; base < pv.world; base += kPeerChunk) {
#pragma unroll
      for (int j = 0; j < kPeerChunk; ++j) {
        if (base + j < pv.world) {
          int p = base + j + pv.rank;
          if (p >= pv.world) p -= pv.world;
          Elems<P, E>::store(pv.data[p] + boff, f);
        }
      }
    }
  }
}

// ---------------------------------------------------------------- epilogues (E elements at a time)
// Epilogue protocol: load<E>(state, elem) is issued BEFORE the peer loads of the same unit so the
// optimizer-state reads overlap the NVLink round trip; apply<E>(g, elem, state) consumes it afterwards.
struct EpiScale {
  float scale;
  template <int E>
  struct State {};
  template <int E>
  __device__ __forceinline__ void load(State<E>&, size_t) const {}
  template <int E>
  __device__ __forceinline__ void apply(float* g, size_t, State<E>&) const {
#pragma unroll
    for (int k = 0; k < E; ++k) g[k] *= scale;
  }
};

template <int E>
__device__ __forceinline__ void ldf(const float* p, float* f) {
#pragma unroll
  for (int k = 0; k < E; k += 4) {
    float4 a = *reinterpret_cast<const float4*>(p + k);
    f[k] = a.x; f[k + 1] = a.y; f[k + 2] = a.z; f[k + 3] = a.w;
  }
}
template <int E>
__device__ __forceinline__ void stf(float* p, const float* f) {
#pragma unroll
  for (int k = 0; k < E; k += 4) *reinterpret_cast<float4*>(p + k) = make_float4(f[k], f[k + 1], f[k + 2], f[k + 3]);
}

__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// g (sum of gradients) -> new weights, updating the fp32 master shard in place.
// `elem` is the flat element index of g[0]; shard_begin is in elements.
struct EpiSGD {
  float* master;
  float* mom;
  size_t shard_begin;
  float scale;
  OptHParams hp;
  static constexpr int kStreams = 2;       // fp32 state streams: master weights, momentum
  template <int E>
  struct State {
    float w[E], m[E];
  };
  __device__ __forceinline__ int active_streams() const { return hp.momentum != 0.f ? 2 : 1; }
  __device__ __forceinline__ float* stream(int i) const { return i == 0 ? master : mom; }
  template <int E>
  __device__ __forceinline__ float* field(State<E>& st, int i) const { return i == 0 ? st.w : st.m; }
  template <int E>
  __device__ __forceinline__ void load(State<E>& st, size_t elem) const {
    const size_t li = elem - shard_begin;
    ldf<E>(master + li, st.w);
    if (hp.momentum != 0.f) ldf<E>(mom + li, st.m);
  }
  // pure math: g (sum of gradients) -> new weights (also left in g), state updated in registers
  template <int E>
  __device__ __forceinline__ void update(float* g, State<E>& st) const {
    const bool has_mom = hp.momentum != 0.f;
    const float gs = scale * hp.grad_scale;
#pragma unroll
    for (int k = 0; k < E; ++k) {
      float gk = g[k] * gs + hp.weight_decay * st.w[k];
      if (has_mom) {
        float b = hp.first_step ? gk : hp.momentum * st.m[k] + (1.f - hp.dampening) * gk;
        st.m[k] = b;
        gk = hp.nesterov ? gk + hp.momentum * b : b;
      }
      st.w[k] -= hp.lr * gk;
      g[k] = st.w[k];
    }
  }
  template <int E>
  __device__ __forceinline__ void apply(float* g, size_t elem, State<E>& st) const {
    const size_t li = elem - shard_begin;
    update<E>(g, st);
    stf<E>(master + li, st.w);
    if (hp.momentum != 0.f) stf<E>(mom + li, st.m);
  }
};

struct EpiAdam {
  float* master;
  float* m1;
  float* m2;
  size_t shard_begin;
  float scale;
  OptHParams hp;
  static constexpr int kStreams = 3;       // master weights, first and second moments
  template <int E>
  struct State {
    float w[E], m[E], v[E];
  };
  __device__ __forceinline__ int active_streams() const { return 3; }
  __device__ __forceinline__ float* stream(int i) const { return i == 0 ? master : (i == 1 ? m1 : m2); }
  template <int E>
  __device__ __forceinline__ float* field(State<E>& st, int i) const {
    return i == 0 ? st.w : (i == 1 ? st.m : st.v);
  }
  template <int E>
  __device__ __forceinline__ void load(State<E>& st, size_t elem) const {
    const size_t li = elem - shard_begin;
    ldf<E>(master + li, st.w);
    ldf<E>(m1 + li, st.m);
    ldf<E>(m2 + li, st.v);
  }
  template <int E>
  __device__ __forceinline__ void update(float* g, State<E>& st) const {
    const float gs = scale * hp.grad_scale;
    const float inv_c1 = 1.f / hp.bias_c1;
    const float inv_c2 = 1.f / hp.bias_c2;
#pragma unroll
    for (int k = 0; k < E; ++k) {
      float gk = g[k] * gs;
      if (hp.adamw) st.w[k] *= (1.f - hp.lr * hp.weight_decay);
      else gk += hp.weight_decay * st.w[k];
      st.m[k] = hp.beta1 * st.m[k] + (1.f - hp.beta1) * gk;
      st.v[k] = hp.beta2 * st.v[k] + (1.f - hp.beta2) * gk * gk;
      // MUFU-based sqrt and reciprocal (<= 2 ulp each): the IEEE-rounded forms cost ~25 more
      // instructions per element and made the Adam epilogue issue-bound (ncu: 520 instr/unit)
      const float denom = sqrt_approx(st.v[k] * inv_c2) + hp.eps;
      st.w[k] -= __fdividef(hp.lr * (st.m[k] * inv_c1), denom);
      g[k] = st.w[k];
    }
  }
  template <int E>
  __device__ __forceinline__ void apply(float* g, size_t elem, State<E>& st) const {
    const size_t li = elem - shard_begin;
    update<E>(g, st);
    stf<E>(master + li, st.w);
    stf<E>(m1 + li, st.m);
    stf<E>(m2 + li, st.v);
  }
};

// ---------------------------------------------------------------- phases
// shard of rank r in UNITS of E elements (host/device agree on groups of 8)
template <int E>
__device__ __forceinline__ void shard_units_of(size_t total_groups, int world, int r, size_t* s0, size_t* s1) {
  size_t b, e;
  shard_units(total_groups, world, r, &b, &e);
  *s0 = b * (8 / E);
  *s1 = e * (8 / E);
}

// Visit the tiles of [s0,s1) that belong to this CTA; fn(first_unit_of_tile).
// Which CTA of how many this one is for the current piece of work.  Ordinary launches use
// (blockIdx.x, gridDim.x); the ring kernel rotates the assignment per descriptor and keeps its
// scheduler CTA out of the count.
struct CtaId {
  int cta, ncta;
  __device__ __forceinline__ CtaId() : cta(blockIdx.x), ncta(gridDim.x) {}
  __device__ __forceinline__ CtaId(int c, int n) : cta(c), ncta(n) {}
};

template <int UNROLL, class F>
__device__ __forceinline__ void for_owned_tiles(size_t s0, size_t s1, F&& fn, CtaId id = CtaId()) {
  const size_t tile = (size_t)blockDim.x * UNROLL;
  for (size_t t = s0 + (size_t)id.cta * tile; t < s1; t += (size_t)id.ncta * tile) fn(t);
}

template <class U, class W, int UNROLL>
__device__ __forceinline__ void pack_phase(const PeerView& pv, const SegDesc* segs, int nsegs, size_t stage_off,
                                           size_t total_groups) {
  constexpr int E = W::kPerVec;
  if (nsegs <= 0) return;
  SegCursor cur;
  bool inited = false;
  char* stage = pv.data[pv.rank] + stage_off;
  for (int r = 0; r < pv.world; ++r) {
    size_t s0, s1;
    shard_units_of<E>(total_groups, pv.world, r, &s0, &s1);
    for_owned_tiles<UNROLL>(s0, s1, [&](size_t t) {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
        if (unit < s1) {
          int64_t e = (int64_t)unit * E;
          if (!inited) {
            cur.init(segs, nsegs, e);
            inited = true;
          }
          float f[E];
          gather_elems<U, E>(cur, e, f);
          st_stream16(stage + unit * 16, W::pack(f));
        }
      }
    });
  }
}

template <class U, class W, int UNROLL>
__device__ __forceinline__ void unpack_phase(const PeerView& pv, const SegDesc* segs, int nsegs, size_t stage_off,
                                             size_t total_groups) {
  constexpr int E = W::kPerVec;
  if (nsegs <= 0) return;
  SegCursor cur;
  bool inited = false;
  const char* stage = pv.data[pv.rank] + stage_off;
  for (int r = 0; r < pv.world; ++r) {
    size_t s0, s1;
    shard_units_of<E>(total_groups, pv.world, r, &s0, &s1);
    for_owned_tiles<UNROLL>(s0, s1, [&](size_t t) {
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
        if (unit < s1) {
          int64_t e = (int64_t)unit * E;
          if (!inited) {
            cur.init(segs, nsegs, e);
            inited = true;
          }
          float f[E];
          W::unpack(ld_stream16(stage + unit * 16), f);
          scatter_elems<U, E>(cur, e, f);
        }
      }
    });
  }
}

// reduce the units of [s0,s1) owned by this CTA; epi.apply<E>(acc, elem); sink(acc, unit)
template <class W, int UNROLL, class Epi, class Sink>
__device__ __forceinline__ void reduce_phase(const PeerView& pv, size_t off, size_t s0, size_t s1, bool nvls, int rot,
                                             Epi& epi, Sink&& sink, CtaId id = CtaId()) {
  constexpr int E = W::kPerVec;
  for_owned_tiles<UNROLL>(s0, s1, [&](size_t t) {
    typename Epi::template State<E> est[UNROLL];
    if (nvls) {
      Vec16 v[UNROLL];
      bool valid[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
        valid[u] = unit < s1;
        if (valid[u]) {
          v[u] = W::mm_reduce(pv.mc_data + off + unit * 16);
          epi.template load<E>(est[u], unit * E);
        }
      }
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (valid[u]) {
          size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
          float acc[E];
          W::unpack(v[u], acc);
          epi.template apply<E>(acc, unit * E, est[u]);
          sink(acc, unit);
        }
      }
    } else {
      size_t idx[UNROLL];
      bool valid[UNROLL];
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        idx[u] = t + (size_t)u * blockDim.x + threadIdx.x;
        valid[u] = idx[u] < s1;
        if (valid[u]) epi.template load<E>(est[u], idx[u] * E);
      }
      float acc[UNROLL][E];
      reduce_units_p2p<W, UNROLL>(pv, off, idx, valid, rot, acc);
#pragma unroll
      for (int u = 0; u < UNROLL; ++u) {
        if (valid[u]) {
          epi.template apply<E>(acc[u], idx[u] * E, est[u]);
          sink(acc[u], idx[u]);
        }
      }
    }
  }, id);
}

// NVLS-only variant with its own unroll: one multimem.ld_reduce per unit keeps 4 registers in flight per
// unit (the P2P path needs 4 x peers), so many more units can be outstanding per thread - the in-switch
// reduction is latency bound per CTA (one tile per switch round trip), bytes in flight are what buys bandwidth.
template <class W, int UNROLL, class Epi, class Sink>
__device__ __forceinline__ void reduce_phase_nvls(const PeerView& pv, size_t off, size_t s0, size_t s1, Epi& epi,
                                                  Sink&& sink, CtaId id = CtaId()) {
  constexpr int E = W::kPerVec;
  for_owned_tiles<UNROLL>(s0, s1, [&](size_t t) {
    typename Epi::template State<E> est[UNROLL];
    Vec16 v[UNROLL];
    bool valid[UNROLL];
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      const size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
      valid[u] = unit < s1;
      if (valid[u]) {
        v[u] = W::mm_reduce(pv.mc_data + off + unit * 16);
        epi.template load<E>(est[u], unit * E);
      }
    }
#pragma unroll
    for (int u = 0; u < UNROLL; ++u) {
      if (valid[u]) {
        const size_t unit = t + (size_t)u * blockDim.x + threadIdx.x;
        float acc[E];
        W::unpack(v[u], acc);
        epi.template apply<E>(acc, unit * E, est[u]);
        sink(acc, unit);
      }
    }
  }, id);
}

__device__ __forceinline__ int rot_of(const PeerView& pv) { return pv.rank + 1 >= pv.world ? 0 : pv.rank + 1; }

}  // namespace

}  // namespace bps
