// Device-side helpers shared by the sm_90a kernels: 128-bit peer loads/stores,
// bf16/fp16 packing, system-scope flag barriers over NVLink peer memory and the
// NVLS multimem wrappers.
#pragma once
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "kernels/peer_view.h"

namespace bps {

struct alignas(16) Vec16 {
  uint32_t x, y, z, w;
};

// ---- global loads/stores ----------------------------------------------------
// Peer (NVLink) reads bypass the local L2 and may only be cached in L1; every
// element is read once, so do not allocate in L1.
__device__ __forceinline__ Vec16 ld_peer16(const void* p) {
  Vec16 v;
  asm volatile("ld.global.relaxed.sys.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_peer16(void* p, const Vec16& v) {
  asm volatile("st.global.relaxed.sys.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ Vec16 ld_stream16(const void* p) {
  Vec16 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_stream16(void* p, const Vec16& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ---- NVLS (multimem) --------------------------------------------------------
// One instruction reduces the same address across every GPU bound to the
// multicast object inside the NVSwitch; one store is replicated to all of them.
__device__ __forceinline__ Vec16 mm_ld_reduce_bf16x8(const void* mc) {
  Vec16 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ Vec16 mm_ld_reduce_f16x8(const void* mc) {
  Vec16 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ Vec16 mm_ld_reduce_f32x4(const void* mc) {
  Vec16 v;
  asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(mc)
               : "memory");
  return v;
}
__device__ __forceinline__ void mm_st16(void* mc, const Vec16& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x), "r"(v.y), "r"(v.z),
               "r"(v.w)
               : "memory");
}

// ---- flags ------------------------------------------------------------------
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }

constexpr long long kBarrierSpinLimit = 60000000000ll;   // ~30 s of SM clocks (default when nothing is configured)
constexpr long long kSpinCheckEvery = 1 << 22;           // clocks between looks at the configured limit

// Watchdog shared by every spin on a peer: after `kSpinCheckEvery` clocks it reads the configured
// limit (BYTEPS_SPIN_TIMEOUT_MS -> RingState::spin_limit) and reports whether it was exceeded.
struct SpinWatch {
  long long t0, limit;
  __device__ __forceinline__ SpinWatch() { reset(); }
  __device__ __forceinline__ void reset() {
    t0 = clock64();
    limit = kSpinCheckEvery;
  }
  __device__ __forceinline__ bool expired(const PeerView& pv) {
    const long long dt = clock64() - t0;
    if (dt <= limit) return false;
    if (limit == kSpinCheckEvery) {      // first slow-path visit: fetch the real limit
      const unsigned long long cfg = *(volatile unsigned long long*)&ring_state_of(pv.epoch)->spin_limit;
      limit = cfg ? (long long)cfg : kBarrierSpinLimit;
      return dt > limit;
    }
    return true;
  }
};

// Cross-rank barrier between the CTAs with the same blockIdx on every rank.
// Slots are single-writer, generations increase monotonically, so no reset is
// ever needed and the state survives CUDA-graph replays (it lives in device
// memory, not in kernel arguments).  Every thread's earlier peer stores are
// ordered before the flag by bar.sync + a system-scope fence in the signalling
// thread; the waiter's acquire + bar.sync orders its later loads after it.
__device__ __forceinline__ void barrier_peers(const PeerView& pv, int channel) {
  __syncthreads();
  // channel < 0: profiling only - one rank runs alone under ncu (which replays the kernel dozens of times
  // while the peers sit idle), so there is nobody to meet; the data path through the switch is unchanged
  if (channel < 0) return;
  const int slot_base = (channel * kMaxBlocks + blockIdx.x);
  if (threadIdx.x < pv.world) {
    const uint32_t target = pv.epoch[slot_base] + 1;
    const int peer = threadIdx.x;
    fence_sys();
    st_release_sys(pv.sig[peer] + slot_base * kMaxRanks + pv.rank, target);
    const uint32_t* mine = pv.sig[pv.rank] + slot_base * kMaxRanks + peer;
    // watchdog: a peer that never arrives (crashed rank, mismatched launch order)
    // turns into a trapped kernel + CUDA error instead of a GPU hung forever
    SpinWatch watch;
    while ((int32_t)(ld_acquire_sys(mine) - target) < 0) {
      if (watch.expired(pv)) {
        printf("byteps_b200: rank %d block %d timed out waiting for peer %d (generation %u)\n", pv.rank,
               (int)blockIdx.x, peer, target);
        __trap();
      }
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) pv.epoch[slot_base] += 1;
}

// "Last block out" pattern: returns true (for the whole block) in the block that arrives last among the `arrivals`
// blocks counting on `counter` (every block of the grid by default), after every earlier block's global writes are
// visible.  The counter is reset to 0 by that block, so it is ready for the next launch on the same stream.
__device__ __forceinline__ bool last_block(uint32_t* counter, uint32_t arrivals) {
  __shared__ uint32_t s_last;
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    const uint32_t prev = atomicAdd(counter, 1u);
    s_last = prev == arrivals - 1 ? 1u : 0u;
    if (s_last) *counter = 0;
    __threadfence();
  }
  __syncthreads();
  return s_last != 0;
}
__device__ __forceinline__ bool last_block(uint32_t* counter) { return last_block(counter, gridDim.x); }

// ---- numeric packing ----------------------------------------------------------
__device__ __forceinline__ float2 bf16x2_to_f2(uint32_t u) {
  return make_float2(__uint_as_float(u << 16), __uint_as_float(u & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(float a, float b) {
  __nv_bfloat162 h = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}
__device__ __forceinline__ float2 f16x2_to_f2(uint32_t u) {
  __half2 h = *reinterpret_cast<__half2*>(&u);
  return __half22float2(h);
}
__device__ __forceinline__ uint32_t f2_to_f16x2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

// Element traits: T = storage type tag, kPerVec = elements per 16-byte vector.
struct TagF32 {
  using type = float;
  static constexpr int kPerVec = 4;
  static constexpr int kBytes = 4;
  __device__ static void unpack(const Vec16& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y); f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  __device__ static Vec16 pack(const float* f) {
    return Vec16{__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3])};
  }
  __device__ static float load1(const void* p, size_t i) { return ((const float*)p)[i]; }
  __device__ static void store1(void* p, size_t i, float v) { ((float*)p)[i] = v; }
  __device__ static Vec16 mm_reduce(const void* mc) { return mm_ld_reduce_f32x4(mc); }
};
struct TagBF16 {
  using type = __nv_bfloat16;
  static constexpr int kPerVec = 8;
  static constexpr int kBytes = 2;
  __device__ static void unpack(const Vec16& v, float* f) {
    float2 a = bf16x2_to_f2(v.x), b = bf16x2_to_f2(v.y), c = bf16x2_to_f2(v.z), d = bf16x2_to_f2(v.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
  }
  __device__ static Vec16 pack(const float* f) {
    return Vec16{f2_to_bf16x2(f[0], f[1]), f2_to_bf16x2(f[2], f[3]), f2_to_bf16x2(f[4], f[5]), f2_to_bf16x2(f[6], f[7])};
  }
  __device__ static float load1(const void* p, size_t i) { return __bfloat162float(((const __nv_bfloat16*)p)[i]); }
  __device__ static void store1(void* p, size_t i, float v) { ((__nv_bfloat16*)p)[i] = __float2bfloat16_rn(v); }
  __device__ static Vec16 mm_reduce(const void* mc) { return mm_ld_reduce_bf16x8(mc); }
};
struct TagF16 {
  using type = __half;
  static constexpr int kPerVec = 8;
  static constexpr int kBytes = 2;
  __device__ static void unpack(const Vec16& v, float* f) {
    float2 a = f16x2_to_f2(v.x), b = f16x2_to_f2(v.y), c = f16x2_to_f2(v.z), d = f16x2_to_f2(v.w);
    f[0] = a.x; f[1] = a.y; f[2] = b.x; f[3] = b.y; f[4] = c.x; f[5] = c.y; f[6] = d.x; f[7] = d.y;
  }
  __device__ static Vec16 pack(const float* f) {
    return Vec16{f2_to_f16x2(f[0], f[1]), f2_to_f16x2(f[2], f[3]), f2_to_f16x2(f[4], f[5]), f2_to_f16x2(f[6], f[7])};
  }
  __device__ static float load1(const void* p, size_t i) { return __half2float(((const __half*)p)[i]); }
  __device__ static void store1(void* p, size_t i, float v) { ((__half*)p)[i] = __float2half_rn(v); }
  __device__ static Vec16 mm_reduce(const void* mc) { return mm_ld_reduce_f16x8(mc); }
};

// ---- dropout bits ---------------------------------------------------------------
// Philox4x32-10 with counter c and key k.  Dropout keeps element i when word i % 4 of the Philox block with counter
// (i / 4, offset) and key seed is below keep = (1 - p) * 2^32; the LayerNorm and attention kernels share the scheme.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int i = 0; i < 10; ++i) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c.x), lo0 = 0xD2511F53u * c.x;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c.z), lo1 = 0xCD9E8D57u * c.z;
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

// the 4 keep bits of Philox block (counter g, offset off): bit j for element 4g + j
__device__ __forceinline__ uint32_t keep_nibble(uint2 key, uint2 off, uint64_t g, uint32_t keep) {
  const uint4 r = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), off.x, off.y), key);
  return (uint32_t)(r.x < keep) | (uint32_t)(r.y < keep) << 1 | (uint32_t)(r.z < keep) << 2 |
         (uint32_t)(r.w < keep) << 3;
}

// keep bits of the 8 elements from element index e (a multiple of 4): bit k for element e + k
__device__ __forceinline__ uint32_t keep_bits(uint2 key, uint2 off, uint64_t e, uint32_t keep) {
  uint32_t bits = 0;
#pragma unroll
  for (int h = 0; h < 2; ++h) bits |= keep_nibble(key, off, (e >> 2) + h, keep) << (4 * h);
  return bits;
}

}  // namespace bps

// ---- mbarrier + bulk async copy (TMA, 1-D form: no tensor map needed) -------------------------
namespace bps {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "DONE:\n\t"
      "}" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// global (local or NVLink peer) -> shared, completion counted on an mbarrier
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// shared -> global (local or NVLink peer), tracked by bulk async-groups
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst), "r"(smem_u32(smem_src)),
               "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait() {
  asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar_sync(int id, int nthreads) {
  asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ void named_bar_arrive(int id, int nthreads) {
  asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}
__device__ __forceinline__ Vec16 lds16(const void* p) {
  Vec16 v;
  asm volatile("ld.shared.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(smem_u32(p)));
  return v;
}
__device__ __forceinline__ void sts16(void* p, const Vec16& v) {
  asm volatile("st.shared.v4.u32 [%0], {%1,%2,%3,%4};" ::"r"(smem_u32(p)), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

}  // namespace bps
