// Fused GPU gradient compression for the NVLink exchange (see compress_fused.cuh).
//
// Round 1 ran the compressors as ~10 separate element-wise passes (EF correct, norm finalize,
// pack, exchange, sum, recompress, unpack), read every peer's payload over NVLink element by
// element and selected top-k with one global atomic per kept element - slower than not compressing
// at all.  Here:
//
//   * ONE producer pass reads the gradient (+ momentum + error feedback), writes the corrected
//     value in place of the error state and emits the payload (sign words / first histogram) -
//     16-byte vector accesses throughout;
//   * payloads are PUSHED into every peer's window (one coalesced copy kernel that ends in the
//     flag barrier), so the consuming kernels read local memory only;
//   * norms / histogram picks are finished by the last block to leave (no extra launches), with a
//     fixed reduction order so every rank derives bit-identical scales;
//   * the consumer pass decompresses all payloads, applies the "server" stage (second error
//     feedback + recompression, server.cc:92-118 in the reference) and finishes the worker's own
//     error update in the same sweep.
//
// Reference semantics: /root/reference/byteps/common/compressor/impl/{onebit,topk,randomk}.cc,
// error_feedback.cc:22-43, momentum.cc:22-36.
#include "kernels/compress_fused.cuh"

#include "kernels/common.cuh"

namespace bps {

namespace {

constexpr int kT = 256;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// block-wide sum with a fixed shape; result valid in thread 0
__device__ __forceinline__ float block_sum(float v) {
  __shared__ float sh[kT / 32];
  v = warp_sum(v);
  const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  __syncthreads();   // sh may still be read from a previous call
  if (l == 0) sh[w] = v;
  __syncthreads();
  float r = 0.f;
  if (w == 0) {
    r = l < kT / 32 ? sh[l] : 0.f;
    r = warp_sum(r);
  }
  return r;
}

// fixed-order sum of `nparts` block partials by one block; result in thread 0
__device__ __forceinline__ float sum_partials(const float* parts, int nparts) {
  float a = 0.f;
  for (int b = threadIdx.x; b < nparts; b += kT) a += __ldcg(parts + b);
  return block_sum(a);
}

// ---- 4 elements at a time ------------------------------------------------------------------------
template <class U>
__device__ __forceinline__ void load4(const void* p, size_t i, size_t n, float* f) {
  if (i + 3 < n) {
    if constexpr (U::kBytes == 4) {
      const float4 v = *reinterpret_cast<const float4*>(reinterpret_cast<const float*>(p) + i);
      f[0] = v.x; f[1] = v.y; f[2] = v.z; f[3] = v.w;
    } else {
      const uint2 v = *reinterpret_cast<const uint2*>(reinterpret_cast<const char*>(p) + i * 2);
      float t[8];
      U::unpack(Vec16{v.x, v.y, 0u, 0u}, t);
      f[0] = t[0]; f[1] = t[1]; f[2] = t[2]; f[3] = t[3];
    }
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q) f[q] = i + q < n ? U::load1(p, i + q) : 0.f;
  }
}
template <class U>
__device__ __forceinline__ void store4(void* p, size_t i, size_t n, const float* f) {
  if (i + 3 < n) {
    if constexpr (U::kBytes == 4) {
      *reinterpret_cast<float4*>(reinterpret_cast<float*>(p) + i) = make_float4(f[0], f[1], f[2], f[3]);
    } else {
      const float t[8] = {f[0], f[1], f[2], f[3], 0.f, 0.f, 0.f, 0.f};
      const Vec16 v = U::pack(t);
      *reinterpret_cast<uint2*>(reinterpret_cast<char*>(p) + i * 2) = make_uint2(v.x, v.y);
    }
  } else {
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (i + q < n) U::store1(p, i + q, f[q]);
  }
}
__device__ __forceinline__ void loadf4(const float* p, size_t i, size_t n, float* f) { load4<TagF32>(p, i, n, f); }
__device__ __forceinline__ void storef4(float* p, size_t i, size_t n, const float* f) { store4<TagF32>(p, i, n, f); }

// corrected value of 4 elements: g (+ nesterov momentum) + ratio * err
template <class U>
__device__ __forceinline__ void corrected4(const void* g, float* mom, float mu, const float* err, float ratio, size_t i,
                                           size_t n, float* p) {
  load4<U>(g, i, n, p);
  if (mom) {
    float m[4];
    loadf4(mom, i, n, m);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      m[q] = mu * m[q] + p[q];
      p[q] += mu * m[q];
    }
    storef4(mom, i, n, m);
  }
  if (err) {
    float e[4];
    loadf4(err, i, n, e);
#pragma unroll
    for (int q = 0; q < 4; ++q) p[q] += ratio * e[q];
  }
}

// ================================================================================================ onebit
// Producer: one warp iteration covers 128 elements = 4 sign words = one 16-byte store.
template <class U>
__global__ void __launch_bounds__(kT) onebit_pre_kernel(const void* g, float* mom, float mu, const float* err,
                                                        float ratio, float* p_out, size_t n, uint32_t* words,
                                                        int use_scale, float* parts, uint32_t* counter) {
  const int lane = threadIdx.x & 31;
  const size_t nwords = (n + 31) / 32;
  const size_t nchunks = (n + 127) / 128;
  const size_t warps = ((size_t)gridDim.x * kT) >> 5;
  float s_abs = 0.f;
  for (size_t c = ((size_t)blockIdx.x * kT + threadIdx.x) >> 5; c < nchunks; c += warps) {
    const size_t i = c * 128 + (size_t)lane * 4;
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    if (i < n) {
      corrected4<U>(g, mom, mu, err, ratio, i, n, p);
      if (p_out) storef4(p_out, i, n, p);
    }
    uint32_t nib = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const bool live = i + q < n;
      if (live) s_abs += fabsf(p[q]);
      nib |= (live && p[q] < 0.f) ? (8u >> q) : 0u;          // first element -> most significant bit
    }
    uint32_t w = nib << (28 - 4 * (lane & 7));               // 8 lanes make one word, lane 0 of the group on top
    w |= __shfl_xor_sync(0xffffffffu, w, 1);
    w |= __shfl_xor_sync(0xffffffffu, w, 2);
    w |= __shfl_xor_sync(0xffffffffu, w, 4);
    const uint32_t w0 = __shfl_sync(0xffffffffu, w, 0), w1 = __shfl_sync(0xffffffffu, w, 8),
                   w2 = __shfl_sync(0xffffffffu, w, 16), w3 = __shfl_sync(0xffffffffu, w, 24);
    if (lane == 0) {
      const size_t wi = c * 4;
      if (wi + 3 < nwords) {
        *reinterpret_cast<uint4*>(words + wi) = make_uint4(w0, w1, w2, w3);
      } else {
        const uint32_t ws[4] = {w0, w1, w2, w3};
        for (int q = 0; q < 4; ++q)
          if (wi + q < nwords) words[wi + q] = ws[q];
      }
    }
  }
  const float b = block_sum(s_abs);
  if (threadIdx.x == 0) parts[blockIdx.x] = b;
  if (last_block(counter)) {
    const float tot = sum_partials(parts, gridDim.x);
    if (threadIdx.x == 0) reinterpret_cast<float*>(words + nwords)[0] = use_scale ? tot / (float)n : 1.0f;
  }
}

// Consumer, pass A: sum of all decompressed payloads (local slots), server-stage correction,
// worker error update.  slots: `world` windows of `slot_bytes` each.
//   c2 = sum_p (+-scale_p) [+ err2]  -> c2_out (two-stage)      | out = mult * sum (one-stage)
//   err = p - sign(p) * scale_me                                    (p is what the producer left in err)
template <class U>
__global__ void __launch_bounds__(kT) onebit_sum_kernel(const char* slots, size_t slot_bytes, int world, int me,
                                                        size_t n, float* err, const float* err2, float* c2_out,
                                                        void* out, float mult, int use_scale2, float* parts,
                                                        uint32_t* counter, float* scale2_out) {
  __shared__ float s_scale[kMaxRanks];
  const size_t nwords = (n + 31) / 32;
  if (threadIdx.x < world)
    s_scale[threadIdx.x] =
        reinterpret_cast<const float*>(slots + (size_t)threadIdx.x * slot_bytes + nwords * 4)[0];
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const size_t nchunks = (n + 127) / 128;
  const size_t warps = ((size_t)gridDim.x * kT) >> 5;
  const float my_scale = s_scale[me];
  float s_abs = 0.f;
  for (size_t c = ((size_t)blockIdx.x * kT + threadIdx.x) >> 5; c < nchunks; c += warps) {
    const size_t i = c * 128 + (size_t)lane * 4;
    if (i >= n) continue;
    const size_t wi = c * 4 + (lane >> 3);
    const int sh = 28 - 4 * (lane & 7);
    float s[4] = {0.f, 0.f, 0.f, 0.f};
    for (int p = 0; p < world; ++p) {
      const uint32_t word = __ldg(reinterpret_cast<const uint32_t*>(slots + (size_t)p * slot_bytes) + wi);
      const uint32_t nib = (word >> sh) & 0xfu;
      const float sc = s_scale[p];
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q] += (nib & (8u >> q)) ? -sc : sc;
    }
    if (err) {   // finish the worker's error feedback: e = p - D(C(p))
      float e[4];
      loadf4(err, i, n, e);
#pragma unroll
      for (int q = 0; q < 4; ++q) e[q] -= (e[q] < 0.f) ? -my_scale : my_scale;
      storef4(err, i, n, e);
    }
    if (c2_out) {
      if (err2) {
        float e2[4];
        loadf4(err2, i, n, e2);
#pragma unroll
        for (int q = 0; q < 4; ++q) s[q] += e2[q];
      }
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (i + q < n) s_abs += fabsf(s[q]);
      storef4(c2_out, i, n, s);
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) s[q] *= mult;
      store4<U>(out, i, n, s);
    }
  }
  if (c2_out) {
    const float b = block_sum(s_abs);
    if (threadIdx.x == 0) parts[blockIdx.x] = b;
    if (last_block(counter)) {
      const float tot = sum_partials(parts, gridDim.x);
      if (threadIdx.x == 0) scale2_out[0] = use_scale2 ? tot / (float)n : 1.0f;
    }
  }
}

// Consumer, pass B (two-stage): out = mult * sign(c2) * scale2 ; err2 = c2 - sign(c2) * scale2
template <class U>
__global__ void __launch_bounds__(kT) onebit_out_kernel(const float* c2, size_t n, const float* scale2_p, float* err2,
                                                        void* out, float mult) {
  const float sc = scale2_p[0];
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    const size_t i = v * 4;
    float c[4], o[4];
    loadf4(c2, i, n, c);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float d = c[q] < 0.f ? -sc : sc;
      o[q] = d * mult;
      c[q] -= d;
    }
    store4<U>(out, i, n, o);
    if (err2) storef4(err2, i, n, c);
  }
}

// ================================================================================================ payload push
// Copy my payload (local slot `me`) into slot `me` of every peer's window, then flag-barrier: when
// the kernel has finished on a rank, every peer's payload has landed in that rank's memory.
__global__ void __launch_bounds__(kT) payload_push_kernel(PeerView pv, size_t win_off, size_t slot_bytes, size_t bytes,
                                                          int channel) {
  const size_t nvec = (bytes + 15) / 16;
  const size_t off = win_off + (size_t)pv.rank * slot_bytes;
  const char* src = pv.data[pv.rank] + off;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < nvec; v += (size_t)gridDim.x * kT) {
    const Vec16 x = ld_stream16(src + v * 16);
    for (int j = 1; j < pv.world; ++j) {
      int p = pv.rank + j;
      if (p >= pv.world) p -= pv.world;
      st_peer16(pv.data[p] + off + v * 16, x);
    }
  }
  barrier_peers(pv, channel);
}

// ================================================================================================ top-k
// Exact selection of the k largest |x| by a 12 + 12 + 7 bit radix select over the fp32 magnitude
// bits.  Histograms are built per block in shared memory and merged with one global atomic per
// non-empty bin; the last block to leave picks the bin that contains the k-th largest key.
constexpr int kTopkBins = 4096;
struct TopkScratch {
  uint32_t hist[kTopkBins];
  uint32_t counter;
  uint32_t prefix;   // key bits decided so far
  uint32_t mask;
  uint32_t k_rem;    // how many still to take among keys that match the prefix
  uint32_t cnt_gt;
  uint32_t cnt_eq;
  uint32_t k;
  uint32_t t_lo;     // keys <= t_lo are not histogrammed at level 0 (sampled lower bound of the k-th largest key)
  uint32_t failed;   // the filtered level-0 histogram held fewer than k keys: redo it unfiltered
  uint32_t n_tie;    // keys equal to the k-th largest key
  uint32_t thr;      // the k-th largest key, once the three key levels are done
  uint32_t k_eq;     // how many of the n_tie ties are kept: the lowest indices (prefix then holds the index cut)
  uint32_t pad[4];
  uint32_t sample[32768];   // |x| keys of the strided sample (topk_sample_*)
};
static_assert(sizeof(TopkScratch) == kTopkScratchBytes, "TopkScratch layout");

__device__ __forceinline__ void topk_level(int level, int* shift, int* bins) {
  if (level == 0) { *shift = 19; *bins = 4096; }
  else if (level == 1) { *shift = 7; *bins = 4096; }
  else { *shift = 0; *bins = 128; }
}

// executed by every thread of ONE block once the global histogram of `level` is complete
__device__ void topk_pick(TopkScratch* sc, int level, bool last_key_level = false) {
  __shared__ uint32_t s_cnt[kT];
  __shared__ uint32_t s_found[3];
  int shift, bins;
  topk_level(level, &shift, &bins);
  const int per = bins / kT > 0 ? bins / kT : 1;          // bins per thread, from the top
  const int t = threadIdx.x;
  const int hi = bins - 1 - t * per;                       // my highest bin
  uint32_t local = 0;
  if (hi >= 0)
    for (int b = hi; b > hi - per && b >= 0; --b) local += __ldcg(&sc->hist[b]);
  s_cnt[t] = local;
  if (t == 0) s_found[0] = 0xffffffffu;
  __syncthreads();
  if (t == 0) {
    // serial scan over 256 thread totals, then inside the thread's bins: ~300 steps, once per level
    const uint32_t k = sc->k_rem;
    uint32_t total = 0;
    for (int q = 0; q < kT; ++q) total += s_cnt[q];
    s_found[1] = total < k ? 1u : 0u;
  }
  __syncthreads();
  if (s_found[1]) {
    // only possible at level 0 with the sampled filter on: too few keys above the guess
    if (t == 0) sc->failed = 1;
    for (int b = t; b < bins; b += kT) sc->hist[b] = 0;
    __threadfence();
    return;
  }
  if (t == 0) {
    sc->failed = 0;
    const uint32_t k = sc->k_rem;
    uint32_t cum = 0;
    int tt = 0;
    for (; tt < kT - 1; ++tt) {
      if (cum + s_cnt[tt] >= k) break;
      cum += s_cnt[tt];
    }
    int b = bins - 1 - tt * per;
    const int lo = b - per + 1 > 0 ? b - per + 1 : 0;
    for (; b > lo; --b) {
      const uint32_t h = __ldcg(&sc->hist[b]);
      if (cum + h >= k) break;
      cum += h;
    }
    sc->prefix |= (uint32_t)b << shift;
    sc->mask |= (uint32_t)(bins - 1) << shift;
    sc->k_rem = k - cum;
    if (last_key_level) sc->n_tie = __ldcg(&sc->hist[b]);
  }
  __syncthreads();
  for (int b = t; b < bins; b += kT) sc->hist[b] = 0;
  __threadfence();
}

__device__ __forceinline__ void hist_flush(uint32_t* sh_hist, TopkScratch* sc, int bins) {
  __syncthreads();
  for (int b = threadIdx.x; b < bins; b += kT) {
    const uint32_t h = sh_hist[b];
    if (h) atomicAdd(&sc->hist[b], h);
  }
}

// Producer: corrected value -> p_out, first-level histogram, pick by the last block.
template <class U>
__global__ void __launch_bounds__(kT) topk_pre_kernel(const void* g, float* mom, float mu, const float* err,
                                                      float ratio, float* p_out, size_t n, TopkScratch* sc) {
  __shared__ uint32_t sh_hist[kTopkBins];
  for (int b = threadIdx.x; b < kTopkBins; b += kT) sh_hist[b] = 0;
  __syncthreads();
  const uint32_t t_lo = sc->t_lo;
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    const size_t i = v * 4;
    float p[4];
    corrected4<U>(g, mom, mu, err, ratio, i, n, p);
    storef4(p_out, i, n, p);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t key = __float_as_uint(p[q]) & 0x7fffffffu;
      if (i + q < n && key >= t_lo) atomicAdd(&sh_hist[key >> 19], 1u);
    }
  }
  hist_flush(sh_hist, sc, kTopkBins);
  if (last_block(&sc->counter)) topk_pick(sc, 0);
}

// Histogram of `level` over the keys that match the prefix decided so far (fp32 input).
// mode 0: plain; mode 1: level 0 with the sampled filter (keys < t_lo skipped); mode 2: level-0 redo
// without the filter, a no-op unless the filtered attempt failed
__global__ void __launch_bounds__(kT) topk_hist_kernel(const float* x, size_t n, int level, int mode, TopkScratch* sc) {
  __shared__ uint32_t sh_hist[kTopkBins];
  if (mode == 2 && !sc->failed) return;
  const uint32_t t_lo = mode == 1 ? sc->t_lo : 0u;
  int shift, bins;
  topk_level(level, &shift, &bins);
  for (int b = threadIdx.x; b < bins; b += kT) sh_hist[b] = 0;
  __syncthreads();
  const uint32_t prefix = sc->prefix, mask = sc->mask;
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    const size_t i = v * 4;
    float p[4];
    loadf4(x, i, n, p);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t key = __float_as_uint(p[q]) & 0x7fffffffu;
      if (i + q < n && (key & mask) == prefix && key >= t_lo)
        atomicAdd(&sh_hist[(key >> shift) & (uint32_t)(bins - 1)], 1u);
    }
  }
  hist_flush(sh_hist, sc, bins);
  if (last_block(&sc->counter)) topk_pick(sc, level, level == 2);
}

// Ties at the threshold are broken by index, lowest first, so that every rank that selects from the same tensor
// keeps the same entries: three more radix levels over the key (2^31 - 1 - i) of the tied elements pick the
// index cut.  A no-op when every tie is kept.
__device__ __forceinline__ uint32_t tie_key(size_t i) { return 0x7fffffffu - (uint32_t)i; }
__global__ void topk_tie_init_kernel(TopkScratch* sc) {
  sc->thr = sc->prefix;
  sc->k_eq = sc->k_rem;
  sc->prefix = 0;
  sc->mask = 0;
}
__global__ void __launch_bounds__(kT) topk_tie_hist_kernel(const float* x, size_t n, int level, TopkScratch* sc) {
  __shared__ uint32_t sh_hist[kTopkBins];
  if (sc->k_eq == sc->n_tie) return;
  int shift, bins;
  topk_level(level, &shift, &bins);
  for (int b = threadIdx.x; b < bins; b += kT) sh_hist[b] = 0;
  __syncthreads();
  const uint32_t thr = sc->thr, prefix = sc->prefix, mask = sc->mask;
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    const size_t i = v * 4;
    float p[4];
    loadf4(x, i, n, p);
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t key = __float_as_uint(p[q]) & 0x7fffffffu, tk = tie_key(i + q);
      if (i + q < n && key == thr && (tk & mask) == prefix)
        atomicAdd(&sh_hist[(tk >> shift) & (uint32_t)(bins - 1)], 1u);
    }
  }
  hist_flush(sh_hist, sc, bins);
  if (last_block(&sc->counter)) topk_pick(sc, level);
}

__global__ void topk_init_kernel(TopkScratch* sc, uint32_t k) {
  for (int b = threadIdx.x; b < kTopkBins; b += blockDim.x) sc->hist[b] = 0;
  if (threadIdx.x == 0) {
    sc->counter = 0;
    sc->prefix = 0;
    sc->mask = 0;
    sc->k_rem = k;
    sc->cnt_gt = 0;
    sc->cnt_eq = 0;
    sc->k = k;
    sc->t_lo = 0;
    sc->failed = 0;
  }
}

// Sampled lower bound of the k-th largest key: the 1% that matter are a tiny part of the 25 M shared-memory
// atomics a full first-level histogram costs, so the first level only counts keys above a guess taken from
// kSampleN strided samples (two radix levels on the sample; the guess aims at ~2x the wanted fraction plus
// four standard deviations, and the pick falls back to an unfiltered pass in the rare case it was too high).
constexpr int kSampleN = 32768;
constexpr int kSampleThreads = 1024;
// step 1 (many blocks): gather the sample keys - one scattered load per thread
template <class U>
__global__ void __launch_bounds__(kT) topk_sample_gather_kernel(const void* g, const float* mom, float mu,
                                                                const float* err, float ratio, size_t n,
                                                                TopkScratch* sc) {
  const size_t S = n < (size_t)kSampleN ? n : (size_t)kSampleN;
  const size_t stride = n / S;
  const size_t j = (size_t)blockIdx.x * kT + threadIdx.x;
  if (j >= S) return;
  const size_t i = j * stride;
  float v = U::load1(g, i);
  if (mom) v += mu * (mu * mom[i] + v);
  if (err) v += ratio * err[i];
  sc->sample[j] = __float_as_uint(v) & 0x7fffffffu;
}
// step 2 (one block): two radix levels over the 32 K sample keys
__global__ void __launch_bounds__(kSampleThreads) topk_sample_pick_kernel(size_t n, uint32_t k, TopkScratch* sc) {
  __shared__ uint32_t sh_hist[kTopkBins];
  __shared__ uint32_t s_pref, s_mask, s_rem;
  const size_t S = n < (size_t)kSampleN ? n : (size_t)kSampleN;
  const double q = (double)k / (double)n;
  // wanted rank inside the sample: 2q + 4 sigma, at least 8; no filter at all for large fractions
  const double want = 2.0 * q * (double)S + 4.0 * sqrt(q * (double)S) + 8.0;
  const bool use = q < 0.125 && want < 0.5 * (double)S;
  if (!use) {
    if (threadIdx.x == 0) sc->t_lo = 0;
    return;
  }
  if (threadIdx.x == 0) {
    s_pref = 0;
    s_mask = 0;
    s_rem = (uint32_t)want;
  }
  for (int level = 0; level < 2; ++level) {
    int shift, bins;
    topk_level(level, &shift, &bins);
    for (int b = threadIdx.x; b < bins; b += kSampleThreads) sh_hist[b] = 0;
    __syncthreads();
    const uint32_t prefix = s_pref, mask = s_mask;
    for (size_t j = threadIdx.x; j < S; j += kSampleThreads) {
      const uint32_t key = sc->sample[j];
      if ((key & mask) == prefix) atomicAdd(&sh_hist[(key >> shift) & (uint32_t)(bins - 1)], 1u);
    }
    __syncthreads();
    if (threadIdx.x < 32) {
      // warp-parallel suffix scan: lane l owns bins [hi - 128 l - 127, hi - 128 l] from the top
      const int lane = threadIdx.x;
      const int per = bins / 32;
      const int hi = bins - 1 - lane * per;
      uint32_t local = 0;
      for (int b = hi; b > hi - per; --b) local += sh_hist[b];
      uint32_t incl = local;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += up;
      }
      const uint32_t kk = s_rem;
      const uint32_t before = incl - local;
      const bool mine = before < kk && incl >= kk;
      const uint32_t who = __ballot_sync(0xffffffffu, mine);
      const int owner = who ? __ffs(who) - 1 : 31;
      if (lane == owner) {
        uint32_t cum = before;
        int b = hi;
        for (; b > hi - per + 1; --b) {
          if (cum + sh_hist[b] >= kk) break;
          cum += sh_hist[b];
        }
        s_pref |= (uint32_t)b << shift;
        s_mask |= (uint32_t)(bins - 1) << shift;
        s_rem = kk - cum;
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) sc->t_lo = s_pref;      // low 7 bits zero: a lower bound of the sampled quantile
}

// Compaction: keys above the threshold take the first k - k_eq payload slots, ties take the rest.
// Slots are handed out with ONE global atomic per block iteration (1024 elements): per-thread counts,
// warp scan, block scan - a per-warp atomic on one address was the whole cost of this pass
// (same-address atomics retire about one per clock).  x_zero: the kept entries of x are
// zeroed, which IS the error-feedback update (the rest of the corrected tensor is already in place).
__global__ void __launch_bounds__(kT) topk_compact_kernel(float* x, size_t n, uint32_t* pairs, int zero_kept,
                                                          TopkScratch* sc) {
  __shared__ uint32_t s_warp[kT / 32];
  __shared__ uint32_t s_base;
  const uint32_t thr = sc->thr, k_eq = sc->k_eq, k = sc->k;
  const uint32_t base_eq = k - k_eq;
  const bool all_ties = k_eq == sc->n_tie;
  const uint32_t cut = sc->prefix;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const size_t n4 = (n + 3) / 4;
  const size_t per_iter = (size_t)gridDim.x * kT;
  const size_t iters = (n4 + per_iter - 1) / per_iter;       // the same trip count for every thread (block syncs)
  for (size_t it = 0; it < iters; ++it) {
    const size_t v = it * per_iter + (size_t)blockIdx.x * kT + threadIdx.x;
    const size_t i = v * 4;
    float p[4] = {0.f, 0.f, 0.f, 0.f};
    if (v < n4) loadf4(x, i, n, p);
    uint32_t gt_mask = 0, eq_mask = 0;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t key = __float_as_uint(p[q]) & 0x7fffffffu;
      const bool live = v < n4 && i + q < n;
      if (live && key > thr) gt_mask |= 1u << q;
      if (live && key == thr && (all_ties || tie_key(i + q) >= cut)) eq_mask |= 1u << q;
    }
    // exclusive prefix of the per-thread counts inside the block
    const uint32_t cnt = (uint32_t)__popc(gt_mask);
    uint32_t incl = cnt;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t up = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += up;
    }
    if (lane == 31) s_warp[warp] = incl;
    __syncthreads();
    if (threadIdx.x == 0) {
      uint32_t tot = 0;
      for (int w = 0; w < kT / 32; ++w) {
        const uint32_t c = s_warp[w];
        s_warp[w] = tot;
        tot += c;
      }
      s_base = tot ? atomicAdd(&sc->cnt_gt, tot) : 0u;
    }
    __syncthreads();
    uint32_t slot = s_base + s_warp[warp] + incl - cnt;
    bool any = false;
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      bool take = false;
      uint32_t my = 0;
      if (gt_mask & (1u << q)) {
        my = slot++;
        take = my < base_eq;
      } else if ((eq_mask & (1u << q)) && k_eq) {
        const uint32_t e = atomicAdd(&sc->cnt_eq, 1u);        // exactly k_eq ties reach here
        if (e < k_eq) {
          my = base_eq + e;
          take = true;
        }
      }
      if (take) {
        *reinterpret_cast<uint2*>(pairs + 2 * (size_t)my) = make_uint2((uint32_t)(i + q), __float_as_uint(p[q]));
        p[q] = 0.f;
        any = true;
      }
    }
    if (zero_kept && any) storef4(x, i, n, p);
    __syncthreads();          // s_warp / s_base are reused by the next iteration
  }
}

// dst[idx] += val for the k pairs of ONE payload (indices are unique inside a payload, payloads are
// added one launch after the other in rank order: the sum is bit-identical on every rank)
__global__ void __launch_bounds__(kT) sparse_add_kernel(const uint32_t* pairs, uint32_t k, size_t n, float* dst) {
  for (uint32_t r = blockIdx.x * kT + threadIdx.x; r < k; r += gridDim.x * kT) {
    const uint2 pr = *reinterpret_cast<const uint2*>(pairs + 2 * (size_t)r);
    if (pr.x < n) dst[pr.x] += __uint_as_float(pr.y);
  }
}

template <class U>
__global__ void __launch_bounds__(kT) cast_scale_kernel(const float* in, size_t n, void* out, float mult) {
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    float p[4];
    loadf4(in, v * 4, n, p);
#pragma unroll
    for (int q = 0; q < 4; ++q) p[q] *= mult;
    store4<U>(out, v * 4, n, p);
  }
}

// out = 0 everywhere, then out[idx] = mult * val for the k pairs (two kernels, same stream)
template <class U>
__global__ void __launch_bounds__(kT) zero_kernel(void* out, size_t n) {
  const size_t n4 = (n + 3) / 4;
  const float z[4] = {0.f, 0.f, 0.f, 0.f};
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT)
    store4<U>(out, v * 4, n, z);
}
template <class U>
__global__ void __launch_bounds__(kT) scatter_kernel(const uint32_t* pairs, uint32_t k, size_t n, void* out, float mult) {
  for (uint32_t r = blockIdx.x * kT + threadIdx.x; r < k; r += gridDim.x * kT) {
    const uint2 pr = *reinterpret_cast<const uint2*>(pairs + 2 * (size_t)r);
    if (pr.x < n) U::store1(out, pr.x, mult * __uint_as_float(pr.y));
  }
}

// ================================================================================================ random-k
// xorshift128+ is sequential, but linear over GF(2): state_{i+J} = T^J state_i.  The host supplies
// T^(2^j) as 128x128 bit matrices (one row = 2 x uint64); every thread jumps to the start of its
// chunk of `per` draws with at most 32 matrix-vector products, then draws sequentially - the exact
// stream of the CPU compressor (csrc/compress/compressor.cc, reference utils.h:74-113) in parallel.
__device__ __forceinline__ void xs_mat_vec(const uint64_t* m, uint64_t a, uint64_t b, uint64_t* oa, uint64_t* ob) {
  uint64_t ra = 0, rb = 0;
  for (int r = 0; r < 128; ++r) {
    const uint64_t par = (uint64_t)((__popcll(m[2 * r] & a) + __popcll(m[2 * r + 1] & b)) & 1);
    if (r < 64) ra |= par << r;
    else rb |= par << (r - 64);
  }
  *oa = ra;
  *ob = rb;
}

// Every thread draws `per` consecutive values.  Its starting state is the base state advanced by
// (block * kT + t) * per draws: the block part is computed once by warp 0 (one matrix per set bit of the
// block offset, 128 rows spread over 32 lanes), the thread part by doubling in shared memory - thread t
// derives its state from thread t - 2^msb(t) with ONE matrix-vector product.  per must be a power of two.
__device__ __forceinline__ void xs_mat_vec_warp(const uint64_t* m, uint64_t a, uint64_t b, int lane, uint64_t* oa,
                                                uint64_t* ob) {
  uint32_t w[4];
#pragma unroll
  for (int part = 0; part < 4; ++part) {
    const int r = part * 32 + lane;
    const bool par = ((__popcll(m[2 * r] & a) + __popcll(m[2 * r + 1] & b)) & 1) != 0;
    w[part] = __ballot_sync(0xffffffffu, par);
  }
  *oa = (uint64_t)w[0] | ((uint64_t)w[1] << 32);
  *ob = (uint64_t)w[2] | ((uint64_t)w[3] << 32);
}

__global__ void __launch_bounds__(kT) randomk_draw_kernel(uint64_t* state, const uint64_t* jump, uint32_t k, uint64_t n,
                                                          uint32_t per, int log2_per, uint32_t* idx) {
  __shared__ uint64_t s_a[kT], s_b[kT];
  const int t = threadIdx.x, lane = t & 31;
  if (t < 32) {
    uint64_t a = state[0], b = state[1];
    uint64_t adv = (uint64_t)blockIdx.x * kT * per;
    for (int j = 0; adv; ++j, adv >>= 1)
      if (adv & 1) xs_mat_vec_warp(jump + (size_t)j * 256, a, b, lane, &a, &b);
    if (t == 0) {
      s_a[0] = a;
      s_b[0] = b;
    }
  }
  __syncthreads();
  for (int level = 0; level < 8; ++level) {          // kT = 256 = 2^8
    const int lo = 1 << level;
    if (t >= lo && t < 2 * lo) {
      // T^(per * 2^level) = jump matrix number log2_per + level
      uint64_t a, b;
      xs_mat_vec(jump + (size_t)(log2_per + level) * 256, s_a[t - lo], s_b[t - lo], &a, &b);
      s_a[t] = a;
      s_b[t] = b;
    }
    __syncthreads();
  }
  const uint64_t first = ((uint64_t)blockIdx.x * kT + t) * per;
  if (first < k) {
    uint64_t a = s_a[t], b = s_b[t];
    const uint64_t end = first + per < k ? first + per : k;
    for (uint64_t i = first; i < end; ++i) {
      uint64_t x = a;
      const uint64_t s = b;
      a = s;
      x ^= x << 23;
      x ^= x >> 17;
      x ^= s ^ (s >> 26);
      b = x;
      idx[i] = (uint32_t)((x + s) % n);
    }
  }
}
// advance the stored state by k draws: 128 threads, one output bit each per matrix (k < 2^32)
__global__ void __launch_bounds__(128) randomk_advance_kernel(uint64_t* state, const uint64_t* jump, uint32_t k) {
  __shared__ uint32_t s_bits[4];
  uint64_t a = state[0], b = state[1];
  const int r = threadIdx.x;
  uint64_t adv = k;
  for (int j = 0; adv; ++j, adv >>= 1) {
    if (!(adv & 1)) continue;
    const uint64_t* m = jump + (size_t)j * 256;
    const bool par = ((__popcll(m[2 * r] & a) + __popcll(m[2 * r + 1] & b)) & 1) != 0;
    const uint32_t bits = __ballot_sync(0xffffffffu, par);
    __syncthreads();
    if ((r & 31) == 0) s_bits[r >> 5] = bits;
    __syncthreads();
    a = (uint64_t)s_bits[0] | ((uint64_t)s_bits[1] << 32);
    b = (uint64_t)s_bits[2] | ((uint64_t)s_bits[3] << 32);
  }
  if (r == 0) {
    state[0] = a;
    state[1] = b;
  }
}

// producer: corrected -> p_out (when error feedback is on), vals[j] = corrected[idx[j]]
template <class U>
__global__ void __launch_bounds__(kT) randomk_gather_kernel(const void* g, float* mom, float mu, const float* err,
                                                            float ratio, size_t n, const uint32_t* idx, uint32_t k,
                                                            float* vals) {
  for (uint32_t r = blockIdx.x * kT + threadIdx.x; r < k; r += gridDim.x * kT) {
    const uint32_t i = idx[r];
    float v = U::load1(g, i);
    if (mom) v += mu * (mu * mom[i] + v);
    if (err) v += ratio * err[i];
    vals[r] = v;
  }
}
// dense EF / momentum update for random-k: err = corrected everywhere (zeroing of the kept entries
// follows in zero_indexed), momentum advanced
template <class U>
__global__ void __launch_bounds__(kT) randomk_state_kernel(const void* g, float* mom, float mu, float* err, float ratio,
                                                           size_t n) {
  const size_t n4 = (n + 3) / 4;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n4; v += (size_t)gridDim.x * kT) {
    float p[4];
    corrected4<U>(g, mom, mu, err, ratio, v * 4, n, p);
    if (err) storef4(err, v * 4, n, p);
  }
}
__global__ void __launch_bounds__(kT) zero_indexed_kernel(const uint32_t* idx, uint32_t k, float* x) {
  for (uint32_t r = blockIdx.x * kT + threadIdx.x; r < k; r += gridDim.x * kT) x[idx[r]] = 0.f;
}
// vals_sum[j] = sum over the local slots, fixed order
__global__ void __launch_bounds__(kT) dense_sum_kernel(const char* slots, size_t slot_bytes, int world, uint32_t k,
                                                       float* out) {
  for (uint32_t r = blockIdx.x * kT + threadIdx.x; r < k; r += gridDim.x * kT) {
    float a = 0.f;
    for (int p = 0; p < world; ++p) a += reinterpret_cast<const float*>(slots + (size_t)p * slot_bytes)[r];
    out[r] = a;
  }
}

// ================================================================================================ dithering
// sum over the local slots of the dense int8 payloads ([n levels][float scale] each; compress.cu's format):
// 16 levels per thread per slot (one 16-byte load), fp32 sum, fixed peer order.
__device__ __forceinline__ float dither_value(int q, int s_levels, int partition) {
  if (partition == 0) return (float)q / (float)s_levels;
  return q == 0 ? 0.f : exp2f((float)(q - 1)) / exp2f((float)(s_levels - 1));
}
__global__ void __launch_bounds__(kT) dither_sum_slots_kernel(const char* slots, size_t slot_bytes, int world, size_t n,
                                                              int s_levels, int partition, float* sum) {
  __shared__ float s_scale[kMaxRanks];
  const size_t lv_bytes = (n + 15) / 16 * 16;
  if (threadIdx.x < world)
    s_scale[threadIdx.x] = reinterpret_cast<const float*>(slots + (size_t)threadIdx.x * slot_bytes + lv_bytes)[0];
  __syncthreads();
  const size_t n16 = (n + 15) / 16;
  for (size_t v = (size_t)blockIdx.x * kT + threadIdx.x; v < n16; v += (size_t)gridDim.x * kT) {
    float acc[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) acc[j] = 0.f;
    for (int p = 0; p < world; ++p) {
      const uint4 raw = __ldg(reinterpret_cast<const uint4*>(slots + (size_t)p * slot_bytes) + v);
      const uint32_t w[4] = {raw.x, raw.y, raw.z, raw.w};
      const float sc = s_scale[p];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        const int q = (int)(int8_t)((w[j >> 2] >> (8 * (j & 3))) & 0xffu);
        const float mag = dither_value(q < 0 ? -q : q, s_levels, partition) * sc;
        acc[j] += q < 0 ? -mag : mag;
      }
    }
    const size_t i = v * 16;
#pragma unroll
    for (int j = 0; j < 16; j += 4) storef4(sum, i + j, n, acc + j);
  }
}

inline int grid_for(size_t items, int cap = 132 * 8) {
  size_t b = (items + kT - 1) / kT;
  if (b < 1) b = 1;
  if (b > (size_t)cap) b = cap;
  return (int)b;
}

#define DISPATCH_U(dtype, STMT)                    \
  switch (dtype) {                                 \
    case 0: { using U = TagF32; STMT; } break;     \
    case 1: { using U = TagBF16; STMT; } break;    \
    case 2: { using U = TagF16; STMT; } break;     \
    default: return cudaErrorInvalidValue;         \
  }

}  // namespace

// ------------------------------------------------------------------------------------------------ host API
cudaError_t launch_onebit_pre(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                              float* p_out, size_t n, uint32_t* words, int use_scale, float* parts, uint32_t* counter,
                              cudaStream_t s) {
  const int grid = grid_for((n + 127) / 128 * 32, kFusedMaxBlocks);
  DISPATCH_U(dtype, (onebit_pre_kernel<U><<<grid, kT, 0, s>>>(g, mom, mu, err, ratio, p_out, n, words, use_scale,
                                                                parts, counter)));
  return cudaGetLastError();
}

cudaError_t launch_onebit_sum(const void* slots, size_t slot_bytes, int world, int me, size_t n, float* err,
                              const float* err2, float* c2_out, void* out, int dtype, float mult, int use_scale2,
                              float* parts, uint32_t* counter, float* scale2_out, cudaStream_t s) {
  if (world < 1 || world > kMaxRanks) return cudaErrorInvalidValue;
  const int grid = grid_for((n + 127) / 128 * 32, kFusedMaxBlocks);
  DISPATCH_U(dtype, (onebit_sum_kernel<U><<<grid, kT, 0, s>>>((const char*)slots, slot_bytes, world, me, n, err, err2,
                                                                c2_out, out, mult, use_scale2, parts, counter,
                                                                scale2_out)));
  return cudaGetLastError();
}

cudaError_t launch_onebit_out(const float* c2, size_t n, const float* scale2, float* err2, void* out, int dtype,
                              float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (onebit_out_kernel<U><<<grid_for((n + 3) / 4), kT, 0, s>>>(c2, n, scale2, err2, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_payload_push(const PeerView& pv, size_t win_off, size_t slot_bytes, size_t bytes, int blocks,
                                int channel, cudaStream_t s) {
  if (blocks < 1 || blocks > kMaxBlocks || (win_off & 15) || (slot_bytes & 15)) return cudaErrorInvalidValue;
  payload_push_kernel<<<blocks, kT, 0, s>>>(pv, win_off, slot_bytes, bytes, channel);
  return cudaGetLastError();
}

cudaError_t launch_topk_pre(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                            float* p_out, size_t n, uint32_t k, void* scratch, cudaStream_t s) {
  if (k == 0 || k > n || !p_out) return cudaErrorInvalidValue;
  TopkScratch* sc = (TopkScratch*)scratch;
  topk_init_kernel<<<1, kT, 0, s>>>(sc, k);
  DISPATCH_U(dtype, (topk_sample_gather_kernel<U><<<kSampleN / kT, kT, 0, s>>>(g, mom, mu, err, ratio, n, sc)));
  topk_sample_pick_kernel<<<1, kSampleThreads, 0, s>>>(n, k, sc);
  DISPATCH_U(dtype, (topk_pre_kernel<U><<<grid_for((n + 3) / 4, kFusedMaxBlocks), kT, 0, s>>>(g, mom, mu, err, ratio,
                                                                                               p_out, n, sc)));
  // the sampled filter was too optimistic (rare): redo level 0 over the corrected tensor, unfiltered
  topk_hist_kernel<<<grid_for((n + 3) / 4, kFusedMaxBlocks), kT, 0, s>>>(p_out, n, 0, 2, sc);
  return cudaGetLastError();
}

cudaError_t launch_topk_finish(float* x, size_t n, uint32_t k, int first_level, uint32_t* pairs, int zero_kept,
                               void* scratch, cudaStream_t s) {
  if (k == 0 || k > n || n > 0x7fffffffu) return cudaErrorInvalidValue;
  TopkScratch* sc = (TopkScratch*)scratch;
  const int grid = grid_for((n + 3) / 4, kFusedMaxBlocks);
  if (first_level == 0) {
    topk_init_kernel<<<1, kT, 0, s>>>(sc, k);
    topk_sample_gather_kernel<TagF32><<<kSampleN / kT, kT, 0, s>>>(x, nullptr, 0.f, nullptr, 0.f, n, sc);
    topk_sample_pick_kernel<<<1, kSampleThreads, 0, s>>>(n, k, sc);
    topk_hist_kernel<<<grid, kT, 0, s>>>(x, n, 0, 1, sc);
    topk_hist_kernel<<<grid, kT, 0, s>>>(x, n, 0, 2, sc);
    first_level = 1;
  }
  for (int level = first_level; level < 3; ++level) topk_hist_kernel<<<grid, kT, 0, s>>>(x, n, level, 0, sc);
  topk_tie_init_kernel<<<1, 1, 0, s>>>(sc);
  for (int level = 0; level < 3; ++level) topk_tie_hist_kernel<<<grid, kT, 0, s>>>(x, n, level, sc);
  topk_compact_kernel<<<grid, kT, 0, s>>>(x, n, pairs, zero_kept, sc);
  return cudaGetLastError();
}

cudaError_t launch_sparse_add_pairs(const uint32_t* pairs, uint32_t k, size_t n, float* dst, cudaStream_t s) {
  sparse_add_kernel<<<grid_for(k), kT, 0, s>>>(pairs, k, n, dst);
  return cudaGetLastError();
}

cudaError_t launch_scatter_pairs(const uint32_t* pairs, uint32_t k, size_t n, void* out, int dtype, float mult,
                                 cudaStream_t s) {
  DISPATCH_U(dtype, (zero_kernel<U><<<grid_for((n + 3) / 4), kT, 0, s>>>(out, n)));
  DISPATCH_U(dtype, (scatter_kernel<U><<<grid_for(k), kT, 0, s>>>(pairs, k, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_cast_scale4(const float* in, size_t n, void* out, int dtype, float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (cast_scale_kernel<U><<<grid_for((n + 3) / 4), kT, 0, s>>>(in, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_randomk_draw(uint64_t* state, const uint64_t* jump, uint32_t k, size_t n, uint32_t* idx,
                                cudaStream_t s) {
  if (k == 0 || n == 0) return cudaErrorInvalidValue;
  const uint32_t per = 16;                  // 2^4 draws per thread
  const uint32_t threads = (k + per - 1) / per;
  randomk_draw_kernel<<<(threads + kT - 1) / kT, kT, 0, s>>>(state, jump, k, (uint64_t)n, per, 4, idx);
  randomk_advance_kernel<<<1, 128, 0, s>>>(state, jump, k);
  return cudaGetLastError();
}

cudaError_t launch_randomk_pre(const void* g, int dtype, float* mom, float mu, float* err, float ratio, size_t n,
                               const uint32_t* idx, uint32_t k, float* vals, cudaStream_t s) {
  DISPATCH_U(dtype, (randomk_gather_kernel<U><<<grid_for(k), kT, 0, s>>>(g, mom, mu, err, ratio, n, idx, k, vals)));
  if (err || mom) {
    DISPATCH_U(dtype, (randomk_state_kernel<U><<<grid_for((n + 3) / 4), kT, 0, s>>>(g, mom, mu, err, ratio, n)));
  }
  if (err) zero_indexed_kernel<<<grid_for(k), kT, 0, s>>>(idx, k, err);
  return cudaGetLastError();
}

cudaError_t launch_dither_sum_slots(const void* slots, size_t slot_bytes, int world, size_t n, int s_levels,
                                    int partition, float* sum, cudaStream_t s) {
  if (world < 1 || world > kMaxRanks) return cudaErrorInvalidValue;
  dither_sum_slots_kernel<<<grid_for((n + 15) / 16), kT, 0, s>>>((const char*)slots, slot_bytes, world, n, s_levels,
                                                                  partition, sum);
  return cudaGetLastError();
}

cudaError_t launch_dense_sum_slots(const void* slots, size_t slot_bytes, int world, uint32_t k, float* out,
                                   cudaStream_t s) {
  dense_sum_kernel<<<grid_for(k), kT, 0, s>>>((const char*)slots, slot_bytes, world, k, out);
  return cudaGetLastError();
}

}  // namespace bps
