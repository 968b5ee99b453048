// Device-side gradient compressors (see compress.cuh).
#include "kernels/compress.cuh"

#include "kernels/common.cuh"

namespace bps {

namespace {

constexpr int kThreads = 256;

inline int grid_for(size_t n, int per_thread = 4, int cap = 132 * 8) {
  size_t b = (n + (size_t)kThreads * per_thread - 1) / ((size_t)kThreads * per_thread);
  if (b < 1) b = 1;
  if (b > (size_t)cap) b = cap;
  return (int)b;
}

template <class U>
__device__ __forceinline__ float load_as_float(const void* p, size_t i) {
  return U::load1(p, i);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---------------------------------------------------------------- error-feedback correction + norms
template <class U>
__global__ void ef_correct_kernel(const void* g, const float* err, float ratio, float* corrected, size_t n,
                                  float* acc) {
  float s_abs = 0.f, s_sq = 0.f, s_max = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = load_as_float<U>(g, i);
    if (err) v += ratio * err[i];
    corrected[i] = v;
    float a = fabsf(v);
    s_abs += a;
    s_sq += v * v;
    s_max = fmaxf(s_max, a);
  }
  __shared__ float sh[3][kThreads / 32];
  s_abs = warp_sum(s_abs);
  s_sq = warp_sum(s_sq);
  s_max = warp_max(s_max);
  int w = threadIdx.x >> 5, l = threadIdx.x & 31;
  if (l == 0) {
    sh[0][w] = s_abs;
    sh[1][w] = s_sq;
    sh[2][w] = s_max;
  }
  __syncthreads();
  if (w == 0) {
    float a = l < kThreads / 32 ? sh[0][l] : 0.f, q = l < kThreads / 32 ? sh[1][l] : 0.f,
          m = l < kThreads / 32 ? sh[2][l] : 0.f;
    a = warp_sum(a);
    q = warp_sum(q);
    m = warp_max(m);
    if (l == 0) {
      // per-block partials; a fixed-shape second pass makes the norms bit-reproducible
      // (every rank must derive the SAME scale from the same data)
      float* part = acc + 4 + 3 * blockIdx.x;
      part[0] = a;
      part[1] = q;
      part[2] = m;
    }
  }
}

__global__ void ef_finalize_kernel(float* acc, int nblocks) {
  __shared__ float sh[3][kThreads];
  float a = 0.f, q = 0.f, m = 0.f;
  for (int b = threadIdx.x; b < nblocks; b += kThreads) {   // fixed assignment, fixed order
    a += acc[4 + 3 * b];
    q += acc[4 + 3 * b + 1];
    m = fmaxf(m, acc[4 + 3 * b + 2]);
  }
  sh[0][threadIdx.x] = a;
  sh[1][threadIdx.x] = q;
  sh[2][threadIdx.x] = m;
  __syncthreads();
  for (int s = kThreads / 2; s > 0; s >>= 1) {
    if (threadIdx.x < s) {
      sh[0][threadIdx.x] += sh[0][threadIdx.x + s];
      sh[1][threadIdx.x] += sh[1][threadIdx.x + s];
      sh[2][threadIdx.x] = fmaxf(sh[2][threadIdx.x], sh[2][threadIdx.x + s]);
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    acc[0] = sh[0][0];
    acc[1] = sh[1][0];
    acc[2] = sh[2][0];
  }
}

// ---------------------------------------------------------------- onebit
__global__ void onebit_pack_kernel(const float* corrected, size_t n, const float* acc, int use_scale, uint32_t* words,
                                   float* err_out) {
  const size_t nwords = (n + 31) / 32;
  const float scale = use_scale ? acc[0] / (float)n : 1.0f;
  const int lane = threadIdx.x & 31;
  const size_t warps = ((size_t)gridDim.x * blockDim.x) >> 5;
  for (size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < nwords; w += warps) {
    size_t i = w * 32 + lane;
    float v = i < n ? corrected[i] : 0.f;
    bool neg = (i < n) && (v < 0.f);
    uint32_t bits = __brev(__ballot_sync(0xffffffffu, neg));   // lane 0 -> MSB
    if (lane == 0) words[w] = bits;
    if (err_out && i < n) err_out[i] = v - (neg ? -scale : scale);
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) reinterpret_cast<float*>(words + nwords)[0] = scale;
}

__global__ void onebit_exchange_sum_kernel(PeerView pv, size_t off, size_t n, float* sum, int channel) {
  barrier_peers(pv, channel);
  const size_t nwords = (n + 31) / 32;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int p = 0; p < pv.world; ++p) {
      const uint32_t* w = reinterpret_cast<const uint32_t*>(pv.data[p] + off);
      const float scale = reinterpret_cast<const float*>(w + nwords)[0];
      const uint32_t word = w[i >> 5];
      acc += ((word >> (31 - (i & 31))) & 1u) ? -scale : scale;
    }
    sum[i] = acc;
  }
  barrier_peers(pv, channel);
}

template <class U>
__global__ void onebit_unpack_kernel(const uint32_t* words, size_t n, void* out, float mult) {
  const size_t nwords = (n + 31) / 32;
  const float scale = reinterpret_cast<const float*>(words + nwords)[0] * mult;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t word = words[i >> 5];
    U::store1(out, i, ((word >> (31 - (i & 31))) & 1u) ? -scale : scale);
  }
}

// ---------------------------------------------------------------- top-k by radix select on |x| bits
// scratch layout (uint32): [0..255] histogram, [256] prefix, [257] mask, [258] k_remaining, [259] cnt_gt,
// [260] cnt_eq, [261] k
__global__ void topk_init_kernel(uint32_t* sc, uint32_t k) {
  int t = threadIdx.x;
  if (t < 256) sc[t] = 0;
  if (t == 0) {
    sc[256] = 0;
    sc[257] = 0;
    sc[258] = k;
    sc[259] = 0;
    sc[260] = 0;
    sc[261] = k;
  }
}

__global__ void topk_hist_kernel(const float* x, size_t n, int shift, uint32_t* sc) {
  __shared__ uint32_t h[256];
  for (int i = threadIdx.x; i < 256; i += blockDim.x) h[i] = 0;
  __syncthreads();
  const uint32_t prefix = sc[256], mask = sc[257];
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    uint32_t key = __float_as_uint(x[i]) & 0x7fffffffu;
    if ((key & mask) == prefix) atomicAdd(&h[(key >> shift) & 0xffu], 1u);
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x)
    if (h[i]) atomicAdd(&sc[i], h[i]);
}

__global__ void topk_pick_kernel(int shift, uint32_t* sc) {
  if (threadIdx.x == 0) {
    uint32_t k = sc[258], cum = 0;
    int d = 255;
    for (; d > 0; --d) {
      if (cum + sc[d] >= k) break;
      cum += sc[d];
    }
    sc[256] |= (uint32_t)d << shift;
    sc[257] |= 0xffu << shift;
    sc[258] = k - cum;   // how many to take among keys sharing the new prefix
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 256; i += blockDim.x) sc[i] = 0;
}

__global__ void topk_compact_kernel(const float* x, size_t n, uint32_t* pairs, float* err_out, uint32_t* sc) {
  const uint32_t thr = sc[256], k_eq = sc[258], k = sc[261];
  const uint32_t base_eq = k - k_eq;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = x[i];
    uint32_t key = __float_as_uint(v) & 0x7fffffffu;
    bool take = false;
    uint32_t slot = 0;
    if (key > thr) {
      slot = atomicAdd(&sc[259], 1u);
      take = slot < base_eq;
    } else if (key == thr) {
      uint32_t e = atomicAdd(&sc[260], 1u);
      if (e < k_eq) {
        slot = base_eq + e;
        take = true;
      }
    }
    if (take) {
      pairs[2 * slot] = (uint32_t)i;
      pairs[2 * slot + 1] = __float_as_uint(v);
    }
    if (err_out) err_out[i] = take ? 0.f : v;
  }
}

__global__ void sparse_exchange_sum_kernel(PeerView pv, size_t off, uint32_t k, size_t n, float* sum, int channel) {
  barrier_peers(pv, channel);
  const size_t total = (size_t)k * pv.world;
  for (size_t j = blockIdx.x * (size_t)blockDim.x + threadIdx.x; j < total; j += (size_t)gridDim.x * blockDim.x) {
    int p = (int)(j / k);
    uint32_t r = (uint32_t)(j % k);
    const uint32_t* pairs = reinterpret_cast<const uint32_t*>(pv.data[p] + off);
    uint32_t idx = pairs[2 * r];
    float val = __uint_as_float(pairs[2 * r + 1]);
    if (idx < n) atomicAdd(&sum[idx], val);
  }
  barrier_peers(pv, channel);
}

// deterministic alternative to the atomic version: one launch per peer, indices are unique within a payload
__global__ void sparse_add_kernel(const uint32_t* pairs, uint32_t k, size_t n, float* sum) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) {
    uint32_t idx = pairs[2 * r];
    if (idx < n) sum[idx] += __uint_as_float(pairs[2 * r + 1]);
  }
}

template <class U>
__global__ void zero_out_kernel(void* out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    U::store1(out, i, 0.f);
}

template <class U>
__global__ void sparse_scatter_kernel(const uint32_t* pairs, uint32_t k, size_t n, void* out, float mult) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) {
    uint32_t idx = pairs[2 * r];
    if (idx < n) U::store1(out, idx, mult * __uint_as_float(pairs[2 * r + 1]));
  }
}

// ---------------------------------------------------------------- random-k
__global__ void randomk_indices_kernel(uint64_t* state, uint32_t k, uint64_t n, uint32_t* idx) {
  if (blockIdx.x == 0 && threadIdx.x == 0) {
    uint64_t a = state[0], b = state[1];
    for (uint32_t i = 0; i < k; ++i) {   // xorshift128+, the CPU compressor's exact stream
      uint64_t t = a;
      const uint64_t s = b;
      a = s;
      t ^= t << 23;
      t ^= t >> 17;
      t ^= s ^ (s >> 26);
      b = t;
      idx[i] = (uint32_t)((t + s) % n);
    }
    state[0] = a;
    state[1] = b;
  }
}

__global__ void copy_kernel(const float* in, float* out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    out[i] = in[i];
}

__global__ void randomk_gather_kernel(const float* corrected, const uint32_t* idx, uint32_t k, float* vals,
                                      float* err_out) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) {
    vals[r] = corrected[idx[r]];
  }
}
__global__ void zero_indexed_kernel(const uint32_t* idx, uint32_t k, float* err) {
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) err[idx[r]] = 0.f;
}

__global__ void dense_exchange_sum_kernel(PeerView pv, size_t off, uint32_t k, float* out, int channel) {
  barrier_peers(pv, channel);
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int p = 0; p < pv.world; ++p) acc += reinterpret_cast<const float*>(pv.data[p] + off)[r];
    out[r] = acc;
  }
  barrier_peers(pv, channel);
}

template <class U>
__global__ void index_scatter_kernel(const uint32_t* idx, const float* vals, uint32_t k, size_t n, void* out,
                                     float mult) {
  // sequential semantics of the reference (later duplicates overwrite): resolve
  // duplicates deterministically by letting the LAST occurrence win.
  for (uint32_t r = blockIdx.x * blockDim.x + threadIdx.x; r < k; r += gridDim.x * blockDim.x) {
    uint32_t i = idx[r];
    bool last = true;
    for (uint32_t q = r + 1; q < k && q < r + 64; ++q) last &= (idx[q] != i);
    if (i < n && last) U::store1(out, i, mult * vals[r]);
  }
}

// ---------------------------------------------------------------- dithering
__device__ __forceinline__ float rng_uniform(uint64_t seed, uint64_t step, uint64_t i) {
  // splitmix64 over (seed, step, index): counter based, reproducible, parallel
  uint64_t z = seed * 0x9E3779B97F4A7C15ull + step * 0xBF58476D1CE4E5B9ull + i * 0x94D049BB133111EBull +
               0x2545F4914F6CDD1Dull;
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  return (float)(z >> 40) * (1.0f / 16777216.0f);
}

__device__ __forceinline__ float dither_level_value(int q, int s_levels, int partition) {
  // q is the (non-negative) level index carried on the wire
  if (partition == 0) return (float)q / (float)s_levels;
  return q == 0 ? 0.f : exp2f((float)(q - 1)) / exp2f((float)(s_levels - 1));
}

__global__ void dither_quantize_kernel(const float* x, size_t n, const float* acc, int s_levels, int partition,
                                       int normalize, uint64_t seed, uint64_t step, int8_t* levels, float* scale_out,
                                       float* err_out) {
  const float scale = normalize == 0 ? acc[2] : sqrtf(acc[1]);
  const float inv = scale > 0.f ? 1.0f / scale : 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = x[i];
    float a = fabsf(v) * inv;   // in [0,1]
    float u = rng_uniform(seed, step, i);
    int q;
    if (partition == 0) {
      float t = a * s_levels;
      float fl = floorf(t);
      q = (int)fl + (u < (t - fl) ? 1 : 0);
      if (q > s_levels) q = s_levels;
    } else {
      // levels 0, 2^-(s-1), ..., 1/2, 1 -> index 0..s
      float t = a * exp2f((float)(s_levels - 1));          // in [0, 2^(s-1)]
      if (t <= 0.f) {
        q = 0;
      } else {
        float lo_idx = floorf(log2f(fmaxf(t, 1e-30f)));     // 2^lo <= t
        if (t < 1.f) {                                       // between 0 and the smallest level
          q = u < t ? 1 : 0;
        } else {
          float lo = exp2f(lo_idx), hi = lo * 2.f;
          int qi = (int)lo_idx + 1;
          q = qi + ((u < (t - lo) / (hi - lo)) ? 1 : 0);
          if (q > s_levels) q = s_levels;
        }
      }
    }
    int8_t sq = (int8_t)(v < 0.f ? -q : q);
    levels[i] = sq;
    if (err_out) err_out[i] = v - (v < 0.f ? -1.f : 1.f) * dither_level_value(q, s_levels, partition) * scale;
  }
  if (blockIdx.x == 0 && threadIdx.x == 0) scale_out[0] = scale;
}

__global__ void dither_exchange_sum_kernel(PeerView pv, size_t off, size_t n, int s_levels, int partition,
                                           float* sum, int channel) {
  barrier_peers(pv, channel);
  const size_t lv_bytes = (n + 15) / 16 * 16;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float acc = 0.f;
    for (int p = 0; p < pv.world; ++p) {
      const int8_t* lv = reinterpret_cast<const int8_t*>(pv.data[p] + off);
      const float scale = reinterpret_cast<const float*>(pv.data[p] + off + lv_bytes)[0];
      int q = lv[i];
      float mag = dither_level_value(q < 0 ? -q : q, s_levels, partition) * scale;
      acc += q < 0 ? -mag : mag;
    }
    sum[i] = acc;
  }
  barrier_peers(pv, channel);
}

template <class U>
__global__ void dither_unpack_kernel(const int8_t* levels, const float* scale_p, size_t n, int s_levels,
                                     int partition, void* out, float mult) {
  const float scale = scale_p[0] * mult;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    int q = levels[i];
    float mag = dither_level_value(q < 0 ? -q : q, s_levels, partition) * scale;
    U::store1(out, i, q < 0 ? -mag : mag);
  }
}

template <class U>
__global__ void cast_scale_kernel(const float* in, size_t n, void* out, float mult) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    U::store1(out, i, in[i] * mult);
}

template <class U>
__global__ void nesterov_kernel(void* g, float* m, float mu, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float gv = U::load1(g, i);
    float mv = mu * m[i] + gv;
    m[i] = mv;
    U::store1(g, i, gv + mu * mv);
  }
}

#define DISPATCH_U(dtype, STMT)                    \
  switch (dtype) {                                 \
    case 0: { using U = TagF32; STMT; } break;     \
    case 1: { using U = TagBF16; STMT; } break;    \
    case 2: { using U = TagF16; STMT; } break;     \
    default: return cudaErrorInvalidValue;         \
  }

}  // namespace

cudaError_t launch_ef_correct(const void* g, int dtype, const float* err, float ratio, float* corrected, size_t n,
                              float* acc, cudaStream_t s) {
  // acc layout: [0..3] results, then 3 floats per block (kEfAccFloats in total)
  const int grid = grid_for(n);
  DISPATCH_U(dtype, (ef_correct_kernel<U><<<grid, kThreads, 0, s>>>(g, err, ratio, corrected, n, acc)));
  ef_finalize_kernel<<<1, kThreads, 0, s>>>(acc, grid);
  return cudaGetLastError();
}

cudaError_t launch_onebit_pack(const float* corrected, size_t n, const float* acc, int use_scale, uint32_t* words,
                               float* err_out, cudaStream_t s) {
  onebit_pack_kernel<<<grid_for(n, 1), kThreads, 0, s>>>(corrected, n, acc, use_scale, words, err_out);
  return cudaGetLastError();
}

cudaError_t launch_onebit_exchange_sum(const PeerView& pv, size_t off, size_t n, float* sum, int blocks, int channel,
                                       cudaStream_t s) {
  if (blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  onebit_exchange_sum_kernel<<<blocks, kThreads, 0, s>>>(pv, off, n, sum, channel);
  return cudaGetLastError();
}

cudaError_t launch_onebit_unpack(const uint32_t* words, size_t n, void* out, int dtype, float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (onebit_unpack_kernel<U><<<grid_for(n), kThreads, 0, s>>>(words, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_topk_select(const float* corrected, size_t n, uint32_t k, uint32_t* pairs, float* err_out,
                               uint32_t* scratch, cudaStream_t s) {
  if (k == 0 || k > n) return cudaErrorInvalidValue;
  topk_init_kernel<<<1, 256, 0, s>>>(scratch, k);
  for (int shift = 24; shift >= 0; shift -= 8) {
    topk_hist_kernel<<<grid_for(n), kThreads, 0, s>>>(corrected, n, shift, scratch);
    topk_pick_kernel<<<1, 256, 0, s>>>(shift, scratch);
  }
  topk_compact_kernel<<<grid_for(n), kThreads, 0, s>>>(corrected, n, pairs, err_out, scratch);
  return cudaGetLastError();
}

cudaError_t launch_sparse_exchange_sum(const PeerView& pv, size_t off, uint32_t k, size_t n, float* sum, int blocks,
                                       int channel, cudaStream_t s) {
  if (blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  cudaError_t e = cudaMemsetAsync(sum, 0, n * sizeof(float), s);
  if (e != cudaSuccess) return e;
  sparse_exchange_sum_kernel<<<blocks, kThreads, 0, s>>>(pv, off, k, n, sum, channel);
  return cudaGetLastError();
}

cudaError_t launch_sparse_add(const uint32_t* pairs, uint32_t k, size_t n, float* sum, cudaStream_t s) {
  sparse_add_kernel<<<grid_for(k, 1), kThreads, 0, s>>>(pairs, k, n, sum);
  return cudaGetLastError();
}

cudaError_t launch_sparse_scatter(const uint32_t* pairs, uint32_t k, size_t n, void* out, int dtype, float mult,
                                  cudaStream_t s) {
  DISPATCH_U(dtype, (zero_out_kernel<U><<<grid_for(n), kThreads, 0, s>>>(out, n)));
  DISPATCH_U(dtype, (sparse_scatter_kernel<U><<<grid_for(k, 1), kThreads, 0, s>>>(pairs, k, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_randomk_indices(uint64_t* state, uint32_t k, size_t n, uint32_t* idx, cudaStream_t s) {
  randomk_indices_kernel<<<1, 32, 0, s>>>(state, k, (uint64_t)n, idx);
  return cudaGetLastError();
}

cudaError_t launch_randomk_gather(const float* corrected, const uint32_t* idx, uint32_t k, size_t n, float* vals,
                                  float* err_out, cudaStream_t s) {
  randomk_gather_kernel<<<grid_for(k, 1), kThreads, 0, s>>>(corrected, idx, k, vals, err_out);
  if (err_out) {
    if (err_out != corrected) copy_kernel<<<grid_for(n), kThreads, 0, s>>>(corrected, err_out, n);
    zero_indexed_kernel<<<grid_for(k, 1), kThreads, 0, s>>>(idx, k, err_out);
  }
  return cudaGetLastError();
}

cudaError_t launch_dense_exchange_sum(const PeerView& pv, size_t off, uint32_t k, float* vals_sum, int blocks,
                                      int channel, cudaStream_t s) {
  if (blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  dense_exchange_sum_kernel<<<blocks, kThreads, 0, s>>>(pv, off, k, vals_sum, channel);
  return cudaGetLastError();
}

cudaError_t launch_index_scatter(const uint32_t* idx, const float* vals, uint32_t k, size_t n, void* out, int dtype,
                                 float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (zero_out_kernel<U><<<grid_for(n), kThreads, 0, s>>>(out, n)));
  DISPATCH_U(dtype, (index_scatter_kernel<U><<<grid_for(k, 1), kThreads, 0, s>>>(idx, vals, k, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_dither_quantize(const float* corrected, size_t n, const float* acc, int s_levels, int partition,
                                   int normalize, uint64_t seed, uint64_t step, int8_t* levels, float* scale_out,
                                   float* err_out, cudaStream_t s) {
  if (s_levels < 1 || s_levels > 126) return cudaErrorInvalidValue;
  dither_quantize_kernel<<<grid_for(n), kThreads, 0, s>>>(corrected, n, acc, s_levels, partition, normalize, seed,
                                                         step, levels, scale_out, err_out);
  return cudaGetLastError();
}

cudaError_t launch_dither_exchange_sum(const PeerView& pv, size_t off, size_t n, int s_levels, int partition,
                                       float* sum, int blocks, int channel, cudaStream_t s) {
  if (blocks < 1 || blocks > kMaxBlocks) return cudaErrorInvalidValue;
  dither_exchange_sum_kernel<<<blocks, kThreads, 0, s>>>(pv, off, n, s_levels, partition, sum, channel);
  return cudaGetLastError();
}

cudaError_t launch_dither_unpack(const int8_t* levels, const float* scale, size_t n, int s_levels, int partition,
                                 void* out, int dtype, float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (dither_unpack_kernel<U><<<grid_for(n), kThreads, 0, s>>>(levels, scale, n, s_levels, partition,
                                                                              out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_cast_scale(const float* in, size_t n, void* out, int dtype, float mult, cudaStream_t s) {
  DISPATCH_U(dtype, (cast_scale_kernel<U><<<grid_for(n), kThreads, 0, s>>>(in, n, out, mult)));
  return cudaGetLastError();
}

cudaError_t launch_nesterov(void* g, int dtype, float* m, float mu, size_t n, cudaStream_t s) {
  DISPATCH_U(dtype, (nesterov_kernel<U><<<grid_for(n), kThreads, 0, s>>>(g, m, mu, n)));
  return cudaGetLastError();
}

}  // namespace bps
