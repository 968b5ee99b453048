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
__global__ void ef_correct_kernel(const void* g, float* mom, float mu, const float* err, float ratio, float* corrected,
                                  size_t n, float* acc) {
  float s_abs = 0.f, s_sq = 0.f, s_max = 0.f;
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float v = load_as_float<U>(g, i);
    if (mom) {   // nesterov in fp32: the user's gradient is only read
      const float m = mu * mom[i] + v;
      mom[i] = m;
      v += mu * m;
    }
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

// ---------------------------------------------------------------- random-k: scatter of the summed values
template <class U>
__global__ void zero_out_kernel(void* out, size_t n) {
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    U::store1(out, i, 0.f);
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

#define DISPATCH_U(dtype, STMT)                    \
  switch (dtype) {                                 \
    case 0: { using U = TagF32; STMT; } break;     \
    case 1: { using U = TagBF16; STMT; } break;    \
    case 2: { using U = TagF16; STMT; } break;     \
    default: return cudaErrorInvalidValue;         \
  }

}  // namespace

cudaError_t launch_ef_correct(const void* g, int dtype, float* mom, float mu, const float* err, float ratio,
                              float* corrected, size_t n, float* acc, cudaStream_t s) {
  // acc layout: [0..3] results, then 3 floats per block (kEfAccFloats in total)
  const int grid = grid_for(n);
  DISPATCH_U(dtype, (ef_correct_kernel<U><<<grid, kThreads, 0, s>>>(g, mom, mu, err, ratio, corrected, n, acc)));
  ef_finalize_kernel<<<1, kThreads, 0, s>>>(acc, grid);
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

}  // namespace bps
