#include "cpu/reducer.h"

// x86 SIMD paths are optional: every kernel has a scalar loop behind it (aarch64 hosts - Grace Hopper
// systems - and x86 without AVX2 build and run; define BPS_NO_X86_SIMD to force the scalar build for testing)
#if (defined(__x86_64__) || defined(__i386__)) && defined(__AVX2__) && defined(__F16C__) && !defined(BPS_NO_X86_SIMD)
#define BPS_X86_SIMD 1
#include <immintrin.h>
#else
#define BPS_X86_SIMD 0
#endif
#include <omp.h>

#include <cmath>
#include <cstring>

#include "core/env.h"
#include "core/log.h"
#include "cpu/half.h"

namespace bps {

CpuReducer::CpuReducer(int num_threads) {
  if (num_threads <= 0) num_threads = (int)env_int("BYTEPS_OMP_THREAD_PER_GPU", 4);
  if (num_threads <= 0) num_threads = 1;
  nthreads_ = num_threads;
}

bool CpuReducer::has_avx512() {
#if BPS_X86_SIMD
  static int v = (__builtin_cpu_supports("avx512f") && __builtin_cpu_supports("avx512bw")) ? 1 : 0;
  return v != 0;
#else
  return false;
#endif
}

// --------------------------------------------------------------------------
// generic typed kernels (the compiler vectorises these under -mavx2)
// --------------------------------------------------------------------------
template <typename T>
static void k_sum2(T* dst, const T* src, size_t n, int nt) {
#pragma omp parallel for simd num_threads(nt) schedule(static)
  for (size_t i = 0; i < n; ++i) dst[i] = dst[i] + src[i];
}
template <typename T>
static void k_sum3(T* dst, const T* a, const T* b, size_t n, int nt) {
#pragma omp parallel for simd num_threads(nt) schedule(static)
  for (size_t i = 0; i < n; ++i) dst[i] = a[i] + b[i];
}
template <typename T>
static void k_axpy2(T* dst, const T* src, size_t n, float alpha, int nt) {
#pragma omp parallel for simd num_threads(nt) schedule(static)
  for (size_t i = 0; i < n; ++i) dst[i] = static_cast<T>(dst[i] + alpha * src[i]);
}
template <typename T>
static void k_axpy3(T* dst, const T* a, const T* b, size_t n, float alpha, int nt) {
#pragma omp parallel for simd num_threads(nt) schedule(static)
  for (size_t i = 0; i < n; ++i) dst[i] = static_cast<T>(a[i] + alpha * b[i]);
}

// --------------------------------------------------------------------------
// 16-bit float kernels: dst = a + alpha*b computed in fp32, 8 lanes (AVX2) or
// 16 lanes (AVX-512) at a time.
// --------------------------------------------------------------------------
#if BPS_X86_SIMD
static inline __m256 load_f16x8(const uint16_t* p) { return _mm256_cvtph_ps(_mm_loadu_si128((const __m128i*)p)); }
static inline void store_f16x8(uint16_t* p, __m256 v) {
  _mm_storeu_si128((__m128i*)p, _mm256_cvtps_ph(v, _MM_FROUND_TO_NEAREST_INT | _MM_FROUND_NO_EXC));
}
static inline __m256 load_bf16x8(const uint16_t* p) {
  __m128i h = _mm_loadu_si128((const __m128i*)p);
  return _mm256_castsi256_ps(_mm256_slli_epi32(_mm256_cvtepu16_epi32(h), 16));
}
static inline void store_bf16x8(uint16_t* p, __m256 v) {
  // round-to-nearest-even on the dropped 16 bits; NaNs stay NaN (quiet bit forced)
  __m256i u = _mm256_castps_si256(v);
  __m256i lsb = _mm256_and_si256(_mm256_srli_epi32(u, 16), _mm256_set1_epi32(1));
  __m256i r = _mm256_add_epi32(u, _mm256_add_epi32(lsb, _mm256_set1_epi32(0x7fff)));
  __m256i isnan = _mm256_castps_si256(_mm256_cmp_ps(v, v, _CMP_UNORD_Q));
  __m256i qnan = _mm256_or_si256(u, _mm256_set1_epi32(0x00400000));
  r = _mm256_blendv_epi8(r, qnan, isnan);
  r = _mm256_srli_epi32(r, 16);
  __m128i lo = _mm256_castsi256_si128(r), hi = _mm256_extracti128_si256(r, 1);
  _mm_storeu_si128((__m128i*)p, _mm_packus_epi32(lo, hi));
}

#endif

template <bool BF>
static void k_half_axpy3(uint16_t* dst, const uint16_t* a, const uint16_t* b, size_t n, float alpha, int nt) {
#if BPS_X86_SIMD
  const size_t nv = n / 8;
  const __m256 va = _mm256_set1_ps(alpha);
#pragma omp parallel for num_threads(nt) schedule(static)
  for (size_t i = 0; i < nv; ++i) {
    __m256 x = BF ? load_bf16x8(a + i * 8) : load_f16x8(a + i * 8);
    __m256 y = BF ? load_bf16x8(b + i * 8) : load_f16x8(b + i * 8);
    __m256 r = _mm256_fmadd_ps(va, y, x);
    if (BF) store_bf16x8(dst + i * 8, r);
    else store_f16x8(dst + i * 8, r);
  }
  const size_t tail = nv * 8;
#else
  const size_t tail = 0;
#endif
#pragma omp parallel for num_threads(nt) schedule(static) if (n - tail > 65536)
  for (size_t i = tail; i < n; ++i) {
    float x = BF ? bf16_to_f32(a[i]) : f16_to_f32(a[i]);
    float y = BF ? bf16_to_f32(b[i]) : f16_to_f32(b[i]);
    float r = x + alpha * y;
    dst[i] = BF ? f32_to_bf16(r) : f32_to_f16(r);
  }
}

#if BPS_X86_SIMD
__attribute__((target("avx512f,avx512bw,avx512vl"))) static void k_f32_sum2_avx512(float* dst, const float* src,
                                                                                  size_t n, int nt) {
  const size_t nv = n / 16;
#pragma omp parallel for num_threads(nt) schedule(static)
  for (size_t i = 0; i < nv; ++i) {
    __m512 x = _mm512_loadu_ps(dst + i * 16), y = _mm512_loadu_ps(src + i * 16);
    _mm512_storeu_ps(dst + i * 16, _mm512_add_ps(x, y));
  }
  for (size_t i = nv * 16; i < n; ++i) dst[i] += src[i];
}

__attribute__((target("avx512f,avx512bw,avx512vl"))) static void k_bf16_axpy3_avx512(uint16_t* dst,
                                                                                    const uint16_t* a,
                                                                                    const uint16_t* b, size_t n,
                                                                                    float alpha, int nt) {
  const size_t nv = n / 16;
  const __m512 va = _mm512_set1_ps(alpha);
#pragma omp parallel for num_threads(nt) schedule(static)
  for (size_t i = 0; i < nv; ++i) {
    __m512 x = _mm512_castsi512_ps(
        _mm512_slli_epi32(_mm512_cvtepu16_epi32(_mm256_loadu_si256((const __m256i*)(a + i * 16))), 16));
    __m512 y = _mm512_castsi512_ps(
        _mm512_slli_epi32(_mm512_cvtepu16_epi32(_mm256_loadu_si256((const __m256i*)(b + i * 16))), 16));
    __m512 r = _mm512_fmadd_ps(va, y, x);
    __m512i u = _mm512_castps_si512(r);
    __m512i lsb = _mm512_and_si512(_mm512_srli_epi32(u, 16), _mm512_set1_epi32(1));
    __m512i rr = _mm512_add_epi32(u, _mm512_add_epi32(lsb, _mm512_set1_epi32(0x7fff)));
    __mmask16 nanm = _mm512_cmp_ps_mask(r, r, _CMP_UNORD_Q);
    rr = _mm512_mask_mov_epi32(rr, nanm, _mm512_or_si512(u, _mm512_set1_epi32(0x00400000)));
    _mm256_storeu_si256((__m256i*)(dst + i * 16), _mm512_cvtepi32_epi16(_mm512_srli_epi32(rr, 16)));
  }
  for (size_t i = nv * 16; i < n; ++i) dst[i] = f32_to_bf16(bf16_to_f32(a[i]) + alpha * bf16_to_f32(b[i]));
}

#else
static void k_f32_sum2_avx512(float*, const float*, size_t, int) {}
static void k_bf16_axpy3_avx512(uint16_t*, const uint16_t*, const uint16_t*, size_t, float, int) {}
#endif

// --------------------------------------------------------------------------
int CpuReducer::sum(void* dst, const void* src, size_t nbytes, int dtype) const {
  return sum(dst, dst, src, nbytes, dtype);
}

int CpuReducer::sum(void* dst, const void* a, const void* b, size_t nbytes, int dtype) const {
  const int nt = nthreads_;
  switch (dtype) {
    case F32:
      if (dst == a && has_avx512()) k_f32_sum2_avx512((float*)dst, (const float*)b, nbytes / 4, nt);
      else k_sum3((float*)dst, (const float*)a, (const float*)b, nbytes / 4, nt);
      break;
    case F64: k_sum3((double*)dst, (const double*)a, (const double*)b, nbytes / 8, nt); break;
    case F16: k_half_axpy3<false>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, 1.0f, nt); break;
    case BF16:
      if (has_avx512()) k_bf16_axpy3_avx512((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, 1.0f, nt);
      else k_half_axpy3<true>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, 1.0f, nt);
      break;
    case U8: k_sum3((uint8_t*)dst, (const uint8_t*)a, (const uint8_t*)b, nbytes, nt); break;
    case I8: k_sum3((int8_t*)dst, (const int8_t*)a, (const int8_t*)b, nbytes, nt); break;
    case I32: k_sum3((int32_t*)dst, (const int32_t*)a, (const int32_t*)b, nbytes / 4, nt); break;
    case I64: k_sum3((int64_t*)dst, (const int64_t*)a, (const int64_t*)b, nbytes / 8, nt); break;
    default: BPS_LOG(ERROR) << "CpuReducer: unsupported dtype " << dtype; return -1;
  }
  return 0;
}

int CpuReducer::sum_scaled(void* dst, const void* src, size_t nbytes, int dtype, float alpha) const {
  return sum_scaled(dst, dst, src, nbytes, dtype, alpha);
}

int CpuReducer::sum_scaled(void* dst, const void* a, const void* b, size_t nbytes, int dtype, float alpha) const {
  const int nt = nthreads_;
  switch (dtype) {
    case F32: k_axpy3((float*)dst, (const float*)a, (const float*)b, nbytes / 4, alpha, nt); break;
    case F64: k_axpy3((double*)dst, (const double*)a, (const double*)b, nbytes / 8, alpha, nt); break;
    case F16: k_half_axpy3<false>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, alpha, nt); break;
    case BF16:
      if (has_avx512()) k_bf16_axpy3_avx512((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, alpha, nt);
      else k_half_axpy3<true>((uint16_t*)dst, (const uint16_t*)a, (const uint16_t*)b, nbytes / 2, alpha, nt);
      break;
    case U8: k_axpy3((uint8_t*)dst, (const uint8_t*)a, (const uint8_t*)b, nbytes, alpha, nt); break;
    case I8: k_axpy3((int8_t*)dst, (const int8_t*)a, (const int8_t*)b, nbytes, alpha, nt); break;
    case I32: k_axpy3((int32_t*)dst, (const int32_t*)a, (const int32_t*)b, nbytes / 4, alpha, nt); break;
    case I64: k_axpy3((int64_t*)dst, (const int64_t*)a, (const int64_t*)b, nbytes / 8, alpha, nt); break;
    default: BPS_LOG(ERROR) << "CpuReducer: unsupported dtype " << dtype; return -1;
  }
  return 0;
}

template <typename T>
static void k_floor_div(T* d, size_t n, long long div, int nt) {
#pragma omp parallel for num_threads(nt) schedule(static)
  for (size_t i = 0; i < n; ++i) {
    long long v = (long long)d[i];
    long long q = v / div;
    if ((v % div != 0) && ((v < 0) != (div < 0))) --q;  // floor semantics like torch.floor_divide
    d[i] = (T)q;
  }
}

int CpuReducer::scale(void* dst, size_t nbytes, int dtype, double alpha) const {
  const int nt = nthreads_;
  const float fa = (float)alpha;
  switch (dtype) {
    case F32: {
      float* d = (float*)dst;
      size_t n = nbytes / 4;
#pragma omp parallel for simd num_threads(nt) schedule(static)
      for (size_t i = 0; i < n; ++i) d[i] *= fa;
      break;
    }
    case F64: {
      double* d = (double*)dst;
      size_t n = nbytes / 8;
#pragma omp parallel for simd num_threads(nt) schedule(static)
      for (size_t i = 0; i < n; ++i) d[i] *= alpha;
      break;
    }
    case F16: {
      uint16_t* d = (uint16_t*)dst;
      size_t n = nbytes / 2;
#pragma omp parallel for num_threads(nt) schedule(static)
      for (size_t i = 0; i < n; ++i) d[i] = f32_to_f16(f16_to_f32(d[i]) * fa);
      break;
    }
    case BF16: {
      uint16_t* d = (uint16_t*)dst;
      size_t n = nbytes / 2;
#pragma omp parallel for num_threads(nt) schedule(static)
      for (size_t i = 0; i < n; ++i) d[i] = f32_to_bf16(bf16_to_f32(d[i]) * fa);
      break;
    }
    case U8: case I8: case I32: case I64: {
      long long div = (long long)std::llround(1.0 / alpha);
      if (div <= 0) div = 1;
      if (dtype == U8) k_floor_div((uint8_t*)dst, nbytes, div, nt);
      else if (dtype == I8) k_floor_div((int8_t*)dst, nbytes, div, nt);
      else if (dtype == I32) k_floor_div((int32_t*)dst, nbytes / 4, div, nt);
      else k_floor_div((int64_t*)dst, nbytes / 8, div, nt);
      break;
    }
    default: return -1;
  }
  return 0;
}

void CpuReducer::copy(void* dst, const void* src, size_t nbytes) const {
  if (dst == src || nbytes == 0) return;
  const int nt = nthreads_;
  const size_t chunk = 1 << 20;
  if (nbytes <= chunk || nt <= 1) {
    memcpy(dst, src, nbytes);
    return;
  }
  const size_t nchunks = (nbytes + chunk - 1) / chunk;
#pragma omp parallel for num_threads(nt) schedule(static)
  for (size_t c = 0; c < nchunks; ++c) {
    size_t off = c * chunk;
    size_t len = (nbytes - off < chunk) ? nbytes - off : chunk;
    memcpy((char*)dst + off, (const char*)src + off, len);
  }
}

}  // namespace bps
