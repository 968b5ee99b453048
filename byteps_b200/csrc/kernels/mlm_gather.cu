// Gather of labelled rows and the scatter of their gradient (see mlm_gather.cuh).
//
// The scan is one CTA of kScanT threads; each thread owns kItems consecutive tokens of a tile, so a block-wide
// exclusive scan of the per-thread counts, plus the count carried from earlier tiles, numbers the labelled tokens in
// token order.  The next tile's labels are loaded before the current tile is scanned.  The copy is one warp per row:
// lanes stride over the row's 16-byte vectors with kUnroll loads in flight, and one kernel serves both directions
// (forward: row j from source token src[j]; backward: token t from slot slot[t]).
#include "kernels/mlm_gather.cuh"

namespace bps {

namespace {

constexpr int kScanT = 1024;
constexpr int kScanW = kScanT / 32;
constexpr int kItems = 8;
constexpr size_t kTile = (size_t)kScanT * kItems;
constexpr int kCopyT = 256;
constexpr int kUnroll = 4;

struct ScanArgs {
  const int64_t* labels;
  int64_t* row_labels;
  int32_t *slot, *src;
  int64_t* dropped;
  size_t T;
  int64_t C, ignore;
};

__device__ __forceinline__ void load_tile(const ScanArgs& a, size_t first, int64_t (&lab)[kItems]) {
#pragma unroll
  for (int k = 0; k < kItems; ++k) lab[k] = first + k < a.T ? __ldg(a.labels + first + k) : a.ignore;
}

__global__ void __launch_bounds__(kScanT) mlm_scan_kernel(ScanArgs a) {
  __shared__ int warp_sum[kScanW];
  const int tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  int64_t carry = 0;   // labelled tokens before this tile
  int64_t nxt[kItems];
  load_tile(a, (size_t)tid * kItems, nxt);
  for (size_t t0 = 0; t0 < a.T; t0 += kTile) {
    const size_t first = t0 + (size_t)tid * kItems;
    int64_t lab[kItems];
    int cnt = 0;
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      lab[k] = nxt[k];
      cnt += lab[k] != a.ignore;
    }
    load_tile(a, first + kTile, nxt);
    int inc = cnt;   // inclusive scan over the warp, then over the warps' totals
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    if (lane == 31) warp_sum[w] = inc;
    __syncthreads();
    if (w == 0) {
      int s = warp_sum[lane];
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const int v = __shfl_up_sync(0xffffffffu, s, o);
        if (lane >= o) s += v;
      }
      warp_sum[lane] = s;
    }
    __syncthreads();
    int64_t n = carry + (w > 0 ? warp_sum[w - 1] : 0) + (inc - cnt);
#pragma unroll
    for (int k = 0; k < kItems; ++k) {
      const size_t t = first + k;
      if (t >= a.T) break;
      int32_t sl = -1;
      if (lab[k] != a.ignore) {
        if (n < a.C) {
          sl = (int32_t)n;
          a.src[n] = (int32_t)t;
          a.row_labels[n] = lab[k];
        }
        ++n;
      }
      a.slot[t] = sl;
    }
    carry += warp_sum[kScanW - 1];
    __syncthreads();   // warp_sum is rewritten by the next tile
  }
  for (int64_t j = (carry < a.C ? carry : a.C) + tid; j < a.C; j += kScanT) {
    a.src[j] = -1;
    a.row_labels[j] = a.ignore;
  }
  if (tid == 0) *a.dropped = carry > a.C ? carry - a.C : 0;
}

// dst row r = src row idx[r], or zeros when idx[r] is outside [0, limit)
__global__ void __launch_bounds__(kCopyT) mlm_copy_rows_kernel(const char* __restrict__ src,
                                                               const int32_t* __restrict__ idx, int64_t limit,
                                                               char* __restrict__ dst, size_t nrows, size_t nvec) {
  const int lane = threadIdx.x & 31;
  const size_t nwarps = (size_t)gridDim.x * (kCopyT / 32);
  const size_t row_bytes = nvec * 16;
  const uint4 zero = make_uint4(0u, 0u, 0u, 0u);
  for (size_t r = ((size_t)blockIdx.x * kCopyT + threadIdx.x) / 32; r < nrows; r += nwarps) {
    const int32_t j = __ldg(idx + r);
    const bool ok = j >= 0 && (int64_t)j < limit;
    const uint4* s = reinterpret_cast<const uint4*>(src + (ok ? (size_t)j : 0) * row_bytes);
    uint4* d = reinterpret_cast<uint4*>(dst + r * row_bytes);
    size_t i = lane;
    for (; i + (kUnroll - 1) * 32 < nvec; i += kUnroll * 32) {
      uint4 v[kUnroll];
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) v[u] = ok ? __ldg(s + i + u * 32) : zero;
#pragma unroll
      for (int u = 0; u < kUnroll; ++u) d[i + u * 32] = v[u];
    }
    for (; i < nvec; i += 32) d[i] = ok ? __ldg(s + i) : zero;
  }
}

int sm_count() {
  int dev = 0, sms = 132;
  if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) sms = 132;
  return sms;
}

bool aligned(const void* p, uintptr_t a) { return p != nullptr && ((uintptr_t)p & (a - 1)) == 0; }

bool bad_shape(size_t T, size_t row_bytes, int64_t C) {
  return T < 1 || T > (size_t)INT32_MAX || row_bytes < 16 || row_bytes % 16 != 0 || C < 1 || C > INT32_MAX;
}

cudaError_t copy_rows(const void* src, const int32_t* idx, int64_t limit, void* dst, size_t nrows, size_t row_bytes,
                      cudaStream_t s) {
  const size_t want = (nrows + kCopyT / 32 - 1) / (kCopyT / 32), cap = (size_t)sm_count() * 8;
  const int grid = (int)(want < cap ? want : cap);
  mlm_copy_rows_kernel<<<grid, kCopyT, 0, s>>>(static_cast<const char*>(src), idx, limit, static_cast<char*>(dst),
                                               nrows, row_bytes / 16);
  return cudaGetLastError();
}

}  // namespace

cudaError_t launch_mlm_gather_fwd(const void* x, const int64_t* labels, size_t T, size_t row_bytes, int64_t C,
                                  int64_t ignore_index, void* rows, int64_t* row_labels, int32_t* slot, int32_t* src,
                                  int64_t* dropped, cudaStream_t s) {
  if (bad_shape(T, row_bytes, C) || !aligned(x, 16) || !aligned(rows, 16) || !aligned(labels, 8) ||
      !aligned(row_labels, 8) || !aligned(dropped, 8) || !aligned(slot, 4) || !aligned(src, 4))
    return cudaErrorInvalidValue;
  mlm_scan_kernel<<<1, kScanT, 0, s>>>(ScanArgs{labels, row_labels, slot, src, dropped, T, C, ignore_index});
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  return copy_rows(x, src, (int64_t)T, rows, (size_t)C, row_bytes, s);
}

cudaError_t launch_mlm_scatter_bwd(const void* drows, const int32_t* slot, size_t T, size_t row_bytes, int64_t C,
                                   void* dx, cudaStream_t s) {
  if (bad_shape(T, row_bytes, C) || !aligned(drows, 16) || !aligned(dx, 16) || !aligned(slot, 4))
    return cudaErrorInvalidValue;
  return copy_rows(drows, slot, C, dx, T, row_bytes, s);
}

}  // namespace bps
