// ResNet's 7x7 / stride-2 stem convolution over a 3-channel bf16 NHWC image, forward and weight gradient, on
// mma.sync.m16n8k16 tensor-core tiles (see stem_conv.cuh and DESIGN.md section 1.17).
//
// Work unit: a segment of up to kSeg pixels of one output row (n, oh).  Its 7 input rows are staged in shared memory
// split by column parity, 4 channel slots per column (the fourth zero):
//   entry e of (kh, even) = x[2 oh - 3 + kh][2 (ow0 + e) - 3][0..2], of (kh, odd) = x[..][2 (ow0 + e) - 2][0..2]
// so that output pixel p = ow - ow0 reads, for each kh, kw = 0, 2, 4, 6 as entries p .. p + 3 of the even row and
// kw = 1, 3, 5 as entries p .. p + 2 of the odd row: 16 and 12 contiguous elements.  K is laid out to match, 14
// k-steps of 16, k-step 2 kh + parity holding slot (kw / 2, c); slot c = 3, and slots 12..15 of an odd step, are
// padding with zero weight and zero A.
#include "kernels/stem_conv.cuh"

#include "kernels/attn_tile.cuh"

namespace bps {

namespace {

constexpr int kSeg = 128;                          // output pixels per unit
constexpr int kEntries = kSeg + 3;                 // staged columns per (kh, parity)
constexpr int kXE = 132;                           // their pitch, in 8-byte entries
constexpr int kSteps = 14;                         // k-steps of 16: 7 kh x 2 parities
constexpr int kKL = kSteps * 16;                   // padded K (224)
constexpr int kK = 147;                            // real K: (kh, kw, c)
constexpr int kCo = 64;
constexpr int kWRow = kKL + 8;                     // weight row pitch in elements: 464 B, conflict-free ldmatrix
constexpr int kXBytes = kSteps * kXE * 8;          // 14,784
constexpr int kWBytes = kCo * kWRow * 2;           // 29,696
constexpr int kFwdThreads = 128;                   // 4 warps x 32 pixels
constexpr int kFwdSmem = kWBytes + kXBytes + 4 * 32 * 128;
constexpr int kWgThreads = 256;                    // 8 warps: 2 halves of co x 4 quarters of K
constexpr int kWgSmem = kXBytes + kSeg * 128;
constexpr int kReduceThreads = 256;

struct Unit {
  int64_t row;   // n * OH + oh
  int oh, ow0, valid;
};

__device__ __forceinline__ Unit unit_at(int64_t u, int nseg, int OH, int OW) {
  Unit r;
  const int seg = (int)(u % nseg);
  r.row = u / nseg;
  r.oh = (int)(r.row % OH);
  r.ow0 = seg * kSeg;
  r.valid = min(kSeg, OW - r.ow0);
  return r;
}

// the 7 input rows of a unit, by column parity, as 8-byte entries (c0, c1, c2, 0); zero outside the image
__device__ __forceinline__ void stage_x(uint8_t* sx, const uint16_t* __restrict__ x, const Unit& u, int OH, int H,
                                        int W) {
  const int64_t n = u.row / OH;
  for (int i = threadIdx.x; i < kSteps * kEntries; i += blockDim.x) {
    const int r = i / kEntries, e = i - r * kEntries;
    const int ih = 2 * u.oh - 3 + (r >> 1), iw = 2 * (u.ow0 + e) - 3 + (r & 1);
    uint32_t lo = 0, hi = 0;
    if ((unsigned)ih < (unsigned)H && (unsigned)iw < (unsigned)W) {
      const uint16_t* p = x + ((n * H + ih) * W + iw) * 3;
      lo = (uint32_t)p[0] | (uint32_t)p[1] << 16;
      hi = p[2];
    }
    *reinterpret_cast<uint2*>(sx + (r * kXE + e) * 8) = make_uint2(lo, hi);
  }
}

// (kh, kw, c) of padded K index kl, or false for a padding slot
__device__ __forceinline__ bool k_of(int kl, int* kh, int* kw, int* c) {
  const int ks = kl >> 4, j = kl & 15;
  *kh = ks >> 1;
  *kw = 2 * (j >> 2) + (ks & 1);
  *c = j & 3;
  return *c < 3 && *kw < 7;
}

__device__ __forceinline__ int w_index(bool w_cl, int co, int kh, int kw, int c) {
  return w_cl ? co * kK + kh * 21 + kw * 3 + c : co * kK + c * 49 + kh * 7 + kw;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__global__ void __launch_bounds__(kFwdThreads) stem_conv_fwd_kernel(const uint16_t* __restrict__ x,
                                                                    const uint16_t* __restrict__ w, bool w_cl,
                                                                    uint16_t* __restrict__ y, int H, int W, int OH,
                                                                    int OW, int nseg, int64_t units) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sw = smem;
  uint8_t* sx = smem + kWBytes;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  uint8_t* so = sx + kXBytes + warp * 32 * 128;
  for (int i = threadIdx.x; i < kCo * kKL; i += blockDim.x) {
    const int co = i / kKL, kl = i - co * kKL;
    int kh, kw, c;
    const uint16_t v = k_of(kl, &kh, &kw, &c) ? w[w_index(w_cl, co, kh, kw, c)] : (uint16_t)0;
    *reinterpret_cast<uint16_t*>(sw + (co * kWRow + kl) * 2) = v;
  }
  const uint32_t swa = smem_u32(sw);
  const int p0 = warp * 32;
  for (int64_t ui = blockIdx.x; ui < units; ui += gridDim.x) {
    const Unit u = unit_at(ui, nseg, OH, OW);
    __syncthreads();   // the weights are packed and every warp is done with the previous unit's rows
    stage_x(sx, x, u, OH, H, W);
    __syncthreads();
    if (p0 >= u.valid) continue;
    float acc[2][8][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int n = 0; n < 8; ++n)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[mt][n][j] = 0.f;
#pragma unroll
    for (int ks = 0; ks < kSteps; ++ks) {
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt) {
        const uint8_t* pa = sx + ks * kXE * 8 + (p0 + 16 * mt + g) * 8 + 4 * t;
        a[mt][0] = *reinterpret_cast<const uint32_t*>(pa);
        a[mt][1] = *reinterpret_cast<const uint32_t*>(pa + 64);
        a[mt][2] = *reinterpret_cast<const uint32_t*>(pa + 16);
        a[mt][3] = *reinterpret_cast<const uint32_t*>(pa + 80);
        if ((ks & 1) && t >= 2) a[mt][2] = a[mt][3] = 0u;   // slots 12..15 of an odd step
      }
#pragma unroll
      for (int np = 0; np < 4; ++np) {
        uint32_t b[4];
        ldsm4(b, swa + (16 * np + (lane & 7) + ((lane >> 4) << 3)) * (kWRow * 2) + (2 * ks + ((lane >> 3) & 1)) * 16);
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) {
          mma<true>(acc[mt][2 * np], a[mt], b[0], b[1]);
          mma<true>(acc[mt][2 * np + 1], a[mt], b[2], b[3]);
        }
      }
    }
    // the warp's 32 x 64 tile through shared memory, then 16-byte stores of whole 128-byte pixels
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int n = 0; n < 8; ++n) {
        const int r = 16 * mt + g;
        *reinterpret_cast<uint32_t*>(so + swz(r, n) + 4 * t) = f2_to_bf16x2(acc[mt][n][0], acc[mt][n][1]);
        *reinterpret_cast<uint32_t*>(so + swz(r + 8, n) + 4 * t) = f2_to_bf16x2(acc[mt][n][2], acc[mt][n][3]);
      }
    __syncwarp();
    uint16_t* yt = y + (u.row * OW + u.ow0 + p0) * kCo;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const int i = lane + 32 * q, r = i >> 3, ch = i & 7;
      if (p0 + r < u.valid)
        *reinterpret_cast<uint4*>(yt + r * kCo + ch * 8) = *reinterpret_cast<const uint4*>(so + swz(r, ch));
    }
    __syncwarp();
  }
}

// Partial dW of the CTA's contiguous range of units: C[co][kl] += sum_p dy[p][co] X[p][kl].  Warp w owns co
// 32 (w & 1) .. + 31 (two m-tiles, A = dy^T by ldmatrix.trans) and kl 56 (w >> 1) .. + 55 (seven n-tiles, B built
// from pairs of staged pixels).
__global__ void __launch_bounds__(kWgThreads) stem_conv_wgrad_kernel(const uint16_t* __restrict__ x,
                                                                     const uint16_t* __restrict__ dy,
                                                                     float* __restrict__ ws, int H, int W, int OH,
                                                                     int OW, int nseg, int64_t units) {
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* sx = smem;
  uint8_t* sdy = smem + kXBytes;
  const uint32_t sdya = smem_u32(sdy);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
  const int mh = warp & 1, kq = warp >> 1;
  int boff[7];   // byte offset of (pixel 0, kl = 56 kq + 8 i + g) in the staged rows
#pragma unroll
  for (int i = 0; i < 7; ++i) {
    const int k = 56 * kq + 8 * i + g, ks = k >> 4, j = k & 15;
    boff[i] = ks * kXE * 8 + (j >> 2) * 8 + (j & 3) * 2;
  }
  float acc[2][7][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int i = 0; i < 7; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[mt][i][j] = 0.f;
  const int64_t u0 = units * blockIdx.x / gridDim.x, u1 = units * (blockIdx.x + 1) / gridDim.x;
  for (int64_t ui = u0; ui < u1; ++ui) {
    const Unit u = unit_at(ui, nseg, OH, OW);
    __syncthreads();   // every warp is done with the previous unit
    stage_x(sx, x, u, OH, H, W);
    const uint16_t* dyt = dy + (u.row * OW + u.ow0) * kCo;
    for (int i = threadIdx.x; i < kSeg * 8; i += blockDim.x) {
      const int r = i >> 3, ch = i & 7;
      const bool ok = r < u.valid;   // pixels past the row read as zero
      cp_async16(sdya + swz(r, ch), ok ? dyt + r * kCo + ch * 8 : dy, ok);
    }
    cp_commit();
    cp_wait<0>();
    __syncthreads();
    for (int p0 = 0; p0 < u.valid; p0 += 16) {
      uint32_t a[2][4];
#pragma unroll
      for (int mt = 0; mt < 2; ++mt)
        ldsm4t(a[mt], sdya + swz(p0 + (lane & 7) + ((lane >> 4) << 3), 4 * mh + 2 * mt + ((lane >> 3) & 1)));
      const uint8_t* px = sx + (p0 + 2 * t) * 8;
#pragma unroll
      for (int i = 0; i < 7; ++i) {
        const uint8_t* q = px + boff[i];
        const uint32_t b0 = (uint32_t)*reinterpret_cast<const uint16_t*>(q) |
                            (uint32_t)*reinterpret_cast<const uint16_t*>(q + 8) << 16;
        const uint32_t b1 = (uint32_t)*reinterpret_cast<const uint16_t*>(q + 64) |
                            (uint32_t)*reinterpret_cast<const uint16_t*>(q + 72) << 16;
        mma<true>(acc[0][i], a[0], b0, b1);
        mma<true>(acc[1][i], a[1], b0, b1);
      }
    }
  }
  float* part = ws + (int64_t)blockIdx.x * kCo * kK;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int i = 0; i < 7; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        int kh, kw, c;
        if (k_of(56 * kq + 8 * i + 2 * t + (j & 1), &kh, &kw, &c))
          part[(32 * mh + 16 * mt + g + 8 * (j >> 1)) * kK + kh * 21 + kw * 3 + c] = acc[mt][i][j];
      }
}

// dW[co, kh, kw, c] = sum of the partials in the order b = 0 .. P - 1, rounded once, in w's layout
__global__ void __launch_bounds__(kReduceThreads) stem_conv_wgrad_reduce_kernel(const float* __restrict__ ws,
                                                                                int partials,
                                                                                uint16_t* __restrict__ dw, bool w_cl) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= kCo * kK) return;
  float s = 0.f;
#pragma unroll 8
  for (int b = 0; b < partials; ++b) s += ws[(int64_t)b * kCo * kK + i];
  const int co = i / kK, k = i - co * kK, kh = k / 21, kw = (k % 21) / 3, c = k % 3;
  dw[w_index(w_cl, co, kh, kw, c)] = (uint16_t)(f2_to_bf16x2(s, 0.f) & 0xffffu);
}

struct Geometry {
  int OH, OW, nseg;
  int64_t units;
};

Geometry geometry(int64_t N, int64_t H, int64_t W) {
  Geometry gm;
  gm.OH = (int)((H - 1) / 2 + 1);
  gm.OW = (int)((W - 1) / 2 + 1);
  gm.nseg = (gm.OW + kSeg - 1) / kSeg;
  gm.units = N * gm.OH * gm.nseg;
  return gm;
}

// resident CTAs of `kernel` per device: SMs x CTAs per SM (0 on error)
template <class K>
int64_t resident(K kernel, int threads, int smem, int* cache) {
  const int dev = device();
  if (cache[dev] == 0) {
    int sms = 0, per = 0;
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
    if (smem > 48 * 1024 &&
        cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem) != cudaSuccess)
      return 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per, kernel, threads, smem) != cudaSuccess) return 0;
    cache[dev] = sms * per;
  }
  return cache[dev];
}

int fwd_resident[kMaxDevices], wgrad_resident[kMaxDevices];

}  // namespace

int stem_conv_wgrad_partials(int64_t N, int64_t H, int64_t W) {
  const int64_t r = resident(stem_conv_wgrad_kernel, kWgThreads, kWgSmem, wgrad_resident);
  const Geometry gm = geometry(N, H, W);
  return (int)(r < gm.units ? r : gm.units);
}

cudaError_t launch_stem_conv_fwd(const void* x, const void* w, bool w_cl, void* y, int64_t N, int64_t H, int64_t W,
                                 cudaStream_t s) {
  const int64_t r = resident(stem_conv_fwd_kernel, kFwdThreads, kFwdSmem, fwd_resident);
  if (r == 0) return cudaErrorInvalidConfiguration;
  const Geometry gm = geometry(N, H, W);
  const int grid = (int)(r < gm.units ? r : gm.units);
  stem_conv_fwd_kernel<<<grid, kFwdThreads, kFwdSmem, s>>>((const uint16_t*)x, (const uint16_t*)w, w_cl,
                                                          (uint16_t*)y, (int)H, (int)W, gm.OH, gm.OW, gm.nseg,
                                                          gm.units);
  return cudaGetLastError();
}

cudaError_t launch_stem_conv_wgrad(const void* x, const void* dy, float* ws, int partials, void* dw, bool w_cl,
                                   int64_t N, int64_t H, int64_t W, cudaStream_t s) {
  const Geometry gm = geometry(N, H, W);
  if (partials < 1 || partials > gm.units) return cudaErrorInvalidValue;
  stem_conv_wgrad_kernel<<<partials, kWgThreads, kWgSmem, s>>>((const uint16_t*)x, (const uint16_t*)dy, ws, (int)H,
                                                              (int)W, gm.OH, gm.OW, gm.nseg, gm.units);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return e;
  stem_conv_wgrad_reduce_kernel<<<(kCo * kK + kReduceThreads - 1) / kReduceThreads, kReduceThreads, 0, s>>>(
      ws, partials, (uint16_t*)dw, w_cl);
  return cudaGetLastError();
}

}  // namespace bps
