// Dynamic loss scaling on the device: the overflow check of the local gradient windows and the cross-rank
// agreement + scaler update (see loss_scale.cuh).  No host round trip, no float atomics: the decision is one
// integer OR per rank, merged in rank order, so every rank computes the same bits.
#include <math.h>

#include <type_traits>

#include "kernels/common.cuh"
#include "kernels/loss_scale.cuh"

namespace bps {
namespace {

constexpr int kCheckThreads = 256;

// Largest magnitude a gradient value on the wire may have (see kLossScaleSumLimit); a value above it, inf or NaN
// counts as an overflow.
__device__ __forceinline__ bool too_big(float v, float limit) { return !(fabsf(v) <= limit); }

// Does any element of one 16-byte vector of gradients (dtype G) overflow on a wire of dtype W?  Each element is
// rounded to the wire as the pack phase rounds it (to nearest even: an fp32 65520 becomes an fp16 inf, 65519.99
// becomes 65504) and compared as a float.
template <class G, class W>
__device__ __forceinline__ bool vec_overflows(const Vec16& v, float limit) {
  float f[G::kPerVec];
  G::unpack(v, f);
  bool bad = false;
#pragma unroll
  for (int k = 0; k < G::kPerVec; ++k) {
    float x = f[k];
    if constexpr (!std::is_same<G, W>::value) {
      if constexpr (std::is_same<W, TagF16>::value) x = __half2float(__float2half_rn(x));
      else x = __bfloat162float(__float2bfloat16_rn(x));
    }
    bad |= too_big(x, limit);
  }
  return bad;
}

template <class G, class W>
__device__ __forceinline__ bool scan(const char* base, size_t nvec, float limit) {
  bool bad = false;
  // plain cached loads: the exchange reads the same bytes right after this kernel
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < nvec; i += (size_t)gridDim.x * blockDim.x) {
    const uint4 u = *reinterpret_cast<const uint4*>(base + i * 16);
    bad |= vec_overflows<G, W>(Vec16{u.x, u.y, u.z, u.w}, limit);
  }
  return bad;
}

__global__ void __launch_bounds__(kCheckThreads) loss_scale_check_kernel(PeerView pv,
                                                                          const LossScaleCheckEntry* __restrict__ table,
                                                                          int nentries, LossScaleState* state) {
  const char* arena = pv.data[pv.rank];
  const float limit = kLossScaleSumLimit / (float)pv.world * fminf(1.f, state->scale);   // S of this step
  bool bad = false;
  for (int i = 0; i < nentries; ++i) {
    const LossScaleCheckEntry e = table[i];
    const char* base = arena + e.off;
    if (e.grad == WIRE_F32) {
      const size_t nvec = e.n / 4;
      if (e.wire == WIRE_F32) bad |= scan<TagF32, TagF32>(base, nvec, limit);
      else if (e.wire == WIRE_BF16) bad |= scan<TagF32, TagBF16>(base, nvec, limit);
      else bad |= scan<TagF32, TagF16>(base, nvec, limit);
    } else if (e.grad == WIRE_BF16) {
      bad |= scan<TagBF16, TagBF16>(base, e.n / 8, limit);
    } else {
      bad |= scan<TagF16, TagF16>(base, e.n / 8, limit);
    }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicOr(&state->found, 1u);
}

// The agreement window of rank r: flags [parity][source rank] at win_off.  The block works in parity g & 1, g being
// its barrier generation in device memory.  A peer block can be at most one participation ahead (to pass barrier
// g + 1 it needs this block there, which this rank's stream starts only after this launch has finished), so a peer
// writing parity (g + 1) & 1 can overlap this block's reads of parity g & 1, and nothing writes parity g & 1 again
// before those reads are done.  Every launch on the stream advances the generation, not only this kernel's, which
// does not change the argument.
__global__ void __launch_bounds__(32) loss_scale_update_kernel(PeerView pv, int channel, size_t win_off,
                                                               LossScaleState* state, int32_t* steps,
                                                               const double* betas, OptHParams* hp, int ngroups,
                                                               int adam) {
  const int W = pv.world, me = pv.rank;
  const uint32_t par = pv.epoch[channel * kMaxBlocks + blockIdx.x] & 1u;
  const uint32_t flag = *(volatile uint32_t*)&state->found;
  if (threadIdx.x < W) {
    uint32_t* dst = reinterpret_cast<uint32_t*>(pv.data[threadIdx.x] + win_off) + par * kMaxRanks + me;
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(dst), "r"(flag) : "memory");
  }
  barrier_peers(pv, channel);
  if (threadIdx.x != 0) return;
  const uint32_t* win = reinterpret_cast<const uint32_t*>(pv.data[me] + win_off) + par * kMaxRanks;
  uint32_t found = 0;
  for (int r = 0; r < W; ++r) found |= *(volatile const uint32_t*)&win[r];
  found = found != 0;

  LossScaleState s = *state;
  const float applied_scale = s.scale;      // what this step's loss was multiplied by
  // torch._amp_update_scale_: products in double, rounded once to the float scale
  if (found) {
    s.scale = (float)((double)s.scale * s.backoff);
    s.tracker = 0;
    s.skipped += 1;
  } else {
    const int32_t successful = s.tracker + 1;
    if (successful == s.interval) {
      const float grown = (float)((double)s.scale * s.growth);
      if (isfinite(grown)) s.scale = grown;
      s.tracker = 0;
    } else {
      s.tracker = successful;
    }
  }
  s.found = 0;
  *state = s;

  const float grad_scale = (float)(1.0 / (double)applied_scale);
  for (int g = 0; g < ngroups; ++g) {
    const int32_t t = steps[g] + 1;          // the step this launch applies (or skips)
    if (!found) steps[g] = t;
    OptHParams& h = hp[g];
    h.grad_scale = grad_scale;
    h.skip = (int)found;
    h.first_step = t == 1;
    if (adam) {
      // 1 - beta^t in float64 from the host's float64 betas, rounded once (what refresh_hparams computes)
      h.bias_c1 = (float)(1.0 - pow(betas[2 * g], (double)t));
      h.bias_c2 = (float)(1.0 - pow(betas[2 * g + 1], (double)t));
    }
  }
}

// one wave of resident blocks at most (the occupancy of this kernel on this device), fewer when the largest window
// has fewer vectors
int check_grid(size_t max_vectors) {
  static int wave = 0;
  if (wave == 0) {
    int dev = 0, sms = 0, per_sm = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, loss_scale_check_kernel, kCheckThreads, 0);
    wave = (sms > 0 ? sms : 1) * (per_sm > 0 ? per_sm : 1);
  }
  const size_t need = (max_vectors + kCheckThreads - 1) / kCheckThreads;
  return (int)(need < 1 ? 1 : (need < (size_t)wave ? need : (size_t)wave));
}

}  // namespace

cudaError_t launch_loss_scale_check(const PeerView& pv, const LossScaleCheckEntry* table, int nentries,
                                    size_t max_vectors, LossScaleState* state, cudaStream_t stream) {
  if (nentries < 1 || table == nullptr || state == nullptr) return cudaErrorInvalidValue;
  loss_scale_check_kernel<<<check_grid(max_vectors), kCheckThreads, 0, stream>>>(pv, table, nentries, state);
  return cudaGetLastError();
}

cudaError_t launch_loss_scale_update(const PeerView& pv, int channel, size_t win_off, LossScaleState* state,
                                     int32_t* steps, const double* betas, OptHParams* hp, int ngroups, int adam,
                                     cudaStream_t stream) {
  if (pv.world < 1 || pv.world > kMaxRanks || channel < 0 || channel > 1 || (win_off & 15) || state == nullptr ||
      steps == nullptr || hp == nullptr || ngroups < 1 || (adam && betas == nullptr))
    return cudaErrorInvalidValue;
  // one block, always block 0: barrier_peers pairs CTAs by index, so every rank meets in the same CTA
  loss_scale_update_kernel<<<1, 32, 0, stream>>>(pv, channel, win_off, state, steps, betas, hp, ngroups, adam);
  return cudaGetLastError();
}

cudaError_t loss_scale_load_kernels() {
  cudaFuncAttributes a;
  cudaError_t e = cudaFuncGetAttributes(&a, (const void*)loss_scale_check_kernel);
  if (e == cudaSuccess) e = cudaFuncGetAttributes(&a, (const void*)loss_scale_update_kernel);
  return e;
}

}  // namespace bps
