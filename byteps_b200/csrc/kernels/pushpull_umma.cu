// wgmma / TMA variant of the in-place push-pull (16-bit wire types).
//
// Idea: the sum over peers IS a GEMM.  View a peer's slice of my shard as a
// matrix X_p[128 rows][64 elems]; stack the peers along K:
//
//     D[128 x 64] (fp32, registers)  =  [ I | I | ... | I ] (128 x 128*P)  x  [ X_0 ; X_1 ; ... ; X_{P-1} ] (128*P x 64)
//
// The B operand is exactly what a 2-D TMA load with SWIZZLE_128B drops into
// shared memory (MN-major canonical layout: 64 contiguous elements per K row,
// 8-row swizzle atoms, SBO = 1024 B), so the NVLink traffic goes
// peer HBM -> TMA -> smem -> tensor core without touching a register.  The A
// operand is the identity, passed as wgmma register fragments: the 64-row
// M half h and the 16-row K slice j only meet on the diagonal (j = 4 h + warp),
// so one warp of the warpgroup holds a 16 x 16 identity and the other three
// hold zeros.  The tensor pipe does the bf16->fp32 conversion and the fp32
// accumulation; the CUDA cores only run the epilogue: scale the fp32 tile,
// pack to 16 bit, stage in smem, bulk-store to every peer.
//
// Warp roles (160 threads, 1 CTA/SM): warps 0-3 = the consumer warpgroup
// (wgmma + epilogue), warp 4 = TMA producer.
#include <cuda.h>

#include "kernels/common.cuh"
#include "kernels/pushpull.cuh"
#include "kernels/pushpull_umma.cuh"

namespace bps {

namespace {

constexpr int kRows = 128;                       // tile rows = K rows per peer = 2 x wgmma M (64)
constexpr int kCols = 64;                        // wgmma N = elements per row (128 B of 16-bit data)
constexpr int kTileElems = kRows * kCols;        // 8192 elements
constexpr int kTileBytes = kTileElems * 2;       // 16 KiB per peer per tile
constexpr int kSlots = 6;                        // ring of peer tiles in flight per CTA
constexpr int kConsumerThreads = 128;            // one warpgroup
constexpr int kThreadsUmma = kConsumerThreads + 32;

struct UmmaSmem {
  uint64_t full[kSlots];
  uint64_t empty[kSlots];
};

// smem layout: [UmmaSmem | pad to 1024][ring: kSlots x 16 KiB (1024-aligned)][out: 16 KiB]
constexpr size_t kSmemHeader = 1024;
constexpr size_t kSmemRing = kSmemHeader;
constexpr size_t kSmemOut = kSmemRing + (size_t)kSlots * kTileBytes;
constexpr size_t kSmemTotal = kSmemOut + kTileBytes + 1024;   // + slack for manual 1024 alignment

__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* map, int c0, int c1, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::
          "r"(smem_u32(smem_dst)),
      "l"(map), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}

// sm_90 matrix descriptor, MN-major, SWIZZLE_128B: 64 contiguous elements per K row, 8-row atoms of 1024 B
__device__ __forceinline__ uint64_t make_desc_b(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFF) >> 4);                 // start address
  d |= (uint64_t)1 << 16;                                  // LBO unused (single atom along N)
  d |= (uint64_t)((1024u >> 4) & 0x3FFF) << 32;            // SBO = 1024 B between 8-row groups along K
  d |= (uint64_t)1 << 62;                                  // layout type 1 = SWIZZLE_128B
  return d;
}

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 64] (+)= A[64 x 16] (registers) x B[16 x 64] (smem, MN-major: imm-trans-b = 1)
template <bool BF16>
__device__ __forceinline__ void wgmma_m64n64k16(float* d, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3,
                                                uint64_t desc_b, uint32_t accumulate) {
#define BPS_WGMMA_ASM(TYPE)                                                                                          \
  asm volatile(                                                                                                      \
      "{\n\t"                                                                                                        \
      ".reg .pred p;\n\t"                                                                                            \
      "setp.ne.b32 p, %37, 0;\n\t"                                                                                   \
      "wgmma.mma_async.sync.aligned.m64n64k16.f32." TYPE "." TYPE " "                                               \
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28," \
      "%29,%30,%31}, {%32,%33,%34,%35}, %36, p, 1, 1, 1;\n\t"                                                        \
      "}"                                                                                                            \
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),             \
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),       \
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),     \
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])      \
      : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(desc_b), "r"(accumulate)                                            \
      : "memory")
  if (BF16)
    BPS_WGMMA_ASM("bf16");
  else
    BPS_WGMMA_ASM("f16");
#undef BPS_WGMMA_ASM
}

template <bool BF16>
__global__ void __launch_bounds__(kThreadsUmma, 1)
    pushpull_inplace_umma_kernel(PeerView pv, const __grid_constant__ UmmaMaps maps, size_t off, size_t total_groups,
                                 float scale, int channel) {
  extern __shared__ unsigned char smem_dyn[];
  // manual 1024-byte alignment (SWIZZLE_128B atoms)
  unsigned char* smem = reinterpret_cast<unsigned char*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
  UmmaSmem* sm = reinterpret_cast<UmmaSmem*>(smem);
  unsigned char* ring = smem + kSmemRing;
  unsigned char* out_smem = smem + kSmemOut;
  const int world = pv.world;
  // warp index broadcast from lane 0: provably warp-uniform, so the role branches below are not divergent paths
  // in which ptxas would have to serialize the wgmma instructions
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;

  size_t b, e;
  shard_units(total_groups, world, pv.rank, &b, &e);
  const size_t shard_elems = (e - b) * 8;                      // my shard, elements
  const size_t shard_off = off + b * 8 * 2;                    // byte offset of my shard in every window
  const size_t ntiles = (shard_elems + kTileElems - 1) / kTileElems;

  // ---- one-time setup
  if (threadIdx.x == 0) {
    for (int s = 0; s < kSlots; ++s) {
      mbar_init(&sm->full[s], 1);
      mbar_init(&sm->empty[s], kConsumerThreads / 32);        // one arrival per consumer warp
    }
    mbar_fence_init();
  }
  barrier_peers(pv, channel);        // __syncthreads inside: setup done AND every peer's input is ready
  fence_proxy_async();

  if (warp == kConsumerThreads / 32) {
    // ===== TMA producer
    if (lane == 0) {
      int s = 0;
      uint32_t phase = 0;
      for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
        for (int p = 0; p < world; ++p) {
          mbar_wait(&sm->empty[s], phase ^ 1);
          mbar_arrive_expect_tx(&sm->full[s], kTileBytes);
          tma_load_2d(ring + (size_t)s * kTileBytes, &maps.m[p], 0, (int)(t * kRows), &sm->full[s]);
          if (++s == kSlots) {
            s = 0;
            phase ^= 1;
          }
        }
      }
    }
  } else {
    // ===== consumer warpgroup: wgmma into two 64 x 64 fp32 accumulators (rows 0-63 / 64-127 of the tile),
    // then registers -> 16-bit -> smem -> bulk store to every peer
    const int g = lane >> 2, q = lane & 3;
    // identity fragment of this thread: a0 = a3 = (row g, cols 2q, 2q+1), a1 = a2 = 0
    const uint32_t one = BF16 ? 0x3F80u : 0x3C00u;
    const uint32_t ident = (g == 2 * q ? one : 0u) | ((g == 2 * q + 1 ? one : 0u) << 16);
    int s = 0;
    uint32_t phase = 0;
    for (size_t t = blockIdx.x; t < ntiles; t += gridDim.x) {
      float acc[2][32];
      for (int p = 0; p < world; ++p) {
        mbar_wait(&sm->full[s], phase);
        const uint32_t b_base = smem_u32(ring + (size_t)s * kTileBytes);
        wgmma_fence();
#pragma unroll
        for (int h = 0; h < 2; ++h) {
#pragma unroll
          for (int w = 0; w < 4; ++w) {                       // K slice j = 4 h + w of this peer's 128 rows
            const uint32_t a = warp == w ? ident : 0u;
            wgmma_m64n64k16<BF16>(acc[h], a, 0u, 0u, a, make_desc_b(b_base + (4 * h + w) * 16 * 128),
                                  (p | w) != 0);
          }
        }
        wgmma_commit();
        wgmma_wait_all();
        if (lane == 0) mbar_arrive(&sm->empty[s]);            // slot reusable: this warp's MMAs have retired
        if (++s == kSlots) {
          s = 0;
          phase ^= 1;
        }
      }
      // the previous tile's bulk stores must have finished reading out_smem
      if (threadIdx.x == 0) bulk_wait_read<0>();
      named_bar_sync(1, kConsumerThreads);
      // accumulator layout: acc[h][4c + i] = row 64 h + 16 warp + g + 8 (i >> 1), column 8 c + 2 q + (i & 1)
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        unsigned char* row0 = out_smem + (size_t)(64 * h + 16 * warp + g) * 128 + q * 4;
#pragma unroll
        for (int c = 0; c < 8; ++c) {
          const float* v = &acc[h][4 * c];
          const uint32_t lo = BF16 ? f2_to_bf16x2(v[0] * scale, v[1] * scale) : f2_to_f16x2(v[0] * scale, v[1] * scale);
          const uint32_t hi = BF16 ? f2_to_bf16x2(v[2] * scale, v[3] * scale) : f2_to_f16x2(v[2] * scale, v[3] * scale);
          *reinterpret_cast<uint32_t*>(row0 + c * 16) = lo;
          *reinterpret_cast<uint32_t*>(row0 + 8 * 128 + c * 16) = hi;
        }
      }
      fence_proxy_async_smem();
      named_bar_sync(1, kConsumerThreads);
      if (threadIdx.x == 0) {
        const size_t done = t * (size_t)kTileElems;
        const size_t left = shard_elems - done;
        const uint32_t bytes = (uint32_t)((left < (size_t)kTileElems ? left : (size_t)kTileElems) * 2);
        for (int j = 0; j < world; ++j) {
          int p = j + pv.rank;
          if (p >= world) p -= world;
          bulk_s2g(pv.data[p] + shard_off + done * 2, out_smem, bytes);
        }
        bulk_commit();
      }
    }
    if (threadIdx.x == 0) {
      bulk_wait<0>();
      fence_proxy_async();
    }
  }
  barrier_peers(pv, channel);
}

}  // namespace

size_t umma_smem_bytes() { return kSmemTotal; }

cudaError_t launch_pushpull_inplace_umma(const PeerView& pv, const UmmaMaps& maps, int wire, size_t off, size_t nelem,
                                         float scale, int blocks, int channel, cudaStream_t stream) {
  if (blocks < 1 || blocks > kMaxBlocks || (off & 127)) return cudaErrorInvalidValue;
  if (wire != WIRE_BF16 && wire != WIRE_F16) return cudaErrorInvalidValue;
  const size_t groups = (nelem + 7) / 8;
  cudaError_t err;
  if (wire == WIRE_BF16) {
    err = cudaFuncSetAttribute(pushpull_inplace_umma_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)kSmemTotal);
    if (err != cudaSuccess) return err;
    pushpull_inplace_umma_kernel<true><<<blocks, kThreadsUmma, kSmemTotal, stream>>>(pv, maps, off, groups, scale,
                                                                                     channel);
  } else {
    err = cudaFuncSetAttribute(pushpull_inplace_umma_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)kSmemTotal);
    if (err != cudaSuccess) return err;
    pushpull_inplace_umma_kernel<false><<<blocks, kThreadsUmma, kSmemTotal, stream>>>(pv, maps, off, groups, scale,
                                                                                      channel);
  }
  return cudaGetLastError();
}

}  // namespace bps
