// wgmma/TMA variant of the in-place push-pull (see pushpull_umma.cu).
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include "kernels/peer_view.h"

namespace bps {

constexpr int kUmmaMaxWorld = 8;

// One 2-D tensor map per peer: [rows][64 elems] 16-bit view of MY shard inside that peer's window,
// box 64 x 128, SWIZZLE_128B.
struct UmmaMaps {
  CUtensorMap m[kUmmaMaxWorld];
};

// Host: encode the maps for the window [off, off + nelem) of the arena described by pv.
// Returns 0 on success (CUresult otherwise; -1 if the driver entry point is missing).
int encode_umma_maps(const PeerView& pv, int wire, size_t off, size_t nelem, UmmaMaps* out);

size_t umma_smem_bytes();

// bf16/fp16 only; off must be 128-byte aligned; world <= 8.
cudaError_t launch_pushpull_inplace_umma(const PeerView& pv, const UmmaMaps& maps, int wire, size_t off, size_t nelem,
                                         float scale, int blocks, int channel, cudaStream_t stream);

}  // namespace bps
