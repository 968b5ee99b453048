// Gather of the labelled rows of a [T, H] activation into C fixed slots, and the scatter of their gradient back
// (two launches forward, one backward).  Rows are copied as raw 16-byte vectors, so the element type only sets the
// row's byte width: row_bytes = H * sizeof(element) must be a multiple of 16 and every row base 16-byte aligned.
// Offsets are 64-bit.  Nothing is read on the host and no launch depends on the labelled count, so both directions
// capture into a CUDA graph; results are bit-identical copies, with no atomics.
//
//   fwd   scan   one CTA walks labels [T] in tiles with a carried prefix.  Token t with labels[t] != ignore_index is
//                the n-th labelled token in token order; it gets slot n if n < C, else -1 (dropped).  Writes slot[T]
//                (int32, -1 for tokens not kept), src[C] (int32 source token of each slot, -1 for an empty slot),
//                row_labels[C] (ignore_index for an empty slot) and *dropped = max(0, labelled - C) (int64).
//         copy   rows[j, :] = x[src[j], :], zeros for an empty slot.
//   bwd   dx[t, :] = drows[slot[t], :], zeros where slot[t] = -1.  Every element of dx is written.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace bps {

cudaError_t launch_mlm_gather_fwd(const void* x, const int64_t* labels, size_t T, size_t row_bytes, int64_t C,
                                  int64_t ignore_index, void* rows, int64_t* row_labels, int32_t* slot, int32_t* src,
                                  int64_t* dropped, cudaStream_t s);
cudaError_t launch_mlm_scatter_bwd(const void* drows, const int32_t* slot, size_t T, size_t row_bytes, int64_t C,
                                   void* dx, cudaStream_t s);

}  // namespace bps
