// Host-side TMA tensor-map encoding for the wgmma push-pull variant.
#include <cuda.h>
#include <cuda_runtime_api.h>

#include <cstring>

#include "kernels/pushpull.cuh"
#include "kernels/pushpull_umma.cuh"

namespace bps {

using EncodeFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                              const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                              CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeFn encode_fn() {
  static EncodeFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
        q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeFn>(p);
  }();
  return fn;
}

int encode_umma_maps(const PeerView& pv, int wire, size_t off, size_t nelem, UmmaMaps* out) {
  EncodeFn enc = encode_fn();
  if (!enc) return -1;
  if (pv.world > kUmmaMaxWorld || (wire != WIRE_BF16 && wire != WIRE_F16)) return -2;
  memset(out, 0, sizeof(*out));
  size_t b, e;
  shard_units((nelem + 7) / 8, pv.world, pv.rank, &b, &e);
  const size_t shard_elems = (e - b) * 8;
  const size_t shard_off = off + b * 8 * 2;
  const cuuint64_t rows = shard_elems ? (shard_elems + 63) / 64 : 1;
  for (int p = 0; p < pv.world; ++p) {
    cuuint64_t dims[2] = {64, rows};
    cuuint64_t strides[1] = {128};          // bytes between rows
    cuuint32_t box[2] = {64, 128};
    cuuint32_t estr[2] = {1, 1};
    CUresult r = enc(&out->m[p], wire == WIRE_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                     2, (void*)(pv.data[p] + shard_off), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return (int)r;
  }
  return 0;
}

}  // namespace bps
