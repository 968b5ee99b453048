// pybind11 surface of the fused self-attention kernels (kernels/attn.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/attn.cuh"
#include "kernels/pushpull.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void check_shape(int dtype, int B, int S, int H, int D, int mask_kind) {
  if (dtype != WIRE_BF16 && dtype != WIRE_F16)
    throw std::invalid_argument("attention: dtype must be WIRE_BF16 or WIRE_F16, got " + std::to_string(dtype));
  if (D != kAttnHeadDim) throw std::invalid_argument("attention: head dimension must be 64, got " + std::to_string(D));
  if (S < 1 || S > kAttnMaxSeq)
    throw std::invalid_argument("attention: sequence length must be in [1, 512], got " + std::to_string(S));
  if (B < 1 || B > 65535 || H < 1 || H > 65535)
    throw std::invalid_argument("attention: batch and heads must be in [1, 65535]");
  if (mask_kind < ATTN_MASK_F32 || mask_kind > ATTN_MASK_BOOL)
    throw std::invalid_argument("attention: unknown mask kind " + std::to_string(mask_kind));
}
}  // namespace

void bind_cuda_attn(py::module_& m) {
  m.attr("ATTN_MASK_F32") = (int)ATTN_MASK_F32;
  m.attr("ATTN_MASK_BF16") = (int)ATTN_MASK_BF16;
  m.attr("ATTN_MASK_F16") = (int)ATTN_MASK_F16;
  m.attr("ATTN_MASK_BOOL") = (int)ATTN_MASK_BOOL;

  m.def("attn_fwd", [](uintptr_t qkv, int dtype, int B, int S, int H, int D, uintptr_t mask, int mask_kind,
                       int64_t mask_bstride, uintptr_t seed, uint32_t keep, float scale, uintptr_t out,
                       uintptr_t lse, uintptr_t s) {
    check_shape(dtype, B, S, H, D, mask_kind);
    chk(launch_attn_fwd((const void*)qkv, dtype, B, S, H, D, (const void*)mask, mask_kind, mask_bstride,
                        (const int64_t*)seed, keep, scale, (void*)out, (float*)lse, (cudaStream_t)s),
        "attn_fwd");
  }, py::arg("qkv"), py::arg("dtype"), py::arg("B"), py::arg("S"), py::arg("H"), py::arg("D"), py::arg("mask"),
     py::arg("mask_kind"), py::arg("mask_bstride"), py::arg("seed"), py::arg("keep"), py::arg("scale"),
     py::arg("out"), py::arg("lse"), py::arg("stream"),
     "out = softmax(Q K^T / 8 + mask) -> dropout -> @ V from qkv [B, S, 3, H, 64]; lse fp32 [B, H, S]; mask 0 or one "
     "value per key (batch stride mask_bstride); seed 0 (no dropout) or device int64 {seed, offset} with keep = "
     "(1 - p) * 2^32 and scale = 1 / (1 - p)");
  m.def("attn_bwd", [](uintptr_t qkv, uintptr_t out, uintptr_t dout, uintptr_t lse, int dtype, int B, int S, int H,
                       int D, uintptr_t mask, int mask_kind, int64_t mask_bstride, uintptr_t seed, uint32_t keep,
                       float scale, uintptr_t delta, uintptr_t dqkv, uintptr_t s) {
    check_shape(dtype, B, S, H, D, mask_kind);
    chk(launch_attn_bwd((const void*)qkv, (const void*)out, (const void*)dout, (const float*)lse, dtype, B, S, H, D,
                        (const void*)mask, mask_kind, mask_bstride, (const int64_t*)seed, keep, scale,
                        (float*)delta, (void*)dqkv, (cudaStream_t)s),
        "attn_bwd");
  }, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("lse"), py::arg("dtype"), py::arg("B"), py::arg("S"),
     py::arg("H"), py::arg("D"), py::arg("mask"), py::arg("mask_kind"), py::arg("mask_bstride"), py::arg("seed"),
     py::arg("keep"), py::arg("scale"), py::arg("delta"), py::arg("dqkv"), py::arg("stream"),
     "dqkv [B, S, 3, H, 64] of attn_fwd's output given dout; delta: fp32 [B, H, S] workspace");
}
