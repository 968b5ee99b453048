// pybind11 surface of the fused self-attention kernels (kernels/attn.cu, attn_varlen.cu and attn_causal.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <initializer_list>
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

void check_varlen(int dtype, int T, int N, int H, int D, int max_seqlen, uintptr_t cu) {
  check_shape(dtype, 1, max_seqlen, H, D, ATTN_MASK_F32);
  if (T < 1) throw std::invalid_argument("attention: token count must be >= 1, got " + std::to_string(T));
  if (N < 1 || N > 65535)
    throw std::invalid_argument("attention: sequence count must be in [1, 65535], got " + std::to_string(N));
  if (cu == 0 || cu % 4 != 0) throw std::invalid_argument("attention: cu_seqlens must be a 4-byte aligned pointer");
}

void check_ptrs(std::initializer_list<uintptr_t> p16, std::initializer_list<uintptr_t> p4) {
  for (uintptr_t p : p16)
    if (p == 0 || p % 16 != 0) throw std::invalid_argument("attention: tensors must be non-null and 16-byte aligned");
  for (uintptr_t p : p4)
    if (p == 0 || p % 4 != 0) throw std::invalid_argument("attention: fp32 tensors must be non-null and aligned");
}
}  // namespace

void bind_cuda_attn(py::module_& m) {
  m.attr("ATTN_MASK_F32") = (int)ATTN_MASK_F32;
  m.attr("ATTN_MASK_BF16") = (int)ATTN_MASK_BF16;
  m.attr("ATTN_MASK_F16") = (int)ATTN_MASK_F16;
  m.attr("ATTN_MASK_BOOL") = (int)ATTN_MASK_BOOL;

  m.def("attn_fwd", [](uintptr_t qkv, int dtype, int B, int S, int H, int D, uintptr_t mask, int mask_kind,
                       int64_t mask_bstride, uintptr_t seed, uint32_t keep, float scale, uintptr_t out,
                       uintptr_t lse, uintptr_t s, bool causal) {
    check_shape(dtype, B, S, H, D, mask_kind);
    chk(launch_attn_fwd((const void*)qkv, dtype, B, S, H, D, (const void*)mask, mask_kind, mask_bstride,
                        (const int64_t*)seed, keep, scale, (void*)out, (float*)lse, (cudaStream_t)s, causal),
        "attn_fwd");
  }, py::arg("qkv"), py::arg("dtype"), py::arg("B"), py::arg("S"), py::arg("H"), py::arg("D"), py::arg("mask"),
     py::arg("mask_kind"), py::arg("mask_bstride"), py::arg("seed"), py::arg("keep"), py::arg("scale"),
     py::arg("out"), py::arg("lse"), py::arg("stream"), py::kw_only(), py::arg("causal") = false,
     "out = softmax(Q K^T / 8 + mask) -> dropout -> @ V from qkv [B, S, 3, H, 64]; lse fp32 [B, H, S]; mask 0 or one "
     "value per key (batch stride mask_bstride); seed 0 (no dropout) or device int64 {seed, offset} with keep = "
     "(1 - p) * 2^32 and scale = 1 / (1 - p); causal: key k attends to query q only when k <= q");
  m.def("attn_bwd", [](uintptr_t qkv, uintptr_t out, uintptr_t dout, uintptr_t lse, int dtype, int B, int S, int H,
                       int D, uintptr_t mask, int mask_kind, int64_t mask_bstride, uintptr_t seed, uint32_t keep,
                       float scale, uintptr_t delta, uintptr_t dqkv, uintptr_t s, bool causal) {
    check_shape(dtype, B, S, H, D, mask_kind);
    chk(launch_attn_bwd((const void*)qkv, (const void*)out, (const void*)dout, (const float*)lse, dtype, B, S, H, D,
                        (const void*)mask, mask_kind, mask_bstride, (const int64_t*)seed, keep, scale,
                        (float*)delta, (void*)dqkv, (cudaStream_t)s, causal),
        "attn_bwd");
  }, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("lse"), py::arg("dtype"), py::arg("B"), py::arg("S"),
     py::arg("H"), py::arg("D"), py::arg("mask"), py::arg("mask_kind"), py::arg("mask_bstride"), py::arg("seed"),
     py::arg("keep"), py::arg("scale"), py::arg("delta"), py::arg("dqkv"), py::arg("stream"), py::kw_only(),
     py::arg("causal") = false,
     "dqkv [B, S, 3, H, 64] of attn_fwd's output given dout; delta: fp32 [B, H, S] workspace; causal as for the "
     "forward");

  m.def("attn_varlen_fwd", [](uintptr_t qkv, int dtype, int T, int N, int H, int D, int max_seqlen,
                              uintptr_t cu_seqlens, uintptr_t seed, uint32_t keep, float scale, uintptr_t out,
                              uintptr_t lse, uintptr_t s, bool causal) {
    check_varlen(dtype, T, N, H, D, max_seqlen, cu_seqlens);
    check_ptrs({qkv, out}, {lse});
    chk(launch_attn_varlen_fwd((const void*)qkv, dtype, T, N, H, D, max_seqlen, (const int*)cu_seqlens,
                               (const int64_t*)seed, keep, scale, (void*)out, (float*)lse, (cudaStream_t)s, causal),
        "attn_varlen_fwd");
  }, py::arg("qkv"), py::arg("dtype"), py::arg("T"), py::arg("N"), py::arg("H"), py::arg("D"),
     py::arg("max_seqlen"), py::arg("cu_seqlens"), py::arg("seed"), py::arg("keep"), py::arg("scale"),
     py::arg("out"), py::arg("lse"), py::arg("stream"), py::kw_only(), py::arg("causal") = false,
     "out [T, E] = attention of qkv [T, 3, H, 64] within the N sequences of device int32 cu_seqlens [N + 1], "
     "each at most max_seqlen (<= 512) long; lse fp32 [H, T]; seed as for attn_fwd; causal: token u of a sequence "
     "attends to token t only when u <= t");
  m.def("attn_varlen_bwd", [](uintptr_t qkv, uintptr_t out, uintptr_t dout, uintptr_t lse, int dtype, int T, int N,
                              int H, int D, int max_seqlen, uintptr_t cu_seqlens, uintptr_t seed, uint32_t keep,
                              float scale, uintptr_t delta, uintptr_t dqkv, uintptr_t s, bool causal) {
    check_varlen(dtype, T, N, H, D, max_seqlen, cu_seqlens);
    check_ptrs({qkv, out, dout, dqkv}, {lse, delta});
    chk(launch_attn_varlen_bwd((const void*)qkv, (const void*)out, (const void*)dout, (const float*)lse, dtype, T,
                               N, H, D, max_seqlen, (const int*)cu_seqlens, (const int64_t*)seed, keep, scale,
                               (float*)delta, (void*)dqkv, (cudaStream_t)s, causal),
        "attn_varlen_bwd");
  }, py::arg("qkv"), py::arg("out"), py::arg("dout"), py::arg("lse"), py::arg("dtype"), py::arg("T"), py::arg("N"),
     py::arg("H"), py::arg("D"), py::arg("max_seqlen"), py::arg("cu_seqlens"), py::arg("seed"), py::arg("keep"),
     py::arg("scale"), py::arg("delta"), py::arg("dqkv"), py::arg("stream"), py::kw_only(), py::arg("causal") = false,
     "dqkv [T, 3, H, 64] of attn_varlen_fwd's output given dout; delta: fp32 [H, T] workspace; causal as for the "
     "forward");
}
