// pybind11 surface of the labelled-row gather of the masked-LM head (kernels/mlm_gather.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <cstdint>
#include <initializer_list>
#include <stdexcept>
#include <string>
#include <utility>

#include "bind/cuda_bind_ext.h"
#include "kernels/mlm_gather.cuh"
#include "kernels/pushpull.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

// bytes of one row of H elements of dtype, after checking the sizes
size_t row_bytes(int dtype, int64_t T, int64_t H, int64_t C) {
  size_t elem = 0;
  if (dtype == WIRE_F32) elem = 4;
  if (dtype == WIRE_BF16 || dtype == WIRE_F16) elem = 2;
  if (elem == 0) throw std::invalid_argument("mlm_gather: dtype must be WIRE_F32, WIRE_BF16 or WIRE_F16");
  if (T < 1 || T > INT32_MAX)
    throw std::invalid_argument("mlm_gather: token count must be in [1, 2^31 - 1], got " + std::to_string(T));
  if (C < 1 || C > INT32_MAX)
    throw std::invalid_argument("mlm_gather: capacity must be in [1, 2^31 - 1], got " + std::to_string(C));
  if (H < 1 || (H * elem) % 16 != 0)
    throw std::invalid_argument("mlm_gather: a row must be a positive multiple of 16 bytes, got H = " +
                                std::to_string(H));
  return (size_t)H * elem;
}

void check_ptrs(std::initializer_list<std::pair<uintptr_t, uintptr_t>> ptrs) {
  for (auto& pa : ptrs)
    if (pa.first == 0 || pa.first % pa.second != 0)
      throw std::invalid_argument("mlm_gather: null or misaligned pointer (need " + std::to_string(pa.second) +
                                  "-byte alignment)");
}
}  // namespace

void bind_cuda_mlm(py::module_& m) {
  m.def("mlm_gather_fwd", [](uintptr_t x, uintptr_t labels, int dtype, int64_t T, int64_t H, int64_t C,
                             int64_t ignore_index, uintptr_t rows, uintptr_t row_labels, uintptr_t slot,
                             uintptr_t src, uintptr_t dropped, uintptr_t s) {
    const size_t rb = row_bytes(dtype, T, H, C);
    check_ptrs({{x, 16}, {rows, 16}, {labels, 8}, {row_labels, 8}, {dropped, 8}, {slot, 4}, {src, 4}});
    chk(launch_mlm_gather_fwd((const void*)x, (const int64_t*)labels, (size_t)T, rb, C, ignore_index, (void*)rows,
                              (int64_t*)row_labels, (int32_t*)slot, (int32_t*)src, (int64_t*)dropped,
                              (cudaStream_t)s),
        "mlm_gather_fwd");
  }, py::arg("x"), py::arg("labels"), py::arg("dtype"), py::arg("T"), py::arg("H"), py::arg("C"),
     py::arg("ignore_index"), py::arg("rows"), py::arg("row_labels"), py::arg("slot"), py::arg("src"),
     py::arg("dropped"), py::arg("stream"),
     "rows [C, H] = the rows of x [T, H] whose int64 label is not ignore_index, in token order, the first C of them "
     "(zeros past the labelled count); row_labels [C] their labels (ignore_index when empty); slot int32 [T] each "
     "token's slot or -1; src int32 [C] workspace; dropped: int64 count of labelled tokens past C");
  m.def("mlm_scatter_bwd", [](uintptr_t drows, uintptr_t slot, int dtype, int64_t T, int64_t H, int64_t C,
                              uintptr_t dx, uintptr_t s) {
    const size_t rb = row_bytes(dtype, T, H, C);
    check_ptrs({{drows, 16}, {dx, 16}, {slot, 4}});
    chk(launch_mlm_scatter_bwd((const void*)drows, (const int32_t*)slot, (size_t)T, rb, C, (void*)dx,
                               (cudaStream_t)s),
        "mlm_scatter_bwd");
  }, py::arg("drows"), py::arg("slot"), py::arg("dtype"), py::arg("T"), py::arg("H"), py::arg("C"), py::arg("dx"),
     py::arg("stream"), "dx [T, H] = drows[slot[t]], zeros where slot[t] = -1; every element is written");
}
