// pybind11 surface of the FP8 cast kernels (kernels/fp8.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/fp8.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void bind_cuda_fp8(py::module_& m) {
  m.attr("FP8_E4M3") = (int)FP8_E4M3;
  m.attr("FP8_E5M2") = (int)FP8_E5M2;
  m.attr("FP8_ROWS") = (int)FP8_ROWS;
  m.attr("FP8_COLS") = (int)FP8_COLS;
  m.attr("FP8_BOTH") = (int)FP8_BOTH;
  m.attr("FP8_HISTORY") = kFp8History;
  m.attr("FP8_STATE_BYTES") = (int)sizeof(Fp8State);
  m.def("fp8_cast_workspace", [](size_t M, int K, int dtype, int fmt, int layout, bool dbias) {
    size_t floats;
    int counters;
    fp8_cast_workspace(M, K, dtype, fmt, layout, dbias, &floats, &counters);
    return py::make_tuple(floats, counters);
  }, py::arg("M"), py::arg("K"), py::arg("dtype"), py::arg("fmt"), py::arg("layout"), py::arg("dbias"),
     "(fp32 workspace floats, zeroed uint32 counters) of one fp8_cast launch");
  m.def("fp8_amax_workspace", [](size_t M, int K, int dtype) {
    size_t floats;
    int counters;
    fp8_amax_workspace(M, K, dtype, &floats, &counters);
    return py::make_tuple(floats, counters);
  }, py::arg("M"), py::arg("K"), py::arg("dtype"),
     "(fp32 workspace floats, zeroed uint32 counters) of one fp8_amax launch");

  m.def("fp8_amax", [](uintptr_t x, int dtype, size_t M, int K, int fmt, uintptr_t state, uintptr_t ws,
                       uintptr_t counters, uintptr_t s) {
    chk(launch_fp8_amax((const void*)x, dtype, M, K, fmt, (Fp8State*)state, (float*)ws, (uint32_t*)counters,
                        (cudaStream_t)s),
        "fp8_amax");
  }, py::arg("x"), py::arg("dtype"), py::arg("M"), py::arg("K"), py::arg("fmt"), py::arg("state"), py::arg("ws"),
     py::arg("counters"), py::arg("stream"), "seed a delayed-scaling state from max |x|");
  m.def("fp8_cast", [](uintptr_t x, int dtype, size_t M, int K, int fmt, int layout, uintptr_t state,
                       uintptr_t out_rows, uintptr_t out_cols, uintptr_t inv, uintptr_t dbias, uintptr_t ws,
                       uintptr_t counters, uintptr_t s) {
    chk(launch_fp8_cast((const void*)x, dtype, M, K, fmt, layout, (Fp8State*)state, (void*)out_rows,
                        (void*)out_cols, (float*)inv, (void*)dbias, (float*)ws, (uint32_t*)counters,
                        (cudaStream_t)s),
        "fp8_cast");
  }, py::arg("x"), py::arg("dtype"), py::arg("M"), py::arg("K"), py::arg("fmt"), py::arg("layout"), py::arg("state"),
     py::arg("out_rows"), py::arg("out_cols"), py::arg("inv"), py::arg("dbias"), py::arg("ws"), py::arg("counters"),
     py::arg("stream"),
     "FP8 copies of x (rows, transposed or both) at the state's scale, the inverse scale applied, the column sums "
     "of x (dbias != 0) and the state's next scale");
}
