// pybind11 surface of the softmax cross-entropy kernels (kernels/xent.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/xent.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void bind_cuda_xent(py::module_& m) {
  m.attr("XENT_NONE") = (int)XENT_NONE;
  m.attr("XENT_SUM") = (int)XENT_SUM;
  m.attr("XENT_MEAN") = (int)XENT_MEAN;
  m.def("xent_workspace", [](size_t M) { return py::make_tuple(xent_workspace_floats(M), xent_counters(M)); },
        py::arg("M"), "(fp32 workspace floats, zeroed uint32 counters) of one xent_fwd launch over M rows");

  m.def("xent_fwd", [](uintptr_t logits, uintptr_t target, int dtype, size_t M, int V, int64_t ignore_index,
                       bool mean, uintptr_t lse, uintptr_t loss_rows, uintptr_t out, uintptr_t count, uintptr_t ws,
                       uintptr_t counters, uintptr_t s) {
    chk(launch_xent_fwd((const void*)logits, (const int64_t*)target, dtype, M, V, ignore_index, mean, (float*)lse,
                        (float*)loss_rows, (float*)out, (int64_t*)count, (float*)ws, (uint32_t*)counters,
                        (cudaStream_t)s),
        "xent_fwd");
  }, py::arg("logits"), py::arg("target"), py::arg("dtype"), py::arg("M"), py::arg("V"), py::arg("ignore_index"),
     py::arg("mean"), py::arg("lse"), py::arg("loss_rows"), py::arg("out"), py::arg("count"), py::arg("ws"),
     py::arg("counters"), py::arg("stream"),
     "per-row lse and loss, the count of rows not ignored (int64) and their loss sum (divided by the count when "
     "mean) in out");
  m.def("xent_bwd", [](uintptr_t logits, uintptr_t target, int dtype, size_t M, int V, int64_t ignore_index,
                       uintptr_t lse, uintptr_t grad, int mode, uintptr_t count, uintptr_t dlogits, uintptr_t s) {
    chk(launch_xent_bwd((const void*)logits, (const int64_t*)target, dtype, M, V, ignore_index, (const float*)lse,
                        (const float*)grad, mode, (const int64_t*)count, (void*)dlogits, (cudaStream_t)s),
        "xent_bwd");
  }, py::arg("logits"), py::arg("target"), py::arg("dtype"), py::arg("M"), py::arg("V"), py::arg("ignore_index"),
     py::arg("lse"), py::arg("grad"), py::arg("mode"), py::arg("count"), py::arg("dlogits"), py::arg("stream"),
     "dlogits = g * (softmax - onehot) in the logits dtype, g = grad[i] (XENT_NONE), grad[0] (XENT_SUM) or "
     "grad[0] / count (XENT_MEAN)");
}
