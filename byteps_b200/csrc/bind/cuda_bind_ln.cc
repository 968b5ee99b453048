// pybind11 surface of the fused dropout / residual add / LayerNorm kernels (kernels/ln.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/ln.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void bind_cuda_ln(py::module_& m) {
  m.def("ln_workspace", [](size_t M, int H) {
    return py::make_tuple(ln_workspace_floats(M, H), ln_counters(M, H));
  }, py::arg("M"), py::arg("H"), "(fp32 workspace floats, zeroed uint32 counters) of one ln_bwd launch at (M, H)");

  m.def("ln_fwd", [](uintptr_t y, uintptr_t residual, int dtype, int wdtype, size_t M, int H, float eps,
                     uintptr_t gamma, uintptr_t beta, uintptr_t seed, uint32_t keep, float scale, uintptr_t z,
                     uintptr_t out, uintptr_t mean, uintptr_t rstd, uintptr_t mask, uintptr_t s) {
    chk(launch_ln_fwd((const void*)y, (const void*)residual, dtype, wdtype, M, H, eps, (const void*)gamma,
                      (const void*)beta, (const int64_t*)seed, keep, scale, (void*)z, (void*)out, (float*)mean,
                      (float*)rstd, (uint8_t*)mask, (cudaStream_t)s),
        "ln_fwd");
  }, py::arg("y"), py::arg("residual"), py::arg("dtype"), py::arg("wdtype"), py::arg("M"), py::arg("H"),
     py::arg("eps"), py::arg("gamma"), py::arg("beta"), py::arg("seed"), py::arg("keep"), py::arg("scale"),
     py::arg("z"), py::arg("out"), py::arg("mean"), py::arg("rstd"), py::arg("mask"), py::arg("stream"),
     "z = residual + dropout(y) (residual, z and mask 0 when absent; seed: device int64 {seed, offset}), "
     "out = layer_norm(z); keep = (1 - p) * 2^32 and scale = 1 / (1 - p) when mask is given");
  m.def("ln_bwd", [](uintptr_t dout, uintptr_t z, uintptr_t mask, int dtype, int wdtype, size_t M, int H, float scale,
                     uintptr_t mean, uintptr_t rstd, uintptr_t gamma, uintptr_t dres, uintptr_t dy, uintptr_t dgamma,
                     uintptr_t dbeta, uintptr_t ws, uintptr_t counters, uintptr_t s) {
    chk(launch_ln_bwd((const void*)dout, (const void*)z, (const uint8_t*)mask, dtype, wdtype, M, H, scale,
                      (const float*)mean, (const float*)rstd, (const void*)gamma, (void*)dres, (void*)dy,
                      (void*)dgamma, (void*)dbeta, (float*)ws, (uint32_t*)counters, (cudaStream_t)s),
        "ln_bwd");
  }, py::arg("dout"), py::arg("z"), py::arg("mask"), py::arg("dtype"), py::arg("wdtype"), py::arg("M"), py::arg("H"),
     py::arg("scale"), py::arg("mean"), py::arg("rstd"), py::arg("gamma"), py::arg("dres"), py::arg("dy"),
     py::arg("dgamma"), py::arg("dbeta"), py::arg("ws"), py::arg("counters"), py::arg("stream"),
     "dres = dz and dy = dz * mask * scale (each 0 when not wanted), dgamma and dbeta in the parameter dtype");
}
