// pybind11 surface of ResNet's stem convolution (kernels/stem_conv.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <cstdint>
#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/pushpull.cuh"
#include "kernels/stem_conv.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void check_shape(int dtype, int64_t N, int64_t H, int64_t W) {
  if (dtype != WIRE_BF16) throw std::invalid_argument("stem_conv: dtype must be WIRE_BF16");
  if (N < 1 || H < 1 || W < 1 || H > INT32_MAX / 2 || W > INT32_MAX / 2)
    throw std::invalid_argument("stem_conv: N, H and W must be in [1, 2^30], got " + std::to_string(N) + ", " +
                                std::to_string(H) + ", " + std::to_string(W));
  const int64_t oh = (H - 1) / 2 + 1;
  if (N > INT64_MAX / (oh * W * 64)) throw std::invalid_argument("stem_conv: tensor too large");
}

void check_ptr(uintptr_t p, uintptr_t align, const char* name) {
  if (p == 0 || p % align != 0)
    throw std::invalid_argument(std::string("stem_conv: ") + name + " is null or not " + std::to_string(align) +
                                "-byte aligned");
}
}  // namespace

void bind_cuda_stem(py::module_& m) {
  m.def("stem_conv_fwd", [](uintptr_t x, uintptr_t w, bool w_cl, uintptr_t y, int dtype, int64_t N, int64_t H,
                            int64_t W, uintptr_t s) {
    check_shape(dtype, N, H, W);
    check_ptr(x, 2, "x");
    check_ptr(w, 2, "w");
    check_ptr(y, 16, "y");
    chk(launch_stem_conv_fwd((const void*)x, (const void*)w, w_cl, (void*)y, N, H, W, (cudaStream_t)s),
        "stem_conv_fwd");
  }, py::arg("x"), py::arg("w"), py::arg("w_cl"), py::arg("y"), py::arg("dtype"), py::arg("N"), py::arg("H"),
     py::arg("W"), py::arg("stream"),
     "y [N, OH, OW, 64] = conv(x [N, H, W, 3], w [64, 3, 7, 7]), stride 2, padding 3; w channels_last if w_cl");
  m.def("stem_conv_wgrad_partials", [](int64_t N, int64_t H, int64_t W) {
    check_shape(WIRE_BF16, N, H, W);
    const int p = stem_conv_wgrad_partials(N, H, W);
    if (p < 1) throw std::runtime_error("stem_conv_wgrad_partials: occupancy query failed");
    return p;
  }, py::arg("N"), py::arg("H"), py::arg("W"),
     "P, the fp32 partials of [64, 147] the weight gradient's workspace holds on the current device");
  m.def("stem_conv_wgrad", [](uintptr_t x, uintptr_t dy, uintptr_t ws, int partials, uintptr_t dw, bool w_cl,
                              int dtype, int64_t N, int64_t H, int64_t W, uintptr_t s) {
    check_shape(dtype, N, H, W);
    check_ptr(x, 2, "x");
    check_ptr(dy, 16, "dy");
    check_ptr(ws, 16, "ws");
    check_ptr(dw, 2, "dw");
    if (partials != stem_conv_wgrad_partials(N, H, W))
      throw std::invalid_argument("stem_conv_wgrad: partials must equal stem_conv_wgrad_partials(N, H, W)");
    chk(launch_stem_conv_wgrad((const void*)x, (const void*)dy, (float*)ws, partials, (void*)dw, w_cl, N, H, W,
                               (cudaStream_t)s),
        "stem_conv_wgrad");
  }, py::arg("x"), py::arg("dy"), py::arg("ws"), py::arg("partials"), py::arg("dw"), py::arg("w_cl"),
     py::arg("dtype"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("stream"),
     "dw [64, 3, 7, 7] (w's layout) = sum over output pixels of dy [N, OH, OW, 64] x the patch of x [N, H, W, 3]; "
     "ws: fp32 workspace of partials x 64 x 147");
}
