// pybind11 surface of the LARS kernels of the fused exchange (kernels/pushpull_lars.cu).  The (start, numel) table,
// the scratch and the window have LAMB's layout: size them with lamb_scratch_bytes / lamb_window_bytes.
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/pushpull_lars.cuh"

namespace py = pybind11;
using namespace bps;

static void chk_lars(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void bind_cuda_lars(py::module_& m) {
  m.def(
      "lars_norms_partial",
      [](const PeerView& pv, int grad_dtype, int wire, uintptr_t segs, int nsegs, size_t stage_off, size_t total_elems,
         float scale, uintptr_t master, uintptr_t params, int nparams, uintptr_t scratch, uintptr_t hp, int blocks,
         int threads, int channel, bool nvls, uintptr_t stream) {
        chk_lars(launch_lars_norms_partial(pv, grad_dtype, wire, (const SegDesc*)segs, nsegs, stage_off, total_elems,
                                           scale, (const float*)master, (const LambParam*)params, nparams,
                                           (double*)scratch, (const OptHParams*)hp, blocks, threads, channel,
                                           nvls ? 1 : 0, (cudaStream_t)stream),
                 "lars_norms_partial");
      },
      py::arg("view"), py::arg("grad_dtype"), py::arg("wire"), py::arg("segs"), py::arg("nsegs"), py::arg("stage_off"),
      py::arg("total_elems"), py::arg("scale"), py::arg("master"), py::arg("params"), py::arg("nparams"),
      py::arg("scratch"), py::arg("hp"), py::arg("blocks"), py::arg("threads") = 512, py::arg("channel") = 0,
      py::arg("nvls") = false, py::arg("stream") = 0,
      "LARS 1/3: pack, reduce this rank's shard, per-parameter partial sums of w^2 and g^2");
  m.def(
      "lars_norms",
      [](const PeerView& pv, int wire, size_t total_elems, uintptr_t params, int nparams, uintptr_t scratch,
         size_t win_off, uintptr_t phi, uintptr_t hp, int blocks, int channel, uintptr_t stream) {
        chk_lars(launch_lars_norms(pv, wire, total_elems, (const LambParam*)params, nparams, (const double*)scratch,
                                   win_off, (float*)phi, (const OptHParams*)hp, blocks, channel, (cudaStream_t)stream),
                 "lars_norms");
      },
      py::arg("view"), py::arg("wire"), py::arg("total_elems"), py::arg("params"), py::arg("nparams"),
      py::arg("scratch"), py::arg("win_off"), py::arg("phi"), py::arg("hp"), py::arg("blocks"), py::arg("channel") = 0,
      py::arg("stream") = 0, "LARS 2/3: exchange the per-parameter partial norms, form the trust ratios");
  m.def(
      "lars_apply",
      [](const PeerView& pv, int grad_dtype, int wire, size_t stage_off, size_t param_off, size_t total_elems,
         float scale, uintptr_t master, uintptr_t mom, uintptr_t params, int nparams, uintptr_t phi, uintptr_t hp,
         int blocks, int threads, int channel, bool nvls, uintptr_t stream) {
        chk_lars(launch_lars_apply(pv, grad_dtype, wire, stage_off, param_off, total_elems, scale, (float*)master,
                                   (float*)mom, (const LambParam*)params, nparams, (const float*)phi,
                                   (const OptHParams*)hp, blocks, threads, channel, nvls ? 1 : 0,
                                   (cudaStream_t)stream),
                 "lars_apply");
      },
      py::arg("view"), py::arg("grad_dtype"), py::arg("wire"), py::arg("stage_off"), py::arg("param_off"),
      py::arg("total_elems"), py::arg("scale"), py::arg("master"), py::arg("mom"), py::arg("params"),
      py::arg("nparams"), py::arg("phi"), py::arg("hp"), py::arg("blocks"), py::arg("threads") = 512,
      py::arg("channel") = 0, py::arg("nvls") = false, py::arg("stream") = 0,
      "LARS 3/3: reduce the shard again, update momentum and master, push the new parameters to every peer");
  m.def("lars_load_kernels", []() { chk_lars(lars_load_kernels(), "lars_load_kernels"); },
        "load the LARS kernels now (before any cross-rank launch)");
}
