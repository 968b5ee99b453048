// pybind11 surface of the LAMB kernels of the fused exchange (kernels/pushpull_lamb.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/pushpull_lamb.cuh"

namespace py = pybind11;
using namespace bps;

static void chk_lamb(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void bind_cuda_lamb(py::module_& m) {
  m.attr("LAMB_PARAM_BYTES") = (int)sizeof(LambParam);
  m.def("lamb_scratch_bytes", &lamb_scratch_bytes, py::arg("shard_elems"), py::arg("nparams"));
  m.def("lamb_window_bytes", &lamb_window_bytes, py::arg("nparams"), py::arg("world"));
  m.def(
      "lamb_moments",
      [](const PeerView& pv, int grad_dtype, int wire, uintptr_t segs, int nsegs, size_t stage_off, size_t total_elems,
         float scale, uintptr_t master, uintptr_t m1, uintptr_t m2, uintptr_t params, int nparams, uintptr_t scratch,
         uintptr_t hp, int blocks, int threads, int channel, bool nvls, uintptr_t stream) {
        chk_lamb(launch_lamb_moments(pv, grad_dtype, wire, (const SegDesc*)segs, nsegs, stage_off, total_elems, scale,
                                     (float*)master, (float*)m1, (float*)m2, (const LambParam*)params, nparams,
                                     (double*)scratch, (const OptHParams*)hp, blocks, threads, channel, nvls ? 1 : 0,
                                     (cudaStream_t)stream),
                 "lamb_moments");
      },
      py::arg("view"), py::arg("grad_dtype"), py::arg("wire"), py::arg("segs"), py::arg("nsegs"), py::arg("stage_off"),
      py::arg("total_elems"), py::arg("scale"), py::arg("master"), py::arg("m1"), py::arg("m2"), py::arg("params"),
      py::arg("nparams"), py::arg("scratch"), py::arg("hp"), py::arg("blocks"), py::arg("threads") = 512,
      py::arg("channel") = 0, py::arg("nvls") = false, py::arg("stream") = 0,
      "LAMB 1/3: pack, reduce this rank's shard, update the moments, per-parameter partial norms");
  m.def(
      "lamb_norms",
      [](const PeerView& pv, int wire, size_t total_elems, uintptr_t params, int nparams, uintptr_t scratch,
         size_t win_off, uintptr_t phi, uintptr_t hp, int blocks, int channel, uintptr_t stream) {
        chk_lamb(launch_lamb_norms(pv, wire, total_elems, (const LambParam*)params, nparams, (const double*)scratch,
                                   win_off, (float*)phi, (const OptHParams*)hp, blocks, channel, (cudaStream_t)stream),
                 "lamb_norms");
      },
      py::arg("view"), py::arg("wire"), py::arg("total_elems"), py::arg("params"), py::arg("nparams"),
      py::arg("scratch"), py::arg("win_off"), py::arg("phi"), py::arg("hp"), py::arg("blocks"), py::arg("channel") = 0,
      py::arg("stream") = 0, "LAMB 2/3: exchange the per-parameter partial norms, form the trust ratios");
  m.def(
      "lamb_apply",
      [](const PeerView& pv, int grad_dtype, int wire, size_t param_off, size_t total_elems, uintptr_t master,
         uintptr_t m1, uintptr_t m2, uintptr_t params, int nparams, uintptr_t phi, uintptr_t hp, int blocks,
         int threads, int channel, bool nvls, uintptr_t stream) {
        chk_lamb(launch_lamb_apply(pv, grad_dtype, wire, param_off, total_elems, (float*)master, (const float*)m1,
                                   (const float*)m2, (const LambParam*)params, nparams, (const float*)phi,
                                   (const OptHParams*)hp, blocks, threads, channel, nvls ? 1 : 0,
                                   (cudaStream_t)stream),
                 "lamb_apply");
      },
      py::arg("view"), py::arg("grad_dtype"), py::arg("wire"), py::arg("param_off"), py::arg("total_elems"),
      py::arg("master"), py::arg("m1"), py::arg("m2"), py::arg("params"), py::arg("nparams"), py::arg("phi"),
      py::arg("hp"), py::arg("blocks"), py::arg("threads") = 512, py::arg("channel") = 0, py::arg("nvls") = false,
      py::arg("stream") = 0, "LAMB 3/3: update the master shard and push the new parameters to every peer");
  m.def("lamb_load_kernels", []() { chk_lamb(lamb_load_kernels(), "lamb_load_kernels"); },
        "load the LAMB kernels now (before any cross-rank launch)");
}
