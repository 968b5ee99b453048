// pybind11 surface of the global gradient-norm clipping kernels of the fused exchange (kernels/grad_clip.cu).  The
// (start, numel) table has LAMB's layout (LambParam).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/grad_clip.cuh"

namespace py = pybind11;
using namespace bps;

static void chk_clip(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

void bind_cuda_clip(py::module_& m) {
  m.attr("CLIP_WINDOW_BYTES") = kClipWindowBytes;
  m.def(
      "clip_norm_partial",
      [](const PeerView& pv, int grad_dtype, int wire, uintptr_t segs, int nsegs, size_t stage_off, size_t total_elems,
         float scale, uintptr_t params, int nparams, uintptr_t row, uintptr_t hp, int blocks, int threads, int channel,
         bool nvls, uintptr_t stream) {
        chk_clip(launch_clip_norm_partial(pv, grad_dtype, wire, (const SegDesc*)segs, nsegs, stage_off, total_elems,
                                          scale, (const LambParam*)params, nparams, (double*)row,
                                          (const OptHParams*)hp, blocks, threads, channel, nvls ? 1 : 0,
                                          (cudaStream_t)stream),
                 "clip_norm_partial");
      },
      py::arg("view"), py::arg("grad_dtype"), py::arg("wire"), py::arg("segs"), py::arg("nsegs"), py::arg("stage_off"),
      py::arg("total_elems"), py::arg("scale"), py::arg("params"), py::arg("nparams"), py::arg("row"), py::arg("hp"),
      py::arg("blocks"), py::arg("threads") = 512, py::arg("channel") = 0, py::arg("nvls") = false,
      py::arg("stream") = 0, "clip 1/2: pack, reduce this rank's shard of a bucket, one float64 sum of g^2 per CTA");
  m.def(
      "clip_norm_update",
      [](const PeerView& pv, int channel, size_t win_off, uintptr_t scratch, int nrows, int row_len, double max_norm,
         uintptr_t grad_norm, uintptr_t hp, int ngroups, uintptr_t stream) {
        chk_clip(launch_clip_norm_update(pv, channel, win_off, (const double*)scratch, nrows, row_len, max_norm,
                                         (float*)grad_norm, (OptHParams*)hp, ngroups, (cudaStream_t)stream),
                 "clip_norm_update");
      },
      py::arg("view"), py::arg("channel"), py::arg("win_off"), py::arg("scratch"), py::arg("nrows"),
      py::arg("row_len"), py::arg("max_norm"), py::arg("grad_norm"), py::arg("hp"), py::arg("ngroups"),
      py::arg("stream") = 0,
      "clip 2/2: the global norm over every rank and bucket, grad_scale of every group multiplied by the coefficient");
  m.def("clip_load_kernels", []() { chk_clip(clip_load_kernels(), "clip_load_kernels"); },
        "load the clipping kernels now (before any cross-rank launch)");
}
