#include "bind/cuda_bind_ext.h"

#include <cuda_runtime_api.h>
#include <pybind11/stl.h>

#include <stdexcept>
#include <string>

#include "comm/nccl_manager.h"
#include "core/gpu_stage.h"
#include "kernels/compress.cuh"
#include "kernels/misc.cuh"
#include "kernels/pushpull.cuh"
#include "kernels/pushpull_umma.cuh"

namespace py = pybind11;
using namespace bps;

static void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}

extern "C" int bps_event_query(void* ev) {
  cudaError_t e = cudaEventQuery((cudaEvent_t)ev);
  if (e == cudaSuccess) return 1;
  if (e != cudaErrorNotReady) cudaGetLastError();
  return 0;
}

namespace bps {
void* gpu_stage_create(int device, int nevents);
void gpu_stage_destroy(void* c);
const BpsGpuStageFns* gpu_stage_fns();
}  // namespace bps

void bind_cuda_ext(py::module_& m) {
  // address of a C function the CUDA-free runtime can call to poll a device event
  m.def("event_query_fn", []() { return (uintptr_t)&bps_event_query; });
  // device stages of the CPU-server pipeline (core/gpu_stage.h): function table + per-device context
  m.def("gpu_stage_fns", []() { return (uintptr_t)gpu_stage_fns(); });
  m.def("gpu_stage_create", [](int device, int nevents) { return (uintptr_t)gpu_stage_create(device, nevents); },
        py::arg("device"), py::arg("nevents") = 8192);
  m.def("gpu_stage_destroy", [](uintptr_t c) { gpu_stage_destroy((void*)c); });
  m.def("stream_wait_event", [](uintptr_t stream, uintptr_t event) {
    chk(cudaStreamWaitEvent((cudaStream_t)stream, (cudaEvent_t)event, 0), "cudaStreamWaitEvent");
  });
  m.def(
      "write_blob",
      [](uintptr_t dst, const py::bytes& data, uintptr_t stream) {
        std::string s(data);
        chk(launch_write_blob((void*)dst, s.data(), s.size(), (cudaStream_t)stream), "write_blob");
      },
      py::arg("dst"), py::arg("data"), py::arg("stream") = 0);
  m.def(
      "l2_flush",
      [](uintptr_t buf, size_t nbytes, uint32_t value, uintptr_t stream) {
        chk(launch_l2_flush((void*)buf, nbytes, value, (cudaStream_t)stream), "l2_flush");
      },
      py::arg("buf"), py::arg("nbytes"), py::arg("value") = 0, py::arg("stream") = 0);

  // ---- native NCCL manager (baseline arm only)
  py::class_<NcclManager>(m, "NcclManager")
      .def(py::init<int, int, int, int, int>(), py::arg("rank"), py::arg("world"), py::arg("device"),
           py::arg("num_rings") = 1, py::arg("group_size") = 4)
      .def_static("available", &NcclManager::available)
      .def_static("make_unique_id", []() { return py::bytes(NcclManager::make_unique_id()); })
      .def("init", [](NcclManager& n, const std::vector<py::bytes>& ids) {
        std::vector<std::string> v;
        for (auto& b : ids) v.push_back(std::string(b));
        py::gil_scoped_release r;
        n.init(v);
      })
      .def("root", &NcclManager::root)
      .def("push_pull", [](NcclManager& n, uintptr_t ptr, size_t nbytes, int dtype, uint64_t first_key,
                           size_t partition_bytes, uintptr_t ready, uintptr_t done) {
        n.push_pull((void*)ptr, nbytes, dtype, first_key, partition_bytes, (cudaEvent_t)ready, (cudaEvent_t)done);
      }, py::arg("ptr"), py::arg("nbytes"), py::arg("dtype"), py::arg("first_key") = 0,
         py::arg("partition_bytes") = 4096000, py::arg("ready") = 0, py::arg("done") = 0)
      .def("tasks_issued", &NcclManager::tasks_issued)
      .def("stream", [](NcclManager& n, int ring) { return (uintptr_t)n.stream(ring); }, py::arg("ring") = 0)
      .def("num_rings", &NcclManager::num_rings);

  // ---- wgmma/TMA push-pull variant
  py::class_<UmmaMaps>(m, "UmmaMaps");
  m.def("make_umma_maps", [](const PeerView& pv, int wire, size_t off, size_t nelem) {
    UmmaMaps maps;
    int r = encode_umma_maps(pv, wire, off, nelem, &maps);
    if (r != 0) throw std::runtime_error("cuTensorMapEncodeTiled failed: " + std::to_string(r));
    return maps;
  });
  m.def("umma_smem_bytes", &umma_smem_bytes);
  m.def(
      "pushpull_inplace_umma",
      [](const PeerView& pv, const UmmaMaps& maps, int wire, size_t off, size_t nelem, float scale, int blocks,
         int channel, uintptr_t stream) {
        chk(launch_pushpull_inplace_umma(pv, maps, wire, off, nelem, scale, blocks, channel, (cudaStream_t)stream),
            "pushpull_inplace_umma");
      },
      py::arg("view"), py::arg("maps"), py::arg("wire"), py::arg("off"), py::arg("nelem"), py::arg("scale"),
      py::arg("blocks"), py::arg("channel") = 0, py::arg("stream") = 0);

  // ---- compression kernels (pointers are raw device addresses)
  using S = cudaStream_t;
  m.def("ef_correct", [](uintptr_t g, int dtype, uintptr_t mom, float mu, uintptr_t err, float ratio,
                         uintptr_t corrected, size_t n, uintptr_t acc, uintptr_t s) {
    chk(launch_ef_correct((const void*)g, dtype, (float*)mom, mu, (const float*)err, ratio, (float*)corrected, n,
                          (float*)acc, (S)s),
        "ef_correct");
  });
  m.def("index_scatter", [](uintptr_t idx, uintptr_t vals, uint32_t k, size_t n, uintptr_t out, int dtype, float mult,
                            uintptr_t s) {
    chk(launch_index_scatter((const uint32_t*)idx, (const float*)vals, k, n, (void*)out, dtype, mult, (S)s),
        "index_scatter");
  });
  m.def("dither_quantize", [](uintptr_t corrected, size_t n, uintptr_t acc, int s_levels, int partition,
                              int normalize, uint64_t seed, uint64_t step, uintptr_t levels, uintptr_t scale_out,
                              uintptr_t err_out, uintptr_t s) {
    chk(launch_dither_quantize((const float*)corrected, n, (const float*)acc, s_levels, partition, normalize, seed,
                               step, (int8_t*)levels, (float*)scale_out, (float*)err_out, (S)s), "dither_quantize");
  });
  m.def("dither_unpack", [](uintptr_t levels, uintptr_t scale, size_t n, int s_levels, int partition, uintptr_t out,
                            int dtype, float mult, uintptr_t s) {
    chk(launch_dither_unpack((const int8_t*)levels, (const float*)scale, n, s_levels, partition, (void*)out, dtype,
                             mult, (S)s), "dither_unpack");
  });
  m.def("cast_scale", [](uintptr_t in, size_t n, uintptr_t out, int dtype, float mult, uintptr_t s) {
    chk(launch_cast_scale((const float*)in, n, (void*)out, dtype, mult, (S)s), "cast_scale");
  });
}
