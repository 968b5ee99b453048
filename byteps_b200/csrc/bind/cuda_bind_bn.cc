// pybind11 surface of the fused batch-norm / residual / ReLU kernels (kernels/bn_act.cu).
#include <cuda_runtime_api.h>
#include <pybind11/pybind11.h>

#include <stdexcept>
#include <string>

#include "bind/cuda_bind_ext.h"
#include "kernels/bn_act.cuh"

namespace py = pybind11;
using namespace bps;

namespace {
void chk(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw std::runtime_error(std::string(what) + ": " + cudaGetErrorString(e));
}
}  // namespace

void bind_cuda_bn(py::module_& m) {
  m.def("bn_act_workspace", [](size_t M, int C) {
    return py::make_tuple(bn_act_workspace_floats(M, C), bn_act_counters(C));
  }, "(fp32 workspace floats, uint32 counters) of one bn_act_fwd_stats / bn_act_bwd_reduce launch");

  m.def("bn_act_fwd_stats", [](uintptr_t x, int dtype, size_t M, int C, float eps, float momentum,
                               uintptr_t running_mean, uintptr_t running_var, uintptr_t save_mean,
                               uintptr_t save_invstd, uintptr_t ws, uintptr_t counters, uintptr_t s) {
    chk(launch_bn_act_fwd_stats((const void*)x, dtype, M, C, eps, momentum, (float*)running_mean, (float*)running_var,
                                (float*)save_mean, (float*)save_invstd, (float*)ws, (uint32_t*)counters,
                                (cudaStream_t)s),
        "bn_act_fwd_stats");
  });
  m.def("bn_act_fwd_apply", [](uintptr_t x, uintptr_t residual, int dtype, size_t M, int C, uintptr_t mean,
                               uintptr_t invstd, uintptr_t weight, uintptr_t bias, bool relu, uintptr_t y,
                               uintptr_t mask, uintptr_t s) {
    chk(launch_bn_act_fwd_apply((const void*)x, (const void*)residual, dtype, M, C, (const float*)mean,
                                (const float*)invstd, (const float*)weight, (const float*)bias, relu ? 1 : 0,
                                (void*)y, (uint8_t*)mask, (cudaStream_t)s),
        "bn_act_fwd_apply");
  });
  m.def("bn_act_bwd_reduce", [](uintptr_t dy, uintptr_t x, uintptr_t mask, int dtype, size_t M, int C, uintptr_t mean,
                                uintptr_t invstd, uintptr_t dweight, uintptr_t dbias, uintptr_t ws, uintptr_t counters,
                                uintptr_t s) {
    chk(launch_bn_act_bwd_reduce((const void*)dy, (const void*)x, (const uint8_t*)mask, dtype, M, C,
                                 (const float*)mean, (const float*)invstd, (float*)dweight, (float*)dbias, (float*)ws,
                                 (uint32_t*)counters, (cudaStream_t)s),
        "bn_act_bwd_reduce");
  });
  m.def("bn_act_bwd_apply", [](uintptr_t dy, uintptr_t x, uintptr_t mask, int dtype, size_t M, int C, uintptr_t mean,
                               uintptr_t invstd, uintptr_t weight, uintptr_t dweight, uintptr_t dbias, uintptr_t dx,
                               uintptr_t dresidual, uintptr_t s, uintptr_t total) {
    chk(launch_bn_act_bwd_apply((const void*)dy, (const void*)x, (const uint8_t*)mask, dtype, M, C,
                                (const float*)mean, (const float*)invstd, (const float*)weight,
                                (const float*)dweight, (const float*)dbias, (void*)dx, (void*)dresidual,
                                (cudaStream_t)s, (const float*)total),
        "bn_act_bwd_apply");
  }, py::arg("dy"), py::arg("x"), py::arg("mask"), py::arg("dtype"), py::arg("M"), py::arg("C"), py::arg("mean"),
     py::arg("invstd"), py::arg("weight"), py::arg("dweight"), py::arg("dbias"), py::arg("dx"), py::arg("dresidual"),
     py::arg("stream"), py::arg("total") = 0,
     "total: device float holding the row count to divide by (bn_sync_stats writes it); 0 divides by M");

  // ---- single-launch passes
  m.def("bn_act_plan", [](int bwd, int dtype, size_t M, int C, long long cap, bool relu, bool residual,
                          bool dy2, int pool_h, int pool_w) -> py::object {
    BnFusedPlan p;
    if (!bn_act_fused_plan(bwd, dtype, M, C, cap, relu ? 1 : 0, residual ? 1 : 0, dy2 ? 1 : 0, &p, pool_h, pool_w))
      return py::none();
    py::dict d;
    d["ws_floats"] = p.ws_floats;
    d["counters"] = p.counters;
    d["rows_per_chunk"] = p.rows_per_chunk;
    d["held_rows"] = p.held_rows;
    d["held_bytes"] = p.held_bytes;
    d["ring_depth"] = p.ring_depth;
    d["smem_bytes"] = p.smem_bytes;
    d["bytes_moved"] = p.bytes_moved;
    d["wave_blocks"] = p.wave_blocks;
    return d;
  }, py::arg("bwd"), py::arg("dtype"), py::arg("M"), py::arg("C"), py::arg("cap") = -1, py::arg("relu") = false,
     py::arg("residual") = false, py::arg("dy2") = false, py::arg("pool_h") = 0, py::arg("pool_w") = 0,
     "plan of the single-launch bn_act_fwd (bwd=0) / bn_act_bwd (bwd=1) at (M, C, dtype) on the current device, or "
     "None when it cannot run there; cap >= 0 limits the bytes of rows a block holds in shared memory.  residual "
     "selects the backward's shared-memory layout; relu, residual and dy2 (a second gradient, backward with a "
     "residual) select the variant whose bytes_moved is reported.  pool_h, pool_w > 0: the pooled passes "
     "(bn_act_fwd_pool / bn_act_bwd_pool, relu without residual) over images of pool_h x pool_w; dy2 then means a "
     "second pooled gradient");
  m.def("bn_act_fwd", [](uintptr_t x, uintptr_t residual, int dtype, size_t M, int C, float eps, float momentum,
                         uintptr_t running_mean, uintptr_t running_var, uintptr_t save_mean, uintptr_t save_invstd,
                         uintptr_t weight, uintptr_t bias, bool relu, uintptr_t y, uintptr_t mask, uintptr_t ws,
                         uintptr_t counters, uintptr_t s, long long cap) {
    chk(launch_bn_act_fwd((const void*)x, (const void*)residual, dtype, M, C, eps, momentum, (float*)running_mean,
                          (float*)running_var, (float*)save_mean, (float*)save_invstd, (const float*)weight,
                          (const float*)bias, relu ? 1 : 0, (void*)y, (uint8_t*)mask, (float*)ws, (uint32_t*)counters,
                          cap, (cudaStream_t)s),
        "bn_act_fwd");
  }, py::arg("x"), py::arg("residual"), py::arg("dtype"), py::arg("M"), py::arg("C"), py::arg("eps"),
     py::arg("momentum"), py::arg("running_mean"), py::arg("running_var"), py::arg("save_mean"),
     py::arg("save_invstd"), py::arg("weight"), py::arg("bias"), py::arg("relu"), py::arg("y"), py::arg("mask"),
     py::arg("ws"), py::arg("counters"), py::arg("stream"), py::arg("cap") = -1);
  m.def("bn_act_bwd", [](uintptr_t dy, uintptr_t x, uintptr_t mask, int dtype, size_t M, int C, uintptr_t mean,
                         uintptr_t invstd, uintptr_t weight, uintptr_t dweight, uintptr_t dbias, uintptr_t dx,
                         uintptr_t dresidual, uintptr_t ws, uintptr_t counters, uintptr_t s, long long cap,
                         uintptr_t dy2) {
    chk(launch_bn_act_bwd((const void*)dy, (const void*)dy2, (const void*)x, (const uint8_t*)mask, dtype, M, C,
                          (const float*)mean, (const float*)invstd, (const float*)weight, (float*)dweight,
                          (float*)dbias, (void*)dx, (void*)dresidual, (float*)ws, (uint32_t*)counters, cap,
                          (cudaStream_t)s),
        "bn_act_bwd");
  }, py::arg("dy"), py::arg("x"), py::arg("mask"), py::arg("dtype"), py::arg("M"), py::arg("C"), py::arg("mean"),
     py::arg("invstd"), py::arg("weight"), py::arg("dweight"), py::arg("dbias"), py::arg("dx"), py::arg("dresidual"),
     py::arg("ws"), py::arg("counters"), py::arg("stream"), py::arg("cap") = -1, py::arg("dy2") = 0,
     "dy2: 0, or a second gradient of the output laid out as dy (M x C, 16-byte aligned; needs dresidual), summed "
     "with dy inside the kernel");

  m.def("bn_act_fwd_pool", [](uintptr_t x, int dtype, int N, int H, int W, int C, float eps, float momentum,
                              uintptr_t running_mean, uintptr_t running_var, uintptr_t save_mean,
                              uintptr_t save_invstd, uintptr_t weight, uintptr_t bias, uintptr_t pooled, uintptr_t code,
                              uintptr_t ws, uintptr_t counters, uintptr_t s, long long cap) {
    chk(launch_bn_act_fwd_pool((const void*)x, dtype, N, H, W, C, eps, momentum, (float*)running_mean,
                               (float*)running_var, (float*)save_mean, (float*)save_invstd, (const float*)weight,
                               (const float*)bias, (void*)pooled, (uint32_t*)code, (float*)ws, (uint32_t*)counters,
                               cap, (cudaStream_t)s),
        "bn_act_fwd_pool");
  }, py::arg("x"), py::arg("dtype"), py::arg("N"), py::arg("H"), py::arg("W"), py::arg("C"), py::arg("eps"),
     py::arg("momentum"), py::arg("running_mean"), py::arg("running_var"), py::arg("save_mean"),
     py::arg("save_invstd"), py::arg("weight"), py::arg("bias"), py::arg("pooled"), py::arg("code"), py::arg("ws"),
     py::arg("counters"), py::arg("stream"), py::arg("cap") = -1,
     "single-launch batch norm, ReLU and 3x3 / stride 2 / padding 1 max pool: the pooled output (N x OH x OW x C) and "
     "its window codes (N * OH * OW * C / 8 uint32)");
  m.def("bn_act_bwd_pool", [](uintptr_t g1, uintptr_t g2, uintptr_t code, uintptr_t x, int dtype, int N, int H, int W,
                              int C, uintptr_t mean, uintptr_t invstd, uintptr_t weight, uintptr_t dweight,
                              uintptr_t dbias, uintptr_t dx, uintptr_t ws, uintptr_t counters, uintptr_t s,
                              long long cap) {
    chk(launch_bn_act_bwd_pool((const void*)g1, (const void*)g2, (const uint32_t*)code, (const void*)x, dtype, N, H, W,
                               C, (const float*)mean, (const float*)invstd, (const float*)weight, (float*)dweight,
                               (float*)dbias, (void*)dx, (float*)ws, (uint32_t*)counters, cap, (cudaStream_t)s),
        "bn_act_bwd_pool");
  }, py::arg("g1"), py::arg("g2"), py::arg("code"), py::arg("x"), py::arg("dtype"), py::arg("N"), py::arg("H"),
     py::arg("W"), py::arg("C"), py::arg("mean"), py::arg("invstd"), py::arg("weight"), py::arg("dweight"),
     py::arg("dbias"), py::arg("dx"), py::arg("ws"), py::arg("counters"), py::arg("stream"), py::arg("cap") = -1,
     "backward of bn_act_fwd_pool for the pooled gradients g1 and g2 (0: none), summed as torch's add");

  // ---- synchronised batch norm
  m.def("bn_act_load_kernels", []() { chk(bn_act_load_kernels(), "bn_act_load_kernels"); },
        "load every batch-norm kernel variant now (before any cross-rank launch)");
  m.def("bn_sync_window_floats", &bn_sync_window_floats, py::arg("world"), py::arg("cmax"));
  m.def("bn_act_fwd_stats_local", [](uintptr_t x, int dtype, size_t M, int C, uintptr_t local_mean,
                                     uintptr_t local_m2, uintptr_t ws, uintptr_t counters, uintptr_t s) {
    chk(launch_bn_act_fwd_stats_local((const void*)x, dtype, M, C, (float*)local_mean, (float*)local_m2, (float*)ws,
                                      (uint32_t*)counters, (cudaStream_t)s),
        "bn_act_fwd_stats_local");
  });
  m.def("bn_sync_stats", [](const PeerView& pv, int channel, size_t win_off, int cmax, int C, uintptr_t local_mean,
                            uintptr_t local_m2, float count, float eps, float momentum, uintptr_t running_mean,
                            uintptr_t running_var, uintptr_t save_mean, uintptr_t save_invstd, uintptr_t total,
                            uintptr_t s) {
    chk(launch_bn_sync_stats(pv, channel, win_off, cmax, C, (const float*)local_mean, (const float*)local_m2, count,
                             eps, momentum, (float*)running_mean, (float*)running_var, (float*)save_mean,
                             (float*)save_invstd, (float*)total, (cudaStream_t)s),
        "bn_sync_stats");
  });
  m.def("bn_sync_grad", [](const PeerView& pv, int channel, size_t win_off, int cmax, int C, uintptr_t dbias,
                           uintptr_t dweight, uintptr_t sum_dbias, uintptr_t sum_dweight, uintptr_t s) {
    chk(launch_bn_sync_grad(pv, channel, win_off, cmax, C, (const float*)dbias, (const float*)dweight,
                            (float*)sum_dbias, (float*)sum_dweight, (cudaStream_t)s),
        "bn_sync_grad");
  });
}
