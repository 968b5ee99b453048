// pybind11 surface of the CUDA-free runtime (module byteps_b200._core).
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "bind/core_bind_ext.h"
#include "compress/compressor.h"
#include "core/env.h"
#include "core/handle_manager.h"
#include "core/log.h"
#include "core/ready_table.h"
#include "core/registry.h"
#include "core/scheduler.h"
#include "core/thread_pool.h"
#include "core/trace.h"
#include "core/types.h"
#include "cpu/half.h"
#include "cpu/reducer.h"

namespace py = pybind11;
using namespace bps;

namespace {

struct PyTask {
  TaskPtr t;
};

class PyCompressor {
 public:
  PyCompressor(const Kwargs& kw, size_t nbytes, int dtype, bool server) {
    c_ = CompressorRegistry::create(kw, nbytes, dtype, server);
    if (!c_) throw std::runtime_error("kwargs name no compressor_type");
  }
  size_t max_compressed_bytes() const { return c_->max_compressed_bytes(); }
  size_t compress(uintptr_t grad, uintptr_t dst) {
    py::gil_scoped_release r;
    return c_->compress((void*)grad, (void*)dst);
  }
  void decompress(uintptr_t src, size_t csize, uintptr_t dst) {
    py::gil_scoped_release r;
    c_->decompress((const void*)src, csize, (void*)dst);
  }
  void decompress_add(uintptr_t src, size_t csize, uintptr_t dst) {
    py::gil_scoped_release r;
    c_->decompress_add((const void*)src, csize, (void*)dst);
  }
  void fast_update_error(uintptr_t err, uintptr_t corr, uintptr_t comp, size_t csize) {
    py::gil_scoped_release r;
    c_->fast_update_error((void*)err, (const void*)corr, (const void*)comp, csize);
  }
  void set_lr(double lr) { c_->set_lr(lr); }
  std::string name() const { return c_->name(); }

 private:
  std::unique_ptr<Compressor> c_;
};

}  // namespace

PYBIND11_MODULE(_core, m) {
  m.doc() = "byteps_b200 native runtime (CUDA-free part)";

  // ---- types
  m.attr("F32") = (int)F32;
  m.attr("F64") = (int)F64;
  m.attr("F16") = (int)F16;
  m.attr("U8") = (int)U8;
  m.attr("I32") = (int)I32;
  m.attr("I8") = (int)I8;
  m.attr("I64") = (int)I64;
  m.attr("BF16") = (int)BF16;
  m.def("dtype_size", &dtype_size);
  m.def("dtype_name", [](int d) { return std::string(dtype_name(d)); });
  m.def("stage_name", [](int s) { return std::string(stage_name(s)); });
  m.attr("STAGE_COUNT") = (int)STAGE_COUNT;
  for (int s = 0; s < STAGE_COUNT; ++s) m.attr(stage_name(s)) = s;
  m.def("command_encode", &command_encode);
  m.def("command_decode", [](int cmd) {
    int r, d;
    command_decode(cmd, &r, &d);
    return py::make_tuple(r, d);
  });
  m.def("make_key", &make_key);
  m.def("key_declared", &key_declared);
  m.def("key_part", &key_part);
  m.def("round_up", &round_up);
  m.def("align_payload", &align_payload);
  m.def("partition_bytes", [](size_t size, size_t bound) {
    std::vector<std::pair<size_t, size_t>> out;
    for (auto& p : partition_bytes(size, bound)) out.emplace_back(p.offset, p.len);
    return out;
  });
  m.def("set_log_level", &set_min_log_level);
  m.def("log_level", &min_log_level);
  m.def("log", [](int lvl, const std::string& msg) {
    if (lvl >= min_log_level() && lvl < L_FATAL) LogMessage("python", 0, lvl).stream() << msg;
  });
  m.def("now_us", &now_us);

  // ---- half helpers (tests)
  m.def("f32_to_bf16", &f32_to_bf16);
  m.def("bf16_to_f32", &bf16_to_f32);
  m.def("f32_to_f16", &f32_to_f16);
  m.def("f16_to_f32", &f16_to_f32);

  // ---- registry
  py::class_<Registry, std::shared_ptr<Registry>>(m, "Registry")
      .def(py::init<>())
      .def("declare", &Registry::declare)
      .def("is_declared", &Registry::is_declared)
      .def("declared_names", &Registry::declared_names)
      .def("size", &Registry::size)
      .def("reset_contexts", &Registry::reset_contexts)
      .def("set_kwargs", &Registry::set_kwargs)
      .def("init_tensor",
           [](Registry& r, const std::string& name, size_t nbytes, int dtype, size_t bound, size_t page) {
             auto ctx = r.context(name);
             if (!ctx) throw std::runtime_error("tensor not declared: " + name);
             r.init_tensor(ctx, nbytes, dtype, bound, page);
             return ctx->keys;
           })
      .def("keys",
           [](Registry& r, const std::string& name) {
             auto ctx = r.context(name);
             if (!ctx) throw std::runtime_error("tensor not declared: " + name);
             return ctx->keys;
           })
      .def("partitions", [](Registry& r, const std::string& name) {
        auto ctx = r.context(name);
        if (!ctx) throw std::runtime_error("tensor not declared: " + name);
        std::vector<std::pair<size_t, size_t>> out;
        for (auto& p : ctx->parts) out.emplace_back(p.offset, p.len);
        return out;
      });

  m.def("hash_naive", &hash_naive);
  m.def("hash_builtin", &hash_builtin);
  m.def("hash_djb2", &hash_djb2);
  m.def("hash_sdbm", &hash_sdbm);
  py::class_<KeyPlacer>(m, "KeyPlacer")
      .def(py::init<const std::string&, int, int, bool, int>(), py::arg("fn") = "djb2", py::arg("num_servers") = 1,
           py::arg("num_workers") = 1, py::arg("mixed_mode") = false, py::arg("mixed_bound") = 101)
      .def("server_of", &KeyPlacer::server_of)
      .def("load", [](KeyPlacer& k) { return k.load(); });

  // ---- ready table + scheduler
  py::class_<ReadyTable, std::shared_ptr<ReadyTable>>(m, "ReadyTable")
      .def(py::init<int, std::string>())
      .def("is_key_ready", &ReadyTable::is_key_ready)
      .def("add_ready_count", &ReadyTable::add_ready_count)
      .def("set_ready_count", &ReadyTable::set_ready_count)
      .def("clear_ready_count", &ReadyTable::clear_ready_count)
      .def("wait_ready", [](ReadyTable& t, uint64_t key, int64_t timeout_ms) {
             py::gil_scoped_release r;
             return t.wait_ready(key, timeout_ms);
           }, py::arg("key"), py::arg("timeout_ms") = -1)
      .def("count", &ReadyTable::count);

  py::class_<PyTask>(m, "Task")
      .def(py::init([](uint64_t key, int priority, size_t len, py::object ready) {
             PyTask p;
             p.t = std::make_shared<Task>();
             p.t->key = key;
             p.t->priority = priority;
             p.t->len = len;
             if (!ready.is_none()) {
               auto fn = std::make_shared<py::object>(ready);
               p.t->ready = [fn]() {
                 py::gil_scoped_acquire g;
                 return (*fn)().cast<bool>();
               };
             }
             return p;
           }),
           py::arg("key"), py::arg("priority") = 0, py::arg("len") = 0, py::arg("ready") = py::none())
      .def_property_readonly("key", [](PyTask& p) { return p.t->key; })
      .def_property_readonly("priority", [](PyTask& p) { return p.t->priority; })
      .def_property_readonly("len", [](PyTask& p) { return p.t->len; });

  py::class_<ScheduledQueue>(m, "ScheduledQueue")
      .def(py::init([](int stage, bool scheduled, uint64_t credits, std::shared_ptr<ReadyTable> rt) {
             return new ScheduledQueue(stage, scheduled, credits, rt.get());
           }),
           py::arg("stage") = 0, py::arg("scheduled") = true, py::arg("credits") = 0, py::arg("ready_table") = nullptr,
           py::keep_alive<1, 5>())
      .def("add", [](ScheduledQueue& q, PyTask& t) { q.add(t.t); })
      .def("get",
           [](ScheduledQueue& q) -> py::object {
             TaskPtr t = q.get();
             if (!t) return py::none();
             return py::cast(PyTask{t});
           })
      .def("get_by_key",
           [](ScheduledQueue& q, uint64_t k) -> py::object {
             TaskPtr t = q.get_by_key(k);
             if (!t) return py::none();
             return py::cast(PyTask{t});
           })
      .def("report_finish", &ScheduledQueue::report_finish)
      .def("pending", &ScheduledQueue::pending)
      .def("credits", &ScheduledQueue::credits)
      .def("reset", &ScheduledQueue::reset);

  // ---- handles
  py::class_<HandleManager, std::shared_ptr<HandleManager>>(m, "HandleManager")
      .def(py::init<>())
      .def("allocate", &HandleManager::allocate)
      .def("mark_done", [](HandleManager& h, int id, int code,
                           const std::string& why) { h.mark_done(id, Status{(StatusCode)code, why}); },
           py::arg("handle"), py::arg("code") = 0, py::arg("reason") = "")
      .def("poll", &HandleManager::poll)
      .def("wait_and_release",
           [](HandleManager& h, int id, int64_t timeout_ms) {
             Status s;
             {
               py::gil_scoped_release r;
               s = h.wait_and_release(id, timeout_ms);
             }
             return py::make_tuple((int)s.code, s.reason);
           },
           py::arg("handle"), py::arg("timeout_ms") = -1)
      .def("outstanding", &HandleManager::outstanding);

  // ---- cpu reducer
  py::class_<CpuReducer>(m, "CpuReducer")
      .def(py::init<int>(), py::arg("num_threads") = 0)
      .def("sum",
           [](CpuReducer& r, uintptr_t dst, uintptr_t src, size_t n, int dt) {
             py::gil_scoped_release g;
             return r.sum((void*)dst, (const void*)src, n, dt);
           })
      .def("sum3",
           [](CpuReducer& r, uintptr_t dst, uintptr_t a, uintptr_t b, size_t n, int dt) {
             py::gil_scoped_release g;
             return r.sum((void*)dst, (const void*)a, (const void*)b, n, dt);
           })
      .def("sum_scaled",
           [](CpuReducer& r, uintptr_t dst, uintptr_t src, size_t n, int dt, float alpha) {
             py::gil_scoped_release g;
             return r.sum_scaled((void*)dst, (const void*)src, n, dt, alpha);
           })
      .def("sum_scaled3",
           [](CpuReducer& r, uintptr_t dst, uintptr_t a, uintptr_t b, size_t n, int dt, float alpha) {
             py::gil_scoped_release g;
             return r.sum_scaled((void*)dst, (const void*)a, (const void*)b, n, dt, alpha);
           })
      .def("scale",
           [](CpuReducer& r, uintptr_t dst, size_t n, int dt, double alpha) {
             py::gil_scoped_release g;
             return r.scale((void*)dst, n, dt, alpha);
           })
      .def("copy",
           [](CpuReducer& r, uintptr_t dst, uintptr_t src, size_t n) {
             py::gil_scoped_release g;
             r.copy((void*)dst, (const void*)src, n);
           })
      .def_property_readonly("num_threads", &CpuReducer::num_threads)
      .def_static("has_avx512", &CpuReducer::has_avx512);

  // ---- compressors
  py::class_<PyCompressor>(m, "Compressor")
      .def(py::init<const Kwargs&, size_t, int, bool>(), py::arg("kwargs"), py::arg("nbytes"), py::arg("dtype"),
           py::arg("server_side") = false)
      .def("max_compressed_bytes", &PyCompressor::max_compressed_bytes)
      .def("compress", &PyCompressor::compress)
      .def("decompress", &PyCompressor::decompress)
      .def("decompress_add", &PyCompressor::decompress_add)
      .def("fast_update_error", &PyCompressor::fast_update_error)
      .def("set_lr", &PyCompressor::set_lr)
      .def("name", &PyCompressor::name);
  m.def("compressor_names", &CompressorRegistry::names);
  m.def("kwargs_serialize", &kwargs_serialize);
  m.def("kwargs_deserialize", &kwargs_deserialize);
  py::class_<XorShift128Plus>(m, "XorShift128Plus")
      .def(py::init<>())
      .def("set_seed", &XorShift128Plus::set_seed)
      .def("next", &XorShift128Plus::next)
      .def("randint", &XorShift128Plus::randint)
      .def(
          "fill_randint_u32",
          [](XorShift128Plus& r, uintptr_t ptr, size_t k, uint64_t high) {
            // k draws of randint(0, high) into a host buffer (random-k index streams for the GPU
            // compressor: the generator is inherently serial, far cheaper on a host core than as a
            // one-thread kernel)
            py::gil_scoped_release nogil;
            uint32_t* p = reinterpret_cast<uint32_t*>(ptr);
            for (size_t i = 0; i < k; ++i) p[i] = (uint32_t)r.randint(0, high);
          },
          py::arg("ptr"), py::arg("k"), py::arg("high"))
      .def("rand", &XorShift128Plus::rand)
      .def("bernoulli", &XorShift128Plus::bernoulli);

  // ---- timeline + telemetry
  py::class_<Timeline, std::shared_ptr<Timeline>>(m, "Timeline")
      .def(py::init<>())
      .def("configure", &Timeline::configure)
      .def("enabled", &Timeline::enabled)
      .def("active", &Timeline::active)
      .def("start_step", &Timeline::start_step)
      .def("end_step", &Timeline::end_step)
      .def("record", &Timeline::record)
      .def("num_events", &Timeline::num_events)
      .def("to_json", &Timeline::to_json)
      .def("dump", &Timeline::dump)
      .def("clear", &Timeline::clear);
  py::class_<Telemetry, std::shared_ptr<Telemetry>>(m, "Telemetry")
      .def(py::init<bool, double>(), py::arg("on") = true, py::arg("interval_s") = 10.0)
      .def("configure", &Telemetry::configure)
      .def("record", &Telemetry::record)
      .def("get",
           [](Telemetry& t) {
             auto e = t.get();
             return py::make_tuple(e.ts_ms, e.mbps);
           })
      .def("should_record", &Telemetry::should_record)
      .def("total_bytes", &Telemetry::total_bytes);

  bind_core_ext(m);
}
