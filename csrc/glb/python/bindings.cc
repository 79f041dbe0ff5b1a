// pybind11 bindings for the host side of the library (stores, rendezvous, tcp
// transport, contexts, point-to-point, new-style + old-style host collectives).
// The CUDA side is registered from bindings_cuda.cc. Buffers cross the boundary
// as raw addresses (int) + sizes; gloo_b200/ops wraps them for numpy / torch.
#include <pybind11/functional.h>
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "glb/allgather.h"
#include "glb/allgatherv.h"
#include "glb/allreduce.h"
#include "glb/alltoall.h"
#include "glb/alltoallv.h"
#include "glb/barrier.h"
#include "glb/broadcast.h"
#include "glb/common/linux.h"
#include "glb/common/logging.h"
#include "glb/common/utils.h"
#include "glb/context.h"
#include "glb/gather.h"
#include "glb/gatherv.h"
#include "glb/math.h"
#include "glb/reduce.h"
#include "glb/reduce_scatter.h"
#include "glb/rendezvous/context.h"
#include "glb/rendezvous/file_store.h"
#include "glb/rendezvous/hash_store.h"
#include "glb/rendezvous/prefix_store.h"
#include "glb/rendezvous/redis_store.h"
#include "glb/transport/ibverbs/device.h"
#include "glb/transport/uv/device.h"
#include "glb/transport/nvl/device.h"
#include "glb/scatter.h"
#include "glb/transport/tcp/device.h"
#include "glb/transport/tcp/tls/device.h"
#include "glb/types.h"

namespace py = pybind11;
using namespace glb;

namespace glb_py {
void registerOldStyle(py::module_& m);  // bindings_algorithms.cc
void registerCuda(py::module_& m);      // bindings_cuda.cc
void registerExtras(py::module_& m);    // bindings_extras.cc
}  // namespace glb_py

namespace {

using ms = std::chrono::milliseconds;

// A store implemented in Python (e.g. wrapping torch.distributed's TCPStore).
class PyStore : public IStore {
 public:
  using IStore::IStore;
  void set(const std::string& key, const Bytes& data) override {
    py::gil_scoped_acquire gil;
    py::function f = py::get_override(this, "set");
    if (!f) throw std::runtime_error("Store.set not implemented");
    f(key, py::bytes(data.data(), data.size()));
  }
  Bytes get(const std::string& key) override {
    py::gil_scoped_acquire gil;
    py::function f = py::get_override(this, "get");
    if (!f) throw std::runtime_error("Store.get not implemented");
    std::string s = py::cast<std::string>(py::bytes(f(key)));
    return Bytes(s.begin(), s.end());
  }
  void wait(const std::vector<std::string>& keys, ms timeout) override {
    py::gil_scoped_acquire gil;
    py::function f = py::get_override(this, "wait");
    if (!f) throw std::runtime_error("Store.wait not implemented");
    f(keys, static_cast<long>(timeout.count()));
  }
  using IStore::wait;
};

inline void* P(uintptr_t p) { return reinterpret_cast<void*>(p); }

std::vector<void*> toPtrs(const std::vector<uintptr_t>& v) {
  std::vector<void*> out;
  for (auto p : v) out.push_back(P(p));
  return out;
}

AllreduceOptions::Func reduceFnFor(int dtype, int op) {
  ReduceFn fn = getReduceFn(static_cast<DataType>(dtype), static_cast<ReduceOp>(op));
  return [fn](void* c, const void* a, const void* b, size_t n) { fn(c, a, b, n); };
}

// Custom reductions written in Python: fn(c_ptr, a_ptr, b_ptr, n) -> None.
AllreduceOptions::Func reduceFnFromPython(py::function f) {
  auto holder = std::make_shared<py::function>(std::move(f));
  return [holder](void* c, const void* a, const void* b, size_t n) {
    py::gil_scoped_acquire gil;
    (*holder)(reinterpret_cast<uintptr_t>(c), reinterpret_cast<uintptr_t>(a), reinterpret_cast<uintptr_t>(b), n);
  };
}

AllreduceOptions::Func pickReduce(int dtype, int op, const py::object& custom) {
  if (!custom.is_none()) return reduceFnFromPython(custom.cast<py::function>());
  return reduceFnFor(dtype, op);
}

ms toMs(long t, const std::shared_ptr<Context>& ctx) { return t < 0 ? ctx->getTimeout() : ms(t); }

}  // namespace

PYBIND11_MODULE(_C, m) {
  m.doc() = "gloo_b200 native core";

  py::register_exception<Exception>(m, "GlbError", PyExc_RuntimeError);
  static py::exception<IoException> ioExc(m, "IoError", m.attr("GlbError").ptr());
  static py::exception<TimeoutException> toExc(m, "TimeoutError", ioExc.ptr());
  static py::exception<InvalidOperationException> invExc(m, "InvalidOperationError", m.attr("GlbError").ptr());
  static py::exception<EnforceNotMet> enfExc(m, "EnforceError", m.attr("GlbError").ptr());
  // Invalid data found on the device: a ValueError, like the host-side argument checks.
  static py::exception<InputException> inExc(m, "InputError", PyExc_ValueError);
  py::register_exception_translator([](std::exception_ptr p) {
    try {
      if (p) std::rethrow_exception(p);
    } catch (const InputException& e) {
      py::set_error(inExc, e.what());
    } catch (const TimeoutException& e) {
      py::set_error(toExc, e.what());
    } catch (const IoException& e) {
      py::set_error(ioExc, e.what());
    } catch (const InvalidOperationException& e) {
      py::set_error(invExc, e.what());
    } catch (const EnforceNotMet& e) {
      py::set_error(enfExc, e.what());
    }
  });

  // ---- common -----------------------------------------------------------------
  m.def("set_log_level", [](int l) { setLogLevel(static_cast<LogLevel>(l)); });
  m.def("log_level", [] { return static_cast<int>(logLevel()); });
  m.def("hostname", &getHostname);
  m.def("pci_devices", &pciDevices, py::arg("pci_class"), py::arg("mask") = 0xffff00);
  m.def("pci_distance", &pciDistance);
  m.def("interface_to_bus_id", &interfaceToBusID);
  m.def("interface_speed", &getInterfaceSpeedByName);
  m.def("list_interfaces", &listInterfaces);
  m.def("kernel_modules", [] {
    auto& s = kernelModules();
    return std::vector<std::string>(s.begin(), s.end());
  });
  m.def("has_simd_half", &hasSimdHalf);
  m.def("element_size", [](int dt) { return elementSize(static_cast<DataType>(dt)); });
  m.def("slot_build", [](int prefix, uint32_t tag, uint64_t delta) {
    return static_cast<uint64_t>(Slot::build(static_cast<uint8_t>(prefix), tag) + delta);
  }, py::arg("prefix"), py::arg("tag"), py::arg("delta") = 0);
  m.def("reduce_local", [](uintptr_t c, uintptr_t a, uintptr_t b, size_t n, int dtype, int op) {
    py::gil_scoped_release nogil;
    getReduceFn(static_cast<DataType>(dtype), static_cast<ReduceOp>(op))(P(c), P(a), P(b), n);
  });
  m.def("float_to_half_bits", [](float f) { return float16::fromFloat(f); });
  m.def("half_bits_to_float", [](uint16_t b) { return float16::toFloat(b); });
  m.def("float_to_bfloat_bits", [](float f) { return bfloat16::fromFloat(f); });
  // FP8 encode / decode of the host types (dtype: DataType.FLOAT8_E4M3 or FLOAT8_E5M2).
  m.def("float_to_fp8_bits", [](float f, int dt) -> uint8_t {
    switch (static_cast<DataType>(dt)) {
      case DataType::FLOAT8_E4M3: return float8_e4m3::fromFloat(f);
      case DataType::FLOAT8_E5M2: return float8_e5m2::fromFloat(f);
      default: GLB_THROW_INVALID_OPERATION_EXCEPTION("float_to_fp8_bits: not an FP8 dtype: ", dt);
    }
  }, py::arg("f"), py::arg("dtype"));
  m.def("fp8_bits_to_float", [](uint8_t b, int dt) -> float {
    switch (static_cast<DataType>(dt)) {
      case DataType::FLOAT8_E4M3: return float8_e4m3::toFloat(b);
      case DataType::FLOAT8_E5M2: return float8_e5m2::toFloat(b);
      default: GLB_THROW_INVALID_OPERATION_EXCEPTION("fp8_bits_to_float: not an FP8 dtype: ", dt);
    }
  }, py::arg("b"), py::arg("dtype"));
  m.def("factorize", &detail::factorize);

  // ---- stores -------------------------------------------------------------------
  py::class_<IStore, PyStore, std::shared_ptr<IStore>>(m, "Store")
      .def(py::init<>())
      .def("set", [](IStore& s, const std::string& k, py::bytes v) {
        std::string sv = v;
        py::gil_scoped_release nogil;
        s.set(k, IStore::Bytes(sv.begin(), sv.end()));
      })
      .def("get", [](IStore& s, const std::string& k) {
        IStore::Bytes b;
        {
          py::gil_scoped_release nogil;
          b = s.get(k);
        }
        return py::bytes(b.data(), b.size());
      })
      .def("wait", [](IStore& s, const std::vector<std::string>& keys, long timeoutMs) {
        py::gil_scoped_release nogil;
        s.wait(keys, ms(timeoutMs));
      }, py::arg("keys"), py::arg("timeout_ms") = 30000)
      .def("add", [](IStore& s, const std::string& k, int64_t v) {
        py::gil_scoped_release nogil;
        return s.add(k, v);
      })
      .def("append", [](IStore& s, const std::string& k, py::bytes v) {
        std::string sv = v;
        py::gil_scoped_release nogil;
        s.append(k, IStore::Bytes(sv.begin(), sv.end()));
      })
      .def("multi_get", [](IStore& s, const std::vector<std::string>& keys) {
        std::vector<IStore::Bytes> r;
        {
          py::gil_scoped_release nogil;
          r = s.multi_get(keys);
        }
        std::vector<py::bytes> out;
        for (auto& b : r) out.emplace_back(b.data(), b.size());
        return out;
      })
      .def("has_extended_api", &IStore::has_extended_api);
  py::class_<rendezvous::HashStore, IStore, std::shared_ptr<rendezvous::HashStore>>(m, "HashStore")
      .def(py::init<>())
      .def("__len__", &rendezvous::HashStore::size);
  py::class_<rendezvous::FileStore, IStore, std::shared_ptr<rendezvous::FileStore>>(m, "FileStore")
      .def(py::init<const std::string&>())
      .def("key_file_paths", &rendezvous::FileStore::getAllKeyFilePaths)
      .def_property_readonly("path", &rendezvous::FileStore::basePath);
  py::class_<rendezvous::PrefixStore, IStore, std::shared_ptr<rendezvous::PrefixStore>>(m, "PrefixStore")
      .def(py::init<const std::string&, std::shared_ptr<IStore>>());
  py::class_<rendezvous::RedisStore, IStore, std::shared_ptr<rendezvous::RedisStore>>(m, "RedisStore")
      .def(py::init<const std::string&, int>(), py::arg("host"), py::arg("port") = 6379,
           py::call_guard<py::gil_scoped_release>())
      .def("check", &rendezvous::RedisStore::check, py::call_guard<py::gil_scoped_release>());

  // ---- transport ------------------------------------------------------------------
  py::class_<transport::Device, std::shared_ptr<transport::Device>>(m, "Device")
      .def("__str__", &transport::Device::str)
      .def("pci_bus_id", &transport::Device::getPCIBusID)
      .def("interface_speed", &transport::Device::getInterfaceSpeed)
      .def("has_gpu_direct", &transport::Device::hasGPUDirect);
  m.def("create_tcp_device", [](const std::string& hostname, const std::string& iface, bool lazy, int numLoops) {
    transport::tcp::attr a;
    a.hostname = hostname;
    a.iface = iface;
    a.numLoops = numLoops;
    return lazy ? transport::tcp::CreateLazyDevice(a) : transport::tcp::CreateDevice(a);
  }, py::arg("hostname") = "", py::arg("iface") = "", py::arg("lazy") = false, py::arg("num_loops") = 1);

  m.def("create_tls_device", [](const std::string& hostname, const std::string& pkey, const std::string& cert,
                                const std::string& caFile, const std::string& caPath) {
    transport::tcp::attr a;
    a.hostname = hostname;
    return transport::tcp::tls::CreateDevice(a, pkey, cert, caFile, caPath);
  }, py::arg("hostname"), py::arg("pkey"), py::arg("cert"), py::arg("ca_file") = "", py::arg("ca_path") = "");
  m.def("tls_available", &transport::tcp::tls::opensslAvailable);
  m.def("create_uv_device", [](const std::string& hostname, const std::string& iface) {
    transport::uv::attr a;
    a.hostname = hostname;
    a.iface = iface;
    return transport::uv::CreateDevice(a);
  }, py::arg("hostname") = "", py::arg("iface") = "",
        "Reference-compatible name for the portable TCP transport; backed by the epoll transport here.");
  m.def("create_nvl_device", [](std::shared_ptr<transport::Device> control, int cudaDevice) {
    transport::nvl::attr a;
    a.control = std::move(control);
    a.cudaDevice = cudaDevice;
    return transport::nvl::CreateDevice(a);
  }, py::arg("control"), py::arg("cuda_device") = -1,
     "NVLink peer-memory transport: device pointers as unbound buffers (send / recv / put / get over NVLink), "
     "host pointers through `control`.");
  m.def("create_ibverbs_device", [](const std::string& name, int port, int index) {
    transport::ibverbs::attr a;
    a.name = name;
    a.port = port;
    a.index = index;
    return transport::ibverbs::CreateDevice(a);
  }, py::arg("name") = "", py::arg("port") = 1, py::arg("index") = 0,
        "Raises InvalidOperationError naming what is missing (library, HCA, or the verbs data path of this build).");
  m.def("ibverbs_device_names", &transport::ibverbs::getDeviceNames);
  m.def("ibverbs_probe", [] {
    auto p = transport::ibverbs::probe();
    py::dict d;
    d["library"] = p.libraryLoaded;
    d["devices"] = p.devices;
    d["peer_memory_module"] = p.peerMemoryModule;
    d["detail"] = p.detail;
    return d;
  });

  py::class_<transport::RemoteKey>(m, "RemoteKey")
      .def_readonly("rank", &transport::RemoteKey::rank)
      .def_readonly("size", &transport::RemoteKey::size)
      .def("serialize", &transport::RemoteKey::serialize);

  py::class_<transport::UnboundBuffer>(m, "UnboundBuffer")
      .def_readonly("size", &transport::UnboundBuffer::size)
      .def("send", [](transport::UnboundBuffer& b, int dst, uint64_t slot, size_t offset, long nbytes) {
        py::gil_scoped_release nogil;
        b.send(dst, slot, offset, nbytes < 0 ? transport::UnboundBuffer::kUnspecifiedByteCount : static_cast<size_t>(nbytes));
      }, py::arg("dst"), py::arg("slot"), py::arg("offset") = 0, py::arg("nbytes") = -1)
      .def("recv", [](transport::UnboundBuffer& b, py::object src, uint64_t slot, size_t offset, long nbytes) {
        std::vector<int> ranks;
        if (py::isinstance<py::int_>(src)) {
          ranks.push_back(src.cast<int>());
        } else {
          ranks = src.cast<std::vector<int>>();
        }
        py::gil_scoped_release nogil;
        b.recv(ranks, slot, offset, nbytes < 0 ? transport::UnboundBuffer::kUnspecifiedByteCount : static_cast<size_t>(nbytes));
      }, py::arg("src"), py::arg("slot"), py::arg("offset") = 0, py::arg("nbytes") = -1)
      .def("wait_recv", [](transport::UnboundBuffer& b, long timeoutMs) -> py::object {
        int rank = -1;
        bool ok;
        {
          py::gil_scoped_release nogil;
          ok = b.waitRecv(&rank, timeoutMs < 0 ? kUnsetTimeout : ms(timeoutMs));
        }
        if (!ok) return py::none();
        return py::int_(rank);
      }, py::arg("timeout_ms") = -1, "Returns the source rank, or None if the wait was aborted.")
      .def("wait_send", [](transport::UnboundBuffer& b, long timeoutMs) -> py::object {
        int rank = -1;
        bool ok;
        {
          py::gil_scoped_release nogil;
          ok = b.waitSend(&rank, timeoutMs < 0 ? kUnsetTimeout : ms(timeoutMs));
        }
        if (!ok) return py::none();
        return py::int_(rank);
      }, py::arg("timeout_ms") = -1)
      .def("abort_wait_recv", &transport::UnboundBuffer::abortWaitRecv)
      .def("abort_wait_send", &transport::UnboundBuffer::abortWaitSend)
      .def("get_remote_key", [](transport::UnboundBuffer& b) { return b.getRemoteKey()->serialize(); })
      .def("put", [](transport::UnboundBuffer& b, std::shared_ptr<Context> ctx, const std::string& key, uint64_t slot,
                     size_t offset, size_t roffset, size_t nbytes) {
        py::gil_scoped_release nogil;
        auto k = ctx->deserializeRemoteKey(key);
        b.put(*k, slot, offset, roffset, nbytes);
      })
      .def("get", [](transport::UnboundBuffer& b, std::shared_ptr<Context> ctx, const std::string& key, uint64_t slot,
                     size_t offset, size_t roffset, size_t nbytes) {
        py::gil_scoped_release nogil;
        auto k = ctx->deserializeRemoteKey(key);
        b.get(*k, slot, offset, roffset, nbytes);
      });

  py::class_<transport::Buffer>(m, "Buffer")
      .def("send", [](transport::Buffer& b, size_t offset, long length, size_t roffset) {
        py::gil_scoped_release nogil;
        b.send(offset, length < 0 ? b.size() - offset : static_cast<size_t>(length), roffset);
      }, py::arg("offset") = 0, py::arg("length") = -1, py::arg("roffset") = 0)
      .def("wait_recv", [](transport::Buffer& b) { py::gil_scoped_release nogil; b.waitRecv(); })
      .def("wait_send", [](transport::Buffer& b) { py::gil_scoped_release nogil; b.waitSend(); })
      .def("set_debug", &transport::Buffer::setDebug);

  py::class_<transport::Pair>(m, "Pair")
      .def("set_sync", [](transport::Pair& p, bool sync, bool busyPoll) {
        py::gil_scoped_release nogil;
        p.setSync(sync, busyPoll);
      }, py::arg("sync"), py::arg("busy_poll") = false)
      .def("is_connected", &transport::Pair::isConnected)
      .def("local_rank", &transport::Pair::getLocalRank)
      .def("close", [](transport::Pair& p) { py::gil_scoped_release nogil; p.close(); })
      .def("create_send_buffer", [](transport::Pair& p, int slot, uintptr_t ptr, size_t size) {
        return p.createSendBuffer(slot, P(ptr), size);
      }, py::keep_alive<0, 1>())
      .def("create_recv_buffer", [](transport::Pair& p, int slot, uintptr_t ptr, size_t size) {
        return p.createRecvBuffer(slot, P(ptr), size);
      }, py::keep_alive<0, 1>());

  // ---- contexts -------------------------------------------------------------------
  py::class_<Context, std::shared_ptr<Context>>(m, "BaseContext")
      .def_readonly("rank", &Context::rank)
      .def_readonly("size", &Context::size)
      .def_readwrite("base", &Context::base)
      .def("set_timeout", [](Context& c, long t) { c.setTimeout(ms(t)); })
      .def("get_timeout", [](Context& c) { return static_cast<long>(c.getTimeout().count()); })
      .def("next_slot", &Context::nextSlot, py::arg("num_slots") = 1)
      .def("close_connections", [](Context& c) { py::gil_scoped_release nogil; c.closeConnections(); })
      .def("get_pair", [](Context& c, int i) -> transport::Pair* {
        py::gil_scoped_release nogil;
        return c.getPair(i).get();
      }, py::return_value_policy::reference_internal)
      .def("device", [](Context& c) { return c.getDevice(); })
      .def("create_unbound_buffer", [](std::shared_ptr<Context> c, uintptr_t ptr, size_t size) {
        return c->createUnboundBuffer(P(ptr), size);
      }, py::keep_alive<0, 1>());
  py::class_<rendezvous::Context, Context, std::shared_ptr<rendezvous::Context>>(m, "Context")
      .def(py::init<int, int, int>(), py::arg("rank"), py::arg("size"), py::arg("base") = 2)
      .def("connect_full_mesh", [](rendezvous::Context& c, std::shared_ptr<IStore> store,
                                   std::shared_ptr<transport::Device> dev) {
        py::gil_scoped_release nogil;
        c.connectFullMesh(std::move(store), dev);
      });
  py::class_<rendezvous::ContextFactory>(m, "ContextFactory")
      .def(py::init<std::shared_ptr<Context>>())
      .def("make_context", [](rendezvous::ContextFactory& f, std::shared_ptr<transport::Device> dev) {
        py::gil_scoped_release nogil;
        return f.makeContext(dev);
      });

  // ---- new-style collectives ------------------------------------------------------
  m.def("allreduce", [](std::shared_ptr<Context> ctx, std::vector<uintptr_t> inputs, std::vector<uintptr_t> outputs,
                        size_t count, int dtype, int op, int algorithm, uint32_t tag, long timeoutMs,
                        size_t maxSegment, py::object custom) {
    AllreduceOptions opts(ctx);
    const size_t es = elementSize(static_cast<DataType>(dtype));
    if (!inputs.empty()) opts.setInputsRaw(toPtrs(inputs), count, es);
    opts.setOutputsRaw(toPtrs(outputs), count, es);
    opts.setReduceFunction(pickReduce(dtype, op, custom));
    opts.setAlgorithm(static_cast<AllreduceOptions::Algorithm>(algorithm));
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    if (maxSegment > 0) opts.setMaxSegmentSize(maxSegment);
    py::gil_scoped_release nogil;
    allreduce(opts);
  }, py::arg("ctx"), py::arg("inputs"), py::arg("outputs"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1,
     py::arg("algorithm") = 0, py::arg("tag") = 0, py::arg("timeout_ms") = -1, py::arg("max_segment") = 0,
     py::arg("custom") = py::none());

  m.def("reduce", [](std::shared_ptr<Context> ctx, uintptr_t input, uintptr_t output, size_t count, int dtype, int op,
                     int root, uint32_t tag, long timeoutMs, py::object custom) {
    ReduceOptions opts(ctx);
    const size_t es = elementSize(static_cast<DataType>(dtype));
    if (input) opts.setInputRaw(P(input), count, es);
    opts.setOutputRaw(P(output), count, es);
    opts.setReduceFunction(pickReduce(dtype, op, custom));
    opts.setRoot(root);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    reduce(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("output"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1,
     py::arg("root") = 0, py::arg("tag") = 0, py::arg("timeout_ms") = -1, py::arg("custom") = py::none());

  m.def("reduce_scatter", [](std::shared_ptr<Context> ctx, uintptr_t input, uintptr_t output, size_t totalCount,
                             std::vector<size_t> recvCounts, int dtype, int op, uint32_t tag, long timeoutMs) {
    ReduceScatterOptions opts(ctx);
    const size_t es = elementSize(static_cast<DataType>(dtype));
    opts.setInputRaw(P(input), totalCount, es);
    size_t mine = recvCounts.empty() ? detail::subRange({0, totalCount}, ctx->size, ctx->rank).len : recvCounts[ctx->rank];
    opts.setOutputRaw(P(output), mine, es);
    opts.setRecvCounts(std::move(recvCounts));
    opts.setReduceFunction(reduceFnFor(dtype, op));
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    reduce_scatter(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("output"), py::arg("total_count"), py::arg("recv_counts"),
     py::arg("dtype"), py::arg("op") = 1, py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("broadcast", [](std::shared_ptr<Context> ctx, uintptr_t input, uintptr_t output, size_t nbytes, int root,
                        uint32_t tag, long timeoutMs) {
    BroadcastOptions opts(ctx);
    if (input) opts.setInputRaw(P(input), nbytes);
    opts.setOutputRaw(P(output), nbytes);
    opts.setRoot(root);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    broadcast(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("output"), py::arg("nbytes"), py::arg("root") = 0, py::arg("tag") = 0,
     py::arg("timeout_ms") = -1);

  m.def("allgather", [](std::shared_ptr<Context> ctx, uintptr_t input, size_t inBytes, uintptr_t output,
                        size_t outBytes, uint32_t tag, long timeoutMs) {
    AllgatherOptions opts(ctx);
    if (input) opts.setInputRaw(P(input), inBytes);
    opts.setOutputRaw(P(output), outBytes);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    allgather(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("in_bytes"), py::arg("output"), py::arg("out_bytes"),
     py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("allgatherv", [](std::shared_ptr<Context> ctx, uintptr_t input, uintptr_t output, std::vector<size_t> counts,
                         size_t elemSize, uint32_t tag, long timeoutMs) {
    AllgathervOptions opts(ctx);
    if (input) opts.setInputRaw(P(input), counts.at(ctx->rank), elemSize);
    opts.setOutputRaw(P(output), counts, elemSize);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    allgatherv(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("output"), py::arg("counts"), py::arg("elem_size"),
     py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("alltoall", [](std::shared_ptr<Context> ctx, uintptr_t input, uintptr_t output, size_t nbytes, uint32_t tag,
                       long timeoutMs) {
    AlltoallOptions opts(ctx);
    opts.setInputRaw(P(input), nbytes);
    opts.setOutputRaw(P(output), nbytes);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    alltoall(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("output"), py::arg("nbytes"), py::arg("tag") = 0,
     py::arg("timeout_ms") = -1);

  m.def("alltoallv", [](std::shared_ptr<Context> ctx, uintptr_t input, std::vector<int64_t> inCounts,
                        uintptr_t output, std::vector<int64_t> outCounts, size_t elemSize, uint32_t tag,
                        long timeoutMs) {
    AlltoallvOptions opts(ctx);
    opts.setInputRaw(P(input), std::move(inCounts), elemSize);
    opts.setOutputRaw(P(output), std::move(outCounts), elemSize);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    alltoallv(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("in_counts"), py::arg("output"), py::arg("out_counts"),
     py::arg("elem_size"), py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("gather", [](std::shared_ptr<Context> ctx, uintptr_t input, size_t inBytes, uintptr_t output, int root,
                     uint32_t tag, long timeoutMs) {
    GatherOptions opts(ctx);
    opts.setInputRaw(P(input), inBytes);
    if (ctx->rank == root) opts.setOutputRaw(P(output), inBytes * ctx->size);
    opts.setRoot(root);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    gather(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("in_bytes"), py::arg("output"), py::arg("root") = 0,
     py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("gatherv", [](std::shared_ptr<Context> ctx, uintptr_t input, size_t inCount, uintptr_t output,
                      std::vector<size_t> counts, size_t elemSize, int root, uint32_t tag, long timeoutMs) {
    GathervOptions opts(ctx);
    opts.setInputRaw(P(input), inCount, elemSize);
    if (ctx->rank == root) opts.setOutputRaw(P(output), std::move(counts), elemSize);
    opts.setRoot(root);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    gatherv(opts);
  }, py::arg("ctx"), py::arg("input"), py::arg("in_count"), py::arg("output"), py::arg("counts"),
     py::arg("elem_size"), py::arg("root") = 0, py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("scatter", [](std::shared_ptr<Context> ctx, std::vector<uintptr_t> inputs, uintptr_t output, size_t nbytes,
                      int root, uint32_t tag, long timeoutMs) {
    ScatterOptions opts(ctx);
    if (ctx->rank == root) opts.setInputsRaw(toPtrs(inputs), nbytes);
    opts.setOutputRaw(P(output), nbytes);
    opts.setRoot(root);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    scatter(opts);
  }, py::arg("ctx"), py::arg("inputs"), py::arg("output"), py::arg("nbytes"), py::arg("root") = 0,
     py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  m.def("barrier", [](std::shared_ptr<Context> ctx, uint32_t tag, long timeoutMs) {
    BarrierOptions opts(ctx);
    opts.setTag(tag);
    opts.setTimeout(toMs(timeoutMs, ctx));
    py::gil_scoped_release nogil;
    barrier(opts);
  }, py::arg("ctx"), py::arg("tag") = 0, py::arg("timeout_ms") = -1);

  glb_py::registerOldStyle(m);
  glb_py::registerCuda(m);
  glb_py::registerExtras(m);
}
