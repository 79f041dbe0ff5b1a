// pybind11 bindings for the CUDA side: PeerContext (topology + symmetric memory),
// peer buffers, fused collectives, tuning knobs, test helpers.
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "glb/cuda/collectives.h"
#include "glb/cuda/cuda_util.h"
#include "glb/cuda/kernels.h"
#include "glb/cuda/peer_context.h"
#include "glb/cuda/selftest.h"
#include "glb/cuda/tuning.h"
#include "glb/cuda/stream.h"

namespace py = pybind11;
using namespace glb;
using namespace glb::cuda;

namespace glb_py {

void registerCudaAlgorithms(py::module_& m);  // bindings_cuda_algorithms.cc

namespace {
inline void* P(uintptr_t p) { return reinterpret_cast<void*>(p); }
inline cudaStream_t S(uintptr_t s) { return reinterpret_cast<cudaStream_t>(s); }

Epilogue makeEpilogue(double scale, int outDtype, const std::vector<uintptr_t>& extra, int blocks, int unroll, int tile) {
  Epilogue ep;
  ep.scale = scale;
  if (outDtype >= 0) {
    ep.castOutput = true;
    ep.outDtype = static_cast<DataType>(outDtype);
  }
  GLB_ENFORCE_LE(extra.size(), static_cast<size_t>(kMaxLocal), "at most ", kMaxLocal, " extra local pointers");
  ep.extra.n = static_cast<int>(extra.size());
  for (size_t i = 0; i < extra.size(); i++) ep.extra.p[i] = P(extra[i]);
  ep.blocks = blocks;
  ep.unroll = unroll;
  ep.tile = tile;
  return ep;
}
}  // namespace

void registerCuda(py::module_& root) {
  auto m = root.def_submodule("cuda", "NVLink peer-memory collectives");

  m.def("device_count", &deviceCount);
  m.def("device_pci_bus_id", &devicePCIBusId);
  m.attr("MAX_RANKS") = kMaxRanks;
  m.attr("THREADS") = kThreads;

  py::class_<DeviceInfo>(m, "DeviceInfo")
      .def_property_readonly("hostname", [](const DeviceInfo& d) { return std::string(d.hostname); })
      .def_readonly("pid", &DeviceInfo::pid)
      .def_readonly("device", &DeviceInfo::device)
      .def_property_readonly("uuid", [](const DeviceInfo& d) {
        return py::bytes(reinterpret_cast<const char*>(d.uuid), 16);
      })
      .def_property_readonly("pci_bus_id", [](const DeviceInfo& d) { return std::string(d.pciBusId); })
      .def_readonly("sm_count", &DeviceInfo::smCount)
      .def_readonly("cc_major", &DeviceInfo::ccMajor)
      .def_readonly("cc_minor", &DeviceInfo::ccMinor)
      .def_readonly("vmm_supported", &DeviceInfo::vmmSupported)
      .def_readonly("multicast_supported", &DeviceInfo::multicastSupported)
      .def_readonly("total_mem", &DeviceInfo::totalMem)
      .def_readonly("nvlink_active", &DeviceInfo::nvlinkActive)
      .def_readonly("nvlink_version", &DeviceInfo::nvlinkVersion)
      .def_readonly("nic_distance", &DeviceInfo::nicDistance)
      .def_property_readonly("nearest_nic", [](const DeviceInfo& d) { return std::string(d.nearestNic); });

  py::class_<PeerBuffer, std::shared_ptr<PeerBuffer>>(m, "PeerBuffer")
      .def_property_readonly("ptr", [](const PeerBuffer& b) { return reinterpret_cast<uintptr_t>(b.local); })
      .def_readonly("nbytes", &PeerBuffer::bytes)
      .def_readonly("vector_ok", &PeerBuffer::vectorOk)
      .def_property_readonly("has_multicast", [](const PeerBuffer& b) { return b.mc != nullptr; })
      .def_property_readonly("multicast_ptr", [](const PeerBuffer& b) { return reinterpret_cast<uintptr_t>(b.mc); })
      .def("peer_ptr", [](const PeerBuffer& b, int r) { return reinterpret_cast<uintptr_t>(b.peer[r]); });

  py::class_<PeerContext, std::shared_ptr<PeerContext>>(m, "PeerContext")
      .def(py::init([](std::shared_ptr<Context> ctx, int device, size_t stageBytes, bool useVmm, bool useNvls) {
        PeerOptions o;
        if (stageBytes > 0) o.stageBytes = stageBytes;
        o.useVmm = useVmm;
        o.useNvls = useNvls;
        py::gil_scoped_release nogil;
        return std::make_shared<PeerContext>(std::move(ctx), device, o);
      }), py::arg("ctx"), py::arg("device"), py::arg("stage_bytes") = 0, py::arg("use_vmm") = true,
          py::arg("use_nvls") = true)
      .def_readonly("rank", &PeerContext::rank)
      .def_readonly("size", &PeerContext::size)
      .def_readonly("device", &PeerContext::device)
      .def("topology", &PeerContext::topology)
      .def("peer_access_everywhere", &PeerContext::peerAccessEverywhere)
      .def("using_vmm", &PeerContext::usingVmm)
      .def("nvls_available", &PeerContext::nvlsAvailable)
      .def("ranks_on_my_device", &PeerContext::ranksOnMyDevice)
      .def("max_blocks", &PeerContext::maxBlocks)
      .def("stage_bytes", &PeerContext::stageBytes)
      .def("describe", &PeerContext::describe)
      .def("alloc_symmetric", [](PeerContext& pc, size_t bytes) {
        py::gil_scoped_release nogil;
        return pc.allocSymmetric(bytes);
      })
      .def("register_buffer", [](PeerContext& pc, uintptr_t ptr, size_t bytes) {
        py::gil_scoped_release nogil;
        return pc.registerBuffer(P(ptr), bytes);
      })
      .def("host_barrier", [](PeerContext& pc) {
        py::gil_scoped_release nogil;
        pc.hostBarrier();
      })
      .def("host_all_same", [](PeerContext& pc, std::vector<int64_t> words) {
        py::gil_scoped_release nogil;
        return pc.hostAllSame(words);
      }, "Collective: whether every rank passed the same list of at most 16 integers.")
      .def("set_timeout", [](PeerContext& pc, long ms) { pc.setTimeout(std::chrono::milliseconds(ms)); },
           "Device-side waits give up after this many milliseconds (0 = never).")
      .def("timeout_ms", [](PeerContext& pc) { return static_cast<long>(pc.timeout().count()); })
      .def("check_health", &PeerContext::checkHealth, "Raises IoException if a device-side wait has timed out.")
      .def("poisoned", &PeerContext::poisoned)
      .def("synchronize", [](PeerContext& pc, uintptr_t stream) {
        py::gil_scoped_release nogil;
        pc.synchronize(S(stream));
      }, py::arg("stream") = 0, "cudaStreamSynchronize + check_health")
      .def("ll_max_bytes", &PeerContext::llMaxBytes)
      .def("co_resident_blocks_two_shot", [](PeerContext& pc, int dtype, int unroll) {
        return pc.coResidentBlocks(twoShotKernelFor(static_cast<DataType>(dtype), pc.size, unroll));
      })
      .def("loopback_selftest", [](PeerContext& pc, uintptr_t stream, size_t count) {
        std::vector<SelfTestResult> res;
        {
          py::gil_scoped_release nogil;
          res = loopbackSelfTest(pc, S(stream), count);
        }
        py::list out;
        for (const auto& r : res) {
          py::dict d;
          d["name"] = r.name;
          d["ok"] = r.ok;
          d["skipped"] = r.skipped;
          d["detail"] = r.detail;
          out.append(d);
        }
        return out;
      }, py::arg("stream") = 0, py::arg("count") = size_t(1) << 18,
         "Run every hot kernel with 2/4/8 virtual ranks on this GPU (profiler safe) and check the results.")
      .def("loopback_timeout_test", [](PeerContext& pc, uintptr_t stream, int timeoutMs) {
        double ms = 0;
        bool raised;
        {
          py::gil_scoped_release nogil;
          raised = loopbackTimeoutTest(pc, S(stream), timeoutMs, &ms);
        }
        return py::make_tuple(raised, ms);
      }, py::arg("stream") = 0, py::arg("timeout_ms") = 200);

  m.def("barrier", [](PeerContext& pc, uintptr_t stream) {
    py::gil_scoped_release nogil;
    barrier(pc, S(stream));
  }, py::arg("pc"), py::arg("stream") = 0);

  m.def("allreduce_registered", [](PeerContext& pc, const PeerBuffer& buf, size_t byteOffset, size_t count, int dtype,
                                   int op, int algo, uintptr_t stream, double scale, std::vector<uintptr_t> extra,
                                   int blocks, int unroll, int tile) {
    const Epilogue ep = makeEpilogue(scale, -1, extra, blocks, unroll, tile);
    py::gil_scoped_release nogil;
    allreduce(pc, buf, byteOffset, count, static_cast<DataType>(dtype), static_cast<ReduceOp>(op),
              static_cast<AllreduceAlgo>(algo), S(stream), ep);
  }, py::arg("pc"), py::arg("buf"), py::arg("byte_offset"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1,
     py::arg("algo") = 0, py::arg("stream") = 0, py::arg("scale") = 1.0, py::arg("extra") = std::vector<uintptr_t>(),
     py::arg("blocks") = 0, py::arg("unroll") = 0, py::arg("tile") = 0);

  m.def("allreduce", [](PeerContext& pc, uintptr_t in, uintptr_t out, size_t count, int dtype, int op, int algo,
                        uintptr_t stream, double scale, int outDtype, std::vector<uintptr_t> extra, int blocks,
                        int tile, int unroll) {
    const Epilogue ep = makeEpilogue(scale, outDtype, extra, blocks, unroll, tile);
    py::gil_scoped_release nogil;
    allreduce(pc, P(in), P(out), count, static_cast<DataType>(dtype), static_cast<ReduceOp>(op),
              static_cast<AllreduceAlgo>(algo), S(stream), ep);
  }, py::arg("pc"), py::arg("input"), py::arg("output"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1,
     py::arg("algo") = 0, py::arg("stream") = 0, py::arg("scale") = 1.0, py::arg("out_dtype") = -1,
     py::arg("extra") = std::vector<uintptr_t>(), py::arg("blocks") = 0, py::arg("tile") = 0, py::arg("unroll") = 0);

  m.def("allreduce_cast", [](PeerContext& pc, const PeerBuffer& in, size_t inOff, const PeerBuffer& out, size_t outOff,
                             size_t count, int dtype, int outDtype, int op, uintptr_t stream, double scale, int blocks) {
    Epilogue ep;
    ep.scale = scale;
    ep.blocks = blocks;
    py::gil_scoped_release nogil;
    allreduceCast(pc, in, inOff, out, outOff, count, static_cast<DataType>(dtype), static_cast<DataType>(outDtype),
                  static_cast<ReduceOp>(op), S(stream), ep);
  }, py::arg("pc"), py::arg("input"), py::arg("in_offset"), py::arg("output"), py::arg("out_offset"), py::arg("count"),
     py::arg("dtype"), py::arg("out_dtype"), py::arg("op") = 1, py::arg("stream") = 0, py::arg("scale") = 1.0,
     py::arg("blocks") = 0);

  m.def("allreduce_residual_norm", [](PeerContext& pc, uintptr_t partial, uintptr_t residual, uintptr_t residualOut,
                                      uintptr_t out, uintptr_t bias, uintptr_t gamma, uintptr_t beta, size_t rows,
                                      size_t hidden, int dtype, int norm, double eps, int algo, uintptr_t stream,
                                      uintptr_t outScales) {
    int v;
    {
      py::gil_scoped_release nogil;
      v = allreduceResidualNorm(pc, P(partial), P(residual), P(residualOut), P(out), P(bias), P(gamma), P(beta), rows,
                                hidden, static_cast<DataType>(dtype), norm, static_cast<float>(eps),
                                static_cast<AllreduceAlgo>(algo), S(stream), reinterpret_cast<float*>(outScales));
    }
    return std::string(normVariantName(v));
  }, py::arg("pc"), py::arg("partial"), py::arg("residual"), py::arg("residual_out"), py::arg("out"), py::arg("bias"),
     py::arg("gamma"), py::arg("beta"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"),
     py::arg("eps"), py::arg("algo") = 0, py::arg("stream") = 0, py::arg("out_scales") = 0,
     "Allreduce of partial sums fused with bias, residual add and a norm (0 none, 1 rms, 2 layer); null pointers are 0. "
     "out_scales set: out holds e4m3 codes and out_scales one fp32 scale per row. Returns the variant that ran.");
  m.def("plan_residual_norm", [](PeerContext& pc, size_t rows, size_t hidden, int dtype, int norm, int algo, bool fp8) {
    const NormPlan p = planResidualNorm(pc, rows, hidden, static_cast<DataType>(dtype), norm,
                                        static_cast<AllreduceAlgo>(algo), fp8);
    py::dict d;
    d["variant"] = std::string(normVariantName(p.variant));
    d["chunk_rows"] = p.chunkRows;
    d["launches"] = p.launches;
    return d;
  }, py::arg("pc"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"), py::arg("algo") = 0,
     py::arg("fp8") = false);
  m.def("reduce_scatter_residual_norm", [](PeerContext& pc, uintptr_t partial, uintptr_t residual,
                                           uintptr_t residualOut, uintptr_t out, uintptr_t bias, uintptr_t gamma,
                                           uintptr_t beta, size_t rows, size_t hidden, int dtype, int norm, double eps,
                                           bool gatherOut, uintptr_t stream, uintptr_t outScales) {
    int v;
    {
      py::gil_scoped_release nogil;
      v = reduceScatterResidualNorm(pc, P(partial), P(residual), P(residualOut), P(out), P(bias), P(gamma), P(beta),
                                    rows, hidden, static_cast<DataType>(dtype), norm, static_cast<float>(eps),
                                    gatherOut, S(stream), reinterpret_cast<float*>(outScales));
    }
    return std::string(normVariantName(v));
  }, py::arg("pc"), py::arg("partial"), py::arg("residual"), py::arg("residual_out"), py::arg("out"), py::arg("bias"),
     py::arg("gamma"), py::arg("beta"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"),
     py::arg("eps"), py::arg("gather_out") = true, py::arg("stream") = 0, py::arg("out_scales") = 0,
     "Reduce-scatter of partial sums over row shards fused with bias, residual add and a norm (0 none, 1 rms, "
     "2 layer), out optionally allgathered; rows is the full row count; null pointers are 0. out_scales set: out "
     "holds e4m3 codes and out_scales one fp32 scale per row. Returns the variant that ran.");
  m.def("plan_reduce_scatter_norm", [](PeerContext& pc, size_t rows, size_t hidden, int dtype, int norm,
                                       bool gatherOut, bool fp8) {
    const NormPlan p = planReduceScatterNorm(pc, rows, hidden, static_cast<DataType>(dtype), norm, gatherOut, fp8);
    py::dict d;
    d["variant"] = std::string(normVariantName(p.variant));
    d["chunk_rows"] = p.chunkRows;
    d["launches"] = p.launches;
    return d;
  }, py::arg("pc"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"), py::arg("gather_out") = true,
     py::arg("fp8") = false);
  m.def("reduce_scatter_residual_norm_backward", [](PeerContext& pc, uintptr_t gradOut, uintptr_t s, uintptr_t gradS,
                                                    uintptr_t gradResidual, uintptr_t gradPartial, uintptr_t gamma,
                                                    uintptr_t gradWeight, uintptr_t gradNormBias, uintptr_t gradBias,
                                                    uintptr_t workspace, size_t workspaceBytes, size_t rows,
                                                    size_t hidden, int dtype, int norm, double eps, bool gatherOut,
                                                    uintptr_t stream) {
    int v;
    {
      py::gil_scoped_release nogil;
      v = reduceScatterResidualNormBackward(pc, P(gradOut), P(s), P(gradS), P(gradResidual), P(gradPartial), P(gamma),
                                            P(gradWeight), P(gradNormBias), P(gradBias), P(workspace), workspaceBytes,
                                            rows, hidden, static_cast<DataType>(dtype), norm, static_cast<float>(eps),
                                            gatherOut, S(stream));
    }
    return std::string(normVariantName(v));
  }, py::arg("pc"), py::arg("grad_out"), py::arg("residual_out"), py::arg("grad_residual_out"),
     py::arg("grad_residual"), py::arg("grad_partial"), py::arg("weight"), py::arg("grad_weight"),
     py::arg("grad_norm_bias"), py::arg("grad_bias"), py::arg("workspace"), py::arg("workspace_bytes"),
     py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"), py::arg("eps"),
     py::arg("gather_out") = true, py::arg("stream") = 0,
     "Backward of reduce_scatter_residual_norm with a norm (1 rms, 2 layer): the norm's backward on this rank's "
     "shard, reduce-scatter of a gathered grad_out before it and allgather of grad_residual into grad_partial "
     "after it, in one kernel; optional column sums (weight, norm bias, bias) need the plan's workspace. rows is "
     "the full row count; null pointers are 0. Returns the variant that ran.");
  m.def("plan_reduce_scatter_norm_backward", [](PeerContext& pc, size_t rows, size_t hidden, int dtype, int norm,
                                                bool gatherOut, int vectors) {
    const NormBackwardPlan p =
        planReduceScatterNormBackward(pc, rows, hidden, static_cast<DataType>(dtype), norm, gatherOut, vectors);
    py::dict d;
    d["variant"] = std::string(normVariantName(p.variant));
    d["chunk_rows"] = p.chunkRows;
    d["launches"] = p.launches;
    d["blocks"] = p.blocks;
    d["workspace_bytes"] = p.workspaceBytes;
    return d;
  }, py::arg("pc"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"), py::arg("gather_out") = true,
     py::arg("vectors") = 0);
  m.def("allreduce_residual_norm_backward", [](PeerContext& pc, uintptr_t gradOut, uintptr_t s, uintptr_t gradS,
                                               uintptr_t gradPartial, uintptr_t gamma, uintptr_t gradWeight,
                                               uintptr_t gradNormBias, uintptr_t gradBias, uintptr_t workspace,
                                               size_t workspaceBytes, size_t rows, size_t hidden, int dtype, int norm,
                                               double eps, int algo, uintptr_t stream) {
    int v;
    {
      py::gil_scoped_release nogil;
      v = allreduceResidualNormBackward(pc, P(gradOut), P(s), P(gradS), P(gradPartial), P(gamma), P(gradWeight),
                                        P(gradNormBias), P(gradBias), P(workspace), workspaceBytes, rows, hidden,
                                        static_cast<DataType>(dtype), norm, static_cast<float>(eps),
                                        static_cast<AllreduceAlgo>(algo), S(stream));
    }
    return std::string(normVariantName(v));
  }, py::arg("pc"), py::arg("grad_out"), py::arg("residual_out"), py::arg("grad_residual_out"),
     py::arg("grad_partial"), py::arg("weight"), py::arg("grad_weight"), py::arg("grad_norm_bias"),
     py::arg("grad_bias"), py::arg("workspace"), py::arg("workspace_bytes"), py::arg("rows"), py::arg("hidden"),
     py::arg("dtype"), py::arg("norm"), py::arg("eps"), py::arg("algo") = 0, py::arg("stream") = 0,
     "Backward of allreduce_residual_norm with a norm (1 rms, 2 layer): allreduce of this rank's partial grad_out, "
     "the norm's backward and the add of grad_residual_out into grad_partial, in one kernel; optional column sums "
     "(weight, norm bias, bias) need the plan's workspace. Null pointers are 0. Returns the variant that ran.");
  m.def("plan_residual_norm_backward", [](PeerContext& pc, size_t rows, size_t hidden, int dtype, int norm,
                                          int vectors, int algo) {
    const NormBackwardPlan p = planResidualNormBackward(pc, rows, hidden, static_cast<DataType>(dtype), norm, vectors,
                                                        static_cast<AllreduceAlgo>(algo));
    py::dict d;
    d["variant"] = std::string(normVariantName(p.variant));
    d["chunk_rows"] = p.chunkRows;
    d["launches"] = p.launches;
    d["blocks"] = p.blocks;
    d["workspace_bytes"] = p.workspaceBytes;
    return d;
  }, py::arg("pc"), py::arg("rows"), py::arg("hidden"), py::arg("dtype"), py::arg("norm"), py::arg("vectors"),
     py::arg("algo") = 0);
  m.attr("MAX_NORM_HIDDEN") = kMaxNormHidden;

  m.def("plan_allreduce", [](PeerContext& pc, size_t bytes, int dtype, int op, int kind) {
    AllreducePlan p = planAllreduce(pc, bytes, static_cast<DataType>(dtype), static_cast<ReduceOp>(op),
                                    static_cast<BufKind>(kind));
    py::dict d;
    d["algo"] = std::string(allreduceAlgoName(p.algo));
    d["blocks"] = p.cfg.blocks;
    d["unroll"] = p.cfg.unroll;
    d["tile"] = p.tile;
    d["from_table"] = p.fromTable;
    return d;
  }, py::arg("pc"), py::arg("bytes"), py::arg("dtype"), py::arg("op") = 1, py::arg("kind") = 0,
     "What AUTO resolves to (kind: 0 symmetric+multicast, 1 registered, 2 plain pointer).");

  // ---- point to point / one-sided ------------------------------------------------------
  m.def("send", [](PeerContext& pc, uintptr_t p, size_t bytes, int dst, uintptr_t st) {
    py::gil_scoped_release nogil;
    send(pc, P(p), bytes, dst, S(st));
  }, py::arg("pc"), py::arg("ptr"), py::arg("bytes"), py::arg("dst"), py::arg("stream") = 0);
  m.def("recv", [](PeerContext& pc, uintptr_t p, size_t bytes, int src, uintptr_t st) {
    py::gil_scoped_release nogil;
    recv(pc, P(p), bytes, src, S(st));
  }, py::arg("pc"), py::arg("ptr"), py::arg("bytes"), py::arg("src"), py::arg("stream") = 0);
  m.def("sendrecv", [](PeerContext& pc, uintptr_t sp, size_t sbytes, int dst, uintptr_t rp, size_t rbytes, int src,
                       uintptr_t st) {
    py::gil_scoped_release nogil;
    sendrecv(pc, P(sp), sbytes, dst, P(rp), rbytes, src, S(st));
  }, py::arg("pc"), py::arg("send_ptr"), py::arg("send_bytes"), py::arg("dst"), py::arg("recv_ptr"),
     py::arg("recv_bytes"), py::arg("src"), py::arg("stream") = 0);
  m.def("exchange", [](PeerContext& pc, uintptr_t sp, size_t sbytes, int dst, const PeerBuffer& rbuf, size_t roff,
                       size_t rbytes, int src, uintptr_t st) {
    py::gil_scoped_release nogil;
    exchange(pc, P(sp), sbytes, dst, rbuf, roff, rbytes, src, S(st));
  }, py::arg("pc"), py::arg("send_ptr"), py::arg("send_bytes"), py::arg("dst"), py::arg("recv_buf"),
     py::arg("recv_offset"), py::arg("recv_bytes"), py::arg("src"), py::arg("stream") = 0);
  m.def("put", [](PeerContext& pc, uintptr_t local, const PeerBuffer& remote, size_t off, size_t bytes, int peer,
                  uintptr_t st) {
    py::gil_scoped_release nogil;
    put(pc, P(local), remote, off, bytes, peer, S(st));
  }, py::arg("pc"), py::arg("local"), py::arg("remote"), py::arg("remote_offset"), py::arg("bytes"), py::arg("peer"),
     py::arg("stream") = 0);
  m.def("get", [](PeerContext& pc, uintptr_t local, const PeerBuffer& remote, size_t off, size_t bytes, int peer,
                  uintptr_t st) {
    py::gil_scoped_release nogil;
    get(pc, P(local), remote, off, bytes, peer, S(st));
  }, py::arg("pc"), py::arg("local"), py::arg("remote"), py::arg("remote_offset"), py::arg("bytes"), py::arg("peer"),
     py::arg("stream") = 0);

  m.def("set_local_shape", [](int ctas, int unroll, bool tiled) { setLocalAllreduceShape(ctas, unroll, tiled); },
        py::arg("ctas_per_sm"), py::arg("unroll"), py::arg("tiled") = false);
  m.def("local_ops_selftest", [](std::vector<int> devices, size_t count) {
    std::vector<SelfTestResult> res;
    {
      py::gil_scoped_release nogil;
      res = localOpsSelfTest(devices, count);
    }
    py::list out;
    for (const auto& r : res) {
      py::dict d;
      d["name"] = r.name;
      d["ok"] = r.ok;
      d["detail"] = r.detail;
      out.append(d);
    }
    return out;
  }, py::arg("devices"), py::arg("count") = 100003,
     "Exercise the LocalOp classes (CudaLocalMemcpy / Native / Host / NCCL reduce + broadcast, dispatchers).");

  // ---- tuning table ---------------------------------------------------------------------
  m.def("tuning_load_file", [](const std::string& path) {
    std::string err;
    int n = TuningTable::get().loadFile(path, &err);
    if (n < 0) GLB_THROW_INVALID_OPERATION_EXCEPTION("tuning table: ", err);
    return n;
  });
  m.def("tuning_load_string", [](const std::string& text) {
    std::string err;
    return TuningTable::get().loadString(text, &err);
  });
  m.def("tuning_clear", [] { TuningTable::get().clear(); });
  m.def("tuning_dump", [] { return TuningTable::get().dump(); });
  m.def("tuning_source", [] { return TuningTable::get().source(); });
  m.def("tuning_lookup", [](const std::string& coll, int P, int kind, size_t bytes) -> py::object {
    const TuneEntry* e = TuningTable::get().lookup(coll, P, static_cast<BufKind>(kind), bytes);
    if (e == nullptr) return py::none();
    py::dict d;
    d["algo"] = e->algo;
    d["blocks"] = e->blocks;
    d["unroll"] = e->unroll;
    d["tile"] = e->tile;
    d["maxbytes"] = e->maxBytes;
    return d;
  });

  m.def("choose_allreduce", [](PeerContext& pc, size_t bytes, int dtype, int op, bool registered, bool mc) {
    return static_cast<int>(chooseAllreduce(pc, bytes, static_cast<DataType>(dtype), static_cast<ReduceOp>(op),
                                            registered, mc));
  });
  m.def("allreduce_algo_name", [](int a) { return std::string(allreduceAlgoName(static_cast<AllreduceAlgo>(a))); });

  // Dedicated (never pooled / shared) streams: torch.cuda.Stream() hands out streams from
  // a 32-entry pool, so two ranks living in one process can end up on the same stream —
  // fatal for kernels that wait for each other on the device.
  m.def("create_stream", [](int device, bool highPriority) {
    DeviceGuard g(device);
    int lo = 0, hi = 0;
    GLB_CUDA_CHECK(cudaDeviceGetStreamPriorityRange(&lo, &hi));
    cudaStream_t s = nullptr;
    GLB_CUDA_CHECK(cudaStreamCreateWithPriority(&s, cudaStreamNonBlocking, highPriority ? hi : lo));
    return reinterpret_cast<uintptr_t>(s);
  }, py::arg("device"), py::arg("high_priority") = false);
  m.def("destroy_stream", [](uintptr_t s) { cudaStreamDestroy(S(s)); });
  m.def("launch_count", &launchCount);
  m.def("get_tuning", [] {
    const auto& t = tuning();
    py::dict d;
    d["one_shot_max_bytes"] = t.oneShotMaxBytes;
    d["nvls_min_bytes"] = t.nvlsMinBytes;
    d["max_blocks"] = t.maxBlocks;
    d["one_shot_blocks"] = t.oneShotBlocks;
    d["ll_max_bytes"] = t.llMaxBytes;
    d["copy_blocks"] = t.copyBlocks;
    d["pipe_tile"] = t.pipeTile;
    d["pipe_exchange_threads"] = t.pipeExchangeThreads;
    return d;
  });
  m.def("set_tuning", [](py::dict d) {
    auto& t = tuning();
    if (d.contains("one_shot_max_bytes")) t.oneShotMaxBytes = d["one_shot_max_bytes"].cast<size_t>();
    if (d.contains("nvls_min_bytes")) t.nvlsMinBytes = d["nvls_min_bytes"].cast<size_t>();
    if (d.contains("max_blocks")) t.maxBlocks = d["max_blocks"].cast<int>();
    if (d.contains("one_shot_blocks")) t.oneShotBlocks = d["one_shot_blocks"].cast<int>();
    if (d.contains("nvls_reduce_scatter")) t.nvlsReduceScatter = d["nvls_reduce_scatter"].cast<bool>();
    if (d.contains("copy_blocks")) t.copyBlocks = d["copy_blocks"].cast<int>();
    if (d.contains("one_shot_push")) setOneShotPush(d["one_shot_push"].cast<bool>());
    if (d.contains("ll_max_bytes")) t.llMaxBytes = d["ll_max_bytes"].cast<size_t>();
    if (d.contains("pipe_tile")) t.pipeTile = d["pipe_tile"].cast<int>();
    if (d.contains("pipe_exchange_threads")) t.pipeExchangeThreads = d["pipe_exchange_threads"].cast<int>();
    if (d.contains("alltoallv_blocks")) t.alltoallvBlocks = d["alltoallv_blocks"].cast<int>();
    if (d.contains("tma_copies")) t.tmaCopies = d["tma_copies"].cast<bool>();
  });

  // ---- local ops / helpers ------------------------------------------------------------
  m.def("local_reduce", [](uintptr_t dst, uintptr_t src, size_t count, int dtype, int op, uintptr_t stream) {
    launchLocalReduce(P(dst), P(src), count, static_cast<DataType>(dtype), static_cast<ReduceOp>(op), S(stream));
    GLB_CUDA_CHECK(cudaGetLastError());
  }, py::arg("dst"), py::arg("src"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1, py::arg("stream") = 0);
  m.def("local_reduce_many", [](uintptr_t dst, std::vector<uintptr_t> srcs, size_t count, int dtype, int op,
                                uintptr_t stream) {
    std::vector<const void*> ps;
    for (auto s : srcs) ps.push_back(P(s));
    launchLocalReduceMany(P(dst), ps.data(), static_cast<int>(ps.size()), count, static_cast<DataType>(dtype),
                          static_cast<ReduceOp>(op), S(stream));
    GLB_CUDA_CHECK(cudaGetLastError());
  }, py::arg("dst"), py::arg("srcs"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1, py::arg("stream") = 0);
  m.def("local_broadcast", [](std::vector<uintptr_t> dsts, uintptr_t src, size_t bytes, uintptr_t stream) {
    std::vector<void*> ps;
    for (auto d : dsts) ps.push_back(P(d));
    launchLocalBroadcast(ps.data(), static_cast<int>(ps.size()), P(src), bytes, S(stream));
    GLB_CUDA_CHECK(cudaGetLastError());
  }, py::arg("dsts"), py::arg("src"), py::arg("bytes"), py::arg("stream") = 0);
  m.def("local_allreduce_many", [](std::vector<uintptr_t> bufs, size_t count, int dtype, int op, double scale,
                                   uintptr_t stream) {
    std::vector<void*> ps;
    for (auto b : bufs) ps.push_back(P(b));
    // A tile counter of this call's own, stream ordered: calls on different streams may overlap.
    unsigned int* tiles = nullptr;
    GLB_CUDA_CHECK(cudaMallocAsync(reinterpret_cast<void**>(&tiles), sizeof(*tiles), S(stream)));
    GLB_CUDA_CHECK(cudaMemsetAsync(tiles, 0, sizeof(*tiles), S(stream)));
    launchLocalAllreduceMany(ps.data(), static_cast<int>(ps.size()), count, static_cast<DataType>(dtype),
                             static_cast<ReduceOp>(op), static_cast<float>(scale), tiles, S(stream));
    noteLaunch();
    const cudaError_t launched = cudaGetLastError();
    GLB_CUDA_CHECK(cudaFreeAsync(tiles, S(stream)));
    GLB_CUDA_CHECK(launched);
  }, py::arg("bufs"), py::arg("count"), py::arg("dtype"), py::arg("op") = 1, py::arg("scale") = 1.0, py::arg("stream") = 0,
     "Every buffer := scale * reduce(all buffers), one kernel, one pass.");
  m.def("local_allreduce_many_uses_bulk", [](std::vector<uintptr_t> bufs, size_t count, int dtype) {
    std::vector<void*> ps;
    for (auto b : bufs) ps.push_back(P(b));
    return localAllreduceUsesBulk(ps.data(), static_cast<int>(ps.size()), count, static_cast<DataType>(dtype));
  }, py::arg("bufs"), py::arg("count"), py::arg("dtype"),
     "Whether local_allreduce_many runs the TMA bulk-copy kernel for these arguments (unless set_local_shape pinned "
     "the LDG/STG kernel).");
  // Whole-buffer closed-form check on the device: returns (mismatches, first bad index or -1).
  m.def("verify", [](uintptr_t buf, size_t count, int dtype, double start, double stride, double rtol, double atol,
                     uintptr_t stream) {
    unsigned long long* dres = nullptr;
    unsigned long long h[2] = {0ull, ~0ull};
    GLB_CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&dres), 16));
    GLB_CUDA_CHECK(cudaMemcpyAsync(dres, h, 16, cudaMemcpyHostToDevice, S(stream)));
    launchVerify(P(buf), count, static_cast<DataType>(dtype), start, stride, rtol, atol, dres, S(stream));
    noteLaunch();
    cudaError_t e1 = cudaMemcpyAsync(h, dres, 16, cudaMemcpyDeviceToHost, S(stream));
    cudaError_t e2 = cudaStreamSynchronize(S(stream));
    cudaFree(dres);
    GLB_CUDA_CHECK(e1);
    GLB_CUDA_CHECK(e2);
    return py::make_tuple(static_cast<size_t>(h[0]), h[1] == ~0ull ? static_cast<long long>(-1) : static_cast<long long>(h[1] - 1));
  }, py::arg("buf"), py::arg("count"), py::arg("dtype"), py::arg("start") = 0.0, py::arg("stride") = 1.0,
     py::arg("rtol") = 1e-5, py::arg("atol") = 0.0, py::arg("stream") = 0);
  m.def("fill", [](uintptr_t dst, size_t count, int dtype, double start, double stride, uintptr_t stream) {
    launchFill(P(dst), count, static_cast<DataType>(dtype), start, stride, S(stream));
    GLB_CUDA_CHECK(cudaGetLastError());
  }, py::arg("dst"), py::arg("count"), py::arg("dtype"), py::arg("start") = 0.0, py::arg("stride") = 1.0,
     py::arg("stream") = 0);
  m.def("spin", [](long long cycles, uintptr_t stream) {
    launchSpin(cycles, S(stream));
    GLB_CUDA_CHECK(cudaGetLastError());
  }, py::arg("cycles"), py::arg("stream") = 0);

  registerCudaAlgorithms(m);
}

}  // namespace glb_py
