// Old-style host Algorithm classes for Python: one type-erased handle created by
// name + dtype (the C++ API is templated; see csrc/glb/allreduce_ring.h etc.).
#include <pybind11/pybind11.h>
#include <pybind11/stl.h>

#include "glb/allgather_ring.h"
#include "glb/allreduce_bcube.h"
#include "glb/allreduce_halving_doubling.h"
#include "glb/allreduce_local.h"
#include "glb/allreduce_ring.h"
#include "glb/allreduce_ring_chunked.h"
#include "glb/barrier_all_to_all.h"
#include "glb/broadcast_one_to_all.h"
#include "glb/pairwise_exchange.h"
#include "glb/reduce_scatter_halving_doubling.h"

namespace py = pybind11;
using namespace glb;

namespace glb_py {

namespace {

template <typename T>
std::vector<T*> typed(const std::vector<uintptr_t>& v) {
  std::vector<T*> out;
  for (auto p : v) out.push_back(reinterpret_cast<T*>(p));
  return out;
}

template <typename T>
std::unique_ptr<Algorithm> makeTyped(const std::string& name, const std::shared_ptr<Context>& ctx,
                                     const std::vector<uintptr_t>& ptrs, size_t count, ReduceOp op, int root,
                                     int rootPtr, const std::vector<int>& recvElems, uintptr_t outPtr) {
  const ReductionFunction<T>* fn = ReductionFunction<T>::get(op);
  GLB_ENFORCE(fn != nullptr, "unsupported reduce op for old-style algorithm");
  if (name == "allreduce_ring") return std::make_unique<AllreduceRing<T>>(ctx, typed<T>(ptrs), count, fn);
  if (name == "allreduce_ring_chunked") return std::make_unique<AllreduceRingChunked<T>>(ctx, typed<T>(ptrs), count, fn);
  if (name == "allreduce_halving_doubling")
    return std::make_unique<AllreduceHalvingDoubling<T>>(ctx, typed<T>(ptrs), count, fn);
  if (name == "allreduce_bcube") return std::make_unique<AllreduceBcube<T>>(ctx, typed<T>(ptrs), count, fn);
  if (name == "allreduce_local") return std::make_unique<AllreduceLocal<T>>(ctx, typed<T>(ptrs), count, fn);
  if (name == "broadcast_one_to_all")
    return std::make_unique<BroadcastOneToAll<T>>(ctx, typed<T>(ptrs), count, root, rootPtr);
  if (name == "reduce_scatter_halving_doubling")
    return std::make_unique<ReduceScatterHalvingDoubling<T>>(ctx, typed<T>(ptrs), count, recvElems, fn);
  if (name == "allgather_ring") {
    std::vector<const T*> ins;
    for (auto p : ptrs) ins.push_back(reinterpret_cast<const T*>(p));
    return std::make_unique<AllgatherRing<T>>(ctx, ins, reinterpret_cast<T*>(outPtr), count);
  }
  GLB_THROW_INVALID_OPERATION_EXCEPTION("unknown algorithm: ", name);
}

}  // namespace

void registerOldStyle(py::module_& m) {
  py::class_<Algorithm>(m, "Algorithm").def("run", [](Algorithm& a) {
    py::gil_scoped_release nogil;
    a.run();
  });

  m.def("make_algorithm", [](const std::string& name, std::shared_ptr<Context> ctx, std::vector<uintptr_t> ptrs,
                             size_t count, int dtype, int op, int root, int rootPtr, std::vector<int> recvElems,
                             uintptr_t outPtr) -> std::unique_ptr<Algorithm> {
    py::gil_scoped_release nogil;
    const ReduceOp rop = static_cast<ReduceOp>(op);
    if (name == "barrier_all_to_all") return std::make_unique<BarrierAllToAll>(ctx);
    if (name == "barrier_all_to_one") return std::make_unique<BarrierAllToOne>(ctx, root);
    if (name == "pairwise_exchange") return std::make_unique<PairwiseExchange>(ctx, static_cast<int>(count), root);
    switch (static_cast<DataType>(dtype)) {
#define GLB_CASE(E, T) \
  case DataType::E: return makeTyped<T>(name, ctx, ptrs, count, rop, root, rootPtr, recvElems, outPtr);
      GLB_CASE(INT8, int8_t)
      GLB_CASE(UINT8, uint8_t)
      GLB_CASE(INT32, int32_t)
      GLB_CASE(INT64, int64_t)
      GLB_CASE(UINT64, uint64_t)
      GLB_CASE(FLOAT32, float)
      GLB_CASE(FLOAT64, double)
      GLB_CASE(FLOAT16, float16)
      GLB_CASE(BFLOAT16, bfloat16)
      GLB_CASE(FLOAT8_E4M3, float8_e4m3)
      GLB_CASE(FLOAT8_E5M2, float8_e5m2)
#undef GLB_CASE
      default: break;
    }
    GLB_THROW_INVALID_OPERATION_EXCEPTION("unsupported dtype for old-style algorithm");
  }, py::arg("name"), py::arg("ctx"), py::arg("ptrs") = std::vector<uintptr_t>(), py::arg("count") = 0,
     py::arg("dtype") = 5, py::arg("op") = 1, py::arg("root") = 0, py::arg("root_pointer") = 0,
     py::arg("recv_elems") = std::vector<int>(), py::arg("out_ptr") = 0, py::keep_alive<0, 2>());
}

}  // namespace glb_py
