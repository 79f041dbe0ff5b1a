// Old-style CUDA algorithm classes: construct once (collective: buffers are
// registered with the peers), run() many times (one fused kernel launch each).
//
//   CudaAllreduceRing / RingChunked / HalvingDoubling (+Pipelined) / Bcube / Local
//   CudaBroadcastOneToAll
//
// Template parameter W selects the workspace, as in the reference
// (cuda_workspace.h:20-30):
//   CudaPeerWorkspace<T>    (default) NVLink peer memory; the kernel variant is
//                           picked per message size (one-shot / two-shot / NVLS)
//                           unless GLB_CUDA_LITERAL_SCHEDULES=1 or the schedule is
//                           requested explicitly, in which case the named schedule
//                           (ring, ring_chunked, halving_doubling, bcube) is
//                           executed literally over peer pointers.
//   CudaHostWorkspace<T>    stage through pinned host memory and run the host
//                           collective over the transport (works across nodes; the
//                           only data path the reference has).
//   CudaDeviceWorkspace<T>  alias of the peer workspace (reference name: GPUDirect).
// If peers are not all P2P-reachable the peer workspace silently degrades to host.
// Streams: without user streams outputs are valid on return; with user streams the
// caller synchronises (docs/cuda.md:7-11 semantics).
// Parity: gloo/cuda_allreduce_*.{h,cc}, cuda_broadcast_one_to_all.{h,cc}.
#pragma once

#include <cuda_runtime.h>

#include <memory>
#include <vector>

#include "glb/algorithm.h"
#include "glb/cuda/collectives.h"
#include "glb/cuda/kernels.h"
#include "glb/cuda/stream.h"

namespace glb {

template <typename T>
struct CudaPeerWorkspace {};
template <typename T>
struct CudaHostWorkspace {};
template <typename T>
using CudaDeviceWorkspace = CudaPeerWorkspace<T>;

namespace cuda {

enum class Workspace { PEER, HOST };

// PeerContext bound to (context, device); created collectively on first use.
std::shared_ptr<PeerContext> peerContextFor(const std::shared_ptr<Context>& ctx, int device,
                                            const PeerOptions& optsIfCreated = PeerOptions());
void releasePeerContexts(const std::shared_ptr<Context>& ctx);
// The variant a reference-named class runs: AUTO (per-size selection) unless literal
// schedules are requested with GLB_CUDA_LITERAL_SCHEDULES=1.
AllreduceAlgo namedAlgo(AllreduceAlgo named);
std::vector<CudaStream> makeStreamsFor(const std::vector<void*>& ptrs, const std::vector<cudaStream_t>& user);

class CudaAllreduceCore {
 public:
  CudaAllreduceCore(std::shared_ptr<Context> ctx, std::vector<void*> ptrs, size_t count, DataType dt, ReduceOp op,
                    std::vector<cudaStream_t> streams, AllreduceAlgo algo, Workspace ws);
  ~CudaAllreduceCore();
  void run();
  AllreduceAlgo resolvedAlgo() const;
  bool usesPeerMemory() const { return pc_ != nullptr; }
  // Fused epilogue: the result is multiplied by `scale` (AVG = 1 / (ranks x local pointers))
  // inside the collective kernel.
  void setScale(double scale) { scale_ = scale; }
  // Launches per run() (1 when the local fold, the exchange and the fan-out are fused).
  int launchesPerRun() const;
  // Pin the launch shape (sweeps / tuner): 0 = tuning table.
  void setLaunchShape(int blocks, int unroll, int tile) {
    shapeBlocks_ = blocks;
    shapeUnroll_ = unroll;
    shapeTile_ = tile;
  }

 private:
  void runHostWorkspace(CudaStream& s0);
  std::shared_ptr<Context> ctx_;
  std::vector<void*> ptrs_;
  size_t count_;
  DataType dt_;
  ReduceOp op_;
  AllreduceAlgo algo_;
  bool syncOutputs_;
  double scale_ = 1.0;
  bool fuseLocal_ = false;   // extra local pointers are folded inside the collective kernel
  int shapeBlocks_ = 0, shapeUnroll_ = 0, shapeTile_ = 0;
  int hostChunks_ = 1;
  std::unique_ptr<CudaStream> h2dStream_;
  std::vector<cudaEvent_t> chunkEvents_;
  std::vector<CudaStream> streams_;
  std::shared_ptr<PeerContext> pc_;
  std::shared_ptr<PeerBuffer> reg_;
  size_t regOffset_ = 0;
  void* hostScratch_ = nullptr;  // pinned, host workspace only
  std::unique_ptr<TileCounter> tiles_;  // the local fused step's: single rank or host workspace only
  struct Literal;
  std::unique_ptr<Literal> literal_;
};

class CudaBroadcastCore {
 public:
  CudaBroadcastCore(std::shared_ptr<Context> ctx, std::vector<void*> ptrs, size_t count, DataType dt, int rootRank,
                    int rootPointerRank, std::vector<cudaStream_t> streams, Workspace ws);
  ~CudaBroadcastCore();
  void run();

 private:
  std::shared_ptr<Context> ctx_;
  std::vector<void*> ptrs_;
  size_t count_;
  DataType dt_;
  int root_;
  int rootPtr_;
  bool syncOutputs_;
  std::vector<CudaStream> streams_;
  std::shared_ptr<PeerContext> pc_;
  std::shared_ptr<PeerBuffer> reg_;
  size_t regOffset_ = 0;
  void* hostScratch_ = nullptr;
};

template <typename W>
struct WorkspaceOf;
template <typename T>
struct WorkspaceOf<CudaPeerWorkspace<T>> {
  static constexpr Workspace value = Workspace::PEER;
};
template <typename T>
struct WorkspaceOf<CudaHostWorkspace<T>> {
  static constexpr Workspace value = Workspace::HOST;
};

template <typename T>
std::vector<void*> eraseType(const std::vector<T*>& ptrs) {
  std::vector<void*> out;
  for (auto* p : ptrs) out.push_back(const_cast<void*>(static_cast<const void*>(p)));
  return out;
}

}  // namespace cuda

// Device reduction function handle (type + op); the actual kernels are selected by
// (dtype, op) at launch. Parity: gloo/cuda.h:286-358.
template <typename T>
class CudaReductionFunction {
 public:
  static const CudaReductionFunction<T>* sum;
  static const CudaReductionFunction<T>* product;
  static const CudaReductionFunction<T>* min;
  static const CudaReductionFunction<T>* max;
  explicit CudaReductionFunction(ReduceOp type) : type_(type) {}
  ReduceOp type() const { return type_; }
  // dst = dst (op) src on `stream` (both device pointers, or host pointers -> CPU).
  void call(T* dst, const T* src, size_t n, cudaStream_t stream) const;
  void callHost(T* dst, const T* src, size_t n) const {
    ReductionFunction<T>::get(type_)->call(dst, src, n);
  }

 private:
  ReduceOp type_;
};
template <typename T>
const CudaReductionFunction<T>* CudaReductionFunction<T>::sum = new CudaReductionFunction<T>(ReduceOp::SUM);
template <typename T>
const CudaReductionFunction<T>* CudaReductionFunction<T>::product = new CudaReductionFunction<T>(ReduceOp::PRODUCT);
template <typename T>
const CudaReductionFunction<T>* CudaReductionFunction<T>::min = new CudaReductionFunction<T>(ReduceOp::MIN);
template <typename T>
const CudaReductionFunction<T>* CudaReductionFunction<T>::max = new CudaReductionFunction<T>(ReduceOp::MAX);

#define GLB_DEFINE_CUDA_ALLREDUCE(Name, Algo)                                                             \
  template <typename T, typename W = CudaPeerWorkspace<T>>                                                \
  class Name : public Algorithm {                                                                         \
   public:                                                                                                \
    Name(const std::shared_ptr<Context>& context, const std::vector<T*>& ptrs, const size_t count,        \
         const std::vector<cudaStream_t>& streams = std::vector<cudaStream_t>(),                         \
         const CudaReductionFunction<T>* fn = CudaReductionFunction<T>::sum)                              \
        : Algorithm(context),                                                                             \
          core_(context, cuda::eraseType(ptrs), count, DataTypeOf<T>::value, fn->type(), streams,         \
                cuda::namedAlgo(cuda::AllreduceAlgo::Algo), cuda::WorkspaceOf<W>::value) {}                                \
    void run() override { core_.run(); }                                                                  \
    cuda::CudaAllreduceCore& core() { return core_; }                                                     \
                                                                                                          \
   private:                                                                                               \
    cuda::CudaAllreduceCore core_;                                                                        \
  };

GLB_DEFINE_CUDA_ALLREDUCE(CudaAllreduceRing, RING)
GLB_DEFINE_CUDA_ALLREDUCE(CudaAllreduceRingChunked, RING_CHUNKED)
GLB_DEFINE_CUDA_ALLREDUCE(CudaAllreduceHalvingDoubling, HALVING_DOUBLING)
GLB_DEFINE_CUDA_ALLREDUCE(CudaAllreduceHalvingDoublingPipelined, HALVING_DOUBLING_PIPELINED)
GLB_DEFINE_CUDA_ALLREDUCE(CudaAllreduceBcube, BCUBE)
#undef GLB_DEFINE_CUDA_ALLREDUCE

// Reduce + broadcast across the local pointers only (no network).
template <typename T>
class CudaAllreduceLocal : public Algorithm {
 public:
  CudaAllreduceLocal(const std::shared_ptr<Context>& context, const std::vector<T*>& ptrs, const size_t count,
                     const std::vector<cudaStream_t>& streams = std::vector<cudaStream_t>());
  void run() override;

 private:
  std::vector<void*> ptrs_;
  size_t count_;
  bool syncOutputs_;
  std::vector<cuda::CudaStream> streams_;
  std::unique_ptr<cuda::TileCounter> tiles_;
};

template <typename T, typename W = CudaPeerWorkspace<T>>
class CudaBroadcastOneToAll : public Algorithm {
 public:
  CudaBroadcastOneToAll(const std::shared_ptr<Context>& context, const std::vector<T*>& ptrs, size_t count,
                        int rootRank = 0, int rootPointerRank = 0,
                        const std::vector<cudaStream_t>& streams = std::vector<cudaStream_t>())
      : Algorithm(context),
        core_(context, cuda::eraseType(ptrs), count, DataTypeOf<T>::value, rootRank, rootPointerRank, streams,
              cuda::WorkspaceOf<W>::value) {}
  void run() override { core_.run(); }

 private:
  cuda::CudaBroadcastCore core_;
};

}  // namespace glb
