// PeerContext — the NVLink/NVSwitch peer-memory data plane ("nvl" transport).
//
// Built on top of a connected glb::Context (the TCP mesh is the control plane):
//   1. topology discovery: every rank publishes {hostname, pid, CUDA device,
//      UUID, PCI bus id, SM count, VMM / multicast capability}; from that each
//      rank derives same-host / same-process / same-device groups and the P2P
//      reachability matrix (the reference only counts same-hostname ranks,
//      transport/context.cc:45-57, and knows PCI distances, common/linux.cc).
//   2. a symmetric pool per rank (signal pad + staging area), mapped into every
//      peer: cuMemCreate + POSIX-fd export passed over unix sockets (SCM_RIGHTS)
//      when the driver supports it — which also lets the pool be bound to an
//      NVLS multicast object — else cudaMalloc + cudaIpc handles. Ranks living in
//      the same process (threads-as-ranks tests) share pointers directly.
//   3. registration of user buffers (registerBuffer) and symmetric allocation
//      (allocSymmetric) so collectives can run zero-copy on them.
//
// This is the natural extension of the reference's RemoteKey/put/get surface
// (transport/unbound_buffer.h:128-152, ibverbs only) to GPU peer memory; nothing
// like it exists in the reference (SURVEY §0.1).
#pragma once

#include <cuda_runtime.h>

#include <chrono>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "glb/context.h"
#include "glb/cuda/cuda_util.h"
#include "glb/cuda/comm_types.h"
#include "glb/cuda/kernels.h"

namespace glb {
namespace cuda {

struct DeviceInfo {
  char hostname[64];
  int32_t pid;
  int32_t device;
  uint8_t uuid[16];
  char pciBusId[24];
  int32_t smCount;
  int32_t ccMajor;
  int32_t ccMinor;
  int32_t vmmSupported;
  int32_t multicastSupported;
  uint64_t totalMem;
  char fdSocket[64];  // abstract unix socket that accepts SCM_RIGHTS messages for this rank
  // NVLink state from NVML (-1 when the library is unavailable) and the PCI position of the
  // GPU relative to the box's network controllers (the reference knows GPU <-> NIC distances
  // only: cuda_private.h:64-100, common/linux.cc).
  int32_t nvlinkActive;     // links in the "active" state
  int32_t nvlinkVersion;    // NVML's NVLink version of link 0 (e.g. 7 for NVLink 5)
  int32_t nicDistance;      // PCI hops to the closest network controller, -1 unknown
  char nearestNic[24];      // its bus id
};

struct PeerOptions {
  size_t stageBytes = 128ull << 20;  // staging area for unregistered buffers (per rank)
  bool useVmm = true;                // try cuMem + fd passing before cudaIpc
  bool useNvls = true;               // bind symmetric memory to a multicast object when possible
  size_t llMaxBytes = 256 * 1024;    // largest message of the flag-in-data (LL) kernels
  size_t p2pSlotBytes = 3u << 20;  // one slot of a point-to-point mailbox ring
  int p2pSlots = 4;                  // slots per (source, destination) ring
  int p2pLanes = 48;                 // CTAs per direction of a point-to-point transfer
  int exchangeBlocks = 32;           // CTAs of a zero-copy exchange (same value on every rank)
};

// A buffer that every rank can address: peer[r] is rank r's copy as mapped here.
struct PeerBuffer {
  void* local = nullptr;
  size_t bytes = 0;
  void* peer[kMaxRanks] = {nullptr};
  void* mc = nullptr;        // multicast (NVLS) alias, or nullptr
  bool vectorOk = false;     // every rank's pointer is 16-byte aligned
  PeerPtrs ptrs() const {
    PeerPtrs p;
    for (int i = 0; i < kMaxRanks; i++) p.p[i] = peer[i];
    return p;
  }
  PeerPtrs ptrsAt(size_t byteOffset) const {
    PeerPtrs p;
    for (int i = 0; i < kMaxRanks; i++) p.p[i] = peer[i] ? static_cast<char*>(peer[i]) + byteOffset : nullptr;
    return p;
  }
  ~PeerBuffer();

 private:
  friend class PeerContext;
  struct Impl;
  std::shared_ptr<Impl> impl_;
};

class FdChannel;

class PeerContext : public std::enable_shared_from_this<PeerContext> {
 public:
  PeerContext(std::shared_ptr<Context> context, int device, PeerOptions opts = PeerOptions());
  ~PeerContext();

  const int rank;
  const int size;
  const int device;

  // The control-plane context (throws if it has been destroyed).
  std::shared_ptr<Context> context() const;
  const std::vector<DeviceInfo>& topology() const { return infos_; }
  // P2P works between every pair of ranks (single host, peer access everywhere).
  bool peerAccessEverywhere() const { return peerOk_; }
  bool usingVmm() const { return vmm_; }
  bool nvlsAvailable() const { return pool_ && pool_->mc != nullptr; }
  int ranksOnMyDevice() const { return ranksOnMyDevice_; }
  // Largest grid a collective kernel may use so that all ranks' CTAs are co-resident
  // (one CTA per SM, shared between the ranks that live on this device).
  int maxBlocks() const { return maxBlocks_; }
  // Same, for a specific kernel: SMs x resident CTAs per SM (occupancy at `threads` and
  // `dynamicSmem` bytes of dynamic shared memory per CTA).
  int coResidentBlocks(const void* kernel, int threads = kThreads, size_t dynamicSmem = 0);
  std::string describe() const;

  // ---- failure detection ---------------------------------------------------------------
  // Device-side waits give up after this long (default: the context's timeout) and the
  // context is poisoned: checkHealth() — called on entry of every collective and by
  // synchronize() — throws IoException from then on, like a failed transport pair
  // (gloo/transport/tcp/unbound_buffer.cc:52-94). Rebuild the context to continue.
  void setTimeout(std::chrono::milliseconds t);
  std::chrono::milliseconds timeout() const { return timeout_; }
  // Also raises InputException (once, then clears it) when a kernel found invalid device-side
  // input, e.g. the splits of alltoallvDev(); that does not poison the context.
  void checkHealth();
  bool poisoned() const { return poisoned_; }
  // Device alias of the host-mapped word such kernels report input errors through.
  InputStatus* inputStatusDevice() const { return inputStatusDev_; }
  // cudaStreamSynchronize + checkHealth: the place where a dead peer surfaces.
  void synchronize(cudaStream_t stream);

  // Collectives of one PeerContext share the barrier epoch in the signal pad, so they must
  // execute one after the other on the device. Calls on the same stream are ordered
  // already; a call on a different stream is made to wait for the previous one here.
  void orderStreams(cudaStream_t stream);
  // Called right after a collective kernel has been launched on `stream`.
  void markLaunched(cudaStream_t stream);
  // The tile counter of the single-rank fused step (launchLocalAllreduceMany); its calls are
  // ordered by orderStreams / markLaunched like the collectives'.
  unsigned int* localTileCounter() const { return localTiles_->get(); }

  // ---- collective calls: every rank, same order ------------------------------------
  std::shared_ptr<PeerBuffer> allocSymmetric(size_t bytes);
  std::shared_ptr<PeerBuffer> registerBuffer(void* ptr, size_t bytes);
  // Collective: true iff `mine` is true on every rank.
  bool agree(bool mine);
  // Resolve [ptr, ptr+bytes) for zero-copy use: if it lies inside one of this context's
  // symmetric allocations ON EVERY RANK the owning PeerBuffer (+ byte offset) is returned
  // (NVLS-capable); otherwise the range is registered through cudaIpc. Collective.
  std::shared_ptr<PeerBuffer> resolveBuffer(void* ptr, size_t bytes, size_t* byteOffset);
  void hostBarrier();
  // Collective: whether every rank passed the same words (at most 16), by an allgather over the context.
  bool hostAllSame(const std::vector<int64_t>& words);
  // Call right before launching a kernel that waits for its peers. When several ranks
  // share one GPU (threads-as-ranks tests) a peer that is still inside a device-
  // synchronising call (cudaMalloc from an allocator, cudaFree, ...) would block behind
  // our spinning kernel and never launch its own: rendezvous on the host first so every
  // rank is at its launch point. No-op with one rank per GPU.
  void launchGuard() {
    if (ranksOnMyDevice_ > 1) hostBarrier();
  }

  // ---- kernel arguments --------------------------------------------------------------
  const CommArgs& comm() const { return comm_; }
  // Staging area (after the signal pad) of every rank's pool, and its size.
  PeerPtrs stagePtrs(size_t byteOffset = 0) const;
  void* stageMc(size_t byteOffset = 0) const;
  size_t stageBytes() const { return stageBytes_; }
  // Flag-in-data region: [parity][source rank][16-byte lines].
  PeerPtrs llPtrs() const;
  size_t llSrcStride() const { return llSrcStride_; }
  size_t llParityStride() const { return llSrcStride_ * static_cast<size_t>(size); }
  size_t llMaxBytes() const { return opts_.llMaxBytes; }
  // Point-to-point mailboxes: box[source rank] = p2pSlots x p2pSlotBytes inside every pool.
  PeerPtrs mailboxPtrs() const;
  size_t mailboxStride() const { return opts_.p2pSlotBytes * static_cast<size_t>(opts_.p2pSlots); }
  const PeerOptions& options() const { return opts_; }
  const PeerBuffer& pool() const { return *pool_; }

  // ---- single-process loopback (profilers, self-test) ----------------------------------
  // Kernel arguments that make ONE launch play rank 0 of `virtualRanks` ranks: every
  // virtual peer's pad is this rank's pad shifted by one flag column, so the barrier
  // flags the kernel posts for its "peers" are exactly the ones it then waits for.
  // Lets Nsight Compute (which serialises kernels and therefore cannot run two ranks
  // that wait for each other) profile the P = 2 / 4 / 8 specialisations, and lets the
  // self-test check them numerically, on one GPU.
  CommArgs loopbackComm(int virtualRanks) const;
  // Single-rank contexts only: a symmetric buffer bound to a ONE-device multicast object, so
  // the multimem (NVLS) kernels can run in loopback. nullptr (+ reason) when unsupported.
  std::shared_ptr<PeerBuffer> tryAllocMulticastLoopback(size_t bytes, std::string* why);

 private:
  uint32_t nextTag() { return 0x7C000000u + (tagSeq_++ & 0xffffffu); }
  void exchangeTopology();
  template <typename T>
  std::vector<T> allgatherStruct(const T& mine);
  std::shared_ptr<PeerBuffer> allocSymmetricImpl(size_t bytes);
  std::shared_ptr<PeerBuffer> allocVmm(size_t bytes, bool wantMc);
  std::shared_ptr<PeerBuffer> allocIpc(size_t bytes);
  std::shared_ptr<PeerBuffer> shareIpc(void* ptr, size_t bytes, bool ownsAllocation);
  bool sameProcess(int r) const;

  std::weak_ptr<Context> context_;  // weak: the context may own this object as an attachment
  PeerOptions opts_;
  std::vector<DeviceInfo> infos_;
  bool peerOk_ = false;
  bool vmm_ = false;
  bool nvlsPossible_ = false;
  int ranksOnMyDevice_ = 1;
  int worstRanksPerDevice_ = 1;
  int minSms_ = 1;
  int maxBlocks_ = 1;
  uint32_t tagSeq_ = 0;
  std::unique_ptr<FdChannel> fdChannel_;
  std::shared_ptr<PeerBuffer> pool_;
  std::mutex symMu_;
  std::vector<std::weak_ptr<PeerBuffer>> symmetric_;  // live allocSymmetric() results
  size_t stageOffset_ = 0;
  size_t stageBytes_ = 0;
  size_t llOffset_ = 0;
  size_t llSrcStride_ = 0;
  size_t mailboxOffset_ = 0;
  CommArgs comm_;
  uint32_t* hostStatus_ = nullptr;     // pinned + mapped: written by kernels that give up
  uint32_t* hostStatusDev_ = nullptr;  // device alias of hostStatus_
  InputStatus* inputStatus_ = nullptr;     // in the same pinned block, after the abort word
  InputStatus* inputStatusDev_ = nullptr;
  std::chrono::milliseconds timeout_{0};
  bool poisoned_ = false;
  std::string poisonReason_;
  cudaStream_t lastStream_ = nullptr;
  bool haveLastStream_ = false;
  cudaEvent_t orderEvent_ = nullptr;
  std::unique_ptr<TileCounter> localTiles_;
  std::mutex occMu_;
  std::map<std::pair<const void*, size_t>, int> occupancy_;  // (kernel, dynamic smem) -> CTAs per SM
  // cudaIpc mappings are per (peer, allocation): cache them, opening twice is an error.
  std::mutex ipcMu_;
  std::map<std::pair<int, std::string>, void*> ipcCache_;
};

}  // namespace cuda
}  // namespace glb
