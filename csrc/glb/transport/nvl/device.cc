#include "glb/transport/nvl/device.h"

#include <cuda_runtime.h>
#include <unistd.h>

#include <atomic>
#include <cstring>
#include <map>
#include <mutex>
#include <sstream>
#include <thread>

#include "glb/common/logging.h"
#include "glb/common/utils.h"
#include "glb/context.h"
#include "glb/cuda/algorithms.h"
#include "glb/cuda/collectives.h"
#include "glb/cuda/cuda_util.h"
#include "glb/cuda/kernels.h"
#include "glb/transport/context.h"

namespace glb {
namespace transport {
namespace nvl {

namespace {

std::string toHex(const void* p, size_t n) {
  static const char* d = "0123456789abcdef";
  std::string s;
  const auto* b = static_cast<const unsigned char*>(p);
  for (size_t i = 0; i < n; i++) {
    s.push_back(d[b[i] >> 4]);
    s.push_back(d[b[i] & 15]);
  }
  return s;
}

bool fromHex(const std::string& s, void* out, size_t n) {
  if (s.size() != 2 * n) return false;
  auto v = [](char c) { return c >= '0' && c <= '9' ? c - '0' : c >= 'a' && c <= 'f' ? c - 'a' + 10 : -1; };
  auto* b = static_cast<unsigned char*>(out);
  for (size_t i = 0; i < n; i++) {
    const int hi = v(s[2 * i]), lo = v(s[2 * i + 1]);
    if (hi < 0 || lo < 0) return false;
    b[i] = static_cast<unsigned char>(hi * 16 + lo);
  }
  return true;
}

struct KeyBlob {
  int32_t rank;
  int32_t pid;
  uint64_t hostHash;
  uint64_t rawPtr;   // the region as seen by its owner
  uint64_t offset;   // region start relative to the base of its allocation
  uint64_t size;
  cudaIpcMemHandle_t handle;
};

uint64_t hostHash() {
  const std::string h = getHostname();
  uint64_t x = 1469598103934665603ull;
  for (char c : h) x = (x ^ static_cast<unsigned char>(c)) * 1099511628211ull;
  return x;
}

class Key : public RemoteKey {
 public:
  explicit Key(const KeyBlob& b) : RemoteKey(b.rank, b.size), blob(b) {}
  std::string serialize() const override { return "nvl:" + toHex(&blob, sizeof(blob)); }
  KeyBlob blob;
};

class Ctx;

// Asynchronous completion of work enqueued on one of the context's side streams.
struct Pending {
  cudaEvent_t event = nullptr;
  int peer = -1;
};

class Buf : public UnboundBuffer {
 public:
  Buf(Ctx* ctx, void* ptr, size_t size) : UnboundBuffer(ptr, size), ctx_(ctx) {}
  ~Buf() override;

  bool waitRecv(int* rank, std::chrono::milliseconds timeout) override { return wait(recvs_, abortRecv_, rank, timeout); }
  bool waitSend(int* rank, std::chrono::milliseconds timeout) override { return wait(sends_, abortSend_, rank, timeout); }
  void abortWaitRecv() override { abortRecv_ = true; }
  void abortWaitSend() override { abortSend_ = true; }

  void send(int dstRank, uint64_t slot, size_t offset, size_t nbytes) override;
  void recv(int srcRank, uint64_t slot, size_t offset, size_t nbytes) override;
  void recv(std::vector<int> srcRanks, uint64_t slot, size_t offset, size_t nbytes) override {
    GLB_ENFORCE_EQ(srcRanks.size(), size_t(1),
                   "nvl: device buffers match in posting order per peer; receive-from-any needs a host buffer");
    recv(srcRanks[0], slot, offset, nbytes);
  }
  std::unique_ptr<RemoteKey> getRemoteKey() const override;
  void put(const RemoteKey& key, uint64_t slot, size_t offset, size_t roffset, size_t nbytes) override;
  void get(const RemoteKey& key, uint64_t slot, size_t offset, size_t roffset, size_t nbytes) override;

 private:
  size_t span(size_t offset, size_t nbytes) const {
    if (nbytes == kUnspecifiedByteCount) {
      GLB_ENFORCE_LE(offset, size, "offset exceeds the buffer");
      nbytes = size - offset;
    }
    GLB_ENFORCE(offset <= size && nbytes <= size - offset, "range exceeds the buffer");
    return nbytes;
  }
  void track(std::vector<Pending>& q, cudaStream_t stream, int peer);
  bool wait(std::vector<Pending>& q, std::atomic<bool>& aborted, int* rank, std::chrono::milliseconds timeout);

  Ctx* ctx_;
  std::mutex mu_;
  std::vector<Pending> sends_, recvs_;
  std::atomic<bool> abortSend_{false}, abortRecv_{false};
};

class Ctx : public Context {
 public:
  Ctx(std::shared_ptr<Context> inner, int cudaDevice)
      : Context(inner->rank, inner->size), inner_(std::move(inner)), device_(cudaDevice) {
    cuda::DeviceGuard g(device_);
    GLB_CUDA_CHECK(cudaStreamCreateWithFlags(&sendStream_, cudaStreamNonBlocking));
    GLB_CUDA_CHECK(cudaStreamCreateWithFlags(&recvStream_, cudaStreamNonBlocking));
  }
  ~Ctx() override {
    cuda::DeviceGuard g(device_);
    cudaStreamSynchronize(sendStream_);
    cudaStreamSynchronize(recvStream_);
    cudaStreamDestroy(sendStream_);
    cudaStreamDestroy(recvStream_);
    for (auto& kv : mapped_) cudaIpcCloseMemHandle(kv.second);
  }

  // ---- everything host side is the wrapped context's business ----------------------------
  std::unique_ptr<Pair>& getPair(int r) override { return inner_->getPair(r); }
  std::unique_ptr<Pair>& createPair(int r) override { return inner_->createPair(r); }
  Pair* peekPair(int r) override { return inner_->peekPair(r); }
  void createAndConnectAllPairs(std::shared_ptr<IStore> store) override { inner_->createAndConnectAllPairs(std::move(store)); }
  std::vector<char> exportRendezvousBlob() override { return inner_->exportRendezvousBlob(); }
  void connectWithBlobs(const std::vector<std::vector<char>>& blobs) override { inner_->connectWithBlobs(blobs); }
  void setTimeout(std::chrono::milliseconds t) override {
    Context::setTimeout(t);
    inner_->setTimeout(t);
  }

  void onAttached(const std::weak_ptr<::glb::Context>& owner) override {
    owner_ = owner;
    auto ctx = owner.lock();
    GLB_ENFORCE(ctx != nullptr, "nvl: the glb::Context must be owned by a shared_ptr");
    cuda::DeviceGuard g(device_);
    // Collective: every rank is inside connectFullMesh / makeContext right now.
    peer_ = cuda::peerContextFor(ctx, device_);
    GLB_ENFORCE(peer_.lock()->peerAccessEverywhere() || size == 1,
                "nvl: the ranks of this context are not all P2P-reachable (single NVLink domain required)");
  }

  std::unique_ptr<UnboundBuffer> createUnboundBuffer(void* ptr, size_t bytes) override {
    if (ptr != nullptr && cuda::deviceForPointer(ptr) >= 0) return std::make_unique<Buf>(this, ptr, bytes);
    return inner_->createUnboundBuffer(ptr, bytes);
  }

  std::unique_ptr<RemoteKey> deserializeRemoteKey(const std::string& s) override {
    if (s.rfind("nvl:", 0) != 0) return inner_->deserializeRemoteKey(s);
    KeyBlob b;
    GLB_ENFORCE(fromHex(s.substr(4), &b, sizeof(b)), "nvl: malformed remote key");
    return std::make_unique<Key>(b);
  }

  std::shared_ptr<cuda::PeerContext> peer() {
    auto p = peer_.lock();
    GLB_ENFORCE(p != nullptr, "nvl: the context is not connected (or has been closed)");
    return p;
  }
  int device() const { return device_; }
  cudaStream_t sendStream() const { return sendStream_; }
  cudaStream_t recvStream() const { return recvStream_; }

  // The target region of `key` as a pointer this process can use on its device.
  char* map(const KeyBlob& b) {
    if (b.hostHash == hostHash() && b.pid == static_cast<int32_t>(::getpid())) {
      return reinterpret_cast<char*>(b.rawPtr);  // same process (threads as ranks): same address space
    }
    GLB_ENFORCE_EQ(b.hostHash, hostHash(), "nvl: remote key from another host");
    std::lock_guard<std::mutex> g(mapMu_);
    const std::string id(reinterpret_cast<const char*>(&b.handle), sizeof(b.handle));
    auto it = mapped_.find(id);
    void* base = nullptr;
    if (it != mapped_.end()) {
      base = it->second;
    } else {
      cuda::DeviceGuard dg(device_);
      cudaError_t e = cudaIpcOpenMemHandle(&base, b.handle, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        cudaGetLastError();
        GLB_THROW_IO_EXCEPTION("nvl: cannot map the remote region of rank ", b.rank, ": ", cudaGetErrorString(e));
      }
      mapped_[id] = base;
    }
    return static_cast<char*>(base) + b.offset;
  }

 private:
  std::shared_ptr<Context> inner_;
  int device_;
  cudaStream_t sendStream_ = nullptr, recvStream_ = nullptr;
  std::weak_ptr<::glb::Context> owner_;
  std::weak_ptr<cuda::PeerContext> peer_;
  std::mutex mapMu_;
  std::map<std::string, void*> mapped_;
};

Buf::~Buf() {
  for (auto* q : {&sends_, &recvs_}) {
    for (auto& p : *q) {
      cudaEventSynchronize(p.event);
      cudaEventDestroy(p.event);
    }
  }
}

void Buf::track(std::vector<Pending>& q, cudaStream_t stream, int peer) {
  Pending p;
  p.peer = peer;
  GLB_CUDA_CHECK(cudaEventCreateWithFlags(&p.event, cudaEventDisableTiming));
  GLB_CUDA_CHECK(cudaEventRecord(p.event, stream));
  std::lock_guard<std::mutex> g(mu_);
  q.push_back(p);
}

bool Buf::wait(std::vector<Pending>& q, std::atomic<bool>& aborted, int* rank, std::chrono::milliseconds timeout) {
  Pending p;
  {
    std::lock_guard<std::mutex> g(mu_);
    GLB_ENFORCE(!q.empty(), "nvl: wait without a pending operation");
    p = q.front();
  }
  if (timeout == kUnsetTimeout) timeout = ctx_->getTimeout();
  const auto start = std::chrono::steady_clock::now();
  cuda::DeviceGuard g(ctx_->device());
  while (true) {
    cudaError_t e = cudaEventQuery(p.event);
    if (e == cudaSuccess) break;
    if (e != cudaErrorNotReady) GLB_CUDA_CHECK(e);
    if (aborted.exchange(false)) return false;
    if (timeout != kNoTimeout && timeout.count() > 0 && std::chrono::steady_clock::now() - start > timeout + std::chrono::seconds(2)) {
      // The device-side wait gives up at `timeout` and lets the kernel end; if even that did
      // not happen the GPU is wedged.
      GLB_THROW_IO_EXCEPTION("nvl: operation with rank ", p.peer, " did not complete within ", timeout.count(), " ms");
    }
    std::this_thread::sleep_for(std::chrono::microseconds(20));
  }
  {
    std::lock_guard<std::mutex> g2(mu_);
    q.erase(q.begin());
  }
  cudaEventDestroy(p.event);
  ctx_->peer()->checkHealth();  // a peer that never showed up surfaces here as IoException
  if (rank != nullptr) *rank = p.peer;
  return true;
}

void Buf::send(int dstRank, uint64_t /*slot*/, size_t offset, size_t nbytes) {
  nbytes = span(offset, nbytes);
  auto pc = ctx_->peer();
  cuda::send(*pc, static_cast<const char*>(ptr) + offset, nbytes, dstRank, ctx_->sendStream());
  track(sends_, ctx_->sendStream(), dstRank);
}

void Buf::recv(int srcRank, uint64_t /*slot*/, size_t offset, size_t nbytes) {
  nbytes = span(offset, nbytes);
  auto pc = ctx_->peer();
  cuda::recv(*pc, static_cast<char*>(ptr) + offset, nbytes, srcRank, ctx_->recvStream());
  track(recvs_, ctx_->recvStream(), srcRank);
}

std::unique_ptr<RemoteKey> Buf::getRemoteKey() const {
  KeyBlob b;
  std::memset(&b, 0, sizeof(b));
  b.rank = ctx_->rank;
  b.pid = static_cast<int32_t>(::getpid());
  b.hostHash = hostHash();
  b.rawPtr = reinterpret_cast<uint64_t>(ptr);
  b.size = size;
  cuda::DeviceGuard g(ctx_->device());
  void* base = ptr;
  try {
    CUdeviceptr bp = 0;
    size_t sz = 0;
    if (cuda::driver().cuMemGetAddressRange(&bp, &sz, reinterpret_cast<CUdeviceptr>(ptr)) == CUDA_SUCCESS && bp != 0) {
      base = reinterpret_cast<void*>(bp);
    }
  } catch (...) {
  }
  b.offset = static_cast<uint64_t>(static_cast<char*>(ptr) - static_cast<char*>(base));
  cudaError_t e = cudaIpcGetMemHandle(&b.handle, base);
  if (e != cudaSuccess) {
    cudaGetLastError();
    // Only peers in this process can use the key then (they need no handle).
    GLB_WARN("nvl: cudaIpcGetMemHandle failed (", cudaGetErrorString(e),
             "); the remote key is usable from ranks of this process only. cudaMalloc'ed memory exports; "
             "cuMemCreate / symmetric allocations do not");
    std::memset(&b.handle, 0, sizeof(b.handle));
  }
  return std::make_unique<Key>(b);
}

void Buf::put(const RemoteKey& key, uint64_t /*slot*/, size_t offset, size_t roffset, size_t nbytes) {
  const auto* k = dynamic_cast<const Key*>(&key);
  GLB_ENFORCE(k != nullptr, "nvl: put() needs an nvl remote key");
  GLB_ENFORCE(offset <= size && nbytes <= size - offset, "put: local range exceeds the buffer");
  GLB_ENFORCE(roffset <= k->size && nbytes <= k->size - roffset, "put: remote range exceeds the region of the key");
  cuda::DeviceGuard g(ctx_->device());
  if (nbytes > 0) {
    cuda::launchPeerCopy(ctx_->map(k->blob) + roffset, static_cast<const char*>(ptr) + offset, nbytes, 64, ctx_->sendStream());
    cuda::noteLaunch();
    GLB_CUDA_CHECK(cudaGetLastError());
  }
  track(sends_, ctx_->sendStream(), k->rank);
}

void Buf::get(const RemoteKey& key, uint64_t /*slot*/, size_t offset, size_t roffset, size_t nbytes) {
  const auto* k = dynamic_cast<const Key*>(&key);
  GLB_ENFORCE(k != nullptr, "nvl: get() needs an nvl remote key");
  GLB_ENFORCE(offset <= size && nbytes <= size - offset, "get: local range exceeds the buffer");
  GLB_ENFORCE(roffset <= k->size && nbytes <= k->size - roffset, "get: remote range exceeds the region of the key");
  cuda::DeviceGuard g(ctx_->device());
  if (nbytes > 0) {
    cuda::launchPeerCopy(static_cast<char*>(ptr) + offset, ctx_->map(k->blob) + roffset, nbytes, 64, ctx_->recvStream());
    cuda::noteLaunch();
    GLB_CUDA_CHECK(cudaGetLastError());
  }
  track(recvs_, ctx_->recvStream(), k->rank);
}

class Dev : public Device {
 public:
  Dev(std::shared_ptr<Device> control, int cudaDevice) : control_(std::move(control)), cudaDevice_(cudaDevice) {
    pci_ = cuda::devicePCIBusId(cudaDevice_);
  }
  std::string str() const override { return strcat_all("nvl(cuda:", cudaDevice_, " ", pci_, ") over ", control_->str()); }
  const std::string& getPCIBusID() const override { return pci_; }
  int getInterfaceSpeed() const override { return 450 * 8 * 1000; }  // Mb/s: 450 GB/s per direction (H100 SXM, NVLink 4)
  bool hasGPUDirect() const override { return true; }
  std::shared_ptr<Context> createContext(int rank, int size) override {
    return std::make_shared<Ctx>(control_->createContext(rank, size), cudaDevice_);
  }

 private:
  std::shared_ptr<Device> control_;
  int cudaDevice_;
  std::string pci_;
};

}  // namespace

std::shared_ptr<::glb::transport::Device> CreateDevice(const attr& a) {
  GLB_ENFORCE(a.control != nullptr, "nvl::CreateDevice needs a control-plane (tcp / tls) device");
  GLB_ENFORCE(cuda::deviceCount() > 0, "nvl::CreateDevice needs a CUDA device");
  int dev = a.cudaDevice;
  if (dev < 0) GLB_CUDA_CHECK(cudaGetDevice(&dev));
  GLB_ENFORCE(dev < cuda::deviceCount(), "invalid CUDA device ", dev);
  return std::make_shared<Dev>(a.control, dev);
}

}  // namespace nvl
}  // namespace transport
}  // namespace glb
