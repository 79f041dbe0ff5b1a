#include "glb/cuda/peer_context.h"

#include <dlfcn.h>
#include <sys/socket.h>
#include <sys/un.h>
#include <poll.h>
#include <unistd.h>

#include <atomic>
#include <cctype>
#include <cerrno>
#include <cstring>
#include <set>
#include <sstream>

#include "glb/allgather.h"
#include "glb/barrier.h"
#include "glb/common/linux.h"
#include "glb/common/utils.h"
#include "glb/cuda/kernels.h"
#include "glb/cuda/tuning.h"

namespace glb {
namespace cuda {

// ---- fd passing over abstract unix datagram sockets ---------------------------------

class FdChannel {
 public:
  FdChannel(int rank) {
    static std::atomic<uint64_t> counter{0};
    fd_ = ::socket(AF_UNIX, SOCK_DGRAM | SOCK_CLOEXEC, 0);
    GLB_ENFORCE_NE(fd_, -1, "socket(AF_UNIX): ", std::strerror(errno));
    name_ = strcat_all("glb-fd-", ::getpid(), "-", counter.fetch_add(1), "-", rank);
    struct sockaddr_un addr;
    socklen_t len = fill(addr, name_);
    GLB_ENFORCE_NE(::bind(fd_, reinterpret_cast<struct sockaddr*>(&addr), len), -1, "bind(", name_,
                   "): ", std::strerror(errno));
  }
  ~FdChannel() {
    for (auto& kv : inbox_) ::close(kv.second);
    if (fd_ >= 0) ::close(fd_);
  }
  const std::string& name() const { return name_; }

  void sendFd(const std::string& peerName, int fd, int srcRank, uint32_t tag) {
    struct sockaddr_un addr;
    socklen_t alen = fill(addr, peerName);
    uint32_t payload[2] = {static_cast<uint32_t>(srcRank), tag};
    struct iovec iov = {payload, sizeof(payload)};
    char ctrl[CMSG_SPACE(sizeof(int))];
    std::memset(ctrl, 0, sizeof(ctrl));
    struct msghdr msg;
    std::memset(&msg, 0, sizeof(msg));
    msg.msg_name = &addr;
    msg.msg_namelen = alen;
    msg.msg_iov = &iov;
    msg.msg_iovlen = 1;
    msg.msg_control = ctrl;
    msg.msg_controllen = sizeof(ctrl);
    struct cmsghdr* cm = CMSG_FIRSTHDR(&msg);
    cm->cmsg_level = SOL_SOCKET;
    cm->cmsg_type = SCM_RIGHTS;
    cm->cmsg_len = CMSG_LEN(sizeof(int));
    std::memcpy(CMSG_DATA(cm), &fd, sizeof(int));
    for (int attempt = 0;; attempt++) {
      ssize_t n = ::sendmsg(fd_, &msg, 0);
      if (n >= 0) return;
      if ((errno == ECONNREFUSED || errno == ENOENT || errno == EAGAIN || errno == ENOBUFS) && attempt < 2000) {
        ::usleep(1000);
        continue;
      }
      GLB_THROW_IO_EXCEPTION("sendmsg(SCM_RIGHTS) to ", peerName, ": ", std::strerror(errno));
    }
  }

  int recvFd(int srcRank, uint32_t tag, std::chrono::milliseconds timeout) {
    const auto key = std::make_pair(srcRank, tag);
    const auto start = std::chrono::steady_clock::now();
    while (true) {
      auto it = inbox_.find(key);
      if (it != inbox_.end()) {
        int fd = it->second;
        inbox_.erase(it);
        return fd;
      }
      struct pollfd pfd = {fd_, POLLIN, 0};
      int rv = ::poll(&pfd, 1, 100);
      if (rv == 0) {
        if (timeout != kNoTimeout && std::chrono::steady_clock::now() - start > timeout) {
          GLB_THROW_IO_EXCEPTION("timed out waiting for a file descriptor from rank ", srcRank);
        }
        continue;
      }
      uint32_t payload[2] = {0, 0};
      struct iovec iov = {payload, sizeof(payload)};
      char ctrl[CMSG_SPACE(sizeof(int))];
      struct msghdr msg;
      std::memset(&msg, 0, sizeof(msg));
      msg.msg_iov = &iov;
      msg.msg_iovlen = 1;
      msg.msg_control = ctrl;
      msg.msg_controllen = sizeof(ctrl);
      ssize_t n = ::recvmsg(fd_, &msg, MSG_CMSG_CLOEXEC);
      if (n < 0) {
        if (errno == EINTR || errno == EAGAIN) continue;
        GLB_THROW_IO_EXCEPTION("recvmsg: ", std::strerror(errno));
      }
      struct cmsghdr* cm = CMSG_FIRSTHDR(&msg);
      if (cm == nullptr || cm->cmsg_type != SCM_RIGHTS) continue;
      int fd = -1;
      std::memcpy(&fd, CMSG_DATA(cm), sizeof(int));
      inbox_[std::make_pair(static_cast<int>(payload[0]), payload[1])] = fd;
    }
  }

 private:
  static socklen_t fill(struct sockaddr_un& addr, const std::string& name) {
    std::memset(&addr, 0, sizeof(addr));
    addr.sun_family = AF_UNIX;
    GLB_ENFORCE_LT(name.size() + 1, sizeof(addr.sun_path));
    std::memcpy(addr.sun_path + 1, name.data(), name.size());  // leading NUL => abstract namespace
    return static_cast<socklen_t>(offsetof(struct sockaddr_un, sun_path) + 1 + name.size());
  }
  int fd_ = -1;
  std::string name_;
  std::map<std::pair<int, uint32_t>, int> inbox_;
};

// ---- PeerBuffer resources ---------------------------------------------------------------

struct PeerBuffer::Impl {
  int device = 0;
  // VMM
  struct Mapping {
    CUdeviceptr va = 0;
    size_t size = 0;
    CUmemGenericAllocationHandle handle = 0;
    bool haveHandle = false;
  };
  std::vector<Mapping> mappings;  // local allocation first, then imported peers, then multicast
  // legacy
  void* owned = nullptr;  // cudaMalloc'ed by us

  ~Impl() {
    DeviceGuard g(device);
    if (!mappings.empty()) {
      try {
        const auto& d = driver();
        for (auto it = mappings.rbegin(); it != mappings.rend(); ++it) {
          if (it->va != 0) {
            d.cuMemUnmap(it->va, it->size);
            d.cuMemAddressFree(it->va, it->size);
          }
          if (it->haveHandle) d.cuMemRelease(it->handle);
        }
      } catch (...) {
      }
    }
    if (owned != nullptr) cudaFree(owned);
  }
};

PeerBuffer::~PeerBuffer() = default;

// ---- PeerContext -------------------------------------------------------------------------

namespace {
bool envOverride(const char* name, bool dflt) { return envFlag(name, dflt); }
}  // namespace

PeerContext::PeerContext(std::shared_ptr<Context> context, int dev, PeerOptions opts)
    : rank(context->rank), size(context->size), device(dev), context_(context), opts_(opts) {
  GLB_ENFORCE_LE(size, kMaxRanks, "PeerContext supports at most ", kMaxRanks, " ranks");
  GLB_ENFORCE(deviceCount() > 0, "PeerContext needs a CUDA device");
  GLB_ENFORCE(device >= 0 && device < deviceCount(), "invalid CUDA device ", device);
  opts_.useVmm = envOverride("CUDA_VMM", opts_.useVmm);
  opts_.useNvls = envOverride("CUDA_NVLS", opts_.useNvls);
  long stageMb = envInt("CUDA_STAGE_MB", -1);
  if (stageMb > 0) opts_.stageBytes = static_cast<size_t>(stageMb) << 20;
  // Point-to-point shape (must be the same on every rank, like every other option here).
  if (long v = envInt("CUDA_P2P_LANES", -1); v > 0) opts_.p2pLanes = static_cast<int>(v);
  if (long v = envInt("CUDA_P2P_SLOTS", -1); v > 0) opts_.p2pSlots = static_cast<int>(v);
  if (long v = envInt("CUDA_P2P_SLOT_KB", -1); v > 0) opts_.p2pSlotBytes = static_cast<size_t>(v) << 10;
  if (long v = envInt("CUDA_EXCHANGE_BLOCKS", -1); v > 0) opts_.exchangeBlocks = static_cast<int>(v);

  DeviceGuard g(device);
  GLB_CUDA_CHECK(cudaFree(nullptr));
  // Load every kernel now, while no peer can be spinning on this device yet.
  preloadAllreduceKernels();
  preloadCollectiveKernels();
  preloadMoeKernels();
  preloadScheduleKernels();
  preloadLocalKernels();
  preloadPipelineKernels();
  preloadP2pKernels();
  preloadAllreduceNormKernels();
  ensureTuningLoaded();
  fdChannel_ = std::make_unique<FdChannel>(rank);
  exchangeTopology();

  // Symmetric pool: [SignalPad | LL lines | p2p mailboxes | staging]. Zero-initialised
  // (epoch 0, no LL line carries a valid sequence number).
  opts_.llMaxBytes = roundUp(std::max<size_t>(opts_.llMaxBytes, 1024), 1024);
  opts_.p2pLanes = std::max(1, std::min(opts_.p2pLanes, kP2pLanes - 2));  // the last two lanes belong to exchange()
  opts_.p2pSlots = std::max(2, opts_.p2pSlots);
  opts_.p2pSlotBytes = roundUp(std::max<size_t>(opts_.p2pSlotBytes, 16u * 1024), static_cast<size_t>(opts_.p2pLanes) * 16);
  llOffset_ = roundUp(sizeof(SignalPad), 4096);
  llSrcStride_ = opts_.llMaxBytes * 2;  // a 16-byte line carries 8 bytes of payload
  mailboxOffset_ = llOffset_ + roundUp(2 * llSrcStride_ * static_cast<size_t>(size), 4096);
  stageOffset_ = mailboxOffset_ + roundUp(mailboxStride() * static_cast<size_t>(size), 4096);
  stageBytes_ = roundUp(opts_.stageBytes, 4096);
  pool_ = allocSymmetric(stageOffset_ + stageBytes_);
  comm_.rank = rank;
  comm_.nranks = size;
  for (int i = 0; i < kMaxRanks; i++) comm_.sig[i] = static_cast<SignalPad*>(i < size ? pool_->peer[i] : nullptr);
  comm_.self = comm_.sig[rank];
  // Status word the kernels raise when a device-side wait gives up.
  GLB_CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&hostStatus_), 64, cudaHostAllocMapped | cudaHostAllocPortable));
  std::memset(hostStatus_, 0, 64);
  GLB_CUDA_CHECK(cudaHostGetDevicePointer(reinterpret_cast<void**>(&hostStatusDev_), hostStatus_, 0));
  comm_.hostStatus = hostStatusDev_;
  static_assert(16 + sizeof(InputStatus) <= 64, "the input status must fit the pinned status block");
  inputStatus_ = reinterpret_cast<InputStatus*>(reinterpret_cast<char*>(hostStatus_) + 16);
  inputStatusDev_ = reinterpret_cast<InputStatus*>(reinterpret_cast<char*>(hostStatusDev_) + 16);
  setTimeout(std::chrono::duration_cast<std::chrono::milliseconds>(context->getTimeout()));
  GLB_CUDA_CHECK(cudaEventCreateWithFlags(&orderEvent_, cudaEventDisableTiming));
  localTiles_ = std::make_unique<TileCounter>(device);
  hostBarrier();
  GLB_INFO(describe());
}

PeerContext::~PeerContext() {
  DeviceGuard g(device);
  cudaDeviceSynchronize();
  if (orderEvent_ != nullptr) cudaEventDestroy(orderEvent_);
  if (hostStatus_ != nullptr) cudaFreeHost(hostStatus_);
  pool_.reset();
  std::lock_guard<std::mutex> lk(ipcMu_);
  for (auto& kv : ipcCache_) cudaIpcCloseMemHandle(kv.second);
  ipcCache_.clear();
}

std::shared_ptr<Context> PeerContext::context() const {
  auto c = context_.lock();
  GLB_ENFORCE(c != nullptr, "the context this PeerContext was built on has been destroyed");
  return c;
}

bool PeerContext::sameProcess(int r) const {
  return infos_[r].pid == infos_[rank].pid && std::strcmp(infos_[r].hostname, infos_[rank].hostname) == 0;
}

template <typename T>
std::vector<T> PeerContext::allgatherStruct(const T& mine) {
  static_assert(std::is_trivially_copyable<T>::value, "POD only");
  std::vector<T> all(size);
  all[rank] = mine;
  if (size > 1) {
    AllgatherOptions o(context());
    o.setOutputRaw(all.data(), all.size() * sizeof(T));
    o.setTag(nextTag());
    allgather(o);
  }
  return all;
}

bool PeerContext::hostAllSame(const std::vector<int64_t>& words) {
  struct Words {
    int64_t n;
    int64_t w[16];
  };
  GLB_ENFORCE(words.size() <= 16, "hostAllSame: at most 16 words");
  Words mine{};
  mine.n = static_cast<int64_t>(words.size());
  std::copy(words.begin(), words.end(), mine.w);
  for (const Words& o : allgatherStruct(mine)) {
    if (std::memcmp(&o, &mine, sizeof(Words)) != 0) return false;
  }
  return true;
}

void PeerContext::hostBarrier() {
  BarrierOptions o(context());
  o.setTag(nextTag());
  barrier(o);
}

namespace {
// NVLink state through NVML, loaded at run time (the library ships with the driver).
void queryNvlink(const char* pciBusId, int32_t* active, int32_t* version) {
  *active = -1;
  *version = -1;
  static void* lib = dlopen("libnvidia-ml.so.1", RTLD_NOW);
  if (lib == nullptr) return;
  using Handle = void*;
  auto init = reinterpret_cast<int (*)()>(dlsym(lib, "nvmlInit_v2"));
  auto byPci = reinterpret_cast<int (*)(const char*, Handle*)>(dlsym(lib, "nvmlDeviceGetHandleByPciBusId_v2"));
  auto state = reinterpret_cast<int (*)(Handle, unsigned, unsigned*)>(dlsym(lib, "nvmlDeviceGetNvLinkState"));
  auto ver = reinterpret_cast<int (*)(Handle, unsigned, unsigned*)>(dlsym(lib, "nvmlDeviceGetNvLinkVersion"));
  if (init == nullptr || byPci == nullptr || state == nullptr || init() != 0) return;
  Handle h = nullptr;
  if (byPci(pciBusId, &h) != 0) return;
  int n = 0;
  for (unsigned link = 0; link < 32; link++) {
    unsigned on = 0;
    if (state(h, link, &on) != 0) break;
    n += on ? 1 : 0;
  }
  *active = n;
  unsigned v = 0;
  if (ver != nullptr && ver(h, 0, &v) == 0) *version = static_cast<int32_t>(v);
}
}  // namespace

void PeerContext::exchangeTopology() {
  DeviceInfo me;
  std::memset(&me, 0, sizeof(me));
  std::strncpy(me.hostname, getHostname().c_str(), sizeof(me.hostname) - 1);
  me.pid = static_cast<int32_t>(::getpid());
  me.device = device;
  cudaDeviceProp prop;
  GLB_CUDA_CHECK(cudaGetDeviceProperties(&prop, device));
  std::memcpy(me.uuid, prop.uuid.bytes, 16);
  std::strncpy(me.pciBusId, devicePCIBusId(device).c_str(), sizeof(me.pciBusId) - 1);
  me.smCount = prop.multiProcessorCount;
  me.ccMajor = prop.major;
  me.ccMinor = prop.minor;
  me.totalMem = prop.totalGlobalMem;
  std::strncpy(me.fdSocket, fdChannel_->name().c_str(), sizeof(me.fdSocket) - 1);
  queryNvlink(me.pciBusId, &me.nvlinkActive, &me.nvlinkVersion);
  me.nicDistance = -1;
  {
    // lower-case bus id as sysfs spells it
    std::string gpu(me.pciBusId);
    for (auto& c : gpu) c = static_cast<char>(std::tolower(static_cast<unsigned char>(c)));
    for (const auto& nic : pciDevices(kPCIClassNetwork, 0xff0000)) {
      const int d = pciDistance(gpu, nic);
      if (d >= 0 && (me.nicDistance < 0 || d < me.nicDistance)) {
        me.nicDistance = d;
        std::strncpy(me.nearestNic, nic.c_str(), sizeof(me.nearestNic) - 1);
      }
    }
  }
  try {
    const auto& d = driver();
    CUdevice cudev;
    GLB_CU_CHECK(d.cuDeviceGet(&cudev, device));
    int v = 0;
    if (d.cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, cudev) == CUDA_SUCCESS) {
      me.vmmSupported = v;
    }
    v = 0;
    if (d.haveMulticast &&
        d.cuDeviceGetAttribute(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, cudev) == CUDA_SUCCESS) {
      me.multicastSupported = v;
    }
  } catch (const std::exception& e) {
    GLB_WARN("CUDA driver API unavailable (", e.what(), "); using cudaIpc only");
  }
  infos_ = allgatherStruct(me);

  bool sameHost = true, allVmm = true, allMc = true;
  std::set<std::string> uuids;
  ranksOnMyDevice_ = 0;
  for (int r = 0; r < size; r++) {
    const auto& in = infos_[r];
    const bool host = std::strcmp(in.hostname, me.hostname) == 0;
    sameHost = sameHost && host;
    allVmm = allVmm && in.vmmSupported;
    allMc = allMc && in.multicastSupported;
    uuids.insert(strcat_all(in.hostname, ":", std::string(reinterpret_cast<const char*>(in.uuid), 16)));
    if (host && std::memcmp(in.uuid, me.uuid, 16) == 0) ranksOnMyDevice_++;
  }
  // Peer access: find each peer's device among the devices visible here (by UUID).
  peerOk_ = sameHost;
  const int ndev = deviceCount();
  for (int r = 0; r < size && peerOk_; r++) {
    if (std::memcmp(infos_[r].uuid, me.uuid, 16) == 0) continue;
    for (int d = 0; d < ndev; d++) {
      cudaDeviceProp p;
      if (cudaGetDeviceProperties(&p, d) != cudaSuccess) continue;
      if (std::memcmp(p.uuid.bytes, infos_[r].uuid, 16) != 0) continue;
      int can = 0;
      cudaDeviceCanAccessPeer(&can, device, d);
      if (!can) peerOk_ = false;
      break;
    }
    // Not visible here: NVSwitch boxes still allow the mapping; failures surface at import time.
  }
  vmm_ = opts_.useVmm && allVmm && sameHost;
  nvlsPossible_ = opts_.useNvls && vmm_ && allMc && size > 1 && static_cast<int>(uuids.size()) == size;
  // Grids must be identical on every rank (CTA b pairs with CTA b of each peer), so the
  // co-residency cap uses the most crowded device and the smallest GPU of the job.
  struct Shape {
    int32_t ranksOnDevice;
    int32_t sms;
  } mineShape{ranksOnMyDevice_, me.smCount};
  auto shapes = allgatherStruct(mineShape);
  worstRanksPerDevice_ = 1;
  minSms_ = me.smCount;
  for (const auto& sh : shapes) {
    worstRanksPerDevice_ = std::max(worstRanksPerDevice_, static_cast<int>(sh.ranksOnDevice));
    minSms_ = std::min(minSms_, static_cast<int>(sh.sms));
  }
  maxBlocks_ = std::max(1, std::min(kMaxBlocks, minSms_ / std::max(1, worstRanksPerDevice_)));
}

std::string PeerContext::describe() const {
  std::ostringstream os;
  os << "PeerContext rank " << rank << "/" << size << " dev " << device << " (" << infos_[rank].pciBusId
     << ", " << infos_[rank].smCount << " SMs, sm_" << infos_[rank].ccMajor << infos_[rank].ccMinor << ")"
     << " peerAccess=" << peerOk_ << " alloc=" << (vmm_ ? "vmm+fd" : "cudaIpc")
     << " nvls=" << (nvlsAvailable() ? "yes" : "no") << " nvlinks=" << infos_[rank].nvlinkActive << "(v"
     << infos_[rank].nvlinkVersion << ") nic=" << (infos_[rank].nearestNic[0] ? infos_[rank].nearestNic : "?") << "@"
     << infos_[rank].nicDistance << " ranksOnDevice=" << ranksOnMyDevice_
     << " maxBlocks=" << maxBlocks_ << " stageMB=" << (stageBytes_ >> 20);
  return os.str();
}

PeerPtrs PeerContext::stagePtrs(size_t byteOffset) const { return pool_->ptrsAt(stageOffset_ + byteOffset); }

PeerPtrs PeerContext::llPtrs() const { return pool_->ptrsAt(llOffset_); }

PeerPtrs PeerContext::mailboxPtrs() const { return pool_->ptrsAt(mailboxOffset_); }

void PeerContext::setTimeout(std::chrono::milliseconds t) {
  timeout_ = t;
  long forced = envInt("CUDA_TIMEOUT_MS", -1);
  if (forced >= 0) timeout_ = std::chrono::milliseconds(forced);
  comm_.timeoutNs = timeout_.count() > 0 ? static_cast<unsigned long long>(timeout_.count()) * 1000000ull : 0ull;
}

void PeerContext::checkHealth() {
  if (!poisoned_) {
    const uint32_t st = *static_cast<volatile uint32_t*>(hostStatus_);
    if (st == 0) {
      volatile InputStatus* in = inputStatus_;
      const uint32_t code = in->code;
      if (code == kInputOk) return;
      const uint32_t who = in->rank;
      const unsigned long long need = in->need, avail = in->avail;
      const uint32_t expert = in->expert;
      in->code = kInputOk;  // raised once; the next call starts clean
      if (code == kInputSlotOverflow) {
        GLB_THROW(InputException, "alltoallv_ll_topk: source rank ", who, " routed ", need, " rows to expert ", expert,
                  " (index rank * experts + e) but a (source, expert) slot group holds max_tokens = ", avail,
                  " rows; none of those rows were sent (a token picked that expert more than once)");
      }
      if (code == kInputOverflow) {
        GLB_THROW(InputException, "alltoallv_dev: rank ", who, " needs ", need, " output rows but has room for ", avail,
                  "; no rows were sent to it");
      }
      GLB_THROW(InputException,
                "alltoallv_dev: invalid splits (a negative or > 2^31-1 count, an offset outside the input, splits "
                "summing to more rows than the input has, a top-k position outside the dispatch input, or arguments "
                "that differ between ranks); nothing was sent");
    }
    poisoned_ = true;
    const uint32_t code = st & 0xffu, who = st >> 8;
    poisonReason_ = code == kAbortTimeout
                        ? strcat_all("rank ", who, " did not reach a device-side barrier within ", timeout_.count(), " ms")
                        : strcat_all("a peer aborted a collective (first missing rank: ", who, ")");
    GLB_ERROR("PeerContext rank ", rank, ": ", poisonReason_, " - the context is unusable from here on");
  }
  GLB_THROW_IO_EXCEPTION("CUDA peer context failed: ", poisonReason_);
}

void PeerContext::synchronize(cudaStream_t stream) {
  DeviceGuard g(device);
  GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
  checkHealth();
}

void PeerContext::orderStreams(cudaStream_t stream) {
  // The previous collective recorded `orderEvent_` right after its launch. The stream handle
  // of that launch is only ever COMPARED here, never used: it may belong to a stream that
  // has been destroyed since.
  if (haveLastStream_ && stream != lastStream_) {
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    cudaStreamIsCapturing(stream, &cs);
    if (cs == cudaStreamCaptureStatusNone) GLB_CUDA_CHECK(cudaStreamWaitEvent(stream, orderEvent_, 0));
  }
}

void PeerContext::markLaunched(cudaStream_t stream) {
  cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
  cudaStreamIsCapturing(stream, &cs);
  if (cs != cudaStreamCaptureStatusNone) return;  // inside a graph the capture order is the order
  GLB_CUDA_CHECK(cudaEventRecord(orderEvent_, stream));
  lastStream_ = stream;
  haveLastStream_ = true;
}

int PeerContext::coResidentBlocks(const void* kernel, int threads, size_t dynamicSmem) {
  std::lock_guard<std::mutex> g(occMu_);
  const auto key = std::make_pair(kernel, dynamicSmem);
  auto it = occupancy_.find(key);
  int perSm = 1;
  if (it != occupancy_.end()) {
    perSm = it->second;
  } else {
    DeviceGuard dg(device);
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kernel, threads, dynamicSmem) == cudaSuccess && n > 0) perSm = n;
    cudaGetLastError();
    occupancy_[key] = perSm;
  }
  return std::max(1, std::min(kMaxBlocks, minSms_ * perSm / std::max(1, worstRanksPerDevice_)));
}

std::shared_ptr<PeerBuffer> PeerContext::tryAllocMulticastLoopback(size_t bytes, std::string* why) {
  std::string dummy;
  std::string& w = why != nullptr ? *why : dummy;
  if (size != 1) {
    w = "needs a single-rank context";
    return nullptr;
  }
  if (!vmm_ || !infos_[rank].multicastSupported) {
    w = "no VMM / multicast support on this device";
    return nullptr;
  }
  try {
    DeviceGuard g(device);
    auto b = allocVmm(bytes, true);
    if (b->mc == nullptr) {
      w = "the driver refused a one-device multicast object";
      return nullptr;
    }
    return b;
  } catch (const std::exception& e) {
    w = e.what();
    return nullptr;
  }
}

CommArgs PeerContext::loopbackComm(int virtualRanks) const {
  GLB_ENFORCE(virtualRanks >= 1 && virtualRanks <= kMaxRanks, "loopback: 1..", kMaxRanks, " virtual ranks");
  CommArgs c = comm_;
  c.rank = 0;
  c.nranks = virtualRanks;
  SignalPad* me = static_cast<SignalPad*>(pool_->local);
  c.self = me;
  for (int i = 0; i < kMaxRanks; i++) {
    // sig[i]->flag[b][0] aliases me->flag[b][i]
    c.sig[i] = i < virtualRanks ? reinterpret_cast<SignalPad*>(reinterpret_cast<uint32_t*>(me) + i) : nullptr;
  }
  return c;
}

void* PeerContext::stageMc(size_t byteOffset) const {
  return pool_->mc ? static_cast<char*>(pool_->mc) + stageOffset_ + byteOffset : nullptr;
}

bool PeerContext::agree(bool mine) {
  auto all = allgatherStruct(static_cast<int>(mine ? 1 : 0));
  for (int v : all) {
    if (!v) return false;
  }
  return true;
}

std::shared_ptr<PeerBuffer> PeerContext::resolveBuffer(void* ptr, size_t bytes, size_t* byteOffset) {
  std::shared_ptr<PeerBuffer> hit;
  size_t off = 0;
  {
    std::lock_guard<std::mutex> g(symMu_);
    for (auto it = symmetric_.begin(); it != symmetric_.end();) {
      auto b = it->lock();
      if (!b) {
        it = symmetric_.erase(it);
        continue;
      }
      char* base = static_cast<char*>(b->local);
      char* p = static_cast<char*>(ptr);
      if (p >= base && p + bytes <= base + b->bytes) {
        hit = b;
        off = static_cast<size_t>(p - base);
      }
      ++it;
    }
  }
  // Symmetric use needs the same offset everywhere (peer pointers are base + offset).
  struct Probe {
    int found;
    int pad;
    uint64_t off;
  } mine{hit ? 1 : 0, 0, off};
  auto all = allgatherStruct(mine);
  bool everywhere = true;
  for (const auto& x : all) everywhere = everywhere && x.found && x.off == all[0].off;
  if (everywhere && hit) {
    *byteOffset = off;
    return hit;
  }
  *byteOffset = 0;
  return registerBuffer(ptr, bytes);
}

std::shared_ptr<PeerBuffer> PeerContext::allocSymmetricImpl(size_t bytes) {
  GLB_ENFORCE(peerOk_ || size == 1, "allocSymmetric: peers are not all P2P-reachable from this device");
  DeviceGuard g(device);
  if (vmm_) {
    // Agree on the path first: a rank whose VMM allocation fails must not leave the others hanging.
    std::shared_ptr<PeerBuffer> buf;
    int ok = 1;
    std::string err;
    try {
      buf = allocVmm(bytes, nvlsPossible_);
    } catch (const std::exception& e) {
      ok = 0;
      err = e.what();
    }
    auto oks = allgatherStruct(ok);
    bool all = true;
    for (int v : oks) all = all && v;
    if (all) return buf;
    if (!err.empty()) GLB_WARN("VMM symmetric allocation failed on rank ", rank, ": ", err, " - falling back to cudaIpc");
    buf.reset();
    vmm_ = false;
    nvlsPossible_ = false;
  }
  return allocIpc(bytes);
}

std::shared_ptr<PeerBuffer> PeerContext::allocSymmetric(size_t bytes) {
  auto b = allocSymmetricImpl(bytes);
  std::lock_guard<std::mutex> g(symMu_);
  symmetric_.push_back(b);
  return b;
}

namespace {
struct VmmExchange {
  uint64_t ptr;
  uint64_t size;
  int32_t ok;
  int32_t pad;
};
}  // namespace

std::shared_ptr<PeerBuffer> PeerContext::allocVmm(size_t bytes, bool wantMc) {
  const auto& d = driver();
  auto impl = std::make_shared<PeerBuffer::Impl>();
  impl->device = device;
  auto buf = std::make_shared<PeerBuffer>();
  buf->impl_ = impl;

  CUmemAllocationProp prop;
  std::memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;

  VmmExchange mine{0, 0, 0, 0};
  int exportedFd = -1;
  CUmemGenericAllocationHandle handle = 0;
  size_t gran = 0, mapSize = 0;
  std::string err;
  try {
    GLB_CU_CHECK(d.cuMemGetAllocationGranularity(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
    if (wantMc) {
      CUmulticastObjectProp mp;
      std::memset(&mp, 0, sizeof(mp));
      mp.numDevices = static_cast<unsigned>(size);
      mp.size = roundUp(bytes, gran);
      mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      size_t mg = 0;
      if (d.cuMulticastGetGranularity(&mg, &mp, CU_MULTICAST_GRANULARITY_RECOMMENDED) == CUDA_SUCCESS && mg > gran) {
        gran = mg;
      }
    }
    mapSize = roundUp(bytes, gran);
    GLB_CU_CHECK(d.cuMemCreate(&handle, mapSize, &prop, 0));
    PeerBuffer::Impl::Mapping m;
    m.handle = handle;
    m.haveHandle = true;
    m.size = mapSize;
    impl->mappings.push_back(m);
    CUdeviceptr va = 0;
    GLB_CU_CHECK(d.cuMemAddressReserve(&va, mapSize, gran, 0, 0));
    impl->mappings.back().va = va;
    GLB_CU_CHECK(d.cuMemMap(va, mapSize, 0, handle, 0));
    // Grant access to this device and to the devices of ranks that live in this
    // process (they use our VA directly).
    std::vector<CUmemAccessDesc> descs;
    std::set<int> devs{device};
    for (int r = 0; r < size; r++) {
      if (sameProcess(r)) devs.insert(infos_[r].device);
    }
    for (int dv : devs) {
      CUmemAccessDesc ad;
      std::memset(&ad, 0, sizeof(ad));
      ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      ad.location.id = dv;
      ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      descs.push_back(ad);
    }
    GLB_CU_CHECK(d.cuMemSetAccess(va, mapSize, descs.data(), descs.size()));
    GLB_CUDA_CHECK(cudaMemset(reinterpret_cast<void*>(va), 0, mapSize));
    GLB_CUDA_CHECK(cudaDeviceSynchronize());
    GLB_CU_CHECK(d.cuMemExportToShareableHandle(&exportedFd, handle, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
    mine.ptr = static_cast<uint64_t>(va);
    mine.size = mapSize;
    mine.ok = 1;
  } catch (const std::exception& e) {
    err = e.what();
  }

  auto all = allgatherStruct(mine);
  bool everyone = true;
  for (const auto& x : all) everyone = everyone && x.ok;
  if (!everyone) {
    if (exportedFd >= 0) ::close(exportedFd);
    GLB_THROW(Exception, "VMM allocation failed on some rank", err.empty() ? "" : ": ", err);
  }

  buf->local = reinterpret_cast<void*>(mine.ptr);
  buf->bytes = bytes;
  buf->peer[rank] = buf->local;
  buf->vectorOk = true;
  const uint32_t tag = nextTag();
  for (int r = 0; r < size; r++) {
    if (r == rank || sameProcess(r)) continue;
    fdChannel_->sendFd(infos_[r].fdSocket, exportedFd, rank, tag);
  }
  int importOk = 1;
  std::string importErr;
  for (int r = 0; r < size; r++) {
    if (r == rank) continue;
    if (sameProcess(r)) {
      buf->peer[r] = reinterpret_cast<void*>(all[r].ptr);
      continue;
    }
    try {
      int fd = fdChannel_->recvFd(r, tag, context()->getTimeout());
      CUmemGenericAllocationHandle h = 0;
      CUresult res = d.cuMemImportFromShareableHandle(&h, reinterpret_cast<void*>(static_cast<uintptr_t>(fd)),
                                                      CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
      ::close(fd);
      GLB_CU_CHECK(res);
      PeerBuffer::Impl::Mapping m;
      m.handle = h;
      m.haveHandle = true;
      m.size = all[r].size;
      impl->mappings.push_back(m);
      CUdeviceptr va = 0;
      GLB_CU_CHECK(d.cuMemAddressReserve(&va, m.size, gran, 0, 0));
      impl->mappings.back().va = va;
      GLB_CU_CHECK(d.cuMemMap(va, m.size, 0, h, 0));
      CUmemAccessDesc ad;
      std::memset(&ad, 0, sizeof(ad));
      ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
      ad.location.id = device;
      ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
      GLB_CU_CHECK(d.cuMemSetAccess(va, m.size, &ad, 1));
      buf->peer[r] = reinterpret_cast<void*>(va);
    } catch (const std::exception& e) {
      importOk = 0;
      importErr = e.what();
    }
  }
  if (exportedFd >= 0) ::close(exportedFd);
  {
    auto oks = allgatherStruct(importOk);
    for (int v : oks) {
      if (!v) GLB_THROW(Exception, "importing a peer allocation failed", importErr.empty() ? "" : ": ", importErr);
    }
  }

  // ---- NVLS: bind the allocation to a multicast object -------------------------------
  if (wantMc) {
    int mcOk = 1;
    std::string mcErr;
    CUmemGenericAllocationHandle mc = 0;
    bool haveMc = false;
    const uint32_t mtag = nextTag();
    try {
      CUmulticastObjectProp mp;
      std::memset(&mp, 0, sizeof(mp));
      mp.numDevices = static_cast<unsigned>(size);
      mp.size = mapSize;
      mp.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
      if (rank == 0) {
        GLB_CU_CHECK(d.cuMulticastCreate(&mc, &mp));
        haveMc = true;
        int mfd = -1;
        GLB_CU_CHECK(d.cuMemExportToShareableHandle(&mfd, mc, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
        for (int r = 1; r < size; r++) fdChannel_->sendFd(infos_[r].fdSocket, mfd, 0, mtag);
        ::close(mfd);
      } else {
        int mfd = fdChannel_->recvFd(0, mtag, context()->getTimeout());
        CUresult res = d.cuMemImportFromShareableHandle(&mc, reinterpret_cast<void*>(static_cast<uintptr_t>(mfd)),
                                                        CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        ::close(mfd);
        GLB_CU_CHECK(res);
        haveMc = true;
      }
      CUdevice cudev;
      GLB_CU_CHECK(d.cuDeviceGet(&cudev, device));
      GLB_CU_CHECK(d.cuMulticastAddDevice(mc, cudev));
    } catch (const std::exception& e) {
      mcOk = 0;
      mcErr = e.what();
    }
    // Everyone must have added its device before anyone binds memory.
    auto oks = allgatherStruct(mcOk);
    bool all1 = true;
    for (int v : oks) all1 = all1 && v;
    if (all1) {
      try {
        GLB_CU_CHECK(d.cuMulticastBindMem(mc, 0, handle, 0, mapSize, 0));
        PeerBuffer::Impl::Mapping m;
        m.handle = mc;
        m.haveHandle = true;
        m.size = mapSize;
        haveMc = false;  // ownership moved to the mapping list
        impl->mappings.push_back(m);
        CUdeviceptr va = 0;
        GLB_CU_CHECK(d.cuMemAddressReserve(&va, mapSize, gran, 0, 0));
        impl->mappings.back().va = va;
        GLB_CU_CHECK(d.cuMemMap(va, mapSize, 0, mc, 0));
        CUmemAccessDesc ad;
        std::memset(&ad, 0, sizeof(ad));
        ad.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
        ad.location.id = device;
        ad.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
        GLB_CU_CHECK(d.cuMemSetAccess(va, mapSize, &ad, 1));
        buf->mc = reinterpret_cast<void*>(va);
      } catch (const std::exception& e) {
        mcOk = 0;
        mcErr = e.what();
      }
      oks = allgatherStruct(mcOk);
      for (int v : oks) all1 = all1 && v;
    }
    if (!all1) {
      if (!mcErr.empty()) GLB_WARN("NVLS multicast setup failed on rank ", rank, ": ", mcErr, " - continuing without NVLS");
      // Not sticky: running out of multicast objects for one allocation must not disable
      // NVLS for the rest of the job.
      buf->mc = nullptr;
      if (haveMc) d.cuMemRelease(mc);
    }
  }
  return buf;
}

std::shared_ptr<PeerBuffer> PeerContext::allocIpc(size_t bytes) {
  void* p = nullptr;
  GLB_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(bytes, 16)));
  GLB_CUDA_CHECK(cudaMemset(p, 0, std::max<size_t>(bytes, 16)));
  GLB_CUDA_CHECK(cudaDeviceSynchronize());
  return shareIpc(p, bytes, /*ownsAllocation=*/true);
}

std::shared_ptr<PeerBuffer> PeerContext::registerBuffer(void* ptr, size_t bytes) {
  GLB_ENFORCE(peerOk_ || size == 1, "registerBuffer: peers are not all P2P-reachable from this device");
  DeviceGuard g(device);
  return shareIpc(ptr, bytes, /*ownsAllocation=*/false);
}

namespace {
struct IpcExchange {
  cudaIpcMemHandle_t handle;
  uint64_t rawPtr;
  uint64_t offset;
  uint64_t bytes;
  int32_t status;  // 1 ok
  int32_t aligned;
};
}  // namespace

std::shared_ptr<PeerBuffer> PeerContext::shareIpc(void* ptr, size_t bytes, bool ownsAllocation) {
  auto impl = std::make_shared<PeerBuffer::Impl>();
  impl->device = device;
  if (ownsAllocation) impl->owned = ptr;
  auto buf = std::make_shared<PeerBuffer>();
  buf->impl_ = impl;
  buf->local = ptr;
  buf->bytes = bytes;

  IpcExchange mine;
  std::memset(&mine, 0, sizeof(mine));
  mine.rawPtr = reinterpret_cast<uint64_t>(ptr);
  mine.bytes = bytes;
  mine.aligned = (reinterpret_cast<uintptr_t>(ptr) % 16 == 0) ? 1 : 0;
  mine.status = 1;
  bool needHandle = false;
  for (int r = 0; r < size; r++) needHandle = needHandle || (r != rank && !sameProcess(r));
  std::string err;
  if (needHandle && ptr != nullptr) {
    // cudaIpc handles name the whole allocation: find its base.
    void* base = ptr;
    try {
      CUdeviceptr b = 0;
      size_t sz = 0;
      if (driver().cuMemGetAddressRange(&b, &sz, reinterpret_cast<CUdeviceptr>(ptr)) == CUDA_SUCCESS && b != 0) {
        base = reinterpret_cast<void*>(b);
      }
    } catch (...) {
    }
    mine.offset = static_cast<uint64_t>(static_cast<char*>(ptr) - static_cast<char*>(base));
    cudaError_t e = cudaIpcGetMemHandle(&mine.handle, base);
    if (e != cudaSuccess) {
      cudaGetLastError();
      mine.status = 0;
      err = strcat_all("cudaIpcGetMemHandle: ", cudaGetErrorString(e));
    }
  }
  auto all = allgatherStruct(mine);
  for (int r = 0; r < size; r++) {
    if (!all[r].status) {
      GLB_THROW(Exception, "rank ", r, " could not export its buffer for peer access", r == rank ? ": " + err : "");
    }
  }
  bool aligned = true;
  int openOk = 1;
  std::string openErr;
  for (int r = 0; r < size; r++) {
    aligned = aligned && all[r].aligned;
    if (r == rank) {
      buf->peer[r] = ptr;
      continue;
    }
    if (sameProcess(r)) {
      buf->peer[r] = reinterpret_cast<void*>(all[r].rawPtr);
      if (infos_[r].device != device) {
        cudaError_t e = cudaDeviceEnablePeerAccess(infos_[r].device, 0);
        if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) {
          openOk = 0;
          openErr = strcat_all("cudaDeviceEnablePeerAccess: ", cudaGetErrorString(e));
        }
        cudaGetLastError();
      }
      continue;
    }
    if (all[r].rawPtr == 0) continue;
    std::lock_guard<std::mutex> lk(ipcMu_);
    auto key = std::make_pair(r, std::string(reinterpret_cast<const char*>(&all[r].handle), sizeof(cudaIpcMemHandle_t)));
    auto it = ipcCache_.find(key);
    void* basePtr = nullptr;
    if (it != ipcCache_.end()) {
      basePtr = it->second;
    } else {
      cudaError_t e = cudaIpcOpenMemHandle(&basePtr, all[r].handle, cudaIpcMemLazyEnablePeerAccess);
      if (e != cudaSuccess) {
        cudaGetLastError();
        openOk = 0;
        openErr = strcat_all("cudaIpcOpenMemHandle(rank ", r, "): ", cudaGetErrorString(e));
        continue;
      }
      ipcCache_[key] = basePtr;
    }
    buf->peer[r] = static_cast<char*>(basePtr) + all[r].offset;
  }
  buf->vectorOk = aligned;
  auto oks = allgatherStruct(openOk);
  for (int v : oks) {
    if (!v) GLB_THROW(Exception, "mapping a peer buffer failed", openErr.empty() ? "" : ": ", openErr);
  }
  return buf;
}

}  // namespace cuda
}  // namespace glb
