#include "glb/cuda/local_ops.h"

#include <set>

#include "glb/common/linux.h"
#include "glb/common/utils.h"
#include "glb/cuda/kernels.h"

namespace glb {

namespace {
template <typename T>
std::vector<CudaDevicePointer<T>> ranges(std::vector<CudaDevicePointer<T>>& ptrs, size_t offset, size_t count) {
  std::vector<CudaDevicePointer<T>> out;
  for (auto& p : ptrs) out.push_back(p.range(offset, count));
  return out;
}

// Stream 0 waits for everything already queued on the other streams (their buffers may
// still be written by earlier work).
void gather(std::vector<CudaStream>& streams) {
  for (size_t i = 1; i < streams.size(); i++) {
    streams[i].record();
    streams[0].waitOn(streams[i]);
  }
}
void scatterOrder(std::vector<CudaStream>& streams) {
  streams[0].record();
  for (size_t i = 1; i < streams.size(); i++) streams[i].waitOn(streams[0]);
}
}  // namespace

// ---- native -------------------------------------------------------------------------------------

template <typename T, typename Dst>
CudaLocalNativeReduce<T, Dst>::CudaLocalNativeReduce(std::vector<CudaStream>& streams,
                                                     std::vector<CudaDevicePointer<T>>& devicePtrs, Dst& target,
                                                     const CudaReductionFunction<T>* fn, size_t offset, size_t count)
    : streams_(streams), srcs_(ranges(devicePtrs, offset, count)), target_(target.range(offset, count)), fn_(fn) {
  GLB_ENFORCE_EQ(streams_.size(), devicePtrs.size(), "one stream per pointer");
  targetIsFirst_ = static_cast<const void*>(*target_) == static_cast<const void*>(*srcs_[0]);
  // Sources on other GPUs are read directly by the reduce kernel.
  cuda::DeviceGuard g(srcs_[0].getDeviceID());
  for (auto& s : srcs_) {
    if (s.getDeviceID() != srcs_[0].getDeviceID()) {
      cudaError_t e = cudaDeviceEnablePeerAccess(s.getDeviceID(), 0);
      if (e != cudaSuccess && e != cudaErrorPeerAccessAlreadyEnabled) GLB_CUDA_CHECK(e);
      cudaGetLastError();
    }
  }
}

template <typename T, typename Dst>
void CudaLocalNativeReduce<T, Dst>::runAsync() {
  cuda::DeviceGuard g(srcs_[0].getDeviceID());
  gather(streams_);
  const size_t n = srcs_[0].getCount();
  if (srcs_.size() > 1) {
    std::vector<const void*> in;
    for (auto& s : srcs_) in.push_back(*s);
    cuda::launchLocalReduceMany(*srcs_[0], in.data(), static_cast<int>(in.size()), n, DataTypeOf<T>::value, fn_->type(),
                                *streams_[0]);
    cuda::noteLaunch();
  }
  if (!targetIsFirst_) streams_[0].copyAsync(*target_, *srcs_[0], n * sizeof(T));
  scatterOrder(streams_);
}

template <typename T, typename Dst>
void CudaLocalNativeReduce<T, Dst>::wait() {
  streams_[0].record();
  streams_[0].wait();
}

template <typename T, typename Src>
CudaLocalNativeBroadcast<T, Src>::CudaLocalNativeBroadcast(std::vector<CudaStream>& streams,
                                                           std::vector<CudaDevicePointer<T>>& devicePtrs, Src& source,
                                                           size_t offset, size_t count)
    : streams_(streams), dsts_(ranges(devicePtrs, offset, count)), source_(source.range(offset, count)) {
  GLB_ENFORCE_EQ(streams_.size(), devicePtrs.size(), "one stream per pointer");
}

template <typename T, typename Src>
void CudaLocalNativeBroadcast<T, Src>::runAsync() {
  // Every destination is filled on its own stream (its own copy engine / device).
  const size_t bytes = source_.getCount() * sizeof(T);
  for (size_t i = 0; i < dsts_.size(); i++) {
    if (static_cast<const void*>(*dsts_[i]) == static_cast<const void*>(*source_)) continue;
    streams_[i].copyAsync(*dsts_[i], *source_, bytes);
  }
}

template <typename T, typename Src>
void CudaLocalNativeBroadcast<T, Src>::wait() {
  for (auto& s : streams_) s.wait();
}

// ---- host ---------------------------------------------------------------------------------------

template <typename T>
CudaLocalHostReduce<T>::CudaLocalHostReduce(std::vector<CudaStream>& streams, std::vector<CudaDevicePointer<T>>& devicePtrs,
                                            CudaHostPointer<T>& target, const CudaReductionFunction<T>* fn, size_t offset,
                                            size_t count)
    : streams_(streams), srcs_(ranges(devicePtrs, offset, count)), target_(target.range(offset, count)), fn_(fn) {
  for (size_t i = 1; i < srcs_.size(); i++) scratch_.push_back(CudaHostPointer<T>::alloc(count));
}

template <typename T>
void CudaLocalHostReduce<T>::runAsync() {
  const size_t bytes = srcs_[0].getCount() * sizeof(T);
  streams_[0].copyAsync(*target_, *srcs_[0], bytes);
  for (size_t i = 1; i < srcs_.size(); i++) streams_[i].copyAsync(*scratch_[i - 1], *srcs_[i], bytes);
}

template <typename T>
void CudaLocalHostReduce<T>::wait() {
  streams_[0].wait();
  for (size_t i = 1; i < srcs_.size(); i++) {
    streams_[i].wait();
    fn_->callHost(*target_, *scratch_[i - 1], srcs_[0].getCount());
  }
}

template <typename T>
CudaLocalHostBroadcast<T>::CudaLocalHostBroadcast(std::vector<CudaStream>& streams,
                                                  std::vector<CudaDevicePointer<T>>& devicePtrs, CudaHostPointer<T>& source,
                                                  size_t offset, size_t count)
    : streams_(streams), dsts_(ranges(devicePtrs, offset, count)), source_(source.range(offset, count)) {}

template <typename T>
void CudaLocalHostBroadcast<T>::runAsync() {
  for (size_t i = 0; i < dsts_.size(); i++) streams_[i].copyAsync(*dsts_[i], *source_, source_.getCount() * sizeof(T));
}

template <typename T>
void CudaLocalHostBroadcast<T>::wait() {
  for (auto& s : streams_) s.wait();
}

// ---- NCCL ---------------------------------------------------------------------------------------

namespace {
template <typename T>
std::vector<int> devicesOf(const std::vector<CudaDevicePointer<T>>& ptrs) {
  std::vector<int> d;
  for (const auto& p : ptrs) d.push_back(p.getDeviceID());
  return d;
}
template <typename T>
int indexOfPointer(const std::vector<CudaDevicePointer<T>>& ptrs, const void* p, const char* what) {
  for (size_t i = 0; i < ptrs.size(); i++) {
    if (static_cast<const void*>(*ptrs[i]) == p) return static_cast<int>(i);
  }
  GLB_THROW_INVALID_OPERATION_EXCEPTION(what, ": the root pointer must be one of the device pointers");
}
}  // namespace

template <typename T>
CudaLocalNCCLReduce<T>::CudaLocalNCCLReduce(std::vector<CudaStream>& streams, std::vector<CudaDevicePointer<T>>& devicePtrs,
                                            CudaDevicePointer<T>& target, const CudaReductionFunction<T>* fn, size_t offset,
                                            size_t count)
    : streams_(streams), srcs_(ranges(devicePtrs, offset, count)), target_(target.range(offset, count)), fn_(fn) {
  root_ = indexOfPointer(srcs_, *target_, "CudaLocalNCCLReduce");
  comms_ = cuda::NcclComm::initAll(devicesOf(srcs_));
}

template <typename T>
void CudaLocalNCCLReduce<T>::runAsync() {
  std::lock_guard<std::mutex> g(cuda::CudaShared::getMutex());
  cuda::NcclComm::groupStart();
  for (size_t i = 0; i < srcs_.size(); i++) {
    cuda::DeviceGuard dg(srcs_[i].getDeviceID());
    comms_[i]->reduce(*srcs_[i], *srcs_[i], srcs_[i].getCount(), DataTypeOf<T>::value, fn_->type(), root_, *streams_[i]);
  }
  cuda::NcclComm::groupEnd();
}

template <typename T>
void CudaLocalNCCLReduce<T>::wait() {
  for (auto& s : streams_) {
    s.record();
    s.wait();
  }
}

template <typename T>
CudaLocalNCCLBroadcast<T>::CudaLocalNCCLBroadcast(std::vector<CudaStream>& streams,
                                                  std::vector<CudaDevicePointer<T>>& devicePtrs, CudaDevicePointer<T>& source,
                                                  size_t offset, size_t count)
    : streams_(streams), dsts_(ranges(devicePtrs, offset, count)), source_(source.range(offset, count)) {
  root_ = indexOfPointer(dsts_, *source_, "CudaLocalNCCLBroadcast");
  comms_ = cuda::NcclComm::initAll(devicesOf(dsts_));
}

template <typename T>
void CudaLocalNCCLBroadcast<T>::runAsync() {
  std::lock_guard<std::mutex> g(cuda::CudaShared::getMutex());
  cuda::NcclComm::groupStart();
  for (size_t i = 0; i < dsts_.size(); i++) {
    cuda::DeviceGuard dg(dsts_[i].getDeviceID());
    comms_[i]->broadcast(*dsts_[i], *dsts_[i], dsts_[i].getCount(), DataTypeOf<T>::value, root_, *streams_[i]);
  }
  cuda::NcclComm::groupEnd();
}

template <typename T>
void CudaLocalNCCLBroadcast<T>::wait() {
  for (auto& s : streams_) {
    s.record();
    s.wait();
  }
}

// ---- dispatch -----------------------------------------------------------------------------------

namespace cuda {
bool localOpsUseNccl(const std::vector<int>& devices, size_t bytes) {
  if (devices.size() < 2 || envFlag("CUDA_LOCAL_NATIVE", false)) return false;
  std::set<int> distinct(devices.begin(), devices.end());
  if (distinct.size() != devices.size()) return false;  // NCCL needs one rank per GPU (nccl.cu:111-116)
  if (bytes < static_cast<size_t>(envInt("CUDA_LOCAL_NCCL_MIN", 256 * 1024))) return false;
  return ncclAvailable();
}
}  // namespace cuda

template <typename T>
std::unique_ptr<LocalOp<T>> cudaDeviceReduce(std::vector<CudaStream>& streams, std::vector<CudaDevicePointer<T>>& devicePtrs,
                                             CudaDevicePointer<T>& targetPtr, const CudaReductionFunction<T>* fn,
                                             size_t offset, size_t count) {
  if (cuda::localOpsUseNccl(devicesOf(devicePtrs), count * sizeof(T))) {
    try {
      return std::make_unique<CudaLocalNCCLReduce<T>>(streams, devicePtrs, targetPtr, fn, offset, count);
    } catch (const std::exception&) {  // root not among the pointers, dtype unknown to NCCL, ...
    }
  }
  return std::make_unique<CudaLocalNativeReduce<T, CudaDevicePointer<T>>>(streams, devicePtrs, targetPtr, fn, offset, count);
}

template <typename T>
std::unique_ptr<LocalOp<T>> cudaDeviceBroadcast(std::vector<CudaStream>& streams,
                                                std::vector<CudaDevicePointer<T>>& devicePtrs,
                                                CudaDevicePointer<T>& sourcePtr, size_t offset, size_t count) {
  if (cuda::localOpsUseNccl(devicesOf(devicePtrs), count * sizeof(T))) {
    try {
      return std::make_unique<CudaLocalNCCLBroadcast<T>>(streams, devicePtrs, sourcePtr, offset, count);
    } catch (const std::exception&) {
    }
  }
  return std::make_unique<CudaLocalNativeBroadcast<T, CudaDevicePointer<T>>>(streams, devicePtrs, sourcePtr, offset, count);
}

template <typename T>
std::unique_ptr<LocalOp<T>> cudaHostReduce(std::vector<CudaStream>& streams, std::vector<CudaDevicePointer<T>>& devicePtrs,
                                           CudaHostPointer<T>& targetPtr, const CudaReductionFunction<T>* fn, size_t offset,
                                           size_t count) {
  // One pointer: plain D2H. Several: reduce on the device first (one kernel, one D2H)
  // unless asked to reduce on the CPU.
  if (devicePtrs.size() > 1 && envFlag("CUDA_LOCAL_HOST_REDUCE", false)) {
    return std::make_unique<CudaLocalHostReduce<T>>(streams, devicePtrs, targetPtr, fn, offset, count);
  }
  return std::make_unique<CudaLocalNativeReduce<T, CudaHostPointer<T>>>(streams, devicePtrs, targetPtr, fn, offset, count);
}

template <typename T>
std::unique_ptr<LocalOp<T>> cudaHostBroadcast(std::vector<CudaStream>& streams, std::vector<CudaDevicePointer<T>>& devicePtrs,
                                              CudaHostPointer<T>& sourcePtr, size_t offset, size_t count) {
  return std::make_unique<CudaLocalHostBroadcast<T>>(streams, devicePtrs, sourcePtr, offset, count);
}

template <typename T>
int findCudaDevicePointerClosestToDevice(std::vector<CudaDevicePointer<T>>& ptrs,
                                         const std::shared_ptr<transport::Device>& dev) {
  if (ptrs.empty() || !dev) return 0;
  const std::string& nic = dev->getPCIBusID();
  if (nic.empty()) return 0;
  int best = 0, bestDist = 1 << 30;
  for (size_t i = 0; i < ptrs.size(); i++) {
    const std::string gpu = cuda::devicePCIBusId(ptrs[i].getDeviceID());
    if (gpu.empty()) continue;
    const int d = pciDistance(nic, gpu);
    if (d >= 0 && d < bestDist) {
      bestDist = d;
      best = static_cast<int>(i);
    }
  }
  return best;
}

#define GLB_INSTANTIATE(T)                                                                                            \
  template class CudaLocalNativeReduce<T, CudaDevicePointer<T>>;                                                      \
  template class CudaLocalNativeReduce<T, CudaHostPointer<T>>;                                                        \
  template class CudaLocalNativeBroadcast<T, CudaDevicePointer<T>>;                                                   \
  template class CudaLocalNativeBroadcast<T, CudaHostPointer<T>>;                                                     \
  template class CudaLocalHostReduce<T>;                                                                              \
  template class CudaLocalHostBroadcast<T>;                                                                           \
  template class CudaLocalNCCLReduce<T>;                                                                              \
  template class CudaLocalNCCLBroadcast<T>;                                                                           \
  template std::unique_ptr<LocalOp<T>> cudaDeviceReduce<T>(std::vector<CudaStream>&, std::vector<CudaDevicePointer<T>>&, \
                                                           CudaDevicePointer<T>&, const CudaReductionFunction<T>*,    \
                                                           size_t, size_t);                                           \
  template std::unique_ptr<LocalOp<T>> cudaDeviceBroadcast<T>(std::vector<CudaStream>&,                               \
                                                              std::vector<CudaDevicePointer<T>>&,                     \
                                                              CudaDevicePointer<T>&, size_t, size_t);                 \
  template std::unique_ptr<LocalOp<T>> cudaHostReduce<T>(std::vector<CudaStream>&, std::vector<CudaDevicePointer<T>>&, \
                                                         CudaHostPointer<T>&, const CudaReductionFunction<T>*, size_t, \
                                                         size_t);                                                     \
  template std::unique_ptr<LocalOp<T>> cudaHostBroadcast<T>(std::vector<CudaStream>&,                                 \
                                                            std::vector<CudaDevicePointer<T>>&, CudaHostPointer<T>&,  \
                                                            size_t, size_t);                                          \
  template int findCudaDevicePointerClosestToDevice<T>(std::vector<CudaDevicePointer<T>>&,                            \
                                                       const std::shared_ptr<transport::Device>&);
GLB_INSTANTIATE(int8_t)
GLB_INSTANTIATE(uint8_t)
GLB_INSTANTIATE(int32_t)
GLB_INSTANTIATE(int64_t)
GLB_INSTANTIATE(uint64_t)
GLB_INSTANTIATE(float)
GLB_INSTANTIATE(double)
GLB_INSTANTIATE(float16)
GLB_INSTANTIATE(bfloat16)
GLB_INSTANTIATE(float8_e4m3)
GLB_INSTANTIATE(float8_e5m2)
#undef GLB_INSTANTIATE

}  // namespace glb
