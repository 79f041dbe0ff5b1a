// Local (single-device-visible) element-wise kernels:
//   localReduce       dst[i] = dst[i] (op) src[i]   — the building block behind
//                     CudaReductionFunction; 128-bit loads/stores, fp32 accumulate
//                     for fp16/bf16, size_t counts, grid sized to the SM count.
//   localReduceMany   dst = reduce(srcs[0..n)) in one pass (multi-pointer local reduce:
//                     srcs may live on peer devices of the same process).
//   localAllreduceMany every buffer := scale * reduce(all buffers), one pass (fused reduce+broadcast).
//   localBroadcast    copy src to n destinations in one pass.
//   verify            whole-buffer closed-form check on the device (bench / smoke).
//   fill / spin       test helpers (pattern fill; delay kernel that surfaces
//                     missing stream synchronisation).
// Parity: gloo/cuda.cu:274-407 (K1-K5), cuda_private.cu:38-61 (K6),
// test/cuda_base_test.cu:15-27 (K7) — rewritten, not ported: the reference kernels
// are scalar, int-indexed, one element per thread.
#include <cstdio>
#include <string>

#include "glb/common/utils.h"
#include "glb/cuda/bulk_copy.cuh"
#include "glb/cuda/cuda_util.h"
#include "glb/cuda/device_common.cuh"
#include "glb/cuda/kernels.h"

namespace glb {
namespace cuda {

namespace {

constexpr int kLocalThreads = 256;
constexpr int kMaxSrcs = 16;
// localAllreduceManyBulkKernel's pipeline (measurements above LocalShape).
constexpr uint32_t kLocalBulkTile = 16 * 1024;  // bytes of one buffer per tile
constexpr int kLocalBulkStages = 3;
constexpr int kLocalBulkCtasPerSm = 1;
constexpr size_t kLocalBulkMinBytes = 1 << 20;  // per buffer; below it the LDG/STG kernel is faster

struct SrcPtrs {
  const void* p[kMaxSrcs];
};
struct DstPtrs {
  void* p[kMaxSrcs];
};

template <typename T>
__global__ void __launch_bounds__(kLocalThreads)
localReduceManyKernel(T* __restrict__ dst, SrcPtrs srcs, int nsrc, size_t count, DevOp op, bool vectorOk) {
  using PT = PackTraits<T>;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t nvec = vectorOk ? count / PT::kElems : 0;
  for (size_t v = tid; v < nvec; v += nthreads) {
    typename PT::AccPack acc = PT::widen(ld128_stream(static_cast<const char*>(srcs.p[0]) + v * 16));
    for (int s = 1; s < nsrc; s++) PT::combine(acc, ld128_stream(static_cast<const char*>(srcs.p[s]) + v * 16), op);
    st128(reinterpret_cast<char*>(dst) + v * 16, PT::narrow(acc));
  }
  using TA = TailAcc<T>;
  for (size_t i = nvec * PT::kElems + tid; i < count; i += nthreads) {
    typename TA::type acc = TA::load(static_cast<const T*>(srcs.p[0])[i]);
    for (int s = 1; s < nsrc; s++) acc = TA::combine(acc, TA::load(static_cast<const T*>(srcs.p[s])[i]), op);
    dst[i] = TA::store(acc);
  }
}

// Elements [first, count) of the fused local allreduce one at a time, grid stride from `tid`.
template <typename T>
__device__ __forceinline__ void localAllreduceScalar(const DstPtrs& bufs, int n, size_t first, size_t count, DevOp op,
                                                     float scale, size_t tid, size_t nthreads) {
  using TA = TailAcc<T>;
  for (size_t i = first + tid; i < count; i += nthreads) {
    typename TA::type acc = TA::load(static_cast<const T*>(bufs.p[0])[i]);
    for (int s = 1; s < n; s++) acc = TA::combine(acc, TA::load(static_cast<const T*>(bufs.p[s])[i]), op);
    if (scale != 1.0f) acc = TA::scale(acc, scale);
    const T res = TA::store(acc);
    for (int s = 0; s < n; s++) static_cast<T*>(bufs.p[s])[i] = res;
  }
}

// Fused local allreduce: every one of the n buffers ends up holding scale * reduce(all n),
// in ONE pass (n reads + n writes per element). This is the whole step when a job has a
// single rank with several local pointers (CudaAllreduce* with ptrs.size() > 1, size == 1,
// and CudaAllreduceLocal): previously a reduce pass followed by a broadcast pass.
// U = 128-bit packs per thread and trip (loads of all trips are issued before the first
// store); kTiled: a CTA works on a contiguous tile of U x blockDim packs per trip (fewer DRAM
// pages open at once) instead of striding the whole grid between the U packs.
template <typename T, int U, bool kTiled>
__global__ void __launch_bounds__(kLocalThreads)
localAllreduceManyKernel(DstPtrs bufs, int n, size_t count, DevOp op, float scale, bool vectorOk) {
  using PT = PackTraits<T>;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t nvec = vectorOk ? count / PT::kElems : 0;
  const size_t first = kTiled ? static_cast<size_t>(blockIdx.x) * blockDim.x * U + threadIdx.x : tid;
  const size_t inner = kTiled ? blockDim.x : nthreads;  // distance between the U packs of one trip
  for (size_t v0 = first; v0 < nvec; v0 += nthreads * U) {
    typename PT::AccPack acc[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * inner;
      if (v < nvec) {
        acc[u] = PT::widen(ld128_stream(static_cast<const char*>(bufs.p[0]) + v * 16));
        for (int s = 1; s < n; s++) PT::combine(acc[u], ld128_stream(static_cast<const char*>(bufs.p[s]) + v * 16), op);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * inner;
      if (v < nvec) {
        if (scale != 1.0f) PT::scale(acc[u], scale);
        const Pack16 r = PT::narrow(acc[u]);
        for (int s = 0; s < n; s++) st128_stream(static_cast<char*>(bufs.p[s]) + v * 16, r);
      }
    }
  }
  localAllreduceScalar<T>(bufs, n, nvec * PT::kElems, count, op, scale, tid, nthreads);
}

// The same step as a TMA (cp.async.bulk) pipeline. The vector is cut into tiles of
// kLocalBulkTile bytes for a persistent grid of one CTA per SM. Each CTA keeps kLocalBulkStages
// stages of n tiles (one per buffer) in dynamic shared memory: thread 0 loads the tile of stage
// k + stages - 1 from every buffer against one mbarrier while the CTA reduces stage k in shared
// memory into the buffer-0 slot, which thread 0 then stores back to all n buffers as one bulk
// group. The arithmetic per 16-byte pack is PackTraits<T>'s in the same order as
// localAllreduceManyKernel, and what is left after the last whole tile goes through the same
// pack and scalar code, so both kernels give the same bits. All pointers must be 16-byte aligned.
//
// Tiles are dealt on demand, so an SM that runs slower than the others takes fewer of them
// instead of ending the step last. A CTA's first stages - 1 tiles are blockIdx.x + j * gridDim.x,
// so the pipeline fills with no atomic on its path; every later one is claimed from `tiles` by
// thread 0, one stage ahead of its load. A CTA stops at its first claim past the end, so a launch
// makes exactly (tiles past the static ones) + gridDim.x claims, and the last of them sets
// *tiles back to zero for the next launch.
template <typename T>
__global__ void __launch_bounds__(kLocalThreads)
localAllreduceManyBulkKernel(DstPtrs bufs, int n, size_t count, DevOp op, float scale, unsigned int* tiles) {
  using PT = PackTraits<T>;
  constexpr uint32_t tile = kLocalBulkTile;
  constexpr int stages = kLocalBulkStages;
  extern __shared__ __align__(128) char smem[];  // [stages][n][tile]
  __shared__ uint64_t full[stages];
  __shared__ size_t slot[stages];  // the tile in each stage; ntiles or more: none, the CTA is done
  const size_t ntiles = count * sizeof(T) / tile;
  const size_t firstClaimed = static_cast<size_t>(stages - 1) * gridDim.x;
  const size_t claims = (ntiles > firstClaimed ? ntiles - firstClaimed : 0) + gridDim.x;
  const size_t stageBytes = static_cast<size_t>(n) * tile;
  if (threadIdx.x == 0) {
    for (int s = 0; s < stages; s++) mbarInit(&full[s], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto claimed = [&](unsigned int c) -> size_t {  // thread 0: the tile that ticket c (from atomicAdd) stands for
    if (c + 1 == claims) *tiles = 0;  // every other claim of this launch has been made
    return firstClaimed + c;
  };
  auto load = [&](size_t k, size_t t) {  // thread 0: tile t into stage k % stages; false past the end
    const int s = static_cast<int>(k % stages);
    slot[s] = t;
    if (t >= ntiles) {
      mbarExpectTx(&full[s], 0);  // completes the phase with no bytes: the waiting threads read `slot` and stop
      return false;
    }
    mbarExpectTx(&full[s], static_cast<uint32_t>(stageBytes));
    for (int b = 0; b < n; b++) bulkLoad(smem + s * stageBytes + b * tile, static_cast<const char*>(bufs.p[b]) + t * tile, tile, &full[s]);
    return true;
  };
  bool more = true;  // thread 0: no claim has come back past the end yet
  if (threadIdx.x == 0) {
    for (int k = 0; more && k < stages - 1; k++) {
      const size_t t = blockIdx.x + static_cast<size_t>(k) * gridDim.x;
      more = load(k, t < ntiles ? t : claimed(atomicAdd(tiles, 1u)));
    }
  }
  const uint32_t packs = tile / 16;
  for (size_t k = 0;; k++) {
    const int s = static_cast<int>(k % stages);
    char* st = smem + s * stageBytes;
    // The ticket for stage k + stages - 1, taken now and first looked at by the refill below, so
    // that warp 0 does not wait for the atomic: its latency hides behind this stage.
    const unsigned int ticket = threadIdx.x == 0 && more ? atomicAdd(tiles, 1u) : 0u;
    mbarWait(&full[s], static_cast<uint32_t>(k / stages) & 1u);
    const size_t t = slot[s];
    if (t >= ntiles) break;
    for (uint32_t v = threadIdx.x; v < packs; v += blockDim.x) {
      typename PT::AccPack acc = PT::widen(*reinterpret_cast<const Pack16*>(st + v * 16));
      for (int b = 1; b < n; b++) PT::combine(acc, *reinterpret_cast<const Pack16*>(st + b * tile + v * 16), op);
      if (scale != 1.0f) PT::scale(acc, scale);
      *reinterpret_cast<Pack16*>(st + v * 16) = PT::narrow(acc);
    }
    fenceProxyAsyncShared();
    __syncthreads();
    if (threadIdx.x == 0) {
      for (int b = 0; b < n; b++) bulkStore(static_cast<char*>(bufs.p[b]) + t * tile, st, tile);
      bulkCommit();
      // Refill the stage of k - 1 once its stores have read it (stage k's may still run).
      if (more) {
        bulkWaitRead<1>();
        more = load(k + stages - 1, claimed(ticket));
      }
    }
  }
  // Past the whole tiles: the remaining packs, then the elements after the last whole pack.
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t nvec = count / PT::kElems;
  for (size_t v = ntiles * (tile / 16) + tid; v < nvec; v += nthreads) {
    typename PT::AccPack acc = PT::widen(ld128_stream(static_cast<const char*>(bufs.p[0]) + v * 16));
    for (int b = 1; b < n; b++) PT::combine(acc, ld128_stream(static_cast<const char*>(bufs.p[b]) + v * 16), op);
    if (scale != 1.0f) PT::scale(acc, scale);
    const Pack16 r = PT::narrow(acc);
    for (int b = 0; b < n; b++) st128_stream(static_cast<char*>(bufs.p[b]) + v * 16, r);
  }
  localAllreduceScalar<T>(bufs, n, nvec * PT::kElems, count, op, scale, tid, nthreads);
  if (threadIdx.x == 0) bulkWaitAll();  // the shared memory the stores read lives as long as the CTA
}

// Whole-buffer check against the closed form start + stride * i (evaluated in fp64, like
// fillKernel): counts elements outside rtol/atol and remembers the first offender.
template <typename T>
__global__ void verifyKernel(const T* buf, size_t count, double start, double stride, double rtol, double atol,
                             unsigned long long* result /* [0]=mismatches, [1]=first bad index + 1 */) {
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  unsigned long long bad = 0;
  for (size_t i = tid; i < count; i += nthreads) {
    const double want = start + stride * static_cast<double>(i);
    const double got = static_cast<double>(Scalar<T>::toAcc(buf[i]));
    const double err = fabs(got - want);
    if (!(err <= atol + rtol * fabs(want))) {
      bad++;
      atomicMin(&result[1], static_cast<unsigned long long>(i) + 1ull);
    }
  }
  if (bad) atomicAdd(&result[0], bad);
}

__global__ void __launch_bounds__(kLocalThreads)
localBroadcastKernel(DstPtrs dsts, int ndst, const char* __restrict__ src, size_t bytes, bool vectorOk) {
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t nvec = vectorOk ? bytes / 16 : 0;
  for (size_t v = tid; v < nvec; v += nthreads) {
    const Pack16 p = ld128_stream(src + v * 16);
    for (int d = 0; d < ndst; d++) st128_stream(static_cast<char*>(dsts.p[d]) + v * 16, p);
  }
  for (size_t i = nvec * 16 + tid; i < bytes; i += nthreads) {
    const char c = src[i];
    for (int d = 0; d < ndst; d++) static_cast<char*>(dsts.p[d])[i] = c;
  }
}

template <typename T>
__global__ void fillKernel(T* dst, size_t count, double start, double stride) {
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = tid; i < count; i += nthreads) {
    const double v = start + stride * static_cast<double>(i);
    dst[i] = Scalar<T>::fromAcc(static_cast<typename Scalar<T>::Acc>(v));
  }
}

__global__ void spinKernel(long long cycles) {
  const long long start = clock64();
  while (clock64() - start < cycles) {
  }
}

// Measured on an H100 80GB HBM3 (SXM, power limit 400 W, max SM clock 1980 MHz), 2 x 400 MB
// fp32, device timed, p50 of 20 launches (scripts/bench_local.py and a sweep in the same
// process, every variant repeated and the repeats within 0.3 %):
//  * localAllreduceManyKernel (LDG/STG): 4 CTAs/SM x 1 pack 0.577 ms (2.77 TB/s). From the
//    earlier sweep on a 700 W card: x 2 packs 0.579, 6 CTAs/SM 0.588, 8 CTAs/SM 0.601,
//    2 CTAs/SM 0.681, the tiled variant within 0.5 % of the grid-stride one.
//  * localAllreduceManyBulkKernel: 16 KB tiles x 3 stages x 1 CTA/SM 0.558 ms (2.87 TB/s).
//    32 KB x 3 and 32 KB x 2 0.558-0.560, 16 KB x 4 and x 6 0.559-0.562, 8 KB x 4 0.564,
//    2 CTAs/SM 0.560-0.575, 4 KB tiles 0.570-1.14. Refilling a stage before the reduction of
//    the next tile instead of after it, and L2 evict-first hints on the copies, were each
//    0.3-2 % slower.
//  * Ceilings in the same process: cudaMemcpyAsync device to device of the same 1.6 GB
//    0.539 ms (2.97 TB/s), the n = 1 in-place copy 0.586 ms through LDG/STG and 0.562 ms
//    through the bulk kernel; one write of both buffers 3.22 TB/s.
//  * Per call with the L2 flushed (p50 of 50): the bulk kernel loses at 256 KB per buffer
//    (64 K floats 8.4 us against 7.4; the mbarrier set-up and the pipeline fill) and wins from
//    1 MB (256 K floats 9.2 against 10.6 us, 1 M 13.7 against 18.3, 10 M 64 against 70).
// On an H100 80GB HBM3 at 700 W (same clock), scripts/bench_local.py: LDG/STG step 0.574 ms
// (2.79 TB/s), bulk step 0.537 ms (2.98 TB/s), cudaMemcpyAsync D2D 0.537 ms (2.98 TB/s), in-place
// copy 0.587 (LDG/STG) and 0.563 ms (bulk), read-only 2.87 TB/s, write-only 3.21 TB/s; bench.py's
// N=1 step 0.535-0.537 ms (median 0.5355 of six runs).
//  * Bulk tiles dealt round-robin (a fixed 184 or 185 per CTA) instead of on demand: median 0.549 ms
//    of six runs alternated with the above (0.548-0.550, one run at 0.556).
//    Per-CTA %globaltimer at exit, p50 over 100 launches: the slowest CTA ended 8.6 us after the
//    median one (1.6 % of the step) and the first 110 us before the last; on demand, 1.6 us (0.3 %).
//    Claiming a tile right before its load instead of a stage ahead was 0.4 % slower.
struct LocalShape {
  int ctasPerSm = 4;
  int unroll = 1;
  bool tiled = false;
  bool pinned = false;  // a shape was set explicitly: every call runs the LDG/STG kernel with it
};

LocalShape localShapeFromEnv() {
  LocalShape s;
  const std::string v = envStr("LOCAL_SHAPE", "");
  int a = 0, b = 0, c = 0;
  if (!v.empty() && std::sscanf(v.c_str(), "%d,%d,%d", &a, &b, &c) == 3) {
    if (a >= 1 && a <= 8) s.ctasPerSm = a;
    if (b == 1 || b == 2 || b == 4) s.unroll = b;
    s.tiled = c != 0;
    s.pinned = true;
  }
  return s;
}

LocalShape& localShape() {
  static LocalShape s = localShapeFromEnv();
  return s;
}

int gridFor(size_t items, int threads, int ctasPerSm = 4) {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  size_t want = (items + threads - 1) / threads;
  size_t cap = static_cast<size_t>(sms) * static_cast<size_t>(ctasPerSm);
  return static_cast<int>(want < 1 ? 1 : (want > cap ? cap : want));
}

// The LDG/STG fused-step instantiation for a launch shape (unroll 1, 2 or 4).
template <typename T>
auto localAllreduceFn(int unroll, bool tiled) {
  if (tiled) {
    if (unroll == 4) return localAllreduceManyKernel<T, 4, true>;
    if (unroll == 1) return localAllreduceManyKernel<T, 1, true>;
    return localAllreduceManyKernel<T, 2, true>;
  }
  if (unroll == 4) return localAllreduceManyKernel<T, 4, false>;
  if (unroll == 1) return localAllreduceManyKernel<T, 1, false>;
  return localAllreduceManyKernel<T, 2, false>;
}

bool aligned16(const void* p) { return reinterpret_cast<uintptr_t>(p) % 16 == 0; }

}  // namespace

void launchLocalReduceMany(void* dst, const void* const* srcs, int nsrc, size_t count, DataType dt, ReduceOp op,
                           cudaStream_t stream) {
  if (count == 0 || nsrc == 0) return;
  SrcPtrs sp;
  bool vectorOk = aligned16(dst);
  for (int i = 0; i < nsrc && i < kMaxSrcs; i++) {
    sp.p[i] = srcs[i];
    vectorOk = vectorOk && aligned16(srcs[i]);
  }
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    const int grid = gridFor(count / PackTraits<T>::kElems + 1, kLocalThreads);
    localReduceManyKernel<T><<<grid, kLocalThreads, 0, stream>>>(static_cast<T*>(dst), sp, nsrc, count,
                                                                static_cast<DevOp>(op), vectorOk);
  });
}

bool localAllreduceUsesBulk(void* const* bufs, int n, size_t count, DataType dt) {
  if (n < 1 || n > kMaxSrcs || count * elementSize(dt) < kLocalBulkMinBytes) return false;
  for (int i = 0; i < n; i++) {
    if (!aligned16(bufs[i])) return false;
  }
  int dev = 0, smemOptin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&smemOptin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  return static_cast<size_t>(kLocalBulkStages) * n * kLocalBulkTile * kLocalBulkCtasPerSm <= static_cast<size_t>(smemOptin);
}

TileCounter::TileCounter(int device) {
  DeviceGuard g(device);
  GLB_CUDA_CHECK(cudaMalloc(&p_, sizeof(*p_)));
  // Zeroed before the constructor returns: the launches that use it may come on any stream,
  // including ones that do not synchronise with the legacy default stream.
  GLB_CUDA_CHECK(cudaMemsetAsync(p_, 0, sizeof(*p_), 0));
  GLB_CUDA_CHECK(cudaStreamSynchronize(0));
}

TileCounter::~TileCounter() { cudaFree(p_); }

void launchLocalAllreduceMany(void* const* bufs, int n, size_t count, DataType dt, ReduceOp op, float scale,
                              unsigned int* tileCounter, cudaStream_t stream) {
  if (count == 0 || n == 0) return;
  DstPtrs bp;
  bool vectorOk = true;
  for (int i = 0; i < n && i < kMaxSrcs; i++) {
    bp.p[i] = bufs[i];
    vectorOk = vectorOk && aligned16(bufs[i]);
  }
  const LocalShape shape = localShape();
  if (!shape.pinned && localAllreduceUsesBulk(bufs, n, count, dt)) {
    const size_t smem = static_cast<size_t>(kLocalBulkStages) * n * kLocalBulkTile;
    dispatchType(dt, [&](auto tag) {
      using T = decltype(tag);
      const auto kernel = localAllreduceManyBulkKernel<T>;
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, static_cast<int>(smem));
      const int grid = gridFor(count * sizeof(T) / kLocalBulkTile * kLocalThreads, kLocalThreads, kLocalBulkCtasPerSm);
      kernel<<<grid, kLocalThreads, smem, stream>>>(bp, n, count, static_cast<DevOp>(op), scale, tileCounter);
    });
    return;
  }
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    // Launch shape: measured on H100 (scripts/bench_local.py); GLB_LOCAL_SHAPE = "<ctas per SM>,<unroll>,<tiled>".
    const int grid = gridFor(count / PackTraits<T>::kElems / shape.unroll + 1, kLocalThreads, shape.ctasPerSm);
    localAllreduceFn<T>(shape.unroll, shape.tiled)<<<grid, kLocalThreads, 0, stream>>>(bp, n, count,
                                                                                     static_cast<DevOp>(op), scale,
                                                                                     vectorOk);
  });
}

void launchVerify(const void* buf, size_t count, DataType dt, double start, double stride, double rtol, double atol,
                  unsigned long long* deviceResult, cudaStream_t stream) {
  if (count == 0) return;
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    verifyKernel<T><<<gridFor(count, 256), 256, 0, stream>>>(static_cast<const T*>(buf), count, start, stride, rtol,
                                                             atol, deviceResult);
  });
}

void launchLocalReduce(void* dst, const void* src, size_t count, DataType dt, ReduceOp op, cudaStream_t stream) {
  const void* srcs[2] = {dst, src};
  launchLocalReduceMany(dst, srcs, 2, count, dt, op, stream);
}

void launchLocalBroadcast(void* const* dsts, int ndst, const void* src, size_t bytes, cudaStream_t stream) {
  if (bytes == 0 || ndst == 0) return;
  DstPtrs dp;
  bool vectorOk = aligned16(src);
  for (int i = 0; i < ndst && i < kMaxSrcs; i++) {
    dp.p[i] = dsts[i];
    vectorOk = vectorOk && aligned16(dsts[i]);
  }
  const int grid = gridFor(bytes / 16 + 1, kLocalThreads);
  localBroadcastKernel<<<grid, kLocalThreads, 0, stream>>>(dp, ndst, static_cast<const char*>(src), bytes, vectorOk);
}

void launchFill(void* dst, size_t count, DataType dt, double start, double stride, cudaStream_t stream) {
  if (count == 0) return;
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    fillKernel<T><<<gridFor(count, 256), 256, 0, stream>>>(static_cast<T*>(dst), count, start, stride);
  });
}

void launchSpin(long long cycles, cudaStream_t stream) { spinKernel<<<1, 1, 0, stream>>>(cycles); }

void setLocalAllreduceShape(int ctasPerSm, int unroll, bool tiled) {
  LocalShape& s = localShape();
  if (ctasPerSm == 0) {
    s = LocalShape();
    return;
  }
  s.pinned = true;
  if (ctasPerSm >= 1 && ctasPerSm <= 8) s.ctasPerSm = ctasPerSm;
  if (unroll == 1 || unroll == 2 || unroll == 4) s.unroll = unroll;
  s.tiled = tiled;
}

void preloadLocalKernels() {
  for (DataType dt : kAllDataTypes) {
    dispatchType(dt, [](auto tag) {
      using T = decltype(tag);
      touchKernel(localReduceManyKernel<T>);
      for (bool tiled : {false, true}) {
        for (int u : {1, 2, 4}) touchKernel(localAllreduceFn<T>(u, tiled));
      }
      touchKernel(localAllreduceManyBulkKernel<T>);
      touchKernel(verifyKernel<T>);
      touchKernel(fillKernel<T>);
    });
  }
  touchKernel(localBroadcastKernel);
  touchKernel(spinKernel);
  cudaGetLastError();
}

}  // namespace cuda
}  // namespace glb
