// TMA bulk copies (cp.async.bulk, SASS: UBLKCP) for the pure data-movement kernels.
//
// A copy kernel built from LDG/STG needs hundreds of resident threads per SM just to keep
// enough 16-byte accesses in flight over a ~2 us NVLink round trip. The Hopper copy
// engine inside each SM (TMA) moves whole chunks asynchronously instead: ONE thread per CTA
// issues  global -> shared  (completion signalled on an mbarrier) and  shared -> global
// (bulk async-groups); the data never touches registers and the SM's warps stay free.
// Source and destination may be local HBM or a peer GPU's memory (mapped over NVLink).
//
// ctaBulkCopy() streams a contiguous byte range through a ring of STAGES shared-memory
// buffers: while chunk i is being stored to its (one or several) destinations, the loads of
// chunks i+1 .. i+STAGES-1 are already in flight. Loading once and storing P times is what an
// allgather / broadcast wants (the block is read from HBM a single time).
#pragma once

#include <cstdint>

#include "glb/cuda/comm_types.h"

namespace glb {
namespace cuda {

constexpr int kBulkStages = 4;
constexpr uint32_t kBulkChunk = 32 * 1024;  // bytes per stage: 4 x 32 KB = 128 KB of shared memory per CTA
constexpr size_t kBulkSmemBytes = static_cast<size_t>(kBulkStages) * kBulkChunk;

__device__ __forceinline__ uint32_t smemAddr(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbarInit(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smemAddr(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbarExpectTx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smemAddr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ bool mbarTryWait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n .reg .pred p;\n mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n selp.u32 %0, 1, 0, p;\n}"
      : "=r"(ok)
      : "r"(smemAddr(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
// global -> shared, completion (byte count) reported to `bar`.
__device__ __forceinline__ void bulkLoad(void* smem, const void* gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smemAddr(smem)),
               "l"(gmem), "r"(bytes), "r"(smemAddr(bar))
               : "memory");
}
// shared -> global, part of the current bulk async-group.
__device__ __forceinline__ void bulkStore(void* gmem, const void* smem, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gmem), "r"(smemAddr(smem)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulkCommit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// All committed groups have finished READING shared memory (their buffers may be refilled).
__device__ __forceinline__ void bulkWaitRead() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
// All committed groups are complete (their writes are performed).
__device__ __forceinline__ void bulkWaitAll() { asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); }

// Per-CTA state of the ring; lives in static shared memory of the calling kernel.
struct BulkRing {
  uint64_t full[kBulkStages];
  uint32_t phase;  // bit s = parity to wait for on full[s]
};

// Call once per kernel by every thread of the CTA (ends with a __syncthreads()).
__device__ __forceinline__ void bulkRingInit(BulkRing& ring) {
  if (threadIdx.x == 0) {
    for (int s = 0; s < kBulkStages; s++) mbarInit(&ring.full[s], 1);
    ring.phase = 0;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
}

// Thread 0 of the CTA copies [0, bytes) from src to every dst[k] (k < ndst). `bytes` must be a
// multiple of 16 and all pointers 16-byte aligned. Returns with every store COMPLETE (and
// ordered before later generic-proxy operations of this thread), other threads fall through.
template <int MAXDST>
__device__ __forceinline__ void ctaBulkCopy(BulkRing& ring, char* smem, const char* src, char* const (&dst)[MAXDST], int ndst,
                                            size_t bytes) {
  if (threadIdx.x != 0 || bytes == 0) return;
  const size_t npieces = (bytes + kBulkChunk - 1) / kBulkChunk;
  constexpr int L = kBulkStages - 1;  // loads in flight ahead of the store
  uint32_t phase = ring.phase;
  for (size_t i = 0; i < npieces + L; i++) {
    if (i < npieces) {
      const int s = static_cast<int>(i % kBulkStages);
      if (i >= static_cast<size_t>(kBulkStages)) bulkWaitRead();  // the stores that read this buffer are done with it
      const size_t off = i * kBulkChunk;
      const uint32_t sz = static_cast<uint32_t>(bytes - off < kBulkChunk ? bytes - off : kBulkChunk);
      mbarExpectTx(&ring.full[s], sz);
      bulkLoad(smem + static_cast<size_t>(s) * kBulkChunk, src + off, sz, &ring.full[s]);
    }
    if (i >= static_cast<size_t>(L)) {
      const size_t j = i - L;
      const int s = static_cast<int>(j % kBulkStages);
      while (!mbarTryWait(&ring.full[s], (phase >> s) & 1u)) {
      }
      phase ^= 1u << s;
      const size_t off = j * kBulkChunk;
      const uint32_t sz = static_cast<uint32_t>(bytes - off < kBulkChunk ? bytes - off : kBulkChunk);
#pragma unroll
      for (int k = 0; k < MAXDST; k++) {
        if (k < ndst) bulkStore(dst[k] + off, smem + static_cast<size_t>(s) * kBulkChunk, sz);
      }
      bulkCommit();
    }
  }
  bulkWaitAll();
  ring.phase = phase;
  // The copies went through the async proxy; make them ordered before the generic-proxy
  // flag stores (barrier) that announce them.
  asm volatile("fence.proxy.async;" ::: "memory");
}

}  // namespace cuda
}  // namespace glb
