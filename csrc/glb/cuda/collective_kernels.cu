// Data-movement collectives over NVLink peer memory (sm_90a): broadcast,
// allgather(v), alltoall(v), reduce_scatter, reduce, gather(v), scatter. All are
// single kernels bracketed by device-side flag barriers; payload moves with
// 128-bit peer loads/stores (or multimem.st through the NVSwitch where a multicast
// alias exists). None of these has a CUDA variant in the reference (SURVEY §0.6).
#include "glb/cuda/device_common.cuh"
#include "glb/cuda/grid_copy.cuh"
#include "glb/cuda/kernels.h"
#include "glb/cuda/peer_reduce.cuh"

namespace glb {
namespace cuda {

namespace {

__device__ __forceinline__ void shareOfB(size_t n, int parts, int r, size_t& begin, size_t& end) {
  const size_t base = n / parts, rem = n % parts;
  begin = r * base + (static_cast<size_t>(r) < rem ? r : rem);
  end = begin + base + (static_cast<size_t>(r) < rem ? 1 : 0);
}

}  // namespace

// ---- broadcast -----------------------------------------------------------------------
// mode 0: root pushes the whole buffer to every peer (latency regime).
// mode 1: scatter + allgather: root pushes slice i to rank i, then every rank
//         pushes its slice to the others; per-GPU egress ~S instead of (P-1)·S.
// mode 2: NVLS: root issues multimem.st, the switch replicates.
// mode 3: relay, chunk-pipelined: the buffer is cut into chunks of (P-1) slices; the root
//         sends slice j of a chunk to relay j ONLY and raises a per-chunk flag; relay j
//         forwards its slice to the other P-2 ranks while the root is already sending the
//         next chunk. Root egress = S, every other GPU's ingress = S and egress
//         S(P-2)/(P-1): all links run at once, nothing is sent twice over the same port
//         (a single multimem.st source is bound by the root's one egress stream).
__global__ void __launch_bounds__(kThreads, 2)
broadcastKernel(CommArgs a, PeerPtrs bufs, char* mc, size_t bytes, int root, int mode, bool vec, int tile) {
  const uint32_t e = loadEpoch(a);
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = a.nranks;
  uint32_t used = mode == 1 ? 3 : 2;
  const size_t relayChunk = static_cast<size_t>(P - 1) * gridDim.x * static_cast<size_t>(tile);  // 16-byte units
  const uint32_t nchunks = mode == 3 ? static_cast<uint32_t>((bytes / 16 + relayChunk - 1) / relayChunk) : 0u;
  if (mode == 3) used = nchunks + 2;  // one flag value per chunk between the two barriers
  if (!blockBarrier<false>(a, e + 1)) {  // every destination may now be overwritten
    retire(a, used, 0);
    return;
  }
  if (mode == 0) {
    if (a.rank == root) {
      const char* src = static_cast<const char*>(bufs.p[root]);
      const size_t nvec = vec ? bytes / 16 : 0;
      constexpr int U = 4;
      for (size_t v0 = tid; v0 < nvec; v0 += nthreads * U) {
        Pack16 p[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t v = v0 + u * nthreads;
          if (v < nvec) p[u] = ld128_stream(src + v * 16);
        }
        for (int i = 1; i < P; i++) {
          char* dst = static_cast<char*>(bufs.p[(root + i) % P]);
#pragma unroll
          for (int u = 0; u < U; u++) {
            const size_t v = v0 + u * nthreads;
            if (v < nvec) st128_stream(dst + v * 16, p[u]);
          }
        }
      }
      for (size_t i = nvec * 16 + tid; i < bytes; i += nthreads) {
        const char c = src[i];
        for (int r = 1; r < P; r++) static_cast<char*>(bufs.p[(root + r) % P])[i] = c;
      }
    }
  } else if (mode == 2) {
    if (a.rank == root) {
      const char* src = static_cast<const char*>(bufs.p[root]);
      const size_t nvec = bytes / 16;
      constexpr int U = 4;
      for (size_t v0 = tid; v0 < nvec; v0 += nthreads * U) {
        Pack16 p[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t v = v0 + u * nthreads;
          if (v < nvec) p[u] = ld128_stream(src + v * 16);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t v = v0 + u * nthreads;
          if (v < nvec) multimemSt128(mc + v * 16, p[u]);
        }
      }
      for (size_t i = nvec * 16 + tid; i < bytes; i += nthreads) {
        const char c = src[i];
        for (int r = 1; r < P; r++) static_cast<char*>(bufs.p[(root + r) % P])[i] = c;
      }
    }
  } else if (mode == 3) {
    const size_t units = bytes / 16;
    const int R = P - 1;
    constexpr int U = 4;
    if (a.rank == root) {
      const char* src = static_cast<const char*>(bufs.p[root]);
      for (uint32_t c = 0; c < nchunks; c++) {
        for (int j = 0; j < R; j++) {
          const size_t lo = ((static_cast<size_t>(c) * R + j) * gridDim.x + blockIdx.x) * tile;
          if (lo >= units) continue;
          const size_t n = units - lo < static_cast<size_t>(tile) ? units - lo : static_cast<size_t>(tile);
          char* dst = static_cast<char*>(bufs.p[(root + 1 + j) % P]) + lo * 16;
          const char* s = src + lo * 16;
          for (size_t v0 = threadIdx.x; v0 < n; v0 += static_cast<size_t>(blockDim.x) * U) {
            Pack16 p[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t v = v0 + static_cast<size_t>(u) * blockDim.x;
              if (v < n) p[u] = ld128_stream(s + v * 16);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t v = v0 + static_cast<size_t>(u) * blockDim.x;
              if (v < n) st128_stream(dst + v * 16, p[u]);
            }
          }
        }
        __syncthreads();
        if (static_cast<int>(threadIdx.x) < R) {
          st_release_sys(&a.sig[(root + 1 + threadIdx.x) % P]->flag[blockIdx.x][root], e + 2 + c);
        }
      }
      for (size_t i = units * 16 + tid; i < bytes; i += nthreads) {
        const char ch = src[i];
        for (int r = 1; r < P; r++) static_cast<char*>(bufs.p[(root + r) % P])[i] = ch;
      }
    } else {
      const int j = (a.rank - root - 1 + P) % P;
      const char* src = static_cast<const char*>(bufs.p[a.rank]);
      for (uint32_t c = 0; c < nchunks; c++) {
        int ok = 1;
        if (threadIdx.x == 0) ok = waitFlag(a, &a.self->flag[blockIdx.x][root], e + 2 + c, root) ? 1 : 0;
        if (!__syncthreads_and(ok)) break;
        const size_t lo = ((static_cast<size_t>(c) * R + j) * gridDim.x + blockIdx.x) * tile;
        if (lo >= units) continue;
        const size_t n = units - lo < static_cast<size_t>(tile) ? units - lo : static_cast<size_t>(tile);
        const char* s = src + lo * 16;
        for (size_t v0 = threadIdx.x; v0 < n; v0 += static_cast<size_t>(blockDim.x) * U) {
          Pack16 p[U];
#pragma unroll
          for (int u = 0; u < U; u++) {
            const size_t v = v0 + static_cast<size_t>(u) * blockDim.x;
            if (v < n) p[u] = ld128_stream(s + v * 16);
          }
          for (int i = 1; i < P; i++) {
            const int d = (a.rank + i) % P;
            if (d == root) continue;
            char* dst = static_cast<char*>(bufs.p[d]) + lo * 16;
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t v = v0 + static_cast<size_t>(u) * blockDim.x;
              if (v < n) st128_stream(dst + v * 16, p[u]);
            }
          }
        }
      }
    }
  } else {
    // Slices are 16-byte granular so every phase stays vectorised.
    const size_t units = bytes / 16;
    if (a.rank == root) {
      for (int i = 1; i < P; i++) {
        const int dst = (root + i) % P;
        size_t b, en;
        shareOfB(units, P, dst, b, en);
        gridCopy(static_cast<char*>(bufs.p[dst]) + b * 16, static_cast<const char*>(bufs.p[root]) + b * 16,
                 (en - b) * 16, vec, tid, nthreads);
      }
      // Unaligned tail goes directly.
      for (size_t i = units * 16 + tid; i < bytes; i += nthreads) {
        const char c = static_cast<const char*>(bufs.p[root])[i];
        for (int r = 1; r < P; r++) static_cast<char*>(bufs.p[(root + r) % P])[i] = c;
      }
    }
    if (!blockBarrier(a, e + 2)) {
      retire(a, used, 0);
      return;
    }
    // Every rank (the root too: nobody else holds its slice) now pushes the slice it
    // owns to all ranks that still miss it, i.e. everyone but itself and the root.
    {
      size_t b, en;
      shareOfB(units, P, a.rank, b, en);
      const char* src = static_cast<const char*>(bufs.p[a.rank]) + b * 16;
      const size_t nvec = vec ? (en - b) : 0;
      for (size_t v = tid; v < nvec; v += nthreads) {
        const Pack16 p = ld128_stream(src + v * 16);
        for (int i = 1; i < P; i++) {
          const int dst = (a.rank + i) % P;
          if (dst != root) st128_stream(static_cast<char*>(bufs.p[dst]) + b * 16 + v * 16, p);
        }
      }
      for (size_t i = nvec * 16 + tid; i < (en - b) * 16; i += nthreads) {
        const char c = src[i];
        for (int r = 1; r < P; r++) {
          const int dst = (a.rank + r) % P;
          if (dst != root) (static_cast<char*>(bufs.p[dst]) + b * 16)[i] = c;
        }
      }
    }
  }
  blockBarrier(a, e + used);
  retire(a, used, 0);
}

void launchBroadcast(const CommArgs& a, const PeerPtrs& bufs, void* mc, size_t bytes, int root, int mode, bool vec,
                     int blocks, int tile, cudaStream_t stream) {
  broadcastKernel<<<blocks, kThreads, 0, stream>>>(a, bufs, static_cast<char*>(mc), bytes, root, mode, vec,
                                                   tile > 0 ? tile : 1024);
}

// ---- allgather(v) / gather(v): push my block into peers' outputs ---------------------------
// Rank r's input block (inBytes[r] bytes at `in`) lands at outOff[r] in the output
// of every rank in [dstBegin, dstEnd) — all ranks for allgather, just the root for
// gather. Outputs are peer-mapped; the input is only read locally.
struct VArgs {
  size_t off[kMaxRanks];
  size_t len[kMaxRanks];
};

__global__ void __launch_bounds__(kThreads, 2)
gatherPushKernel(CommArgs a, const char* __restrict__ in, PeerPtrs outs, char* mcOut, VArgs va, int onlyDst,
                 bool vec) {
  const uint32_t e = loadEpoch(a);
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = a.nranks;
  if (!blockBarrier<false>(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  const size_t off = va.off[a.rank];
  const size_t len = va.len[a.rank];
  const bool v16 = vec && off % 16 == 0;
  const size_t nvec = v16 ? len / 16 : 0;
  if (onlyDst >= 0) {
    gridCopy(static_cast<char*>(outs.p[onlyDst]) + off, in, len, v16, tid, nthreads);
  } else if (mcOut != nullptr && v16) {
    for (size_t v = tid; v < nvec; v += nthreads) multimemSt128(mcOut + off + v * 16, ld128_stream(in + v * 16));
    for (size_t i = nvec * 16 + tid; i < len; i += nthreads) {
      const char c = in[i];
      for (int r = 0; r < P; r++) (static_cast<char*>(outs.p[r]) + off)[i] = c;
    }
  } else {
    constexpr int U = 4;
    for (size_t v0 = tid; v0 < nvec; v0 += nthreads * U) {
      Pack16 p[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t v = v0 + u * nthreads;
        if (v < nvec) p[u] = ld128_stream(in + v * 16);
      }
      for (int i = 0; i < P; i++) {
        char* dst = static_cast<char*>(outs.p[(a.rank + i) % P]) + off;
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t v = v0 + u * nthreads;
          if (v < nvec) st128_stream(dst + v * 16, p[u]);
        }
      }
    }
    for (size_t i = nvec * 16 + tid; i < len; i += nthreads) {
      const char c = in[i];
      for (int r = 0; r < P; r++) (static_cast<char*>(outs.p[r]) + off)[i] = c;
    }
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

void launchGatherPush(const CommArgs& a, const void* in, const PeerPtrs& outs, void* mcOut, const size_t* offs,
                      const size_t* lens, int onlyDst, bool vec, int blocks, cudaStream_t stream) {
  VArgs va;
  for (int i = 0; i < kMaxRanks; i++) {
    va.off[i] = i < a.nranks ? offs[i] : 0;
    va.len[i] = i < a.nranks ? lens[i] : 0;
  }
  gatherPushKernel<<<blocks, kThreads, 0, stream>>>(a, static_cast<const char*>(in), outs, static_cast<char*>(mcOut),
                                                    va, onlyDst, vec);
}

// ---- alltoall(v) / scatter: push chunk j of my input into slot (me) of rank j's output -------
// sendOff/sendLen index my input per destination; recvOff[r] (same on all ranks by
// symmetry of the exchange tables) is where MY chunk lands in rank r's output.
__global__ void __launch_bounds__(kThreads)
alltoallPushKernel(CommArgs a, const char* __restrict__ in, PeerPtrs outs, VArgs send, VArgs dstOff, VArgs myRecv,
                   VArgs blk, bool exchange, int onlySrc, bool vec) {
  const uint32_t e = loadEpoch(a);
  const int P = a.nranks;
  // v-variant: publish where I expect each source's chunk; peers read it after the
  // barrier (every CTA writes the same values, so no cross-CTA ordering is needed).
  if (exchange && threadIdx.x < P) a.self->xchg[threadIdx.x] = myRecv.off[threadIdx.x];
  if (!blockBarrier(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  if (onlySrc < 0 || onlySrc == a.rank) {
    // CTAs are dealt to destinations in proportion to the bytes each one gets (the host
    // fills blk.off = first CTA, blk.len = CTA count per destination), so every link is
    // busy at once and uneven (v-variant) splits stay balanced. With fewer CTAs than
    // destinations every CTA walks all destinations.
    const bool partitioned = blk.len[0] + blk.off[P - 1] > 0 && static_cast<size_t>(gridDim.x) >= static_cast<size_t>(P);
    for (int i = 0; i < P; i++) {
      const int dst = (a.rank + i) % P;
      size_t tid, nthreads;
      if (partitioned) {
        const size_t b0 = blk.off[dst], nb = blk.len[dst];
        if (blockIdx.x < b0 || blockIdx.x >= b0 + nb) continue;
        tid = (blockIdx.x - b0) * blockDim.x + threadIdx.x;
        nthreads = nb * blockDim.x;
      } else {
        tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
        nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      }
      const size_t so = send.off[dst], sl = send.len[dst];
      const size_t dofs = exchange ? static_cast<size_t>(*reinterpret_cast<volatile unsigned long long*>(
                                         &a.sig[dst]->xchg[a.rank]))
                                   : dstOff.off[dst];
      gridCopy(static_cast<char*>(outs.p[dst]) + dofs, in + so, sl, vec, tid, nthreads);
    }
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

void launchAlltoallPush(const CommArgs& a, const void* in, const PeerPtrs& outs, const size_t* sendOff,
                        const size_t* sendLen, const size_t* dstOff, const size_t* recvOffTable, int onlySrc,
                        bool vec, int blocks, cudaStream_t stream) {
  VArgs s, d, rcv;
  for (int i = 0; i < kMaxRanks; i++) {
    s.off[i] = i < a.nranks ? sendOff[i] : 0;
    s.len[i] = i < a.nranks ? sendLen[i] : 0;
    d.off[i] = i < a.nranks ? dstOff[i] : 0;
    d.len[i] = 0;
    rcv.off[i] = (recvOffTable != nullptr && i < a.nranks) ? recvOffTable[i] : 0;
    rcv.len[i] = 0;
  }
  // CTA ranges per destination, proportional to payload (at least one each).
  VArgs blk;
  for (int i = 0; i < kMaxRanks; i++) blk.off[i] = blk.len[i] = 0;
  if (blocks >= a.nranks) {
    size_t total = 0;
    for (int i = 0; i < a.nranks; i++) total += s.len[i];
    size_t used = 0;
    int spare = blocks - a.nranks;
    for (int i = 0; i < a.nranks; i++) {
      size_t extra = total > 0 ? static_cast<size_t>(spare) * s.len[i] / total : 0;
      blk.off[i] = used;
      blk.len[i] = 1 + extra;
      used += blk.len[i];
    }
  }
  alltoallPushKernel<<<blocks, kThreads, 0, stream>>>(a, static_cast<const char*>(in), outs, s, d, rcv, blk,
                                                      recvOffTable != nullptr, onlySrc, vec);
}

// ---- device-split all-to-all-v (expert-parallel dispatch / combine) ----------------------------
// Splits are device arrays of row counts; nothing about them passes through the host. P ranks,
// E local experts per rank, K = P·E chunks per rank. Count matrix M[s][k] = entry k of rank s's
// in_splits, read after the first barrier from column s of the a2aCount table of my own pad.
//   forward: k = j·E + e = rows of rank s for expert e of rank j; input packed in k order; on
//            rank j expert e's segment starts at a multiple of `align` rows and holds the rows of
//            sources 0..P-1 one after the other.
//   inverse: k = e·P + s = rows of my expert e that go back to rank s, read at in_offsets[k]; on
//            rank s they land packed in (holder j, e) order: where s's forward input rows were.
// A destination whose rows exceed the capacity it published receives nothing; invalid input
// anywhere (negative or oversized split, offsets out of range, headers that differ) moves
// nothing anywhere. Both are reported to the host of every rank through InputStatus.
namespace {

constexpr uint32_t kA2aBad = 0xffffffffu;  // a count that is not a valid row count

// Spin until the grid-barrier generation moves past `g`, bounded like every other device-side
// wait: 0 when it moved, kAbortTimeout / kAbortPeer when the wait was abandoned.
static __device__ __noinline__ uint32_t waitGenSlow(const volatile uint32_t* gen, uint32_t g, uint32_t* abortWord,
                                                    unsigned long long timeoutNs) {
  const unsigned long long t0 = globalTimerNs();
  uint32_t polls = 0;
  while (*gen == g) {
    if ((++polls & 127u) == 0u) {
      if (ld_relaxed_sys(abortWord) != 0u) return kAbortPeer;
      if (timeoutNs != 0ull && globalTimerNs() - t0 > timeoutNs) {
        atomicCAS(abortWord, 0u, static_cast<uint32_t>(kAbortTimeout));
        return kAbortTimeout;
      }
    }
  }
  return 0u;
}

// Grid barrier among the CTAs of THIS launch on this rank. It relies on every CTA being resident
// (the grid is capped by coResidentBlocks); should that fail, e.g. because another process holds
// SMs, the wait gives up after the context timeout like a barrier does, raises the abort word and
// returns false. Every CTA still counts its arrival, so the last one to arrive resets the counter
// and the next launch starts clean. Everything a CTA wrote before, at system scope, is visible to
// every CTA after it, and is covered by their later release stores.
__device__ __forceinline__ bool localGridSync(const CommArgs& a) {
  SignalPad* me = a.self;
  __syncthreads();
  int ok = 1;
  if (threadIdx.x == 0) {
    volatile uint32_t* gen = &me->a2aGen;
    const uint32_t g = *gen;
    __threadfence_system();
    if (atomicAdd(&me->a2aArrive, 1u) == gridDim.x - 1) {
      atomicExch(&me->a2aArrive, 0u);
      __threadfence();
      atomicAdd(&me->a2aGen, 1u);
    } else if (*gen == g) {
      const uint32_t rc = waitGenSlow(gen, g, &me->abort, a.timeoutNs);
      if (rc != 0u) {
        reportAbort(a, rc, a.rank);
        ok = 0;
      }
    }
    __threadfence();
  }
  return __syncthreads_and(ok) != 0;
}

// Exclusive prefix sum over the CTA (one value per thread); `total` gets the sum.
__device__ __forceinline__ unsigned long long blockExclusiveScan(unsigned long long v, unsigned long long* warpSums,
                                                                 unsigned long long& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warpSums[w] = x;
  __syncthreads();
  if (w == 0) {
    unsigned long long s = lane < nw ? warpSums[lane] : 0ull;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warpSums[lane] = s;
  }
  __syncthreads();
  total = warpSums[nw - 1];
  const unsigned long long r = x - v + (w > 0 ? warpSums[w - 1] : 0ull);
  __syncthreads();
  return r;
}

__device__ __forceinline__ uint32_t ldPad(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }

// Before barrier 1: my header and my P·E row counts (kA2aBad for one that is not a valid row count)
// into column `me` of every rank's a2aHdr / a2aCount, spread over the grid.
__device__ __forceinline__ void a2aPublish(const CommArgs& a, const long long* inSplits, int K, unsigned long long rb,
                                           int E, int align, uint32_t direction, uint32_t capRows, bool localBad) {
  const int P = a.nranks, me = a.rank, t = threadIdx.x;
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = gtid; i < static_cast<size_t>(P) * K; i += gthreads) {
    const int peer = static_cast<int>(i / K), k = static_cast<int>(i % K);
    const long long x = inSplits[k];
    a.sig[peer]->a2aCount[k][me] = (x < 0 || x > 0x7fffffffll) ? kA2aBad : static_cast<uint32_t>(x);
  }
  if (blockIdx.x == 0 && t < P) {
    uint32_t* h = &a.sig[t]->a2aHdr[0][me];
    const uint32_t hdr[kA2aHdrWords] = {static_cast<uint32_t>(rb), static_cast<uint32_t>(E), static_cast<uint32_t>(align),
                                        direction, capRows, localBad ? 1u : 0u};
#pragma unroll
    for (int w = 0; w < kA2aHdrWords; w++) h[w * kMaxRanks] = hdr[w];
  }
}

// After barrier 1: whether any rank's header differs from mine or reports bad input of its own,
// or any count is not a valid row count. sCap[s] gets rank s's capacity.
__device__ __forceinline__ bool a2aHeadersBad(const SignalPad* pad, int P, int K, unsigned long long rb, int E, int align,
                                              uint32_t direction, unsigned long long* sCap) {
  const int t = threadIdx.x;
  bool b = false;
  if (t < P) {
    const uint32_t want[4] = {static_cast<uint32_t>(rb), static_cast<uint32_t>(E), static_cast<uint32_t>(align), direction};
#pragma unroll
    for (int w = 0; w < 4; w++) b = b || ldPad(&pad->a2aHdr[w][t]) != want[w];
    b = b || ldPad(&pad->a2aHdr[5][t]) != 0u;
    sCap[t] = ldPad(&pad->a2aHdr[4][t]);
  }
  for (int i = t; i < P * K; i += blockDim.x) b = b || ldPad(&pad->a2aCount[i % K][i / K]) == kA2aBad;
  return __syncthreads_or(b) != 0;
}

// The forward layout from the count matrix. Chunk k = j·E + e of my input lands on rank j at row
// sDst[k] + sAux[k]: sDst[k] = rows of sources before me in that segment, sAux[k] = where expert e's
// segment starts on j (a multiple of `align`). sNeed[j] = rows rank j needs, up to the end of its
// last segment.
__device__ __forceinline__ void a2aForwardLayout(const SignalPad* pad, int P, int E, int K, int me, int align,
                                                 unsigned long long* sDst, unsigned long long* sAux,
                                                 unsigned long long* sNeed) {
  const int t = threadIdx.x;
  if (t < K) {
    unsigned long long before = 0, all = 0;
    for (int s = 0; s < P; s++) {
      const unsigned long long m = ldPad(&pad->a2aCount[t][s]);
      before += s < me ? m : 0ull;
      all += m;
    }
    sDst[t] = before;
    sAux[t] = all;
  }
  __syncthreads();
  if (t < P) {
    unsigned long long base = 0;
    for (int e = 0; e < E; e++) {
      const unsigned long long n = sAux[t * E + e];
      sAux[t * E + e] = base;
      base += n;
      if (e + 1 < E) base = (base + align - 1) / align * align;
    }
    sNeed[t] = base;
  }
  __syncthreads();
}

// Thread 0 of CTA 0, once every rank's input is known: raise the first error, if any, on the host.
// An overflow names the first rank whose layout needs more rows than it has.
__device__ __forceinline__ void a2aReport(InputStatus* status, bool invalid, int P, const unsigned long long* sNeed,
                                          const unsigned long long* sCap) {
  int over = -1;
  if (!invalid) {
    for (int j = P - 1; j >= 0; j--) over = sNeed[j] > sCap[j] ? j : over;
  }
  volatile InputStatus* st = status;
  if (st != nullptr && (invalid || over >= 0) && st->code == kInputOk) {
    st->rank = over >= 0 ? static_cast<uint32_t>(over) : 0u;
    st->need = over >= 0 ? sNeed[over] : 0ull;
    st->avail = over >= 0 ? sCap[over] : 0ull;
    __threadfence_system();
    st->code = invalid ? kInputInvalid : kInputOverflow;
  }
}

}  // namespace

struct A2aDevArgs {
  const char* in;
  unsigned long long inRows;
  unsigned long long rowBytes;
  const long long* inSplits;
  const long long* inOffsets;  // inverse only
  long long* outSplits;        // forward only, may be null
  long long* outOffsets;
  char* stagedOut;             // plain output: copied from my staging after barrier 2; null = zero copy
  uint32_t capRows;
  int experts;
  int align;
  int inverse;
  InputStatus* status;  // host-mapped
};

// The quantising dispatch (kQuant): bf16 rows of H elements in, e4m3 codes (rowBytes = H) and
// one fp32 scale per 128-element block out. The scales of rank j go to `scales.p[j]`, row-major
// (rows, H / 128), or, staged, into j's staging area right after its `capRows` rows of codes.
// Its own type, so that the copying form keeps its parameter block.
template <bool kQuant>
struct A2aDevKernelArgs : A2aDevArgs {};
template <>
struct A2aDevKernelArgs<true> : A2aDevArgs {
  PeerPtrs scales;     // zero copy: every rank's out_scales
  float* stagedScales; // plain output: copied from my staging after barrier 2; null = zero copy
};

constexpr int kQuantUnroll = 4;      // blocks in flight per half-warp
constexpr float kE4m3Max = 448.0f;
constexpr float kQuantMinAmax = 1e-4f;

// Header word 3: bit 0 = inverse, bit 1 = quantising. Ranks that disagree on either read the
// call as invalid, like differing row sizes.
template <bool kQuant>
__device__ __forceinline__ uint32_t a2aDirection(int inverse) {
  return static_cast<uint32_t>(inverse) | (kQuant ? 2u : 0u);
}

// Chunk of `nblk` blocks: bf16 at `in`, codes to `codes`, scales to `scales`. A half-warp owns a
// block: each lane loads 8 elements (16 bytes), the block amax takes 4 shuffles within the 16
// lanes, each lane stores 8 codes (8 bytes), lane 0 of the half stores the scale. The loop is
// warp-uniform so the shuffles run with a full mask; lanes past the end take part with zeros.
// `tid` / `nthreads` are multiples of 32 apart from the lane, like every caller of gridCopy.
// Numerics: amax = max(max |x|, 1e-4f); code = e4m3(x * (448 * (1 / amax))); scale = amax / 448,
// each step a correctly rounded fp32 operation (no contraction, no approximate division). The
// multiplier is a rounded reciprocal times 448, not a rounded 448 / amax: that is what torch
// evaluates for `448.0 / amax` (a scalar over a tensor), so torch code reproduces every byte.
// One block in a half-warp: `v` is this lane's 8 bf16 elements; returns its 8 codes and sets
// `amax` (the scale is amax / 448). Every lane of the warp must call it: the amax shuffles run
// with a full mask and stay within each half.
__device__ __forceinline__ uint2 quantBlock(const uint4& v, float& amax) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  float f[8];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
  amax = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(f[i]));
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  amax = fmaxf(amax, kQuantMinAmax);
  const float s = __fmul_rn(__frcp_rn(amax), kE4m3Max);
  uint32_t c[4];
#pragma unroll
  for (int i = 0; i < 4; i++) c[i] = float2ToFp8x2<__nv_fp8_e4m3>(__fmul_rn(f[2 * i], s), __fmul_rn(f[2 * i + 1], s));
  return make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
}

__device__ __forceinline__ void quantCopy(char* codes, float* scales, const char* in, unsigned long long nblk,
                                          size_t tid, size_t nthreads) {
  const int lane = static_cast<int>(tid & 31), half = lane >> 4, hl = lane & 15;
  const unsigned long long nwarps = nthreads / 32, warp = tid / 32;
  for (unsigned long long base = warp * (2 * kQuantUnroll); base < nblk; base += nwarps * (2 * kQuantUnroll)) {
    uint4 v[kQuantUnroll];
#pragma unroll
    for (int u = 0; u < kQuantUnroll; u++) {
      const unsigned long long blk = base + 2 * u + half;
      v[u] = blk < nblk ? *reinterpret_cast<const uint4*>(in + blk * (2 * kFp8Block) + hl * 16)
                        : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int u = 0; u < kQuantUnroll; u++) {
      const unsigned long long blk = base + 2 * u + half;
      float amax;
      const uint2 c = quantBlock(v[u], amax);
      if (blk < nblk) {
        *reinterpret_cast<uint2*>(codes + blk * kFp8Block + hl * 8) = c;
        if (hl == 0) scales[blk] = __fdiv_rn(amax, kE4m3Max);
      }
    }
  }
}

// Forward form, after a2aForwardLayout: my receive segment t = e·P + s starts at row sRcv[t] and
// holds sRcvCnt[t] rows.
__device__ __forceinline__ void a2aRecvSegments(const SignalPad* pad, int P, int E, int K, int me,
                                                const unsigned long long* sAux, unsigned long long* sRcv,
                                                uint32_t* sRcvCnt) {
  const int t = threadIdx.x;
  if (t < K) {
    const int e = t / P, s = t % P;
    unsigned long long off = sAux[me * E + e];
    for (int s2 = 0; s2 < s; s2++) off += ldPad(&pad->a2aCount[me * E + e][s2]);
    sRcv[t] = off;
    sRcvCnt[t] = ldPad(&pad->a2aCount[me * E + e][s]);
  }
}

// Forward form, plain output, once every CTA of every peer has pushed: my receive segments from my
// staging area to `out`, segment by segment, so that alignment gaps of `out` stay untouched. The
// quantising form's scales follow my capRows rows of codes in the staging area.
template <bool kQuant>
__device__ __forceinline__ void a2aCopyOutSegments(char* out, float* outScales, const char* stage,
                                                   const unsigned long long* sRcv, const uint32_t* sRcvCnt, int K,
                                                   unsigned long long rb, const unsigned long long& capRows /* in shared memory */, size_t tid,
                                                   size_t nthreads) {
  for (int k = 0; k < K; k++) {
    const unsigned long long n = sRcvCnt[k];
    if (n > 0) gridCopy(out + sRcv[k] * rb, stage + sRcv[k] * rb, n * rb, true, tid, nthreads);
    if constexpr (kQuant) {
      const unsigned long long sb = rb / kFp8Block * sizeof(float);  // scale bytes per row
      if (n > 0) {
        gridCopy(reinterpret_cast<char*>(outScales) + sRcv[k] * sb, stage + capRows * rb + sRcv[k] * sb, n * sb, true,
                 tid, nthreads);
      }
    }
  }
}

template <bool kQuant>
__global__ void __launch_bounds__(kThreads)
alltoallvDevKernel(CommArgs a, PeerPtrs outs, A2aDevKernelArgs<kQuant> d) {
  constexpr int kMaxK = kMaxRanks * kMaxA2aExperts;
  __shared__ unsigned long long sSrc[kMaxK];  // my chunk k: first input row
  __shared__ unsigned long long sDst[kMaxK];  //             first row in its destination's output
  __shared__ unsigned long long sAux[kMaxK];  // forward: column sums, then expert bases; inverse: R[j][s]
  __shared__ unsigned long long sRcv[kMaxK];  // forward: first row of my receive segment e·P+s
  __shared__ uint32_t sRcvCnt[kMaxK];         //          and its rows
  __shared__ uint32_t sCnt[kMaxK];            // my chunk k: rows
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks], sBytes[kMaxRanks];
  __shared__ unsigned long long sBlkOff[kMaxRanks], sBlkLen[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;

  // ---- my own splits: validate, and where each chunk starts in my input ----
  long long v = 0, o = 0;
  bool bad = false;
  if (t < K) {
    v = d.inSplits[t];
    bad = v < 0 || v > 0x7fffffffll;
    if (d.inverse) {
      o = d.inOffsets[t];
      bad = bad || o < 0 || static_cast<unsigned long long>(o) > d.inRows ||
            (!bad && static_cast<unsigned long long>(v) > d.inRows - static_cast<unsigned long long>(o));
    }
  }
  const unsigned long long c = bad ? 0ull : static_cast<unsigned long long>(v);
  unsigned long long inTotal;
  const unsigned long long prefix = blockExclusiveScan(t < K ? c : 0ull, sWarp, inTotal);
  if (t < K) {
    sCnt[t] = static_cast<uint32_t>(c);
    sSrc[t] = d.inverse ? static_cast<unsigned long long>(o) : prefix;
  }
  const bool localBad = __syncthreads_or(bad || (!d.inverse && inTotal > d.inRows)) != 0;

  // ---- publish: header + counts into column `me` of every rank's tables, spread over the grid ----
  a2aPublish(a, d.inSplits, K, rb, E, d.align, a2aDirection<kQuant>(d.inverse), d.capRows, localBad);
  // CTA b's release at the barrier must cover what the other CTAs published.
  const bool ok1 = localGridSync(a) && blockBarrier(a, ep + 1);

  // ---- the count matrix: validity, capacities, every offset ----
  const SignalPad* pad = a.self;
  bool invalid = false;
  if (ok1) invalid = a2aHeadersBad(pad, P, K, rb, E, d.align, a2aDirection<kQuant>(d.inverse), sCap);
  if (ok1 && !invalid) {
    if (!d.inverse) {
      a2aForwardLayout(pad, P, E, K, me, d.align, sDst, sAux, sNeed);
      if (t < K) sDst[t] += sAux[t];
      a2aRecvSegments(pad, P, E, K, me, sAux, sRcv, sRcvCnt);
    } else {
      // R[j][s] = rows holder j returns to rank s.
      for (int i = t; i < P * P; i += blockDim.x) {
        const int j = i / P, s = i % P;
        unsigned long long r = 0;
        for (int e = 0; e < E; e++) r += ldPad(&pad->a2aCount[e * P + s][j]);
        sAux[i] = r;
      }
      __syncthreads();
      if (t < P) {
        unsigned long long need = 0, base = 0;
        for (int j = 0; j < P; j++) {
          need += sAux[j * P + t];
          base += j < me ? sAux[j * P + t] : 0ull;
        }
        sNeed[t] = need;
        for (int e = 0; e < E; e++) {
          sDst[e * P + t] = base;
          base += sCnt[e * P + t];
        }
      }
    }
    __syncthreads();
    if (t < P) {
      unsigned long long rows = 0;
      for (int i = 0; i < E; i++) rows += sCnt[d.inverse ? i * P + t : t * E + i];
      sBytes[t] = sNeed[t] > sCap[t] ? 0ull : rows * rb;  // an overflowing destination gets nothing
    }
    __syncthreads();
    if (t == 0) {
      // CTAs dealt to destinations in proportion to their bytes, at least one each (as launchAlltoallPush).
      // The share is computed in double (spare x bytes may not fit 64 bits) and the running total
      // is clamped, so rounding can never deal out more CTAs than the grid has.
      unsigned long long total = 0, used = 0, extraUsed = 0;
      for (int j = 0; j < P; j++) total += sBytes[j];
      const unsigned long long spare = gridDim.x > static_cast<unsigned>(P) ? gridDim.x - P : 0u;
      for (int j = 0; j < P; j++) {
        unsigned long long extra =
            total > 0 ? static_cast<unsigned long long>(static_cast<double>(spare) * static_cast<double>(sBytes[j]) /
                                                        static_cast<double>(total))
                      : 0ull;
        extra = extra < spare - extraUsed ? extra : spare - extraUsed;
        extraUsed += extra;
        sBlkOff[j] = used;
        sBlkLen[j] = 1 + extra;
        used += sBlkLen[j];
      }
    }
    __syncthreads();
  }

  // ---- report, receive metadata, payload ----
  if (ok1 && blockIdx.x == 0) {
    if (t == 0) a2aReport(d.status, invalid, P, sNeed, sCap);
    if (!invalid && !d.inverse && d.outSplits != nullptr && t < K) {
      d.outSplits[t] = sRcvCnt[t];
      d.outOffsets[t] = static_cast<long long>(sRcv[t]);
    }
  }
  if (ok1 && !invalid) {
    const bool partitioned = gridDim.x >= static_cast<unsigned>(P);
    for (int i = 0; i < P; i++) {
      const int dst = (me + i) % P;
      if (sBytes[dst] == 0) continue;
      size_t tid, nthreads;
      if (partitioned) {
        const size_t b0 = sBlkOff[dst], nb = sBlkLen[dst];
        if (blockIdx.x < b0 || blockIdx.x >= b0 + nb) continue;
        tid = (blockIdx.x - b0) * blockDim.x + t;
        nthreads = nb * blockDim.x;
      } else {
        tid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
        nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      }
      for (int x = 0; x < E; x++) {
        const int k = d.inverse ? x * P + dst : dst * E + x;
        if (sCnt[k] == 0) continue;
        if constexpr (kQuant) {
          // Input rows are 2·rb bytes (bf16); a row is rb / 128 blocks.
          const unsigned long long bpr = rb / kFp8Block;
          char* codes = static_cast<char*>(outs.p[dst]);
          float* scales = d.stagedScales != nullptr ? reinterpret_cast<float*>(codes + sCap[dst] * rb)
                                                    : static_cast<float*>(d.scales.p[dst]);
          quantCopy(codes + sDst[k] * rb, scales + sDst[k] * bpr, d.in + sSrc[k] * rb * 2, sCnt[k] * bpr, tid, nthreads);
        } else {
          gridCopy(static_cast<char*>(outs.p[dst]) + sDst[k] * rb, d.in + sSrc[k] * rb, sCnt[k] * rb, true, tid, nthreads);
        }
      }
    }
  }
  blockBarrier(a, ep + 2);
  // NO pad table reads from here on. Once every CTA of every rank has arrived at barrier 2 a peer
  // may finish and start its next launch, which rewrites its column of my tables before its own
  // barrier 1 without waiting for anything. Everything below comes from shared memory.

  // ---- plain output: my staging -> out, once every CTA of every peer has pushed ----
  if (d.stagedOut != nullptr) {
    const bool synced = localGridSync(a);
    if (synced && ok1 && !invalid && sNeed[me] <= sCap[me] && ld_relaxed_sys(&a.self->abort) == 0u) {
      const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
      const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      const char* stage = static_cast<const char*>(outs.p[me]);
      if (d.inverse) {
        gridCopy(d.stagedOut, stage, sNeed[me] * rb, true, tid, nthreads);
      } else {
        float* stagedScales = nullptr;
        if constexpr (kQuant) stagedScales = d.stagedScales;
        a2aCopyOutSegments<kQuant>(d.stagedOut, stagedScales, stage, sRcv, sRcvCnt, K, rb, sCap[me], tid, nthreads);
      }
    }
  }
  retire(a, 2, 0);
}

void launchAlltoallvDev(const CommArgs& a, const PeerPtrs& outs, const void* in, size_t inRows, size_t rowBytes,
                        const long long* inSplits, const long long* inOffsets, long long* outSplits,
                        long long* outOffsets, void* stagedOut, uint32_t capRows, int experts, int align, bool inverse,
                        InputStatus* status, int blocks, cudaStream_t stream) {
  A2aDevKernelArgs<false> d;
  d.in = static_cast<const char*>(in);
  d.inRows = inRows;
  d.rowBytes = rowBytes;
  d.inSplits = inSplits;
  d.inOffsets = inOffsets;
  d.outSplits = outSplits;
  d.outOffsets = outOffsets;
  d.stagedOut = static_cast<char*>(stagedOut);
  d.capRows = capRows;
  d.experts = experts;
  d.align = align;
  d.inverse = inverse ? 1 : 0;
  d.status = status;
  alltoallvDevKernel<false><<<blocks, kThreads, 0, stream>>>(a, outs, d);
}

void launchAlltoallvDevFp8(const CommArgs& a, const PeerPtrs& outs, const PeerPtrs& scales, const void* in,
                           size_t inRows, size_t hidden, const long long* inSplits, long long* outSplits,
                           long long* outOffsets, void* stagedOut, float* stagedScales, uint32_t capRows, int experts,
                           int align, InputStatus* status, int blocks, cudaStream_t stream) {
  A2aDevKernelArgs<true> d;
  d.in = static_cast<const char*>(in);
  d.inRows = inRows;
  d.rowBytes = hidden;  // e4m3 codes: one byte per element
  d.inSplits = inSplits;
  d.inOffsets = nullptr;
  d.outSplits = outSplits;
  d.outOffsets = outOffsets;
  d.stagedOut = static_cast<char*>(stagedOut);
  d.capRows = capRows;
  d.experts = experts;
  d.align = align;
  d.inverse = 0;
  d.status = status;
  d.scales = scales;
  d.stagedScales = stagedScales;
  alltoallvDevKernel<true><<<blocks, kThreads, 0, stream>>>(a, outs, d);
}

// ---- top-k MoE combine: pull each token's expert rows and sum them with its gate weights ---------
// The mirror of the forward dispatch, run by the source. Chunk k = j·E + e of my dispatch input
// (splits[k] rows, starting at row sSrc[k]) lies on holder j from row sDst[k] on, sDst as the
// dispatch computes it from the same count matrix; so input row p of chunk k is holder row
// sDst[k] + (p - sSrc[k]). Each token's warp reads its k rows there and writes one row locally.
//   barrier 1  headers and counts published, with the dispatch's code
//   barrier 2  a plain expert_out copied into its holder's staging area; every rank's bad-pos word
//              published. The grid sync before it puts every local CTA's stores under CTA b's release:
//              the barrier pairs CTA b with CTA b only.
//   barrier 3  every rank has read its rows: holders may reuse expert_out and the staging area.
// Every path passes all three barriers, so ranks never wait for a different count.
struct A2aTopkArgs {
  const long long* splits;   // my dispatch in_splits, P·E entries in j·E + e order
  const long long* pos;      // (tokens, topk): row of my dispatch input, -1 = not sent
  const float* weights;      // (tokens, topk)
  char* out;                 // (tokens, rowBytes), written locally
  const char* stagedIn;      // plain expert_out: copied into my staging area (srcs.p[me]); null = zero copy
  unsigned long long tokens;
  unsigned long long rowBytes;
  uint32_t capRows;
  int topk;
  int experts;
  int align;
  InputStatus* status;  // host-mapped
};

// Header word 3 of the top-k combine: bit 2 marks the form, bit 3 a staged (plain) expert_out, so
// ranks that mix the form with the dispatch, or symmetric with plain expert_out, read it as invalid.
constexpr uint32_t kA2aTopkDir = 4u;
constexpr uint32_t kA2aTopkStaged = 8u;
constexpr int kTopkInFlight = 4;  // choices whose packs a lane loads before it adds them
constexpr int kTopkPacks = 2;     // packs of one row per lane per step

template <typename T>
__global__ void __launch_bounds__(kThreads)
moeCombineTopkKernel(CommArgs a, PeerPtrs srcs, A2aTopkArgs d) {
  using PT = PackTraits<T>;
  constexpr int kMaxK = kMaxRanks * kMaxA2aExperts;
  __shared__ unsigned long long sSrc[kMaxK];  // my chunk k: first row in my dispatch input
  __shared__ unsigned long long sDst[kMaxK];  //             first row on its holder
  __shared__ unsigned long long sAux[kMaxK];  // column sums, then expert bases
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks];
  __shared__ const char* sBase[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;
  const uint32_t dir = kA2aTopkDir | (d.stagedIn != nullptr ? kA2aTopkStaged : 0u);
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;

  // ---- 1. my splits, where each chunk starts in my input; publish; clear my bad-pos word ----
  const long long v = t < K ? d.splits[t] : 0ll;
  const bool bad = v < 0 || v > 0x7fffffffll;
  unsigned long long inRows;
  const unsigned long long prefix = blockExclusiveScan(bad ? 0ull : static_cast<unsigned long long>(v), sWarp, inRows);
  if (t < K) sSrc[t] = prefix;
  if (t < P) sBase[t] = static_cast<const char*>(srcs.p[t]);
  const bool localBad = __syncthreads_or(bad) != 0;
  a2aPublish(a, d.splits, K, rb, E, d.align, dir, d.capRows, localBad);
  if (blockIdx.x == 0 && t < P) a.sig[t]->a2aPosBad[me] = 0u;
  const bool ok1 = localGridSync(a) && blockBarrier(a, ep + 1);

  // ---- 2. the layout; stage a plain expert_out; check pos ----
  const SignalPad* pad = a.self;
  bool invalid = false, over = false;
  if (ok1) invalid = a2aHeadersBad(pad, P, K, rb, E, d.align, dir, sCap);
  if (ok1 && !invalid) {
    a2aForwardLayout(pad, P, E, K, me, d.align, sDst, sAux, sNeed);
    if (t < K) sDst[t] += sAux[t];
    over = __syncthreads_or(t < P && sNeed[t] > sCap[t]) != 0;
  }
  const bool go = ok1 && !invalid && !over;
  if (go && d.stagedIn != nullptr) gridCopy(const_cast<char*>(sBase[me]), d.stagedIn, sNeed[me] * rb, true, gtid, gthreads);
  if (go) {
    bool b = false;
    const unsigned long long n = d.tokens * static_cast<unsigned long long>(d.topk);
    for (size_t i = gtid; i < n; i += gthreads) {
      const long long p = d.pos[i];
      b = b || p < -1 || (p >= 0 && static_cast<unsigned long long>(p) >= inRows);
    }
    if (__syncthreads_or(b) != 0 && t < P) a.sig[t]->a2aPosBad[me] = 1u;
  }
  const bool ok2 = localGridSync(a) && blockBarrier(a, ep + 2);

  // ---- 3. every rank's verdict; pull and reduce ----
  bool posBad = false;
  if (ok2 && go) posBad = __syncthreads_or(t < P && ldPad(&pad->a2aPosBad[t]) != 0u) != 0;
  if (ok1 && ok2 && blockIdx.x == 0 && t == 0) a2aReport(d.status, invalid || posBad, P, sNeed, sCap);
  if (ok2 && go && !posBad) {
    const int lane = t & 31, k = d.topk;
    const unsigned long long npk = rb / 16;
    for (unsigned long long tok = gtid / 32; tok < d.tokens; tok += gthreads / 32) {
      // Lane j < k: where choice j's row lies. The last chunk starting at or before p holds it
      // (an empty chunk starts where the next one does).
      const char* src = nullptr;
      float w = 0.0f;
      if (lane < k) {
        const long long p = d.pos[tok * k + lane];
        if (p >= 0) {
          int lo = 0, hi = K - 1;
          while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (sSrc[mid] <= static_cast<unsigned long long>(p)) lo = mid; else hi = mid - 1;
          }
          src = sBase[lo / E] + (sDst[lo] + (static_cast<unsigned long long>(p) - sSrc[lo])) * rb;
          w = d.weights[tok * k + lane];
        }
      }
      char* dst = d.out + tok * rb;
      // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
      for (unsigned long long v0 = lane; v0 - lane < npk; v0 += 32 * kTopkPacks) {
        typename PT::AccPack acc[kTopkPacks];
#pragma unroll
        for (int u = 0; u < kTopkPacks; u++) {
#pragma unroll
          for (int i = 0; i < PT::kElems; i++) acc[u].v[i] = 0.0f;
        }
        for (int j0 = 0; j0 < k; j0 += kTopkInFlight) {
          const char* s[kTopkInFlight];
          float ws[kTopkInFlight];
          Pack16 x[kTopkInFlight][kTopkPacks];
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
            s[c] = reinterpret_cast<const char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(src), (j0 + c) & 31));
            ws[c] = __shfl_sync(0xffffffffu, w, (j0 + c) & 31);
            if (j0 + c >= k) s[c] = nullptr;
#pragma unroll
            for (int u = 0; u < kTopkPacks; u++) {
              const unsigned long long pk = v0 + 32ull * u;
              if (s[c] != nullptr && pk < npk) x[c][u] = ld128_stream(s[c] + pk * 16);
            }
          }
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
            if (s[c] == nullptr) continue;
#pragma unroll
            for (int u = 0; u < kTopkPacks; u++) {
              const typename PT::AccPack xf = PT::widen(x[c][u]);
#pragma unroll
              for (int i = 0; i < PT::kElems; i++) acc[u].v[i] = __fadd_rn(acc[u].v[i], __fmul_rn(ws[c], xf.v[i]));
            }
          }
        }
#pragma unroll
        for (int u = 0; u < kTopkPacks; u++) {
          const unsigned long long pk = v0 + 32ull * u;
          if (pk < npk) st128(dst + pk * 16, PT::narrow(acc[u]));
        }
      }
    }
  }
  blockBarrier(a, ep + 3);
  // NO pad table or peer reads from here on: a peer that has passed barrier 3 may start its next
  // launch, which rewrites its columns of my tables and its staging area.
  retire(a, 3, 0);
}

namespace {
// The top-k combine instantiation for dt: float, bfloat16 or float16 rows (null for any other).
using TopkCombineFn = void (*)(CommArgs, PeerPtrs, A2aTopkArgs);
TopkCombineFn topkCombineFn(DataType dt) {
  switch (dt) {
    case DataType::FLOAT32: return moeCombineTopkKernel<float>;
    case DataType::BFLOAT16: return moeCombineTopkKernel<__nv_bfloat16>;
    case DataType::FLOAT16: return moeCombineTopkKernel<__half>;
    default: return nullptr;
  }
}
}  // namespace

void launchMoeCombineTopk(const CommArgs& a, const PeerPtrs& srcs, const void* stagedIn, void* out, size_t tokens,
                          int topk, const long long* pos, const float* weights, const long long* splits, size_t rowBytes,
                          DataType dt, uint32_t capRows, int experts, int align, InputStatus* status, int blocks,
                          cudaStream_t stream) {
  A2aTopkArgs d;
  d.splits = splits;
  d.pos = pos;
  d.weights = weights;
  d.out = static_cast<char*>(out);
  d.stagedIn = static_cast<const char*>(stagedIn);
  d.tokens = tokens;
  d.rowBytes = rowBytes;
  d.capRows = capRows;
  d.topk = topk;
  d.experts = experts;
  d.align = align;
  d.status = status;
  topkCombineFn(dt)<<<blocks, kThreads, 0, stream>>>(a, srcs, d);
}

// ---- top-k MoE dispatch: route each token from its gate indices and push its row to every choice ----
// The forward dispatch of route(x, topk_idx) without its T·k-row copy: each token's row is read
// once (and quantised once) and stored to each of its k destination rows. The layout, splits and
// pos are those of route() + the forward alltoallvDevKernel, byte for byte.
//   route (before barrier 1, local): group g = topk_idx entry, in 0..P·E-1 (anything else is not
//     routed). CTA b owns a contiguous slice of tokens. It counts every choice of every token
//     (the totals, which every CTA needs for pos) and those before its slice (its base), then ranks
//     its slice's choices in (token, choice) order: within a warp by __match_any_sync, across the
//     warps of a round in warp order through shared running counts. No atomic decides a place.
//     pos = (rows of groups before g) + (choices of g before this one); CTA 0 writes splits.
//   publish / barrier 1 / layout: the dispatch's helpers; header word 3 carries bit 4 (this form),
//     bit 1 (quantising) and bit 3 (staged output), so ranks that mix forms read it as invalid.
//   push: one warp per token of my slice; a lane per choice finds its destination row
//     sDst[g] + (pos - sSrc[g]) on rank g / E, then the warp reads each 16-byte pack (or, quantising,
//     each 128-element block) once and stores it to every destination that does not overflow.
//   barrier 2, staged copy-out and retire as in the dispatch.
struct MoeDispatchTopkArgs {
  const char* x;              // (tokens, rowBytes); quantising: bf16 (tokens, rowBytes) elements
  const long long* idx;       // (tokens, topk) group per choice
  long long* splits;          // (P·E) out: routed choices per group
  long long* pos;             // (tokens, topk) out: row of route()'s rows, -1 = not routed
  long long* outSplits;
  long long* outOffsets;
  char* stagedOut;            // plain output: copied from my staging after barrier 2; null = zero copy
  unsigned long long tokens;
  unsigned long long rowBytes;  // of an output row (quantising: H codes)
  uint32_t capRows;
  int topk;
  int experts;
  int align;
  InputStatus* status;  // host-mapped
};
template <bool kQuant>
struct MoeDispatchTopkKernelArgs : MoeDispatchTopkArgs {};
template <>
struct MoeDispatchTopkKernelArgs<true> : MoeDispatchTopkArgs {
  PeerPtrs scales;      // zero copy: every rank's out_scales
  float* stagedScales;  // plain output: copied from my staging after barrier 2; null = zero copy
};

constexpr uint32_t kA2aTopkDispatchDir = 16u;  // header word 3, bit 4: the top-k dispatch
constexpr int kTopkPushUnroll = 4;             // packs of a row in flight per lane
static_assert(kThreads >= kMaxRanks * kMaxA2aExperts, "one scan slot per group");

__device__ __forceinline__ int topkGroup(long long v, int K) { return v >= 0 && v < K ? static_cast<int>(v) : K; }

template <bool kQuant>
__global__ void __launch_bounds__(kThreads)
moeDispatchTopkKernel(CommArgs a, PeerPtrs outs, MoeDispatchTopkKernelArgs<kQuant> d) {
  constexpr int kMaxK = kMaxRanks * kMaxA2aExperts;
  __shared__ unsigned long long sSrc[kMaxK];  // group g: first row of route()'s rows
  __shared__ unsigned long long sDst[kMaxK];  //          first row on rank g / E
  __shared__ unsigned long long sAux[kMaxK];  // my splits (published), then column sums / expert bases
  __shared__ unsigned long long sRcv[kMaxK];  // first row of my receive segment e·P+s
  __shared__ uint32_t sRcvCnt[kMaxK];         // and its rows
  __shared__ uint32_t sTot[kMaxK];            // group g: routed choices of all my tokens
  __shared__ uint32_t sRun[kMaxK];            //          of the tokens before my slice, then running
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = blockDim.x >> 5;
  const unsigned long long rb = d.rowBytes, k = static_cast<unsigned long long>(d.topk);
  const uint32_t dir = kA2aTopkDispatchDir | (kQuant ? 2u : 0u) | (d.stagedOut != nullptr ? kA2aTopkStaged : 0u);

  // ---- route: counts, then pos of my slice ----
  const unsigned long long n = d.tokens * k;
  const unsigned long long per = (d.tokens + gridDim.x - 1) / gridDim.x;
  const unsigned long long tok0 = min(d.tokens, blockIdx.x * per), tok1 = min(d.tokens, tok0 + per);
  const unsigned long long lo = tok0 * k, hi = tok1 * k;
  for (int g = t; g < K; g += blockDim.x) sTot[g] = sRun[g] = 0u;
  __syncthreads();
  for (unsigned long long b = static_cast<unsigned long long>(warp) * 32; b < n; b += blockDim.x) {
    const unsigned long long i = b + lane;
    const int g = i < n ? topkGroup(d.idx[i], K) : K;
    const bool before = i < lo;
    const unsigned m = __match_any_sync(0xffffffffu, 2 * g + (before ? 1 : 0));
    if (g < K && lane == __ffs(m) - 1) {
      atomicAdd(&sTot[g], static_cast<uint32_t>(__popc(m)));
      if (before) atomicAdd(&sRun[g], static_cast<uint32_t>(__popc(m)));
    }
  }
  __syncthreads();
  unsigned long long routed;
  const unsigned long long first = blockExclusiveScan(t < K ? sTot[t] : 0u, sWarp, routed);
  if (t < K) {
    sSrc[t] = first;
    sAux[t] = sTot[t];
    if (blockIdx.x == 0) d.splits[t] = sTot[t];
  }
  __syncthreads();
  for (unsigned long long b = lo; b < hi; b += blockDim.x) {
    const unsigned long long i = b + t;
    const int g = i < hi ? topkGroup(d.idx[i], K) : K;
    const unsigned m = __match_any_sync(0xffffffffu, g);
    const unsigned below = m & ((1u << lane) - 1u);
    long long p = -1;
    for (int w = 0; w < nw; w++) {
      if (warp == w && g < K) {
        const uint32_t r = sRun[g];
        __syncwarp(m);
        if (below == 0u) sRun[g] = r + static_cast<uint32_t>(__popc(m));
        p = static_cast<long long>(sSrc[g] + r + static_cast<uint32_t>(__popc(below)));
      }
      __syncthreads();
    }
    if (i < hi) d.pos[i] = p;
  }

  // ---- publish: header + my splits; the layout ----
  a2aPublish(a, reinterpret_cast<const long long*>(sAux), K, rb, E, d.align, dir, d.capRows, false);
  const bool ok1 = localGridSync(a) && blockBarrier(a, ep + 1);
  const SignalPad* pad = a.self;
  bool invalid = false;
  if (ok1) invalid = a2aHeadersBad(pad, P, K, rb, E, d.align, dir, sCap);
  if (ok1 && !invalid) {
    a2aForwardLayout(pad, P, E, K, me, d.align, sDst, sAux, sNeed);
    if (t < K) sDst[t] += sAux[t];
    a2aRecvSegments(pad, P, E, K, me, sAux, sRcv, sRcvCnt);
    __syncthreads();
  }
  if (ok1 && blockIdx.x == 0) {
    if (t == 0) a2aReport(d.status, invalid, P, sNeed, sCap);
    if (!invalid && t < K) {
      d.outSplits[t] = sRcvCnt[t];
      d.outOffsets[t] = static_cast<long long>(sRcv[t]);
    }
  }

  // ---- push: one warp per token of my slice ----
  if (ok1 && !invalid) {
    for (unsigned long long tok = tok0 + warp; tok < tok1; tok += nw) {
      // Lane c < k: where choice c's row goes; null when it is not routed or its rank overflows.
      char* dst = nullptr;
      float* dsc = nullptr;
      if (static_cast<unsigned long long>(lane) < k) {
        const unsigned long long i = tok * k + lane;
        const int g = topkGroup(d.idx[i], K);
        if (g < K && sNeed[g / E] <= sCap[g / E]) {
          const int j = g / E;
          const unsigned long long row = sDst[g] + (static_cast<unsigned long long>(d.pos[i]) - sSrc[g]);
          dst = static_cast<char*>(outs.p[j]) + row * rb;
          if constexpr (kQuant) {
            float* sc = d.stagedScales != nullptr ? reinterpret_cast<float*>(static_cast<char*>(outs.p[j]) + sCap[j] * rb)
                                                  : static_cast<float*>(d.scales.p[j]);
            dsc = sc + row * (rb / kFp8Block);
          }
        }
      }
      if constexpr (kQuant) {
        // Half-warps take 128-element blocks, as quantCopy: one amax and one set of codes per block.
        const int half = lane >> 4, hl = lane & 15;
        const unsigned long long nblk = rb / kFp8Block;
        const char* src = d.x + tok * rb * 2;
        for (unsigned long long b0 = 0; b0 < nblk; b0 += 2 * kQuantUnroll) {
          uint4 v[kQuantUnroll];
#pragma unroll
          for (int u = 0; u < kQuantUnroll; u++) {
            const unsigned long long blk = b0 + 2 * u + half;
            v[u] = blk < nblk ? *reinterpret_cast<const uint4*>(src + blk * (2 * kFp8Block) + hl * 16)
                              : make_uint4(0u, 0u, 0u, 0u);
          }
          uint2 c[kQuantUnroll];
          float amax[kQuantUnroll];
#pragma unroll
          for (int u = 0; u < kQuantUnroll; u++) c[u] = quantBlock(v[u], amax[u]);
          for (int ch = 0; ch < d.topk; ch++) {
            char* q = reinterpret_cast<char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dst), ch));
            float* qs = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dsc), ch));
            if (q == nullptr) continue;
#pragma unroll
            for (int u = 0; u < kQuantUnroll; u++) {
              const unsigned long long blk = b0 + 2 * u + half;
              if (blk < nblk) {
                *reinterpret_cast<uint2*>(q + blk * kFp8Block + hl * 8) = c[u];
                if (hl == 0) qs[blk] = __fdiv_rn(amax[u], kE4m3Max);
              }
            }
          }
        }
      } else {
        const unsigned long long npk = rb / 16;
        const char* src = d.x + tok * rb;
        // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
        for (unsigned long long v0 = lane; v0 - lane < npk; v0 += 32 * kTopkPushUnroll) {
          Pack16 x[kTopkPushUnroll];
#pragma unroll
          for (int u = 0; u < kTopkPushUnroll; u++) {
            const unsigned long long pk = v0 + 32ull * u;
            if (pk < npk) x[u] = ld128_stream(src + pk * 16);
          }
          for (int ch = 0; ch < d.topk; ch++) {
            char* q = reinterpret_cast<char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dst), ch));
            if (q == nullptr) continue;
#pragma unroll
            for (int u = 0; u < kTopkPushUnroll; u++) {
              const unsigned long long pk = v0 + 32ull * u;
              if (pk < npk) st128_stream(q + pk * 16, x[u]);
            }
          }
        }
      }
    }
  }
  blockBarrier(a, ep + 2);
  // NO pad table reads from here on (see alltoallvDevKernel).

  // ---- plain output: my staging -> out, once every CTA of every peer has pushed ----
  if (d.stagedOut != nullptr) {
    const bool synced = localGridSync(a);
    if (synced && ok1 && !invalid && sNeed[me] <= sCap[me] && ld_relaxed_sys(&a.self->abort) == 0u) {
      const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
      const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      float* stagedScales = nullptr;
      if constexpr (kQuant) stagedScales = d.stagedScales;
      a2aCopyOutSegments<kQuant>(d.stagedOut, stagedScales, static_cast<const char*>(outs.p[me]), sRcv, sRcvCnt, K,
                                 rb, sCap[me], tid, nthreads);
    }
  }
  retire(a, 2, 0);
}

namespace {
void fillDispatchTopk(MoeDispatchTopkArgs& d, const void* x, size_t tokens, int topk, const long long* idx,
                      long long* splits, long long* pos, long long* outSplits, long long* outOffsets, void* stagedOut,
                      size_t rowBytes, uint32_t capRows, int experts, int align, InputStatus* status) {
  d.x = static_cast<const char*>(x);
  d.idx = idx;
  d.splits = splits;
  d.pos = pos;
  d.outSplits = outSplits;
  d.outOffsets = outOffsets;
  d.stagedOut = static_cast<char*>(stagedOut);
  d.tokens = tokens;
  d.rowBytes = rowBytes;
  d.capRows = capRows;
  d.topk = topk;
  d.experts = experts;
  d.align = align;
  d.status = status;
}
}  // namespace

void launchMoeDispatchTopk(const CommArgs& a, const PeerPtrs& outs, const void* x, size_t tokens, int topk,
                           const long long* idx, long long* splits, long long* pos, long long* outSplits,
                           long long* outOffsets, void* stagedOut, size_t rowBytes, uint32_t capRows, int experts,
                           int align, InputStatus* status, int blocks, cudaStream_t stream) {
  MoeDispatchTopkKernelArgs<false> d;
  fillDispatchTopk(d, x, tokens, topk, idx, splits, pos, outSplits, outOffsets, stagedOut, rowBytes, capRows, experts,
                   align, status);
  moeDispatchTopkKernel<false><<<blocks, kThreads, 0, stream>>>(a, outs, d);
}

void launchMoeDispatchTopkFp8(const CommArgs& a, const PeerPtrs& outs, const PeerPtrs& scales, const void* x,
                              size_t tokens, int topk, const long long* idx, long long* splits, long long* pos,
                              long long* outSplits, long long* outOffsets, void* stagedOut, float* stagedScales,
                              size_t hidden, uint32_t capRows, int experts, int align, InputStatus* status, int blocks,
                              cudaStream_t stream) {
  MoeDispatchTopkKernelArgs<true> d;
  fillDispatchTopk(d, x, tokens, topk, idx, splits, pos, outSplits, outOffsets, stagedOut, hidden, capRows, experts,
                   align, status);
  d.scales = scales;
  d.stagedScales = stagedScales;
  moeDispatchTopkKernel<true><<<blocks, kThreads, 0, stream>>>(a, outs, d);
}

// ---- reduce_scatter / reduce: pull my slice from every peer's input, reduce, store -----------
// Inputs are peer-mapped. Rank r reduces elements [elemOff[r], elemOff[r]+elemLen[r])
// and writes them to `out` (local pointer; for reduce() it is the root's peer-mapped
// output at the same offset).
struct EArgs {
  size_t off[kMaxRanks];
  size_t len[kMaxRanks];
};

template <typename T, int NR, int UNROLL>
__global__ void __launch_bounds__(kThreads)
reducePullKernel(CommArgs a, PeerPtrs ins, char* mcIn, T* __restrict__ out, EArgs ea, DevOp op, float scale,
                 bool vec, bool useMc) {
  using PT = PackTraits<T>;
  const uint32_t e = loadEpoch(a);
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = NR > 0 ? NR : a.nranks;
  if (!blockBarrier<false>(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  const size_t off = ea.off[a.rank], len = ea.len[a.rank];
  const bool v16 = vec && (off * sizeof(T)) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
  const size_t nvec = v16 ? len / PT::kElems : 0;
  const size_t byteOff = off * sizeof(T);
  auto store = [&](size_t v, const Pack16& r) { st128(reinterpret_cast<char*>(out) + v * 16, r); };
  if (useMc && v16) {
    if constexpr (hasMultimem<T>()) reduceMultimem<T, 4>(mcIn + byteOff, tid, nvec, nthreads, scale, store);
  } else {
    constexpr int kSlots = NR > 0 ? NR : kMaxRanks;
    const char* peer[kSlots];
#pragma unroll
    for (int i = 0; i < kSlots; i++) {
      peer[i] = i < P ? static_cast<const char*>(ins.p[(a.rank + i) % P]) + byteOff : nullptr;
    }
    reducePeers<T, kSlots, UNROLL, 0>(P, tid, nvec, nthreads, op, scale, [&](int i) { return peer[i]; }, store);
  }
  using TA = TailAcc<T>;
  for (size_t i = nvec * PT::kElems + tid; i < len; i += nthreads) {
    typename TA::type acc = TA::load(static_cast<const T*>(ins.p[0])[off + i]);
    for (int r = 1; r < P; r++) acc = TA::combine(acc, TA::load(static_cast<const T*>(ins.p[r])[off + i]), op);
    if (scale != 1.0f) acc = TA::scale(acc, scale);
    out[i] = TA::store(acc);
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

namespace {
// The reduce-pull instantiation for (T, P).
template <typename T>
auto reducePullFn(int nranks) {
  if constexpr (isHotType<T>()) {
    if (nranks == 2) return reducePullKernel<T, 2, 4>;
    if (nranks == 4) return reducePullKernel<T, 4, 2>;
    if (nranks == 8) return reducePullKernel<T, 8, 2>;
  }
  return reducePullKernel<T, 0, 1>;
}
}  // namespace

void launchReducePull(const CommArgs& a, const PeerPtrs& ins, void* mcIn, void* out, const size_t* elemOff,
                      const size_t* elemLen, DataType dt, ReduceOp op, float scale, bool vec, bool useMc, int blocks,
                      cudaStream_t stream) {
  EArgs ea;
  for (int i = 0; i < kMaxRanks; i++) {
    ea.off[i] = i < a.nranks ? elemOff[i] : 0;
    ea.len[i] = i < a.nranks ? elemLen[i] : 0;
  }
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    reducePullFn<T>(a.nranks)<<<blocks, kThreads, 0, stream>>>(a, ins, static_cast<char*>(mcIn), static_cast<T*>(out),
                                                               ea, static_cast<DevOp>(op), scale, vec, useMc);
  });
}

// ---- small allgather / alltoall without a barrier: flag-in-data lines -------------------------
// Same protocol and pool region as llAllreduceKernel (every rank hears from every peer in a
// launch, which is what makes two parity halves sufficient). Payload unit: 8 bytes.
namespace {
__device__ __forceinline__ void load8(const char* p, size_t avail, bool aligned, uint32_t& d0, uint32_t& d1) {
  if (aligned && avail >= 8) {
    const uint2 v = *reinterpret_cast<const uint2*>(p);
    d0 = v.x;
    d1 = v.y;
    return;
  }
  unsigned long long w = 0;
  for (int k = 0; k < 8; k++) {
    if (static_cast<size_t>(k) < avail) w |= static_cast<unsigned long long>(static_cast<unsigned char>(p[k])) << (8 * k);
  }
  d0 = static_cast<uint32_t>(w);
  d1 = static_cast<uint32_t>(w >> 32);
}
__device__ __forceinline__ void store8(char* p, size_t avail, bool aligned, uint32_t d0, uint32_t d1) {
  if (aligned && avail >= 8) {
    *reinterpret_cast<uint2*>(p) = make_uint2(d0, d1);
    return;
  }
  const unsigned long long w = static_cast<unsigned long long>(d0) | (static_cast<unsigned long long>(d1) << 32);
  for (int k = 0; k < 8; k++) {
    if (static_cast<size_t>(k) < avail) p[k] = static_cast<char>(w >> (8 * k));
  }
}
}  // namespace

__global__ void __launch_bounds__(kThreads)
llExchangeKernel(CommArgs a, const char* __restrict__ in, char* __restrict__ out, size_t bytes, int mode, PeerPtrs ll,
                 size_t srcStride, size_t parityStride) {
  const uint32_t seq = ld_relaxed_sys(&a.self->llSeq) + 1u;
  const size_t base = (seq & 1u) * parityStride;
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = a.nranks;
  const size_t nunits = (bytes + 7) / 8;
  const size_t items = static_cast<size_t>(P) * nunits;
  const bool inAligned = reinterpret_cast<uintptr_t>(in) % 8 == 0 && bytes % 8 == 0;
  const bool outAligned = reinterpret_cast<uintptr_t>(out) % 8 == 0 && bytes % 8 == 0;
  // send: item = (peer slot i, unit u); peers rotated by rank
  for (size_t it = tid; it < items; it += nthreads) {
    const int i = static_cast<int>(it / nunits);
    const size_t u = it % nunits;
    const int dst = (a.rank + i) % P;
    const char* src = in + (mode == 1 ? static_cast<size_t>(dst) * bytes : 0) + u * 8;
    uint32_t d0, d1;
    load8(src, bytes - u * 8, inAligned, d0, d1);
    if (dst == a.rank) {
      store8(out + static_cast<size_t>(a.rank) * bytes + u * 8, bytes - u * 8, outAligned, d0, d1);
    } else {
      llStore(static_cast<char*>(ll.p[dst]) + base + static_cast<size_t>(a.rank) * srcStride + u * 16, d0, d1, seq);
    }
  }
  // receive
  const char* mine = static_cast<const char*>(ll.p[a.rank]) + base;
  for (size_t it = tid; it < items; it += nthreads) {
    const int i = static_cast<int>(it / nunits);
    const size_t u = it % nunits;
    const int src = (a.rank + i) % P;
    if (src == a.rank) continue;
    uint32_t d0, d1;
    if (!llLoad(a, mine + static_cast<size_t>(src) * srcStride + u * 16, seq, d0, d1, src)) break;
    store8(out + static_cast<size_t>(src) * bytes + u * 8, bytes - u * 8, outAligned, d0, d1);
  }
  retire(a, 0, 0, 1);
}

void launchLLExchange(const CommArgs& a, const void* in, void* out, size_t bytes, int mode, const PeerPtrs& ll,
                      size_t srcStride, size_t parityStride, int blocks, int threads, cudaStream_t stream) {
  llExchangeKernel<<<blocks, threads, 0, stream>>>(a, static_cast<const char*>(in), static_cast<char*>(out), bytes, mode,
                                                   ll, srcStride, parityStride);
}

const void* broadcastKernelPtr() { return reinterpret_cast<const void*>(broadcastKernel); }
const void* gatherPushKernelPtr() { return reinterpret_cast<const void*>(gatherPushKernel); }
const void* alltoallPushKernelPtr() { return reinterpret_cast<const void*>(alltoallPushKernel); }
const void* alltoallvDevKernelPtr(bool fp8) {
  return fp8 ? reinterpret_cast<const void*>(alltoallvDevKernel<true>)
             : reinterpret_cast<const void*>(alltoallvDevKernel<false>);
}
const void* moeCombineTopkKernelPtr(DataType dt) { return reinterpret_cast<const void*>(topkCombineFn(dt)); }
const void* moeDispatchTopkKernelPtr(bool fp8) {
  return fp8 ? reinterpret_cast<const void*>(moeDispatchTopkKernel<true>)
             : reinterpret_cast<const void*>(moeDispatchTopkKernel<false>);
}
const void* reducePullKernelPtr(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(reducePullFn<decltype(tag)>(nranks)); });
  return k;
}

void preloadCollectiveKernels() {
  touchKernel(broadcastKernel);
  touchKernel(gatherPushKernel);
  touchKernel(alltoallPushKernel);
  touchKernel(alltoallvDevKernel<false>);
  touchKernel(alltoallvDevKernel<true>);
  for (DataType dt : {DataType::FLOAT32, DataType::BFLOAT16, DataType::FLOAT16}) touchKernel(topkCombineFn(dt));
  touchKernel(moeDispatchTopkKernel<false>);
  touchKernel(moeDispatchTopkKernel<true>);
  touchKernel(llExchangeKernel);
  for (DataType dt : kAllDataTypes) {
    dispatchType(dt, [&](auto tag) {
      for (int P : {0, 2, 4, 8}) touchKernel(reducePullFn<decltype(tag)>(P));
    });
  }
  cudaGetLastError();
}

}  // namespace cuda
}  // namespace glb
