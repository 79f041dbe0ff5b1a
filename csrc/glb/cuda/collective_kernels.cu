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

// The cast allgather(v): my block is float32 at `in`; it is rounded to TO (round to nearest even,
// overflow to +-inf, NaN stays NaN) as it is read, and only TO bytes are pushed. va counts TO
// elements. `vec`: `in` and every output are 16-byte aligned.
template <typename TO>
__global__ void __launch_bounds__(kThreads, 2)
castGatherPushKernel(CommArgs a, const float* __restrict__ in, PeerPtrs outs, VArgs va, bool vec) {
  const uint32_t e = loadEpoch(a);
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = a.nranks;
  if (!blockBarrier<false>(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  const size_t off = va.off[a.rank], len = va.len[a.rank];
  const size_t nitems = vec && (off * sizeof(TO)) % 16 == 0 ? len / 8 : 0;
  for (size_t it = tid; it < nitems; it += nthreads) {
    float v[8];
    Item8<float>::load(in + it * 8, v);
    for (int i = 0; i < P; i++) Item8<TO>::store(static_cast<TO*>(outs.p[(a.rank + i) % P]) + off + it * 8, v);
  }
  for (size_t i = nitems * 8 + tid; i < len; i += nthreads) {
    const TO c = Scalar<TO>::fromAcc(in[i]);
    for (int r = 0; r < P; r++) static_cast<TO*>(outs.p[r])[off + i] = c;
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

namespace {
VArgs vargs(int nranks, const size_t* offs, const size_t* lens) {
  VArgs va;
  for (int i = 0; i < kMaxRanks; i++) {
    va.off[i] = i < nranks ? offs[i] : 0;
    va.len[i] = i < nranks ? lens[i] : 0;
  }
  return va;
}
}  // namespace

void launchCastGatherPush(const CommArgs& a, const void* in, const PeerPtrs& outs, DataType outDt, const size_t* offs,
                          const size_t* counts, bool vec, int blocks, cudaStream_t stream) {
  dispatchHalfType(outDt, [&](auto tag) {
    castGatherPushKernel<decltype(tag)><<<blocks, kThreads, 0, stream>>>(a, static_cast<const float*>(in), outs,
                                                                          vargs(a.nranks, offs, counts), vec);
  });
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

// The cast reduce_scatter: 16-bit inputs, float32 `out`, SUM. Rank r's share is accumulated in
// fp32 in peer order, scaled in fp32 and stored as fp32: it is never rounded to 16 bits. No
// multimem form: multimem.ld_reduce on 16-bit data would return a 16-bit sum.
template <typename TI, int NR, int UNROLL>
__global__ void __launch_bounds__(kThreads)
castReducePullKernel(CommArgs a, PeerPtrs ins, float* __restrict__ out, EArgs ea, float scale, bool vec) {
  using PT = PackTraits<TI>;
  const uint32_t e = loadEpoch(a);
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const int P = NR > 0 ? NR : a.nranks;
  if (!blockBarrier<false>(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  const size_t off = ea.off[a.rank], len = ea.len[a.rank];
  const bool v16 = vec && (off * sizeof(TI)) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
  const size_t nvec = v16 ? len / PT::kElems : 0;
  const size_t byteOff = off * sizeof(TI);
  constexpr int kSlots = NR > 0 ? NR : kMaxRanks;
  const char* peer[kSlots];
#pragma unroll
  for (int i = 0; i < kSlots; i++) {
    peer[i] = i < P ? static_cast<const char*>(ins.p[(a.rank + i) % P]) + byteOff : nullptr;
  }
  reducePeers<TI, kSlots, UNROLL, 0, false>(
      P, tid, nvec, nthreads, DevOp::SUM, scale, [&](int i) { return peer[i]; },
      [&](size_t v, const typename PT::AccPack& r) { Item8<float>::store(out + v * PT::kElems, r.v); });
  for (size_t i = nvec * PT::kElems + tid; i < len; i += nthreads) {
    float acc = Scalar<TI>::toAcc(static_cast<const TI*>(ins.p[0])[off + i]);
    for (int r = 1; r < P; r++) acc += Scalar<TI>::toAcc(static_cast<const TI*>(ins.p[r])[off + i]);
    if (scale != 1.0f) acc *= scale;
    out[i] = acc;
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

namespace {
// The cast reduce-pull instantiation for (TI, P).
template <typename TI>
auto castReducePullFn(int nranks) {
  if (nranks == 2) return castReducePullKernel<TI, 2, 4>;
  if (nranks == 4) return castReducePullKernel<TI, 4, 2>;
  if (nranks == 8) return castReducePullKernel<TI, 8, 2>;
  return castReducePullKernel<TI, 0, 1>;
}
}  // namespace

void launchCastReducePull(const CommArgs& a, const PeerPtrs& ins, float* out, const size_t* elemOff,
                          const size_t* elemLen, DataType dt, float scale, bool vec, int blocks, cudaStream_t stream) {
  EArgs ea;
  for (int i = 0; i < kMaxRanks; i++) {
    ea.off[i] = i < a.nranks ? elemOff[i] : 0;
    ea.len[i] = i < a.nranks ? elemLen[i] : 0;
  }
  dispatchHalfType(dt, [&](auto tag) {
    castReducePullFn<decltype(tag)>(a.nranks)<<<blocks, kThreads, 0, stream>>>(a, ins, out, ea, scale, vec);
  });
}

// ---- one rank: out = TO(float(in) * scale) -----------------------------------------------------
// The P = 1 form of the cast reduce_scatter (16-bit in, float32 out) and allgather (float32 in,
// 16-bit out): the conversion and the scale of the collective, with nothing to exchange.
template <typename TI, typename TO>
__global__ void __launch_bounds__(kThreads)
castScaleKernel(const TI* __restrict__ in, TO* __restrict__ out, size_t count, float scale, bool vec) {
  const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
  const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  const size_t nitems = vec ? count / 8 : 0;
  for (size_t it = tid; it < nitems; it += nthreads) {
    float v[8];
    Item8<TI>::load(in + it * 8, v);
    if (scale != 1.0f) {
#pragma unroll
      for (int k = 0; k < 8; k++) v[k] *= scale;
    }
    Item8<TO>::store(out + it * 8, v);
  }
  for (size_t i = nitems * 8 + tid; i < count; i += nthreads) {
    float x = Scalar<TI>::toAcc(in[i]);
    if (scale != 1.0f) x *= scale;
    out[i] = Scalar<TO>::fromAcc(x);
  }
}

namespace {
// Calls f(TI{}, TO{}) for the pairs of the cast reduce_scatter and allgather.
template <typename F>
void dispatchCastLocal(DataType in, DataType out, F&& f) {
  if (in == DataType::FLOAT32) {
    dispatchHalfType(out, [&](auto to) { f(float{}, to); });
  } else if (out == DataType::FLOAT32) {
    dispatchHalfType(in, [&](auto ti) { f(ti, float{}); });
  }
}
}  // namespace

void launchCastScale(const void* in, DataType inDt, void* out, DataType outDt, size_t count, float scale, int blocks,
                     cudaStream_t stream) {
  const bool vec = (reinterpret_cast<uintptr_t>(in) | reinterpret_cast<uintptr_t>(out)) % 16 == 0;
  dispatchCastLocal(inDt, outDt, [&](auto ti, auto to) {
    using TI = decltype(ti);
    using TO = decltype(to);
    castScaleKernel<TI, TO><<<blocks, kThreads, 0, stream>>>(static_cast<const TI*>(in), static_cast<TO*>(out), count,
                                                             scale, vec);
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
const void* reducePullKernelPtr(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(reducePullFn<decltype(tag)>(nranks)); });
  return k;
}

const void* castReducePullKernelPtr(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchHalfType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(castReducePullFn<decltype(tag)>(nranks)); });
  return k;
}
const void* castGatherPushKernelPtr(DataType outDt) {
  const void* k = nullptr;
  dispatchHalfType(outDt, [&](auto tag) { k = reinterpret_cast<const void*>(castGatherPushKernel<decltype(tag)>); });
  return k;
}

void preloadCollectiveKernels() {
  touchKernel(broadcastKernel);
  touchKernel(gatherPushKernel);
  touchKernel(alltoallPushKernel);
  touchKernel(llExchangeKernel);
  for (DataType dt : kAllDataTypes) {
    dispatchType(dt, [&](auto tag) {
      for (int P : {0, 2, 4, 8}) touchKernel(reducePullFn<decltype(tag)>(P));
    });
    dispatchHalfType(dt, [&](auto tag) {
      using T = decltype(tag);
      for (int P : {0, 2, 4, 8}) touchKernel(castReducePullFn<T>(P));
      touchKernel(castGatherPushKernel<T>);
      touchKernel(castScaleKernel<T, float>);
      touchKernel(castScaleKernel<float, T>);
    });
  }
  cudaGetLastError();
}

}  // namespace cuda
}  // namespace glb
