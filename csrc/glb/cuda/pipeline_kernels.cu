// Pipelined allreduce for ARBITRARY device pointers (sm_90a).
//
// The reference API takes plain `T*` (cuda_allreduce_ring_chunked.h:30-36); a pointer that
// is neither registered nor symmetric cannot be read by the peers (and cannot be bound to an
// NVSwitch multicast object), so the data has to pass through the symmetric pool. Instead
// of copy-in / collective / copy-out as three passes, ONE persistent kernel runs a
// three-stage software pipeline over chunks of the vector, one device barrier per step:
//
//     step i:   A(i)    copy chunk i        user input  -> pool slot i % 3      (local HBM)
//               B(i-1)  reduce chunk i-1    in the pool: multimem.ld_reduce + multimem.st
//                                           through the NVSwitch (or peer loads + stores)
//               C(i-2)  copy chunk i-2      pool slot -> user output              (local HBM)
//
// The three stages of a step touch three different slots, so they run concurrently: the
// warps of every CTA are split into an exchange group (B, NVLink-bound) and a copy group
// (A and C, HBM-bound) and the local copies hide under the NVLink time.
//
// Ownership: a chunk is P shares x G tiles x T 16-byte groups; CTA b owns tile b of every
// share in every stage, so the CTA-to-CTA flag barrier is all the synchronisation needed
// (the CTA that reads a peer's tile is barrier-paired with the CTA that wrote it).
//
// allgather(v) / gather(v) and reduce_scatter of plain pointers use the same framework with
// two stages, and both PULL:
//
//     step i:   A(i)    copy chunk i of my data     user input -> my pool slot i % 2   (local HBM)
//               B(i-1)  load chunk i-1 from slot (i-1) % 2 of every peer, (reduce,) store to
//                       the user output                                                 (NVLink)
//
// Chunk i covers bytes [i*C, (i+1)*C) of EVERY rank's block (allgather) or share
// (reduce_scatter), C = G*T*16. The chunk count comes from the largest block, so the grid and
// the number of steps (chunks + 1, one barrier each) are the same on every rank.
//
// Two slots are enough: nothing is written back into the pool to be read again later. The slot
// a rank fills in step i+1 is the slot its peers read in step i; the rank starts step i+1 only
// after barrier i, and it passes barrier i only when CTA b of every peer has finished step i.
//
// alltoall(v) / scatter and reduce use the same framework and also pull:
//  * pipelinedAlltoallKernel: two slots of P sub-slots of C bytes. A(i) copies chunk i of my block
//    for rank j into sub-slot j of my slot i % 2 (my own block straight to the output); B(i-1)
//    pulls sub-slot `me` of slot (i-1) % 2 of every peer into the output. Two slots are enough for
//    the reason above. The v-variant's lengths are rank-local, so the ranks agree on the chunk
//    count on the device: each publishes its need before barrier 1 (SignalPad::pipeChunks) and
//    all run max(maximum, 1) + 1 steps. Even when every block is empty there are two barriers,
//    so the table is read before the final barrier (see SignalPad::pipeChunks).
//  * pipelinedReduceKernel: the input slots of reduce_scatter plus two result slots of C bytes,
//    three stages and chunks + 2 steps. B(i-1) reduces my share of chunk i-1; the root stores it
//    to the output, every other rank to its own result slot (i-1) % 2. C(i-2), root only, pulls
//    share q of chunk i-2 from peer q's result slot (i-2) % 2. Two result slots are enough: a rank
//    rewrites result slot k in step k+2, after barrier k+1, which it passes only when the root's
//    CTA b has finished step k+1, the step in which the root reads that slot.
//
// Pool rules, which every kernel that uses the bulk region keeps, so that consecutive calls
// need no other synchronisation:
//  * Before its first barrier, a kernel writes only its own pool. A peer may still be reading
//    its own bulk region at that point: the staged paths copy out of the pool with a
//    cudaMemcpyAsync after their kernel's final barrier. Pulling keeps this rule without an
//    entry barrier (gatherPushKernel, which pushes, pays one before its first remote store).
//  * A kernel reads a peer's pool for the last time before its own final barrier.
//
// Why pull: a pushed chunk lands in the receiver's pool and has to be read again to reach the
// output, an extra (P-1)·s pass over the receiver's HBM; pulling costs one extra s (my own
// block into my pool).
#include "glb/cuda/device_common.cuh"
#include "glb/cuda/grid_copy.cuh"
#include "glb/cuda/kernels.h"
#include "glb/cuda/peer_reduce.cuh"

namespace glb {
namespace cuda {

namespace {

template <typename T>
__device__ __forceinline__ Pack16 loadGroupP(const T* base, size_t g, size_t count, bool aligned) {
  constexpr int K = 16 / sizeof(T);
  const size_t i0 = g * K;
  if (aligned && i0 + K <= count) return ld128_stream(reinterpret_cast<const char*>(base) + g * 16);
  Pack16 p;
  p.w[0] = p.w[1] = p.w[2] = p.w[3] = 0u;
  T* t = reinterpret_cast<T*>(&p);
#pragma unroll
  for (int k = 0; k < K; k++) {
    if (i0 + k < count) t[k] = base[i0 + k];
  }
  return p;
}

template <typename T>
__device__ __forceinline__ void storeGroupP(T* base, size_t g, size_t count, bool aligned, const Pack16& p) {
  constexpr int K = 16 / sizeof(T);
  const size_t i0 = g * K;
  if (aligned && i0 + K <= count) {
    st128_stream(reinterpret_cast<char*>(base) + g * 16, p);
    return;
  }
  const T* t = reinterpret_cast<const T*>(&p);
#pragma unroll
  for (int k = 0; k < K; k++) {
    if (i0 + k < count) base[i0 + k] = t[k];
  }
}

}  // namespace

template <typename T, bool MC, int NR>
__global__ void __launch_bounds__(kThreads)
pipelinedAllreduceKernel(CommArgs a, const T* in, T* out, size_t count, DevOp op, float scale, PeerPtrs stage,
                         char* mcStage, int tileVecs, int exchangeThreads, LocalPtrs extra) {
  using PT = PackTraits<T>;
  const int P = NR > 0 ? NR : a.nranks;
  const int G = gridDim.x;
  const int b = blockIdx.x;
  const size_t T_ = static_cast<size_t>(tileVecs);  // power of two (host enforces)
  const int tileShift = 31 - __clz(tileVecs);
  const size_t chunkVecs = static_cast<size_t>(P) * G * T_;
  const size_t slotBytes = chunkVecs * 16;
  const size_t ngroups = (count + PT::kElems - 1) / PT::kElems;
  const size_t nchunks = (ngroups + chunkVecs - 1) / chunkVecs;
  const uint32_t e = loadEpoch(a);
  char* myStage = static_cast<char*>(stage.p[a.rank]);

  bool aligned = reinterpret_cast<uintptr_t>(in) % 16 == 0 && reinterpret_cast<uintptr_t>(out) % 16 == 0;
  for (int k = 0; k < extra.n; k++) aligned = aligned && reinterpret_cast<uintptr_t>(extra.p[k]) % 16 == 0;

  const bool exchanger = static_cast<int>(threadIdx.x) < exchangeThreads;
  const int xt = threadIdx.x, xn = exchangeThreads;                            // exchange group
  const int ct = threadIdx.x - exchangeThreads, cn = blockDim.x - exchangeThreads;  // copy group

  uint32_t used = 0;
  for (size_t i = 0; i < nchunks + 2; i++) {
    if (exchanger) {
      // ---- B(i-1): reduce my share's tile of chunk i-1 in the pool, deliver to everyone ----
      if (i >= 1 && i - 1 < nchunks) {
        const size_t slot = ((i - 1) % 3) * slotBytes;
        const size_t w0 = (static_cast<size_t>(a.rank) * G + b) * T_;
        // Not reduceMultimem / reducePeers: through them this kernel's registers are allocated
        // differently, and the instantiations that already spill spill other amounts.
        if constexpr (MC) {
          char* mc = mcStage + slot + w0 * 16;
          constexpr int U = 4;
          for (size_t o0 = xt; o0 < T_; o0 += static_cast<size_t>(xn) * U) {
            Pack16 r[U];
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t o = o0 + static_cast<size_t>(u) * xn;
              if (o < T_) r[u] = Multimem<T>::ldReduceAdd(mc + o * 16);
            }
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t o = o0 + static_cast<size_t>(u) * xn;
              if (o < T_) {
                if (scale != 1.0f) {
                  typename PT::AccPack acc = PT::widen(r[u]);
                  PT::scale(acc, scale);
                  r[u] = PT::narrow(acc);
                }
                multimemSt128(mc + o * 16, r[u]);
              }
            }
          }
        } else {
          // Peer exchange inside the pool, like the two-shot kernel: kSlots x U independent
          // 128-bit loads in flight per thread (an NVLink round trip is ~2 us).
          constexpr int kSlots = NR > 0 ? NR : kMaxRanks;
          // 16-lane (FP8) packs widen to twice the fp32 registers of 8-lane ones: half the packs in
          // flight keeps the exchange free of spills (-Xptxas -v).
          constexpr int kWide = PT::kElems > 8 ? 2 : 1;
          constexpr int U0 = NR == 2 ? 8 : (NR == 4 ? 4 : (NR == 8 ? 2 : 1));
          constexpr int U = U0 / kWide > 0 ? U0 / kWide : 1;
          char* peer[kSlots];
#pragma unroll
          for (int q = 0; q < kSlots; q++) {
            peer[q] = q < P ? static_cast<char*>(stage.p[(a.rank + q) % P]) + slot + w0 * 16 : nullptr;
          }
          if constexpr (kWide > 1 && kSlots > 8) {
            // Any P with 16-lane packs: the peers' packs come in two batches of 8 (same order).
            for (size_t o = xt; o < T_; o += static_cast<size_t>(xn)) {
              typename PT::AccPack acc;
#pragma unroll
              for (int b0 = 0; b0 < kSlots; b0 += 8) {
                Pack16 v[8];
#pragma unroll
                for (int q = 0; q < 8; q++) {
                  if (b0 + q < P) v[q] = ld128_stream(peer[b0 + q] + o * 16);
                }
#pragma unroll
                for (int q = 0; q < 8; q++) {
                  if (b0 + q == 0) {
                    acc = PT::widen(v[q]);
                  } else if (b0 + q < P) {
                    PT::combine(acc, v[q], op);
                  }
                }
              }
              if (scale != 1.0f) PT::scale(acc, scale);
              const Pack16 res = PT::narrow(acc);
#pragma unroll
              for (int q = 0; q < kSlots; q++) {
                if (q < P) st128_stream(peer[q] + o * 16, res);
              }
            }
          } else {
            for (size_t o0 = xt; o0 < T_; o0 += static_cast<size_t>(xn) * U) {
              Pack16 v[U][kSlots];
#pragma unroll
              for (int u = 0; u < U; u++) {
                const size_t o = o0 + static_cast<size_t>(u) * xn;
                if (o < T_) {
#pragma unroll
                  for (int q = 0; q < kSlots; q++) {
                    if (q < P) v[u][q] = ld128_stream(peer[q] + o * 16);
                  }
                }
              }
#pragma unroll
              for (int u = 0; u < U; u++) {
                const size_t o = o0 + static_cast<size_t>(u) * xn;
                if (o < T_) {
                  typename PT::AccPack acc = PT::widen(v[u][0]);
#pragma unroll
                  for (int q = 1; q < kSlots; q++) {
                    if (q < P) PT::combine(acc, v[u][q], op);
                  }
                  if (scale != 1.0f) PT::scale(acc, scale);
                  const Pack16 res = PT::narrow(acc);
#pragma unroll
                  for (int q = 0; q < kSlots; q++) {
                    if (q < P) st128_stream(peer[q] + o * 16, res);
                  }
                }
              }
            }
          }
        }
      }
    } else {
      // independent 128-bit accesses in flight per copy thread (half for 16-lane packs, as above)
      constexpr int CU = PT::kElems > 8 ? 2 : 4;
      const size_t PT_ = static_cast<size_t>(P) * T_;
      // ---- C(i-2): pool -> user output ----------------------------------------------------
      if (i >= 2) {
        const size_t c = i - 2;
        const char* slot = myStage + (c % 3) * slotBytes;
        const size_t g0 = c * chunkVecs;
        for (size_t j0 = ct; j0 < PT_; j0 += static_cast<size_t>(cn) * CU) {
          Pack16 p[CU];
          size_t g[CU];
#pragma unroll
          for (int u = 0; u < CU; u++) {
            const size_t j = j0 + static_cast<size_t>(u) * cn;
            const size_t w = (((j >> tileShift) * G + b) << tileShift) + (j & (T_ - 1));
            g[u] = j < PT_ ? g0 + w : ngroups;
            if (g[u] < ngroups) p[u] = ld128(slot + w * 16);
          }
#pragma unroll
          for (int u = 0; u < CU; u++) {
            if (g[u] < ngroups) {
              storeGroupP(out, g[u], count, aligned, p[u]);
              for (int k = 0; k < extra.n; k++) storeGroupP(static_cast<T*>(extra.p[k]), g[u], count, aligned, p[u]);
            }
          }
        }
      }
      // ---- A(i): user input -> pool -------------------------------------------------------
      if (i < nchunks) {
        char* slot = myStage + (i % 3) * slotBytes;
        const size_t g0 = i * chunkVecs;
        for (size_t j0 = ct; j0 < PT_; j0 += static_cast<size_t>(cn) * CU) {
          Pack16 p[CU];
          size_t w[CU];
#pragma unroll
          for (int u = 0; u < CU; u++) {
            const size_t j = j0 + static_cast<size_t>(u) * cn;
            w[u] = j < PT_ ? (((j >> tileShift) * G + b) << tileShift) + (j & (T_ - 1)) : chunkVecs;
            const size_t g = g0 + w[u];
            if (w[u] < chunkVecs && g < ngroups) {
              p[u] = loadGroupP(in, g, count, aligned);
              if (extra.n > 0) {
                typename PT::AccPack acc = PT::widen(p[u]);
                for (int k = 0; k < extra.n; k++) {
                  PT::combine(acc, loadGroupP(static_cast<const T*>(extra.p[k]), g, count, aligned), op);
                }
                p[u] = PT::narrow(acc);
              }
            } else {
              p[u].w[0] = p[u].w[1] = p[u].w[2] = p[u].w[3] = 0u;  // keep the reduction of the padding finite
            }
          }
#pragma unroll
          for (int u = 0; u < CU; u++) {
            if (w[u] < chunkVecs) st128(slot + w[u] * 16, p[u]);
          }
        }
      }
    }
    used++;
    if (!blockBarrier(a, e + used)) break;
  }
  retire(a, static_cast<uint32_t>(nchunks + 2), 0);
}

namespace {
// The pipelined instantiation for (T, multicast stage, P).
template <typename T>
auto pipeFn(bool mc, int nranks) {
  if constexpr (hasMultimem<T>()) {
    if (mc) return pipelinedAllreduceKernel<T, true, 0>;
  }
  if constexpr (isHotType<T>()) {
    if (nranks == 2) return pipelinedAllreduceKernel<T, false, 2>;
    if (nranks == 4) return pipelinedAllreduceKernel<T, false, 4>;
    if (nranks == 8) return pipelinedAllreduceKernel<T, false, 8>;
  }
  return pipelinedAllreduceKernel<T, false, 0>;
}
}  // namespace

const void* pipelinedKernelFor(DataType dt, bool mc, int nranks) {
  const void* k = nullptr;
  dispatchType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(pipeFn<decltype(tag)>(mc, nranks)); });
  return k;
}

void launchPipelinedAllreduce(const CommArgs& a, const void* in, void* out, size_t count, DataType dt, ReduceOp op,
                              float scale, const PeerPtrs& stage, void* mcStage, int tileVecs, int exchangeThreads,
                              const LocalPtrs& extra, int blocks, cudaStream_t stream) {
  const bool mc = mcStage != nullptr && nvlsSupports(dt, op);
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    pipeFn<T>(mc, a.nranks)<<<blocks, kThreads, 0, stream>>>(a, static_cast<const T*>(in), static_cast<T*>(out), count,
                                                             static_cast<DevOp>(op), scale, stage,
                                                             mc ? static_cast<char*>(mcStage) : nullptr, tileVecs,
                                                             exchangeThreads, extra);
  });
}

// Per-rank blocks (allgather: bytes) or shares (reduce_scatter: elements).
struct PipeBlocks {
  size_t off[kMaxRanks];
  size_t len[kMaxRanks];
};

namespace {
// Part of a block of `len` units that falls into tile b of chunk c (units per tile: tileUnits).
__device__ __forceinline__ size_t tilePart(size_t len, size_t c, size_t chunkUnits, size_t tileUnits) {
  const size_t s = c * chunkUnits + blockIdx.x * tileUnits;
  return len > s ? (len - s < tileUnits ? len - s : tileUnits) : 0;
}

__device__ __forceinline__ size_t largestOf(const PipeBlocks& pb, int P) {
  size_t m = 0;
  for (int q = 0; q < P; q++) m = pb.len[q] > m ? pb.len[q] : m;
  return m;
}
}  // namespace

// n float32 elements of src rounded to TO (nearest even, overflow to +-inf, NaN stays NaN) at dst
// and, unless it is null, at dst2; by thread t of a team of nt.
template <typename TO>
__device__ __forceinline__ void castCopy(TO* dst, TO* dst2, const float* src, size_t n, int t, int nt) {
  const uintptr_t all = reinterpret_cast<uintptr_t>(src) | reinterpret_cast<uintptr_t>(dst) |
                        reinterpret_cast<uintptr_t>(dst2);
  const size_t items = all % 16 == 0 ? n / 8 : 0;
  for (size_t it = t; it < items; it += nt) {
    float v[8];
    Item8<float>::load(src + it * 8, v);
    Item8<TO>::store(dst + it * 8, v);
    if (dst2 != nullptr) Item8<TO>::store(dst2 + it * 8, v);
  }
  for (size_t i = items * 8 + t; i < n; i += nt) {
    const TO c = Scalar<TO>::fromAcc(src[i]);
    dst[i] = c;
    if (dst2 != nullptr) dst2[i] = c;
  }
}

// Slot: C bytes, my chunk. A(i): my chunk i -> my slot, and to out + off[me] unless `in` already
// is that address (in place) or I receive nothing (gather, not the root). B(i-1): chunk i-1 of
// every peer's slot -> out + off[q] (only the root for gather: a non-root never writes its out).
// TO = char copies bytes. TO = __half / __nv_bfloat16 is the cast allgather: `in` holds float32
// elements, A(i) rounds them to TO as it reads them, and the blocks, the slots and the pulls are
// in TO bytes, so only TO bytes cross NVLink.
template <typename TO>
__device__ __forceinline__ void allgatherPipe(CommArgs& a, const char* in, char* out, const PipeBlocks& pb, int onlyDst,
                                              const PeerPtrs& stage, int tileVecs, int exchangeThreads) {
  const int P = a.nranks, me = a.rank;
  const size_t tileBytes = static_cast<size_t>(tileVecs) * 16;
  const size_t C = gridDim.x * tileBytes;
  const size_t nchunks = (largestOf(pb, P) + C - 1) / C;
  const size_t tileOff = blockIdx.x * tileBytes;
  const uint32_t e = loadEpoch(a);
  char* myStage = static_cast<char*>(stage.p[me]);
  const bool receiver = onlyDst < 0 || onlyDst == me;
  const bool copyOwn = receiver && out + pb.off[me] != in;
  const bool exchanger = static_cast<int>(threadIdx.x) < exchangeThreads;
  const int xt = threadIdx.x, xn = exchangeThreads;
  const int ct = threadIdx.x - exchangeThreads, cn = blockDim.x - exchangeThreads;

  for (size_t i = 0; i < nchunks + 1; i++) {
    if (exchanger) {
      // ---- B(i-1): pull every peer's chunk i-1 into my output ----
      if (i >= 1 && receiver) {
        const size_t c = i - 1;
        for (int k = 1; k < P; k++) {
          const int q = (me + k) % P;
          const size_t n = tilePart(pb.len[q], c, C, tileBytes);
          if (n > 0) {
            gridCopy(out + pb.off[q] + c * C + tileOff,
                     static_cast<const char*>(stage.p[q]) + (c % 2) * C + tileOff, n, true, xt, xn);
          }
        }
      }
    } else if (i < nchunks) {
      // ---- A(i): my chunk i -> my slot (and my own block of the output) ----
      const size_t n = tilePart(pb.len[me], i, C, tileBytes);
      if (n > 0) {
        if constexpr (std::is_same<TO, char>::value) {
          const char* src = in + i * C + tileOff;
          gridCopy(myStage + (i % 2) * C + tileOff, src, n, true, ct, cn);
          if (copyOwn) gridCopy(out + pb.off[me] + i * C + tileOff, src, n, true, ct, cn);
        } else {
          const float* src = reinterpret_cast<const float*>(in) + (i * C + tileOff) / sizeof(TO);
          castCopy(reinterpret_cast<TO*>(myStage + (i % 2) * C + tileOff),
                   copyOwn ? reinterpret_cast<TO*>(out + pb.off[me] + i * C + tileOff) : nullptr, src, n / sizeof(TO),
                   ct, cn);
        }
      }
    }
    if (!blockBarrier(a, e + static_cast<uint32_t>(i) + 1)) break;
  }
  retire(a, static_cast<uint32_t>(nchunks + 1), 0);
}

__global__ void __launch_bounds__(kThreads)
pipelinedAllgatherKernel(CommArgs a, const char* in, char* out, PipeBlocks pb, int onlyDst, PeerPtrs stage,
                         int tileVecs, int exchangeThreads) {
  allgatherPipe<char>(a, in, out, pb, onlyDst, stage, tileVecs, exchangeThreads);
}

template <typename TO>
__global__ void __launch_bounds__(kThreads)
castPipelinedAllgatherKernel(CommArgs a, const char* in, char* out, PipeBlocks pb, PeerPtrs stage, int tileVecs,
                             int exchangeThreads) {
  allgatherPipe<TO>(a, in, out, pb, -1, stage, tileVecs, exchangeThreads);
}

// A stage of reduce_scatter and reduce: chunk i of every share of `in` -> sub-slot q of `slot`
// (tile b of it; `slot` already points at the tile).
template <typename T>
__device__ __forceinline__ void stageShares(const T* in, const PipeBlocks& pb, int P, size_t i, size_t chunkElems,
                                            size_t tileElems, size_t C, char* slot, int ct, int cn) {
  using PT = PackTraits<T>;
  constexpr int CU = PT::kElems > 8 ? 2 : 4;
  for (int q = 0; q < P; q++) {
    const size_t n = tilePart(pb.len[q], i, chunkElems, tileElems);
    if (n == 0) continue;
    const size_t ng = (n + PT::kElems - 1) / PT::kElems;
    const T* src = in + pb.off[q] + i * chunkElems + blockIdx.x * tileElems;
    const bool aligned = reinterpret_cast<uintptr_t>(src) % 16 == 0;
    for (size_t j0 = ct; j0 < ng; j0 += static_cast<size_t>(cn) * CU) {
      Pack16 p[CU];
#pragma unroll
      for (int u = 0; u < CU; u++) {
        const size_t j = j0 + static_cast<size_t>(u) * cn;
        if (j < ng) p[u] = loadGroupP(src, j, n, aligned);
      }
#pragma unroll
      for (int u = 0; u < CU; u++) {
        const size_t j = j0 + static_cast<size_t>(u) * cn;
        if (j < ng) st128(slot + q * C + j * 16, p[u]);
      }
    }
  }
}

// Slot: P sub-slots of C bytes, sub-slot q = chunk i of share q. A(i): chunk i of every share of
// `in` -> my slot i % 2. B(i-1): sub-slot `me` of slot (i-1) % 2 from all P pools, reduced in the
// accumulator type of PackTraits (fp32 for the 16-bit and FP8 types), scaled, rounded once and
// stored to out + (i-1)·C. Counts are in elements: a share of `in`, and `out`, may start at an
// address that is not 16-byte aligned (element-wise loads / stores at their groups).
// TO = float with a 16-bit T is the cast reduce_scatter: the pool holds T, and the fp32
// accumulator is stored as it is, never rounded to T.
template <typename T, int NR, typename TO>
__device__ __forceinline__ void reduceScatterPipe(CommArgs& a, const T* in, TO* out, const PipeBlocks& pb, DevOp op,
                                                  float scale, const PeerPtrs& stage, int tileVecs,
                                                  int exchangeThreads) {
  using PT = PackTraits<T>;
  const int P = NR > 0 ? NR : a.nranks;
  const int me = a.rank;
  const size_t T_ = static_cast<size_t>(tileVecs);
  const size_t tileElems = T_ * PT::kElems;
  const size_t chunkElems = gridDim.x * tileElems;
  const size_t C = chunkElems * sizeof(T);  // = G*T*16 bytes
  const size_t slotBytes = static_cast<size_t>(P) * C;
  const size_t nchunks = (largestOf(pb, P) + chunkElems - 1) / chunkElems;
  const size_t tileOff = blockIdx.x * T_ * 16;
  const uint32_t e = loadEpoch(a);
  char* myStage = static_cast<char*>(stage.p[me]);
  const bool outAligned = reinterpret_cast<uintptr_t>(out) % 16 == 0;
  const bool exchanger = static_cast<int>(threadIdx.x) < exchangeThreads;
  const int xt = threadIdx.x, xn = exchangeThreads;
  const int ct = threadIdx.x - exchangeThreads, cn = blockDim.x - exchangeThreads;

  for (size_t i = 0; i < nchunks + 1; i++) {
    if (exchanger) {
      // ---- B(i-1): reduce my share's tile of chunk i-1 from every pool ----
      const size_t c = i - 1;
      const size_t n = i >= 1 ? tilePart(pb.len[me], c, chunkElems, tileElems) : 0;
      if (n > 0) {
        const size_t ng = (n + PT::kElems - 1) / PT::kElems;
        TO* dst = out + c * chunkElems + blockIdx.x * tileElems;
        // Half the packs for 16-lane FP8, as in the allreduce pipeline. U is 6 rather than 8 at
        // P = 2, and any P loads in batches (of 4 for 8-byte lanes): the element-wise output path
        // needs the registers, and this keeps every instantiation free of spills (-Xptxas -v).
        constexpr int kSlots = NR > 0 ? NR : kMaxRanks;
        constexpr int kWide = PT::kElems > 8 ? 2 : 1;
        constexpr int U0 = NR == 2 ? 6 : (NR == 4 ? 4 : (NR == 8 ? 2 : 1));
        constexpr int U = U0 / kWide > 0 ? U0 / kWide : 1;
        constexpr int kBatch = kSlots <= 8 ? 0 : (sizeof(T) == 8 ? 4 : 8);
        const char* peer[kSlots];
#pragma unroll
        for (int q = 0; q < kSlots; q++) {
          peer[q] = q < P ? static_cast<const char*>(stage.p[(me + q) % P]) + (c % 2) * slotBytes + me * C + tileOff
                          : nullptr;
        }
        if constexpr (std::is_same<T, TO>::value) {
          reducePeers<T, kSlots, U, kBatch>(P, xt, ng, xn, op, scale, [&](int q) { return peer[q]; },
                                            [&](size_t o, const Pack16& r) { storeGroupP(dst, o, n, outAligned, r); });
        } else {
          // group o of T is groups 2o and 2o + 1 of the float32 out
          static_assert(PT::kElems == 8, "the cast form takes 16-bit inputs");
          reducePeers<T, kSlots, U, kBatch, false>(
              P, xt, ng, xn, op, scale, [&](int q) { return peer[q]; }, [&](size_t o, const typename PT::AccPack& r) {
                Pack16 lo, hi;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                  lo.w[k] = __float_as_uint(r.v[k]);
                  hi.w[k] = __float_as_uint(r.v[4 + k]);
                }
                storeGroupP(dst, 2 * o, n, outAligned, lo);
                storeGroupP(dst, 2 * o + 1, n, outAligned, hi);
              });
        }
      }
    } else if (i < nchunks) {
      // ---- A(i): chunk i of every share -> my slot (zero past a share's end) ----
      stageShares(in, pb, P, i, chunkElems, tileElems, C, myStage + (i % 2) * slotBytes + tileOff, ct, cn);
    }
    if (!blockBarrier(a, e + static_cast<uint32_t>(i) + 1)) break;
  }
  retire(a, static_cast<uint32_t>(nchunks + 1), 0);
}

template <typename T, int NR>
__global__ void __launch_bounds__(kThreads)
pipelinedReduceScatterKernel(CommArgs a, const T* in, T* out, PipeBlocks pb, DevOp op, float scale, PeerPtrs stage,
                             int tileVecs, int exchangeThreads) {
  reduceScatterPipe<T, NR, T>(a, in, out, pb, op, scale, stage, tileVecs, exchangeThreads);
}

// The cast reduce_scatter (16-bit TI in, float32 out, SUM) of plain pointers of any size.
template <typename TI, int NR>
__global__ void __launch_bounds__(kThreads)
castPipelinedReduceScatterKernel(CommArgs a, const TI* in, float* out, PipeBlocks pb, float scale, PeerPtrs stage,
                                 int tileVecs, int exchangeThreads) {
  reduceScatterPipe<TI, NR, float>(a, in, out, pb, DevOp::SUM, scale, stage, tileVecs, exchangeThreads);
}

// reduce to `root`: the shares are those of reduce_scatter, with three stages and two more pool
// slots of C bytes (the result slots) after the two input slots.
//   A(i)    chunk i of every share of `in` -> my input slot i % 2                     (local HBM)
//   B(i-1)  sub-slot `me` of input slot (i-1) % 2 from all P pools, reduced; the root stores
//           its share to `out`, every other rank to its OWN result slot (i-1) % 2       (NVLink)
//   C(i-2)  root only: share q of chunk i-2 from result slot (i-2) % 2 of peer q -> out (NVLink)
// chunks + 2 steps, one barrier each. A non-root never touches `out` (it may be null).
template <typename T, int NR>
__global__ void __launch_bounds__(kThreads)
pipelinedReduceKernel(CommArgs a, const T* in, T* out, PipeBlocks pb, int root, DevOp op, PeerPtrs stage, int tileVecs,
                      int exchangeThreads) {
  using PT = PackTraits<T>;
  const int P = NR > 0 ? NR : a.nranks;
  const int me = a.rank;
  const bool isRoot = me == root;
  const size_t T_ = static_cast<size_t>(tileVecs);
  const size_t tileElems = T_ * PT::kElems;
  const size_t chunkElems = gridDim.x * tileElems;
  const size_t C = chunkElems * sizeof(T);
  const size_t slotBytes = static_cast<size_t>(P) * C;
  const size_t resultOff = 2 * slotBytes;
  const size_t nchunks = (largestOf(pb, P) + chunkElems - 1) / chunkElems;
  const size_t tileOff = blockIdx.x * T_ * 16;
  const uint32_t e = loadEpoch(a);
  char* myStage = static_cast<char*>(stage.p[me]);
  const bool outAligned = !isRoot || reinterpret_cast<uintptr_t>(out + pb.off[me]) % 16 == 0;
  const bool exchanger = static_cast<int>(threadIdx.x) < exchangeThreads;
  const int xt = threadIdx.x, xn = exchangeThreads;
  const int ct = threadIdx.x - exchangeThreads, cn = blockDim.x - exchangeThreads;

  for (size_t i = 0; i < nchunks + 2; i++) {
    if (exchanger) {
      // ---- B(i-1): reduce my share's tile of chunk i-1 from every pool ----
      const size_t c = i - 1;
      const size_t n = i >= 1 && c < nchunks ? tilePart(pb.len[me], c, chunkElems, tileElems) : 0;
      if (n > 0) {
        T* dst = isRoot ? out + pb.off[me] + c * chunkElems + blockIdx.x * tileElems
                        : reinterpret_cast<T*>(myStage + resultOff + (c % 2) * C + tileOff);
        const size_t srcOff = (c % 2) * slotBytes + me * C + tileOff;
        const size_t ng = (n + PT::kElems - 1) / PT::kElems;
        auto store = [&](size_t o, const Pack16& r) { storeGroupP(dst, o, n, outAligned, r); };
        // Half of reduce_scatter's depth: the kernel also carries the root's pull stage. Any P takes
        // each peer's address from `stage` at its load instead of holding 16 pointers in registers.
        // Both keep every instantiation free of spills (-Xptxas -v).
        constexpr int kSlots = NR > 0 ? NR : kMaxRanks;
        constexpr int kWide = PT::kElems > 8 ? 2 : 1;
        constexpr int U0 = NR == 2 ? 4 : (NR == 4 ? 2 : 1);
        constexpr int U = U0 / kWide > 0 ? U0 / kWide : 1;
        if constexpr (kSlots > 8) {
          constexpr int kBatch = sizeof(T) == 8 || kWide > 1 ? 2 : 4;
          auto peer = [&](int q) {
            return static_cast<const char*>(stage.p[me + q < P ? me + q : me + q - P]) + srcOff;
          };
          reducePeers<T, kSlots, U, kBatch>(P, xt, ng, xn, op, 1.0f, peer, store);
        } else {
          const char* peer[kSlots];
#pragma unroll
          for (int q = 0; q < kSlots; q++) {
            peer[q] = q < P ? static_cast<const char*>(stage.p[(me + q) % P]) + srcOff : nullptr;
          }
          reducePeers<T, kSlots, U, 0>(P, xt, ng, xn, op, 1.0f, [&](int q) { return peer[q]; }, store);
        }
      }
    } else {
      // ---- C(i-2): the root pulls every peer's reduced share of chunk i-2 ----
      if (isRoot && i >= 2) {
        const size_t c = i - 2;
        for (int k = 1; k < P; k++) {
          const int q = (me + k) % P;
          const size_t n = tilePart(pb.len[q], c, chunkElems, tileElems);
          if (n > 0) {
            gridCopy(reinterpret_cast<char*>(out + pb.off[q] + c * chunkElems + blockIdx.x * tileElems),
                     static_cast<const char*>(stage.p[q]) + resultOff + (c % 2) * C + tileOff, n * sizeof(T), true, ct,
                     cn);
          }
        }
      }
      // ---- A(i): chunk i of every share -> my input slot ----
      if (i < nchunks) {
        stageShares(in, pb, P, i, chunkElems, tileElems, C, myStage + (i % 2) * slotBytes + tileOff, ct, cn);
      }
    }
    if (!blockBarrier(a, e + static_cast<uint32_t>(i) + 1)) break;
  }
  retire(a, static_cast<uint32_t>(nchunks + 2), 0);
}

// alltoall(v) and scatter. Slot: P sub-slots of C bytes, sub-slot j = chunk i of my block for
// destination j. Block j of `in` is send.len[j] bytes at send.off[j]; the block from source q lands
// at out + recv.off[q] (recv.len[q] bytes).
//   A(i)    chunk i of my block for every destination j != me -> sub-slot j of my slot i % 2; my
//           own block straight from `in` to out + recv.off[me]                         (local HBM)
//   B(i-1)  sub-slot `me` of slot (i-1) % 2 of every peer q -> out + recv.off[q] + (i-1)·C (NVLink)
// Scatter is the form in which only the root has blocks to send and every rank receives from the
// root only: a non-root never reads `in`.
// The step count: the lengths are rank-local (alltoallv), so each rank publishes the chunks it
// needs in the pipeChunks table before barrier 1 and every rank runs max(max, 1) + 1 steps. A(0)
// depends only on my own lengths, so it runs before that maximum is known. At least one chunk, so
// at least two barriers, even when every block is empty: the table is read between barrier 1 and
// the final barrier, and a peer rewrites its column in its next launch only after passing that
// final barrier, i.e. after every reader has read. With a single barrier, a peer could pass it,
// start its next launch and rewrite its column before a slow CTA here has read this launch's value.
__global__ void __launch_bounds__(kThreads)
pipelinedAlltoallKernel(CommArgs a, const char* in, char* out, PipeBlocks send, PipeBlocks recv, PeerPtrs stage,
                        int tileVecs, int exchangeThreads) {
  const int P = a.nranks, me = a.rank;
  const size_t tileBytes = static_cast<size_t>(tileVecs) * 16;
  const size_t C = gridDim.x * tileBytes;
  const size_t slotBytes = static_cast<size_t>(P) * C;
  const size_t tileOff = blockIdx.x * tileBytes;
  const uint32_t e = loadEpoch(a);
  char* myStage = static_cast<char*>(stage.p[me]);
  const size_t ownLen = send.len[me] < recv.len[me] ? send.len[me] : recv.len[me];
  const bool exchanger = static_cast<int>(threadIdx.x) < exchangeThreads;
  const int xt = threadIdx.x, xn = exchangeThreads;
  const int ct = threadIdx.x - exchangeThreads, cn = blockDim.x - exchangeThreads;
  // Every CTA writes the same value: the barrier pairs CTA b with CTA b only, so the column a CTA
  // reads must have been written by its own twin. The thread that writes peer q's pad is the one
  // that releases the barrier flag to q.
  if (threadIdx.x < P) {
    const size_t largest = largestOf(send, P) > largestOf(recv, P) ? largestOf(send, P) : largestOf(recv, P);
    st_relaxed_sys(&a.sig[threadIdx.x]->pipeChunks[me], static_cast<uint32_t>((largest + C - 1) / C));
  }

  size_t nchunks = 0;  // known after barrier 1
  for (size_t i = 0; i < nchunks + 1; i++) {
    if (exchanger) {
      // ---- B(i-1): pull my sub-slot of chunk i-1 from every peer ----
      if (i >= 1) {
        const size_t c = i - 1;
        for (int k = 1; k < P; k++) {
          const int q = (me + k) % P;
          const size_t n = tilePart(recv.len[q], c, C, tileBytes);
          if (n > 0) {
            gridCopy(out + recv.off[q] + c * C + tileOff,
                     static_cast<const char*>(stage.p[q]) + (c % 2) * slotBytes + me * C + tileOff, n, true, xt, xn);
          }
        }
      }
    } else {
      // ---- A(i): chunk i of every block -> my slot (my own block -> out) ----
      for (int k = 0; k < P; k++) {
        const int j = (me + k) % P;
        const size_t n = tilePart(j == me ? ownLen : send.len[j], i, C, tileBytes);
        if (n > 0) {
          char* dst = j == me ? out + recv.off[me] + i * C + tileOff : myStage + (i % 2) * slotBytes + j * C + tileOff;
          gridCopy(dst, in + send.off[j] + i * C + tileOff, n, true, ct, cn);
        }
      }
    }
    if (!blockBarrier(a, e + static_cast<uint32_t>(i) + 1)) break;
    if (i == 0) {
      nchunks = 1;  // at least two barriers: the read below must come before the final one
      for (int q = 0; q < P; q++) {
        const size_t need = ld_relaxed_sys(&a.self->pipeChunks[q]);
        nchunks = need > nchunks ? need : nchunks;
      }
    }
  }
  retire(a, static_cast<uint32_t>(nchunks + 1), 0);
}

namespace {
// The pipelined reduce_scatter instantiation for (T, P).
template <typename T>
auto pipeRsFn(int nranks) {
  if constexpr (isHotType<T>()) {
    if (nranks == 2) return pipelinedReduceScatterKernel<T, 2>;
    if (nranks == 4) return pipelinedReduceScatterKernel<T, 4>;
    if (nranks == 8) return pipelinedReduceScatterKernel<T, 8>;
  }
  return pipelinedReduceScatterKernel<T, 0>;
}

// The cast pipelined reduce_scatter instantiation for (TI, P).
template <typename TI>
auto castPipeRsFn(int nranks) {
  if (nranks == 2) return castPipelinedReduceScatterKernel<TI, 2>;
  if (nranks == 4) return castPipelinedReduceScatterKernel<TI, 4>;
  if (nranks == 8) return castPipelinedReduceScatterKernel<TI, 8>;
  return castPipelinedReduceScatterKernel<TI, 0>;
}

// The pipelined reduce instantiation for (T, P).
template <typename T>
auto pipeReduceFn(int nranks) {
  if constexpr (isHotType<T>()) {
    if (nranks == 2) return pipelinedReduceKernel<T, 2>;
    if (nranks == 4) return pipelinedReduceKernel<T, 4>;
    if (nranks == 8) return pipelinedReduceKernel<T, 8>;
  }
  return pipelinedReduceKernel<T, 0>;
}

PipeBlocks pipeBlocks(int nranks, const size_t* offs, const size_t* lens) {
  PipeBlocks pb;
  for (int i = 0; i < kMaxRanks; i++) {
    pb.off[i] = i < nranks ? offs[i] : 0;
    pb.len[i] = i < nranks ? lens[i] : 0;
  }
  return pb;
}
}  // namespace

const void* pipelinedAllgatherKernelPtr() { return reinterpret_cast<const void*>(pipelinedAllgatherKernel); }
const void* pipelinedAlltoallKernelPtr() { return reinterpret_cast<const void*>(pipelinedAlltoallKernel); }

const void* pipelinedReduceScatterKernelFor(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(pipeRsFn<decltype(tag)>(nranks)); });
  return k;
}

const void* castPipelinedReduceScatterKernelFor(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchHalfType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(castPipeRsFn<decltype(tag)>(nranks)); });
  return k;
}

const void* castPipelinedAllgatherKernelFor(DataType outDt) {
  const void* k = nullptr;
  dispatchHalfType(outDt, [&](auto tag) { k = reinterpret_cast<const void*>(castPipelinedAllgatherKernel<decltype(tag)>); });
  return k;
}

const void* pipelinedReduceKernelFor(DataType dt, int nranks) {
  const void* k = nullptr;
  dispatchType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(pipeReduceFn<decltype(tag)>(nranks)); });
  return k;
}

void launchPipelinedAllgather(const CommArgs& a, const void* in, void* out, const size_t* offs, const size_t* lens,
                              int onlyDst, const PeerPtrs& stage, int tileVecs, int exchangeThreads, int blocks,
                              cudaStream_t stream) {
  pipelinedAllgatherKernel<<<blocks, kThreads, 0, stream>>>(a, static_cast<const char*>(in), static_cast<char*>(out),
                                                            pipeBlocks(a.nranks, offs, lens), onlyDst, stage, tileVecs,
                                                            exchangeThreads);
}

void launchPipelinedReduceScatter(const CommArgs& a, const void* in, void* out, const size_t* elemOff,
                                  const size_t* elemLen, DataType dt, ReduceOp op, float scale, const PeerPtrs& stage,
                                  int tileVecs, int exchangeThreads, int blocks, cudaStream_t stream) {
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    pipeRsFn<T>(a.nranks)<<<blocks, kThreads, 0, stream>>>(a, static_cast<const T*>(in), static_cast<T*>(out),
                                                           pipeBlocks(a.nranks, elemOff, elemLen),
                                                           static_cast<DevOp>(op), scale, stage, tileVecs,
                                                           exchangeThreads);
  });
}

void launchCastPipelinedAllgather(const CommArgs& a, const void* in, void* out, DataType outDt, const size_t* offs,
                                  const size_t* lens, const PeerPtrs& stage, int tileVecs, int exchangeThreads,
                                  int blocks, cudaStream_t stream) {
  dispatchHalfType(outDt, [&](auto tag) {
    castPipelinedAllgatherKernel<decltype(tag)><<<blocks, kThreads, 0, stream>>>(
        a, static_cast<const char*>(in), static_cast<char*>(out), pipeBlocks(a.nranks, offs, lens), stage, tileVecs,
        exchangeThreads);
  });
}

void launchCastPipelinedReduceScatter(const CommArgs& a, const void* in, float* out, const size_t* elemOff,
                                      const size_t* elemLen, DataType dt, float scale, const PeerPtrs& stage,
                                      int tileVecs, int exchangeThreads, int blocks, cudaStream_t stream) {
  dispatchHalfType(dt, [&](auto tag) {
    using TI = decltype(tag);
    castPipeRsFn<TI>(a.nranks)<<<blocks, kThreads, 0, stream>>>(a, static_cast<const TI*>(in), out,
                                                                pipeBlocks(a.nranks, elemOff, elemLen), scale, stage,
                                                                tileVecs, exchangeThreads);
  });
}

void launchPipelinedReduce(const CommArgs& a, const void* in, void* out, const size_t* elemOff, const size_t* elemLen,
                           int root, DataType dt, ReduceOp op, const PeerPtrs& stage, int tileVecs, int exchangeThreads,
                           int blocks, cudaStream_t stream) {
  dispatchType(dt, [&](auto tag) {
    using T = decltype(tag);
    pipeReduceFn<T>(a.nranks)<<<blocks, kThreads, 0, stream>>>(a, static_cast<const T*>(in), static_cast<T*>(out),
                                                               pipeBlocks(a.nranks, elemOff, elemLen), root,
                                                               static_cast<DevOp>(op), stage, tileVecs, exchangeThreads);
  });
}

void launchPipelinedAlltoall(const CommArgs& a, const void* in, void* out, const size_t* sendOff, const size_t* sendLen,
                             const size_t* recvOff, const size_t* recvLen, const PeerPtrs& stage, int tileVecs,
                             int exchangeThreads, int blocks, cudaStream_t stream) {
  pipelinedAlltoallKernel<<<blocks, kThreads, 0, stream>>>(a, static_cast<const char*>(in), static_cast<char*>(out),
                                                           pipeBlocks(a.nranks, sendOff, sendLen),
                                                           pipeBlocks(a.nranks, recvOff, recvLen), stage, tileVecs,
                                                           exchangeThreads);
}

void preloadPipelineKernels() {
  for (DataType dt : kAllDataTypes) {
    dispatchType(dt, [](auto tag) {
      for (bool mc : {false, true}) {
        for (int nr : {0, 2, 4, 8}) touchKernel(pipeFn<decltype(tag)>(mc, nr));
      }
      for (int nr : {0, 2, 4, 8}) {
        touchKernel(pipeRsFn<decltype(tag)>(nr));
        touchKernel(pipeReduceFn<decltype(tag)>(nr));
      }
    });
  }
  for (DataType dt : kAllDataTypes) {
    dispatchHalfType(dt, [](auto tag) {
      for (int nr : {0, 2, 4, 8}) touchKernel(castPipeRsFn<decltype(tag)>(nr));
      touchKernel(castPipelinedAllgatherKernel<decltype(tag)>);
    });
  }
  touchKernel(pipelinedAllgatherKernel);
  touchKernel(pipelinedAlltoallKernel);
  cudaGetLastError();
}

}  // namespace cuda
}  // namespace glb
