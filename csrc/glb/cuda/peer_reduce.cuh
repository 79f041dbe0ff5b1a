// The inner loops of every kernel that reduces 16-byte packs pulled from the peers (sm_90a).
#pragma once

#include "glb/cuda/device_common.cuh"

namespace glb {
namespace cuda {

// Reduces packs [begin, end) with stride `stride` over P peers: pack o of rotated peer q is at
// peer(q) + o * 16. Each result is widened to the PackTraits accumulator in peer order, scaled,
// rounded once and handed to sink(o, pack). With kNarrow false the scaled accumulator itself
// (PackTraits<T>::AccPack, fp32 lanes for the 16-bit types) goes to the sink, unrounded.
//
// kSlots >= P is the number of peers the code is written for (kMaxRanks for any P). With
// kBatch == 0 each thread keeps kSlots x U independent 128-bit loads in flight, as many as it can
// afford (an NVLink round trip is ~2 us); with kBatch > 0 it reduces one pack at a time and loads
// the peers' packs in batches of kBatch, in the same order, which bounds the registers at any P.
template <typename T, int kSlots, int U, int kBatch, bool kNarrow = true, typename Peer, typename Sink>
__device__ __forceinline__ void reducePeers(int P, size_t begin, size_t end, size_t stride, DevOp op, float scale,
                                            Peer&& peer, Sink&& sink) {
  using PT = PackTraits<T>;
  if constexpr (kBatch > 0) {
    for (size_t o = begin; o < end; o += stride) {
      typename PT::AccPack acc;
#pragma unroll
      for (int b0 = 0; b0 < kSlots; b0 += kBatch) {
        Pack16 v[kBatch];
#pragma unroll
        for (int q = 0; q < kBatch; q++) {
          if (b0 + q < P) v[q] = ld128_stream(peer(b0 + q) + o * 16);
        }
#pragma unroll
        for (int q = 0; q < kBatch; q++) {
          if (b0 + q == 0) {
            acc = PT::widen(v[q]);
          } else if (b0 + q < P) {
            PT::combine(acc, v[q], op);
          }
        }
      }
      if (scale != 1.0f) PT::scale(acc, scale);
      if constexpr (kNarrow) {
        sink(o, PT::narrow(acc));
      } else {
        sink(o, acc);
      }
    }
  } else {
    for (size_t o0 = begin; o0 < end; o0 += stride * U) {
      Pack16 v[U][kSlots];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t o = o0 + static_cast<size_t>(u) * stride;
        if (o < end) {
#pragma unroll
          for (int q = 0; q < kSlots; q++) {
            if (q < P) v[u][q] = ld128_stream(peer(q) + o * 16);
          }
        }
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t o = o0 + static_cast<size_t>(u) * stride;
        if (o < end) {
          typename PT::AccPack acc = PT::widen(v[u][0]);
#pragma unroll
          for (int q = 1; q < kSlots; q++) {
            if (q < P) PT::combine(acc, v[u][q], op);
          }
          if (scale != 1.0f) PT::scale(acc, scale);
          if constexpr (kNarrow) {
            sink(o, PT::narrow(acc));
          } else {
            sink(o, acc);
          }
        }
      }
    }
  }
}

template <typename T>
__device__ __forceinline__ Pack16 scalePack(const Pack16& p, float s) {
  using PT = PackTraits<T>;
  typename PT::AccPack acc = PT::widen(p);
  PT::scale(acc, s);
  return PT::narrow(acc);
}

// Packs [begin, end) with stride `stride` of a multicast range: multimem.ld_reduce (a SUM inside the
// NVSwitch), U loads in flight per thread, scaled, handed to sink(v, pack).
template <typename T, int U, typename Sink>
__device__ __forceinline__ void reduceMultimem(const char* mc, size_t begin, size_t end, size_t stride, float scale,
                                               Sink&& sink) {
  for (size_t v0 = begin; v0 < end; v0 += stride * U) {
    Pack16 r[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + static_cast<size_t>(u) * stride;
      if (v < end) r[u] = Multimem<T>::ldReduceAdd(mc + v * 16);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + static_cast<size_t>(u) * stride;
      if (v < end) sink(v, scale != 1.0f ? scalePack<T>(r[u], scale) : r[u]);
    }
  }
}

}  // namespace cuda
}  // namespace glb
