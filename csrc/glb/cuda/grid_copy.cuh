// Byte copies by a team of threads (a whole grid, or one warp group of a CTA): `tid` is the
// thread's index in the team, `nthreads` the team's size.
#pragma once

#include "glb/cuda/device_common.cuh"

namespace glb {
namespace cuda {

template <typename W>
__device__ __forceinline__ void gridCopyWords(char* dst, const char* src, size_t bytes, size_t tid, size_t nthreads) {
  const size_t n = bytes / sizeof(W);
  constexpr int U = 4;
  for (size_t i0 = tid; i0 < n; i0 += nthreads * U) {
    W w[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + u * nthreads;
      if (i < n) w[u] = reinterpret_cast<const W*>(src)[i];
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + u * nthreads;
      if (i < n) reinterpret_cast<W*>(dst)[i] = w[u];
    }
  }
  for (size_t i = n * sizeof(W) + tid; i < bytes; i += nthreads) dst[i] = src[i];
}

// 16 bytes from a source that is only W-byte aligned (W = 8 or 4), as one pack.
template <typename W>
__device__ __forceinline__ Pack16 ldPackWords(const char* src) {
  Pack16 p;
  W* w = reinterpret_cast<W*>(&p);
#pragma unroll
  for (int i = 0; i < static_cast<int>(16 / sizeof(W)); i++) w[i] = reinterpret_cast<const W*>(src)[i];
  return p;
}

template <typename W>
__device__ __forceinline__ void gridCopyBody(char* dst, const char* src, size_t nvec, size_t tid, size_t nthreads) {
  constexpr int U = 4;
  for (size_t v0 = tid; v0 < nvec; v0 += nthreads * U) {
    Pack16 p[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * nthreads;
      if (v < nvec) {
        if constexpr (sizeof(W) == 16) {
          p[u] = ld128_stream(src + v * 16);
        } else {
          p[u] = ldPackWords<W>(src + v * 16);
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * nthreads;
      if (v < nvec) st128_stream(dst + v * 16, p[u]);
    }
  }
}

// Body copy for a source that is 4-byte (not 8-byte) congruent with the 16-byte aligned
// destination: instead of four 4-byte loads per pack, load the two ALIGNED packs that straddle
// it and pick the words (the second load of one pack is the first load of the next and hits L1/L2).
// The first and last pack use word loads so that no byte outside [src, src + 16 * nvec) is read.
__device__ __forceinline__ void gridCopyBodyShifted(char* dst, const char* src, size_t nvec, size_t tid, size_t nthreads) {
  const int shift = static_cast<int>((reinterpret_cast<uintptr_t>(src) % 16) / 4);  // 1..3 words
  const char* base = src - shift * 4;                                                // 16-byte aligned
  if (tid == 0 && nvec > 0) st128_stream(dst, ldPackWords<unsigned int>(src));
  if (tid == 1 % nthreads && nvec > 1) st128_stream(dst + (nvec - 1) * 16, ldPackWords<unsigned int>(src + (nvec - 1) * 16));
  constexpr int U = 4;
  for (size_t v0 = 1 + tid; v0 + 1 < nvec; v0 += nthreads * U) {
    Pack16 lo[U], hi[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * nthreads;
      if (v + 1 < nvec) {
        lo[u] = ld128(base + v * 16);
        hi[u] = ld128(base + v * 16 + 16);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t v = v0 + u * nthreads;
      if (v + 1 < nvec) {
        Pack16 o;
        if (shift == 1) {
          o.w[0] = lo[u].w[1]; o.w[1] = lo[u].w[2]; o.w[2] = lo[u].w[3]; o.w[3] = hi[u].w[0];
        } else if (shift == 2) {
          o.w[0] = lo[u].w[2]; o.w[1] = lo[u].w[3]; o.w[2] = hi[u].w[0]; o.w[3] = hi[u].w[1];
        } else {
          o.w[0] = lo[u].w[3]; o.w[1] = hi[u].w[0]; o.w[2] = hi[u].w[1]; o.w[3] = hi[u].w[2];
        }
        st128_stream(dst + v * 16, o);
      }
    }
  }
}

// Copy `bytes` from src to dst with the whole grid. The DESTINATION side (usually a peer,
// i.e. NVLink stores) always moves in 128-bit stores: a byte-wise head brings dst to a
// 16-byte boundary, the body loads with the widest access the (local) source allows at
// that point (16 / 8 / 4 bytes) and a byte-wise tail finishes. Only sources that are
// not even 4-byte congruent with the destination fall back to narrow word copies.
__device__ __forceinline__ void gridCopy(char* dst, const char* src, size_t bytes, bool /*vecHint*/, size_t tid,
                                         size_t nthreads) {
  const size_t mis = reinterpret_cast<uintptr_t>(dst) % 16;
  size_t head = mis ? 16 - mis : 0;
  if (head > bytes) head = bytes;
  const uintptr_t srcBody = reinterpret_cast<uintptr_t>(src + head) % 16;
  if (srcBody % 4 != 0) {
    const uintptr_t both = reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(src);
    if (both % 2 == 0) {
      gridCopyWords<unsigned short>(dst, src, bytes, tid, nthreads);
    } else {
      for (size_t i = tid; i < bytes; i += nthreads) dst[i] = src[i];
    }
    return;
  }
  for (size_t i = tid; i < head; i += nthreads) dst[i] = src[i];
  const size_t nvec = (bytes - head) / 16;
  if (srcBody == 0) {
    gridCopyBody<Pack16>(dst + head, src + head, nvec, tid, nthreads);
  } else if (srcBody % 8 == 0) {
    gridCopyBody<unsigned long long>(dst + head, src + head, nvec, tid, nthreads);
  } else {
    gridCopyBodyShifted(dst + head, src + head, nvec, tid, nthreads);
  }
  for (size_t i = head + nvec * 16 + tid; i < bytes; i += nthreads) dst[i] = src[i];
}

}  // namespace cuda
}  // namespace glb
