// Device-side building blocks shared by every collective kernel (sm_90a):
//
//  * CommArgs / SignalPad — per-rank signal page mapped into every peer. A kernel
//    synchronises with its peers by storing a monotonically increasing epoch into
//    the peers' pads (st.release.sys) and spinning on its own pad
//    (ld.acquire.sys): this replaces the host-side stream.wait() + notification
//    Buffers of the reference (cuda_allreduce_ring_chunked.cc:177-208).
//  * 16-byte vector packs with fp32 accumulation for 16-bit and 8-bit float types and a
//    runtime reduction op (uniform branch; these kernels are link/HBM bound).
//  * multimem.* wrappers for the NVLS (NVSwitch multicast) path.
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_fp8.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <type_traits>

#include "glb/cuda/comm_types.h"
#include "glb/types.h"

namespace glb {
namespace cuda {

enum class DevOp : int { SUM = 1, PRODUCT = 2, MAX = 3, MIN = 4 };

// ---- memory-ordering primitives -------------------------------------------------

__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ uint32_t ld_relaxed_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ unsigned long long globalTimerNs() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// ---- failure detection ------------------------------------------------------------
// The reference bounds every wait with the context timeout and turns a silent peer into an
// IoException (transport/tcp/unbound_buffer.cc:52-94). The device-side equivalent: a flag
// wait that exceeds CommArgs::timeoutNs raises the abort word in every rank's pad and in a
// host-mapped status word, after which every barrier returns false at once and the kernels
// run to their end without touching anything else. PeerContext::checkHealth() turns the
// status word into the exception and poisons the context.
// The slow paths take scalars only: handing `const CommArgs&` (a kernel parameter) to a
// non-inlined function would force a copy of the whole struct into local memory in every
// kernel.
// Returns 0 when the flag arrived, kAbortTimeout when the wait timed out (the local abort
// word is raised here), kAbortPeer when somebody else had raised it.
static __device__ __noinline__ uint32_t waitFlagSlow(const uint32_t* flag, uint32_t want, uint32_t* abortWord,
                                                     unsigned long long timeoutNs) {
  const unsigned long long t0 = globalTimerNs();
  uint32_t polls = 0;
  while (static_cast<int32_t>(ld_acquire_sys(flag) - want) < 0) {
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

// After a failed wait: tell every peer (their waits end early instead of running into their
// own time-out) and the host.
__device__ __forceinline__ void reportAbort(const CommArgs& a, uint32_t code, int missingPeer) {
  if (code == kAbortTimeout) {
    a.self->abortRank = static_cast<uint32_t>(missingPeer);
    for (int r = 0; r < a.nranks; r++) {
      if (r != a.rank) st_relaxed_sys(&a.sig[r]->abort, static_cast<uint32_t>(kAbortPeer));
    }
  }
  if (a.hostStatus != nullptr && ld_relaxed_sys(a.hostStatus) == 0u) {
    st_relaxed_sys(a.hostStatus, code | (static_cast<uint32_t>(missingPeer) << 8));
  }
  __threadfence_system();
}

// Spin until *flag has reached `want` (wrap-safe). Returns false when the wait was abandoned.
__device__ __forceinline__ bool waitFlag(const CommArgs& a, const uint32_t* flag, uint32_t want, int peer) {
  if (static_cast<int32_t>(ld_acquire_sys(flag) - want) >= 0) return true;
  const uint32_t rc = waitFlagSlow(flag, want, &a.self->abort, a.timeoutNs);
  if (rc == 0u) return true;
  reportAbort(a, rc, peer);
  return false;
}

// All CTAs with the same blockIdx on every rank rendezvous. Everything the
// callers wrote before (including stores into peer memory) is visible to every
// peer's block after it returns (bar.sync + cumulative release/acquire at .sys).
// kRelease=false is for the FIRST barrier of a kernel that has not written anything a
// peer will read: "my kernel has started" needs no fence (the inputs were produced by
// earlier kernels and are already visible system-wide), which saves a MEMBAR.SYS.
// Returns false (on every thread of the CTA) when a peer did not show up in time.
template <bool kRelease = true>
__device__ __forceinline__ bool blockBarrier(const CommArgs& a, uint32_t epoch) {
  __syncthreads();
  int ok = 1;
  if (threadIdx.x < a.nranks) {
    const int peer = threadIdx.x;
    if (kRelease) {
      st_release_sys(&a.sig[peer]->flag[blockIdx.x][a.rank], epoch);
    } else {
      st_relaxed_sys(&a.sig[peer]->flag[blockIdx.x][a.rank], epoch);
    }
    ok = waitFlag(a, &a.self->flag[blockIdx.x][peer], epoch, peer) ? 1 : 0;
  }
  return __syncthreads_and(ok) != 0;
}

// Read the epoch at kernel entry (all CTAs see the same value: it only changes
// when the LAST CTA of a launch retires, after every CTA has read it).
__device__ __forceinline__ uint32_t loadEpoch(const CommArgs& a) { return ld_relaxed_sys(&a.self->epoch); }

// Called by every CTA at the very end; the last one publishes the new counters.
__device__ __forceinline__ void retire(const CommArgs& a, uint32_t barriersUsed, uint32_t stagedLaunch,
                                       uint32_t llLaunch = 0) {
  __syncthreads();
  if (threadIdx.x == 0) {
    SignalPad* me = a.self;
    // No fences: the ticket is an L2 atomic (the last CTA sees every earlier arrival) and
    // the counters are next read by the NEXT launch, after this kernel has retired.
    uint32_t ticket = atomicAdd(&me->done, 1u);
    if (ticket == gridDim.x - 1) {
      me->done = 0;
      me->epoch += barriersUsed;
      me->stageSeq += stagedLaunch;
      me->llSeq += llLaunch;
    }
  }
}

// ---- flag-in-data ("LL") lines ------------------------------------------------------
// A 16-byte line carries 8 bytes of payload and two copies of the launch's sequence
// number: {d0, seq, d1, seq}. Each 8-byte half is written atomically, so a reader that
// sees both flags equal to `seq` has both payload words; no barrier and no MEMBAR.SYS on
// the critical path (one posted store + one poll).
__device__ __forceinline__ void llStore(void* p, uint32_t d0, uint32_t d1, uint32_t seq) {
  asm volatile("st.volatile.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(d0), "r"(seq), "r"(d1), "r"(seq) : "memory");
}
__device__ __forceinline__ bool llTryLoad(const void* p, uint32_t seq, uint32_t& d0, uint32_t& d1) {
  uint32_t f0, f1;
  asm volatile("ld.volatile.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(d0), "=r"(f0), "=r"(d1), "=r"(f1) : "l"(p) : "memory");
  return f0 == seq && f1 == seq;
}
static __device__ __noinline__ uint32_t llLoadSlow(const void* p, uint32_t seq, uint32_t& d0, uint32_t& d1,
                                                   uint32_t* abortWord, unsigned long long timeoutNs) {
  const unsigned long long t0 = globalTimerNs();
  uint32_t polls = 0;
  while (!llTryLoad(p, seq, d0, d1)) {
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
__device__ __forceinline__ bool llLoad(const CommArgs& a, const void* p, uint32_t seq, uint32_t& d0, uint32_t& d1, int peer) {
  if (llTryLoad(p, seq, d0, d1)) return true;
  const uint32_t rc = llLoadSlow(p, seq, d0, d1, &a.self->abort, a.timeoutNs);
  if (rc == 0u) return true;
  reportAbort(a, rc, peer);
  return false;
}

// ---- 16-byte packs ----------------------------------------------------------------

struct alignas(16) Pack16 {
  uint32_t w[4];
};

__device__ __forceinline__ Pack16 ld128(const void* p) {
  Pack16 v;
  asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p)
               : "memory");
  return v;
}
// Streaming variants: do not allocate in L1 (peer / single-use data).
__device__ __forceinline__ Pack16 ld128_stream(const void* p) {
  Pack16 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st128(void* p, const Pack16& v) {
  asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]), "r"(v.w[2]), "r"(v.w[3])
               : "memory");
}
__device__ __forceinline__ void st128_stream(void* p, const Pack16& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.w[0]), "r"(v.w[1]),
               "r"(v.w[2]), "r"(v.w[3])
               : "memory");
}

template <typename T>
__device__ __forceinline__ T applyOp(T a, T b, DevOp op) {
  switch (op) {
    case DevOp::SUM: return a + b;
    case DevOp::PRODUCT: return a * b;
    case DevOp::MAX: return b > a ? b : a;
    default: return b < a ? b : a;
  }
}

// Accumulator traits: how one 16-byte pack of T is widened, combined, narrowed.
template <typename T>
struct PackTraits {
  static constexpr int kElems = 16 / sizeof(T);
  using Acc = T;
  struct AccPack {
    T v[kElems];
  };
  __device__ static AccPack widen(const Pack16& p) {
    AccPack a;
    const T* t = reinterpret_cast<const T*>(&p);
#pragma unroll
    for (int i = 0; i < kElems; i++) a.v[i] = t[i];
    return a;
  }
  __device__ static void combine(AccPack& a, const Pack16& p, DevOp op) {
    const T* t = reinterpret_cast<const T*>(&p);
#pragma unroll
    for (int i = 0; i < kElems; i++) a.v[i] = applyOp<T>(a.v[i], t[i], op);
  }
  __device__ static Pack16 narrow(const AccPack& a) {
    Pack16 p;
    T* t = reinterpret_cast<T*>(&p);
#pragma unroll
    for (int i = 0; i < kElems; i++) t[i] = a.v[i];
    return p;
  }
  __device__ static T one(const T* p) { return *p; }
  __device__ static T combineOne(T a, T b, DevOp op) { return applyOp<T>(a, b, op); }
  // Epilogue: multiply the reduced value (floating types only; the host rejects a scale
  // on integer buffers).
  __device__ static void scale(AccPack& a, float s) {
    if constexpr (std::is_floating_point<T>::value) {
#pragma unroll
      for (int i = 0; i < kElems; i++) a.v[i] = static_cast<T>(a.v[i] * s);
    }
  }
  __device__ static T scaleOne(T a, float s) {
    if constexpr (std::is_floating_point<T>::value) return static_cast<T>(a * s);
    return a;
  }
};

template <>
struct PackTraits<__half> {
  static constexpr int kElems = 8;
  struct AccPack {
    float v[8];
  };
  __device__ static AccPack widen(const Pack16& p) {
    AccPack a;
    const __half2* h = reinterpret_cast<const __half2*>(&p);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float2 f = __half22float2(h[i]);
      a.v[2 * i] = f.x;
      a.v[2 * i + 1] = f.y;
    }
    return a;
  }
  __device__ static void combine(AccPack& a, const Pack16& p, DevOp op) {
    const __half2* h = reinterpret_cast<const __half2*>(&p);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float2 f = __half22float2(h[i]);
      a.v[2 * i] = applyOp<float>(a.v[2 * i], f.x, op);
      a.v[2 * i + 1] = applyOp<float>(a.v[2 * i + 1], f.y, op);
    }
  }
  __device__ static Pack16 narrow(const AccPack& a) {
    Pack16 p;
    __half2* h = reinterpret_cast<__half2*>(&p);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2half2_rn(a.v[2 * i], a.v[2 * i + 1]);
    return p;
  }
  __device__ static __half combineOne(__half a, __half b, DevOp op) {
    return __float2half_rn(applyOp<float>(__half2float(a), __half2float(b), op));
  }
  __device__ static void scale(AccPack& a, float s) {
#pragma unroll
    for (int i = 0; i < 8; i++) a.v[i] *= s;
  }
  __device__ static __half scaleOne(__half a, float s) { return __float2half_rn(__half2float(a) * s); }
};

template <>
struct PackTraits<__nv_bfloat16> {
  static constexpr int kElems = 8;
  struct AccPack {
    float v[8];
  };
  __device__ static AccPack widen(const Pack16& p) {
    AccPack a;
    // bf16 -> fp32 is a 16-bit shift.
#pragma unroll
    for (int i = 0; i < 4; i++) {
      a.v[2 * i] = __uint_as_float(p.w[i] << 16);
      a.v[2 * i + 1] = __uint_as_float(p.w[i] & 0xffff0000u);
    }
    return a;
  }
  __device__ static void combine(AccPack& a, const Pack16& p, DevOp op) {
#pragma unroll
    for (int i = 0; i < 4; i++) {
      a.v[2 * i] = applyOp<float>(a.v[2 * i], __uint_as_float(p.w[i] << 16), op);
      a.v[2 * i + 1] = applyOp<float>(a.v[2 * i + 1], __uint_as_float(p.w[i] & 0xffff0000u), op);
    }
  }
  __device__ static Pack16 narrow(const AccPack& a) {
    Pack16 p;
    __nv_bfloat162* h = reinterpret_cast<__nv_bfloat162*>(&p);
#pragma unroll
    for (int i = 0; i < 4; i++) h[i] = __floats2bfloat162_rn(a.v[2 * i], a.v[2 * i + 1]);
    return p;
  }
  __device__ static __nv_bfloat16 combineOne(__nv_bfloat16 a, __nv_bfloat16 b, DevOp op) {
    return __float2bfloat16_rn(applyOp<float>(__bfloat162float(a), __bfloat162float(b), op));
  }
  __device__ static void scale(AccPack& a, float s) {
#pragma unroll
    for (int i = 0; i < 8; i++) a.v[i] *= s;
  }
  __device__ static __nv_bfloat16 scaleOne(__nv_bfloat16 a, float s) {
    return __float2bfloat16_rn(__bfloat162float(a) * s);
  }
};

// FP8 (e4m3 / e5m2): 16 lanes per pack, fp32 accumulator. Widening is exact (fp8 -> f16x2 ->
// f32x2); narrowing rounds to nearest even and saturates to +-max finite
// (cvt.rn.satfinite.{e4m3,e5m2}x2.f32, the only fp32 -> fp8 conversion on sm_90a).
template <typename T>
struct Fp8Format;
template <>
struct Fp8Format<__nv_fp8_e4m3> {
  static constexpr __nv_fp8_interpretation_t value = __NV_E4M3;
};
template <>
struct Fp8Format<__nv_fp8_e5m2> {
  static constexpr __nv_fp8_interpretation_t value = __NV_E5M2;
};

template <typename T>
__device__ __forceinline__ float2 fp8x2ToFloat2(uint32_t x2) {
  const __half2 h = __half2(__nv_cvt_fp8x2_to_halfraw2(static_cast<__nv_fp8x2_storage_t>(x2), Fp8Format<T>::value));
  return __half22float2(h);
}
template <typename T>
__device__ __forceinline__ uint32_t float2ToFp8x2(float a, float b) {
  return __nv_cvt_float2_to_fp8x2(make_float2(a, b), __NV_SATFINITE, Fp8Format<T>::value);
}
template <typename T>
__device__ __forceinline__ float fp8ToFloat(T x) {
  return __half2float(__half(__nv_cvt_fp8_to_halfraw(x.__x, Fp8Format<T>::value)));
}
template <typename T>
__device__ __forceinline__ T floatToFp8(float x) {
  T r;
  r.__x = __nv_cvt_float_to_fp8(x, __NV_SATFINITE, Fp8Format<T>::value);
  return r;
}

// One element of T as its fp32 value (16-bit and FP8 types) or as itself (every other type),
// and back: widening is exact, narrowing rounds to nearest even (FP8 also saturates).
template <typename T>
struct Scalar {
  using Acc = T;
  __device__ static T toAcc(T x) { return x; }
  __device__ static T fromAcc(T x) { return x; }
};
template <>
struct Scalar<__half> {
  using Acc = float;
  __device__ static float toAcc(__half x) { return __half2float(x); }
  __device__ static __half fromAcc(float x) { return __float2half_rn(x); }
};
template <>
struct Scalar<__nv_bfloat16> {
  using Acc = float;
  __device__ static float toAcc(__nv_bfloat16 x) { return __bfloat162float(x); }
  __device__ static __nv_bfloat16 fromAcc(float x) { return __float2bfloat16_rn(x); }
};
template <typename T>
struct Fp8Scalar {
  using Acc = float;
  __device__ static float toAcc(T x) { return fp8ToFloat(x); }
  __device__ static T fromAcc(float x) { return floatToFp8<T>(x); }
};
template <>
struct Scalar<__nv_fp8_e4m3> : Fp8Scalar<__nv_fp8_e4m3> {};
template <>
struct Scalar<__nv_fp8_e5m2> : Fp8Scalar<__nv_fp8_e5m2> {};

template <typename T>
struct Fp8PackTraits {
  static constexpr int kElems = 16;
  struct AccPack {
    float v[16];
  };
  __device__ static AccPack widen(const Pack16& p) {
    AccPack a;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const float2 lo = fp8x2ToFloat2<T>(p.w[i] & 0xffffu), hi = fp8x2ToFloat2<T>(p.w[i] >> 16);
      a.v[4 * i] = lo.x;
      a.v[4 * i + 1] = lo.y;
      a.v[4 * i + 2] = hi.x;
      a.v[4 * i + 3] = hi.y;
    }
    return a;
  }
  __device__ static void combine(AccPack& a, const Pack16& p, DevOp op) {
    // two lanes at a time: widening the whole pack first keeps 16 more registers live
#pragma unroll
    for (int i = 0; i < 8; i++) {
      const float2 f = fp8x2ToFloat2<T>((p.w[i / 2] >> (16 * (i % 2))) & 0xffffu);
      a.v[2 * i] = applyOp<float>(a.v[2 * i], f.x, op);
      a.v[2 * i + 1] = applyOp<float>(a.v[2 * i + 1], f.y, op);
    }
  }
  __device__ static Pack16 narrow(const AccPack& a) {
    Pack16 p;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      p.w[i] = float2ToFp8x2<T>(a.v[4 * i], a.v[4 * i + 1]) | (float2ToFp8x2<T>(a.v[4 * i + 2], a.v[4 * i + 3]) << 16);
    }
    return p;
  }
  __device__ static T combineOne(T a, T b, DevOp op) {
    return floatToFp8<T>(applyOp<float>(fp8ToFloat(a), fp8ToFloat(b), op));
  }
  __device__ static void scale(AccPack& a, float s) {
#pragma unroll
    for (int i = 0; i < 16; i++) a.v[i] *= s;
  }
  __device__ static T scaleOne(T a, float s) { return floatToFp8<T>(fp8ToFloat(a) * s); }
};
template <>
struct PackTraits<__nv_fp8_e4m3> : Fp8PackTraits<__nv_fp8_e4m3> {};
template <>
struct PackTraits<__nv_fp8_e5m2> : Fp8PackTraits<__nv_fp8_e5m2> {};

template <typename T>
constexpr bool isFp8Type() {
  return std::is_same<T, __nv_fp8_e4m3>::value || std::is_same<T, __nv_fp8_e5m2>::value;
}

// Quantisation to e4m3 codes with one fp32 scale per block of values (the MoE FP8 dispatch: 1 x
// 128 blocks; the fused residual norm's FP8 out: one block per row). Numerics: amax = max(max |x|,
// 1e-4f); code = e4m3(x * (448 * (1 / amax))) (round to nearest even, saturating); scale = amax /
// 448, each step a correctly rounded fp32 operation (no contraction, no approximate division). The
// multiplier is a rounded reciprocal times 448, not a rounded 448 / amax: that is what torch
// evaluates for `448.0 / amax` (a scalar over a tensor), so torch code reproduces every byte.
constexpr float kE4m3Max = 448.0f;
constexpr float kQuantMinAmax = 1e-4f;

// The block's amax from the largest |x| of its values.
__device__ __forceinline__ float quantAmax(float absMax) { return fmaxf(absMax, kQuantMinAmax); }
// The multiplier that takes the block's values to codes.
__device__ __forceinline__ float e4m3Multiplier(float amax) { return __fmul_rn(__frcp_rn(amax), kE4m3Max); }
// Two values to two codes (low byte: a).
__device__ __forceinline__ uint32_t e4m3Codes2(float a, float b, float multiplier) {
  return float2ToFp8x2<__nv_fp8_e4m3>(__fmul_rn(a, multiplier), __fmul_rn(b, multiplier));
}
// The block's scale: x ~= code * scale.
__device__ __forceinline__ float e4m3Scale(float amax) { return __fdiv_rn(amax, kE4m3Max); }

// Scalar tails (elements after the last whole pack). 16-bit and FP8 types accumulate them in
// fp32, scale in fp32 and round once, like their packs; every other type accumulates in itself.
template <typename T>
struct TailAcc {
  using type = T;
  __device__ static T load(T x) { return x; }
  __device__ static T store(T x) { return x; }
  __device__ static T combine(T a, T b, DevOp op) { return PackTraits<T>::combineOne(a, b, op); }
  __device__ static T scale(T a, float s) { return PackTraits<T>::scaleOne(a, s); }
};
template <typename T>
struct Fp32TailAcc {
  using type = float;
  __device__ static float load(T x) { return Scalar<T>::toAcc(x); }
  __device__ static T store(float x) { return Scalar<T>::fromAcc(x); }
  __device__ static float combine(float a, float b, DevOp op) { return applyOp<float>(a, b, op); }
  __device__ static float scale(float a, float s) { return a * s; }
};
template <>
struct TailAcc<__half> : Fp32TailAcc<__half> {};
template <>
struct TailAcc<__nv_bfloat16> : Fp32TailAcc<__nv_bfloat16> {};
template <>
struct TailAcc<__nv_fp8_e4m3> : Fp32TailAcc<__nv_fp8_e4m3> {};
template <>
struct TailAcc<__nv_fp8_e5m2> : Fp32TailAcc<__nv_fp8_e5m2> {};
// Element types that get the P-specialised (two-shot, pipelined, reduce-pull) instantiations.
template <typename T>
constexpr bool isHotType() {
  return std::is_same<T, float>::value || std::is_same<T, __half>::value || std::is_same<T, __nv_bfloat16>::value ||
         isFp8Type<T>();
}
// Element types multimem.ld_reduce can add on sm_90a (NVLS, hybrid, multicast pipelines).
// It has no e4m3 / e5m2 form on this target, so FP8 never takes those paths.
template <typename T>
constexpr bool hasMultimem() {
  return std::is_same<T, float>::value || std::is_same<T, __half>::value || std::is_same<T, __nv_bfloat16>::value;
}

// ---- mixed-precision items (cast epilogue) --------------------------------------------
// Eight consecutive elements of T as fp32 lanes: 2 x 16 B for float, 1 x 16 B for the
// 16-bit types. Used by the kernels whose output dtype differs from the input dtype
// (fp32 accumulate -> bf16/fp16 store, or 16-bit inputs -> fp32 result).
template <typename T>
struct Item8;
template <>
struct Item8<float> {
  static constexpr int kBytes = 32;
  __device__ static void load(const void* p, float (&v)[8]) {
    const Pack16 a = ld128_stream(p), b = ld128_stream(static_cast<const char*>(p) + 16);
#pragma unroll
    for (int i = 0; i < 4; i++) {
      v[i] = __uint_as_float(a.w[i]);
      v[4 + i] = __uint_as_float(b.w[i]);
    }
  }
  __device__ static void store(void* p, const float (&v)[8]) {
    Pack16 a, b;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      a.w[i] = __float_as_uint(v[i]);
      b.w[i] = __float_as_uint(v[4 + i]);
    }
    st128_stream(p, a);
    st128_stream(static_cast<char*>(p) + 16, b);
  }
};
template <>
struct Item8<__half> {
  static constexpr int kBytes = 16;
  __device__ static void load(const void* p, float (&v)[8]) {
    const auto a = PackTraits<__half>::widen(ld128_stream(p));
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = a.v[i];
  }
  __device__ static void store(void* p, const float (&v)[8]) {
    PackTraits<__half>::AccPack a;
#pragma unroll
    for (int i = 0; i < 8; i++) a.v[i] = v[i];
    st128_stream(p, PackTraits<__half>::narrow(a));
  }
};
template <>
struct Item8<__nv_bfloat16> {
  static constexpr int kBytes = 16;
  __device__ static void load(const void* p, float (&v)[8]) {
    const auto a = PackTraits<__nv_bfloat16>::widen(ld128_stream(p));
#pragma unroll
    for (int i = 0; i < 8; i++) v[i] = a.v[i];
  }
  __device__ static void store(void* p, const float (&v)[8]) {
    PackTraits<__nv_bfloat16>::AccPack a;
#pragma unroll
    for (int i = 0; i < 8; i++) a.v[i] = v[i];
    st128_stream(p, PackTraits<__nv_bfloat16>::narrow(a));
  }
};

// FP8: 8 elements are 8 bytes (one 64-bit access).
template <typename T>
struct Fp8Item8 {
  static constexpr int kBytes = 8;
  __device__ static void load(const void* p, float (&v)[8]) {
    const uint2 x = *static_cast<const uint2*>(p);
    const uint32_t w[2] = {x.x, x.y};
#pragma unroll
    for (int i = 0; i < 2; i++) {
      const float2 lo = fp8x2ToFloat2<T>(w[i] & 0xffffu), hi = fp8x2ToFloat2<T>(w[i] >> 16);
      v[4 * i] = lo.x;
      v[4 * i + 1] = lo.y;
      v[4 * i + 2] = hi.x;
      v[4 * i + 3] = hi.y;
    }
  }
  __device__ static void store(void* p, const float (&v)[8]) {
    uint2 x;
    x.x = float2ToFp8x2<T>(v[0], v[1]) | (float2ToFp8x2<T>(v[2], v[3]) << 16);
    x.y = float2ToFp8x2<T>(v[4], v[5]) | (float2ToFp8x2<T>(v[6], v[7]) << 16);
    *static_cast<uint2*>(p) = x;
  }
};
template <>
struct Item8<__nv_fp8_e4m3> : Fp8Item8<__nv_fp8_e4m3> {};
template <>
struct Item8<__nv_fp8_e5m2> : Fp8Item8<__nv_fp8_e5m2> {};

// ---- NVLS (multimem) --------------------------------------------------------------
// ld_reduce returns the reduction of the same address across every GPU bound to
// the multicast object (performed inside the NVSwitch); st broadcasts to all.

template <typename T>
struct Multimem;  // only add for float / half / bf16 (see hasMultimem)

template <>
struct Multimem<float> {
  __device__ static Pack16 ldReduceAdd(const void* mc) {
    Pack16 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(mc)
                 : "memory");
    return v;
  }
};
template <>
struct Multimem<__half> {
  __device__ static Pack16 ldReduceAdd(const void* mc) {
    Pack16 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(mc)
                 : "memory");
    return v;
  }
};
template <>
struct Multimem<__nv_bfloat16> {
  __device__ static Pack16 ldReduceAdd(const void* mc) {
    Pack16 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.w[0]), "=r"(v.w[1]), "=r"(v.w[2]), "=r"(v.w[3])
                 : "l"(mc)
                 : "memory");
    return v;
  }
};

__device__ __forceinline__ void multimemSt128(void* mc, const Pack16& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.w[0]), "r"(v.w[1]),
               "r"(v.w[2]), "r"(v.w[3])
               : "memory");
}

// ---- host side: dtype dispatch and kernel preloading ----------------------------------

// Calls f(T{}) with the device element type T of dt. Each kernel family picks its
// instantiation from T in one selector, which the launcher, the occupancy query and the
// preload all call.
template <typename F>
void dispatchType(DataType dt, F&& f) {
  switch (dt) {
    case DataType::INT8: f(int8_t{}); break;
    case DataType::UINT8: f(uint8_t{}); break;
    case DataType::INT16: f(int16_t{}); break;
    case DataType::INT32: f(int32_t{}); break;
    case DataType::UINT32: f(uint32_t{}); break;
    case DataType::INT64: f(0LL); break;
    case DataType::UINT64: f(0ULL); break;
    case DataType::FLOAT32: f(float{}); break;
    case DataType::FLOAT64: f(double{}); break;
    case DataType::FLOAT16: f(__half{}); break;
    case DataType::BFLOAT16: f(__nv_bfloat16{}); break;
    case DataType::FLOAT8_E4M3: f(__nv_fp8_e4m3{}); break;
    case DataType::FLOAT8_E5M2: f(__nv_fp8_e5m2{}); break;
  }
}

// Calls f(T{}) when dt is a 16-bit floating type (float16, bfloat16); returns whether it is one.
// The cast reduce-scatter and allgather take these on their 16-bit side.
template <typename F>
bool dispatchHalfType(DataType dt, F&& f) {
  if (dt == DataType::FLOAT16) {
    f(__half{});
  } else if (dt == DataType::BFLOAT16) {
    f(__nv_bfloat16{});
  } else {
    return false;
  }
  return true;
}

constexpr DataType kAllDataTypes[] = {DataType::INT8,    DataType::UINT8,       DataType::INT16,      DataType::INT32,
                                      DataType::UINT32,  DataType::INT64,       DataType::UINT64,     DataType::FLOAT32,
                                      DataType::FLOAT64, DataType::FLOAT16,     DataType::BFLOAT16,   DataType::FLOAT8_E4M3,
                                      DataType::FLOAT8_E5M2};

// Force-load one kernel. With CUDA's lazy module loading the first launch of a kernel may
// have to synchronise the context; if a peer rank on the same device is already spinning
// inside its collective kernel, that launch never happens (DESIGN.md, "Running ranks that
// share one GPU"). So the preload*Kernels() functions touch every kernel a launcher can start,
// by calling each selector over its whole domain (a selector returns nullptr for arguments
// that have no kernel).
template <typename K>
void touchKernel(K kernel) {
  if (kernel == nullptr) return;
  cudaFuncAttributes attr;
  cudaFuncGetAttributes(&attr, reinterpret_cast<const void*>(kernel));
}

}  // namespace cuda
}  // namespace glb
