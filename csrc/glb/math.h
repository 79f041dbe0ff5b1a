// Host reduction kernels. Every function computes c[i] = a[i] (op) b[i]; `c` may
// alias `a` (the in-place form the collectives use). Typed templates for the
// old-style API plus a (dtype, op) -> function-pointer table for the new-style
// API whose reduce callback is type-erased.
//
// float16 / bfloat16 go through fp32; when the CPU has AVX2+F16C the 16-bit paths
// run 8 lanes at a time (runtime-dispatched, so the binary still runs on CPUs
// without them). float8_e4m3 / float8_e5m2 use the generic scalar templates below: every
// element is widened to fp32, combined, and rounded back (RNE, saturating). Parity: gloo/math.h:15-95, math.cc:17-98.
#pragma once

#include <cstddef>

#include "glb/types.h"

namespace glb {

using ReduceFn = void (*)(void* c, const void* a, const void* b, size_t n);

template <typename T>
void sum(void* c, const void* a, const void* b, size_t n) {
  T* tc = static_cast<T*>(c);
  const T* ta = static_cast<const T*>(a);
  const T* tb = static_cast<const T*>(b);
  for (size_t i = 0; i < n; i++) tc[i] = ta[i] + tb[i];
}

template <typename T>
void product(void* c, const void* a, const void* b, size_t n) {
  T* tc = static_cast<T*>(c);
  const T* ta = static_cast<const T*>(a);
  const T* tb = static_cast<const T*>(b);
  for (size_t i = 0; i < n; i++) tc[i] = ta[i] * tb[i];
}

template <typename T>
void max(void* c, const void* a, const void* b, size_t n) {
  T* tc = static_cast<T*>(c);
  const T* ta = static_cast<const T*>(a);
  const T* tb = static_cast<const T*>(b);
  for (size_t i = 0; i < n; i++) tc[i] = (tb[i] > ta[i]) ? tb[i] : ta[i];
}

template <typename T>
void min(void* c, const void* a, const void* b, size_t n) {
  T* tc = static_cast<T*>(c);
  const T* ta = static_cast<const T*>(a);
  const T* tb = static_cast<const T*>(b);
  for (size_t i = 0; i < n; i++) tc[i] = (tb[i] < ta[i]) ? tb[i] : ta[i];
}

// 16-bit specialisations (SIMD when available).
template <>
void sum<float16>(void* c, const void* a, const void* b, size_t n);
template <>
void product<float16>(void* c, const void* a, const void* b, size_t n);
template <>
void max<float16>(void* c, const void* a, const void* b, size_t n);
template <>
void min<float16>(void* c, const void* a, const void* b, size_t n);
template <>
void sum<bfloat16>(void* c, const void* a, const void* b, size_t n);
template <>
void product<bfloat16>(void* c, const void* a, const void* b, size_t n);
template <>
void max<bfloat16>(void* c, const void* a, const void* b, size_t n);
template <>
void min<bfloat16>(void* c, const void* a, const void* b, size_t n);

// Scalar reference versions of the 16-bit ops (used by tests to validate SIMD).
void sumScalarF16(float16* c, const float16* a, const float16* b, size_t n);
void sumScalarBF16(bfloat16* c, const bfloat16* a, const bfloat16* b, size_t n);

// True when the SIMD 16-bit paths are active on this CPU.
bool hasSimdHalf();

// Lookup for the type-erased API. Throws for CUSTOM.
ReduceFn getReduceFn(DataType dtype, ReduceOp op);

}  // namespace glb
