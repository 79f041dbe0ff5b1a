#include "glb/math.h"

#include <immintrin.h>

#include "glb/common/logging.h"

namespace glb {

namespace {

bool cpuHasF16C() {
  static const bool v = __builtin_cpu_supports("avx2") && __builtin_cpu_supports("f16c");
  return v;
}

enum class Op { Sum, Product, Max, Min };

template <Op op>
inline float apply(float x, float y) {
  if constexpr (op == Op::Sum) return x + y;
  if constexpr (op == Op::Product) return x * y;
  if constexpr (op == Op::Max) return (y > x) ? y : x;
  return (y < x) ? y : x;
}

template <Op op>
__attribute__((target("avx2,f16c"))) inline __m256 applyV(__m256 x, __m256 y) {
  if constexpr (op == Op::Sum) return _mm256_add_ps(x, y);
  if constexpr (op == Op::Product) return _mm256_mul_ps(x, y);
  // blendv keeps x unless the comparison holds: identical NaN behaviour to the scalar form.
  if constexpr (op == Op::Max) return _mm256_blendv_ps(x, y, _mm256_cmp_ps(y, x, _CMP_GT_OQ));
  return _mm256_blendv_ps(x, y, _mm256_cmp_ps(y, x, _CMP_LT_OQ));
}

template <Op op>
__attribute__((target("avx2,f16c"))) void f16Simd(float16* c, const float16* a, const float16* b, size_t n) {
  size_t i = 0;
  for (; i + 8 <= n; i += 8) {
    __m256 va = _mm256_cvtph_ps(_mm_loadu_si128(reinterpret_cast<const __m128i*>(a + i)));
    __m256 vb = _mm256_cvtph_ps(_mm_loadu_si128(reinterpret_cast<const __m128i*>(b + i)));
    __m256 vc = applyV<op>(va, vb);
    _mm_storeu_si128(reinterpret_cast<__m128i*>(c + i), _mm256_cvtps_ph(vc, _MM_FROUND_TO_NEAREST_INT));
  }
  for (; i < n; i++) c[i] = float16(apply<op>(float(a[i]), float(b[i])));
}

template <Op op>
__attribute__((target("avx2"))) void bf16Simd(bfloat16* c, const bfloat16* a, const bfloat16* b, size_t n) {
  size_t i = 0;
  const __m256i bias = _mm256_set1_epi32(0x7fff);
  const __m256i one = _mm256_set1_epi32(1);
  for (; i + 8 <= n; i += 8) {
    __m256i ia = _mm256_slli_epi32(
        _mm256_cvtepu16_epi32(_mm_loadu_si128(reinterpret_cast<const __m128i*>(a + i))), 16);
    __m256i ib = _mm256_slli_epi32(
        _mm256_cvtepu16_epi32(_mm_loadu_si128(reinterpret_cast<const __m128i*>(b + i))), 16);
    __m256 vc = applyV<op>(_mm256_castsi256_ps(ia), _mm256_castsi256_ps(ib));
    __m256i u = _mm256_castps_si256(vc);
    // round to nearest even: u += 0x7fff + ((u >> 16) & 1)
    __m256i lsb = _mm256_and_si256(_mm256_srli_epi32(u, 16), one);
    __m256i r = _mm256_srli_epi32(_mm256_add_epi32(u, _mm256_add_epi32(bias, lsb)), 16);
    // NaN inputs: keep a quiet NaN (rounding could carry into the exponent).
    __m256 isnan = _mm256_cmp_ps(vc, vc, _CMP_UNORD_Q);
    __m256i qnan = _mm256_or_si256(_mm256_srli_epi32(u, 16), _mm256_set1_epi32(0x40));
    r = _mm256_blendv_epi8(r, qnan, _mm256_castps_si256(isnan));
    __m128i lo = _mm256_castsi256_si128(r);
    __m128i hi = _mm256_extracti128_si256(r, 1);
    _mm_storeu_si128(reinterpret_cast<__m128i*>(c + i), _mm_packus_epi32(lo, hi));
  }
  for (; i < n; i++) c[i] = bfloat16(apply<op>(float(a[i]), float(b[i])));
}

template <typename T, Op op>
void halfScalar(T* c, const T* a, const T* b, size_t n) {
  for (size_t i = 0; i < n; i++) c[i] = T(apply<op>(float(a[i]), float(b[i])));
}

template <Op op>
void f16Dispatch(void* c, const void* a, const void* b, size_t n) {
  auto* tc = static_cast<float16*>(c);
  auto* ta = static_cast<const float16*>(a);
  auto* tb = static_cast<const float16*>(b);
  if (cpuHasF16C()) {
    f16Simd<op>(tc, ta, tb, n);
  } else {
    halfScalar<float16, op>(tc, ta, tb, n);
  }
}

template <Op op>
void bf16Dispatch(void* c, const void* a, const void* b, size_t n) {
  auto* tc = static_cast<bfloat16*>(c);
  auto* ta = static_cast<const bfloat16*>(a);
  auto* tb = static_cast<const bfloat16*>(b);
  if (cpuHasF16C()) {
    bf16Simd<op>(tc, ta, tb, n);
  } else {
    halfScalar<bfloat16, op>(tc, ta, tb, n);
  }
}

}  // namespace

bool hasSimdHalf() { return cpuHasF16C(); }

template <>
void sum<float16>(void* c, const void* a, const void* b, size_t n) { f16Dispatch<Op::Sum>(c, a, b, n); }
template <>
void product<float16>(void* c, const void* a, const void* b, size_t n) { f16Dispatch<Op::Product>(c, a, b, n); }
template <>
void max<float16>(void* c, const void* a, const void* b, size_t n) { f16Dispatch<Op::Max>(c, a, b, n); }
template <>
void min<float16>(void* c, const void* a, const void* b, size_t n) { f16Dispatch<Op::Min>(c, a, b, n); }
template <>
void sum<bfloat16>(void* c, const void* a, const void* b, size_t n) { bf16Dispatch<Op::Sum>(c, a, b, n); }
template <>
void product<bfloat16>(void* c, const void* a, const void* b, size_t n) { bf16Dispatch<Op::Product>(c, a, b, n); }
template <>
void max<bfloat16>(void* c, const void* a, const void* b, size_t n) { bf16Dispatch<Op::Max>(c, a, b, n); }
template <>
void min<bfloat16>(void* c, const void* a, const void* b, size_t n) { bf16Dispatch<Op::Min>(c, a, b, n); }

void sumScalarF16(float16* c, const float16* a, const float16* b, size_t n) {
  halfScalar<float16, Op::Sum>(c, a, b, n);
}
void sumScalarBF16(bfloat16* c, const bfloat16* a, const bfloat16* b, size_t n) {
  halfScalar<bfloat16, Op::Sum>(c, a, b, n);
}

namespace {
template <typename T>
ReduceFn pick(ReduceOp op) {
  switch (op) {
    case ReduceOp::SUM: return &sum<T>;
    case ReduceOp::PRODUCT: return &product<T>;
    case ReduceOp::MAX: return &max<T>;
    case ReduceOp::MIN: return &min<T>;
    default: break;
  }
  GLB_THROW_INVALID_OPERATION_EXCEPTION("no built-in reduce function for op ", reduceOpName(op));
}
}  // namespace

ReduceFn getReduceFn(DataType dtype, ReduceOp op) {
  switch (dtype) {
    case DataType::INT8: return pick<int8_t>(op);
    case DataType::UINT8: return pick<uint8_t>(op);
    case DataType::INT16: return pick<int16_t>(op);
    case DataType::INT32: return pick<int32_t>(op);
    case DataType::UINT32: return pick<uint32_t>(op);
    case DataType::INT64: return pick<int64_t>(op);
    case DataType::UINT64: return pick<uint64_t>(op);
    case DataType::FLOAT32: return pick<float>(op);
    case DataType::FLOAT64: return pick<double>(op);
    case DataType::FLOAT16: return pick<float16>(op);
    case DataType::BFLOAT16: return pick<bfloat16>(op);
    case DataType::FLOAT8_E4M3: return pick<float8_e4m3>(op);
    case DataType::FLOAT8_E5M2: return pick<float8_e5m2>(op);
  }
  GLB_THROW_INVALID_OPERATION_EXCEPTION("unknown dtype");
}

}  // namespace glb
