// Fundamental value types: Slot (64-bit message tag algebra), float16 / bfloat16 /
// float8_e4m3 / float8_e5m2 (host-side storage types with software conversion),
// DataType / ReduceOp enums shared by the host and CUDA paths.
// Parity: gloo/types.h:40-335, types.cc:16-32.
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <iosfwd>
#include <limits>
#include <type_traits>

#ifdef __CUDACC__
#define GLB_HOST_DEVICE __host__ __device__
#else
#define GLB_HOST_DEVICE
#endif

namespace glb {

// ---- Slot -------------------------------------------------------------------
// Layout: [ prefix:8 | tag:32 | delta:24 ].
// `prefix` identifies the collective family, `tag` is the user tag that lets
// concurrent collectives share a context, `delta` is consumed by `slot + n`
// inside an algorithm (per-step / per-segment sub-channels). The reference
// reserves only 8 bits for delta (types.h:76-91); we widen it to 24 so deep
// pipelines (many segments in flight) never alias, and still throw on overflow.
constexpr uint8_t kGatherSlotPrefix = 0x01;
constexpr uint8_t kAllgatherSlotPrefix = 0x02;
constexpr uint8_t kReduceSlotPrefix = 0x03;
constexpr uint8_t kAllreduceSlotPrefix = 0x04;
constexpr uint8_t kScatterSlotPrefix = 0x05;
constexpr uint8_t kBroadcastSlotPrefix = 0x06;
constexpr uint8_t kBarrierSlotPrefix = 0x07;
constexpr uint8_t kAlltoallSlotPrefix = 0x08;
constexpr uint8_t kReduceScatterSlotPrefix = 0x09;
constexpr uint8_t kInternalSlotPrefix = 0x7f;  // context factory, key exchange, ...

class Slot {
 public:
  static constexpr int kDeltaBits = 24;
  static constexpr uint64_t kDeltaMask = (1ull << kDeltaBits) - 1;

  static Slot build(uint8_t prefix, uint32_t tag);

  operator uint64_t() const { return base_ + delta_; }
  // slot + n: throws EnforceNotMet when delta overflows. Templated so that every
  // integral type binds here rather than to the built-in operator via uint64_t().
  template <typename I, typename = typename std::enable_if<std::is_integral<I>::value>::type>
  Slot operator+(I i) const {
    return add(static_cast<uint64_t>(i));
  }
  uint8_t prefix() const { return static_cast<uint8_t>(base_ >> 56); }
  uint32_t tag() const { return static_cast<uint32_t>((base_ >> kDeltaBits) & 0xffffffffu); }
  uint64_t delta() const { return delta_; }

 private:
  Slot add(uint64_t i) const;
  explicit Slot(uint64_t base, uint64_t delta) : base_(base), delta_(delta) {}
  const uint64_t base_;
  const uint64_t delta_;
};

// ---- 16-bit float storage types ----------------------------------------------
namespace detail {
GLB_HOST_DEVICE inline uint32_t f2u(float f) {
  uint32_t u;
#ifdef __CUDA_ARCH__
  u = __float_as_uint(f);
#else
  std::memcpy(&u, &f, 4);
#endif
  return u;
}
GLB_HOST_DEVICE inline float u2f(uint32_t u) {
  float f;
#ifdef __CUDA_ARCH__
  f = __uint_as_float(u);
#else
  std::memcpy(&f, &u, 4);
#endif
  return f;
}
}  // namespace detail

// IEEE binary16. Conversions are round-to-nearest-even and handle subnormals,
// infinities and NaN. Arithmetic goes through fp32.
struct alignas(2) float16 {
  uint16_t x = 0;

  float16() = default;
  GLB_HOST_DEVICE float16(float f) : x(fromFloat(f)) {}
  GLB_HOST_DEVICE explicit float16(double d) : x(fromFloat(static_cast<float>(d))) {}
  GLB_HOST_DEVICE float16(int v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE explicit float16(long v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE explicit float16(unsigned long v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE static float16 fromBits(uint16_t b) {
    float16 h;
    h.x = b;
    return h;
  }

  GLB_HOST_DEVICE operator float() const { return toFloat(x); }

  GLB_HOST_DEVICE static uint16_t fromFloat(float f) {
    uint32_t u = detail::f2u(f);
    uint32_t sign = (u >> 16) & 0x8000u;
    uint32_t mag = u & 0x7fffffffu;
    if (mag >= 0x7f800000u) {  // inf / nan
      return static_cast<uint16_t>(sign | 0x7c00u | ((mag > 0x7f800000u) ? 0x0200u : 0));
    }
    if (mag >= 0x477ff000u) {  // rounds to >= 65520 -> inf
      return static_cast<uint16_t>(sign | 0x7c00u);
    }
    if (mag < 0x33000001u) {  // < 2^-25 (or exactly): rounds to zero
      return static_cast<uint16_t>(sign);
    }
    int32_t exp = static_cast<int32_t>(mag >> 23) - 127;
    uint32_t man = (mag & 0x7fffffu) | 0x800000u;
    uint32_t shift;
    uint32_t hexp;
    if (exp < -14) {  // subnormal half
      shift = static_cast<uint32_t>(13 + (-14 - exp));
      hexp = 0;
    } else {
      shift = 13;
      hexp = static_cast<uint32_t>(exp + 15);
    }
    uint32_t half = man >> shift;
    uint32_t rem = man & ((1u << shift) - 1);
    uint32_t mid = 1u << (shift - 1);
    if (rem > mid || (rem == mid && (half & 1u))) half++;
    // For normals `half` carries the implicit bit at 0x400: adding (hexp-1)<<10
    // folds it into the exponent, and a mantissa carry naturally bumps the exponent.
    uint32_t out = (hexp == 0) ? half : (((hexp - 1) << 10) + half);
    return static_cast<uint16_t>(sign | out);
  }

  GLB_HOST_DEVICE static float toFloat(uint16_t h) {
    uint32_t sign = (static_cast<uint32_t>(h) & 0x8000u) << 16;
    uint32_t exp = (h >> 10) & 0x1fu;
    uint32_t man = h & 0x3ffu;
    uint32_t u;
    if (exp == 0) {
      if (man == 0) {
        u = sign;
      } else {  // subnormal: normalise
        int e = -1;
        do {
          e++;
          man <<= 1;
        } while ((man & 0x400u) == 0);
        u = sign | (static_cast<uint32_t>(127 - 15 - e) << 23) | ((man & 0x3ffu) << 13);
      }
    } else if (exp == 31) {
      u = sign | 0x7f800000u | (man << 13);
    } else {
      u = sign | ((exp + 112) << 23) | (man << 13);
    }
    return detail::u2f(u);
  }

  GLB_HOST_DEVICE float16& operator+=(const float16& o) { return *this = float16(float(*this) + float(o)); }
  GLB_HOST_DEVICE float16& operator-=(const float16& o) { return *this = float16(float(*this) - float(o)); }
  GLB_HOST_DEVICE float16& operator*=(const float16& o) { return *this = float16(float(*this) * float(o)); }
  GLB_HOST_DEVICE float16& operator/=(const float16& o) { return *this = float16(float(*this) / float(o)); }
};

// bfloat16: top 16 bits of an fp32, round-to-nearest-even.
struct alignas(2) bfloat16 {
  uint16_t x = 0;

  bfloat16() = default;
  GLB_HOST_DEVICE bfloat16(float f) : x(fromFloat(f)) {}
  GLB_HOST_DEVICE explicit bfloat16(double d) : x(fromFloat(static_cast<float>(d))) {}
  GLB_HOST_DEVICE bfloat16(int v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE explicit bfloat16(long v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE explicit bfloat16(unsigned long v) : x(fromFloat(static_cast<float>(v))) {}
  GLB_HOST_DEVICE static bfloat16 fromBits(uint16_t b) {
    bfloat16 h;
    h.x = b;
    return h;
  }
  GLB_HOST_DEVICE operator float() const { return detail::u2f(static_cast<uint32_t>(x) << 16); }

  GLB_HOST_DEVICE static uint16_t fromFloat(float f) {
    uint32_t u = detail::f2u(f);
    if ((u & 0x7fffffffu) > 0x7f800000u) return static_cast<uint16_t>((u >> 16) | 0x0040u);  // quiet NaN
    uint32_t lsb = (u >> 16) & 1u;
    u += 0x7fffu + lsb;
    return static_cast<uint16_t>(u >> 16);
  }

  GLB_HOST_DEVICE bfloat16& operator+=(const bfloat16& o) { return *this = bfloat16(float(*this) + float(o)); }
  GLB_HOST_DEVICE bfloat16& operator-=(const bfloat16& o) { return *this = bfloat16(float(*this) - float(o)); }
  GLB_HOST_DEVICE bfloat16& operator*=(const bfloat16& o) { return *this = bfloat16(float(*this) * float(o)); }
  GLB_HOST_DEVICE bfloat16& operator/=(const bfloat16& o) { return *this = bfloat16(float(*this) / float(o)); }
};

// ---- 8-bit float storage types ------------------------------------------------------
// OCP FP8. E4M3 ("fn"): bias 7, no infinities, S.1111.111 is NaN, max finite 448.
// E5M2: bias 15, IEEE-style infinities and NaNs, max finite 57344.
// Decoding is exact. Encoding rounds to nearest even and SATURATES to +-max finite, which is
// what the only fp32 -> fp8 conversion on sm_90a does (cvt.rn.satfinite); torch's CPU .to()
// instead turns an overflow into NaN (e4m3fn) or inf (e5m2). NaN stays NaN.
namespace detail {
template <int kExpBits, int kManBits, uint8_t kMaxCode>
struct Fp8Codec {
  static constexpr int kBias = (1 << (kExpBits - 1)) - 1;

  GLB_HOST_DEVICE static uint8_t encode(float f) {
    const uint32_t u = f2u(f);
    const uint32_t sign = (u >> 24) & 0x80u;
    const uint32_t mag = u & 0x7fffffffu;
    if (mag > 0x7f800000u) return static_cast<uint8_t>(sign | 0x7fu);  // NaN
    // At most half the smallest subnormal 2^(1 - bias - man): rounds to (signed) zero.
    if (mag <= (static_cast<uint32_t>(127 - kBias - kManBits) << 23)) return static_cast<uint8_t>(sign);
    const int32_t exp = static_cast<int32_t>(mag >> 23) - 127;
    const uint32_t man = (mag & 0x7fffffu) | 0x800000u;
    uint32_t shift = 23 - kManBits;
    uint32_t hexp = 0;
    if (exp < 1 - kBias) {
      shift += static_cast<uint32_t>(1 - kBias - exp);  // subnormal result
    } else {
      hexp = static_cast<uint32_t>(exp + kBias);
    }
    uint32_t q = man >> shift;
    const uint32_t rem = man & ((1u << shift) - 1), mid = 1u << (shift - 1);
    if (rem > mid || (rem == mid && (q & 1u))) q++;
    // As in float16::fromFloat: the implicit bit of q folds into the exponent field.
    uint32_t code = hexp == 0 ? q : ((hexp - 1) << kManBits) + q;
    if (code > kMaxCode) code = kMaxCode;  // saturate (also the inf / NaN codes of the format)
    return static_cast<uint8_t>(sign | code);
  }

  GLB_HOST_DEVICE static float decode(uint8_t b) {
    const uint32_t sign = (static_cast<uint32_t>(b) & 0x80u) << 24;
    const uint32_t exp = (b >> kManBits) & ((1u << kExpBits) - 1);
    const uint32_t man = b & ((1u << kManBits) - 1);
    if (kExpBits == 4 && exp == 15 && man == 7) return u2f(sign | 0x7fc00000u);
    if (kExpBits == 5 && exp == 31) return u2f(sign | 0x7f800000u | (man != 0 ? 0x400000u : 0u));
    if (exp == 0) {  // subnormal: man * 2^(1 - bias - man bits), exact in fp32
      const float v = static_cast<float>(man) * u2f(static_cast<uint32_t>(127 + 1 - kBias - kManBits) << 23);
      return u2f(sign | f2u(v));
    }
    return u2f(sign | ((exp - kBias + 127) << 23) | (man << (23 - kManBits)));
  }
};
}  // namespace detail

#define GLB_DEFINE_FP8(NAME, EXP, MAN, MAXCODE)                                                    \
  struct alignas(1) NAME {                                                                         \
    using Codec = detail::Fp8Codec<EXP, MAN, MAXCODE>;                                             \
    uint8_t x = 0;                                                                                 \
    NAME() = default;                                                                              \
    GLB_HOST_DEVICE NAME(float f) : x(Codec::encode(f)) {}                                         \
    GLB_HOST_DEVICE explicit NAME(double d) : x(Codec::encode(static_cast<float>(d))) {}           \
    GLB_HOST_DEVICE NAME(int v) : x(Codec::encode(static_cast<float>(v))) {}                       \
    GLB_HOST_DEVICE explicit NAME(long v) : x(Codec::encode(static_cast<float>(v))) {}             \
    GLB_HOST_DEVICE explicit NAME(unsigned long v) : x(Codec::encode(static_cast<float>(v))) {}    \
    GLB_HOST_DEVICE static NAME fromBits(uint8_t b) {                                              \
      NAME h;                                                                                      \
      h.x = b;                                                                                     \
      return h;                                                                                    \
    }                                                                                              \
    GLB_HOST_DEVICE static uint8_t fromFloat(float f) { return Codec::encode(f); }                 \
    GLB_HOST_DEVICE static float toFloat(uint8_t b) { return Codec::decode(b); }                   \
    GLB_HOST_DEVICE operator float() const { return Codec::decode(x); }                            \
    GLB_HOST_DEVICE NAME& operator+=(const NAME& o) { return *this = NAME(float(*this) + float(o)); } \
    GLB_HOST_DEVICE NAME& operator-=(const NAME& o) { return *this = NAME(float(*this) - float(o)); } \
    GLB_HOST_DEVICE NAME& operator*=(const NAME& o) { return *this = NAME(float(*this) * float(o)); } \
    GLB_HOST_DEVICE NAME& operator/=(const NAME& o) { return *this = NAME(float(*this) / float(o)); } \
  };
GLB_DEFINE_FP8(float8_e4m3, 4, 3, 0x7e)  // 0x7e = 448
GLB_DEFINE_FP8(float8_e5m2, 5, 2, 0x7b)  // 0x7b = 57344
#undef GLB_DEFINE_FP8

#define GLB_DEFINE_HALF_BINOPS(T)                                                                   \
  GLB_HOST_DEVICE inline T operator+(const T& a, const T& b) { return T(float(a) + float(b)); }     \
  GLB_HOST_DEVICE inline T operator-(const T& a, const T& b) { return T(float(a) - float(b)); }     \
  GLB_HOST_DEVICE inline T operator*(const T& a, const T& b) { return T(float(a) * float(b)); }     \
  GLB_HOST_DEVICE inline T operator/(const T& a, const T& b) { return T(float(a) / float(b)); }     \
  GLB_HOST_DEVICE inline bool operator<(const T& a, const T& b) { return float(a) < float(b); }     \
  GLB_HOST_DEVICE inline bool operator<=(const T& a, const T& b) { return float(a) <= float(b); }   \
  GLB_HOST_DEVICE inline bool operator>(const T& a, const T& b) { return float(a) > float(b); }     \
  GLB_HOST_DEVICE inline bool operator>=(const T& a, const T& b) { return float(a) >= float(b); }   \
  GLB_HOST_DEVICE inline bool operator==(const T& a, const T& b) { return float(a) == float(b); }   \
  GLB_HOST_DEVICE inline bool operator!=(const T& a, const T& b) { return float(a) != float(b); }
GLB_DEFINE_HALF_BINOPS(float16)
GLB_DEFINE_HALF_BINOPS(bfloat16)
GLB_DEFINE_HALF_BINOPS(float8_e4m3)
GLB_DEFINE_HALF_BINOPS(float8_e5m2)
#undef GLB_DEFINE_HALF_BINOPS

std::ostream& operator<<(std::ostream& os, const float16& v);
std::ostream& operator<<(std::ostream& os, const bfloat16& v);
std::ostream& operator<<(std::ostream& os, const float8_e4m3& v);
std::ostream& operator<<(std::ostream& os, const float8_e5m2& v);

// ---- runtime type / op tags --------------------------------------------------
enum class DataType : int {
  INT8 = 0,
  UINT8 = 1,
  INT32 = 2,
  INT64 = 3,
  UINT64 = 4,
  FLOAT32 = 5,
  FLOAT64 = 6,
  FLOAT16 = 7,
  BFLOAT16 = 8,
  UINT32 = 9,
  INT16 = 10,
  FLOAT8_E4M3 = 11,
  FLOAT8_E5M2 = 12,
};

enum class ReduceOp : int { SUM = 1, PRODUCT = 2, MAX = 3, MIN = 4, CUSTOM = 1000 };

inline bool isFp8(DataType t) { return t == DataType::FLOAT8_E4M3 || t == DataType::FLOAT8_E5M2; }

size_t elementSize(DataType t);
const char* dataTypeName(DataType t);
const char* reduceOpName(ReduceOp op);

template <typename T>
struct DataTypeOf;
#define GLB_DTYPE(T, E)                          \
  template <>                                    \
  struct DataTypeOf<T> {                         \
    static constexpr DataType value = DataType::E; \
  };
GLB_DTYPE(int8_t, INT8)
GLB_DTYPE(char, INT8)
GLB_DTYPE(uint8_t, UINT8)
GLB_DTYPE(int16_t, INT16)
GLB_DTYPE(int32_t, INT32)
GLB_DTYPE(uint32_t, UINT32)
GLB_DTYPE(int64_t, INT64)
GLB_DTYPE(long long, INT64)
GLB_DTYPE(uint64_t, UINT64)
GLB_DTYPE(unsigned long long, UINT64)
GLB_DTYPE(float, FLOAT32)
GLB_DTYPE(double, FLOAT64)
GLB_DTYPE(float16, FLOAT16)
GLB_DTYPE(bfloat16, BFLOAT16)
GLB_DTYPE(float8_e4m3, FLOAT8_E4M3)
GLB_DTYPE(float8_e5m2, FLOAT8_E5M2)
#undef GLB_DTYPE

}  // namespace glb
