#include "glb/types.h"

#include <ostream>

#include "glb/common/logging.h"

namespace glb {

Slot Slot::build(uint8_t prefix, uint32_t tag) {
  uint64_t base = (static_cast<uint64_t>(prefix) << 56) | (static_cast<uint64_t>(tag) << kDeltaBits);
  return Slot(base, 0);
}

Slot Slot::add(uint64_t i) const {
  uint64_t d = delta_ + i;
  GLB_ENFORCE_LE(d, kDeltaMask, "Slot overflow: delta ", delta_, " + ", i);
  return Slot(base_, d);
}

std::ostream& operator<<(std::ostream& os, const float16& v) { return os << static_cast<float>(v); }
std::ostream& operator<<(std::ostream& os, const bfloat16& v) { return os << static_cast<float>(v); }
std::ostream& operator<<(std::ostream& os, const float8_e4m3& v) { return os << static_cast<float>(v); }
std::ostream& operator<<(std::ostream& os, const float8_e5m2& v) { return os << static_cast<float>(v); }

size_t elementSize(DataType t) {
  switch (t) {
    case DataType::INT8:
    case DataType::UINT8:
    case DataType::FLOAT8_E4M3:
    case DataType::FLOAT8_E5M2: return 1;
    case DataType::FLOAT16:
    case DataType::BFLOAT16:
    case DataType::INT16: return 2;
    case DataType::INT32:
    case DataType::UINT32:
    case DataType::FLOAT32: return 4;
    case DataType::INT64:
    case DataType::UINT64:
    case DataType::FLOAT64: return 8;
  }
  GLB_THROW_INVALID_OPERATION_EXCEPTION("unknown dtype ", static_cast<int>(t));
}

const char* dataTypeName(DataType t) {
  switch (t) {
    case DataType::INT8: return "int8";
    case DataType::UINT8: return "uint8";
    case DataType::INT16: return "int16";
    case DataType::INT32: return "int32";
    case DataType::UINT32: return "uint32";
    case DataType::INT64: return "int64";
    case DataType::UINT64: return "uint64";
    case DataType::FLOAT32: return "float32";
    case DataType::FLOAT64: return "float64";
    case DataType::FLOAT16: return "float16";
    case DataType::BFLOAT16: return "bfloat16";
    case DataType::FLOAT8_E4M3: return "float8_e4m3";
    case DataType::FLOAT8_E5M2: return "float8_e5m2";
  }
  return "?";
}

const char* reduceOpName(ReduceOp op) {
  switch (op) {
    case ReduceOp::SUM: return "sum";
    case ReduceOp::PRODUCT: return "product";
    case ReduceOp::MAX: return "max";
    case ReduceOp::MIN: return "min";
    case ReduceOp::CUSTOM: return "custom";
  }
  return "?";
}

}  // namespace glb
