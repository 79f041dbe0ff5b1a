// Exception taxonomy.
//
//   Exception                       base of everything thrown by the library
//   ├── InvalidOperationException   API misuse (wrong rank, unsupported op, ...)
//   ├── IoException                 transport failure; the context is poisoned and
//   │   └── TimeoutException        must be re-created (same contract as the
//   │                               reference, docs/errors.md:5-13)
//   ├── InputException              bad input: data found on the device (a collective's
//   │                               device-side counts) or buffers a collective cannot
//   │                               take (overlapping input and output); the context
//   │                               stays usable
//   └── EnforceNotMet               failed GLB_ENFORCE (logging.h)
//
// Parity: gloo/common/error.h:21-48.
#pragma once

#include <chrono>
#include <exception>
#include <stdexcept>
#include <string>

#include "glb/common/string.h"

namespace glb {

// 0 ms means "wait forever"; -1 ms means "inherit the context timeout".
constexpr std::chrono::milliseconds kNoTimeout = std::chrono::milliseconds::zero();
constexpr std::chrono::milliseconds kUnsetTimeout = std::chrono::milliseconds(-1);

struct Exception : public std::runtime_error {
  explicit Exception(const std::string& msg) : std::runtime_error(msg) {}
};

struct InvalidOperationException : public Exception {
  explicit InvalidOperationException(const std::string& msg) : Exception(msg) {}
};

struct InputException : public Exception {
  explicit InputException(const std::string& msg) : Exception(msg) {}
};

struct IoException : public Exception {
  explicit IoException(const std::string& msg) : Exception(msg) {}
};

struct TimeoutException : public IoException {
  explicit TimeoutException(const std::string& msg) : IoException(msg) {}
};

}  // namespace glb

#define GLB_THROW(ExcType, ...) \
  throw ExcType(::glb::strcat_all("[", __FILE__, ":", __LINE__, "] ", __VA_ARGS__))

#define GLB_THROW_INVALID_OPERATION_EXCEPTION(...) \
  GLB_THROW(::glb::InvalidOperationException, __VA_ARGS__)
#define GLB_THROW_IO_EXCEPTION(...) GLB_THROW(::glb::IoException, __VA_ARGS__)
#define GLB_THROW_TIMEOUT(...) GLB_THROW(::glb::TimeoutException, __VA_ARGS__)
