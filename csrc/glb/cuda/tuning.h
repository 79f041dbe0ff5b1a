// Measured tuning table for the CUDA collectives.
//
// Which kernel variant is fastest for a message, and with how many CTAs / how much
// unrolling, depends on P, on the kind of buffer (multicast-bound symmetric memory,
// peer-registered, plain user pointer) and on the size. None of that is guessed at run
// time: `python -m gloo_b200.tune` (scripts/glb_tune.py) measures every variant and launch
// shape on the box and writes a table; the library loads it at start-up
// (GLB_TUNE_FILE, else <package>/tuning/<device>.tune) and `choose*` consult it. Without
// a table the built-in defaults of collectives.h apply.
//
// File format, one entry per line ('#' starts a comment):
//   <collective> P=<ranks> buf=<sym|reg|user> maxbytes=<N|inf> algo=<name> blocks=<n> [unroll=<n>] [tile=<n>]
// Entries of one (collective, P, buf) group are searched in ascending maxbytes order; the
// first with bytes <= maxbytes wins.
#pragma once

#include <cstddef>
#include <map>
#include <mutex>
#include <string>
#include <tuple>
#include <vector>

namespace glb {
namespace cuda {

enum class BufKind : int {
  SYMMETRIC = 0,   // library symmetric allocation with an NVSwitch multicast alias
  REGISTERED = 1,  // peer-mapped (cudaIpc / VMM) without multicast
  USER = 2,        // arbitrary device pointer: data passes through the pool
};
const char* bufKindName(BufKind k);

struct TuneEntry {
  size_t maxBytes = ~size_t(0);
  std::string algo;   // collective specific ("ll", "one_shot", "two_shot", "nvls", "pipelined", "direct", ...)
  int blocks = 0;     // 0 = library default
  int unroll = 0;
  int tile = 0;
};

class TuningTable {
 public:
  static TuningTable& get();

  void clear();
  // Returns the number of entries added; malformed lines are reported in *err (and skipped).
  int loadString(const std::string& text, std::string* err = nullptr);
  int loadFile(const std::string& path, std::string* err = nullptr);
  void add(const std::string& coll, int P, BufKind kind, TuneEntry e);
  // nullptr when the table has no group for (coll, P, kind).
  const TuneEntry* lookup(const std::string& coll, int P, BufKind kind, size_t bytes) const;
  std::string dump() const;
  size_t size() const;
  const std::string& source() const { return source_; }

 private:
  using Key = std::tuple<std::string, int, int>;
  mutable std::mutex mu_;
  std::map<Key, std::vector<TuneEntry>> groups_;
  std::string source_ = "built-in";
};

// Loads GLB_TUNE_FILE or the packaged table once per process (idempotent).
void ensureTuningLoaded();

}  // namespace cuda
}  // namespace glb
