#include "glb/cuda/tuning.h"

#include <dlfcn.h>

#include <algorithm>
#include <cstdlib>
#include <fstream>
#include <sstream>

#include "glb/common/logging.h"
#include "glb/common/utils.h"

namespace glb {
namespace cuda {

const char* bufKindName(BufKind k) {
  switch (k) {
    case BufKind::SYMMETRIC: return "sym";
    case BufKind::REGISTERED: return "reg";
    case BufKind::USER: return "user";
  }
  return "?";
}

TuningTable& TuningTable::get() {
  static TuningTable t;
  return t;
}

void TuningTable::clear() {
  std::lock_guard<std::mutex> g(mu_);
  groups_.clear();
  source_ = "built-in";
}

size_t TuningTable::size() const {
  std::lock_guard<std::mutex> g(mu_);
  size_t n = 0;
  for (const auto& kv : groups_) n += kv.second.size();
  return n;
}

void TuningTable::add(const std::string& coll, int P, BufKind kind, TuneEntry e) {
  std::lock_guard<std::mutex> g(mu_);
  auto& v = groups_[Key(coll, P, static_cast<int>(kind))];
  v.push_back(std::move(e));
  std::stable_sort(v.begin(), v.end(), [](const TuneEntry& a, const TuneEntry& b) { return a.maxBytes < b.maxBytes; });
}

const TuneEntry* TuningTable::lookup(const std::string& coll, int P, BufKind kind, size_t bytes) const {
  std::lock_guard<std::mutex> g(mu_);
  auto it = groups_.find(Key(coll, P, static_cast<int>(kind)));
  if (it == groups_.end() || it->second.empty()) return nullptr;
  for (const auto& e : it->second) {
    if (bytes <= e.maxBytes) return &e;
  }
  return &it->second.back();
}

int TuningTable::loadString(const std::string& text, std::string* err) {
  std::istringstream in(text);
  std::string line;
  int added = 0, lineno = 0;
  while (std::getline(in, line)) {
    lineno++;
    auto hash = line.find('#');
    if (hash != std::string::npos) line.resize(hash);
    std::istringstream ls(line);
    std::string coll;
    if (!(ls >> coll)) continue;
    TuneEntry e;
    int P = 0;
    int kind = -1;
    bool ok = true;
    std::string tok;
    while (ls >> tok) {
      auto eq = tok.find('=');
      if (eq == std::string::npos) {
        ok = false;
        break;
      }
      const std::string k = tok.substr(0, eq), v = tok.substr(eq + 1);
      try {
        if (k == "P") {
          P = std::stoi(v);
        } else if (k == "buf") {
          kind = v == "sym" ? 0 : v == "reg" ? 1 : v == "user" ? 2 : -1;
        } else if (k == "maxbytes") {
          e.maxBytes = v == "inf" ? ~size_t(0) : static_cast<size_t>(std::stoull(v));
        } else if (k == "algo") {
          e.algo = v;
        } else if (k == "blocks") {
          e.blocks = std::stoi(v);
        } else if (k == "unroll") {
          e.unroll = std::stoi(v);
        } else if (k == "tile") {
          e.tile = std::stoi(v);
        }  // unknown keys (e.g. measured us=) are informational
      } catch (const std::exception&) {
        ok = false;
        break;
      }
    }
    if (!ok || P <= 0 || kind < 0 || e.algo.empty()) {
      if (err != nullptr) *err += strcat_all("line ", lineno, ": cannot parse '", line, "'\n");
      continue;
    }
    add(coll, P, static_cast<BufKind>(kind), e);
    added++;
  }
  return added;
}

int TuningTable::loadFile(const std::string& path, std::string* err) {
  std::ifstream f(path);
  if (!f) {
    if (err != nullptr) *err += strcat_all("cannot open ", path, "\n");
    return -1;
  }
  std::stringstream ss;
  ss << f.rdbuf();
  int n = loadString(ss.str(), err);
  if (n > 0) {
    std::lock_guard<std::mutex> g(mu_);
    source_ = path;
  }
  return n;
}

std::string TuningTable::dump() const {
  std::lock_guard<std::mutex> g(mu_);
  std::ostringstream os;
  for (const auto& kv : groups_) {
    for (const auto& e : kv.second) {
      os << std::get<0>(kv.first) << " P=" << std::get<1>(kv.first)
         << " buf=" << bufKindName(static_cast<BufKind>(std::get<2>(kv.first))) << " maxbytes=";
      if (e.maxBytes == ~size_t(0)) {
        os << "inf";
      } else {
        os << e.maxBytes;
      }
      os << " algo=" << e.algo << " blocks=" << e.blocks;
      if (e.unroll) os << " unroll=" << e.unroll;
      if (e.tile) os << " tile=" << e.tile;
      os << "\n";
    }
  }
  return os.str();
}

namespace {
std::string libraryDir() {
  Dl_info info;
  if (dladdr(reinterpret_cast<const void*>(&ensureTuningLoaded), &info) == 0 || info.dli_fname == nullptr) return "";
  std::string p(info.dli_fname);
  auto slash = p.rfind('/');
  return slash == std::string::npos ? "." : p.substr(0, slash);
}
}  // namespace

void ensureTuningLoaded() {
  static std::once_flag once;
  std::call_once(once, [] {
    if (envFlag("CUDA_TUNE_DISABLE", false)) return;
    std::vector<std::string> candidates;
    if (const char* f = std::getenv("GLB_TUNE_FILE")) candidates.push_back(f);
    const std::string dir = libraryDir();
    if (!dir.empty()) {
      candidates.push_back(dir + "/tuning/h100.tune");     // next to _C.so (python package)
      candidates.push_back(dir + "/../tuning/h100.tune");  // next to lib/libglb.so
    }
    for (const auto& c : candidates) {
      std::string err;
      int n = TuningTable::get().loadFile(c, &err);
      if (n > 0) {
        GLB_INFO("tuning table: ", n, " entries from ", c);
        return;
      }
    }
  });
}

}  // namespace cuda
}  // namespace glb
