#include "glb/cuda/collectives.h"

#include <algorithm>
#include <atomic>
#include <numeric>

#include "glb/common/utils.h"
#include "glb/cuda/kernels.h"
#include "glb/cuda/trace.h"

namespace glb {
namespace cuda {

const char* allreduceAlgoName(AllreduceAlgo a) {
  switch (a) {
    case AllreduceAlgo::AUTO: return "auto";
    case AllreduceAlgo::ONE_SHOT: return "one_shot";
    case AllreduceAlgo::TWO_SHOT: return "two_shot";
    case AllreduceAlgo::NVLS: return "nvls";
    case AllreduceAlgo::LL: return "ll";
    case AllreduceAlgo::PIPELINED: return "pipelined";
    case AllreduceAlgo::HYBRID: return "hybrid";
    case AllreduceAlgo::RING: return "ring";
    case AllreduceAlgo::RING_CHUNKED: return "ring_chunked";
    case AllreduceAlgo::HALVING_DOUBLING: return "halving_doubling";
    case AllreduceAlgo::BCUBE: return "bcube";
    case AllreduceAlgo::HALVING_DOUBLING_PIPELINED: return "halving_doubling_pipelined";
  }
  return "?";
}

AllreduceAlgo allreduceAlgoFromName(const std::string& n) {
  for (AllreduceAlgo a : {AllreduceAlgo::AUTO, AllreduceAlgo::ONE_SHOT, AllreduceAlgo::TWO_SHOT, AllreduceAlgo::NVLS,
                          AllreduceAlgo::LL, AllreduceAlgo::PIPELINED, AllreduceAlgo::HYBRID, AllreduceAlgo::RING,
                          AllreduceAlgo::RING_CHUNKED,
                          AllreduceAlgo::HALVING_DOUBLING, AllreduceAlgo::BCUBE,
                          AllreduceAlgo::HALVING_DOUBLING_PIPELINED}) {
    if (n == allreduceAlgoName(a)) return a;
  }
  return AllreduceAlgo::AUTO;
}

Tuning& tuning() {
  static Tuning t = [] {
    Tuning x;
    x.llMaxBytes = static_cast<size_t>(envInt("CUDA_LL_MAX", static_cast<long>(x.llMaxBytes)));
    x.oneShotMaxBytes = static_cast<size_t>(envInt("CUDA_ONESHOT_MAX", static_cast<long>(x.oneShotMaxBytes)));
    x.nvlsMinBytes = static_cast<size_t>(envInt("CUDA_NVLS_MIN", static_cast<long>(x.nvlsMinBytes)));
    x.maxBlocks = static_cast<int>(envInt("CUDA_BLOCKS", x.maxBlocks));
    x.oneShotBlocks = static_cast<int>(envInt("CUDA_ONESHOT_BLOCKS", x.oneShotBlocks));
    x.copyBlocks = static_cast<int>(envInt("CUDA_COPY_BLOCKS", x.copyBlocks));
    x.alltoallvBlocks = static_cast<int>(envInt("CUDA_ALLTOALLV_BLOCKS", x.alltoallvBlocks));
    x.nvlsReduceScatter = envFlag("CUDA_NVLS_REDUCE_SCATTER", x.nvlsReduceScatter);
    setOneShotPush(envFlag("CUDA_ONESHOT_PUSH", true));
    x.bcastDirectMaxBytes = static_cast<size_t>(envInt("CUDA_BCAST_DIRECT_MAX", static_cast<long>(x.bcastDirectMaxBytes)));
    x.bcastRelayMinBytes = static_cast<size_t>(envInt("CUDA_BCAST_RELAY_MIN", static_cast<long>(x.bcastRelayMinBytes)));
    x.pipeTile = static_cast<int>(envInt("CUDA_PIPE_TILE", x.pipeTile));
    x.pipeExchangeThreads = static_cast<int>(envInt("CUDA_PIPE_XTHREADS", x.pipeExchangeThreads));
    x.tmaCopies = envFlag("CUDA_TMA", x.tmaCopies);
    return x;
  }();
  return t;
}

namespace {

// Layout of the staging area: two one-shot halves, then the bulk region.
struct StageLayout {
  size_t half;       // bytes of one one-shot half
  size_t bulkOff;    // start of the bulk (pipelined / staged collectives) region
  size_t bulkBytes;
};

StageLayout layoutOf(const PeerContext& pc) {
  StageLayout l;
  l.half = std::min<size_t>(roundUp(std::max<size_t>(tuning().oneShotMaxBytes, 4096), 4096), pc.stageBytes() / 4);
  l.bulkOff = 2 * l.half;
  l.bulkBytes = pc.stageBytes() - l.bulkOff;
  return l;
}

int blocksFor(const PeerContext& pc, size_t vecsPerRank, int unrollHint, int cap) {
  size_t want = ceilDiv(std::max<size_t>(vecsPerRank, 1), static_cast<size_t>(kThreads) * unrollHint);
  int b = static_cast<int>(std::min<size_t>(want, static_cast<size_t>(cap)));
  return std::max(1, std::min(b, pc.maxBlocks()));
}

std::atomic<uint64_t> gLaunches{0};

void checkLaunch(const char* what) {
  gLaunches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) GLB_THROW(Exception, what, ": kernel launch failed: ", cudaGetErrorString(e));
}

// Everything a collective does before it launches: device, health, stream order, and the
// host rendezvous needed when ranks share a GPU.
void prologue(PeerContext& pc, cudaStream_t stream) {
  pc.checkHealth();
  pc.orderStreams(stream);
  pc.launchGuard();
}

// ... and after it has launched.
void finish(PeerContext& pc, cudaStream_t stream, const char* what) {
  checkLaunch(what);
  pc.markLaunched(stream);
}

float scaleOf(const Epilogue& ep, DataType dt) {
  if (ep.scale == 1.0) return 1.0f;
  GLB_ENFORCE(dt == DataType::FLOAT32 || dt == DataType::FLOAT64 || dt == DataType::FLOAT16 || dt == DataType::BFLOAT16 ||
                  isFp8(dt),
              "a scale epilogue needs a floating-point buffer");
  return static_cast<float>(ep.scale);
}

// Grid of a bandwidth kernel: enough CTAs for the work, never more than the table / knob
// says, never more than can be co-resident.
int clampBlocks(PeerContext& pc, const void* kernel, int wanted, size_t vecsPerRank, int unroll) {
  const size_t need = ceilDiv(std::max<size_t>(vecsPerRank, 1), static_cast<size_t>(kThreads) * std::max(unroll, 1));
  int b = static_cast<int>(std::min<size_t>(need, static_cast<size_t>(std::max(wanted, 1))));
  return std::max(1, std::min(b, pc.coResidentBlocks(kernel)));
}

// multimem.ld_reduce has no FP8 form on sm_90a: an explicit request for a multicast variant
// on an FP8 buffer is an error rather than a silent change of algorithm.
void rejectFp8Multicast(AllreduceAlgo algo, DataType dt) {
  if (isFp8(dt) && (algo == AllreduceAlgo::NVLS || algo == AllreduceAlgo::HYBRID)) {
    GLB_THROW_INVALID_OPERATION_EXCEPTION("allreduce: ", allreduceAlgoName(algo), " has no ", dataTypeName(dt),
                                          " reduction (multimem.ld_reduce on sm_90a reduces f32 / f16 / bf16 only)");
  }
}

int defaultUnroll(AllreduceAlgo a, int P) {
  if (a == AllreduceAlgo::NVLS) return 4;
  return P == 2 ? 4 : 2;
}

}  // namespace

uint64_t launchCount() { return gLaunches.load(); }
void noteLaunch(unsigned n) { gLaunches.fetch_add(n, std::memory_order_relaxed); }

AllreducePlan planAllreduce(PeerContext& pc, size_t bytes, DataType dt, ReduceOp op, BufKind kind) {
  const auto& t = tuning();
  const int P = std::max(pc.size, 1);
  const auto l = layoutOf(pc);
  AllreducePlan plan;
  auto usable = [&](AllreduceAlgo a) {
    switch (a) {
      case AllreduceAlgo::LL: return bytes <= pc.llMaxBytes();
      case AllreduceAlgo::ONE_SHOT: return roundUp(bytes, 16) <= l.half;
      case AllreduceAlgo::NVLS: return kind == BufKind::SYMMETRIC && nvlsSupports(dt, op);
      case AllreduceAlgo::HYBRID:
        return kind == BufKind::SYMMETRIC && nvlsSupports(dt, op) && hybridKernelFor(dt, pc.size) != nullptr;
      case AllreduceAlgo::TWO_SHOT: return kind != BufKind::USER;
      case AllreduceAlgo::PIPELINED: return kind == BufKind::USER;
      default: return false;
    }
  };
  if (const TuneEntry* e = TuningTable::get().lookup("allreduce", P, kind, bytes)) {
    AllreduceAlgo a = allreduceAlgoFromName(e->algo);
    if (a != AllreduceAlgo::AUTO && usable(a)) {
      plan.algo = a;
      plan.cfg.blocks = e->blocks;
      plan.cfg.unroll = e->unroll;
      plan.tile = e->tile;
      plan.fromTable = true;
      return plan;
    }
  }
  // Built-in fallback. One-shot moves (P-1)*S into every GPU, so its break-even shrinks
  // with P; in-switch reduction moves ~S(1+1/P) per direction against 2S(P-1)/P for
  // two-shot: a win from P = 4 up, a loss at P = 2.
  if (bytes <= t.llMaxBytes && usable(AllreduceAlgo::LL)) {
    plan.algo = AllreduceAlgo::LL;
  } else if (bytes <= t.oneShotMaxBytes / static_cast<size_t>(P) && usable(AllreduceAlgo::ONE_SHOT)) {
    plan.algo = AllreduceAlgo::ONE_SHOT;
  } else if (kind == BufKind::USER) {
    plan.algo = AllreduceAlgo::PIPELINED;
  } else if (P > 2 && bytes >= t.nvlsMinBytes && usable(AllreduceAlgo::NVLS)) {
    plan.algo = AllreduceAlgo::NVLS;
  } else {
    plan.algo = AllreduceAlgo::TWO_SHOT;
  }
  plan.cfg.blocks = 0;
  plan.cfg.unroll = 0;
  return plan;
}

AllreduceAlgo chooseAllreduce(PeerContext& pc, size_t bytes, DataType dt, ReduceOp op, bool registered,
                              bool hasMulticast) {
  const BufKind kind = !registered ? BufKind::USER : (hasMulticast ? BufKind::SYMMETRIC : BufKind::REGISTERED);
  return planAllreduce(pc, bytes, dt, op, kind).algo;
}

void barrier(PeerContext& pc, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::barrier");
  DeviceGuard g(pc.device);
  prologue(pc, stream);
  launchBarrier(pc.comm(), stream);
  finish(pc, stream, "barrier");
}

namespace {

void runLL(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, DataType outDt, ReduceOp op,
           float scale, const LocalPtrs& extra, int blocksHint, cudaStream_t stream) {
  const size_t es = elementSize(dt);
  GLB_ENFORCE_LE(count * es, pc.llMaxBytes(), "LL allreduce limited to ", pc.llMaxBytes(), " bytes");
  const size_t units = ceilDiv(count * es, size_t(8));
  int threads = static_cast<int>(std::min<size_t>(kThreads, roundUp(std::max<size_t>(units, 32), 32)));
  int blocks = static_cast<int>(ceilDiv(units, static_cast<size_t>(threads)));
  blocks = std::max(1, std::min({blocks, blocksHint > 0 ? blocksHint : 16, pc.maxBlocks()}));  // no barrier: no co-residency need
  launchLLAllreduce(pc.comm(), in, out, count, dt, outDt, op, scale, pc.llPtrs(), pc.llSrcStride(), pc.llParityStride(),
                    extra, blocks, threads, stream);
}

void runOneShot(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op, float scale,
                const LocalPtrs& extra, int blocksHint, cudaStream_t stream) {
  const auto l = layoutOf(pc);
  const size_t bytes = count * elementSize(dt);
  GLB_ENFORCE_LE(roundUp(bytes, 16), l.half, "one-shot allreduce limited to ", l.half, " bytes");
  const int blocks = blocksFor(pc, ceilDiv(bytes, size_t(16)), 1, blocksHint > 0 ? blocksHint : tuning().oneShotBlocks);
  launchOneShotAllreduce(pc.comm(), in, out, count, dt, op, scale, pc.stagePtrs(0), l.half, extra, blocks, stream);
}

// Launch shape of a kernel that pipelines plain pointers through `slots` pool slots, each of
// `shares` x blocks x tile 16-byte groups. `payloadBytes` is the largest payload in the same
// units as one slot (the whole vector for the allreduce, P x the largest share for
// reduce_scatter and reduce, the largest block for allgather, P x the block for alltoall and
// scatter, and the bulk region for alltoallv, whose byte counts are rank-local). A zero hint takes
// the tuning default.
struct PipeShape {
  int blocks = 1;
  int tile = 16;
  int xthreads = 32;
};

PipeShape pipeShape(PeerContext& pc, const void* kernel, int slots, int shares, size_t payloadBytes, int blocksHint,
                    int tileHint, int xthreadsHint, const char* what) {
  const auto l = layoutOf(pc);
  PipeShape sh;
  sh.blocks = std::max(1, std::min(blocksHint > 0 ? blocksHint : tuning().maxBlocks, pc.coResidentBlocks(kernel)));
  // Tile: a power of two, small enough for every slot in the bulk region and for a few
  // steps of pipelining on mid-sized messages.
  const int tile = tileHint > 0 ? tileHint : tuning().pipeTile;
  auto slotBytes = [&](int tl, int bl) { return static_cast<size_t>(shares) * bl * tl * 16; };
  while (sh.tile * 2 <= tile) sh.tile *= 2;
  while (sh.tile > 16 && (slots * slotBytes(sh.tile, sh.blocks) > l.bulkBytes ||
                          payloadBytes < 4 * slotBytes(sh.tile, sh.blocks))) {
    sh.tile /= 2;
  }
  while (sh.blocks > 1 && payloadBytes < slotBytes(sh.tile, sh.blocks)) sh.blocks = (sh.blocks + 1) / 2;  // tiny messages: fewer CTAs
  GLB_ENFORCE_LE(slots * slotBytes(sh.tile, sh.blocks), l.bulkBytes, "staging pool too small for the pipelined ", what,
                 "; raise GLB_CUDA_STAGE_MB (CudaContext stage_bytes)");
  const int x = xthreadsHint > 0 ? xthreadsHint : tuning().pipeExchangeThreads;
  sh.xthreads = std::max(32, std::min(kThreads - 32, x / 32 * 32));
  return sh;
}

void runPipelined(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op, float scale,
                  const LocalPtrs& extra, const AllreducePlan& plan, cudaStream_t stream) {
  const auto l = layoutOf(pc);
  const size_t es = elementSize(dt);
  const size_t groups = ceilDiv(count * es, size_t(16));
  const bool mc = pc.nvlsAvailable() && pc.size > 2 && nvlsSupports(dt, op);
  // cfg.unroll doubles as "exchange warps" for this kernel (0 = the pipeExchangeThreads knob).
  const PipeShape sh = pipeShape(pc, pipelinedKernelFor(dt, mc, pc.size), 3, pc.size, groups * 16, plan.cfg.blocks,
                                 plan.tile, plan.cfg.unroll * 32, "allreduce");
  launchPipelinedAllreduce(pc.comm(), in, out, count, dt, op, scale, pc.stagePtrs(l.bulkOff),
                           mc ? pc.stageMc(l.bulkOff) : nullptr, sh.tile, sh.xthreads, extra, sh.blocks, stream);
}

}  // namespace

void allreduce(PeerContext& pc, const PeerBuffer& buf, size_t byteOffset, size_t count, DataType dt, ReduceOp op,
               AllreduceAlgo algo, cudaStream_t stream, const Epilogue& ep) {
  GLB_TRACE_RANGE("glb::cuda::allreduce");
  pc.checkHealth();
  if (count == 0) return;
  const size_t es = elementSize(dt);
  const size_t bytes = count * es;
  GLB_ENFORCE_LE(byteOffset + bytes, buf.bytes, "allreduce range exceeds the registered buffer");
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  GLB_ENFORCE(!ep.castOutput || ep.outDtype == dt, "in-place allreduce cannot change the dtype; use allreduceCast");
  rejectFp8Multicast(algo, dt);
  const float scale = scaleOf(ep, dt);
  DeviceGuard g(pc.device);
  char* local = static_cast<char*>(buf.local) + byteOffset;
  // Single rank: the buffer already holds the result unless there is something to fold or
  // scale. GLB_CUDA_FORCE_KERNELS=1 still launches the collective kernel (loopback on local
  // memory) so it can be profiled with Nsight Compute.
  if (pc.size == 1 && !envFlag("CUDA_FORCE_KERNELS", false)) {
    if (ep.extra.n > 0 || scale != 1.0f) {
      std::vector<void*> all{local};
      for (int k = 0; k < ep.extra.n; k++) all.push_back(ep.extra.p[k]);
      pc.orderStreams(stream);
      launchLocalAllreduceMany(all.data(), static_cast<int>(all.size()), count, dt, op, scale, pc.localTileCounter(), stream);
      finish(pc, stream, "allreduce(local)");
    }
    return;
  }
  const bool hasMc = buf.mc != nullptr && byteOffset % 16 == 0;
  const BufKind kind = hasMc ? BufKind::SYMMETRIC : BufKind::REGISTERED;
  // The two-shot and NVLS kernels fold and fan out the extra pointers in 16-byte packs.
  bool extraAligned = true;
  for (int k = 0; k < ep.extra.n; k++) extraAligned = extraAligned && reinterpret_cast<uintptr_t>(ep.extra.p[k]) % 16 == 0;
  AllreducePlan plan;
  if (algo == AllreduceAlgo::AUTO) {
    plan = planAllreduce(pc, bytes, dt, op, kind);
    algo = plan.algo;
    if (algo == AllreduceAlgo::HYBRID && ep.extra.n > 0) {  // the hybrid kernel takes one pointer
      algo = AllreduceAlgo::NVLS;
      plan.cfg = LaunchCfg();
    }
    if (algo == AllreduceAlgo::NVLS && !extraAligned) {
      algo = AllreduceAlgo::TWO_SHOT;
      plan.cfg = LaunchCfg();
    }
  }
  if (ep.blocks > 0) plan.cfg.blocks = ep.blocks;
  if (ep.unroll > 0) plan.cfg.unroll = ep.unroll;
  prologue(pc, stream);
  switch (algo) {
    case AllreduceAlgo::LL:
      runLL(pc, local, local, count, dt, dt, op, scale, ep.extra, plan.cfg.blocks, stream);
      break;
    case AllreduceAlgo::ONE_SHOT:
      runOneShot(pc, local, local, count, dt, op, scale, ep.extra, plan.cfg.blocks, stream);
      break;
    case AllreduceAlgo::NVLS: {
      GLB_ENFORCE(hasMc, "NVLS allreduce needs a multicast-bound (symmetric) buffer");
      GLB_ENFORCE(nvlsSupports(dt, op), "NVLS supports sum over float32/float16/bfloat16 only");
      GLB_ENFORCE(extraAligned, "NVLS allreduce needs 16-byte aligned extra pointers");
      LaunchCfg cfg = plan.cfg;
      if (cfg.unroll == 0) cfg.unroll = defaultUnroll(algo, pc.size);
      cfg.blocks = clampBlocks(pc, nvlsKernelFor(dt, cfg.unroll), cfg.blocks > 0 ? cfg.blocks : tuning().maxBlocks,
                               ceilDiv(bytes, size_t(16)) / pc.size, cfg.unroll);
      launchNvlsAllreduce(pc.comm(), static_cast<char*>(buf.mc) + byteOffset, buf.ptrsAt(byteOffset), count, dt, scale,
                          ep.extra, cfg, stream);
      break;
    }
    case AllreduceAlgo::HYBRID: {
      GLB_ENFORCE(hasMc && nvlsSupports(dt, op) && hybridKernelFor(dt, pc.size) != nullptr && ep.extra.n == 0,
                  "hybrid allreduce: sum of f32/f16/bf16 on a multicast-bound buffer, 4 or 8 ranks, one pointer");
      // cfg.blocks = all CTAs, cfg.unroll = CTAs of the NVLS part, tile = per-mille of the vector done peer to peer
      int blocks = plan.cfg.blocks > 0 ? plan.cfg.blocks : 132;
      blocks = std::max(2, std::min(blocks, pc.coResidentBlocks(hybridKernelFor(dt, pc.size))));
      const int nvlsBlocks = std::max(1, std::min(plan.cfg.unroll > 0 ? plan.cfg.unroll : 32, blocks - 1));
      const int permille = std::max(0, std::min((ep.tile > 0 ? ep.tile : plan.tile > 0 ? plan.tile : 175), 900));
      launchHybridAllreduce(pc.comm(), static_cast<char*>(buf.mc) + byteOffset, buf.ptrsAt(byteOffset), count, dt, scale,
                            blocks, nvlsBlocks, static_cast<unsigned>(permille), stream);
      break;
    }
    case AllreduceAlgo::TWO_SHOT: {
      const bool vectorOk = buf.vectorOk && byteOffset % 16 == 0 && extraAligned;
      LaunchCfg cfg = plan.cfg;
      if (cfg.unroll == 0) cfg.unroll = defaultUnroll(algo, pc.size);
      cfg.blocks = clampBlocks(pc, twoShotKernelFor(dt, pc.size, cfg.unroll), cfg.blocks > 0 ? cfg.blocks : tuning().maxBlocks,
                               bytes / 16 / pc.size, cfg.unroll);
      launchTwoShotAllreduce(pc.comm(), buf.ptrsAt(byteOffset), count, dt, op, scale, vectorOk, ep.extra, cfg, stream);
      break;
    }
    case AllreduceAlgo::PIPELINED:
      plan.tile = ep.tile > 0 ? ep.tile : plan.tile;
      runPipelined(pc, local, local, count, dt, op, scale, ep.extra, plan, stream);
      break;
    default:
      GLB_THROW_INVALID_OPERATION_EXCEPTION("allreduce: algorithm ", allreduceAlgoName(algo),
                                            " is not available on this entry point");
  }
  finish(pc, stream, "allreduce");
}

void allreduce(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op,
               AllreduceAlgo algo, cudaStream_t stream, const Epilogue& ep) {
  GLB_TRACE_RANGE("glb::cuda::allreduce(user pointers)");
  pc.checkHealth();
  if (count == 0) return;
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  rejectFp8Multicast(algo, dt);
  DeviceGuard g(pc.device);
  const size_t es = elementSize(dt);
  const size_t bytes = count * es;
  const DataType outDt = ep.castOutput ? ep.outDtype : dt;
  GLB_ENFORCE(castSupported(dt, outDt), "allreduce: unsupported dtype conversion in the epilogue");
  const float scale = scaleOf(ep, dt);
  if (pc.size == 1 && !envFlag("CUDA_FORCE_KERNELS", false)) {
    if (outDt != dt) {
      // Single rank with a cast: the LL kernel degenerates to a fused fold / scale / convert.
      GLB_ENFORCE_LE(bytes, pc.llMaxBytes(), "allreduce with a dtype conversion on plain pointers is limited to ",
                     pc.llMaxBytes(), " bytes; register the buffers (allreduceCast)");
      pc.checkHealth();
      runLL(pc, in, out, count, dt, outDt, op, scale, ep.extra, 0, stream);
      checkLaunch("allreduce(ll)");
      return;
    }
    if (ep.extra.n > 0 || scale != 1.0f) {
      if (in != out) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
      std::vector<void*> all{out};
      for (int k = 0; k < ep.extra.n; k++) all.push_back(ep.extra.p[k]);
      pc.orderStreams(stream);
      launchLocalAllreduceMany(all.data(), static_cast<int>(all.size()), count, dt, op, scale, pc.localTileCounter(), stream);
      finish(pc, stream, "allreduce(local)");
    } else if (in != out) {
      GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    }
    return;
  }
  AllreducePlan plan;
  if (algo == AllreduceAlgo::AUTO) {
    plan = planAllreduce(pc, bytes, dt, op, BufKind::USER);
    algo = plan.algo;
  }
  if (ep.blocks > 0) plan.cfg.blocks = ep.blocks;
  if (ep.unroll > 0) plan.cfg.unroll = ep.unroll;
  if (ep.tile > 0) plan.tile = ep.tile;
  if (outDt != dt) {
    GLB_ENFORCE_LE(bytes, pc.llMaxBytes(), "allreduce with a dtype conversion on plain pointers is limited to ",
                   pc.llMaxBytes(), " bytes; register the buffers (allreduceCast)");
    algo = AllreduceAlgo::LL;
  }
  // Variants that need peer-visible user memory fall back to the pool path.
  if (algo == AllreduceAlgo::TWO_SHOT || algo == AllreduceAlgo::NVLS) algo = AllreduceAlgo::PIPELINED;
  if (algo == AllreduceAlgo::ONE_SHOT && roundUp(bytes, 16) > layoutOf(pc).half) algo = AllreduceAlgo::PIPELINED;
  if (algo == AllreduceAlgo::LL && bytes > pc.llMaxBytes()) algo = AllreduceAlgo::PIPELINED;
  prologue(pc, stream);
  switch (algo) {
    case AllreduceAlgo::LL: runLL(pc, in, out, count, dt, outDt, op, scale, ep.extra, plan.cfg.blocks, stream); break;
    case AllreduceAlgo::ONE_SHOT: runOneShot(pc, in, out, count, dt, op, scale, ep.extra, plan.cfg.blocks, stream); break;
    case AllreduceAlgo::PIPELINED: runPipelined(pc, in, out, count, dt, op, scale, ep.extra, plan, stream); break;
    default:
      GLB_THROW_INVALID_OPERATION_EXCEPTION("allreduce: algorithm ", allreduceAlgoName(algo), " needs registered buffers");
  }
  finish(pc, stream, "allreduce(user pointers)");
}

void allreduceCast(PeerContext& pc, const PeerBuffer& in, size_t inOffset, const PeerBuffer& out, size_t outOffset,
                   size_t count, DataType dt, DataType outDt, ReduceOp op, cudaStream_t stream, const Epilogue& ep) {
  GLB_TRACE_RANGE("glb::cuda::allreduceCast");
  if (count == 0) return;
  GLB_ENFORCE(dt != outDt && castSupported(dt, outDt), "allreduceCast: supported conversions are f32 <-> f16 / bf16, fp8 -> f32 / bf16 and f32 / bf16 -> fp8");
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  GLB_ENFORCE_LE(inOffset + count * elementSize(dt), in.bytes, "allreduceCast input range exceeds the buffer");
  GLB_ENFORCE_LE(outOffset + count * elementSize(outDt), out.bytes, "allreduceCast output range exceeds the buffer");
  GLB_ENFORCE(ep.extra.n == 0, "allreduceCast takes one input per rank");
  const float scale = scaleOf(ep, DataType::FLOAT32);
  DeviceGuard g(pc.device);
  if (pc.size == 1 && !envFlag("CUDA_FORCE_KERNELS", false)) {
    // Degenerate: convert (and scale) locally, in pieces the LL kernel accepts.
    const size_t piece = pc.llMaxBytes() / elementSize(dt);
    pc.checkHealth();
    for (size_t done = 0; done < count; done += piece) {
      const size_t n = std::min(piece, count - done);
      runLL(pc, static_cast<const char*>(in.local) + inOffset + done * elementSize(dt),
            static_cast<char*>(out.local) + outOffset + done * elementSize(outDt), n, dt, outDt, op, scale, LocalPtrs(), 0,
            stream);
      checkLaunch("allreduceCast(local)");
    }
    return;
  }
  const bool vec = in.vectorOk && out.vectorOk && inOffset % 32 == 0 && outOffset % 32 == 0;
  const bool useMc = in.mc != nullptr && vec && pc.size > 2 && nvlsSupports(dt, op) &&
                     count * elementSize(dt) >= tuning().nvlsMinBytes;
  const void* kernel = castKernelFor(dt, outDt);
  const int wanted = ep.blocks > 0 ? ep.blocks : tuning().maxBlocks;
  const int blocks = clampBlocks(pc, kernel, wanted, ceilDiv(count, size_t(8)) / pc.size, 1);
  prologue(pc, stream);
  launchCastAllreduce(pc.comm(), in.ptrsAt(inOffset), useMc ? static_cast<char*>(in.mc) + inOffset : nullptr,
                      out.ptrsAt(outOffset), count, dt, outDt, op, scale, vec, blocks, stream);
  finish(pc, stream, "allreduceCast");
}


// ---- allreduce fused with bias, residual add and a norm ----------------------------------

// The bytes of one row of out in the pool: a T row, or with `quant` hidden e4m3 codes and a scale.
size_t poolOutRowBytes(size_t hidden, DataType dt, bool quant) {
  return quant ? hidden + sizeof(float) : hidden * elementSize(dt);
}

NormPlan planResidualNorm(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm, AllreduceAlgo algo,
                          bool quant) {
  const size_t rowBytes = hidden * elementSize(dt);
  const size_t bytes = rows * rowBytes;
  const auto l = layoutOf(pc);
  NormPlan p;
  p.variant = kNormLocal;
  p.chunkRows = std::max<size_t>(rows, 1);
  if (pc.size > 1) {
    if (algo != AllreduceAlgo::AUTO && algo != AllreduceAlgo::LL && algo != AllreduceAlgo::ONE_SHOT &&
        algo != AllreduceAlgo::TWO_SHOT) {
      GLB_THROW(InputException, "allreduce_residual_norm: algo must be auto, ll, one_shot or two_shot, got ",
                allreduceAlgoName(algo));
    }
    // The allreduce's choice for a plain buffer of the same size: the tuning table and the
    // CUDA_LL_MAX / CUDA_ONESHOT_MAX knobs govern this operation too. As in allreduce(algo=), a
    // variant whose region cannot hold the rows runs as the row-sharded two-shot.
    if (algo == AllreduceAlgo::AUTO) algo = planAllreduce(pc, bytes, dt, ReduceOp::SUM, BufKind::USER).algo;
    if (algo == AllreduceAlgo::LL && bytes <= pc.llMaxBytes()) {
      p.variant = kNormLL;
    } else if (algo == AllreduceAlgo::ONE_SHOT && roundUp(bytes, 16) <= l.half) {
      p.variant = kNormOneShot;
    } else {
      p.variant = kNormTwoShot;
      // One launch while the staged rows (partials, and out with a norm) fit the bulk region.
      const size_t perRow = rowBytes + (norm != kNormNone ? poolOutRowBytes(hidden, dt, quant) : 0);
      if (perRow > l.bulkBytes) {
        GLB_THROW(InputException, "allreduce_residual_norm: the pool's bulk region holds no row of ", rowBytes,
                  " bytes; raise GLB_CUDA_STAGE_MB (CudaContext stage_bytes)");
      }
      p.chunkRows = std::min(p.chunkRows, l.bulkBytes / perRow);
    }
  }
  p.launches = rows == 0 ? 0 : ceilDiv(rows, p.chunkRows);
  return p;
}

NormPlan planReduceScatterNorm(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm, bool gatherOut,
                               bool quant) {
  const size_t P = static_cast<size_t>(pc.size);
  if (rows % P != 0) {
    GLB_THROW(InputException, "reduce_scatter_residual_norm: ", rows, " rows do not split into ", P, " equal shards");
  }
  // One rank: the shard is every row, and the allreduce form's local launch computes it.
  if (P == 1) return planResidualNorm(pc, rows, hidden, dt, norm, AllreduceAlgo::AUTO, quant);
  const size_t rowBytes = hidden * elementSize(dt), shard = rows / P;
  const auto l = layoutOf(pc);
  // One launch while the staged rows of every shard (and the gathered out) fit the bulk region;
  // beyond it, consecutive chunks of chunkRows rows of every shard.
  const size_t perRow = P * (rowBytes + (norm != kNormNone && gatherOut ? poolOutRowBytes(hidden, dt, quant) : 0));
  if (perRow > l.bulkBytes) {
    GLB_THROW(InputException, "reduce_scatter_residual_norm: the pool's bulk region holds no row of ", rowBytes,
              " bytes from each of ", P, " shards; raise GLB_CUDA_STAGE_MB (CudaContext stage_bytes)");
  }
  NormPlan p;
  p.variant = kNormScatter;
  p.chunkRows = std::min(std::max<size_t>(shard, 1), l.bulkBytes / perRow);
  p.launches = shard == 0 ? 0 : ceilDiv(shard, p.chunkRows);
  return p;
}

NormBackwardPlan planReduceScatterNormBackward(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm,
                                               bool gatherOut, int vectors) {
  const char* op = "reduce_scatter_residual_norm_backward";
  const size_t P = static_cast<size_t>(pc.size);
  if (rows % P != 0) GLB_THROW(InputException, op, ": ", rows, " rows do not split into ", P, " equal shards");
  if (norm != kNormRms && norm != kNormLayer) GLB_THROW(InputException, op, ": needs a norm (rms or layer)");
  if (!normSupports(dt)) GLB_THROW(InputException, op, ": rows must be float32, bfloat16 or float16");
  if (vectors < 0 || vectors > 3) GLB_THROW(InputException, op, ": ", vectors, " vector gradients asked for");
  const size_t rowBytes = hidden * elementSize(dt), shard = rows / P;
  NormBackwardPlan p;
  size_t gridRows;
  if (P == 1) {
    // One rank: the local launch over every row, no exchange.
    p.variant = kNormLocal;
    p.chunkRows = std::max<size_t>(rows, 1);
    gridRows = p.chunkRows;
  } else {
    // The forward's chunking: P rows of pool per chunk row for grad_partial, and P more for the
    // staged grad_out when it was gathered.
    const auto l = layoutOf(pc);
    const size_t perRow = P * (gatherOut ? 2 : 1) * rowBytes;
    if (perRow > l.bulkBytes) {
      GLB_THROW(InputException, op, ": the pool's bulk region holds no row of ", rowBytes, " bytes from each of ", P,
                " shards; raise GLB_CUDA_STAGE_MB (CudaContext stage_bytes)");
    }
    p.variant = kNormScatter;
    p.chunkRows = std::min(std::max<size_t>(shard, 1), l.bulkBytes / perRow);
    gridRows = P * p.chunkRows;
  }
  const void* kernel = normBackwardKernelFor(dt, norm, p.variant);
  p.blocks = static_cast<int>(std::min<size_t>(
      gridRows, static_cast<size_t>(pc.coResidentBlocks(kernel, kThreads, normBackwardSmemBytes(vectors)))));
  p.launches = shard == 0 ? 0 : ceilDiv(shard, p.chunkRows);
  // The column sums: one fp32 vector per CTA and vector, finished by one more launch.
  p.workspaceBytes = vectors > 0 ? static_cast<size_t>(p.blocks) * vectors * hidden * sizeof(float) : 0;
  if (vectors > 0 && p.launches > 0) p.launches += 1;
  return p;
}

NormBackwardPlan planResidualNormBackward(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm,
                                          int vectors, AllreduceAlgo algo) {
  const char* op = "allreduce_residual_norm_backward";
  if (norm != kNormRms && norm != kNormLayer) GLB_THROW(InputException, op, ": needs a norm (rms or layer)");
  if (!normSupports(dt)) GLB_THROW(InputException, op, ": rows must be float32, bfloat16 or float16");
  if (vectors < 0 || vectors > 3) GLB_THROW(InputException, op, ": ", vectors, " vector gradients asked for");
  if (algo != AllreduceAlgo::AUTO && algo != AllreduceAlgo::ONE_SHOT && algo != AllreduceAlgo::TWO_SHOT) {
    GLB_THROW(InputException, op, ": algo must be auto, one_shot or two_shot, got ", allreduceAlgoName(algo));
  }
  const size_t rowBytes = hidden * elementSize(dt);
  NormBackwardPlan p;
  p.variant = kNormLocal;
  p.chunkRows = std::max<size_t>(rows, 1);
  if (pc.size > 1) {
    // auto: the forward's variant for these rows (no LL backward: its LL is the one-shot here);
    // a one-shot whose rows do not fit a pool half runs as the two-shot, as in the forward.
    const auto l = layoutOf(pc);
    int v = algo == AllreduceAlgo::ONE_SHOT ? kNormOneShot : kNormTwoShot;
    if (algo == AllreduceAlgo::AUTO) v = planResidualNorm(pc, rows, hidden, dt, kNormNone, algo).variant;
    p.variant = (v == kNormLL || v == kNormOneShot) && roundUp(rows * rowBytes, 16) <= l.half ? kNormOneShot
                                                                                               : kNormTwoShot;
    if (p.variant == kNormTwoShot) {
      if (rowBytes > l.bulkBytes || vectors * hidden * sizeof(float) > l.bulkBytes) {
        GLB_THROW(InputException, op, ": the pool's bulk region holds no row of ", rowBytes, " bytes or no ",
                  vectors, " fp32 column sums of ", hidden, "; raise GLB_CUDA_STAGE_MB (CudaContext stage_bytes)");
      }
      // One pool row per row: the owner's gradPartial overwrites the staged gradOut.
      p.chunkRows = std::min(p.chunkRows, l.bulkBytes / rowBytes);
    }
  }
  const void* kernel = normBackwardKernelFor(dt, norm, p.variant);
  p.blocks = static_cast<int>(std::min<size_t>(
      p.chunkRows, static_cast<size_t>(pc.coResidentBlocks(kernel, kThreads, normBackwardSmemBytes(vectors)))));
  p.launches = rows == 0 ? 0 : ceilDiv(rows, p.chunkRows);
  p.workspaceBytes = vectors > 0 ? static_cast<size_t>(p.blocks) * vectors * hidden * sizeof(float) : 0;
  if (vectors > 0 && p.launches > 0) p.launches += 1;
  return p;
}

const char* normVariantName(int variant) {
  switch (variant) {
    case kNormLL: return "ll";
    case kNormOneShot: return "one_shot";
    case kNormTwoShot: return "two_shot";
    case kNormScatter: return "reduce_scatter";
    default: return "local";
  }
}

namespace {

// A tensor argument of the fused operations: `bytes` bytes at p (null: absent).
struct NormRange {
  const char* name;
  const void* p;
  size_t bytes;
};

#define GLB_NORM_CHECK(cond, ...) \
  do {                            \
    if (!(cond)) GLB_THROW(InputException, op, ": ", __VA_ARGS__); \
  } while (0)

// What the fused operations check before anything is launched: dtype, norm, row width,
// `required` (whether the tensors `requiredWhat` names are there), 16-byte alignment, and that no
// output overlaps an input or another output, except outputs[0] == inputs[inPlace] exactly (in
// place: each row is read before it is written). Null tensors are absent.
template <size_t NI, size_t NO>
void checkNormCall(const char* op, DataType dt, int norm, size_t hidden, bool required, const char* requiredWhat,
                   const NormRange (&inputs)[NI], const NormRange (&outputs)[NO], size_t inPlace) {
  GLB_NORM_CHECK(normSupports(dt), "rows must be float32, bfloat16 or float16, got ", dataTypeName(dt));
  GLB_NORM_CHECK(norm == kNormNone || norm == kNormRms || norm == kNormLayer, "unknown norm ", norm);
  const size_t es = elementSize(dt);
  GLB_NORM_CHECK(hidden > 0 && hidden * es % 16 == 0, "a row of ", hidden, " ", dataTypeName(dt),
                 " elements is not a positive multiple of 16 bytes");
  GLB_NORM_CHECK(hidden <= static_cast<size_t>(kMaxNormHidden), "rows of ", hidden, " elements exceed the limit of ",
                 kMaxNormHidden);
  GLB_NORM_CHECK(required, requiredWhat);
  for (const NormRange& r : inputs) {
    GLB_NORM_CHECK(reinterpret_cast<uintptr_t>(r.p) % 16 == 0, r.name, " must be 16-byte aligned");
  }
  for (const NormRange& r : outputs) {
    GLB_NORM_CHECK(reinterpret_cast<uintptr_t>(r.p) % 16 == 0, r.name, " must be 16-byte aligned");
  }
  auto overlap = [&](const NormRange& a, const NormRange& b) {
    const uintptr_t x = reinterpret_cast<uintptr_t>(a.p), y = reinterpret_cast<uintptr_t>(b.p);
    return a.p != nullptr && b.p != nullptr && a.bytes > 0 && b.bytes > 0 && x < y + b.bytes && y < x + a.bytes;
  };
  for (const NormRange& o : outputs) {
    for (const NormRange& i : inputs) {
      const bool inPlaceOk = &o == &outputs[0] && &i == &inputs[inPlace] && o.p == i.p;
      GLB_NORM_CHECK(inPlaceOk || !overlap(o, i), o.name, " overlaps ", i.name);
    }
  }
  for (size_t a = 0; a < NO; a++) {
    for (size_t b = a + 1; b < NO; b++) {
      GLB_NORM_CHECK(!overlap(outputs[a], outputs[b]), outputs[a].name, " overlaps ", outputs[b].name);
    }
  }
}

// The forward's required tensors: partial, residual, residual_out and, with a norm, out.
constexpr const char* kNormRequired = "partial, residual, residual_out and (with a norm) out are required";
bool normRequired(size_t rows, const NormRange (&inputs)[5], const NormRange (&outputs)[3], int norm) {
  return rows == 0 || (inputs[0].p != nullptr && inputs[1].p != nullptr && outputs[0].p != nullptr &&
                       (norm == kNormNone || outputs[1].p != nullptr));
}

// The forward's outputs: residual_out (`residualRows` rows) and out (`outRows` rows of T, or with
// outScales of e4m3 codes, plus their fp32 scales).
struct NormOutputs {
  NormRange r[3];
};
NormOutputs normOutputs(void* residualOut, void* out, float* outScales, size_t residualRows, size_t outRows,
                        size_t hidden, DataType dt, int norm) {
  const size_t rb = hidden * elementSize(dt);
  const bool quant = outScales != nullptr;
  return {{{"residual_out", residualOut, residualRows * rb},
           {"out", norm != kNormNone ? out : nullptr, outRows * (quant ? hidden : rb)},
           {"out_scales", outScales, outRows * sizeof(float)}}};
}

// The quantising form's own limits: a norm, and rows of codes that are whole 16-byte packs.
void checkNormQuant(const char* op, int norm, size_t hidden, const float* outScales) {
  if (outScales == nullptr) return;
  GLB_NORM_CHECK(norm != kNormNone, "the FP8 out (out_scales) needs a norm (rms or layer)");
  GLB_NORM_CHECK(hidden % 16 == 0, "the FP8 out needs rows of a multiple of 16 elements, got ", hidden);
}

// Points a chunk's out at its codes and scales (the quantising form): rows from row r0 on.
void quantChunk(NormArgs& a, void* out, float* outScales, size_t r0, size_t hidden) {
  if (outScales == nullptr) return;
  a.out = static_cast<char*>(out) + r0 * hidden;
  a.outScales = outScales + r0;
}

// The arguments of one chunk: n rows from `off` bytes into every row tensor.
NormArgs chunkArgs(const void* partial, const void* residual, void* residualOut, void* out, const void* bias,
                   const void* gamma, const void* beta, size_t off, size_t n, size_t hidden, int norm, float eps) {
  NormArgs a;
  a.partial = static_cast<const char*>(partial) + off;
  a.residual = static_cast<const char*>(residual) + off;
  a.residualOut = static_cast<char*>(residualOut) + off;
  a.out = norm != kNormNone ? static_cast<char*>(out) + off : nullptr;
  a.bias = bias;
  a.gamma = gamma;
  a.beta = beta;
  a.rows = n;
  a.hidden = hidden;
  a.eps = eps;
  return a;
}

// One launch of the fused kernel whose grid-stride loops cover `gridRows` rows.
void launchNormChunk(PeerContext& pc, const NormArgs& a, const NormXchg& x, DataType dt, int norm, int variant,
                     size_t gridRows, cudaStream_t stream, const char* op) {
  // Every CTA waits for its twin on the peers: the grid must be co-resident.
  const void* kernel = allreduceNormKernelFor(dt, norm, variant, a.outScales != nullptr);
  const int blocks = static_cast<int>(std::min<size_t>(gridRows, static_cast<size_t>(pc.coResidentBlocks(kernel))));
  prologue(pc, stream);
  launchAllreduceNorm(pc.comm(), a, x, dt, norm, variant, blocks, stream);
  finish(pc, stream, op);
}

// The column sums a backward call asks for, in workspace order: vec[kind] is the slot of kind k
// (0 weight, 1 norm bias, 2 bias; -1: not asked for), out[slot] its output.
struct VecSlots {
  int vec[3];
  int vectors = 0;
  void* out[3] = {nullptr, nullptr, nullptr};
};
VecSlots vecSlots(void* const (&vecOut)[3]) {
  VecSlots v;
  for (int k = 0; k < 3; k++) {
    v.vec[k] = vecOut[k] != nullptr ? v.vectors : -1;
    if (vecOut[k] != nullptr) v.out[v.vectors++] = vecOut[k];
  }
  return v;
}

// The backward's arguments of one chunk: n rows from `off` bytes into every row tensor.
NormBwdArgs bwdChunkArgs(const void* gradOut, const void* s, const void* gradS, void* gradResidual, void* gradPartial,
                         const void* gamma, void* workspace, size_t off, size_t n, size_t hidden, float eps,
                         const VecSlots& v, bool first) {
  NormBwdArgs a;
  a.gradOut = static_cast<const char*>(gradOut) + off;
  a.s = static_cast<const char*>(s) + off;
  a.gradS = gradS != nullptr ? static_cast<const char*>(gradS) + off : nullptr;
  a.gradResidual = gradResidual != nullptr ? static_cast<char*>(gradResidual) + off : nullptr;
  a.gradPartial = static_cast<char*>(gradPartial) + off;
  a.gamma = gamma;
  a.ws = static_cast<float*>(workspace);
  a.rows = n;
  a.hidden = hidden;
  a.eps = eps;
  a.vectors = v.vectors;
  a.vecWeight = v.vec[0];
  a.vecNormBias = v.vec[1];
  a.vecBias = v.vec[2];
  a.first = first ? 1 : 0;
  return a;
}

}  // namespace

int allreduceResidualNorm(PeerContext& pc, const void* partial, const void* residual, void* residualOut, void* out,
                          const void* bias, const void* gamma, const void* beta, size_t rows, size_t hidden,
                          DataType dt, int norm, float eps, AllreduceAlgo algo, cudaStream_t stream,
                          float* outScales) {
  GLB_TRACE_RANGE("glb::cuda::allreduceResidualNorm");
  pc.checkHealth();
  const char* op = "allreduce_residual_norm";
  const size_t rb = hidden * elementSize(dt);
  const NormRange inputs[] = {{"partial", partial, rows * rb}, {"residual", residual, rows * rb}, {"bias", bias, rb},
                              {"weight", gamma, rb}, {"norm_bias", beta, rb}};
  const NormOutputs outputs = normOutputs(residualOut, out, outScales, rows, rows, hidden, dt, norm);
  checkNormCall(op, dt, norm, hidden, normRequired(rows, inputs, outputs.r, norm), kNormRequired, inputs, outputs.r, 1);
  checkNormQuant(op, norm, hidden, outScales);
  if (rows == 0) return kNormLocal;
  const NormPlan plan = planResidualNorm(pc, rows, hidden, dt, norm, algo, outScales != nullptr);
  DeviceGuard g(pc.device);
  const auto l = layoutOf(pc);
  const size_t rowBytes = hidden * elementSize(dt);
  for (size_t r0 = 0; r0 < rows; r0 += plan.chunkRows) {
    const size_t n = std::min(plan.chunkRows, rows - r0);
    NormArgs a = chunkArgs(partial, residual, residualOut, out, bias, gamma, beta, r0 * rowBytes, n, hidden, norm, eps);
    quantChunk(a, out, outScales, r0, hidden);
    NormXchg x{};
    switch (plan.variant) {
      case kNormLL:
        x.peers = pc.llPtrs();
        x.srcStride = pc.llSrcStride();
        x.parityStride = pc.llParityStride();
        break;
      case kNormOneShot:
        x.peers = pc.stagePtrs(0);
        x.parityStride = l.half;
        break;
      case kNormTwoShot: x.peers = pc.stagePtrs(l.bulkOff); break;
      default: break;
    }
    x.mine = x.peers.p[pc.rank];
    launchNormChunk(pc, a, x, dt, norm, plan.variant, n, stream, op);
  }
  return plan.variant;
}

int reduceScatterResidualNorm(PeerContext& pc, const void* partial, const void* residual, void* residualOut, void* out,
                              const void* bias, const void* gamma, const void* beta, size_t rows, size_t hidden,
                              DataType dt, int norm, float eps, bool gatherOut, cudaStream_t stream,
                              float* outScales) {
  GLB_TRACE_RANGE("glb::cuda::reduceScatterResidualNorm");
  pc.checkHealth();
  const char* op = "reduce_scatter_residual_norm";
  const size_t P = static_cast<size_t>(pc.size), shard = rows / P;
  const size_t rb = hidden * elementSize(dt);
  const NormRange inputs[] = {{"partial", partial, rows * rb}, {"residual", residual, shard * rb}, {"bias", bias, rb},
                              {"weight", gamma, rb}, {"norm_bias", beta, rb}};
  const NormOutputs outputs = normOutputs(residualOut, out, outScales, shard, gatherOut ? rows : shard, hidden, dt, norm);
  checkNormCall(op, dt, norm, hidden, normRequired(rows, inputs, outputs.r, norm), kNormRequired, inputs, outputs.r, 1);
  checkNormQuant(op, norm, hidden, outScales);
  GLB_NORM_CHECK(rows % P == 0, rows, " rows do not split into ", P, " equal shards");
  if (P == 1) {
    return allreduceResidualNorm(pc, partial, residual, residualOut, out, bias, gamma, beta, rows, hidden, dt, norm,
                                 eps, AllreduceAlgo::AUTO, stream, outScales);
  }
  if (rows == 0) return kNormScatter;
  const NormPlan plan = planReduceScatterNorm(pc, rows, hidden, dt, norm, gatherOut, outScales != nullptr);
  DeviceGuard g(pc.device);
  const size_t rowBytes = hidden * elementSize(dt);
  NormXchg x{};
  x.peers = pc.stagePtrs(layoutOf(pc).bulkOff);
  x.mine = x.peers.p[pc.rank];
  x.shardRows = shard;
  x.gather = gatherOut ? 1 : 0;
  // Chunk rows [r0, r0 + n) of every shard: the same byte offset into the partial, the shard
  // tensors and a gathered out, whose other shards lie shardRows further on.
  for (size_t r0 = 0; r0 < shard; r0 += plan.chunkRows) {
    const size_t n = std::min(plan.chunkRows, shard - r0);
    NormArgs a = chunkArgs(partial, residual, residualOut, out, bias, gamma, beta, r0 * rowBytes, n, hidden, norm, eps);
    quantChunk(a, out, outScales, r0, hidden);
    launchNormChunk(pc, a, x, dt, norm, kNormScatter, P * n, stream, op);
  }
  return kNormScatter;
}

int reduceScatterResidualNormBackward(PeerContext& pc, const void* gradOut, const void* s, const void* gradS,
                                      void* gradResidual, void* gradPartial, const void* gamma, void* gradWeight,
                                      void* gradNormBias, void* gradBias, void* workspace, size_t workspaceBytes,
                                      size_t rows, size_t hidden, DataType dt, int norm, float eps, bool gatherOut,
                                      cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::reduceScatterResidualNormBackward");
  pc.checkHealth();
  const char* op = "reduce_scatter_residual_norm_backward";
  const size_t P = static_cast<size_t>(pc.size), shard = rows / P;
  GLB_NORM_CHECK(norm == kNormRms || norm == kNormLayer, "needs a norm (rms or layer), got ", norm);
  GLB_NORM_CHECK(norm == kNormLayer || gradNormBias == nullptr, "grad_norm_bias needs a layer norm");
  const size_t rb = hidden * elementSize(dt);
  const NormRange inputs[] = {{"grad_out", gradOut, (gatherOut ? rows : shard) * rb},
                              {"residual_out", s, shard * rb},
                              {"grad_residual_out", gradS, shard * rb},
                              {"weight", gamma, rb}};
  const NormRange outputs[] = {{"grad_residual", gradResidual, shard * rb}, {"grad_partial", gradPartial, rows * rb},
                               {"grad_weight", gradWeight, rb}, {"grad_norm_bias", gradNormBias, rb},
                               {"grad_bias", gradBias, rb}, {"workspace", workspace, workspaceBytes}};
  checkNormCall(op, dt, norm, hidden, rows == 0 || (gradOut != nullptr && s != nullptr && gradPartial != nullptr),
                "grad_out, residual_out and grad_partial are required", inputs, outputs, 2);
  GLB_NORM_CHECK(rows % P == 0, rows, " rows do not split into ", P, " equal shards");
  void* const vecOut[3] = {gradWeight, gradNormBias, gradBias};
  const VecSlots slots = vecSlots(vecOut);
  const int vectors = slots.vectors;
  const NormBackwardPlan plan = planReduceScatterNormBackward(pc, rows, hidden, dt, norm, gatherOut, vectors);
  GLB_NORM_CHECK(workspaceBytes >= plan.workspaceBytes, "the workspace of ", workspaceBytes, " bytes is below the ",
                 plan.workspaceBytes, " the plan needs");
  GLB_NORM_CHECK(plan.workspaceBytes == 0 || workspace != nullptr, "the column sums need a workspace");
  DeviceGuard g(pc.device);
  if (shard == 0) {
    // Nothing to sum: the vector gradients are zero.
    for (void* v : vecOut) {
      if (v != nullptr) GLB_CUDA_CHECK(cudaMemsetAsync(v, 0, rb, stream));
    }
    return plan.variant;
  }
  NormXchg x{};
  if (plan.variant == kNormScatter) {
    x.peers = pc.stagePtrs(layoutOf(pc).bulkOff);
    x.mine = x.peers.p[pc.rank];
    x.shardRows = shard;
    x.gather = gatherOut ? 1 : 0;
  }
  // Chunk rows [r0, r0 + n) of every shard, as in the forward. The grid of every chunk but a
  // shorter last one is plan.blocks; CTA b carries its column sums in workspace slot b.
  for (size_t r0 = 0; r0 < shard; r0 += plan.chunkRows) {
    const size_t n = std::min(plan.chunkRows, shard - r0);
    const NormBwdArgs a = bwdChunkArgs(gradOut, s, gradS, gradResidual, gradPartial, gamma, workspace, r0 * rb, n,
                                       hidden, eps, slots, r0 == 0);
    const size_t gridRows = plan.variant == kNormScatter ? P * n : n;
    const int blocks = static_cast<int>(std::min<size_t>(gridRows, static_cast<size_t>(plan.blocks)));
    prologue(pc, stream);
    launchNormBackward(pc.comm(), a, x, dt, norm, plan.variant, blocks, stream);
    finish(pc, stream, op);
  }
  if (vectors > 0) {
    // The first chunk's grid is plan.blocks and wrote every slot; later chunks use a prefix.
    launchNormBackwardFinish(static_cast<const float*>(workspace), plan.blocks, vectors, hidden, slots.out, dt, stream);
    checkLaunch(op);
  }
  return plan.variant;
}

int allreduceResidualNormBackward(PeerContext& pc, const void* gradOut, const void* s, const void* gradS,
                                  void* gradPartial, const void* gamma, void* gradWeight, void* gradNormBias,
                                  void* gradBias, void* workspace, size_t workspaceBytes, size_t rows, size_t hidden,
                                  DataType dt, int norm, float eps, AllreduceAlgo algo, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::allreduceResidualNormBackward");
  pc.checkHealth();
  const char* op = "allreduce_residual_norm_backward";
  GLB_NORM_CHECK(norm == kNormRms || norm == kNormLayer, "needs a norm (rms or layer), got ", norm);
  GLB_NORM_CHECK(norm == kNormLayer || gradNormBias == nullptr, "grad_norm_bias needs a layer norm");
  const size_t rb = hidden * elementSize(dt);
  const NormRange inputs[] = {{"grad_out", gradOut, rows * rb},
                              {"residual_out", s, rows * rb},
                              {"grad_residual_out", gradS, rows * rb},
                              {"weight", gamma, rb}};
  const NormRange outputs[] = {{"grad_partial", gradPartial, rows * rb}, {"grad_weight", gradWeight, rb},
                               {"grad_norm_bias", gradNormBias, rb},     {"grad_bias", gradBias, rb},
                               {"workspace", workspace, workspaceBytes}};
  checkNormCall(op, dt, norm, hidden, rows == 0 || (gradOut != nullptr && s != nullptr && gradPartial != nullptr),
                "grad_out, residual_out and grad_partial are required", inputs, outputs, 2);
  void* const vecOut[3] = {gradWeight, gradNormBias, gradBias};
  const VecSlots slots = vecSlots(vecOut);
  const int vectors = slots.vectors;
  const NormBackwardPlan plan = planResidualNormBackward(pc, rows, hidden, dt, norm, vectors, algo);
  GLB_NORM_CHECK(workspaceBytes >= plan.workspaceBytes, "the workspace of ", workspaceBytes, " bytes is below the ",
                 plan.workspaceBytes, " the plan needs");
  GLB_NORM_CHECK(plan.workspaceBytes == 0 || workspace != nullptr, "the column sums need a workspace");
  DeviceGuard g(pc.device);
  if (rows == 0) {
    // Nothing to sum: the vector gradients are zero.
    for (void* v : vecOut) {
      if (v != nullptr) GLB_CUDA_CHECK(cudaMemsetAsync(v, 0, rb, stream));
    }
    return plan.variant;
  }
  const auto l = layoutOf(pc);
  NormXchg x{};
  if (plan.variant == kNormOneShot) {
    x.peers = pc.stagePtrs(0);
    x.parityStride = l.half;
  } else if (plan.variant == kNormTwoShot) {
    x.peers = pc.stagePtrs(l.bulkOff);
  }
  x.mine = x.peers.p[pc.rank];
  // The grid of every chunk but a shorter last one is plan.blocks; CTA b carries its column sums in
  // workspace slot b.
  for (size_t r0 = 0; r0 < rows; r0 += plan.chunkRows) {
    const size_t n = std::min(plan.chunkRows, rows - r0);
    const NormBwdArgs a = bwdChunkArgs(gradOut, s, gradS, nullptr, gradPartial, gamma, workspace, r0 * rb, n, hidden,
                                       eps, slots, r0 == 0);
    const int blocks = static_cast<int>(std::min<size_t>(n, static_cast<size_t>(plan.blocks)));
    prologue(pc, stream);
    launchNormBackward(pc.comm(), a, x, dt, norm, plan.variant, blocks, stream);
    finish(pc, stream, op);
  }
  if (vectors == 0) return plan.variant;
  const float* ws = static_cast<const float*>(workspace);
  if (plan.variant == kNormTwoShot) {
    // The CTA sums cover this rank's rows: a collective finish sums them over the ranks.
    const int threads = normBackwardFinishThreads();
    const int blocks = static_cast<int>(std::min<size_t>(
        ceilDiv(static_cast<size_t>(vectors) * hidden, static_cast<size_t>(threads)),
        static_cast<size_t>(pc.coResidentBlocks(normBackwardFinishAllreduceKernelFor(dt), threads))));
    prologue(pc, stream);
    launchNormBackwardFinishAllreduce(pc.comm(), ws, plan.blocks, vectors, hidden, slots.out, x.peers, dt, blocks,
                                      stream);
    finish(pc, stream, op);
  } else {
    launchNormBackwardFinish(ws, plan.blocks, vectors, hidden, slots.out, dt, stream);
    checkLaunch(op);
  }
  return plan.variant;
}

#undef GLB_NORM_CHECK


// ---- data movement ---------------------------------------------------------------------

namespace {

std::vector<size_t> prefix(const std::vector<size_t>& v) {
  std::vector<size_t> off(v.size() + 1, 0);
  for (size_t i = 0; i < v.size(); i++) off[i + 1] = off[i] + v[i];
  return off;
}

// A view of the pool's bulk region as a PeerBuffer-like target for staged calls.
struct StagedOut {
  PeerPtrs ptrs;
  void* mc;
  char* mine;
};

StagedOut stagedBulk(const PeerContext& pc, size_t needBytes, const char* what) {
  const auto l = layoutOf(pc);
  GLB_ENFORCE_LE(needBytes, l.bulkBytes, what, ": ", needBytes,
                 " bytes do not fit the staging pool; register the buffer (PeerContext::registerBuffer / "
                 "allocSymmetric) or raise GLB_CUDA_STAGE_MB");
  StagedOut s;
  s.ptrs = pc.stagePtrs(l.bulkOff);
  s.mc = pc.stageMc(l.bulkOff);
  s.mine = static_cast<char*>(s.ptrs.p[pc.rank]);
  return s;
}

// Store-only kernels (broadcast / gather / alltoall pushes) are light on registers, so two
// CTAs per SM stay co-resident: their cap is 2x the reduce kernels'.
// Grid of a store-only kernel: enough CTAs for `workBytes`, at most what the tuning table (keyed
// by `keyBytes`) or the copyBlocks knob allows, and never more than can be co-resident for THIS
// kernel (occupancy query: every CTA waits for its twin on the peers, so all must be running).
int bwBlocks(PeerContext& pc, const char* coll, const void* kernel, size_t workBytes, size_t keyBytes = ~size_t(0)) {
  if (keyBytes == ~size_t(0)) keyBytes = workBytes;
  size_t want = ceilDiv(std::max<size_t>(workBytes / 16, 1), static_cast<size_t>(kThreads) * 4);
  const int resident = kernel != nullptr ? pc.coResidentBlocks(kernel) : pc.maxBlocks();
  int cap = std::min({tuning().copyBlocks, resident, kMaxBlocks});
  if (const TuneEntry* e = TuningTable::get().lookup(coll, pc.size, BufKind::REGISTERED, keyBytes)) {
    if (e->blocks > 0) cap = std::min({e->blocks, resident, kMaxBlocks});
  }
  return std::max(1, static_cast<int>(std::min<size_t>(want, static_cast<size_t>(cap))));
}

}  // namespace

namespace {
// Launch shape of one broadcast kernel. mode 0 = root pushes everything, 1 = scatter +
// allgather, 2 = multimem.st, 3 = chunk-pipelined relay (see broadcastKernel).
struct BcastShape {
  int mode = 0;
  int blocks = 1;
  int tile = 0;
};

BcastShape planBroadcast(PeerContext& pc, size_t bytes, bool vec, bool hasMc) {
  const auto& t = tuning();
  BcastShape sh;
  const TuneEntry* e = TuningTable::get().lookup("broadcast", pc.size, BufKind::REGISTERED, bytes);
  // multimem.st pays off when the root would otherwise send P-1 copies: P > 2. From
  // bcastRelayMinBytes up the pipelined relay keeps every link busy instead.
  if (pc.size > 2 && vec && bytes >= t.bcastRelayMinBytes) {
    sh.mode = 3;
  } else if (hasMc && vec && pc.size > 2 && bytes >= t.bcastDirectMaxBytes) {
    sh.mode = 2;
  } else if (bytes > t.bcastDirectMaxBytes && pc.size > 2) {
    sh.mode = 1;
  }
  if (e != nullptr) {
    if (e->algo == "relay" && vec && pc.size > 2) sh.mode = 3;
    if (e->algo == "nvls" && hasMc && vec) sh.mode = 2;
    if (e->algo == "scatter" && pc.size > 2) sh.mode = 1;
    if (e->algo == "direct") sh.mode = 0;
  }
  long forced = envInt("CUDA_BCAST_MODE", -1);
  if (forced >= 0 && forced <= 3 && (forced != 2 || (hasMc && vec)) && (forced != 3 || (vec && pc.size > 2))) {
    sh.mode = static_cast<int>(forced);
  }
  sh.blocks = bwBlocks(pc, "broadcast", broadcastKernelPtr(), sh.mode == 1 ? bytes / pc.size * 2 : bytes, bytes);
  if (sh.mode == 3) {
    // Tiles of at least 8 KB per CTA (one full pass of the CTA), at least ~4 chunks in flight
    // behind each other; small payloads use fewer CTAs rather than smaller tiles.
    const size_t units = bytes / 16;
    const size_t R = static_cast<size_t>(pc.size - 1);
    long tile = envInt("CUDA_BCAST_TILE", e != nullptr && e->tile > 0 ? e->tile : 0);
    if (tile <= 0) {
      tile = 512;
      while (tile < 4096 && units / (R * static_cast<size_t>(sh.blocks) * static_cast<size_t>(tile) * 2) >= 8) tile *= 2;
    }
    sh.tile = static_cast<int>(tile);
    const size_t fit = std::max<size_t>(units / (R * static_cast<size_t>(sh.tile) * 4), 1);
    sh.blocks = static_cast<int>(std::min<size_t>(static_cast<size_t>(sh.blocks), fit));
  }
  return sh;
}
}  // namespace

void broadcast(PeerContext& pc, const PeerBuffer& buf, size_t byteOffset, size_t bytes, int root,
               cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::broadcast");
  if (bytes == 0 || pc.size == 1) return;
  GLB_ENFORCE(root >= 0 && root < pc.size, "broadcast: invalid root ", root);
  GLB_ENFORCE_LE(byteOffset + bytes, buf.bytes, "broadcast range exceeds the registered buffer");
  DeviceGuard g(pc.device);
  const bool vec = buf.vectorOk && byteOffset % 16 == 0;
  const BcastShape sh = planBroadcast(pc, bytes, vec, buf.mc != nullptr);
  prologue(pc, stream);
  launchBroadcast(pc.comm(), buf.ptrsAt(byteOffset), buf.mc ? static_cast<char*>(buf.mc) + byteOffset : nullptr,
                  bytes, root, sh.mode, vec, sh.blocks, sh.tile, stream);
  finish(pc, stream, "broadcast");
}

void broadcast(PeerContext& pc, void* ptr, size_t bytes, int root, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::broadcast(staged)");
  if (bytes == 0 || pc.size == 1) return;
  DeviceGuard g(pc.device);
  const auto l = layoutOf(pc);
  const size_t piece = l.bulkBytes / 16 * 16;
  PeerPtrs stage = pc.stagePtrs(l.bulkOff);
  char* mine = static_cast<char*>(stage.p[pc.rank]);
  for (size_t done = 0; done < bytes; done += piece) {
    const size_t n = std::min(piece, bytes - done);
    char* p = static_cast<char*>(ptr) + done;
    if (pc.rank == root) GLB_CUDA_CHECK(cudaMemcpyAsync(mine, p, n, cudaMemcpyDeviceToDevice, stream));
    const BcastShape sh = planBroadcast(pc, n, true, pc.nvlsAvailable());
    prologue(pc, stream);
    launchBroadcast(pc.comm(), stage, pc.stageMc(l.bulkOff), n, root, sh.mode, true, sh.blocks, sh.tile, stream);
    finish(pc, stream, "broadcast(staged)");
    if (pc.rank != root) GLB_CUDA_CHECK(cudaMemcpyAsync(p, mine, n, cudaMemcpyDeviceToDevice, stream));
  }
}

namespace {
void gatherCommon(PeerContext& pc, const void* in, const PeerPtrs& outs, void* mcOut, bool vecOut,
                  const std::vector<size_t>& bytesPerRank, int onlyDst, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::allgather/gather");
  GLB_ENFORCE_EQ(static_cast<int>(bytesPerRank.size()), pc.size, "need one byte count per rank");
  auto off = prefix(bytesPerRank);
  const bool vec = vecOut && reinterpret_cast<uintptr_t>(in) % 16 == 0;
  // The barrier pairs CTA b with CTA b of every peer: the grid must be the same on every
  // rank, so it is sized from the LARGEST block (every rank holds the whole size vector).
  const size_t largest = *std::max_element(bytesPerRank.begin(), bytesPerRank.end());
  prologue(pc, stream);
  launchGatherPush(pc.comm(), in, outs, mcOut, off.data(), bytesPerRank.data(), onlyDst, vec,
                   bwBlocks(pc, "allgather", gatherPushKernelPtr(), largest), stream);
  finish(pc, stream, "allgather/gather");
}

// Plain pointers whose payload is larger than the pool's bulk region: one kernel pipelines
// copy-in and pull through two pool slots (pipeline_kernels.cu). Every rank holds the whole
// size vector and the same pool size, so all ranks pick this path together.
bool exceedsBulk(const PeerContext& pc, size_t bytes) { return bytes > layoutOf(pc).bulkBytes; }

void runPipelinedGather(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& bytesPerRank, int onlyDst,
                        cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::allgather/gather(pipelined)");
  GLB_ENFORCE_EQ(static_cast<int>(bytesPerRank.size()), pc.size, "need one byte count per rank");
  auto off = prefix(bytesPerRank);
  const size_t largest = *std::max_element(bytesPerRank.begin(), bytesPerRank.end());
  const PipeShape sh = pipeShape(pc, pipelinedAllgatherKernelPtr(), 2, 1, largest, 0, 0, 0, "allgather / gather");
  prologue(pc, stream);
  launchPipelinedAllgather(pc.comm(), in, out, off.data(), bytesPerRank.data(), onlyDst,
                           pc.stagePtrs(layoutOf(pc).bulkOff), sh.tile, sh.xthreads, sh.blocks, stream);
  finish(pc, stream, "allgather/gather(pipelined)");
}

bool allEqual(const std::vector<size_t>& v) {
  for (size_t x : v) {
    if (x != v[0]) return false;
  }
  return true;
}

// Small uniform allgather / alltoall: flag-in-data lines, no barrier, any output pointer.
bool tryLLExchange(PeerContext& pc, const void* in, void* outLocal, size_t bytesPerBlock, int mode,
                   cudaStream_t stream) {
  size_t limit = std::min(tuning().llMaxBytes, pc.llMaxBytes());
  if (const TuneEntry* e = TuningTable::get().lookup(mode == 0 ? "allgather" : "alltoall", pc.size, BufKind::REGISTERED,
                                                     bytesPerBlock)) {
    if (e->algo != "ll") return false;
    limit = pc.llMaxBytes();
  }
  if (bytesPerBlock == 0 || bytesPerBlock > limit || envFlag("CUDA_LL_DISABLE", false)) return false;
  const size_t units = ceilDiv(bytesPerBlock, size_t(8)) * pc.size;
  int threads = static_cast<int>(std::min<size_t>(kThreads, roundUp(std::max<size_t>(units, 32), 32)));
  int blocks = static_cast<int>(std::min<size_t>(ceilDiv(units, static_cast<size_t>(threads)), 16));
  blocks = std::max(1, std::min(blocks, pc.maxBlocks()));
  prologue(pc, stream);
  launchLLExchange(pc.comm(), in, outLocal, bytesPerBlock, mode, pc.llPtrs(), pc.llSrcStride(), pc.llParityStride(), blocks,
                   threads, stream);
  finish(pc, stream, "ll exchange");
  return true;
}
}  // namespace

void allgatherv(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset,
                const std::vector<size_t>& bytesPerRank, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  auto off = prefix(bytesPerRank);
  GLB_ENFORCE_LE(outOffset + off.back(), out.bytes, "allgather output exceeds the registered buffer");
  if (pc.size == 1) {
    char* dst = static_cast<char*>(out.local) + outOffset;
    if (dst != in && off.back() > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, in, off.back(), cudaMemcpyDeviceToDevice, stream));
    return;
  }
  if (allEqual(bytesPerRank) &&
      tryLLExchange(pc, in, static_cast<char*>(out.local) + outOffset, bytesPerRank[0], 0, stream)) {
    return;
  }
  // No multicast here: an allgather's bottleneck is what every GPU RECEIVES ((P-1)/P of the
  // output either way); multimem.st would only relieve the uplink and additionally deliver
  // each block back to its sender.
  gatherCommon(pc, in, out.ptrsAt(outOffset), nullptr, out.vectorOk && outOffset % 16 == 0, bytesPerRank, -1, stream);
}

void allgatherv(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& bytesPerRank,
                cudaStream_t stream) {
  DeviceGuard g(pc.device);
  auto off = prefix(bytesPerRank);
  if (pc.size == 1) {
    if (out != in && off.back() > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, off.back(), cudaMemcpyDeviceToDevice, stream));
    return;
  }
  if (allEqual(bytesPerRank) && tryLLExchange(pc, in, out, bytesPerRank[0], 0, stream)) return;
  if (exceedsBulk(pc, off.back())) {
    runPipelinedGather(pc, in, out, bytesPerRank, -1, stream);
    return;
  }
  auto st = stagedBulk(pc, off.back(), "allgather");
  gatherCommon(pc, in, st.ptrs, nullptr, true, bytesPerRank, -1, stream);
  if (off.back() > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, st.mine, off.back(), cudaMemcpyDeviceToDevice, stream));
}

void gatherv(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset,
             const std::vector<size_t>& bytesPerRank, int root, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_ENFORCE(root >= 0 && root < pc.size, "gather: invalid root ", root);
  if (pc.size == 1) {
    char* dst = static_cast<char*>(out.local) + outOffset;
    if (dst != in && bytesPerRank[0] > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, in, bytesPerRank[0], cudaMemcpyDeviceToDevice, stream));
    return;
  }
  gatherCommon(pc, in, out.ptrsAt(outOffset), nullptr, out.vectorOk && outOffset % 16 == 0, bytesPerRank, root, stream);
}

void gatherv(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& bytesPerRank, int root,
             cudaStream_t stream) {
  DeviceGuard g(pc.device);
  auto off = prefix(bytesPerRank);
  if (pc.size == 1) {
    if (out != in && off.back() > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, off.back(), cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(root >= 0 && root < pc.size, "gather: invalid root ", root);
  if (exceedsBulk(pc, off.back())) {
    runPipelinedGather(pc, in, out, bytesPerRank, root, stream);
    return;
  }
  auto st = stagedBulk(pc, off.back(), "gather");
  gatherCommon(pc, in, st.ptrs, nullptr, true, bytesPerRank, root, stream);
  if (pc.rank == root && off.back() > 0) {
    GLB_CUDA_CHECK(cudaMemcpyAsync(out, st.mine, off.back(), cudaMemcpyDeviceToDevice, stream));
  }
}

namespace {
// `uniform` is a property of the ENTRY POINT (alltoall() vs alltoallv()), never derived from
// this rank's own tables: ranks of one alltoallv call may hold tables that look uniform
// locally while a peer's do not, and they must all run the same protocol. The v-variant
// therefore always exchanges receive offsets through the signal pads and always launches
// the same fixed grid (its byte counts are rank-local, the grid must not be).
void alltoallCommon(PeerContext& pc, const void* in, const std::vector<size_t>& sendBytes, const PeerPtrs& outs,
                    bool vecOut, const std::vector<size_t>& recvBytes, bool uniform, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::alltoall");
  GLB_ENFORCE_EQ(static_cast<int>(sendBytes.size()), pc.size, "alltoall: need one send size per rank");
  GLB_ENFORCE_EQ(static_cast<int>(recvBytes.size()), pc.size, "alltoall: need one recv size per rank");
  auto soff = prefix(sendBytes);
  auto roff = prefix(recvBytes);
  // dstOff[j] = where my chunk lands in rank j's output = rank j's receive offset
  // for source `me`. For the uniform case that is me * chunk; for the v-variant the
  // kernel reads it from rank j's pad (published there before the first barrier).
  std::vector<size_t> dstOff(pc.size);
  for (int j = 0; j < pc.size; j++) dstOff[j] = uniform ? static_cast<size_t>(pc.rank) * sendBytes[0] : ~size_t(0);
  const bool vec = vecOut && reinterpret_cast<uintptr_t>(in) % 16 == 0;
  int blocks;
  if (uniform) {
    blocks = bwBlocks(pc, "alltoall", alltoallPushKernelPtr(), soff.back(), sendBytes[0]);
  } else {
    blocks = std::max(1, std::min({tuning().alltoallvBlocks, pc.coResidentBlocks(alltoallPushKernelPtr()), kMaxBlocks}));
  }
  prologue(pc, stream);
  launchAlltoallPush(pc.comm(), in, outs, soff.data(), sendBytes.data(), dstOff.data(), uniform ? nullptr : roff.data(),
                     -1, vec, blocks, stream);
  finish(pc, stream, "alltoall");
}

// Plain pointers beyond the staged path: one kernel streams the blocks through two pool slots
// (pipeline_kernels.cu). `shapeBytes` sizes the launch and must be the same on every rank: the grid
// and the tile feed the step count and the barrier pairing.
void runPipelinedAlltoall(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& sendBytes,
                          const std::vector<size_t>& recvBytes, size_t shapeBytes, const char* what,
                          cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::alltoall/scatter(pipelined)");
  GLB_ENFORCE_EQ(static_cast<int>(sendBytes.size()), pc.size, what, ": need one send size per rank");
  GLB_ENFORCE_EQ(static_cast<int>(recvBytes.size()), pc.size, what, ": need one recv size per rank");
  auto soff = prefix(sendBytes);
  auto roff = prefix(recvBytes);
  const PipeShape sh = pipeShape(pc, pipelinedAlltoallKernelPtr(), 2, pc.size, shapeBytes, 0, 0, 0, what);
  prologue(pc, stream);
  launchPipelinedAlltoall(pc.comm(), in, out, soff.data(), sendBytes.data(), roff.data(), recvBytes.data(),
                          pc.stagePtrs(layoutOf(pc).bulkOff), sh.tile, sh.xthreads, sh.blocks, stream);
  finish(pc, stream, what);
}

// The pipelined exchange writes the output while later chunks of the input are still to be read,
// so, as in NCCL, the two buffers must not overlap. The check sees this rank's pointers only: a
// rank that raises here does not launch, and peers that did launch wait for it until the timeout.
void rejectOverlap(const void* in, size_t inBytes, const void* out, size_t outBytes, const char* what) {
  const uintptr_t i = reinterpret_cast<uintptr_t>(in), o = reinterpret_cast<uintptr_t>(out);
  if (inBytes > 0 && outBytes > 0 && i < o + outBytes && o < i + inBytes) {
    GLB_THROW(InputException, what, ": the input and output buffers overlap, which is not supported");
  }
}
}  // namespace

void alltoall(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset, size_t bytes,
              cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_ENFORCE_LE(outOffset + bytes * pc.size, out.bytes, "alltoall output exceeds the registered buffer");
  char* dst = static_cast<char*>(out.local) + outOffset;
  if (pc.size == 1) {
    if (dst != in && bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  if (tryLLExchange(pc, in, dst, bytes, 1, stream)) return;
  // The push kernel stores my chunk for rank j into rank j's output while rank j may still be
  // reading its own chunk for me from that address: in place, that would be a race.
  rejectOverlap(in, bytes * pc.size, dst, bytes * pc.size, "alltoall");
  std::vector<size_t> sizes(pc.size, bytes);
  alltoallCommon(pc, in, sizes, out.ptrsAt(outOffset), out.vectorOk && outOffset % 16 == 0, sizes, true, stream);
}

void alltoall(PeerContext& pc, const void* in, void* out, size_t bytes, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  if (pc.size == 1) {
    if (out != in && bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  if (tryLLExchange(pc, in, out, bytes, 1, stream)) return;
  if (exceedsBulk(pc, bytes * pc.size)) {
    rejectOverlap(in, bytes * pc.size, out, bytes * pc.size, "alltoall");
    std::vector<size_t> sizes(pc.size, bytes);
    runPipelinedAlltoall(pc, in, out, sizes, sizes, bytes * pc.size, "alltoall(pipelined)", stream);
    return;
  }
  auto st = stagedBulk(pc, bytes * pc.size, "alltoall");
  std::vector<size_t> sizes(pc.size, bytes);
  alltoallCommon(pc, in, sizes, st.ptrs, true, sizes, true, stream);
  if (bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, st.mine, bytes * pc.size, cudaMemcpyDeviceToDevice, stream));
}

void alltoallv(PeerContext& pc, const void* in, const std::vector<size_t>& sendBytes, const PeerBuffer& out,
               size_t outOffset, const std::vector<size_t>& recvBytes, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  auto roff = prefix(recvBytes);
  GLB_ENFORCE_LE(outOffset + roff.back(), out.bytes, "alltoall output exceeds the registered buffer");
  if (pc.size == 1) {
    char* dst = static_cast<char*>(out.local) + outOffset;
    if (dst != in && sendBytes[0] > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, in, sendBytes[0], cudaMemcpyDeviceToDevice, stream));
    return;
  }
  // As for alltoall: the push kernel writes peers' outputs while they still read their inputs.
  rejectOverlap(in, prefix(sendBytes).back(), static_cast<const char*>(out.local) + outOffset, roff.back(), "alltoallv");
  alltoallCommon(pc, in, sendBytes, out.ptrsAt(outOffset), out.vectorOk && outOffset % 16 == 0, recvBytes, false, stream);
}

void alltoallv(PeerContext& pc, const void* in, const std::vector<size_t>& sendBytes, void* out,
               const std::vector<size_t>& recvBytes, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  if (pc.size == 1) {
    if (out != in && sendBytes[0] > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, sendBytes[0], cudaMemcpyDeviceToDevice, stream));
    return;
  }
  rejectOverlap(in, prefix(sendBytes).back(), out, prefix(recvBytes).back(), "alltoallv");
  // Always the pipelined kernel: the byte counts are rank-local, so no rule that every rank
  // evaluates alike could choose between it and a staged launch. The kernel agrees on its step
  // count on the device, and its launch shape comes from the pool size alone.
  runPipelinedAlltoall(pc, in, out, sendBytes, recvBytes, layoutOf(pc).bulkBytes, "alltoallv(pipelined)", stream);
}

namespace {
// The limits the device-split MoE calls share, named after the public operation. Rows are
// `rowBytes` (quantising: H codes, H a multiple of kFp8Block) and a multiple of `rowMultiple`.
void checkMoeLimits(const char* name, int experts, int align, size_t rowBytes, size_t rowMultiple) {
  GLB_ENFORCE(experts >= 1 && experts <= kMaxA2aExperts, name, ": experts per rank must be in 1..", kMaxA2aExperts,
              ", got ", experts);
  GLB_ENFORCE(align >= 1, name, ": align must be at least 1, got ", align);
  GLB_ENFORCE(rowBytes > 0 && rowBytes <= 0xffffffffull, name, ": row size must be 1 byte .. 4 GB, got ", rowBytes);
  GLB_ENFORCE(rowBytes % rowMultiple == 0, name, ": the row size must be a positive multiple of ", rowMultiple,
              " bytes, got ", rowBytes);
}

void checkTopk(const char* name, int topk) {
  GLB_ENFORCE(topk >= 1 && topk <= 32, name, ": topk must be in 1..32, got ", topk);
}

void checkAligned16(const char* name, const void* a, const void* b, const char* what) {
  GLB_ENFORCE(reinterpret_cast<uintptr_t>(a) % 16 == 0 && reinterpret_cast<uintptr_t>(b) % 16 == 0, name, ": ", what,
              " must be 16-byte aligned");
}

// What a kernel needs from a MoeOut (and, quantising, its scales): every rank's rows in place or
// its staging area, my staged pointers, and the capacity in rows. Registered: bounds-checked
// against the registration, zero copy. Plain: staged through the pool's bulk region, where a row
// takes rowBytes, plus its scales after the capacity's codes (hidden is a multiple of 128, so they
// start 16-byte aligned); that caps the capacity.
// The combine's backward adds a gradient buffer of expert_out's shape (`grad`), of the same kind:
// registered, every rank's in place; plain, the rows after the staged expert_out's capacity in
// each staging area, so a row then takes 2·rowBytes of the pool.
struct MoeTarget {
  PeerPtrs peers;
  MoeScales scales;
  const char* mine;  // my rows, wherever they are read or written by this rank's caller
  char* staged;      // my plain tensor (null if it is empty)
  bool plain;
  size_t capRows;
  PeerPtrs grads;       // registered grad only
  char* gradMine;       // my grad rows
};

MoeTarget resolveMoeOut(const PeerContext& pc, const char* name, const char* what, const MoeOut& out,
                        const MoeOut* scales, size_t capacityRows, size_t rowBytes, const MoeOut* grad = nullptr) {
  if (scales != nullptr && (out.buf == nullptr) != (scales->buf == nullptr)) {
    GLB_THROW(InputException, name, ": out and out_scales must both be registered / symmetric or both plain");
  }
  if (grad != nullptr && (out.buf == nullptr) != (grad->buf == nullptr)) {
    GLB_THROW(InputException, name, ": expert_out and grad_expert_out must both be registered / symmetric or both plain");
  }
  const size_t scaleBytes = scales != nullptr ? rowBytes / kFp8Block * sizeof(float) : 0;
  const size_t gradBytes = grad != nullptr ? rowBytes : 0;
  MoeTarget t{};
  if (out.buf != nullptr) {
    GLB_ENFORCE_LE(out.offset + capacityRows * rowBytes, out.buf->bytes, name, ": ", what,
                   " exceeds the registered buffer");
    t.peers = out.buf->ptrsAt(out.offset);
    t.mine = static_cast<const char*>(out.buf->local) + out.offset;
    t.capRows = capacityRows;
    if (grad != nullptr) {
      GLB_ENFORCE_LE(grad->offset + capacityRows * rowBytes, grad->buf->bytes, name,
                     ": grad_expert_out exceeds the registered buffer");
      t.grads = grad->buf->ptrsAt(grad->offset);
      t.gradMine = static_cast<char*>(grad->buf->local) + grad->offset;
    }
    if (scales != nullptr) {
      GLB_ENFORCE_LE(scales->offset + capacityRows * scaleBytes, scales->buf->bytes, name,
                     ": output scales exceed the registered buffer");
      GLB_ENFORCE(scales->offset % sizeof(float) == 0, name, ": output scales must be 4-byte aligned");
      t.scales.scales = scales->buf->ptrsAt(scales->offset);
    }
  } else {
    const auto l = layoutOf(pc);
    t.peers = pc.stagePtrs(l.bulkOff);
    t.mine = static_cast<const char*>(out.ptr);
    t.staged = static_cast<char*>(out.ptr);
    t.plain = true;
    t.capRows = std::min(capacityRows, l.bulkBytes / (rowBytes + scaleBytes + gradBytes));
    if (grad != nullptr) t.gradMine = static_cast<char*>(grad->ptr);
    if (scales != nullptr) {
      GLB_ENFORCE(reinterpret_cast<uintptr_t>(scales->ptr) % sizeof(float) == 0, name,
                  ": output scales must be 4-byte aligned");
      t.scales.stagedScales = static_cast<float*>(scales->ptr);
    }
  }
  return t;
}

MoeArgs moeArgs(PeerContext& pc, const MoeTarget& t, size_t rowBytes, int experts, int align) {
  MoeArgs d{};
  d.rowBytes = rowBytes;
  d.staged = t.staged;
  d.status = pc.inputStatusDevice();
  d.capRows = static_cast<uint32_t>(std::min<size_t>(t.capRows, 0xfffffffeull));
  d.experts = experts;
  d.align = align;
  d.plain = t.plain ? 1 : 0;
  return d;
}

// Like the host-count v-variant the grid is fixed (the sizes are only known on the device, the
// grid must be the same on every rank), and P = 1 runs the same kernel: the layouts still apply.
int moeBlocks(PeerContext& pc, const void* kernel) {
  return std::max(1, std::min({tuning().alltoallvBlocks, pc.coResidentBlocks(kernel), kMaxBlocks}));
}
}  // namespace

void alltoallvDev(PeerContext& pc, const void* in, size_t inRows, size_t rowBytes, const int64_t* inSplits,
                  const int64_t* inOffsets, const MoeOut& out, size_t capacityRows, int64_t* outSplits,
                  int64_t* outOffsets, int experts, int align, bool inverse, cudaStream_t stream,
                  const MoeOut* outScales) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_dev");
  const char* name = "alltoallv_dev";
  const bool fp8 = outScales != nullptr;
  checkMoeLimits(name, experts, align, rowBytes, fp8 ? kFp8Block : 1);
  GLB_ENFORCE(inSplits != nullptr, name, ": no input splits");
  GLB_ENFORCE(!inverse || (inOffsets != nullptr && !fp8), name,
              ": the inverse exchange needs the input offsets and does not quantise");
  GLB_ENFORCE(inverse || (outSplits != nullptr && outOffsets != nullptr),
              name, ": the forward exchange needs output splits and offsets");
  const MoeTarget t = resolveMoeOut(pc, name, "out", out, outScales, capacityRows, rowBytes);
  if (fp8) checkAligned16(name, in, t.mine, "input and output");
  const int blocks = moeBlocks(pc, alltoallvDevKernelPtr(fp8));
  prologue(pc, stream);
  launchAlltoallvDev(pc.comm(), t.peers, moeArgs(pc, t, rowBytes, experts, align), fp8 ? &t.scales : nullptr, in,
                     inRows, reinterpret_cast<const long long*>(inSplits), reinterpret_cast<const long long*>(inOffsets),
                     reinterpret_cast<long long*>(outSplits), reinterpret_cast<long long*>(outOffsets), inverse, blocks,
                     stream);
  finish(pc, stream, name);
}

void alltoallvDevTopk(PeerContext& pc, const void* x, size_t tokens, size_t rowBytes, int topk, const int64_t* topkIdx,
                      int64_t* splits, int64_t* pos, const MoeOut& out, size_t capacityRows, int64_t* outSplits,
                      int64_t* outOffsets, int experts, int align, cudaStream_t stream, const MoeOut* outScales) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_dev_topk");
  const char* name = "alltoallv_dev_topk";
  const bool fp8 = outScales != nullptr;
  checkTopk(name, topk);
  checkMoeLimits(name, experts, align, rowBytes, fp8 ? kFp8Block : 16);
  GLB_ENFORCE(tokens * static_cast<size_t>(topk) <= 0x7fffffffull, name, ": tokens x topk must be below 2^31, got ",
              tokens, " x ", topk);
  GLB_ENFORCE(splits != nullptr && outSplits != nullptr && outOffsets != nullptr &&
                  (tokens == 0 || (x != nullptr && topkIdx != nullptr && pos != nullptr)),
              name, ": missing x, topk_idx, splits, pos, out_splits or out_offsets");
  const MoeTarget t = resolveMoeOut(pc, name, "out", out, outScales, capacityRows, rowBytes);
  checkAligned16(name, x, t.mine, "x and out");
  // Peers write my out while I still read my x.
  rejectOverlap(x, tokens * rowBytes * (fp8 ? 2 : 1), t.mine, capacityRows * rowBytes, name);
  const int blocks = moeBlocks(pc, moeDispatchTopkKernelPtr(fp8));
  prologue(pc, stream);
  launchMoeDispatchTopk(pc.comm(), t.peers, moeArgs(pc, t, rowBytes, experts, align), fp8 ? &t.scales : nullptr, x,
                        tokens, topk, reinterpret_cast<const long long*>(topkIdx), reinterpret_cast<long long*>(splits),
                        reinterpret_cast<long long*>(pos), reinterpret_cast<long long*>(outSplits),
                        reinterpret_cast<long long*>(outOffsets), blocks, stream);
  finish(pc, stream, name);
}

void alltoallvDevCombineTopk(PeerContext& pc, void* out, size_t tokens, int topk, const int64_t* pos,
                             const float* weights, const int64_t* splits, const MoeOut& expertOut, size_t capacityRows,
                             size_t rowBytes, DataType dt, int experts, int align, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_dev_combine_topk");
  const char* name = "alltoallv_dev_combine_topk";
  GLB_ENFORCE(dt == DataType::FLOAT32 || dt == DataType::BFLOAT16 || dt == DataType::FLOAT16, name,
              ": rows must be float32, bfloat16 or float16");
  checkTopk(name, topk);
  checkMoeLimits(name, experts, align, rowBytes, 16);
  GLB_ENFORCE(splits != nullptr && (tokens == 0 || (pos != nullptr && out != nullptr)), name,
              ": missing splits, pos or out");
  // A plain expert_out is copied into my staging area, where my peers read it.
  const MoeTarget t = resolveMoeOut(pc, name, "expert_out", expertOut, nullptr, capacityRows, rowBytes);
  checkAligned16(name, out, t.mine, "out and expert_out");
  // Peers read my expert_out while I write my out.
  rejectOverlap(t.mine, capacityRows * rowBytes, out, tokens * rowBytes, name);
  const int blocks = moeBlocks(pc, moeCombineTopkKernelPtr(dt));
  prologue(pc, stream);
  launchMoeCombineTopk(pc.comm(), t.peers, moeArgs(pc, t, rowBytes, experts, align), out, tokens, topk,
                       reinterpret_cast<const long long*>(pos), weights, reinterpret_cast<const long long*>(splits), dt,
                       blocks, stream);
  finish(pc, stream, name);
}

void alltoallvDevCombineTopkBackward(PeerContext& pc, const MoeOut& gradExpertOut, float* gradWeights,
                                     const void* gradOut, const MoeOut& expertOut, size_t tokens, int topk,
                                     const int64_t* pos, const float* weights, const int64_t* splits,
                                     size_t capacityRows, size_t rowBytes, DataType dt, int experts, int align,
                                     cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_dev_combine_topk_backward");
  const char* name = "alltoallv_dev_combine_topk_backward";
  GLB_ENFORCE(dt == DataType::FLOAT32 || dt == DataType::BFLOAT16 || dt == DataType::FLOAT16, name,
              ": rows must be float32, bfloat16 or float16");
  checkTopk(name, topk);
  checkMoeLimits(name, experts, align, rowBytes, 16);
  GLB_ENFORCE(splits != nullptr &&
                  (tokens == 0 || (pos != nullptr && weights != nullptr && gradOut != nullptr && gradWeights != nullptr)),
              name, ": missing splits, pos, weights, grad_out or grad_weights");
  // Plain expert_out and grad_expert_out both go through my staging area: rows, then gradient rows.
  const MoeTarget t = resolveMoeOut(pc, name, "expert_out", expertOut, nullptr, capacityRows, rowBytes, &gradExpertOut);
  checkAligned16(name, gradOut, t.mine, "grad_out and expert_out");
  checkAligned16(name, t.gradMine, t.gradMine, "grad_expert_out");
  // Peers write my grad_expert_out while I read my expert_out, grad_out and write grad_weights.
  const size_t capBytes = capacityRows * rowBytes;
  rejectOverlap(t.mine, capBytes, t.gradMine, capBytes, name);
  rejectOverlap(gradOut, tokens * rowBytes, t.gradMine, capBytes, name);
  rejectOverlap(gradWeights, tokens * topk * sizeof(float), t.gradMine, capBytes, name);
  const int blocks = moeBlocks(pc, moeCombineTopkBackwardKernelPtr(dt));
  prologue(pc, stream);
  launchMoeCombineTopkBackward(pc.comm(), t.peers, t.plain ? t.peers : t.grads, moeArgs(pc, t, rowBytes, experts, align),
                               t.plain ? t.gradMine : nullptr, capacityRows, gradOut, gradWeights, tokens, topk,
                               reinterpret_cast<const long long*>(pos), weights,
                               reinterpret_cast<const long long*>(splits), dt, blocks, stream);
  finish(pc, stream, name);
}

MoeLLLayout moeLLLayout(int nranks, int experts, int maxTokens, int topk, size_t hidden, size_t elemBytes, bool fp8) {
  const char* name = "moe_ll_buffer";
  GLB_ENFORCE(nranks >= 1 && nranks <= kMaxRanks, name, ": at most ", kMaxRanks, " ranks, got ", nranks);
  checkTopk(name, topk);
  GLB_ENFORCE(maxTokens >= 1 && static_cast<int64_t>(maxTokens) * topk <= 0x7fffffffll, name,
              ": max_tokens must be at least 1 and max_tokens x topk at most 2^31 - 1, got ", maxTokens, " x ", topk);
  GLB_ENFORCE(!fp8 || elemBytes == 2, name, ": the quantising form takes bfloat16 rows");
  checkMoeLimits(name, experts, 1, fp8 ? hidden : hidden * elemBytes, fp8 ? kFp8Block : 16);
  MoeLLLayout l{};
  l.rowBytes = fp8 ? hidden : hidden * elemBytes;
  l.scaleBytes = fp8 ? hidden / kFp8Block * sizeof(float) : 0;
  l.combineRowBytes = hidden * elemBytes;
  const unsigned long long slots = static_cast<unsigned long long>(experts) * nranks * maxTokens;
  const unsigned long long choices = static_cast<unsigned long long>(maxTokens) * topk;
  unsigned long long at = 0;
  auto take = [&](unsigned long long n) {
    const unsigned long long o = at;
    at += (n + 15) / 16 * 16;
    return o;
  };
  l.slots = take(slots * l.rowBytes);
  l.scales = take(slots * l.scaleBytes);
  l.tags = take(slots * sizeof(int32_t));
  l.dispatchSig = take(static_cast<unsigned long long>(experts) * nranks * 8);
  l.combineSlots = take(choices * l.combineRowBytes);
  l.combineSig = take(static_cast<unsigned long long>(nranks) * 8);
  l.choices = take(choices * sizeof(int32_t));
  l.ctrl = take(16);
  l.bytes = at;
  l.experts = experts;
  l.maxTokens = maxTokens;
  l.topk = topk;
  l.fp8 = fp8 ? 1 : 0;
  return l;
}

namespace {
MoeLLArgs moeLLArgs(PeerContext& pc, const char* name, const PeerBuffer& buf, size_t offset, const MoeLLLayout& l) {
  GLB_ENFORCE(offset % 16 == 0 && offset + l.bytes <= buf.bytes, name, ": the buffer (", l.bytes,
              " bytes) does not fit the registration at offset ", offset);
  MoeLLArgs L{};
  L.bufs = buf.ptrsAt(offset);
  L.l = l;
  L.status = pc.inputStatusDevice();
  return L;
}
}  // namespace

void alltoallvLLTopk(PeerContext& pc, const PeerBuffer& buf, size_t offset, const MoeLLLayout& l, const void* x,
                     size_t tokens, const int64_t* topkIdx, void* out, float* outScales, int64_t* outSplits,
                     cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_ll_topk");
  const char* name = "alltoallv_ll_topk";
  GLB_ENFORCE(tokens <= static_cast<size_t>(l.maxTokens), name, ": ", tokens, " tokens; the buffer holds max_tokens = ",
              l.maxTokens);
  GLB_ENFORCE(out != nullptr && outSplits != nullptr && (!l.fp8 || outScales != nullptr) &&
                  (tokens == 0 || (x != nullptr && topkIdx != nullptr)),
              name, ": missing x, topk_idx, out, out_scales or out_splits");
  checkAligned16(name, x, out, "x and out");
  const MoeLLArgs L = moeLLArgs(pc, name, buf, offset, l);
  const int blocks = moeBlocks(pc, moeLLDispatchKernelPtr(l.fp8 != 0));
  prologue(pc, stream);
  launchMoeLLDispatch(pc.comm(), L, x, tokens, reinterpret_cast<const long long*>(topkIdx), out, outScales,
                      reinterpret_cast<long long*>(outSplits), blocks, stream);
  finish(pc, stream, name);
}

void alltoallvLLCombineTopk(PeerContext& pc, const PeerBuffer& buf, size_t offset, const MoeLLLayout& l, void* y,
                            size_t tokens, const void* expertOut, const float* weights, DataType dt,
                            cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_TRACE_RANGE("glb::cuda::alltoallv_ll_combine_topk");
  const char* name = "alltoallv_ll_combine_topk";
  GLB_ENFORCE(dt == DataType::FLOAT32 || dt == DataType::BFLOAT16 || dt == DataType::FLOAT16, name,
              ": rows must be float32, bfloat16 or float16");
  GLB_ENFORCE(l.combineRowBytes % 16 == 0, name, ": rows must be a multiple of 16 bytes");
  GLB_ENFORCE(tokens <= static_cast<size_t>(l.maxTokens), name, ": ", tokens, " tokens; the buffer holds max_tokens = ",
              l.maxTokens);
  GLB_ENFORCE(expertOut != nullptr && (tokens == 0 || y != nullptr), name, ": missing expert_out or y");
  checkAligned16(name, y, expertOut, "y and expert_out");
  const MoeLLArgs L = moeLLArgs(pc, name, buf, offset, l);
  // Sized like the dispatch, whose CTAs need more of an SM: ranks sharing a GPU may run one rank's
  // dispatch beside the others' combines, and every CTA of that dispatch must still be resident.
  const int blocks = moeBlocks(pc, moeLLDispatchKernelPtr(l.fp8 != 0));
  prologue(pc, stream);
  launchMoeLLCombine(pc.comm(), L, expertOut, weights, y, tokens, dt, blocks, stream);
  finish(pc, stream, name);
}

void scatter(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset, size_t bytes, int root,
             cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_ENFORCE(root >= 0 && root < pc.size, "scatter: invalid root ", root);
  GLB_ENFORCE_LE(outOffset + bytes, out.bytes, "scatter output exceeds the registered buffer");
  if (pc.size == 1) {
    char* dst = static_cast<char*>(out.local) + outOffset;
    if (dst != in && bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  std::vector<size_t> soff(pc.size), slen(pc.size, bytes), doff(pc.size, 0);
  for (int j = 0; j < pc.size; j++) soff[j] = static_cast<size_t>(j) * bytes;
  const bool vec = out.vectorOk && outOffset % 16 == 0 && (pc.rank != root || reinterpret_cast<uintptr_t>(in) % 16 == 0);
  prologue(pc, stream);
  launchAlltoallPush(pc.comm(), in, out.ptrsAt(outOffset), soff.data(), slen.data(), doff.data(), nullptr, root, vec,
                     bwBlocks(pc, "alltoall", alltoallPushKernelPtr(), bytes * pc.size, bytes), stream);
  finish(pc, stream, "scatter");
}

void scatter(PeerContext& pc, const void* in, void* out, size_t bytes, int root, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  if (pc.size == 1) {
    if (out != in && bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, bytes, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(root >= 0 && root < pc.size, "scatter: invalid root ", root);
  if (exceedsBulk(pc, bytes)) {
    // Only the root sends; every rank receives its block from the root.
    std::vector<size_t> send(pc.size, pc.rank == root ? bytes : 0), recv(pc.size, 0);
    recv[root] = bytes;
    runPipelinedAlltoall(pc, in, out, send, recv, bytes * pc.size, "scatter(pipelined)", stream);
    return;
  }
  auto st = stagedBulk(pc, bytes, "scatter");
  std::vector<size_t> soff(pc.size), slen(pc.size, bytes), doff(pc.size, 0);
  for (int j = 0; j < pc.size; j++) soff[j] = static_cast<size_t>(j) * bytes;
  prologue(pc, stream);
  launchAlltoallPush(pc.comm(), in, st.ptrs, soff.data(), slen.data(), doff.data(), nullptr, root,
                     pc.rank != root || reinterpret_cast<uintptr_t>(in) % 16 == 0,
                     bwBlocks(pc, "alltoall", alltoallPushKernelPtr(), bytes * pc.size, bytes), stream);
  finish(pc, stream, "scatter(staged)");
  if (bytes > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, st.mine, bytes, cudaMemcpyDeviceToDevice, stream));
}

namespace {
void reducePullCommon(PeerContext& pc, const PeerPtrs& ins, void* mcIn, bool vecIn, void* out,
                      const std::vector<size_t>& counts, DataType dt, ReduceOp op, double scaleD, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::reduce_scatter/reduce");
  GLB_ENFORCE_EQ(static_cast<int>(counts.size()), pc.size, "need one element count per rank");
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  auto off = prefix(counts);
  const size_t es = elementSize(dt);
  // In-switch reduction only for P > 2 (at P = 2 it doubles the uplink traffic).
  // Decisions that shape the launch use the LARGEST share: identical on every rank.
  const size_t largest = *std::max_element(counts.begin(), counts.end());
  bool wantMc = tuning().nvlsReduceScatter;
  int cap = tuning().maxBlocks;
  if (const TuneEntry* e = TuningTable::get().lookup("reduce_scatter", pc.size, mcIn ? BufKind::SYMMETRIC : BufKind::REGISTERED,
                                                     largest * es)) {
    wantMc = e->algo == "nvls";
    if (e->blocks > 0) cap = e->blocks;
  }
  const bool useMc = mcIn != nullptr && pc.size > 2 && wantMc && nvlsSupports(dt, op) && largest * es >= tuning().nvlsMinBytes;
  Epilogue ep;
  ep.scale = scaleD;
  const float scale = scaleOf(ep, dt);
  prologue(pc, stream);
  launchReducePull(pc.comm(), ins, mcIn, out, off.data(), counts.data(), dt, op, scale, vecIn, useMc,
                   std::min(blocksFor(pc, largest * es / 16, 1, cap), pc.coResidentBlocks(reducePullKernelPtr(dt, pc.size))),
                   stream);
  finish(pc, stream, "reduce_scatter");
}
}  // namespace

namespace {
// Small reduce_scatter with equal shares: flag-in-data lines, no barrier, any input pointer.
bool tryLLReduceScatter(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& counts, DataType dt,
                        ReduceOp op, double scaleD, cudaStream_t stream) {
  if (pc.size < 2 || !allEqual(counts) || counts[0] == 0 || envFlag("CUDA_LL_DISABLE", false)) return false;
  const size_t bytes = counts[0] * elementSize(dt);
  size_t limit = std::min(tuning().llMaxBytes, pc.llMaxBytes());
  if (const TuneEntry* e = TuningTable::get().lookup("reduce_scatter", pc.size, BufKind::REGISTERED, bytes)) {
    if (e->algo != "ll") return false;
    limit = pc.llMaxBytes();
  }
  if (bytes > limit) return false;
  Epilogue ep;
  ep.scale = scaleD;
  const float scale = scaleOf(ep, dt);
  const size_t units = ceilDiv(bytes, size_t(8)) * pc.size;
  int threads = static_cast<int>(std::min<size_t>(kThreads, roundUp(std::max<size_t>(units, 32), 32)));
  int blocks = static_cast<int>(std::min<size_t>(ceilDiv(units, static_cast<size_t>(threads)), 16));
  prologue(pc, stream);
  launchLLReduceScatter(pc.comm(), in, out, counts[0], dt, op, scale, pc.llPtrs(), pc.llSrcStride(), pc.llParityStride(),
                        std::max(1, blocks), threads, stream);
  finish(pc, stream, "reduce_scatter(ll)");
  return true;
}
}  // namespace

void reduce_scatter(PeerContext& pc, const PeerBuffer& in, size_t inOffset, void* out,
                    const std::vector<size_t>& counts, DataType dt, ReduceOp op, cudaStream_t stream, double scale) {
  DeviceGuard g(pc.device);
  auto off = prefix(counts);
  const size_t es = elementSize(dt);
  GLB_ENFORCE_LE(inOffset + off.back() * es, in.bytes, "reduce_scatter input exceeds the registered buffer");
  if (pc.size == 1) {
    const char* src = static_cast<const char*>(in.local) + inOffset;
    if (src != out && counts[0] > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, src, counts[0] * es, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  if (tryLLReduceScatter(pc, static_cast<const char*>(in.local) + inOffset, out, counts, dt, op, scale, stream)) return;
  reducePullCommon(pc, in.ptrsAt(inOffset), in.mc ? static_cast<char*>(in.mc) + inOffset : nullptr,
                   in.vectorOk && inOffset % 16 == 0, out, counts, dt, op, scale, stream);
}

void reduce_scatter(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& counts, DataType dt,
                    ReduceOp op, cudaStream_t stream, double scale) {
  DeviceGuard g(pc.device);
  auto off = prefix(counts);
  const size_t es = elementSize(dt);
  if (pc.size == 1) {
    if (in != out && counts[0] > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, counts[0] * es, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
  if (tryLLReduceScatter(pc, in, out, counts, dt, op, scale, stream)) return;
  if (exceedsBulk(pc, off.back() * es)) {
    GLB_TRACE_RANGE("glb::cuda::reduce_scatter(pipelined)");
    GLB_ENFORCE_EQ(static_cast<int>(counts.size()), pc.size, "need one element count per rank");
    Epilogue ep;
    ep.scale = scale;
    const float s = scaleOf(ep, dt);
    const size_t largest = *std::max_element(counts.begin(), counts.end());
    const PipeShape sh = pipeShape(pc, pipelinedReduceScatterKernelFor(dt, pc.size), 2, pc.size,
                                   largest * es * pc.size, 0, 0, 0, "reduce_scatter");
    prologue(pc, stream);
    launchPipelinedReduceScatter(pc.comm(), in, out, off.data(), counts.data(), dt, op, s,
                                 pc.stagePtrs(layoutOf(pc).bulkOff), sh.tile, sh.xthreads, sh.blocks, stream);
    finish(pc, stream, "reduce_scatter(pipelined)");
    return;
  }
  auto st = stagedBulk(pc, off.back() * es, "reduce_scatter");
  if (off.back() > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(st.mine, in, off.back() * es, cudaMemcpyDeviceToDevice, stream));
  reducePullCommon(pc, st.ptrs, st.mc, true, out, counts, dt, op, scale, stream);
}

// ---- cast reduce_scatter / allgather(v) ---------------------------------------------------------

namespace {
bool isHalf(DataType t) { return t == DataType::FLOAT16 || t == DataType::BFLOAT16; }

// What every cast call checks before it launches anything, on this rank's arguments: the dtype
// pair (16-bit -> float32 for reduce_scatter, float32 -> 16-bit for allgather), SUM, one count per
// rank, and disjoint input and output ranges (in place is impossible across dtypes). inBytes /
// outBytes are the ranges the call reads and writes here.
void checkCast(const PeerContext& pc, const char* what, bool reduce, DataType inDt, DataType outDt, ReduceOp op,
               const std::vector<size_t>& counts, const void* in, size_t inBytes, const void* out, size_t outBytes) {
  if (reduce ? !(isHalf(inDt) && outDt == DataType::FLOAT32) : !(inDt == DataType::FLOAT32 && isHalf(outDt))) {
    GLB_THROW(InputException, what, ": the cast form takes ",
              reduce ? "float16 / bfloat16 input and a float32 output" : "float32 input and a float16 / bfloat16 output",
              ", got ", dataTypeName(inDt), " -> ", dataTypeName(outDt));
  }
  if (reduce && op != ReduceOp::SUM) GLB_THROW(InputException, what, ": the cast form reduces with SUM only");
  if (static_cast<int>(counts.size()) != pc.size) {
    GLB_THROW(InputException, what, ": ", counts.size(), " counts for ", pc.size, " ranks");
  }
  const uintptr_t i = reinterpret_cast<uintptr_t>(in), o = reinterpret_cast<uintptr_t>(out);
  if (inBytes > 0 && outBytes > 0 && i < o + outBytes && o < i + inBytes) {
    GLB_THROW(InputException, what, ": the input and output overlap; a cast cannot run in place");
  }
}

size_t total(const std::vector<size_t>& counts) { return std::accumulate(counts.begin(), counts.end(), size_t(0)); }

// One rank: the conversion and the scale, one local launch (none for an empty share).
void castLocal(PeerContext& pc, const void* in, DataType inDt, void* out, DataType outDt, size_t count, float scale,
               cudaStream_t stream, const char* what) {
  if (count == 0) return;
  pc.orderStreams(stream);
  launchCastScale(in, inDt, out, outDt, count, scale, blocksFor(pc, ceilDiv(count, size_t(8)), 1, tuning().maxBlocks),
                  stream);
  finish(pc, stream, what);
}

void castReducePull(PeerContext& pc, const PeerPtrs& ins, bool vecIn, void* out, const std::vector<size_t>& counts,
                    DataType dt, float scale, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::reduce_scatter(cast)");
  auto off = prefix(counts);
  const size_t largest = *std::max_element(counts.begin(), counts.end());
  const int blocks = std::min(blocksFor(pc, largest * elementSize(dt) / 16, 1, tuning().maxBlocks),
                              pc.coResidentBlocks(castReducePullKernelPtr(dt, pc.size)));
  prologue(pc, stream);
  launchCastReducePull(pc.comm(), ins, static_cast<float*>(out), off.data(), counts.data(), dt, scale, vecIn, blocks,
                       stream);
  finish(pc, stream, "reduce_scatter(cast)");
}

void castGatherPush(PeerContext& pc, const void* in, const PeerPtrs& outs, bool vecOut, const std::vector<size_t>& counts,
                    DataType outDt, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::allgather(cast)");
  auto off = prefix(counts);
  const size_t largest = *std::max_element(counts.begin(), counts.end());
  const bool vec = vecOut && reinterpret_cast<uintptr_t>(in) % 16 == 0;
  prologue(pc, stream);
  launchCastGatherPush(pc.comm(), in, outs, outDt, off.data(), counts.data(), vec,
                       bwBlocks(pc, "allgather", castGatherPushKernelPtr(outDt), largest * elementSize(outDt)), stream);
  finish(pc, stream, "allgather(cast)");
}
}  // namespace

void reduce_scatter(PeerContext& pc, const PeerBuffer& in, size_t inOffset, void* out, const std::vector<size_t>& counts,
                    DataType dt, DataType outDt, ReduceOp op, cudaStream_t stream, double scale) {
  if (outDt == dt) {
    reduce_scatter(pc, in, inOffset, out, counts, dt, op, stream, scale);
    return;
  }
  DeviceGuard g(pc.device);
  const char* src = static_cast<const char*>(in.local) + inOffset;
  const size_t n = total(counts), mine = pc.rank < static_cast<int>(counts.size()) ? counts[pc.rank] : 0;
  checkCast(pc, "reduce_scatter", true, dt, outDt, op, counts, src, n * elementSize(dt), out, mine * sizeof(float));
  if (inOffset + n * elementSize(dt) > in.bytes) {
    GLB_THROW(InputException, "reduce_scatter: the input range exceeds the registered buffer");
  }
  if (pc.size == 1) {
    castLocal(pc, src, dt, out, outDt, mine, static_cast<float>(scale), stream, "reduce_scatter(cast, local)");
    return;
  }
  castReducePull(pc, in.ptrsAt(inOffset), in.vectorOk && inOffset % 16 == 0, out, counts, dt, static_cast<float>(scale),
                 stream);
}

void reduce_scatter(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& counts, DataType dt,
                    DataType outDt, ReduceOp op, cudaStream_t stream, double scale) {
  if (outDt == dt) {
    reduce_scatter(pc, in, out, counts, dt, op, stream, scale);
    return;
  }
  DeviceGuard g(pc.device);
  const size_t es = elementSize(dt);
  const size_t n = total(counts), mine = pc.rank < static_cast<int>(counts.size()) ? counts[pc.rank] : 0;
  checkCast(pc, "reduce_scatter", true, dt, outDt, op, counts, in, n * es, out, mine * sizeof(float));
  const float s = static_cast<float>(scale);
  if (pc.size == 1) {
    castLocal(pc, in, dt, out, outDt, mine, s, stream, "reduce_scatter(cast, local)");
    return;
  }
  if (exceedsBulk(pc, n * es)) {
    GLB_TRACE_RANGE("glb::cuda::reduce_scatter(cast, pipelined)");
    auto off = prefix(counts);
    const size_t largest = *std::max_element(counts.begin(), counts.end());
    const PipeShape sh = pipeShape(pc, castPipelinedReduceScatterKernelFor(dt, pc.size), 2, pc.size,
                                   largest * es * pc.size, 0, 0, 0, "reduce_scatter");
    prologue(pc, stream);
    launchCastPipelinedReduceScatter(pc.comm(), in, static_cast<float*>(out), off.data(), counts.data(), dt, s,
                                     pc.stagePtrs(layoutOf(pc).bulkOff), sh.tile, sh.xthreads, sh.blocks, stream);
    finish(pc, stream, "reduce_scatter(cast, pipelined)");
    return;
  }
  auto st = stagedBulk(pc, n * es, "reduce_scatter");
  if (n > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(st.mine, in, n * es, cudaMemcpyDeviceToDevice, stream));
  castReducePull(pc, st.ptrs, true, out, counts, dt, s, stream);
}

void allgatherv(PeerContext& pc, const void* in, DataType inDt, const PeerBuffer& out, size_t outOffset,
                const std::vector<size_t>& counts, DataType outDt, cudaStream_t stream) {
  const size_t es = elementSize(outDt);
  if (inDt == outDt) {
    std::vector<size_t> bytes(counts);
    for (auto& b : bytes) b *= es;
    allgatherv(pc, in, out, outOffset, bytes, stream);
    return;
  }
  DeviceGuard g(pc.device);
  char* dst = static_cast<char*>(out.local) + outOffset;
  const size_t n = total(counts), mine = pc.rank < static_cast<int>(counts.size()) ? counts[pc.rank] : 0;
  checkCast(pc, "allgather", false, inDt, outDt, ReduceOp::SUM, counts, in, mine * sizeof(float), dst, n * es);
  if (outOffset + n * es > out.bytes) {
    GLB_THROW(InputException, "allgather: the output range exceeds the registered buffer");
  }
  if (pc.size == 1) {
    castLocal(pc, in, inDt, dst, outDt, mine, 1.0f, stream, "allgather(cast, local)");
    return;
  }
  castGatherPush(pc, in, out.ptrsAt(outOffset), out.vectorOk && outOffset % 16 == 0, counts, outDt, stream);
}

void allgatherv(PeerContext& pc, const void* in, DataType inDt, void* out, const std::vector<size_t>& counts,
                DataType outDt, cudaStream_t stream) {
  const size_t es = elementSize(outDt);
  if (inDt == outDt) {
    std::vector<size_t> bytes(counts);
    for (auto& b : bytes) b *= es;
    allgatherv(pc, in, out, bytes, stream);
    return;
  }
  DeviceGuard g(pc.device);
  const size_t n = total(counts), mine = pc.rank < static_cast<int>(counts.size()) ? counts[pc.rank] : 0;
  checkCast(pc, "allgather", false, inDt, outDt, ReduceOp::SUM, counts, in, mine * sizeof(float), out, n * es);
  if (pc.size == 1) {
    castLocal(pc, in, inDt, out, outDt, mine, 1.0f, stream, "allgather(cast, local)");
    return;
  }
  if (exceedsBulk(pc, n * es)) {
    GLB_TRACE_RANGE("glb::cuda::allgather(cast, pipelined)");
    std::vector<size_t> bytes(counts);
    for (auto& b : bytes) b *= es;
    auto off = prefix(bytes);
    const size_t largest = *std::max_element(bytes.begin(), bytes.end());
    const PipeShape sh = pipeShape(pc, castPipelinedAllgatherKernelFor(outDt), 2, 1, largest, 0, 0, 0, "allgather");
    prologue(pc, stream);
    launchCastPipelinedAllgather(pc.comm(), in, out, outDt, off.data(), bytes.data(), pc.stagePtrs(layoutOf(pc).bulkOff),
                                 sh.tile, sh.xthreads, sh.blocks, stream);
    finish(pc, stream, "allgather(cast, pipelined)");
    return;
  }
  auto st = stagedBulk(pc, n * es, "allgather");
  castGatherPush(pc, in, st.ptrs, true, counts, outDt, stream);
  if (n > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, st.mine, n * es, cudaMemcpyDeviceToDevice, stream));
}

void reduce(PeerContext& pc, const PeerBuffer& in, size_t inOffset, const PeerBuffer& out, size_t outOffset,
            size_t count, DataType dt, ReduceOp op, int root, cudaStream_t stream) {
  DeviceGuard g(pc.device);
  GLB_ENFORCE(root >= 0 && root < pc.size, "reduce: invalid root ", root);
  const size_t es = elementSize(dt);
  GLB_ENFORCE_LE(inOffset + count * es, in.bytes, "reduce input exceeds the registered buffer");
  if (pc.size == 1) {
    const char* src = static_cast<const char*>(in.local) + inOffset;
    char* dst = static_cast<char*>(out.local) + outOffset;
    if (src != dst && count > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(dst, src, count * es, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(out.peer[root] != nullptr, "reduce: the root's output is not registered");
  // Each rank reduces an equal slice and stores it straight into the root's output.
  std::vector<size_t> counts(pc.size);
  for (int r = 0; r < pc.size; r++) counts[r] = count / pc.size + (static_cast<size_t>(r) < count % pc.size ? 1 : 0);
  auto off = prefix(counts);
  char* dst = static_cast<char*>(out.peer[root]) + outOffset + off[pc.rank] * es;
  reducePullCommon(pc, in.ptrsAt(inOffset), in.mc ? static_cast<char*>(in.mc) + inOffset : nullptr,
                   in.vectorOk && inOffset % 16 == 0, dst, counts, dt, op, 1.0, stream);
}

void reduce(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op, int root,
            cudaStream_t stream) {
  DeviceGuard g(pc.device);
  const size_t es = elementSize(dt);
  if (pc.size == 1) {
    if (in != out && count > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(out, in, count * es, cudaMemcpyDeviceToDevice, stream));
    return;
  }
  GLB_ENFORCE(root >= 0 && root < pc.size, "reduce: invalid root ", root);
  std::vector<size_t> counts(pc.size);
  for (int r = 0; r < pc.size; r++) counts[r] = count / pc.size + (static_cast<size_t>(r) < count % pc.size ? 1 : 0);
  auto off = prefix(counts);
  const auto l = layoutOf(pc);
  const size_t half = l.bulkBytes / 2 / 16 * 16;
  if (count * es > half) {
    // Larger than the staged path takes: one kernel streams the shares through the pool and the
    // root pulls the reduced shares (pipeline_kernels.cu). count and the pool size are the same on
    // every rank, so every rank takes this path together.
    GLB_TRACE_RANGE("glb::cuda::reduce(pipelined)");
    GLB_ENFORCE(op != ReduceOp::CUSTOM, "custom reductions run on the host path only");
    const PipeShape sh = pipeShape(pc, pipelinedReduceKernelFor(dt, pc.size), 2, pc.size + 1, counts[0] * es * pc.size,
                                   0, 0, 0, "reduce");
    prologue(pc, stream);
    launchPipelinedReduce(pc.comm(), in, out, off.data(), counts.data(), root, dt, op, pc.stagePtrs(l.bulkOff), sh.tile,
                          sh.xthreads, sh.blocks, stream);
    finish(pc, stream, "reduce(pipelined)");
    return;
  }
  // Stage inputs in the first half of the bulk region, collect results in the second.
  PeerPtrs ins = pc.stagePtrs(l.bulkOff);
  PeerPtrs outs = pc.stagePtrs(l.bulkOff + half);
  char* mine = static_cast<char*>(ins.p[pc.rank]);
  if (count > 0) GLB_CUDA_CHECK(cudaMemcpyAsync(mine, in, count * es, cudaMemcpyDeviceToDevice, stream));
  char* dst = static_cast<char*>(outs.p[root]) + off[pc.rank] * es;
  reducePullCommon(pc, ins, pc.stageMc(l.bulkOff), true, dst, counts, dt, op, 1.0, stream);
  if (pc.rank == root && count > 0) {
    GLB_CUDA_CHECK(cudaMemcpyAsync(out, static_cast<char*>(outs.p[root]), count * es, cudaMemcpyDeviceToDevice, stream));
  }
}

// ---- point to point ------------------------------------------------------------------------------

namespace {
void p2pCommon(PeerContext& pc, const void* sendPtr, size_t sendBytes, int dst, void* recvPtr, size_t recvBytes,
               int src, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::p2p");
  DeviceGuard g(pc.device);
  GLB_ENFORCE(sendBytes == 0 || (dst >= 0 && dst < pc.size && dst != pc.rank), "send: invalid destination rank ", dst);
  GLB_ENFORCE(recvBytes == 0 || (src >= 0 && src < pc.size && src != pc.rank), "recv: invalid source rank ", src);
  if (sendBytes == 0 && recvBytes == 0) return;
  pc.checkHealth();
  // No orderStreams / launchGuard: p2p kernels do not use the barrier epoch, and a host
  // rendezvous of ALL ranks would deadlock a pairwise operation.
  const auto& o = pc.options();
  // Both ends must cut a slot into the same stripes: the lane count comes from job-wide
  // values only. Sender and receiver CTAs wait for each other, so they must be co-resident.
  const int lanes = std::max(1, std::min(o.p2pLanes, pc.maxBlocks() / 2));
  launchP2p(pc.comm(), sendPtr, sendBytes, sendBytes ? dst : 0, recvPtr, recvBytes, recvBytes ? src : 0, pc.mailboxPtrs(),
            pc.mailboxStride(), o.p2pSlotBytes, o.p2pSlots, lanes, stream);
  checkLaunch("p2p");
}
}  // namespace

void send(PeerContext& pc, const void* ptr, size_t bytes, int dst, cudaStream_t stream) {
  p2pCommon(pc, ptr, bytes, dst, nullptr, 0, 0, stream);
}

void recv(PeerContext& pc, void* ptr, size_t bytes, int src, cudaStream_t stream) {
  p2pCommon(pc, nullptr, 0, 0, ptr, bytes, src, stream);
}

void sendrecv(PeerContext& pc, const void* sendPtr, size_t sendBytes, int dst, void* recvPtr, size_t recvBytes,
              int src, cudaStream_t stream) {
  p2pCommon(pc, sendPtr, sendBytes, dst, recvPtr, recvBytes, src, stream);
}

void exchange(PeerContext& pc, const void* sendPtr, size_t sendBytes, int dst, const PeerBuffer& recvBuf,
              size_t recvOffset, size_t recvBytes, int src, cudaStream_t stream) {
  GLB_TRACE_RANGE("glb::cuda::exchange");
  DeviceGuard g(pc.device);
  GLB_ENFORCE(sendBytes == 0 || (dst >= 0 && dst < pc.size && dst != pc.rank), "exchange: invalid destination rank ", dst);
  GLB_ENFORCE(recvBytes == 0 || (src >= 0 && src < pc.size && src != pc.rank), "exchange: invalid source rank ", src);
  if (sendBytes == 0 && recvBytes == 0) return;
  GLB_ENFORCE(sendBytes == 0 || recvBuf.peer[dst] != nullptr, "exchange: rank ", dst, " has no mapping of the receive buffer");
  GLB_ENFORCE_LE(recvOffset + std::max(sendBytes, recvBytes), recvBuf.bytes, "exchange: range exceeds the receive buffer");
  pc.checkHealth();
  // Pairwise like send / recv: no barrier epoch, no host rendezvous. The arrival counter
  // counts CTAs, so the grid is a job-wide value.
  const int blocks = std::max(1, std::min(pc.options().exchangeBlocks, pc.maxBlocks()));
  char* remote = sendBytes ? static_cast<char*>(recvBuf.peer[dst]) + recvOffset : nullptr;
  launchExchange(pc.comm(), sendPtr, sendBytes, sendBytes ? dst : 0, remote, recvBytes, recvBytes ? src : 0, blocks,
                 tuning().tmaCopies && std::max(sendBytes, recvBytes) >= 64 * 1024, stream);
  checkLaunch("exchange");
}

void put(PeerContext& pc, const void* local, const PeerBuffer& remote, size_t remoteOffset, size_t bytes, int peer,
         cudaStream_t stream) {
  GLB_ENFORCE(peer >= 0 && peer < pc.size && remote.peer[peer] != nullptr, "put: rank ", peer, " has no mapping of this buffer");
  GLB_ENFORCE_LE(remoteOffset + bytes, remote.bytes, "put: range exceeds the remote buffer");
  if (bytes == 0) return;
  DeviceGuard g(pc.device);
  pc.checkHealth();
  launchPeerCopy(static_cast<char*>(remote.peer[peer]) + remoteOffset, local, bytes, bwBlocks(pc, "put", nullptr, bytes), stream,
                 tuning().tmaCopies);
  checkLaunch("put");
}

void get(PeerContext& pc, void* local, const PeerBuffer& remote, size_t remoteOffset, size_t bytes, int peer,
         cudaStream_t stream) {
  GLB_ENFORCE(peer >= 0 && peer < pc.size && remote.peer[peer] != nullptr, "get: rank ", peer, " has no mapping of this buffer");
  GLB_ENFORCE_LE(remoteOffset + bytes, remote.bytes, "get: range exceeds the remote buffer");
  if (bytes == 0) return;
  DeviceGuard g(pc.device);
  pc.checkHealth();
  launchPeerCopy(local, static_cast<const char*>(remote.peer[peer]) + remoteOffset, bytes, bwBlocks(pc, "get", nullptr, bytes), stream,
                 tuning().tmaCopies);
  checkLaunch("get");
}

}  // namespace cuda
}  // namespace glb
