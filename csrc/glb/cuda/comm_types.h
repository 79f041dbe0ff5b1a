// Plain structs shared between host code and device kernels (safe to include
// from .cc files): the per-rank signal pad and the by-value kernel arguments.
#pragma once

#include <cstddef>
#include <cstdint>

namespace glb {
namespace cuda {

constexpr int kMaxRanks = 16;
constexpr int kMaxBlocks = 512;   // upper bound on CTAs of one collective kernel
constexpr int kThreads = 512;     // threads per CTA of the data-moving kernels
constexpr int kP2pLanes = 64;     // max CTAs per direction of a point-to-point transfer
constexpr int kMaxA2aExperts = 32;  // local experts per rank of the device-split all-to-all-v
constexpr int kA2aHdrWords = 6;     // its per-rank header: rowBytes, E, align, direction, capacity, bad input
constexpr int kFp8Block = 128;      // elements per fp32 scale of its quantising (bf16 -> e4m3) form

// Why a kernel gave up (SignalPad::abort / the host status word).
enum AbortCode : uint32_t {
  kAbortNone = 0,
  kAbortTimeout = 1,   // a peer did not reach the barrier within the timeout
  kAbortPeer = 2,      // a peer (or another CTA) aborted first and told us
};

// Data error found on the device by the device-split all-to-all-v. It is reported through a
// host-mapped word of its own (not the abort word): the context stays usable, and the next host
// call raises it as an input error.
enum InputCode : uint32_t {
  kInputOk = 0,
  kInputOverflow = 1,  // a destination needs more output rows than it has
  kInputInvalid = 2,   // a negative or oversized split, an offset out of range, or headers that differ
  kInputSlotOverflow = 3,  // low-latency exchange: a (source, expert) group has more rows than max_tokens
};
struct InputStatus {
  uint32_t code;             // InputCode; written last, cleared by the host when it raises
  uint32_t rank;             // the overflowing destination (slot overflow: the source)
  unsigned long long need;   // rows it needs
  unsigned long long avail;  // rows it has (slot overflow: max_tokens)
  uint32_t expert;           // slot overflow: the global expert index j·E + e
};

// One per rank, at the start of its symmetric pool. `flag[b][s]` is written by
// rank s's block b; everything else is only touched by the owning rank (except
// `abort`, which any rank may raise).
struct alignas(128) SignalPad {
  uint32_t flag[kMaxBlocks][kMaxRanks];
  uint32_t epoch;      // barrier epoch consumed so far (advanced by the last CTA to finish)
  uint32_t stageSeq;   // number of staged (one-shot) launches so far -> double-buffer parity
  uint32_t done;       // CTA completion ticket
  uint32_t llSeq;      // number of flag-in-data (LL) launches so far -> flag value / parity
  uint32_t abort;      // != 0: a barrier timed out somewhere; every later barrier returns at once
  uint32_t abortRank;  // who was missing when the first local time-out fired
  uint32_t pad[26];
  // Scratch for in-kernel metadata exchange (alltoallv receive offsets).
  unsigned long long xchg[kMaxRanks];
  // Point-to-point lanes (p2p_kernels.cu). Lane l of the pair (s -> d) counts mailbox chunks:
  //   d.pad.p2pHead[l][s]  written by s: chunks published so far
  //   s.pad.p2pTail[l][d]  written by d: chunks consumed so far
  //   p2pSent / p2pRecvd   the owners' own running totals (persist across launches)
  uint32_t p2pHead[kP2pLanes][kMaxRanks];
  uint32_t p2pTail[kP2pLanes][kMaxRanks];
  uint32_t p2pSent[kP2pLanes][kMaxRanks];
  uint32_t p2pRecvd[kP2pLanes][kMaxRanks];
  // Device-split all-to-all-v (alltoallvDevKernel). Before its first barrier rank s writes its
  // header and its P·E row counts into column s of these tables in EVERY rank's pad (the layout
  // of `flag`), so after the barrier each rank reads the whole count matrix from its own pad.
  // Rank s writes them again only in its next launch, after all of its CTAs have passed the
  // second barrier of this one, i.e. after every reader has finished. That holds because no rank
  // reads the tables after its own second barrier.
  uint32_t a2aHdr[kA2aHdrWords][kMaxRanks];
  uint32_t a2aCount[kMaxRanks * kMaxA2aExperts][kMaxRanks];
  // Grid barrier among this rank's own CTAs of one launch: arrivals, generation.
  uint32_t a2aArrive;
  uint32_t a2aGen;
  // Pipelined all-to-all (pipelinedAlltoallKernel): before its first barrier rank s writes the
  // number of chunks it needs into column s of this table in EVERY rank's pad (the layout of
  // `flag`), so after the barrier each rank takes the maximum over its own row. Rank s rewrites its
  // column only in a later launch, after all its CTAs have passed this launch's final barrier, and
  // CTA b of every reader arrives there only after it has read (it reads right after barrier 1).
  // That needs the final barrier to be a later one than barrier 1: the kernel runs at least two
  // steps, even when every block is empty. 32-bit entries: in the loopback self-test peer pads are
  // this pad shifted by one column, which keeps them aligned.
  uint32_t pipeChunks[kMaxRanks];
  // Top-k MoE combine (moeCombineTopkKernel): rank s clears column s of this table in EVERY rank's
  // pad with its header, before barrier 1, and sets it between barriers 1 and 2 if one of its `pos`
  // entries is out of range; every rank reads its own row between barriers 2 and 3. Rank s rewrites
  // its column only in a later launch, after every CTA of every rank has arrived at barrier 3.
  uint32_t a2aPosBad[kMaxRanks];
};

struct CommArgs {
  int rank;
  int nranks;
  SignalPad* sig[kMaxRanks];  // sig[r] = rank r's pad as mapped in this process
  SignalPad* self;            // == sig[rank]; a plain field so that kernels need no dynamic
                              // index into their parameter space to reach their own pad
  // Failure detection: a barrier that waits longer than this sets the abort word,
  // reports through `hostStatus` (mapped pinned host memory) and lets the kernel exit.
  unsigned long long timeoutNs;  // 0 = wait forever
  uint32_t* hostStatus;          // may be null
};

struct PeerPtrs {
  void* p[kMaxRanks];
};

// Extra local pointers of a multi-pointer call (beyond the one that takes part in the
// exchange): folded into it before, and overwritten with the result after, inside the
// same kernel.
constexpr int kMaxLocal = 7;
struct LocalPtrs {
  int n = 0;
  void* p[kMaxLocal] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
};

// How a bandwidth kernel is launched: CTAs and the per-thread unroll (independent
// 128-bit accesses in flight). Filled from the tuning table (tuning.h).
struct LaunchCfg {
  int blocks = 64;
  int unroll = 0;  // 0 = the kernel's default for this P
};

}  // namespace cuda
}  // namespace glb
