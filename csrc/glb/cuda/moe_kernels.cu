// Device-split MoE exchange over NVLink peer memory (sm_90a): the all-to-all-v with device-side
// counts (forward and inverse, copying and quantising to FP8), the top-k dispatch and the top-k
// combine. Every form runs the same protocol, written once below: publish a header and the row
// counts, agree at barrier 1, derive the layout from the count matrix, move the rows, and for the
// dispatches copy a plain output out of the staging area after barrier 2.
//
// Splits are device arrays of row counts; nothing about them passes through the host. P ranks,
// E local experts per rank, K = P·E chunks per rank. Count matrix M[s][k] = entry k of rank s's
// in_splits, read after the first barrier from column s of the a2aCount table of my own pad.
//   forward: k = j·E + e = rows of rank s for expert e of rank j; input packed in k order; on
//            rank j expert e's segment starts at a multiple of `align` rows and holds the rows of
//            sources 0..P-1 one after the other.
//   inverse: k = e·P + s = rows of my expert e that go back to rank s, read at in_offsets[k]; on
//            rank s they land packed in (holder j, e) order: where s's forward input rows were.
// A destination whose rows exceed the capacity it published receives nothing; invalid input
// anywhere (negative or oversized split, offsets out of range, headers that differ) moves
// nothing anywhere. Both are reported to the host of every rank through InputStatus.
#include <type_traits>

#include "glb/cuda/device_common.cuh"
#include "glb/cuda/grid_copy.cuh"
#include "glb/cuda/kernels.h"

namespace glb {
namespace cuda {

namespace {

constexpr uint32_t kA2aBad = 0xffffffffu;  // a count that is not a valid row count
constexpr int kMaxK = kMaxRanks * kMaxA2aExperts;

// Header word 3: which form of the exchange a rank runs. Ranks that disagree on any bit read the
// call as invalid, like differing row sizes. Bit 1 marks the quantising forms, bit 3 a staged
// (plain) output or expert_out: a rank whose peers push into its registered buffer and a rank
// whose peers push into its staging area would each write where the other does not read.
enum class A2aForm : uint32_t {
  kForward = 0u,
  kInverse = 1u,
  kCombineTopk = 4u,
  kDispatchTopk = 16u,
  kCombineTopkBackward = 32u
};
__device__ __forceinline__ uint32_t a2aHeaderWord(A2aForm form, bool quant, bool staged) {
  return static_cast<uint32_t>(form) | (quant ? 2u : 0u) | (staged ? 8u : 0u);
}

// The fields of a call: the copying forms take MoeArgs, the quantising ones MoeQuantArgs, so that
// the copying kernels' parameter block does not carry the scales.
template <bool kQuant>
using MoeKernelArgs = std::conditional_t<kQuant, MoeQuantArgs, MoeArgs>;

// Spin until the grid-barrier generation moves past `g`, bounded like every other device-side
// wait: 0 when it moved, kAbortTimeout / kAbortPeer when the wait was abandoned.
static __device__ __noinline__ uint32_t waitGenSlow(const volatile uint32_t* gen, uint32_t g, uint32_t* abortWord,
                                                    unsigned long long timeoutNs) {
  const unsigned long long t0 = globalTimerNs();
  uint32_t polls = 0;
  while (*gen == g) {
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

// Grid barrier among the CTAs of THIS launch on this rank. It relies on every CTA being resident
// (the grid is capped by coResidentBlocks); should that fail, e.g. because another process holds
// SMs, the wait gives up after the context timeout like a barrier does, raises the abort word and
// returns false. Every CTA still counts its arrival, so the last one to arrive resets the counter
// and the next launch starts clean. Everything a CTA wrote before, at system scope, is visible to
// every CTA after it, and is covered by their later release stores.
__device__ __forceinline__ bool localGridSync(const CommArgs& a) {
  SignalPad* me = a.self;
  __syncthreads();
  int ok = 1;
  if (threadIdx.x == 0) {
    volatile uint32_t* gen = &me->a2aGen;
    const uint32_t g = *gen;
    __threadfence_system();
    if (atomicAdd(&me->a2aArrive, 1u) == gridDim.x - 1) {
      atomicExch(&me->a2aArrive, 0u);
      __threadfence();
      atomicAdd(&me->a2aGen, 1u);
    } else if (*gen == g) {
      const uint32_t rc = waitGenSlow(gen, g, &me->abort, a.timeoutNs);
      if (rc != 0u) {
        reportAbort(a, rc, a.rank);
        ok = 0;
      }
    }
    __threadfence();
  }
  return __syncthreads_and(ok) != 0;
}

// Exclusive prefix sum over the CTA (one value per thread); `total` gets the sum.
__device__ __forceinline__ unsigned long long blockExclusiveScan(unsigned long long v, unsigned long long* warpSums,
                                                                 unsigned long long& total) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  unsigned long long x = v;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warpSums[w] = x;
  __syncthreads();
  if (w == 0) {
    unsigned long long s = lane < nw ? warpSums[lane] : 0ull;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long y = __shfl_up_sync(0xffffffffu, s, o);
      if (lane >= o) s += y;
    }
    if (lane < nw) warpSums[lane] = s;
  }
  __syncthreads();
  total = warpSums[nw - 1];
  const unsigned long long r = x - v + (w > 0 ? warpSums[w - 1] : 0ull);
  __syncthreads();
  return r;
}

__device__ __forceinline__ uint32_t ldPad(const uint32_t* p) { return *reinterpret_cast<const volatile uint32_t*>(p); }

// ---- agree: publish, barrier 1, check ---------------------------------------------------------
// My header and my P·E row counts (kA2aBad for one that is not a valid row count) go into column
// `me` of every rank's a2aHdr / a2aCount, spread over the grid; the combine also clears its column
// of every rank's a2aPosBad. After barrier 1, `invalid` tells whether any rank's header differs
// from mine or reports bad input of its own, or any count is not a valid row count, and sCap[s]
// holds rank s's capacity. Returns whether barrier 1 (and the grid sync before it) held.
__device__ __forceinline__ bool a2aAgree(const CommArgs& a, uint32_t ep, const long long* splits, const MoeArgs& d,
                                         uint32_t word, bool localBad, bool clearPosBad, unsigned long long* sCap,
                                         bool& invalid) {
  const int P = a.nranks, K = P * d.experts, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
  for (size_t i = gtid; i < static_cast<size_t>(P) * K; i += gthreads) {
    const int peer = static_cast<int>(i / K), k = static_cast<int>(i % K);
    const long long x = splits[k];
    a.sig[peer]->a2aCount[k][me] = (x < 0 || x > 0x7fffffffll) ? kA2aBad : static_cast<uint32_t>(x);
  }
  if (blockIdx.x == 0 && t < P) {
    uint32_t* h = &a.sig[t]->a2aHdr[0][me];
    const uint32_t hdr[kA2aHdrWords] = {static_cast<uint32_t>(rb), static_cast<uint32_t>(d.experts),
                                        static_cast<uint32_t>(d.align), word, d.capRows, localBad ? 1u : 0u};
#pragma unroll
    for (int w = 0; w < kA2aHdrWords; w++) h[w * kMaxRanks] = hdr[w];
    if (clearPosBad) a.sig[t]->a2aPosBad[me] = 0u;
  }
  // CTA b's release at the barrier must cover what the other CTAs published.
  const bool ok1 = localGridSync(a) && blockBarrier(a, ep + 1);
  invalid = false;
  if (!ok1) return false;
  const SignalPad* pad = a.self;
  bool b = false;
  if (t < P) {
    const uint32_t want[4] = {static_cast<uint32_t>(rb), static_cast<uint32_t>(d.experts),
                              static_cast<uint32_t>(d.align), word};
#pragma unroll
    for (int w = 0; w < 4; w++) b = b || ldPad(&pad->a2aHdr[w][t]) != want[w];
    b = b || ldPad(&pad->a2aHdr[5][t]) != 0u;
    sCap[t] = ldPad(&pad->a2aHdr[4][t]);
  }
  for (int i = t; i < P * K; i += blockDim.x) b = b || ldPad(&pad->a2aCount[i % K][i / K]) == kA2aBad;
  invalid = __syncthreads_or(b) != 0;
  return true;
}

// Thread 0 of CTA 0, once every rank's input is known: raise the first error, if any, on the host.
// An overflow names the first rank whose layout needs more rows than it has.
__device__ __forceinline__ void a2aReport(InputStatus* status, bool invalid, int P, const unsigned long long* sNeed,
                                          const unsigned long long* sCap) {
  int over = -1;
  if (!invalid) {
    for (int j = P - 1; j >= 0; j--) over = sNeed[j] > sCap[j] ? j : over;
  }
  volatile InputStatus* st = status;
  if (st != nullptr && (invalid || over >= 0) && st->code == kInputOk) {
    st->rank = over >= 0 ? static_cast<uint32_t>(over) : 0u;
    st->need = over >= 0 ? sNeed[over] : 0ull;
    st->avail = over >= 0 ? sCap[over] : 0ull;
    __threadfence_system();
    st->code = invalid ? kInputInvalid : kInputOverflow;
  }
}

// ---- forward layout ----------------------------------------------------------------------------
// From the count matrix: chunk k = j·E + e of my input lands on rank j from row sDst[k] on, which
// is where expert e's segment starts on j (a multiple of `align`) plus the rows of sources before
// me in it. sAux[k] ends as that segment start, sNeed[j] as the rows rank j needs, up to the end
// of its last segment.
__device__ __forceinline__ void a2aForwardLayout(const SignalPad* pad, int P, int E, int me, int align,
                                                 unsigned long long* sDst, unsigned long long* sAux,
                                                 unsigned long long* sNeed) {
  const int t = threadIdx.x, K = P * E;
  if (t < K) {
    unsigned long long before = 0, all = 0;
    for (int s = 0; s < P; s++) {
      const unsigned long long m = ldPad(&pad->a2aCount[t][s]);
      before += s < me ? m : 0ull;
      all += m;
    }
    sDst[t] = before;
    sAux[t] = all;
  }
  __syncthreads();
  if (t < P) {
    unsigned long long base = 0;
    for (int e = 0; e < E; e++) {
      const unsigned long long n = sAux[t * E + e];
      sAux[t * E + e] = base;
      base += n;
      if (e + 1 < E) base = (base + align - 1) / align * align;
    }
    sNeed[t] = base;
  }
  __syncthreads();
  if (t < K) sDst[t] += sAux[t];
}

// After a2aForwardLayout: my receive segment t = e·P + s (first row sRcv[t], sRcvCnt[t] rows).
__device__ __forceinline__ void a2aReceiveSegments(const SignalPad* pad, int P, int E, int me,
                                                   const unsigned long long* sAux, unsigned long long* sRcv,
                                                   uint32_t* sRcvCnt) {
  const int t = threadIdx.x;
  if (t < P * E) {
    const int e = t / P, s = t % P;
    unsigned long long off = sAux[me * E + e];
    for (int s2 = 0; s2 < s; s2++) off += ldPad(&pad->a2aCount[me * E + e][s2]);
    sRcv[t] = off;
    sRcvCnt[t] = ldPad(&pad->a2aCount[me * E + e][s]);
  }
  __syncthreads();
}

// The dispatches' layout: a2aForwardLayout and a2aReceiveSegments; CTA 0 reports the outcome and,
// when the call is valid and they are given, stores the segments to outSplits / outOffsets.
__device__ __forceinline__ void a2aDispatchLayout(const CommArgs& a, bool ok1, bool invalid, const MoeArgs& d,
                                                  long long* outSplits, long long* outOffsets,
                                                  unsigned long long* sDst, unsigned long long* sAux,
                                                  unsigned long long* sNeed, const unsigned long long* sCap,
                                                  unsigned long long* sRcv, uint32_t* sRcvCnt) {
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const SignalPad* pad = a.self;
  if (ok1 && !invalid) {
    a2aForwardLayout(pad, P, E, me, d.align, sDst, sAux, sNeed);
    a2aReceiveSegments(pad, P, E, me, sAux, sRcv, sRcvCnt);
  }
  if (ok1 && blockIdx.x == 0) {
    if (t == 0) a2aReport(d.status, invalid, P, sNeed, sCap);
    if (!invalid && outSplits != nullptr && t < K) {
      outSplits[t] = sRcvCnt[t];
      outOffsets[t] = static_cast<long long>(sRcv[t]);
    }
  }
}

// ---- finish a dispatch: barrier 2, staged copy-out, retire --------------------------------------
// A plain output is copied from my staging area (`stage`) once every CTA of every peer has pushed:
// the forward forms segment by segment, so that alignment gaps of the output stay untouched (the
// quantising forms' scales follow my `capRows` rows of codes there); the inverse form in one piece.
// The segment-by-segment copy: rows of `rb` bytes from `stage` to `out`, and, quantising, their
// scales from after `capRows` rows of codes in `stage` to `outScales`.
template <bool kQuant>
__device__ __forceinline__ void a2aCopyOut(char* out, float* outScales, const char* stage, unsigned long long rb,
                                           unsigned long long capRows, int K, const unsigned long long* sRcv,
                                           const uint32_t* sRcvCnt, size_t tid, size_t nthreads) {
  for (int k = 0; k < K; k++) {
    const unsigned long long n = sRcvCnt[k];
    if (n > 0) gridCopy(out + sRcv[k] * rb, stage + sRcv[k] * rb, n * rb, true, tid, nthreads);
    if constexpr (kQuant) {
      const unsigned long long sb = rb / kFp8Block * sizeof(float);  // scale bytes per row
      if (n > 0) {
        gridCopy(reinterpret_cast<char*>(outScales) + sRcv[k] * sb, stage + capRows * rb + sRcv[k] * sb, n * sb, true,
                 tid, nthreads);
      }
    }
  }
}

template <bool kQuant>
__device__ __forceinline__ void a2aFinish(const CommArgs& a, uint32_t ep, bool moved, const MoeKernelArgs<kQuant>& d,
                                          bool inverse, const unsigned long long* sRcv, const uint32_t* sRcvCnt,
                                          const unsigned long long* sNeed, const unsigned long long* sCap, int K,
                                          const char* stage) {
  blockBarrier(a, ep + 2);
  // NO pad table reads from here on. Once every CTA of every rank has arrived at barrier 2 a peer
  // may finish and start its next launch, which rewrites its column of my tables before its own
  // barrier 1 without waiting for anything. Everything below comes from shared memory.
  if (d.staged != nullptr) {
    const int me = a.rank;
    const bool synced = localGridSync(a);
    if (synced && moved && sNeed[me] <= sCap[me] && ld_relaxed_sys(&a.self->abort) == 0u) {
      const unsigned long long rb = d.rowBytes;
      const size_t tid = static_cast<size_t>(blockIdx.x) * blockDim.x + threadIdx.x;
      const size_t nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      if (inverse) {
        gridCopy(d.staged, stage, sNeed[me] * rb, true, tid, nthreads);
      } else {
        float* outScales = nullptr;
        if constexpr (kQuant) outScales = d.stagedScales;
        a2aCopyOut<kQuant>(d.staged, outScales, stage, rb, sCap[me], K, sRcv, sRcvCnt, tid, nthreads);
      }
    }
  }
  retire(a, 2, 0);
}

// ---- quantise: bf16 blocks of kFp8Block elements to e4m3 codes and one fp32 scale ---------------
constexpr int kQuantUnroll = 4;      // blocks in flight per half-warp

// A half-warp owns a block: each lane loads 8 elements (16 bytes), the block amax takes 4 shuffles
// within the 16 lanes, each lane stores 8 codes (8 bytes), lane 0 of the half stores the scale.
// Numerics: quantAmax / e4m3Multiplier / e4m3Codes2 / e4m3Scale (device_common.cuh).
// One block in a half-warp: `v` is this lane's 8 bf16 elements; returns its 8 codes and sets
// `amax` (the scale is amax / 448). Every lane of the warp must call it: the amax shuffles run
// with a full mask and stay within each half.
__device__ __forceinline__ uint2 quantBlock(const uint4& v, float& amax) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  float f[8];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
  amax = 0.0f;
#pragma unroll
  for (int i = 0; i < 8; i++) amax = fmaxf(amax, fabsf(f[i]));
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  amax = quantAmax(amax);
  const float s = e4m3Multiplier(amax);
  uint32_t c[4];
#pragma unroll
  for (int i = 0; i < 4; i++) c[i] = e4m3Codes2(f[2 * i], f[2 * i + 1], s);
  return make_uint2(c[0] | (c[1] << 16), c[2] | (c[3] << 16));
}

// One step of a warp: blocks b0 + 2·u + half (u < kQuantUnroll) of the `nblk` blocks at `in`
// are loaded, then quantised one by one, each handed to `emit(u, blk, codes, amax)`. Warp-uniform,
// so the shuffles run with a full mask; lanes past the end take part with zeros.
template <typename Emit>
__device__ __forceinline__ void quantStep(const char* in, unsigned long long b0, unsigned long long nblk, int lane,
                                          Emit&& emit) {
  const int half = lane >> 4, hl = lane & 15;
  uint4 v[kQuantUnroll];
#pragma unroll
  for (int u = 0; u < kQuantUnroll; u++) {
    const unsigned long long blk = b0 + 2 * u + half;
    v[u] = blk < nblk ? *reinterpret_cast<const uint4*>(in + blk * (2 * kFp8Block) + hl * 16) : make_uint4(0u, 0u, 0u, 0u);
  }
#pragma unroll
  for (int u = 0; u < kQuantUnroll; u++) {
    float amax;
    const uint2 c = quantBlock(v[u], amax);
    emit(u, b0 + 2 * u + half, c, amax);
  }
}

// Store one block's codes and scale to a destination (`codes`, `scales` at block 0).
__device__ __forceinline__ void quantStore(char* codes, float* scales, unsigned long long blk, unsigned long long nblk,
                                           int lane, uint2 c, float amax) {
  const int hl = lane & 15;
  if (blk < nblk) {
    *reinterpret_cast<uint2*>(codes + blk * kFp8Block + hl * 8) = c;
    if (hl == 0) scales[blk] = e4m3Scale(amax);
  }
}

// A chunk of `nblk` blocks, grid-strided: bf16 at `in`, codes to `codes`, scales to `scales`.
// `tid` / `nthreads` are multiples of 32 apart from the lane, like every caller of gridCopy.
__device__ __forceinline__ void quantCopy(char* codes, float* scales, const char* in, unsigned long long nblk,
                                          size_t tid, size_t nthreads) {
  const int lane = static_cast<int>(tid & 31);
  const unsigned long long nwarps = nthreads / 32, warp = tid / 32;
  for (unsigned long long b0 = warp * (2 * kQuantUnroll); b0 < nblk; b0 += nwarps * (2 * kQuantUnroll)) {
    quantStep(in, b0, nblk, lane, [&](int, unsigned long long blk, uint2 c, float amax) {
      quantStore(codes, scales, blk, nblk, lane, c, amax);
    });
  }
}

}  // namespace

// ---- device-split all-to-all-v -----------------------------------------------------------------
// The quantising form (kQuant): bf16 rows of H elements in, e4m3 codes (rowBytes = H) and one fp32
// scale per 128-element block out. The scales of rank j go to `scales.p[j]`, row-major
// (rows, H / 128), or, staged, into j's staging area right after its `capRows` rows of codes.
template <bool kQuant>
__global__ void __launch_bounds__(kThreads)
alltoallvDevKernel(CommArgs a, PeerPtrs outs, const char* in, unsigned long long inRows, const long long* inSplits,
                   const long long* inOffsets, long long* outSplits, long long* outOffsets, int inverse,
                   MoeKernelArgs<kQuant> d) {
  __shared__ unsigned long long sSrc[kMaxK];  // my chunk k: first input row
  __shared__ unsigned long long sDst[kMaxK];  //             first row in its destination's output
  __shared__ unsigned long long sAux[kMaxK];  // forward: column sums, then expert bases; inverse: R[j][s]
  __shared__ unsigned long long sRcv[kMaxK];  // forward: first row of my receive segment e·P+s
  __shared__ uint32_t sRcvCnt[kMaxK];         //          and its rows
  __shared__ uint32_t sCnt[kMaxK];            // my chunk k: rows
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks], sBytes[kMaxRanks];
  __shared__ unsigned long long sBlkOff[kMaxRanks], sBlkLen[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;

  // ---- my own splits: validate, and where each chunk starts in my input ----
  long long v = 0, o = 0;
  bool bad = false;
  if (t < K) {
    v = inSplits[t];
    bad = v < 0 || v > 0x7fffffffll;
    if (inverse) {
      o = inOffsets[t];
      bad = bad || o < 0 || static_cast<unsigned long long>(o) > inRows ||
            (!bad && static_cast<unsigned long long>(v) > inRows - static_cast<unsigned long long>(o));
    }
  }
  const unsigned long long c = bad ? 0ull : static_cast<unsigned long long>(v);
  unsigned long long inTotal;
  const unsigned long long prefix = blockExclusiveScan(t < K ? c : 0ull, sWarp, inTotal);
  if (t < K) {
    sCnt[t] = static_cast<uint32_t>(c);
    sSrc[t] = inverse ? static_cast<unsigned long long>(o) : prefix;
  }
  const bool localBad = __syncthreads_or(bad || (!inverse && inTotal > inRows)) != 0;

  // ---- agree, then every offset from the count matrix ----
  const uint32_t word = a2aHeaderWord(inverse ? A2aForm::kInverse : A2aForm::kForward, kQuant, d.plain != 0);
  bool invalid;
  const bool ok1 = a2aAgree(a, ep, inSplits, d, word, localBad, false, sCap, invalid);
  if (!inverse) {
    a2aDispatchLayout(a, ok1, invalid, d, outSplits, outOffsets, sDst, sAux, sNeed, sCap, sRcv, sRcvCnt);
  } else {
    if (ok1 && !invalid) {
      // R[j][s] = rows holder j returns to rank s.
      const SignalPad* pad = a.self;
      for (int i = t; i < P * P; i += blockDim.x) {
        const int j = i / P, s = i % P;
        unsigned long long r = 0;
        for (int e = 0; e < E; e++) r += ldPad(&pad->a2aCount[e * P + s][j]);
        sAux[i] = r;
      }
      __syncthreads();
      if (t < P) {
        unsigned long long need = 0, base = 0;
        for (int j = 0; j < P; j++) {
          need += sAux[j * P + t];
          base += j < me ? sAux[j * P + t] : 0ull;
        }
        sNeed[t] = need;
        for (int e = 0; e < E; e++) {
          sDst[e * P + t] = base;
          base += sCnt[e * P + t];
        }
      }
      __syncthreads();
    }
    if (ok1 && blockIdx.x == 0 && t == 0) a2aReport(d.status, invalid, P, sNeed, sCap);
  }
  if (ok1 && !invalid) {
    if (t < P) {
      unsigned long long rows = 0;
      for (int i = 0; i < E; i++) rows += sCnt[inverse ? i * P + t : t * E + i];
      sBytes[t] = sNeed[t] > sCap[t] ? 0ull : rows * rb;  // an overflowing destination gets nothing
    }
    __syncthreads();
    if (t == 0) {
      // CTAs dealt to destinations in proportion to their bytes, at least one each (as launchAlltoallPush).
      // The share is computed in double (spare x bytes may not fit 64 bits) and the running total
      // is clamped, so rounding can never deal out more CTAs than the grid has.
      unsigned long long total = 0, used = 0, extraUsed = 0;
      for (int j = 0; j < P; j++) total += sBytes[j];
      const unsigned long long spare = gridDim.x > static_cast<unsigned>(P) ? gridDim.x - P : 0u;
      for (int j = 0; j < P; j++) {
        unsigned long long extra =
            total > 0 ? static_cast<unsigned long long>(static_cast<double>(spare) * static_cast<double>(sBytes[j]) /
                                                        static_cast<double>(total))
                      : 0ull;
        extra = extra < spare - extraUsed ? extra : spare - extraUsed;
        extraUsed += extra;
        sBlkOff[j] = used;
        sBlkLen[j] = 1 + extra;
        used += sBlkLen[j];
      }
    }
    __syncthreads();

    // ---- payload ----
    const bool partitioned = gridDim.x >= static_cast<unsigned>(P);
    for (int i = 0; i < P; i++) {
      const int dst = (me + i) % P;
      if (sBytes[dst] == 0) continue;
      size_t tid, nthreads;
      if (partitioned) {
        const size_t b0 = sBlkOff[dst], nb = sBlkLen[dst];
        if (blockIdx.x < b0 || blockIdx.x >= b0 + nb) continue;
        tid = (blockIdx.x - b0) * blockDim.x + t;
        nthreads = nb * blockDim.x;
      } else {
        tid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
        nthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      }
      for (int x = 0; x < E; x++) {
        const int k = inverse ? x * P + dst : dst * E + x;
        if (sCnt[k] == 0) continue;
        if constexpr (kQuant) {
          // Input rows are 2·rb bytes (bf16); a row is rb / 128 blocks.
          const unsigned long long bpr = rb / kFp8Block;
          char* codes = static_cast<char*>(outs.p[dst]);
          float* scales = d.plain ? reinterpret_cast<float*>(codes + sCap[dst] * rb)
                                  : static_cast<float*>(d.scales.p[dst]);
          quantCopy(codes + sDst[k] * rb, scales + sDst[k] * bpr, in + sSrc[k] * rb * 2, sCnt[k] * bpr, tid, nthreads);
        } else {
          gridCopy(static_cast<char*>(outs.p[dst]) + sDst[k] * rb, in + sSrc[k] * rb, sCnt[k] * rb, true, tid, nthreads);
        }
      }
    }
  }
  a2aFinish<kQuant>(a, ep, ok1 && !invalid, d, inverse != 0, sRcv, sRcvCnt, sNeed, sCap, K,
                    static_cast<const char*>(outs.p[me]));
}

void launchAlltoallvDev(const CommArgs& a, const PeerPtrs& outs, const MoeArgs& d, const MoeScales* scales,
                        const void* in, size_t inRows, const long long* inSplits, const long long* inOffsets,
                        long long* outSplits, long long* outOffsets, bool inverse, int blocks, cudaStream_t stream) {
  const char* x = static_cast<const char*>(in);
  if (scales != nullptr) {
    alltoallvDevKernel<true><<<blocks, kThreads, 0, stream>>>(a, outs, x, inRows, inSplits, inOffsets, outSplits,
                                                              outOffsets, inverse, MoeQuantArgs{d, *scales});
  } else {
    alltoallvDevKernel<false><<<blocks, kThreads, 0, stream>>>(a, outs, x, inRows, inSplits, inOffsets, outSplits,
                                                               outOffsets, inverse, d);
  }
}

// ---- top-k MoE combine: pull each token's expert rows and sum them with its gate weights ---------
// The mirror of the forward dispatch, run by the source. Chunk k = j·E + e of my dispatch input
// (splits[k] rows, starting at row sSrc[k]) lies on holder j from row sDst[k] on, sDst as the
// dispatch computes it from the same count matrix; so input row p of chunk k is holder row
// sDst[k] + (p - sSrc[k]). Each token's warp reads its k rows there and writes one row locally.
//   barrier 1  headers and counts published, with the dispatch's code
//   barrier 2  a plain expert_out copied into its holder's staging area; every rank's bad-pos word
//              published. The grid sync before it puts every local CTA's stores under CTA b's release:
//              the barrier pairs CTA b with CTA b only.
//   barrier 3  every rank has read its rows: holders may reuse expert_out and the staging area.
// Every path passes all three barriers, so ranks never wait for a different count. The backward
// below runs the same protocol up to the pull (topkPullPrologue) and the same choice lookup.
constexpr int kTopkInFlight = 4;  // choices whose packs a lane loads before it adds them
constexpr int kTopkPacks = 2;     // packs of one row per lane per step

namespace {
// The pulling forms up to barrier 2 and its verdict: where each chunk of my dispatch input starts
// (sSrc), every holder's expert_out (sBase), agree on `word`, the forward layout, a plain expert_out
// (d.staged) copied into my staging area, my `choices` pos entries checked, the grid sync and
// barrier 2, and every rank's verdict, which CTA 0 reports. Returns whether this rank may pull:
// every rank's input is valid and no holder overflows.
__device__ __forceinline__ bool topkPullPrologue(const CommArgs& a, uint32_t ep, const PeerPtrs& srcs,
                                                 const long long* splits, const long long* posIn,
                                                 unsigned long long choices, const MoeArgs& d, uint32_t word,
                                                 unsigned long long* sSrc, unsigned long long* sDst,
                                                 unsigned long long* sAux, unsigned long long* sNeed,
                                                 unsigned long long* sCap, const char** sBase,
                                                 unsigned long long* sWarp) {
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;

  // ---- 1. my splits, where each chunk starts in my input; agree ----
  const long long v = t < K ? splits[t] : 0ll;
  const bool bad = v < 0 || v > 0x7fffffffll;
  unsigned long long inRows;
  const unsigned long long prefix = blockExclusiveScan(bad ? 0ull : static_cast<unsigned long long>(v), sWarp, inRows);
  if (t < K) sSrc[t] = prefix;
  if (t < P) sBase[t] = static_cast<const char*>(srcs.p[t]);
  const bool localBad = __syncthreads_or(bad) != 0;
  bool invalid;
  const bool ok1 = a2aAgree(a, ep, splits, d, word, localBad, true, sCap, invalid);

  // ---- 2. the layout; stage a plain expert_out; check pos ----
  const SignalPad* pad = a.self;
  bool over = false;
  if (ok1 && !invalid) {
    a2aForwardLayout(pad, P, E, me, d.align, sDst, sAux, sNeed);
    over = __syncthreads_or(t < P && sNeed[t] > sCap[t]) != 0;
  }
  const bool go = ok1 && !invalid && !over;
  if (go && d.staged != nullptr) gridCopy(const_cast<char*>(sBase[me]), d.staged, sNeed[me] * rb, true, gtid, gthreads);
  if (go) {
    bool b = false;
    for (size_t i = gtid; i < choices; i += gthreads) {
      const long long p = posIn[i];
      b = b || p < -1 || (p >= 0 && static_cast<unsigned long long>(p) >= inRows);
    }
    if (__syncthreads_or(b) != 0 && t < P) a.sig[t]->a2aPosBad[me] = 1u;
  }
  const bool ok2 = localGridSync(a) && blockBarrier(a, ep + 2);

  // ---- 3. every rank's verdict ----
  bool posBad = false;
  if (ok2 && go) posBad = __syncthreads_or(t < P && ldPad(&pad->a2aPosBad[t]) != 0u) != 0;
  if (ok1 && ok2 && blockIdx.x == 0 && t == 0) a2aReport(d.status, invalid || posBad, P, sNeed, sCap);
  return ok2 && go && !posBad;
}

// Where row p of my dispatch input lies: the last chunk starting at or before p holds it (an empty
// chunk starts where the next one does); its holder is chunk / E, the row there is returned.
__device__ __forceinline__ unsigned long long topkHolderRow(const unsigned long long* sSrc,
                                                            const unsigned long long* sDst, int K, int E,
                                                            unsigned long long p, int& holder) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sSrc[mid] <= p) lo = mid; else hi = mid - 1;
  }
  holder = lo / E;
  return sDst[lo] + (p - sSrc[lo]);
}

// The combines' accumulate step: acc += w · float(x) for each element of a 16-byte pack, a correctly
// rounded fp32 multiply, then a correctly rounded add (never contracted to a fused multiply-add).
template <typename T>
__device__ __forceinline__ void topkAccumulate(typename PackTraits<T>::AccPack& acc, float w, const Pack16& x) {
  using PT = PackTraits<T>;
  const typename PT::AccPack xf = PT::widen(x);
#pragma unroll
  for (int i = 0; i < PT::kElems; i++) acc.v[i] = __fadd_rn(acc.v[i], __fmul_rn(w, xf.v[i]));
}
}  // namespace

template <typename T>
__global__ void __launch_bounds__(kThreads)
moeCombineTopkKernel(CommArgs a, PeerPtrs srcs, const long long* splits, const long long* posIn, const float* weights,
                     char* out, unsigned long long tokens, int topk, MoeArgs d) {
  using PT = PackTraits<T>;
  __shared__ unsigned long long sSrc[kMaxK];  // my chunk k: first row in my dispatch input
  __shared__ unsigned long long sDst[kMaxK];  //             first row on its holder
  __shared__ unsigned long long sAux[kMaxK];  // column sums, then expert bases
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks];
  __shared__ const char* sBase[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int K = a.nranks * d.experts, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;

  const bool pull = topkPullPrologue(a, ep, srcs, splits, posIn, tokens * static_cast<unsigned long long>(topk), d,
                                     a2aHeaderWord(A2aForm::kCombineTopk, false, d.plain != 0), sSrc, sDst, sAux,
                                     sNeed, sCap, sBase, sWarp);
  // ---- pull and reduce ----
  if (pull) {
    const int lane = t & 31, k = topk;
    const unsigned long long npk = rb / 16;
    for (unsigned long long tok = gtid / 32; tok < tokens; tok += gthreads / 32) {
      // Lane j < k: where choice j's row lies, and its weight (1 without weights).
      const char* src = nullptr;
      float w = 0.0f;
      if (lane < k) {
        const long long p = posIn[tok * k + lane];
        if (p >= 0) {
          int j;
          const unsigned long long row = topkHolderRow(sSrc, sDst, K, d.experts, static_cast<unsigned long long>(p), j);
          src = sBase[j] + row * rb;
          w = weights != nullptr ? weights[tok * k + lane] : 1.0f;
        }
      }
      char* dst = out + tok * rb;
      // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
      for (unsigned long long v0 = lane; v0 - lane < npk; v0 += 32 * kTopkPacks) {
        typename PT::AccPack acc[kTopkPacks];
#pragma unroll
        for (int u = 0; u < kTopkPacks; u++) {
#pragma unroll
          for (int i = 0; i < PT::kElems; i++) acc[u].v[i] = 0.0f;
        }
        for (int j0 = 0; j0 < k; j0 += kTopkInFlight) {
          const char* s[kTopkInFlight];
          float ws[kTopkInFlight];
          Pack16 x[kTopkInFlight][kTopkPacks];
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
            s[c] = reinterpret_cast<const char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(src), (j0 + c) & 31));
            ws[c] = __shfl_sync(0xffffffffu, w, (j0 + c) & 31);
            if (j0 + c >= k) s[c] = nullptr;
#pragma unroll
            for (int u = 0; u < kTopkPacks; u++) {
              const unsigned long long pk = v0 + 32ull * u;
              if (s[c] != nullptr && pk < npk) x[c][u] = ld128_stream(s[c] + pk * 16);
            }
          }
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
            if (s[c] == nullptr) continue;
#pragma unroll
            for (int u = 0; u < kTopkPacks; u++) topkAccumulate<T>(acc[u], ws[c], x[c][u]);
          }
        }
#pragma unroll
        for (int u = 0; u < kTopkPacks; u++) {
          const unsigned long long pk = v0 + 32ull * u;
          if (pk < npk) st128(dst + pk * 16, PT::narrow(acc[u]));
        }
      }
    }
  }
  blockBarrier(a, ep + 3);
  // NO pad table or peer reads from here on: a peer that has passed barrier 3 may start its next
  // launch, which rewrites its columns of my tables and its staging area.
  retire(a, 3, 0);
}

// ---- top-k MoE combine backward: pull, dot and push in one pass --------------------------------
// The backward of the weighted combine y[t] = sum_j w[t, j] · expert_out[row(t, j)], run by the
// source like the combine, with the same protocol up to the pull and the same (holder, row) of each
// choice. For each routed choice it reads the expert row over NVLink once and
//   grad_w[t, j]                  = <dy[t], expert_out[row]>, fp32 (+0.0 when pos = -1)
//   grad_expert_out[row] on holder = round_T(w[t, j] · float(dy[t])), one correctly rounded multiply
// The dot's order is fixed, so its bits do not depend on the grid: lane l sums, in fp32 with one
// fused multiply-add per element, the elements of packs l, l + 32, l + 64, ... in that order (each
// pack's elements in order), then a shfl_xor butterfly over distances 16, 8, 4, 2, 1 adds the lanes.
//   barrier 1, barrier 2  as in the combine
//   between 2 and 3       only if every rank's verdict is valid: pull, dot and push; each holder also
//                         writes +0 to every row of its grad_expert_out outside its receive segments
//                         (alignment gaps and the tail), so no rank writes anything when a call fails.
//   barrier 3             every rank has read its rows and pushed its gradient rows
//   after barrier 3       a plain grad_expert_out is copied out of my staging area, segment by segment.
// Staged (plain expert_out and grad_expert_out), a holder's staging area holds its expert_out copy
// in rows [0, cap) and the pushed gradient rows in [cap, 2·cap); senders take cap from its header.
// pos must name each routed dispatch-input row at most once (route() and the top-k dispatch do);
// staged, a segment row that no choice names is copied out with unspecified contents.
constexpr int kTopkBackPacks = 1;  // packs of one row per lane per step: dy, 4 choices' rows, 4 dots in registers

namespace {
__device__ __forceinline__ void gridZero(char* dst, unsigned long long bytes, size_t tid, size_t nthreads) {
  const Pack16 z = {{0u, 0u, 0u, 0u}};
  for (unsigned long long i = tid; i < bytes / 16; i += nthreads) st128(dst + i * 16, z);
}
}  // namespace

template <typename T>
__global__ void __launch_bounds__(kThreads)
moeCombineTopkBackwardKernel(CommArgs a, PeerPtrs srcs, PeerPtrs grads, const long long* splits,
                             const long long* posIn, const float* weights, const char* dy, float* gradW,
                             char* stagedGrad, unsigned long long tokens, unsigned long long capacity, int topk,
                             MoeArgs d) {
  using PT = PackTraits<T>;
  __shared__ unsigned long long sSrc[kMaxK];  // my chunk k: first row in my dispatch input
  __shared__ unsigned long long sDst[kMaxK];  //             first row on its holder
  __shared__ unsigned long long sAux[kMaxK];  // column sums, then expert bases
  __shared__ unsigned long long sRcv[kMaxK];  // first row of my receive segment e·P+s
  __shared__ uint32_t sRcvCnt[kMaxK];         // and its rows
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks];
  __shared__ const char* sBase[kMaxRanks];
  __shared__ char* sGrad[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const unsigned long long rb = d.rowBytes;
  const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
  const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;

  const bool pull = topkPullPrologue(a, ep, srcs, splits, posIn, tokens * static_cast<unsigned long long>(topk), d,
                                     a2aHeaderWord(A2aForm::kCombineTopkBackward, false, d.plain != 0), sSrc, sDst,
                                     sAux, sNeed, sCap, sBase, sWarp);
  if (pull) {
    a2aReceiveSegments(a.self, P, E, me, sAux, sRcv, sRcvCnt);
    if (t < P) sGrad[t] = d.plain ? const_cast<char*>(sBase[t]) + sCap[t] * rb : static_cast<char*>(grads.p[t]);
    __syncthreads();

    // ---- zero my rows outside the receive segments: the gap after each expert, the tail ----
    char* mine = d.plain ? stagedGrad : sGrad[me];
    if (mine != nullptr) {
      for (int e = 0; e < E; e++) {
        const int last = e * P + P - 1;
        const unsigned long long lo = sRcv[last] + sRcvCnt[last];
        const unsigned long long hi = e + 1 < E ? sAux[me * E + e + 1] : capacity;
        if (hi > lo) gridZero(mine + lo * rb, (hi - lo) * rb, gtid, gthreads);
      }
    }

    // ---- pull, dot and push: one warp per token ----
    const int lane = t & 31, k = topk;
    const unsigned long long npk = rb / 16;
    for (unsigned long long tok = gtid / 32; tok < tokens; tok += gthreads / 32) {
      // Lane j < k: choice j's expert row, its gradient row and its weight.
      const char* src = nullptr;
      char* dstG = nullptr;
      float w = 0.0f;
      if (lane < k) {
        const long long p = posIn[tok * k + lane];
        if (p >= 0) {
          int j;
          const unsigned long long row = topkHolderRow(sSrc, sDst, K, E, static_cast<unsigned long long>(p), j);
          src = sBase[j] + row * rb;
          dstG = sGrad[j] + row * rb;
          w = weights[tok * k + lane];
        }
      }
      const char* g = dy + tok * rb;
      for (int j0 = 0; j0 < k; j0 += kTopkInFlight) {
        const char* s[kTopkInFlight];
        char* q[kTopkInFlight];
        float ws[kTopkInFlight], part[kTopkInFlight];
#pragma unroll
        for (int c = 0; c < kTopkInFlight; c++) {
          s[c] = reinterpret_cast<const char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(src), (j0 + c) & 31));
          q[c] = reinterpret_cast<char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dstG), (j0 + c) & 31));
          ws[c] = __shfl_sync(0xffffffffu, w, (j0 + c) & 31);
          if (j0 + c >= k) s[c] = nullptr;
          part[c] = 0.0f;
        }
        // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
        for (unsigned long long v0 = lane; v0 - lane < npk; v0 += 32 * kTopkBackPacks) {
          Pack16 gv[kTopkBackPacks], x[kTopkInFlight][kTopkBackPacks];
#pragma unroll
          for (int u = 0; u < kTopkBackPacks; u++) {
            const unsigned long long pk = v0 + 32ull * u;
            if (pk < npk) gv[u] = ld128(g + pk * 16);
          }
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
#pragma unroll
            for (int u = 0; u < kTopkBackPacks; u++) {
              const unsigned long long pk = v0 + 32ull * u;
              if (s[c] != nullptr && pk < npk) x[c][u] = ld128_stream(s[c] + pk * 16);
            }
          }
#pragma unroll
          for (int u = 0; u < kTopkBackPacks; u++) {
            const unsigned long long pk = v0 + 32ull * u;
            if (pk >= npk) continue;
            const typename PT::AccPack gf = PT::widen(gv[u]);
#pragma unroll
            for (int c = 0; c < kTopkInFlight; c++) {
              if (s[c] == nullptr) continue;
              const typename PT::AccPack xf = PT::widen(x[c][u]);
              typename PT::AccPack o;
#pragma unroll
              for (int i = 0; i < PT::kElems; i++) {
                part[c] = __fmaf_rn(gf.v[i], xf.v[i], part[c]);
                o.v[i] = __fmul_rn(ws[c], gf.v[i]);
              }
              st128(q[c] + pk * 16, PT::narrow(o));
            }
          }
        }
#pragma unroll
        for (int c = 0; c < kTopkInFlight; c++) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) part[c] = __fadd_rn(part[c], __shfl_xor_sync(0xffffffffu, part[c], o));
        }
        if (lane == 0) {
#pragma unroll
          for (int c = 0; c < kTopkInFlight; c++) {
            if (j0 + c < k) gradW[tok * k + j0 + c] = s[c] != nullptr ? part[c] : 0.0f;
          }
        }
      }
    }
  }
  blockBarrier(a, ep + 3);
  // NO pad table or peer reads from here on (as in the combine). Every peer has pushed its rows
  // into my staging area: once every local CTA is past barrier 3, copy them out.
  if (stagedGrad != nullptr) {
    const bool synced = localGridSync(a);
    if (synced && pull && ld_relaxed_sys(&a.self->abort) == 0u) {
      a2aCopyOut<false>(stagedGrad, nullptr, sGrad[me], rb, 0, K, sRcv, sRcvCnt, gtid, gthreads);
    }
  }
  retire(a, 3, 0);
}

namespace {
// The top-k combine instantiation for dt: float, bfloat16 or float16 rows (null for any other).
using TopkCombineFn = void (*)(CommArgs, PeerPtrs, const long long*, const long long*, const float*, char*,
                               unsigned long long, int, MoeArgs);
TopkCombineFn topkCombineFn(DataType dt) {
  switch (dt) {
    case DataType::FLOAT32: return moeCombineTopkKernel<float>;
    case DataType::BFLOAT16: return moeCombineTopkKernel<__nv_bfloat16>;
    case DataType::FLOAT16: return moeCombineTopkKernel<__half>;
    default: return nullptr;
  }
}
// Its backward, for the same row types.
using TopkCombineBackwardFn = void (*)(CommArgs, PeerPtrs, PeerPtrs, const long long*, const long long*, const float*,
                                       const char*, float*, char*, unsigned long long, unsigned long long, int, MoeArgs);
TopkCombineBackwardFn topkCombineBackwardFn(DataType dt) {
  switch (dt) {
    case DataType::FLOAT32: return moeCombineTopkBackwardKernel<float>;
    case DataType::BFLOAT16: return moeCombineTopkBackwardKernel<__nv_bfloat16>;
    case DataType::FLOAT16: return moeCombineTopkBackwardKernel<__half>;
    default: return nullptr;
  }
}
}  // namespace

void launchMoeCombineTopkBackward(const CommArgs& a, const PeerPtrs& srcs, const PeerPtrs& grads, const MoeArgs& d,
                                  void* stagedGrad, size_t capacityRows, const void* dy, float* gradWeights,
                                  size_t tokens, int topk, const long long* pos, const float* weights,
                                  const long long* splits, DataType dt, int blocks, cudaStream_t stream) {
  topkCombineBackwardFn(dt)<<<blocks, kThreads, 0, stream>>>(a, srcs, grads, splits, pos, weights,
                                                             static_cast<const char*>(dy), gradWeights,
                                                             static_cast<char*>(stagedGrad), tokens, capacityRows,
                                                             topk, d);
}

void launchMoeCombineTopk(const CommArgs& a, const PeerPtrs& srcs, const MoeArgs& d, void* out, size_t tokens,
                          int topk, const long long* pos, const float* weights, const long long* splits, DataType dt,
                          int blocks, cudaStream_t stream) {
  topkCombineFn(dt)<<<blocks, kThreads, 0, stream>>>(a, srcs, splits, pos, weights, static_cast<char*>(out), tokens,
                                                     topk, d);
}

// ---- top-k MoE dispatch: route each token from its gate indices and push its row to every choice ----
// The forward dispatch of route(x, topk_idx) without its T·k-row copy: each token's row is read
// once (and quantised once) and stored to each of its k destination rows. The layout, splits and
// pos are those of route() + the forward alltoallvDevKernel, byte for byte.
//   route (before barrier 1, local): group g = topk_idx entry, in 0..P·E-1 (anything else is not
//     routed). CTA b owns a contiguous slice of tokens. It counts every choice of every token
//     (the totals, which every CTA needs for pos) and those before its slice (its base), then ranks
//     its slice's choices in (token, choice) order: within a warp by __match_any_sync, across the
//     warps of a round in warp order through shared running counts. No atomic decides a place.
//     pos = (rows of groups before g) + (choices of g before this one); CTA 0 writes splits.
//   agree / dispatch layout: as the forward exchange, with its own form in the header.
//   push: one warp per token of my slice; a lane per choice finds its destination row
//     sDst[g] + (pos - sSrc[g]) on rank g / E, then the warp reads each 16-byte pack (or, quantising,
//     each 128-element block) once and stores it to every destination that does not overflow.
//   barrier 2, staged copy-out and retire as in the forward exchange.
constexpr int kTopkPushUnroll = 4;  // packs of a row in flight per lane
static_assert(kThreads >= kMaxRanks * kMaxA2aExperts, "one scan slot per group");

__device__ __forceinline__ int topkGroup(long long v, int K) { return v >= 0 && v < K ? static_cast<int>(v) : K; }

namespace {
// Route, first half: the routed choices of every group g over all `n` choices (sTot[g]), route()'s
// first row of g (sSrc[g], their exclusive prefix) and the choices of g before choice `lo`, where my
// CTA's slice starts (sRun[g]). `totals(g)` runs for each g on thread g once sTot[g] is final.
template <typename Totals>
__device__ __forceinline__ void topkRouteCount(const long long* idx, unsigned long long n, unsigned long long lo, int K,
                                               uint32_t* sTot, uint32_t* sRun, unsigned long long* sSrc,
                                               unsigned long long* sWarp, Totals&& totals) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  for (int g = t; g < K; g += blockDim.x) sTot[g] = sRun[g] = 0u;
  __syncthreads();
  for (unsigned long long b = static_cast<unsigned long long>(warp) * 32; b < n; b += blockDim.x) {
    const unsigned long long i = b + lane;
    const int g = i < n ? topkGroup(idx[i], K) : K;
    const bool before = i < lo;
    const unsigned m = __match_any_sync(0xffffffffu, 2 * g + (before ? 1 : 0));
    if (g < K && lane == __ffs(m) - 1) {
      atomicAdd(&sTot[g], static_cast<uint32_t>(__popc(m)));
      if (before) atomicAdd(&sRun[g], static_cast<uint32_t>(__popc(m)));
    }
  }
  __syncthreads();
  unsigned long long routed;
  const unsigned long long first = blockExclusiveScan(t < K ? sTot[t] : 0u, sWarp, routed);
  if (t < K) {
    sSrc[t] = first;
    totals(t);
  }
  __syncthreads();
}

// Route, second half: rank the choices [lo, hi) of my slice in (token, choice) order, within a warp by
// __match_any_sync, across the warps of a round in warp order through the running counts sRun.
// `emit(i, g, p)` gets choice i's group (K: not routed) and pos (-1: not routed).
template <typename Emit>
__device__ __forceinline__ void topkRouteRank(const long long* idx, unsigned long long lo, unsigned long long hi, int K,
                                              const unsigned long long* sSrc, uint32_t* sRun, Emit&& emit) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, nw = blockDim.x >> 5;
  for (unsigned long long b = lo; b < hi; b += blockDim.x) {
    const unsigned long long i = b + t;
    const int g = i < hi ? topkGroup(idx[i], K) : K;
    const unsigned m = __match_any_sync(0xffffffffu, g);
    const unsigned below = m & ((1u << lane) - 1u);
    long long p = -1;
    for (int w = 0; w < nw; w++) {
      if (warp == w && g < K) {
        const uint32_t r = sRun[g];
        __syncwarp(m);
        if (below == 0u) sRun[g] = r + static_cast<uint32_t>(__popc(m));
        p = static_cast<long long>(sSrc[g] + r + static_cast<uint32_t>(__popc(below)));
      }
      __syncthreads();
    }
    if (i < hi) emit(i, g, p);
  }
}

// Push one token's row `src` (rb bytes; quantising: rb / 128 bf16 blocks of 2 · 128 bytes) to every
// choice c < topk whose lane holds a destination `dst` (and, quantising, its scales `dsc`): each
// 16-byte pack, or each 128-element block, is read and quantised once. Called by the whole warp.
template <bool kQuant>
__device__ __forceinline__ void topkPushRow(const char* src, unsigned long long rb, int lane, int topk, char* dst,
                                            float* dsc) {
  if constexpr (kQuant) {
    // Half-warps take 128-element blocks, as quantCopy: one amax and one set of codes per block.
    const unsigned long long nblk = rb / kFp8Block;
    for (unsigned long long b0 = 0; b0 < nblk; b0 += 2 * kQuantUnroll) {
      uint2 c[kQuantUnroll];
      float amax[kQuantUnroll];
      quantStep(src, b0, nblk, lane, [&](int u, unsigned long long, uint2 cu, float au) {
        c[u] = cu;
        amax[u] = au;
      });
      for (int ch = 0; ch < topk; ch++) {
        char* q = reinterpret_cast<char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dst), ch));
        float* qs = reinterpret_cast<float*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dsc), ch));
        if (q == nullptr) continue;
#pragma unroll
        for (int u = 0; u < kQuantUnroll; u++) quantStore(q, qs, b0 + 2 * u + (lane >> 4), nblk, lane, c[u], amax[u]);
      }
    }
  } else {
    const unsigned long long npk = rb / 16;
    // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
    for (unsigned long long v0 = lane; v0 - lane < npk; v0 += 32 * kTopkPushUnroll) {
      Pack16 xv[kTopkPushUnroll];
#pragma unroll
      for (int u = 0; u < kTopkPushUnroll; u++) {
        const unsigned long long pk = v0 + 32ull * u;
        if (pk < npk) xv[u] = ld128_stream(src + pk * 16);
      }
      for (int ch = 0; ch < topk; ch++) {
        char* q = reinterpret_cast<char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(dst), ch));
        if (q == nullptr) continue;
#pragma unroll
        for (int u = 0; u < kTopkPushUnroll; u++) {
          const unsigned long long pk = v0 + 32ull * u;
          if (pk < npk) st128_stream(q + pk * 16, xv[u]);
        }
      }
    }
  }
}
}  // namespace

template <bool kQuant>
__global__ void __launch_bounds__(kThreads)
moeDispatchTopkKernel(CommArgs a, PeerPtrs outs, const char* x, const long long* idx, long long* splits, long long* pos,
                      long long* outSplits, long long* outOffsets, unsigned long long tokens, int topk,
                      MoeKernelArgs<kQuant> d) {
  __shared__ unsigned long long sSrc[kMaxK];  // group g: first row of route()'s rows
  __shared__ unsigned long long sDst[kMaxK];  //          first row on rank g / E
  __shared__ unsigned long long sAux[kMaxK];  // my splits (published), then column sums / expert bases
  __shared__ unsigned long long sRcv[kMaxK];  // first row of my receive segment e·P+s
  __shared__ uint32_t sRcvCnt[kMaxK];         // and its rows
  __shared__ uint32_t sTot[kMaxK];            // group g: routed choices of all my tokens
  __shared__ uint32_t sRun[kMaxK];            //          of the tokens before my slice, then running
  __shared__ unsigned long long sNeed[kMaxRanks], sCap[kMaxRanks];
  __shared__ unsigned long long sWarp[32];
  const uint32_t ep = loadEpoch(a);
  const int P = a.nranks, E = d.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = blockDim.x >> 5;
  const unsigned long long rb = d.rowBytes, k = static_cast<unsigned long long>(topk);

  // ---- route: counts, then pos of my slice ----
  const unsigned long long per = (tokens + gridDim.x - 1) / gridDim.x;
  const unsigned long long tok0 = min(tokens, blockIdx.x * per), tok1 = min(tokens, tok0 + per);
  const unsigned long long lo = tok0 * k, hi = tok1 * k;
  topkRouteCount(idx, tokens * k, lo, K, sTot, sRun, sSrc, sWarp, [&](int g) {
    sAux[g] = sTot[g];
    if (blockIdx.x == 0) splits[g] = sTot[g];
  });
  topkRouteRank(idx, lo, hi, K, sSrc, sRun, [&](unsigned long long i, int, long long p) { pos[i] = p; });

  // ---- agree on my splits; the layout ----
  bool invalid;
  const bool ok1 = a2aAgree(a, ep, reinterpret_cast<const long long*>(sAux), d,
                            a2aHeaderWord(A2aForm::kDispatchTopk, kQuant, d.plain != 0), false, false, sCap,
                            invalid);
  a2aDispatchLayout(a, ok1, invalid, d, outSplits, outOffsets, sDst, sAux, sNeed, sCap, sRcv, sRcvCnt);

  // ---- push: one warp per token of my slice ----
  if (ok1 && !invalid) {
    for (unsigned long long tok = tok0 + warp; tok < tok1; tok += nw) {
      // Lane c < k: where choice c's row goes; null when it is not routed or its rank overflows.
      char* dst = nullptr;
      float* dsc = nullptr;
      if (static_cast<unsigned long long>(lane) < k) {
        const unsigned long long i = tok * k + lane;
        const int g = topkGroup(idx[i], K);
        if (g < K && sNeed[g / E] <= sCap[g / E]) {
          const int j = g / E;
          const unsigned long long row = sDst[g] + (static_cast<unsigned long long>(pos[i]) - sSrc[g]);
          dst = static_cast<char*>(outs.p[j]) + row * rb;
          if constexpr (kQuant) {
            float* sc = d.plain ? reinterpret_cast<float*>(static_cast<char*>(outs.p[j]) + sCap[j] * rb)
                                : static_cast<float*>(d.scales.p[j]);
            dsc = sc + row * (rb / kFp8Block);
          }
        }
      }
      topkPushRow<kQuant>(x + tok * rb * (kQuant ? 2 : 1), rb, lane, topk, dst, dsc);
    }
  }
  a2aFinish<kQuant>(a, ep, ok1 && !invalid, d, false, sRcv, sRcvCnt, sNeed, sCap, K,
                    static_cast<const char*>(outs.p[me]));
}

void launchMoeDispatchTopk(const CommArgs& a, const PeerPtrs& outs, const MoeArgs& d, const MoeScales* scales,
                           const void* x, size_t tokens, int topk, const long long* idx, long long* splits,
                           long long* pos, long long* outSplits, long long* outOffsets, int blocks, cudaStream_t stream) {
  const char* xc = static_cast<const char*>(x);
  if (scales != nullptr) {
    moeDispatchTopkKernel<true><<<blocks, kThreads, 0, stream>>>(a, outs, xc, idx, splits, pos, outSplits, outOffsets,
                                                                 tokens, topk, MoeQuantArgs{d, *scales});
  } else {
    moeDispatchTopkKernel<false><<<blocks, kThreads, 0, stream>>>(a, outs, xc, idx, splits, pos, outSplits, outOffsets,
                                                                  tokens, topk, d);
  }
}

// ---- low-latency top-k exchange: fixed slots, one signal round each way ------------------------
// For decoding, where a layer moves a handful of rows and the variable layout's barriers dominate.
// Every rank owns a buffer of one layout (MoeLLLayout, agreed on the host when it is created), so
// nothing about shapes is agreed on the device: expert e of rank j has a fixed slot range
// [e][s][0, maxTokens) for each source s, and a source writes there without asking.
//   dispatch  route (as moeDispatchTopkKernel); push each routed choice of group g = j·E + e to slot
//             (e, me, r) of rank j, r its rank in g in (token, choice) order, with the int32 tag t·k + c;
//             a group with more than maxTokens rows (a token that picks an expert twice) sends nothing
//             and its choices are marked unsent. Local grid sync, then one release word per (j, e):
//             [e][me] on rank j = (call, form, rows). Wait for my E·P words of this call, pack expert
//             e's rows into out[e] in source order, write out_splits.
//   combine   every packed row of my experts goes to its source's combine slot named by its tag;
//             local grid sync, one release word to each source; wait for my P words and sum each
//             token's sent choices with its weights, as moeCombineTopkKernel.
// Waits are bounded by the context timeout and the abort word, as every barrier is. The call count
// lives in the buffer: every CTA reads it at entry and the last CTA to finish advances it, so CUDA
// graph replays keep counting. Dispatch and combine alternate on a buffer (the host enforces it):
// a source's next dispatch starts only after its combine has seen every holder's word, which each
// holder sends after it has read its slots and tags, so one set of slots serves every call.
namespace {
__device__ __forceinline__ void st_release_sys_u64(unsigned long long* p, unsigned long long v) {
  asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ unsigned long long ld_acquire_sys_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

// A signal word: bits 63..36 the call (count + 1, modulo 2^28), 35..32 the form, 31..0 the rows. A
// word is only ever compared for equality with the call a reader expects; the stale word it replaces
// is two calls older, and a fresh buffer's zero never names a call.
__host__ __device__ __forceinline__ unsigned long long llWord(uint32_t seq, uint32_t form, uint32_t count) {
  return (static_cast<unsigned long long>(((seq & 0x0fffffffu) << 4) | form) << 32) | count;
}
__device__ __forceinline__ bool llArrived(unsigned long long w, uint32_t seq) {
  return static_cast<uint32_t>(w >> 36) == (seq & 0x0fffffffu);
}
__device__ __forceinline__ uint32_t llForm(unsigned long long w) { return static_cast<uint32_t>(w >> 32) & 15u; }

__device__ __forceinline__ uint32_t llWaitSlow(const unsigned long long* w, uint32_t seq, uint32_t* abortWord,
                                                   unsigned long long timeoutNs) {
  const unsigned long long t0 = globalTimerNs();
  uint32_t polls = 0;
  while (!llArrived(ld_acquire_sys_u64(w), seq)) {
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

// Wait for call `seq`'s word at `w`, written by `peer`; false when the wait was abandoned.
__device__ __forceinline__ bool llWait(const CommArgs& a, const unsigned long long* w, uint32_t seq, int peer,
                                       unsigned long long& v) {
  v = ld_acquire_sys_u64(w);
  if (llArrived(v, seq)) return true;
  const uint32_t rc = llWaitSlow(w, seq, &a.self->abort, a.timeoutNs);
  if (rc == 0u) {
    v = ld_acquire_sys_u64(w);
    return true;
  }
  reportAbort(a, rc, peer);
  return false;
}

// Thread 0 of CTA 0: raise an input error on the host, unless one is pending.
__device__ __forceinline__ void llReport(InputStatus* status, uint32_t code, uint32_t source, uint32_t expert,
                                         unsigned long long rows, unsigned long long maxTokens) {
  volatile InputStatus* st = status;
  if (st != nullptr && st->code == kInputOk) {
    st->rank = source;
    st->expert = expert;
    st->need = rows;
    st->avail = maxTokens;
    __threadfence_system();
    st->code = code;
  }
}

// Every CTA at its end: the last one advances the buffer's call count.
__device__ __forceinline__ void llRetire(uint32_t* ctrl) {
  __syncthreads();
  if (threadIdx.x == 0 && atomicAdd(&ctrl[1], 1u) == gridDim.x - 1) {
    ctrl[1] = 0u;
    ctrl[0] += 1u;
  }
}

// My receive groups g = e·P + s from the dispatch words: sN[g] rows (0 for an overflowed group or a
// word of another form) and sAll[g], their exclusive prefix over g; `bad` when a word is of another
// form. Expert e's rows from source s start at row sAll[g] - sAll[e·P] of its packed segment.
__device__ __forceinline__ bool llGroups(const unsigned long long* words, uint32_t form, unsigned long long M, int K,
                                         uint32_t* sN, unsigned long long* sAll, unsigned long long* sWarp,
                                         unsigned long long& total) {
  const int t = threadIdx.x;
  uint32_t n = 0u;
  bool bad = false;
  if (t < K) {
    const unsigned long long w = ld_acquire_sys_u64(words + t);
    bad = llForm(w) != form;
    n = bad || static_cast<uint32_t>(w) > M ? 0u : static_cast<uint32_t>(w);
    sN[t] = n;
  }
  const unsigned long long first = blockExclusiveScan(n, sWarp, total);
  if (t < K) sAll[t] = first;
  return __syncthreads_or(bad) != 0;
}

// The last group starting at or before packed row q (an empty group starts where the next one does).
__device__ __forceinline__ int llGroupOf(const unsigned long long* sAll, int K, unsigned long long q) {
  int lo = 0, hi = K - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (sAll[mid] <= q) lo = mid; else hi = mid - 1;
  }
  return lo;
}
}  // namespace

unsigned long long moeLLSignal(uint32_t seq, uint32_t form, uint32_t count) { return llWord(seq, form, count); }

template <bool kQuant>
__global__ void __launch_bounds__(kThreads)
moeLLDispatchKernel(CommArgs a, MoeLLArgs L, const char* x, const long long* idx, unsigned long long tokens, char* out,
                    float* outScales, long long* outSplits) {
  __shared__ unsigned long long sSrc[kMaxK];  // group g = j·E + e: route()'s first row of g
  __shared__ uint32_t sTot[kMaxK];            //   routed choices of all my tokens
  __shared__ uint32_t sRun[kMaxK];            //   of the tokens before my slice, then running
  __shared__ uint32_t sN[kMaxK];              // my receive group e·P + s: rows
  __shared__ unsigned long long sAll[kMaxK];  //   their exclusive prefix
  __shared__ unsigned long long sWarp[32];
  const int P = a.nranks, E = L.l.experts, K = P * E, me = a.rank, t = threadIdx.x;
  const int lane = t & 31, warp = t >> 5, nw = blockDim.x >> 5;
  const unsigned long long rb = L.l.rowBytes, sb = L.l.scaleBytes, k = L.l.topk, M = L.l.maxTokens;
  char* mine = static_cast<char*>(L.bufs.p[me]);
  uint32_t* ctrl = reinterpret_cast<uint32_t*>(mine + L.l.ctrl);
  int* choices = reinterpret_cast<int*>(mine + L.l.choices);
  const unsigned long long* words = reinterpret_cast<const unsigned long long*>(mine + L.l.dispatchSig);
  const uint32_t seq = *reinterpret_cast<volatile uint32_t*>(ctrl) + 1u;
  const uint32_t form = kQuant ? kMoeLLDispatchFp8 : kMoeLLDispatch;

  // ---- 1. route: my slice's choices get their rank in their group, or -1 (not routed, overflow) ----
  const unsigned long long per = (tokens + gridDim.x - 1) / gridDim.x;
  const unsigned long long tok0 = min(tokens, blockIdx.x * per), tok1 = min(tokens, tok0 + per);
  topkRouteCount(idx, tokens * k, tok0 * k, K, sTot, sRun, sSrc, sWarp, [](int) {});
  topkRouteRank(idx, tok0 * k, tok1 * k, K, sSrc, sRun, [&](unsigned long long i, int g, long long p) {
    choices[i] = p >= 0 && sTot[g] <= M ? static_cast<int>(p - static_cast<long long>(sSrc[g])) : -1;
  });
  __syncthreads();

  // ---- 2. push: one warp per token of my slice, to slot (e, me, r) of rank j with its tag ----
  for (unsigned long long tok = tok0 + warp; tok < tok1; tok += nw) {
    char* dst = nullptr;
    float* dsc = nullptr;
    if (static_cast<unsigned long long>(lane) < k) {
      const unsigned long long i = tok * k + lane;
      const int r = choices[i];
      if (r >= 0) {
        const int g = topkGroup(idx[i], K), j = g / E, e = g % E;
        const unsigned long long slot = (static_cast<unsigned long long>(e) * P + me) * M + r;
        char* b = static_cast<char*>(L.bufs.p[j]);
        dst = b + L.l.slots + slot * rb;
        if constexpr (kQuant) dsc = reinterpret_cast<float*>(b + L.l.scales + slot * sb);
        reinterpret_cast<int*>(b + L.l.tags)[slot] = static_cast<int>(i);
      }
    }
    topkPushRow<kQuant>(x + tok * rb * (kQuant ? 2 : 1), rb, lane, static_cast<int>(k), dst, dsc);
  }

  // ---- 3. signal: word [e][me] on rank j ----
  bool ok = localGridSync(a);
  if (ok && blockIdx.x == 0 && t < K) {
    const int j = t / E, e = t % E;
    unsigned long long* w = reinterpret_cast<unsigned long long*>(static_cast<char*>(L.bufs.p[j]) + L.l.dispatchSig);
    st_release_sys_u64(w + e * P + me, llWord(seq, form, sTot[t]));
  }

  // ---- 4. receive my E·P words, pack ----
  if (ok) {
    bool gone = false;
    if (t < K) {
      unsigned long long w;
      gone = !llWait(a, words + t, seq, t % P, w);
    }
    ok = __syncthreads_or(gone) == 0;
  }
  if (ok) {
    unsigned long long total;
    const bool bad = llGroups(words, form, M, K, sN, sAll, sWarp, total);
    if (!bad) {
      const size_t gtid = static_cast<size_t>(blockIdx.x) * blockDim.x + t;
      const size_t gthreads = static_cast<size_t>(gridDim.x) * blockDim.x;
      for (int g = 0; g < K; g++) {
        const unsigned long long n = sN[g];
        if (n == 0) continue;
        const int e = g / P;
        const unsigned long long row = static_cast<unsigned long long>(e) * P * M + (sAll[g] - sAll[e * P]);
        gridCopy(out + row * rb, mine + L.l.slots + g * M * rb, n * rb, true, gtid, gthreads);
        if constexpr (kQuant) {
          gridCopy(reinterpret_cast<char*>(outScales) + row * sb, mine + L.l.scales + g * M * sb, n * sb, true, gtid,
                   gthreads);
        }
      }
      if (blockIdx.x == 0 && t < K) outSplits[t] = sN[t];
    }
    // An overflow is raised on its source and on its holder; the first error of a call wins.
    if (blockIdx.x == 0 && t == 0) {
      if (bad) llReport(L.status, kInputInvalid, 0u, 0u, 0ull, 0ull);
      for (int g = 0; g < K; g++) {
        if (sTot[g] > M) llReport(L.status, kInputSlotOverflow, me, g, sTot[g], M);
      }
      for (int g = 0; g < K && !bad; g++) {
        const uint32_t n = static_cast<uint32_t>(words[g]);
        if (n > M) llReport(L.status, kInputSlotOverflow, g % P, me * E + g / P, n, M);
      }
    }
  }
  llRetire(ctrl);
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
moeLLCombineKernel(CommArgs a, MoeLLArgs L, const char* expertOut, const float* weights, char* y,
                   unsigned long long tokens) {
  using PT = PackTraits<T>;
  __shared__ uint32_t sN[kMaxK];              // my receive group e·P + s: rows
  __shared__ unsigned long long sAll[kMaxK];  //   their exclusive prefix
  __shared__ unsigned long long sWarp[32];
  const int P = a.nranks, me = a.rank, t = threadIdx.x, lane = t & 31;
  const unsigned long long crb = L.l.combineRowBytes, k = L.l.topk, M = L.l.maxTokens;
  // Derived from the parameters where they are used: little stays live across the grid sync's call.
  auto mine = [&]() { return static_cast<char*>(L.bufs.p[me]); };
  uint32_t* ctrl = reinterpret_cast<uint32_t*>(mine() + L.l.ctrl);
  const uint32_t seq = *reinterpret_cast<volatile uint32_t*>(ctrl) + 1u;
  const size_t gwarp = (static_cast<size_t>(blockIdx.x) * blockDim.x + t) / 32;
  const size_t nwarps = static_cast<size_t>(gridDim.x) * blockDim.x / 32;

  // ---- 1. holder push: packed row q of my experts goes to its source's combine slot, by its tag ----
  {
    const int K = P * L.l.experts;
    const int* tags = reinterpret_cast<const int*>(mine() + L.l.tags);
    unsigned long long total;
    llGroups(reinterpret_cast<const unsigned long long*>(mine() + L.l.dispatchSig),
             L.l.fp8 ? kMoeLLDispatchFp8 : kMoeLLDispatch, M, K, sN, sAll, sWarp, total);
    for (unsigned long long q = gwarp; q < total; q += nwarps) {
      const int g = llGroupOf(sAll, K, q), e = g / P, s = g % P;
      const unsigned long long r = q - sAll[g];
      const long long tag = tags[g * M + r];
      if (tag < 0 || static_cast<unsigned long long>(tag) >= M * k) continue;
      const char* src = expertOut + (static_cast<unsigned long long>(e) * P * M + (sAll[g] - sAll[e * P]) + r) * crb;
      char* dst = static_cast<char*>(L.bufs.p[s]) + L.l.combineSlots + static_cast<unsigned long long>(tag) * crb;
      for (unsigned long long pk = lane; pk < crb / 16; pk += 32) st128(dst + pk * 16, ld128(src + pk * 16));
    }
  }

  // ---- 2. signal every source ----
  bool ok = localGridSync(a);
  const int* choices = reinterpret_cast<const int*>(mine() + L.l.choices);
  const unsigned long long* cwords = reinterpret_cast<const unsigned long long*>(mine() + L.l.combineSig);
  const unsigned long long npk = crb / 16;
  if (ok && blockIdx.x == 0 && t < P) {
    unsigned long long* w = reinterpret_cast<unsigned long long*>(static_cast<char*>(L.bufs.p[t]) + L.l.combineSig);
    st_release_sys_u64(w + me, llWord(seq, kMoeLLCombine, 0u));
  }

  // ---- 3. wait for every holder, then sum each token's sent choices ----
  bool bad = false;
  if (ok) {
    bool gone = false;
    if (t < P) {
      unsigned long long w;
      gone = !llWait(a, cwords + t, seq, t, w);
      bad = !gone && llForm(w) != kMoeLLCombine;
    }
    ok = __syncthreads_or(gone) == 0;
    bad = __syncthreads_or(bad) != 0;
  }
  if (ok && !bad) {
    for (unsigned long long tok = gwarp; tok < tokens; tok += nwarps) {
      // Lane c < k: choice c's row in my combine slots and its weight, when it was sent.
      const char* src = nullptr;
      float w = 0.0f;
      if (static_cast<unsigned long long>(lane) < k) {
        const unsigned long long i = tok * k + lane;
        if (choices[i] >= 0) {
          src = mine() + L.l.combineSlots + i * crb;
          w = weights != nullptr ? weights[i] : 1.0f;
        }
      }
      // Warp-uniform trip count: every lane takes part in the shuffles, lanes past the row end idle.
      for (unsigned long long pk = lane; pk - lane < npk; pk += 32) {
        typename PT::AccPack acc;
#pragma unroll
        for (int i = 0; i < PT::kElems; i++) acc.v[i] = 0.0f;
        for (int c = 0; c < static_cast<int>(k); c++) {
          const char* sc = reinterpret_cast<const char*>(__shfl_sync(0xffffffffu, reinterpret_cast<uintptr_t>(src), c));
          const float wc = __shfl_sync(0xffffffffu, w, c);
          if (sc != nullptr && pk < npk) topkAccumulate<T>(acc, wc, ld128(sc + pk * 16));
        }
        if (pk < npk) st128(y + tok * crb + pk * 16, PT::narrow(acc));
      }
    }
  }
  if (ok && bad && blockIdx.x == 0 && t == 0) llReport(L.status, kInputInvalid, 0u, 0u, 0ull, 0ull);
  llRetire(ctrl);
}

namespace {
using LLCombineFn = void (*)(CommArgs, MoeLLArgs, const char*, const float*, char*, unsigned long long);
LLCombineFn llCombineFn(DataType dt) {
  switch (dt) {
    case DataType::FLOAT32: return moeLLCombineKernel<float>;
    case DataType::BFLOAT16: return moeLLCombineKernel<__nv_bfloat16>;
    case DataType::FLOAT16: return moeLLCombineKernel<__half>;
    default: return nullptr;
  }
}
}  // namespace

void launchMoeLLDispatch(const CommArgs& a, const MoeLLArgs& L, const void* x, size_t tokens, const long long* idx,
                         void* out, float* outScales, long long* outSplits, int blocks, cudaStream_t stream) {
  const char* xc = static_cast<const char*>(x);
  char* o = static_cast<char*>(out);
  if (L.l.fp8) {
    moeLLDispatchKernel<true><<<blocks, kThreads, 0, stream>>>(a, L, xc, idx, tokens, o, outScales, outSplits);
  } else {
    moeLLDispatchKernel<false><<<blocks, kThreads, 0, stream>>>(a, L, xc, idx, tokens, o, outScales, outSplits);
  }
}

void launchMoeLLCombine(const CommArgs& a, const MoeLLArgs& L, const void* expertOut, const float* weights, void* y,
                        size_t tokens, DataType dt, int blocks, cudaStream_t stream) {
  llCombineFn(dt)<<<blocks, kThreads, 0, stream>>>(a, L, static_cast<const char*>(expertOut), weights,
                                                   static_cast<char*>(y), tokens);
}

const void* moeLLDispatchKernelPtr(bool fp8) {
  return fp8 ? reinterpret_cast<const void*>(moeLLDispatchKernel<true>)
             : reinterpret_cast<const void*>(moeLLDispatchKernel<false>);
}
const void* moeLLCombineKernelPtr(DataType dt) { return reinterpret_cast<const void*>(llCombineFn(dt)); }

const void* alltoallvDevKernelPtr(bool fp8) {
  return fp8 ? reinterpret_cast<const void*>(alltoallvDevKernel<true>)
             : reinterpret_cast<const void*>(alltoallvDevKernel<false>);
}
const void* moeCombineTopkKernelPtr(DataType dt) { return reinterpret_cast<const void*>(topkCombineFn(dt)); }
const void* moeCombineTopkBackwardKernelPtr(DataType dt) {
  return reinterpret_cast<const void*>(topkCombineBackwardFn(dt));
}
const void* moeDispatchTopkKernelPtr(bool fp8) {
  return fp8 ? reinterpret_cast<const void*>(moeDispatchTopkKernel<true>)
             : reinterpret_cast<const void*>(moeDispatchTopkKernel<false>);
}

void preloadMoeKernels() {
  touchKernel(alltoallvDevKernel<false>);
  touchKernel(alltoallvDevKernel<true>);
  for (DataType dt : {DataType::FLOAT32, DataType::BFLOAT16, DataType::FLOAT16}) {
    touchKernel(topkCombineFn(dt));
    touchKernel(topkCombineBackwardFn(dt));
    touchKernel(llCombineFn(dt));
  }
  touchKernel(moeDispatchTopkKernel<false>);
  touchKernel(moeDispatchTopkKernel<true>);
  touchKernel(moeLLDispatchKernel<false>);
  touchKernel(moeLLDispatchKernel<true>);
  cudaGetLastError();
}

}  // namespace cuda
}  // namespace glb
