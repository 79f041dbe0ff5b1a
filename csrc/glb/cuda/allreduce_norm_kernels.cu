// Tensor-parallel allreduce fused with bias, residual add and RMSNorm / LayerNorm (sm_90a).
//
// For every row i of a (rows, H) problem, with p_r the partial sums of rank r:
//
//   s_i             = sum_r p_r[i] (+ bias) + residual[i]    fp32, rounded once -> residualOut[i]
//   x_i             = residualOut[i] as fp32
//   out[i] (rms)    = x_i * 1 / sqrt(mean(x_i^2) + eps) * gamma
//   out[i] (layer)  = (x_i - mean(x_i)) * 1 / sqrt(var(x_i) + eps) * gamma + beta
//
// A CTA owns whole rows (grid-stride loop over rows); row i always belongs to CTA i % gridDim.x,
// on every rank, so the barrier pairing of CTA b across ranks pairs the CTAs that touch the same
// rows. Thread t holds 16-byte packs t, t + kThreads, ... of its row in registers (at most
// NormRow<T>::kPacks of them at H = kMaxNormHidden), so a row is read once and the statistics come from a
// block reduction over registers. Every sum has a fixed order (partials in rank order, then bias,
// then residual; the block reduction by thread and warp index), and the same code runs on every
// rank, so ranks that reduce the same row write the same bytes.
//
//   LL        flag-in-data lines of the partial into every peer's LL region (the protocol of
//             llAllreduceKernel); every rank reduces every row. No barrier.
//   ONE_SHOT  each rank stages its partial in its pool half (launch parity), one barrier, then
//             every rank reads the P staged copies of each row and runs the epilogue itself.
//   TWO_SHOT  stage in the pool's bulk region, barrier, rank r reduces the rows of its share and
//             stores both result rows into every peer's pool (residualOut over the staged partial,
//             which only the row's owner reads; out after the partials), barrier, every rank
//             copies its pool rows out to its own residualOut / out.
//   LOCAL     one rank: the epilogue on the partial, no exchange.
//   SCATTER   the reduce-scatter form (sequence parallelism): residual / residualOut / an
//             ungathered out are this rank's shard of the rows. Stage every shard's chunk in the
//             bulk region, barrier, rank r reduces the rows of shard r and writes residualOut
//             (and an ungathered out) straight to its own tensors; with `gather` it stores out
//             into every peer's pool, barrier, and every rank copies all P shards of out.
//
// The quantising form (Q, with a norm): out is e4m3 codes (rows, H) and n.outScales one fp32 scale
// per row. The epilogue rounds each out value to T (the bytes the unquantised form writes), takes
// the row's amax with one more block reduction and stores quantAmax / e4m3Multiplier codes and the
// e4m3Scale (device_common.cuh) from the registers. What the two-shot and the gathered scatter
// exchange is then H code bytes and one scale per row instead of an H-element row of T.
#include "glb/cuda/device_common.cuh"
#include "glb/cuda/kernels.h"

namespace glb {
namespace cuda {

namespace {

template <typename T>
struct NormRow {
  using PT = PackTraits<T>;
  static constexpr int kE = PT::kElems;  // elements per 16-byte pack
  static constexpr int kPacks = kMaxNormHidden * static_cast<int>(sizeof(T)) / 16 / kThreads;
  using Acc = typename PT::AccPack;
};

// Sum of v over the CTA, the same value on every thread; fixed order (warp butterfly, then the
// warps' sums in warp order). Starts with a barrier so that back-to-back calls can reuse `sh`.
__device__ __forceinline__ float blockSum(float v, float* sh) {
#pragma unroll
  for (int d = 16; d >= 1; d /= 2) v += __shfl_xor_sync(0xffffffffu, v, d);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.0f;
#pragma unroll
  for (int w = 0; w < kThreads / 32; w++) s += sh[w];
  return s;
}

// gridDim.x read again where used (a volatile read of %nctaid.x) rather than held across the row
// loop, where it would spill at the widest rows (fp32 LayerNorm).
__device__ __forceinline__ unsigned gridCtas() {
  unsigned n;
  asm volatile("mov.u32 %0, %%nctaid.x;" : "=r"(n));
  return n;
}

// Max of v over the CTA, the same value on every thread; blockSum's order.
__device__ __forceinline__ float blockMax(float v, float* sh) {
#pragma unroll
  for (int d = 16; d >= 1; d /= 2) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, d));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float m = 0.0f;
#pragma unroll
  for (int w = 0; w < kThreads / 32; w++) m = fmaxf(m, sh[w]);
  return m;
}

// The e4m3 codes of one pack of T (kE elements, kE bytes: a uint32_t for float, a uint2 for the
// 16-bit types), and their store at `p`.
template <typename T>
using QCodes = typename std::conditional<NormRow<T>::kE == 8, uint2, uint32_t>::type;
__device__ __forceinline__ void stCodes(char* p, uint32_t c) { *reinterpret_cast<uint32_t*>(p) = c; }
__device__ __forceinline__ void stCodes(char* p, uint2 c) { *reinterpret_cast<uint2*>(p) = c; }

template <typename T>
__device__ __forceinline__ QCodes<T> packCodes(const typename NormRow<T>::Acc& x, float multiplier) {
  uint32_t w[NormRow<T>::kE / 4];
#pragma unroll
  for (int i = 0; i < NormRow<T>::kE / 4; i++) {
    w[i] = e4m3Codes2(x.v[4 * i], x.v[4 * i + 1], multiplier) |
           (e4m3Codes2(x.v[4 * i + 2], x.v[4 * i + 3], multiplier) << 16);
  }
  if constexpr (NormRow<T>::kE == 8) {
    return make_uint2(w[0], w[1]);
  } else {
    return w[0];
  }
}

__device__ __forceinline__ const char* rowPtr(const void* base, size_t row, size_t rowBytes) {
  return static_cast<const char*>(base) + row * rowBytes;
}

// The norm's statistics of a row whose rounded values are x (pack k of this thread at x[k]), in
// one fixed order: the forward epilogue and the backward both compute them so, and the backward
// sees the forward's statistics bit for bit. statAdd folds one pack (the packs in k order) into
// this thread's sum; rowStats finishes from it: mean (0 for rms) and rinv = 1 / sqrt(var + eps)
// (layer) or 1 / sqrt(mean(x^2) + eps) (rms).
template <typename T, int NORM>
__device__ __forceinline__ void statAdd(float& sum, const typename NormRow<T>::Acc& x) {
#pragma unroll
  for (int e = 0; e < NormRow<T>::kE; e++) {
    if constexpr (NORM == kNormLayer) {
      sum += x.v[e];
    } else if constexpr (NORM == kNormRms) {
      sum = fmaf(x.v[e], x.v[e], sum);
    }
  }
}

template <typename T, int NORM>
__device__ __forceinline__ void rowStats(const typename NormRow<T>::Acc (&x)[NormRow<T>::kPacks], float sum, int npacks,
                                         float eps, float* sh, float& mean, float& rinv) {
  using R = NormRow<T>;
  const int t = threadIdx.x;
  const float hidden = static_cast<float>(npacks * R::kE);
  mean = 0.0f;
  if constexpr (NORM == kNormLayer) {
    mean = blockSum(sum, sh) / hidden;
    float sq = 0.0f;
#pragma unroll
    for (int k = 0; k < R::kPacks; k++) {
      if (t + k * kThreads < npacks) {
#pragma unroll
        for (int e = 0; e < R::kE; e++) {
          const float d = x[k].v[e] - mean;
          sq = fmaf(d, d, sq);
        }
      }
    }
    rinv = 1.0f / sqrtf(blockSum(sq, sh) / hidden + eps);
  } else {
    rinv = 1.0f / sqrtf(blockSum(sum, sh) / hidden + eps);
  }
}

// The row epilogue on the reduced partials `acc` of row `row`: adds bias and residual, rounds
// once, and hands each pack of residualOut and out to store(k, resid, out). `npacks` packs per
// row; pack k of this thread is t + k * kThreads. Q (with a norm): store's out is to be dropped;
// the row's codes go to storeQ(pk, codes, scale) once its amax is known, pack by pack, and the
// thread that has pack 0 stores the scale.
template <typename T, int NORM, bool Q, typename Store, typename StoreQ>
__device__ __forceinline__ void rowEpilogue(typename NormRow<T>::Acc (&acc)[NormRow<T>::kPacks], const NormArgs& n,
                                            size_t row, int npacks, float* sh, Store&& store, StoreQ&& storeQ) {
  using R = NormRow<T>;
  using PT = typename R::PT;
  const int t = threadIdx.x;
  const size_t rb = static_cast<size_t>(npacks) * 16;
  float sum = 0.0f;
#pragma unroll
  for (int k = 0; k < R::kPacks; k++) {
    const int pk = t + k * kThreads;
    if (pk < npacks) {
      if (n.bias != nullptr) PT::combine(acc[k], ld128(static_cast<const char*>(n.bias) + pk * 16), DevOp::SUM);
      PT::combine(acc[k], ld128_stream(rowPtr(n.residual, row, rb) + pk * 16), DevOp::SUM);
      const Pack16 r = PT::narrow(acc[k]);
      if constexpr (NORM == kNormNone) store(pk, r, r);
      acc[k] = PT::widen(r);  // the rounded value: what the next layer sees
      statAdd<T, NORM>(sum, acc[k]);
    }
  }
  if constexpr (NORM != kNormNone) {
    float mean, rinv, absMax = 0.0f;
    rowStats<T, NORM>(acc, sum, npacks, n.eps, sh, mean, rinv);
#pragma unroll
    for (int k = 0; k < R::kPacks; k++) {
      const int pk = t + k * kThreads;
      if (pk < npacks) {
        const Pack16 r = PT::narrow(acc[k]);  // exact: acc holds rounded values
        typename R::Acc g, b;
        if (n.gamma != nullptr) g = PT::widen(ld128(static_cast<const char*>(n.gamma) + pk * 16));
        if (NORM == kNormLayer && n.beta != nullptr) b = PT::widen(ld128(static_cast<const char*>(n.beta) + pk * 16));
#pragma unroll
        for (int e = 0; e < R::kE; e++) {
          float y = (acc[k].v[e] - mean) * rinv;
          if (n.gamma != nullptr) y *= g.v[e];
          if (NORM == kNormLayer && n.beta != nullptr) y += b.v[e];
          acc[k].v[e] = y;
        }
        if constexpr (Q) {
          const Pack16 o = PT::narrow(acc[k]);
          store(pk, r, o);
          acc[k] = PT::widen(o);  // out as the unquantised form writes it
#pragma unroll
          for (int e = 0; e < R::kE; e++) absMax = fmaxf(absMax, fabsf(acc[k].v[e]));
        } else {
          store(pk, r, PT::narrow(acc[k]));
        }
      }
    }
    if constexpr (Q) {
      const float amax = quantAmax(blockMax(absMax, sh));
      const float mul = e4m3Multiplier(amax), scale = e4m3Scale(amax);
#pragma unroll
      for (int k = 0; k < R::kPacks; k++) {
        const int pk = t + k * kThreads;
        if (pk < npacks) storeQ(pk, packCodes<T>(acc[k], mul), scale);
      }
    }
  }
}

template <typename T>
__device__ __forceinline__ void zeroAcc(typename NormRow<T>::Acc (&acc)[NormRow<T>::kPacks]) {
#pragma unroll
  for (int k = 0; k < NormRow<T>::kPacks; k++) {
#pragma unroll
    for (int e = 0; e < NormRow<T>::kE; e++) acc[k].v[e] = 0.0f;
  }
}

// Adds the packs of one staged row (a copy of some rank's partial) to acc.
template <typename T>
__device__ __forceinline__ void addRow(typename NormRow<T>::Acc (&acc)[NormRow<T>::kPacks], const char* row,
                                       int npacks) {
#pragma unroll
  for (int k = 0; k < NormRow<T>::kPacks; k++) {
    const int pk = threadIdx.x + k * kThreads;
    if (pk < npacks) PackTraits<T>::combine(acc[k], ld128_stream(row + pk * 16), DevOp::SUM);
  }
}

template <typename T>
__device__ __forceinline__ void copyRow(char* dst, const char* src, int npacks) {
  for (int pk = threadIdx.x; pk < npacks; pk += kThreads) st128(dst + pk * 16, ld128(src + pk * 16));
}

// Row i of the problem is handled by CTA i % gridDim.x of every rank. Q: the quantising form.
template <typename T, int NORM, int V, bool Q>
__global__ void __launch_bounds__(kThreads, 1)
allreduceNormKernel(CommArgs a, NormArgs n, NormXchg x) {
  using R = NormRow<T>;
  __shared__ float sh[kThreads / 32];
  // The peers' pointers, indexed by a run-time rank: from shared memory rather than the
  // parameter space (a dynamic parameter index copies the struct to local memory) or a register
  // per rank (which spills at the widest rows).
  __shared__ char* peers[kMaxRanks];
  if (threadIdx.x < kMaxRanks) peers[threadIdx.x] = static_cast<char*>(x.peers.p[threadIdx.x]);
  __syncthreads();
  const int P = a.nranks;
  const int me = a.rank;
  const int npacks = static_cast<int>(n.hidden * sizeof(T) / 16);
  const size_t rb = static_cast<size_t>(npacks) * 16;
  // Q: a row of codes is hidden bytes; the pools hold a region of code rows, then its scales.
  const size_t qb = n.hidden;
  auto toUser = [&](size_t row) {
    return [&, row](int pk, const Pack16& r, const Pack16& o) {
      st128(static_cast<char*>(n.residualOut) + row * rb + pk * 16, r);
      if (NORM != kNormNone && !Q) st128(static_cast<char*>(n.out) + row * rb + pk * 16, o);
    };
  };
  auto toUserQ = [&](size_t row) {
    return [&, row](int pk, const QCodes<T>& c, float scale) {
      stCodes(static_cast<char*>(n.out) + row * qb + pk * R::kE, c);
      if (pk == 0) n.outScales[row] = scale;
    };
  };
  typename R::Acc acc[R::kPacks];

  if constexpr (V == kNormLocal) {
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
      zeroAcc<T>(acc);
      addRow<T>(acc, rowPtr(n.partial, i, rb), npacks);
      rowEpilogue<T, NORM, Q>(acc, n, i, npacks, sh, toUser(i), toUserQ(i));
    }
  } else if constexpr (V == kNormLL) {
    // x.peers.p[r]: rank r's LL region; lines [parity][source][unit], two 8-byte units per pack.
    const uint32_t seq = ld_relaxed_sys(&a.self->llSeq) + 1u;
    const size_t base = (seq & 1u) * x.parityStride;
    const char* myRegion = static_cast<const char*>(x.mine) + base;
    const size_t mySlot = base + static_cast<size_t>(me) * x.srcStride;
    bool alive = true;
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
#pragma unroll
      for (int k = 0; k < R::kPacks; k++) {
        const int pk = threadIdx.x + k * kThreads;
        if (pk < npacks) {
          const Pack16 own = ld128(rowPtr(n.partial, i, rb) + pk * 16);
          const size_t line = (i * npacks + pk) * 32;
          for (int r = 0; r < P; r++) {
            if (r != me) {
              char* dst = peers[r] + mySlot + line;
              llStore(dst, own.w[0], own.w[1], seq);
              llStore(dst + 16, own.w[2], own.w[3], seq);
            }
          }
        }
      }
      zeroAcc<T>(acc);
#pragma unroll
      for (int k = 0; k < R::kPacks; k++) {
        const int pk = threadIdx.x + k * kThreads;
        if (pk < npacks) {
          const size_t line = (i * npacks + pk) * 32;
          for (int r = 0; r < P && alive; r++) {
            Pack16 p;
            if (r == me) {
              p = ld128(rowPtr(n.partial, i, rb) + pk * 16);  // mine, read again: cached, saves registers
            } else {
              const char* src = myRegion + static_cast<size_t>(r) * x.srcStride + line;
              alive = llLoad(a, src, seq, p.w[0], p.w[1], r) && llLoad(a, src + 16, seq, p.w[2], p.w[3], r);
            }
            if (alive) PackTraits<T>::combine(acc[k], p, DevOp::SUM);
          }
        }
      }
      // A timed-out poll ends the row loop on the whole CTA before the block reductions.
      alive = __syncthreads_and(alive) != 0;
      if (!alive) break;
      rowEpilogue<T, NORM, Q>(acc, n, i, npacks, sh, toUser(i), toUserQ(i));
    }
    retire(a, 0, 0, 1);
  } else if constexpr (V == kNormOneShot) {
    const uint32_t e = loadEpoch(a);
    const size_t off = (ld_relaxed_sys(&a.self->stageSeq) & 1u) * x.parityStride;
    char* myStage = static_cast<char*>(x.mine) + off;
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) copyRow<T>(myStage + i * rb, rowPtr(n.partial, i, rb), npacks);
    if (!blockBarrier(a, e + 1)) {
      retire(a, 1, 1);
      return;
    }
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
      zeroAcc<T>(acc);
      for (int r = 0; r < P; r++) addRow<T>(acc, peers[r] + off + i * rb, npacks);
      rowEpilogue<T, NORM, Q>(acc, n, i, npacks, sh, toUser(i), toUserQ(i));
    }
    retire(a, 1, 1);
  } else if constexpr (V == kNormTwoShot) {
    // Pool rows: [0, rows) the staged partials, overwritten with residualOut by the row's owner;
    // [rows, 2 rows) out, or with Q rows code rows of qb bytes and then rows fp32 scales.
    const uint32_t e = loadEpoch(a);
    char* mine = static_cast<char*>(x.mine);
    // Q: each peer's code rows and scales, from shared memory like `peers`: held in registers across
    // the row loop, their offsets spill at 16-bit LayerNorm. So do the grid size and the epoch,
    // which Q reads again where it uses them (the epoch only changes when the launch's last CTA
    // retires).
    __shared__ char* qPeers[Q ? kMaxRanks : 1];
    __shared__ float* sPeers[Q ? kMaxRanks : 1];
    if (Q && threadIdx.x < kMaxRanks) {
      qPeers[threadIdx.x] = peers[threadIdx.x] + n.rows * rb;
      sPeers[threadIdx.x] = reinterpret_cast<float*>(peers[threadIdx.x] + n.rows * (rb + qb));
    }
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) copyRow<T>(mine + i * rb, rowPtr(n.partial, i, rb), npacks);
    if (!blockBarrier(a, e + 1)) {
      retire(a, 2, 0);
      return;
    }
    size_t sb, se;
    {
      const size_t q = n.rows / P, rem = n.rows % P;
      sb = me * q + (static_cast<size_t>(me) < rem ? me : rem);
      se = sb + q + (static_cast<size_t>(me) < rem ? 1 : 0);
    }
    const size_t first = sb + (blockIdx.x + gridDim.x - sb % gridDim.x) % gridDim.x;
    for (size_t i = first; i < se; i += (Q ? gridCtas() : gridDim.x)) {
      zeroAcc<T>(acc);
      for (int r = 0; r < P; r++) addRow<T>(acc, peers[r] + i * rb, npacks);
      rowEpilogue<T, NORM, Q>(
          acc, n, i, npacks, sh,
          [&](int pk, const Pack16& rr, const Pack16& o) {
            for (int r = 0; r < P; r++) {
              st128_stream(peers[r] + i * rb + pk * 16, rr);
              if (NORM != kNormNone && !Q) st128_stream(peers[r] + (n.rows + i) * rb + pk * 16, o);
            }
          },
          [&](int pk, const QCodes<T>& c, float scale) {
            for (int r = 0; r < P; r++) {
              stCodes(qPeers[r] + i * qb + pk * R::kE, c);
              if (pk == 0) sPeers[r][i] = scale;
            }
          });
    }
    if (blockBarrier(a, (Q ? loadEpoch(a) : e) + 2)) {
      for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
        copyRow<T>(static_cast<char*>(n.residualOut) + i * rb, mine + i * rb, npacks);
        if constexpr (Q) {
          copyRow<T>(static_cast<char*>(n.out) + i * qb, qPeers[me] + i * qb, static_cast<int>(qb / 16));
          if (threadIdx.x == 0) n.outScales[i] = sPeers[me][i];
        } else if (NORM != kNormNone) {
          copyRow<T>(static_cast<char*>(n.out) + i * rb, mine + (n.rows + i) * rb, npacks);
        }
      }
    }
    retire(a, 2, 0);
  } else {
    // n.rows rows of every shard. Pool rows: [0, P rows) the staged partials, row q * rows + i =
    // the user's partial row q * shardRows + i; with a gathered out, [P rows, 2 P rows) out in the
    // same order (Q: P rows code rows of qb bytes, then P rows fp32 scales). Rank me owns pool rows
    // [me * rows, (me + 1) * rows), shard row i = j - me * rows.
    // Two barriers either way: with a gathered out the second orders the out stores before the
    // copy out; without one it is a closing barrier, so that no rank restages its pool (in its
    // next launch) while a peer may still be reading the rows it staged.
    const uint32_t e = loadEpoch(a);
    char* mine = static_cast<char*>(x.mine);
    const size_t rows = n.rows, all = static_cast<size_t>(P) * rows;
    const bool gather = NORM != kNormNone && x.gather != 0;
    auto userRow = [&](size_t j) { return j / rows * x.shardRows + j % rows; };
    for (size_t j = blockIdx.x; j < all; j += gridDim.x) copyRow<T>(mine + j * rb, rowPtr(n.partial, userRow(j), rb), npacks);
    if (!blockBarrier(a, e + 1)) {
      retire(a, 2, 0);
      return;
    }
    const size_t sb = me * rows, se = sb + rows;
    const size_t first = sb + (blockIdx.x + gridDim.x - sb % gridDim.x) % gridDim.x;
    for (size_t j = first; j < se; j += gridDim.x) {
      const size_t i = j - sb;
      zeroAcc<T>(acc);
      for (int r = 0; r < P; r++) addRow<T>(acc, peers[r] + j * rb, npacks);
      rowEpilogue<T, NORM, Q>(
          acc, n, i, npacks, sh,
          [&](int pk, const Pack16& rr, const Pack16& o) {
            st128(static_cast<char*>(n.residualOut) + i * rb + pk * 16, rr);
            if (NORM == kNormNone || Q) return;
            if (gather) {
              for (int r = 0; r < P; r++) st128_stream(peers[r] + (all + j) * rb + pk * 16, o);
            } else {
              st128(static_cast<char*>(n.out) + i * rb + pk * 16, o);
            }
          },
          [&](int pk, const QCodes<T>& c, float scale) {
            if (gather) {
              for (int r = 0; r < P; r++) {
                char* q = peers[r] + all * rb;
                stCodes(q + j * qb + pk * R::kE, c);
                if (pk == 0) reinterpret_cast<float*>(q + all * qb)[j] = scale;
              }
            } else {
              stCodes(static_cast<char*>(n.out) + i * qb + pk * R::kE, c);
              if (pk == 0) n.outScales[i] = scale;
            }
          });
    }
    if (blockBarrier(a, (Q ? loadEpoch(a) : e) + 2) && gather) {  // Q: the epoch as in the two-shot
      for (size_t j = blockIdx.x; j < all; j += gridDim.x) {
        if constexpr (Q) {
          const char* q = mine + all * rb;
          copyRow<T>(static_cast<char*>(n.out) + userRow(j) * qb, q + j * qb, static_cast<int>(qb / 16));
          if (threadIdx.x == 0) n.outScales[userRow(j)] = reinterpret_cast<const float*>(q + all * qb)[j];
        } else {
          copyRow<T>(static_cast<char*>(n.out) + userRow(j) * rb, mine + (all + j) * rb, npacks);
        }
      }
    }
    retire(a, 2, 0);
  }
}

// ---- backward of the reduce-scatter form -----------------------------------------------------
// Per row, in fp32, with g the row's gradient of out and s the saved residual_out row:
//   mean, rinv from s (rowStats: the forward's statistics bit for bit), xh = (s - mean) rinv,
//   gg = g gamma, dx = rinv (gg - mean(gg) - xh mean(gg xh))   (rms: no mean(gg) term),
//   gradResidual = round(gradS + dx);  column sums: g xh (weight), g (norm bias), the rounded
//   gradResidual (bias).

// The CTA's column sums in dynamic shared memory, one fixed region of kMaxNormHidden floats per
// kind (0 weight, 1 norm bias, 2 bias): slot (k, e) of thread t at ((kind * kPacks + k) * kE + e)
// * kThreads + t. Thread t holds the same packs of every row, so only it touches its slots: no
// synchronisation, no bank conflicts, and every address is a constant offset. At this kernel's
// registers a CTA fills an SM's register file, so the fixed size costs no occupancy.
template <typename T>
__device__ __forceinline__ float& colSum(float* sums, int kind, int k, int e) {
  using R = NormRow<T>;
  return sums[((kind * R::kPacks + k) * R::kE + e) * kThreads + threadIdx.x];
}

// Moves this thread's column sums between shared memory and the CTA's vectors in ws: in before
// the rows (zero in the first chunk), out after them.
template <typename T>
__device__ __forceinline__ void moveSums(const NormBwdArgs& n, float* sums, int npacks, bool in) {
  using R = NormRow<T>;
  // The base through a volatile move: the two calls (before and after the row loop) each compute
  // the address rather than share one held across the loop, where it would spill.
  float* ws = n.ws;
  asm volatile("mov.b64 %0, %0;" : "+l"(ws));
  ws += static_cast<size_t>(blockIdx.x) * n.vectors * n.hidden;
  const int vec[3] = {n.vecWeight, n.vecNormBias, n.vecBias};
#pragma unroll
  for (int kind = 0; kind < 3; kind++) {
    if (vec[kind] < 0) continue;
#pragma unroll
    for (int k = 0; k < R::kPacks; k++) {
      const int pk = threadIdx.x + k * kThreads;
      if (pk >= npacks) continue;
#pragma unroll
      for (int e = 0; e < R::kE; e += 4) {
        float4* p = reinterpret_cast<float4*>(ws + vec[kind] * n.hidden + pk * R::kE + e);
        if (in) {
          const float4 v = n.first ? make_float4(0.0f, 0.0f, 0.0f, 0.0f) : *p;
          colSum<T>(sums, kind, k, e) = v.x;
          colSum<T>(sums, kind, k, e + 1) = v.y;
          colSum<T>(sums, kind, k, e + 2) = v.z;
          colSum<T>(sums, kind, k, e + 3) = v.w;
        } else {
          *p = make_float4(colSum<T>(sums, kind, k, e), colSum<T>(sums, kind, k, e + 1), colSum<T>(sums, kind, k, e + 2),
                           colSum<T>(sums, kind, k, e + 3));
        }
      }
    }
  }
}

// The address p, opaque to the optimiser: per-pack pointers of a row then stay immediate offsets
// of one base instead of becoming loop-carried 64-bit pointers, one per pack, which spill at the
// widest rows.
template <typename P>
__device__ __forceinline__ P* opaque(P* p) {
  asm("mov.b64 %0, %0;" : "+l"(p));
  return p;
}

// Row i of the shard: loadG(g) puts the row's fp32 gradient of out in g (pack k of this thread
// at g[k]) once the statistics are known. Hands each pack of gradResidual to store(pk, pack) and
// adds this thread's columns to the CTA's sums. Only g stays in registers across the block
// reductions; the s row is read again where xh is needed (from L1 / L2), which keeps the widest
// rows free of spills.
template <typename T, int NORM, typename LoadG, typename Store>
__device__ __forceinline__ void rowBackward(const NormBwdArgs& n, size_t i, int npacks, float* sh,
                                            float* sums, LoadG&& loadG, Store&& store) {
  using R = NormRow<T>;
  using PT = typename R::PT;
  const int t = threadIdx.x;
  const size_t rb = static_cast<size_t>(npacks) * 16;
  const char* s = opaque(rowPtr(n.s, i, rb));
  const char* gs = n.gradS != nullptr ? opaque(rowPtr(n.gradS, i, rb)) : nullptr;
  const char* gamma = n.gamma != nullptr ? opaque(static_cast<const char*>(n.gamma)) : nullptr;
  float mean, rinv;
  {
    typename R::Acc x[R::kPacks];
    float sum = 0.0f;
#pragma unroll
    for (int k = 0; k < R::kPacks; k++) {
      const int pk = t + k * kThreads;
      if (pk < npacks) {
        x[k] = PT::widen(ld128(s + pk * 16));
        statAdd<T, NORM>(sum, x[k]);
      }
    }
    rowStats<T, NORM>(x, sum, npacks, n.eps, sh, mean, rinv);
  }
  typename R::Acc g[R::kPacks];
  loadG(g);
  float sgg = 0.0f, sggx = 0.0f;
#pragma unroll
  for (int k = 0; k < R::kPacks; k++) {
    const int pk = t + k * kThreads;
    if (pk < npacks) {
      const typename R::Acc x = PT::widen(ld128(s + pk * 16));
      typename R::Acc w;
      if (gamma != nullptr) w = PT::widen(ld128(gamma + pk * 16));
#pragma unroll
      for (int e = 0; e < R::kE; e++) {
        const float xh = (x.v[e] - mean) * rinv;
        if (n.vecWeight >= 0) colSum<T>(sums, 0, k, e) += g[k].v[e] * xh;
        if (n.vecNormBias >= 0) colSum<T>(sums, 1, k, e) += g[k].v[e];
        if (gamma != nullptr) g[k].v[e] *= w.v[e];
        sgg += g[k].v[e];
        sggx = fmaf(g[k].v[e], xh, sggx);
      }
    }
  }
  const float hidden = static_cast<float>(npacks * R::kE);
  const float mggx = blockSum(sggx, sh) / hidden;
  float mgg = 0.0f;
  if constexpr (NORM == kNormLayer) mgg = blockSum(sgg, sh) / hidden;
#pragma unroll
  for (int k = 0; k < R::kPacks; k++) {
    const int pk = t + k * kThreads;
    if (pk < npacks) {
      const typename R::Acc x = PT::widen(ld128(s + pk * 16));
      typename R::Acc r;
      if (gs != nullptr) {
        r = PT::widen(ld128(gs + pk * 16));
      } else {
#pragma unroll
        for (int e = 0; e < R::kE; e++) r.v[e] = 0.0f;
      }
#pragma unroll
      for (int e = 0; e < R::kE; e++) {
        const float xh = (x.v[e] - mean) * rinv;
        const float dx = NORM == kNormLayer ? rinv * (g[k].v[e] - mgg - xh * mggx) : rinv * (g[k].v[e] - xh * mggx);
        r.v[e] += dx;
      }
      const Pack16 o = PT::narrow(r);
      if (n.vecBias >= 0) {
        const typename R::Acc ro = PT::widen(o);
#pragma unroll
        for (int e = 0; e < R::kE; e++) colSum<T>(sums, 2, k, e) += ro.v[e];
      }
      store(pk, o);
    }
  }
}

// The backward, V = kNormScatter (P ranks) or kNormLocal (one rank). Scatter: with a gathered out,
// stage every shard's chunk of gradOut in the bulk region (pool rows [0, P rows), in the forward's
// order); barrier; the owner of each row reduces its P staged rows (in rank order, fp32, not
// rounded), runs rowBackward and stores gradResidual into every peer's pool (rows [P rows,
// 2 P rows), or [0, P rows) without a gather); barrier; every rank copies all P shards out to
// gradPartial. Row j of the pool belongs to CTA j % gridDim.x in every phase, so each barrier
// pairs the CTAs that touch the same rows. Without a gather nothing is staged, and the first
// barrier only keeps the owners' stores out of a peer's pool until that peer has finished the
// launch before, which may still be reading it.
//
// The allreduce forms (tensor parallelism): every rank holds all rows of s and gradS, gradOut is
// its partial of out's gradient, and gradPartial = round(gradS + dx) gets every row.
//   ONE_SHOT  stage gradOut in the pool half of this launch's parity, barrier, every rank sums the
//             P staged copies of every row in rank order and runs rowBackward on all of them, so
//             its column sums cover every row.
//   TWO_SHOT  stage gradOut in the bulk region, barrier, the owner of each row (the forward
//             two-shot's row split) sums the P staged rows in rank order, runs rowBackward and
//             stores gradPartial into every peer's pool over the staged row (which only the owner
//             reads), barrier, every rank copies all rows out. The column sums cover this rank's
//             rows: normBackwardFinishAllreduceKernel completes them.
template <typename T, int NORM, int V>
__global__ void __launch_bounds__(kThreads, 1)
normBackwardKernel(CommArgs a, NormBwdArgs n, NormXchg x) {
  using R = NormRow<T>;
  extern __shared__ float colSums[];
  __shared__ float sh[kThreads / 32];
  __shared__ char* peers[kMaxRanks];
  if (threadIdx.x < kMaxRanks) {
    char* p = static_cast<char*>(x.peers.p[threadIdx.x]);
    // One-shot: the pool half of this launch, folded into the peers' pointers once.
    if constexpr (V == kNormOneShot) p += (ld_relaxed_sys(&a.self->stageSeq) & 1u) * x.parityStride;
    peers[threadIdx.x] = p;
  }
  const int npacks = static_cast<int>(n.hidden * sizeof(T) / 16);
  const size_t rb = static_cast<size_t>(npacks) * 16;
  moveSums<T>(n, colSums, npacks, true);
  __syncthreads();

  if constexpr (V == kNormLocal) {
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
      auto loadG = [&](typename R::Acc(&g)[R::kPacks]) {
        zeroAcc<T>(g);
        addRow<T>(g, rowPtr(n.gradOut, i, rb), npacks);
      };
      rowBackward<T, NORM>(n, i, npacks, sh, colSums, loadG, [&](int pk, const Pack16& o) {
        if (n.gradResidual != nullptr) st128(static_cast<char*>(n.gradResidual) + i * rb + pk * 16, o);
        st128(static_cast<char*>(n.gradPartial) + i * rb + pk * 16, o);
      });
    }
  } else if constexpr (V == kNormOneShot) {
    for (size_t i = blockIdx.x; i < n.rows; i += gridCtas()) {
      copyRow<T>(peers[a.rank] + i * rb, rowPtr(n.gradOut, i, rb), npacks);
    }
    if (!blockBarrier(a, loadEpoch(a) + 1)) {
      retire(a, 1, 1);
      return;
    }
    for (size_t i = blockIdx.x; i < n.rows; i += gridCtas()) {
      auto loadG = [&](typename R::Acc(&g)[R::kPacks]) {
        zeroAcc<T>(g);
        for (int r = 0; r < a.nranks; r++) addRow<T>(g, opaque(peers[r] + i * rb), npacks);
      };
      rowBackward<T, NORM>(n, i, npacks, sh, colSums, loadG, [&](int pk, const Pack16& o) {
        st128(static_cast<char*>(n.gradPartial) + i * rb + pk * 16, o);
      });
    }
  } else if constexpr (V == kNormTwoShot) {
    // Pool rows [0, rows): the staged gradOut, overwritten with gradPartial by the row's owner.
    const int P = a.nranks;
    char* mine = static_cast<char*>(x.mine);
    for (size_t i = blockIdx.x; i < n.rows; i += gridCtas()) copyRow<T>(mine + i * rb, rowPtr(n.gradOut, i, rb), npacks);
    if (!blockBarrier(a, loadEpoch(a) + 1)) {
      retire(a, 2, 0);
      return;
    }
    // This rank's rows [sb, se), the forward two-shot's split. The end is read from shared memory
    // where it is tested rather than held across the row loop, where it would spill (fp32 layer).
    __shared__ size_t ownEnd;
    size_t sb;
    {
      const size_t q = n.rows / P, rem = n.rows % P, me = static_cast<size_t>(a.rank);
      sb = me * q + (me < rem ? me : rem);
      if (threadIdx.x == 0) ownEnd = sb + q + (me < rem ? 1 : 0);
    }
    __syncthreads();
    const unsigned ctas = gridCtas();
    for (size_t i = sb + (blockIdx.x + ctas - sb % ctas) % ctas; i < ownEnd; i += gridCtas()) {
      auto loadG = [&](typename R::Acc(&g)[R::kPacks]) {
        zeroAcc<T>(g);
        for (int r = 0; r < P; r++) addRow<T>(g, opaque(peers[r] + i * rb), npacks);
      };
      rowBackward<T, NORM>(n, i, npacks, sh, colSums, loadG, [&](int pk, const Pack16& o) {
        for (int r = 0; r < P; r++) st128_stream(opaque(peers[r] + i * rb) + pk * 16, o);
      });
    }
    if (blockBarrier(a, loadEpoch(a) + 2)) {
      for (size_t i = blockIdx.x; i < n.rows; i += gridCtas()) {
        copyRow<T>(static_cast<char*>(n.gradPartial) + i * rb, mine + i * rb, npacks);
      }
    }
  } else {
    const int P = a.nranks;
    char* mine = static_cast<char*>(x.mine);
    const size_t rows = n.rows, all = static_cast<size_t>(P) * rows;
    const bool gather = x.gather != 0;
    const size_t gathered = gather ? all : 0;  // the pool row of gradResidual row 0
    auto userRow = [&](size_t j) { return j / rows * x.shardRows + j % rows; };
    if (gather) {
      for (size_t j = blockIdx.x; j < all; j += gridCtas()) copyRow<T>(mine + j * rb, rowPtr(n.gradOut, userRow(j), rb), npacks);
    }
    if (!blockBarrier(a, loadEpoch(a) + 1)) {
      retire(a, 2, 0);
      return;
    }
    const size_t sb = static_cast<size_t>(a.rank) * rows, se = sb + rows;
    const unsigned ctas = gridCtas();
    const size_t first = sb + (blockIdx.x + ctas - sb % ctas) % ctas;
    for (size_t j = first; j < se; j += gridCtas()) {
      const size_t i = j - sb;
      auto loadG = [&](typename R::Acc(&g)[R::kPacks]) {
        zeroAcc<T>(g);
        if (gather) {
          for (int r = 0; r < P; r++) addRow<T>(g, opaque(peers[r] + j * rb), npacks);
        } else {
          addRow<T>(g, opaque(rowPtr(n.gradOut, i, rb)), npacks);
        }
      };
      rowBackward<T, NORM>(n, i, npacks, sh, colSums, loadG, [&](int pk, const Pack16& o) {
        if (n.gradResidual != nullptr) st128(static_cast<char*>(n.gradResidual) + i * rb + pk * 16, o);
        for (int r = 0; r < P; r++) st128_stream(opaque(peers[r] + (gathered + j) * rb) + pk * 16, o);
      });
    }
    // The epoch read again rather than held across the row loop, where it would spill: it only
    // changes when the launch's last CTA retires.
    if (blockBarrier(a, loadEpoch(a) + 2)) {
      for (size_t j = blockIdx.x; j < all; j += gridCtas()) {
        copyRow<T>(static_cast<char*>(n.gradPartial) + userRow(j) * rb, mine + (gathered + j) * rb, npacks);
      }
    }
  }
  moveSums<T>(n, colSums, npacks, false);
  if constexpr (V == kNormOneShot) {
    retire(a, 1, 1);
  } else if constexpr (V != kNormLocal) {
    retire(a, 2, 0);
  }
}

constexpr int kFinishThreads = 256;
struct VecOuts {
  void* p[3];
};

// One column of one vector per thread: the CTAs' sums in CTA order, rounded once.
template <typename T>
__global__ void __launch_bounds__(kFinishThreads)
normBackwardFinishKernel(const float* ws, int slots, int vectors, unsigned long long hidden, VecOuts outs) {
  const size_t c = static_cast<size_t>(blockIdx.x) * kFinishThreads + threadIdx.x;
  const int v = blockIdx.y;
  if (c >= hidden || outs.p[v] == nullptr) return;
  float s = 0.0f;
  for (int b = 0; b < slots; b++) s += ws[(static_cast<size_t>(b) * vectors + v) * hidden + c];
  static_cast<T*>(outs.p[v])[c] = Scalar<T>::fromAcc(s);
}

// The two-shot allreduce backward's finish, a collective: its CTA sums cover this rank's rows only.
// Element k of the [vectors][hidden] vector per thread (grid-stride): this rank's CTA sums in CTA
// order (fp32), staged in its pool; barrier; the P staged vectors in rank order, rounded once, the
// same bytes on every rank; a closing barrier, so that no rank restages its pool while a peer still
// reads it. CTA b handles the same elements on every rank, so each barrier pairs the right CTAs.
template <typename T>
__global__ void __launch_bounds__(kFinishThreads)
normBackwardFinishAllreduceKernel(CommArgs a, const float* ws, int slots, int vectors, unsigned long long hidden,
                                  VecOuts outs, PeerPtrs pool) {
  // Indexed by a run-time rank / vector: from shared memory, filled with constant indices (a
  // dynamic index into the parameter space copies the struct to local memory).
  __shared__ const float* peers[kMaxRanks];
  __shared__ T* out[3];
  if (threadIdx.x == 0) {
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++) peers[r] = static_cast<const float*>(pool.p[r]);
#pragma unroll
    for (int v = 0; v < 3; v++) out[v] = static_cast<T*>(outs.p[v]);
  }
  __syncthreads();
  const uint32_t e = loadEpoch(a);
  const size_t len = static_cast<size_t>(vectors) * hidden, stride = static_cast<size_t>(gridDim.x) * kFinishThreads;
  float* mine = const_cast<float*>(peers[a.rank]);
  for (size_t k = static_cast<size_t>(blockIdx.x) * kFinishThreads + threadIdx.x; k < len; k += stride) {
    float s = 0.0f;
    for (int b = 0; b < slots; b++) s += ws[static_cast<size_t>(b) * len + k];
    mine[k] = s;
  }
  if (!blockBarrier(a, e + 1)) {
    retire(a, 2, 0);
    return;
  }
  for (size_t k = static_cast<size_t>(blockIdx.x) * kFinishThreads + threadIdx.x; k < len; k += stride) {
    float s = 0.0f;
    for (int r = 0; r < a.nranks; r++) s += peers[r][k];
    out[k / hidden][k % hidden] = Scalar<T>::fromAcc(s);
  }
  blockBarrier(a, e + 2);
  retire(a, 2, 0);
}

// The one place that names a backward instantiation: the launch, the occupancy query and the preload.
template <typename T>
auto normBwdFn(int norm, int variant) -> decltype(&normBackwardKernel<T, kNormRms, kNormLocal>) {
  auto byVariant = [&](auto normTag) -> decltype(&normBackwardKernel<T, kNormRms, kNormLocal>) {
    constexpr int N = decltype(normTag)::value;
    switch (variant) {
      case kNormScatter: return normBackwardKernel<T, N, kNormScatter>;
      case kNormLocal: return normBackwardKernel<T, N, kNormLocal>;
      case kNormOneShot: return normBackwardKernel<T, N, kNormOneShot>;
      case kNormTwoShot: return normBackwardKernel<T, N, kNormTwoShot>;
      default: return nullptr;
    }
  };
  switch (norm) {
    case kNormRms: return byVariant(std::integral_constant<int, kNormRms>{});
    case kNormLayer: return byVariant(std::integral_constant<int, kNormLayer>{});
    default: return nullptr;
  }
}

// The one place that names an instantiation: the launch, the occupancy query and the preload.
// The quantising form exists with a norm only.
template <typename T>
auto normFn(int norm, int variant, bool quant) -> decltype(&allreduceNormKernel<T, kNormNone, kNormLocal, false>) {
  using Fn = decltype(&allreduceNormKernel<T, kNormNone, kNormLocal, false>);
  auto byVariant = [&](auto normTag, auto quantTag) -> Fn {
    constexpr int N = decltype(normTag)::value;
    constexpr bool Q = decltype(quantTag)::value;
    switch (variant) {
      case kNormLL: return allreduceNormKernel<T, N, kNormLL, Q>;
      case kNormOneShot: return allreduceNormKernel<T, N, kNormOneShot, Q>;
      case kNormTwoShot: return allreduceNormKernel<T, N, kNormTwoShot, Q>;
      case kNormLocal: return allreduceNormKernel<T, N, kNormLocal, Q>;
      case kNormScatter: return allreduceNormKernel<T, N, kNormScatter, Q>;
      default: return nullptr;
    }
  };
  auto byQuant = [&](auto normTag) -> Fn {
    if (!quant) return byVariant(normTag, std::false_type{});
    if constexpr (decltype(normTag)::value != kNormNone) return byVariant(normTag, std::true_type{});
    return nullptr;
  };
  switch (norm) {
    case kNormNone: return byQuant(std::integral_constant<int, kNormNone>{});
    case kNormRms: return byQuant(std::integral_constant<int, kNormRms>{});
    case kNormLayer: return byQuant(std::integral_constant<int, kNormLayer>{});
    default: return nullptr;
  }
}

// Calls f(T{}) for the dtypes the fused operation takes; returns whether dt is one.
template <typename F>
bool dispatchNormType(DataType dt, F&& f) {
  switch (dt) {
    case DataType::FLOAT32: f(float{}); return true;
    case DataType::BFLOAT16: f(__nv_bfloat16{}); return true;
    case DataType::FLOAT16: f(__half{}); return true;
    default: return false;
  }
}

}  // namespace

bool normSupports(DataType dt) {
  return dispatchNormType(dt, [](auto) {});
}

const void* allreduceNormKernelFor(DataType dt, int norm, int variant, bool quant) {
  const void* k = nullptr;
  dispatchNormType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(normFn<decltype(tag)>(norm, variant, quant)); });
  return k;
}

void preloadAllreduceNormKernels() {
  for (DataType dt : {DataType::FLOAT32, DataType::BFLOAT16, DataType::FLOAT16}) {
    for (int norm : {kNormNone, kNormRms, kNormLayer}) {
      for (int v : {kNormLL, kNormOneShot, kNormTwoShot, kNormLocal, kNormScatter}) {
        for (bool quant : {false, true}) {
          if (quant && norm == kNormNone) continue;
          dispatchNormType(dt, [&](auto tag) { touchKernel(normFn<decltype(tag)>(norm, v, quant)); });
        }
      }
    }
    // The backward's column sums of the widest row take more than the default 48 KB.
    for (int norm : {kNormRms, kNormLayer}) {
      for (int v : {kNormScatter, kNormLocal, kNormOneShot, kNormTwoShot}) {
        dispatchNormType(dt, [&](auto tag) {
          const auto k = normBwdFn<decltype(tag)>(norm, v);
          touchKernel(k);
          cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               static_cast<int>(normBackwardSmemBytes(3)));
        });
      }
    }
    dispatchNormType(dt, [&](auto tag) {
      touchKernel(normBackwardFinishKernel<decltype(tag)>);
      touchKernel(normBackwardFinishAllreduceKernel<decltype(tag)>);
    });
  }
  cudaGetLastError();
}

void launchAllreduceNorm(const CommArgs& a, const NormArgs& n, const NormXchg& x, DataType dt, int norm, int variant,
                         int blocks, cudaStream_t stream) {
  dispatchNormType(dt, [&](auto tag) {
    if (auto k = normFn<decltype(tag)>(norm, variant, n.outScales != nullptr)) k<<<blocks, kThreads, 0, stream>>>(a, n, x);
  });
}

const void* normBackwardKernelFor(DataType dt, int norm, int variant) {
  const void* k = nullptr;
  dispatchNormType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(normBwdFn<decltype(tag)>(norm, variant)); });
  return k;
}

size_t normBackwardSmemBytes(int vectors) { return vectors > 0 ? 3 * kMaxNormHidden * sizeof(float) : 0; }

void launchNormBackward(const CommArgs& a, const NormBwdArgs& n, const NormXchg& x, DataType dt, int norm, int variant,
                        int blocks, cudaStream_t stream) {
  const size_t smem = normBackwardSmemBytes(n.vectors);
  dispatchNormType(dt, [&](auto tag) {
    if (auto k = normBwdFn<decltype(tag)>(norm, variant)) k<<<blocks, kThreads, smem, stream>>>(a, n, x);
  });
}

void launchNormBackwardFinish(const float* ws, int slots, int vectors, size_t hidden, void* const (&outs)[3],
                              DataType dt, cudaStream_t stream) {
  VecOuts o{{outs[0], outs[1], outs[2]}};
  const dim3 grid(static_cast<unsigned>((hidden + kFinishThreads - 1) / kFinishThreads), static_cast<unsigned>(vectors));
  dispatchNormType(dt, [&](auto tag) {
    normBackwardFinishKernel<decltype(tag)><<<grid, kFinishThreads, 0, stream>>>(ws, slots, vectors, hidden, o);
  });
}

const void* normBackwardFinishAllreduceKernelFor(DataType dt) {
  const void* k = nullptr;
  dispatchNormType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(normBackwardFinishAllreduceKernel<decltype(tag)>); });
  return k;
}

int normBackwardFinishThreads() { return kFinishThreads; }

void launchNormBackwardFinishAllreduce(const CommArgs& a, const float* ws, int slots, int vectors, size_t hidden,
                                       void* const (&outs)[3], const PeerPtrs& pool, DataType dt, int blocks,
                                       cudaStream_t stream) {
  VecOuts o{{outs[0], outs[1], outs[2]}};
  dispatchNormType(dt, [&](auto tag) {
    normBackwardFinishAllreduceKernel<decltype(tag)><<<blocks, kFinishThreads, 0, stream>>>(a, ws, slots, vectors, hidden,
                                                                                           o, pool);
  });
}

}  // namespace cuda
}  // namespace glb
