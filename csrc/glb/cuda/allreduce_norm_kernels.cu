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

__device__ __forceinline__ const char* rowPtr(const void* base, size_t row, size_t rowBytes) {
  return static_cast<const char*>(base) + row * rowBytes;
}

// The row epilogue on the reduced partials `acc` of row `row`: adds bias and residual, rounds
// once, and hands each pack of residualOut and out to store(k, resid, out). `npacks` packs per
// row; pack k of this thread is t + k * kThreads.
template <typename T, int NORM, typename Store>
__device__ __forceinline__ void rowEpilogue(typename NormRow<T>::Acc (&acc)[NormRow<T>::kPacks], const NormArgs& n,
                                            size_t row, int npacks, float* sh, Store&& store) {
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
      if constexpr (NORM == kNormLayer) {
#pragma unroll
        for (int e = 0; e < R::kE; e++) sum += acc[k].v[e];
      } else if constexpr (NORM == kNormRms) {
#pragma unroll
        for (int e = 0; e < R::kE; e++) sum = fmaf(acc[k].v[e], acc[k].v[e], sum);
      }
    }
  }
  if constexpr (NORM != kNormNone) {
    const float hidden = static_cast<float>(npacks * R::kE);
    float mean = 0.0f, rinv;
    if constexpr (NORM == kNormLayer) {
      mean = blockSum(sum, sh) / hidden;
      float sq = 0.0f;
#pragma unroll
      for (int k = 0; k < R::kPacks; k++) {
        if (t + k * kThreads < npacks) {
#pragma unroll
          for (int e = 0; e < R::kE; e++) {
            const float d = acc[k].v[e] - mean;
            sq = fmaf(d, d, sq);
          }
        }
      }
      rinv = 1.0f / sqrtf(blockSum(sq, sh) / hidden + n.eps);
    } else {
      rinv = 1.0f / sqrtf(blockSum(sum, sh) / hidden + n.eps);
    }
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
        store(pk, r, PT::narrow(acc[k]));
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

// Row i of the problem is handled by CTA i % gridDim.x of every rank.
template <typename T, int NORM, int V>
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
  auto toUser = [&](size_t row) {
    return [&, row](int pk, const Pack16& r, const Pack16& o) {
      st128(static_cast<char*>(n.residualOut) + row * rb + pk * 16, r);
      if (NORM != kNormNone) st128(static_cast<char*>(n.out) + row * rb + pk * 16, o);
    };
  };
  typename R::Acc acc[R::kPacks];

  if constexpr (V == kNormLocal) {
    for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
      zeroAcc<T>(acc);
      addRow<T>(acc, rowPtr(n.partial, i, rb), npacks);
      rowEpilogue<T, NORM>(acc, n, i, npacks, sh, toUser(i));
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
      rowEpilogue<T, NORM>(acc, n, i, npacks, sh, toUser(i));
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
      rowEpilogue<T, NORM>(acc, n, i, npacks, sh, toUser(i));
    }
    retire(a, 1, 1);
  } else if constexpr (V == kNormTwoShot) {
    // Pool rows: [0, rows) the staged partials, overwritten with residualOut by the row's owner;
    // [rows, 2 rows) out.
    const uint32_t e = loadEpoch(a);
    char* mine = static_cast<char*>(x.mine);
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
    for (size_t i = first; i < se; i += gridDim.x) {
      zeroAcc<T>(acc);
      for (int r = 0; r < P; r++) addRow<T>(acc, peers[r] + i * rb, npacks);
      rowEpilogue<T, NORM>(acc, n, i, npacks, sh, [&](int pk, const Pack16& rr, const Pack16& o) {
        for (int r = 0; r < P; r++) {
          st128_stream(peers[r] + i * rb + pk * 16, rr);
          if (NORM != kNormNone) st128_stream(peers[r] + (n.rows + i) * rb + pk * 16, o);
        }
      });
    }
    if (blockBarrier(a, e + 2)) {
      for (size_t i = blockIdx.x; i < n.rows; i += gridDim.x) {
        copyRow<T>(static_cast<char*>(n.residualOut) + i * rb, mine + i * rb, npacks);
        if (NORM != kNormNone) copyRow<T>(static_cast<char*>(n.out) + i * rb, mine + (n.rows + i) * rb, npacks);
      }
    }
    retire(a, 2, 0);
  } else {
    // n.rows rows of every shard. Pool rows: [0, P rows) the staged partials, row q * rows + i =
    // the user's partial row q * shardRows + i; with a gathered out, [P rows, 2 P rows) out in the
    // same order. Rank me owns pool rows [me * rows, (me + 1) * rows), shard row i = j - me * rows.
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
      rowEpilogue<T, NORM>(acc, n, i, npacks, sh, [&](int pk, const Pack16& rr, const Pack16& o) {
        st128(static_cast<char*>(n.residualOut) + i * rb + pk * 16, rr);
        if (NORM == kNormNone) return;
        if (gather) {
          for (int r = 0; r < P; r++) st128_stream(peers[r] + (all + j) * rb + pk * 16, o);
        } else {
          st128(static_cast<char*>(n.out) + i * rb + pk * 16, o);
        }
      });
    }
    if (blockBarrier(a, e + 2) && gather) {
      for (size_t j = blockIdx.x; j < all; j += gridDim.x) {
        copyRow<T>(static_cast<char*>(n.out) + userRow(j) * rb, mine + (all + j) * rb, npacks);
      }
    }
    retire(a, 2, 0);
  }
}

// The one place that names an instantiation: the launch, the occupancy query and the preload.
template <typename T>
auto normFn(int norm, int variant) -> decltype(&allreduceNormKernel<T, kNormNone, kNormLocal>) {
  auto byVariant = [&](auto normTag) -> decltype(&allreduceNormKernel<T, kNormNone, kNormLocal>) {
    constexpr int N = decltype(normTag)::value;
    switch (variant) {
      case kNormLL: return allreduceNormKernel<T, N, kNormLL>;
      case kNormOneShot: return allreduceNormKernel<T, N, kNormOneShot>;
      case kNormTwoShot: return allreduceNormKernel<T, N, kNormTwoShot>;
      case kNormLocal: return allreduceNormKernel<T, N, kNormLocal>;
      case kNormScatter: return allreduceNormKernel<T, N, kNormScatter>;
      default: return nullptr;
    }
  };
  switch (norm) {
    case kNormNone: return byVariant(std::integral_constant<int, kNormNone>{});
    case kNormRms: return byVariant(std::integral_constant<int, kNormRms>{});
    case kNormLayer: return byVariant(std::integral_constant<int, kNormLayer>{});
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

const void* allreduceNormKernelFor(DataType dt, int norm, int variant) {
  const void* k = nullptr;
  dispatchNormType(dt, [&](auto tag) { k = reinterpret_cast<const void*>(normFn<decltype(tag)>(norm, variant)); });
  return k;
}

void preloadAllreduceNormKernels() {
  for (DataType dt : {DataType::FLOAT32, DataType::BFLOAT16, DataType::FLOAT16}) {
    for (int norm : {kNormNone, kNormRms, kNormLayer}) {
      for (int v : {kNormLL, kNormOneShot, kNormTwoShot, kNormLocal, kNormScatter}) {
        dispatchNormType(dt, [&](auto tag) { touchKernel(normFn<decltype(tag)>(norm, v)); });
      }
    }
  }
  cudaGetLastError();
}

void launchAllreduceNorm(const CommArgs& a, const NormArgs& n, const NormXchg& x, DataType dt, int norm, int variant,
                         int blocks, cudaStream_t stream) {
  dispatchNormType(dt, [&](auto tag) {
    if (auto k = normFn<decltype(tag)>(norm, variant)) k<<<blocks, kThreads, 0, stream>>>(a, n, x);
  });
}

}  // namespace cuda
}  // namespace glb
