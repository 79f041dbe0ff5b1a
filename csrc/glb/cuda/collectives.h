// Host-side API of the CUDA-buffer collectives: argument checking, variant
// selection per message size and kernel launch. Every call is asynchronous on the
// given stream (a single kernel launch for registered buffers) and must be issued
// in the same order by every rank of the PeerContext.
//
// Buffers come in two flavours:
//   * PeerBuffer (registerBuffer / allocSymmetric): zero-copy, kernels read and
//     write the peers' copies directly;
//   * arbitrary device pointers: staged through the symmetric pool.
#pragma once

#include <cuda_runtime.h>

#include <string>
#include <vector>

#include "glb/cuda/kernels.h"
#include "glb/cuda/peer_context.h"
#include "glb/cuda/tuning.h"
#include "glb/types.h"

namespace glb {
namespace cuda {

enum class AllreduceAlgo : int {
  AUTO = 0,
  ONE_SHOT = 1,
  TWO_SHOT = 2,
  NVLS = 3,
  LL = 4,         // flag-in-data one-shot, no barrier (smallest messages)
  PIPELINED = 5,  // arbitrary pointers: in-kernel copy-in / exchange / copy-out pipeline through the pool
  HYBRID = 6,     // NVLS on one part of the vector + peer-to-peer two-shot on the rest, concurrently
  // Literal schedules of the reference's named algorithms, executed by the
  // step-table kernel over peer pointers (schedule_kernels.cu).
  RING = 10,
  RING_CHUNKED = 11,
  HALVING_DOUBLING = 12,
  BCUBE = 13,
  HALVING_DOUBLING_PIPELINED = 14,
};

const char* allreduceAlgoName(AllreduceAlgo a);

AllreduceAlgo allreduceAlgoFromName(const std::string& name);

// Process-wide knobs (initialised from GLB_CUDA_* env vars). Per-size decisions come from
// the tuning table (tuning.h); these are the fallbacks and global caps.
struct Tuning {
  size_t llMaxBytes = 16 * 1024;        // flag-in-data one-shot while bytes <= this
  size_t oneShotMaxBytes = 256 * 1024;  // barrier one-shot while bytes <= this / P; above: two-shot / NVLS
  size_t nvlsMinBytes = 32 * 1024;      // >= : NVLS when the buffer has a multicast alias (and P > 2)
  int maxBlocks = 128;                  // CTAs for the bandwidth kernels (clamped to the co-residency cap)
  int oneShotBlocks = 8;
  bool nvlsReduceScatter = false;       // multimem.ld_reduce in reduce_scatter / reduce instead of the P2P pull
                                        // (GLB_CUDA_NVLS_REDUCE_SCATTER); off by default
  int copyBlocks = 264;                 // CTAs for the store-only kernels (40 regs: 2-3 CTAs per SM; 2 x 132 SMs)
  int alltoallvBlocks = 64;             // fixed grid of the v-variant (sizes are rank-local, the grid must not be)
  size_t bcastDirectMaxBytes = 256 * 1024;  // <= : root pushes everything itself
  size_t bcastRelayMinBytes = 64u << 20;    // >= : chunk-pipelined relay broadcast (P > 2)
  int pipeTile = 1024;                  // 16-byte groups per tile of the pipelined kernel (power of two)
  int pipeExchangeThreads = 256;        // threads of each CTA that drive NVLink in the pipelined kernel
  bool tmaCopies = false;               // put / get / exchange through cp.async.bulk (TMA) instead of LDG/STG
                                        // when no table entry decides (GLB_CUDA_TMA)
};
Tuning& tuning();
// Number of collective kernels launched by this process so far.
uint64_t launchCount();
void noteLaunch(unsigned n = 1);  // local (non-collective) kernels report here

// What AUTO resolves to for a call, with the launch shape from the tuning table.
struct AllreducePlan {
  AllreduceAlgo algo = AllreduceAlgo::AUTO;
  LaunchCfg cfg;
  int tile = 0;
  bool fromTable = false;
};
AllreducePlan planAllreduce(PeerContext& pc, size_t bytes, DataType dt, ReduceOp op, BufKind kind);
// Which variant AUTO resolves to for this call (legacy signature).
AllreduceAlgo chooseAllreduce(PeerContext& pc, size_t bytes, DataType dt, ReduceOp op, bool registered,
                              bool hasMulticast);

// Optional per-call arguments of allreduce / reduce_scatter / reduce: the fused epilogue.
struct Epilogue {
  double scale = 1.0;           // multiply the reduced value before the final rounding (AVG: 1 / P)
  bool castOutput = false;      // store as `outDtype` instead of the input dtype
  DataType outDtype = DataType::FLOAT32;
  LocalPtrs extra;              // more local inputs (same count / dtype): folded in, and overwritten with the result
  // Pin the launch shape (tuner / sweeps); 0 = from the tuning table.
  int blocks = 0;
  int unroll = 0;
  int tile = 0;
};

void barrier(PeerContext& pc, cudaStream_t stream);

// In place on a registered / symmetric buffer (count elements from byteOffset).
void allreduce(PeerContext& pc, const PeerBuffer& buf, size_t byteOffset, size_t count, DataType dt, ReduceOp op,
               AllreduceAlgo algo, cudaStream_t stream, const Epilogue& ep = Epilogue());

// Arbitrary device pointers (in may equal out): LL / one-shot for small messages, the
// pipelined kernel above. With ep.castOutput `out` holds ep.outDtype elements (small
// messages only; larger ones need registered buffers, see allreduceCast).
void allreduce(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op,
               AllreduceAlgo algo, cudaStream_t stream, const Epilogue& ep = Epilogue());

// Out of place between two registered buffers with different dtypes (f32 <-> f16 / bf16):
// fp32 accumulation, one rounding to `outDt`.
void allreduceCast(PeerContext& pc, const PeerBuffer& in, size_t inOffset, const PeerBuffer& out, size_t outOffset,
                   size_t count, DataType dt, DataType outDt, ReduceOp op, cudaStream_t stream,
                   const Epilogue& ep = Epilogue());


// Allreduce of the partial sums `partial` ((rows, hidden), dt) fused with bias, residual add and
// a norm, one launch (docs/cuda.md, "Allreduce + residual + norm"): residualOut = round(sum of
// the partials + bias + residual), out = norm(residualOut) (kNormRms / kNormLayer; kNormNone
// writes residualOut only). dt is float32, bfloat16 or float16 for every tensor; hidden * element
// size is a multiple of 16 bytes and at most kMaxNormHidden elements; pointers are 16-byte aligned;
// bias / gamma / beta may be null. residualOut may be residual; no other output may overlap an
// input. Every rank passes the same residual, bias, gamma and beta, and gets the same bytes.
// Invalid arguments raise InputException before anything is launched. Returns the NormVariant.
// outScales set: the FP8 form (docs/cuda.md, "FP8 out"), with a norm and hidden a multiple of 16.
// out then holds e4m3 codes (rows, hidden) of the row o that the call without outScales writes,
// and outScales one fp32 scale per row (16-byte aligned): amax = max(max |o|, 1e-4), code =
// e4m3(o * (448 * (1 / amax))), scale = amax / 448. residualOut is unchanged; neither range may
// overlap an input or another output.
int allreduceResidualNorm(PeerContext& pc, const void* partial, const void* residual, void* residualOut, void* out,
                          const void* bias, const void* gamma, const void* beta, size_t rows, size_t hidden,
                          DataType dt, int norm, float eps, AllreduceAlgo algo, cudaStream_t stream,
                          float* outScales = nullptr);
// The variant that call runs (the planAllreduce choice for a plain buffer of its bytes, or an
// explicit LL / ONE_SHOT / TWO_SHOT), and its launches: the two-shot stages its rows in the pool's
// bulk region, so beyond what that holds it runs as consecutive chunks of chunkRows rows (`quant`:
// the FP8 form, whose out rows there are hidden code bytes and a scale).
struct NormPlan {
  int variant;
  size_t chunkRows;
  size_t launches;
};
NormPlan planResidualNorm(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm, AllreduceAlgo algo,
                          bool quant = false);
const char* normVariantName(int variant);

// The reduce-scatter form of allreduceResidualNorm, for sequence parallelism (docs/cuda.md,
// "Reduce-scatter + residual + norm"). `partial` holds rows = P x Ts rows on every rank; rank r
// owns rows [r Ts, (r + 1) Ts), and residual / residualOut are its shard of Ts rows:
// residualOut[i] = round(sum of the partials' row r Ts + i + bias + residual[i]), with the sum
// order, rounding and limits of allreduceResidualNorm, so the bytes equal the matching rows of
// its outputs. out = norm(residualOut): this rank's Ts rows, or with gatherOut all P shards
// (rows rows, shard q at row q Ts) on every rank. rows % P == 0. One rank runs the allreduce
// form's local launch. Invalid arguments raise InputException before anything is launched.
// outScales set: the FP8 form of allreduceResidualNorm, out and outScales with out's rows (a
// gathered out: shard q's codes and scales at row q Ts).
int reduceScatterResidualNorm(PeerContext& pc, const void* partial, const void* residual, void* residualOut, void* out,
                              const void* bias, const void* gamma, const void* beta, size_t rows, size_t hidden,
                              DataType dt, int norm, float eps, bool gatherOut, cudaStream_t stream,
                              float* outScales = nullptr);
// Its variant (kNormScatter, or kNormLocal for one rank) and launches: it stages every shard's rows
// (and a gathered out) in the pool's bulk region, so beyond what that holds it runs as consecutive
// chunks of chunkRows rows of every shard.
NormPlan planReduceScatterNorm(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm, bool gatherOut,
                               bool quant = false);

// The backward of reduceScatterResidualNorm with a norm (kNormRms / kNormLayer), for training with
// sequence parallelism (docs/cuda.md, "Backward of the reduce-scatter norm"), on the forward's
// exchange and chunking. rows = P x Ts; s is the saved residualOut shard (Ts rows), gradS the
// gradient of it (null: zero), gradOut the gradient of out: rows rows (a partial per rank) with
// gatherOut, this rank's Ts rows without. Per shard row, in fp32: g = the sum over ranks of gradOut
// in rank order (or gradOut), the statistics recomputed from s exactly as the forward computed
// them, gradResidual = round(gradS + the norm's input gradient). gradPartial (rows rows) gets every
// rank's gradResidual shards, shard q at row q Ts, the same bytes on every rank; gradResidual
// (optional, may be gradS) this rank's. Optional column sums over this rank's rows, fp32, rounded
// once, in a fixed order (no floating-point atomics): gradWeight = sum g xh, gradNormBias = sum g
// (layer only), gradBias = sum of the rounded gradResidual rows. They need `workspace` (16-byte
// aligned, at least the plan's workspaceBytes). Ts = 0 launches nothing and zeroes the column sums.
// One rank runs a local launch. Invalid arguments raise InputException before anything is launched.
int reduceScatterResidualNormBackward(PeerContext& pc, const void* gradOut, const void* s, const void* gradS,
                                      void* gradResidual, void* gradPartial, const void* gamma, void* gradWeight,
                                      void* gradNormBias, void* gradBias, void* workspace, size_t workspaceBytes,
                                      size_t rows, size_t hidden, DataType dt, int norm, float eps, bool gatherOut,
                                      cudaStream_t stream);
// Its variant (kNormScatter, or kNormLocal for one rank), chunk rows and launches (the chunks, plus
// one that finishes the column sums when `vectors` > 0 of them are asked for), the grid, and the
// fp32 workspace of the column sums: blocks x vectors x hidden floats.
struct NormBackwardPlan {
  int variant;
  size_t chunkRows;
  size_t launches;
  int blocks;
  size_t workspaceBytes;
};
NormBackwardPlan planReduceScatterNormBackward(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm,
                                               bool gatherOut, int vectors);

// The backward of allreduceResidualNorm with a norm (kNormRms / kNormLayer), for training with
// tensor parallelism (docs/cuda.md, "Backward of the allreduce norm"). Every rank holds all rows of
// s (the saved residualOut) and gradS (its gradient, null: zero); gradOut is this rank's partial of
// out's gradient. Per row, in fp32: g = the sum over ranks of gradOut in rank order, the statistics
// recomputed from s exactly as the forward computed them, gradPartial = round(gradS + the norm's
// input gradient), the same bytes on every rank and for both variants; it is also the gradient of
// the residual, and may be gradS itself. Optional column sums over all rows, fp32, rounded once, in
// a fixed order, the same bytes on every rank: gradWeight = sum g xh, gradNormBias = sum g (layer
// only), gradBias = sum of the rounded gradPartial rows. They need `workspace` (16-byte aligned, at
// least the plan's workspaceBytes). rows = 0 launches nothing and zeroes the column sums. algo:
// AUTO, ONE_SHOT or TWO_SHOT; one rank runs a local launch. Invalid arguments raise InputException
// before anything is launched. Returns the NormVariant.
int allreduceResidualNormBackward(PeerContext& pc, const void* gradOut, const void* s, const void* gradS,
                                  void* gradPartial, const void* gamma, void* gradWeight, void* gradNormBias,
                                  void* gradBias, void* workspace, size_t workspaceBytes, size_t rows, size_t hidden,
                                  DataType dt, int norm, float eps, AllreduceAlgo algo, cudaStream_t stream);
// Its variant (kNormOneShot, kNormTwoShot or kNormLocal; AUTO takes the forward's variant for these
// rows, its LL as the one-shot), chunk rows (the two-shot stages one pool row per row), launches
// (chunks, plus one that finishes the column sums when `vectors` > 0), grid and workspace, as
// planReduceScatterNormBackward reports them.
NormBackwardPlan planResidualNormBackward(PeerContext& pc, size_t rows, size_t hidden, DataType dt, int norm,
                                          int vectors, AllreduceAlgo algo);


// ---- data movement -------------------------------------------------------------------
// `buf`/`out` arguments are registered or symmetric buffers; plain-pointer
// overloads stage through the pool (payload limited to the pool's bulk region).

// In place: root's bytes replace everyone's.
void broadcast(PeerContext& pc, const PeerBuffer& buf, size_t byteOffset, size_t bytes, int root,
               cudaStream_t stream);
void broadcast(PeerContext& pc, void* ptr, size_t bytes, int root, cudaStream_t stream);

// Rank r's `in` (bytesPerRank[r] bytes) lands at the prefix-sum offset in every out.
void allgatherv(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset,
                const std::vector<size_t>& bytesPerRank, cudaStream_t stream);
void allgatherv(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& bytesPerRank,
                cudaStream_t stream);
// The cast form (docs/cuda.md, "Cast reduce-scatter / allgather"): rank r's `in` holds counts[r]
// float32 elements (inDt), and lands in every out as outDt (float16 / bfloat16), rounded once on
// the sender (to nearest even; overflow to +-inf, NaN stays NaN), so only 16-bit bytes cross
// NVLink. Counts are in elements; inDt == outDt is the byte form above. Another pair, an `in` that
// overlaps the output or an output range beyond the registered buffer raises InputException
// before any launch. Never LL; one launch per call at P > 1 (one local kernel at P = 1).
void allgatherv(PeerContext& pc, const void* in, DataType inDt, const PeerBuffer& out, size_t outOffset,
                const std::vector<size_t>& counts, DataType outDt, cudaStream_t stream);
void allgatherv(PeerContext& pc, const void* in, DataType inDt, void* out, const std::vector<size_t>& counts,
                DataType outDt, cudaStream_t stream);
// Only `root` receives.
void gatherv(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset,
             const std::vector<size_t>& bytesPerRank, int root, cudaStream_t stream);
void gatherv(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& bytesPerRank, int root,
             cudaStream_t stream);

// Chunk j of my input (sendBytes[j] at the prefix-sum offset) goes to rank j, which
// stores what it gets from rank i at the prefix-sum offset of ITS recvBytes[i].
void alltoallv(PeerContext& pc, const void* in, const std::vector<size_t>& sendBytes, const PeerBuffer& out,
               size_t outOffset, const std::vector<size_t>& recvBytes, cudaStream_t stream);
void alltoallv(PeerContext& pc, const void* in, const std::vector<size_t>& sendBytes, void* out,
               const std::vector<size_t>& recvBytes, cudaStream_t stream);

// Where the rows of a device-split MoE call live on this rank: a registered buffer at `offset`
// (zero copy), or, with `buf` null, a plain device pointer (staged through the pool, which also
// caps the capacity). Every rank must pass the same kind; a mix is invalid input on every rank.
struct MoeOut {
  const PeerBuffer* buf = nullptr;
  size_t offset = 0;
  void* ptr = nullptr;
};

// All-to-all-v whose row counts live on the device (expert-parallel dispatch / combine): one
// kernel, no host value depends on the device data, so it needs no synchronisation and can be
// captured in a CUDA graph. A row is `rowBytes` on every rank; `in` holds `inRows` rows.
// `inSplits` has P·E int64 entries.
//   forward (inverse = false): entry j·E + e = my rows for expert e of rank j, packed in that
//     order in `in`. Each rank receives expert-major: expert e's segment starts at a multiple of
//     `align` rows and holds the rows of sources 0..P-1 in order; it writes outSplits[e·P + s] /
//     outOffsets[e·P + s] (int64, rows) for its segment from source s.
//   inverse: `inSplits` / `inOffsets` (entry e·P + s) describe the forward output layout; the
//     rows go back to where they came from, packed in (holder, expert) order.
// An output that would need more than its capacity (`capacityRows`, and for a plain pointer also
// what fits the staging pool) receives nothing; invalid splits or offsets move nothing. Either
// is raised as InputException by the next checkHealth() on every rank that runs after the kernel
// has (synchronize() is the dependable place: earlier calls may not see it yet).
// `outScales` set: the quantising forward form (FP8 expert dispatch). `in` holds `inRows` bf16
// rows of `rowBytes` = hidden elements (a multiple of kFp8Block); each row arrives as `hidden`
// e4m3 codes in `out` and hidden / kFp8Block fp32 scales in `outScales` (row-major, capacityRows
// rows), at the same row index, so x ~= code * scale. Per block of kFp8Block elements: amax =
// max(max|x|, 1e-4), code = e4m3(x * (448 * (1 / amax))) (round to nearest even, saturating),
// scale = amax / 448, each a correctly rounded fp32 operation. `in` and `out` must be 16-byte
// aligned, and out and outScales of one kind. For plain pointers the capacity is capped by what
// fits the staging pool at hidden + hidden / 32 bytes a row.
void alltoallvDev(PeerContext& pc, const void* in, size_t inRows, size_t rowBytes, const int64_t* inSplits,
                  const int64_t* inOffsets, const MoeOut& out, size_t capacityRows, int64_t* outSplits,
                  int64_t* outOffsets, int experts, int align, bool inverse, cudaStream_t stream,
                  const MoeOut* outScales = nullptr);
// Top-k MoE dispatch: route() + the forward alltoallvDev in one kernel. `x` holds `tokens` rows
// of `rowBytes` (a multiple of 16; x and out 16-byte aligned, disjoint); `topkIdx` is int64
// (tokens, topk), 1 <= topk <= 32, tokens x topk < 2^31: entry j·E + e chooses local expert e
// of rank j, anything outside 0..P·E-1 is not routed. Writes `splits` (P·E: routed choices per
// (rank, expert)) and `pos` ((tokens, topk): the row of route()'s rows that carries each choice,
// -1 if not routed), from this rank's input alone, even when the call fails. out, outSplits and
// outOffsets then equal those of alltoallvDev(route()'s rows, splits) byte for byte: within a
// (rank, expert) group rows go by token, then by choice. Each token is read once and stored to
// each of its choices. Capacity, paths and error reporting are those of alltoallvDev.
// `outScales` set: the quantising form, with alltoallvDev's input, outputs, numerics and checks;
// each token is quantised once and the same codes and scales are stored to all its choices.
void alltoallvDevTopk(PeerContext& pc, const void* x, size_t tokens, size_t rowBytes, int topk, const int64_t* topkIdx,
                      int64_t* splits, int64_t* pos, const MoeOut& out, size_t capacityRows, int64_t* outSplits,
                      int64_t* outOffsets, int experts, int align, cudaStream_t stream,
                      const MoeOut* outScales = nullptr);
// Top-k MoE combine: the inverse of the forward alltoallvDev fused with the gate-weighted sum.
// `splits` is the in_splits this rank passed to the dispatch; `expertOut` holds, on every rank, the
// experts' output rows (`rowBytes` each, dtype dt: float, bfloat16 or float16) in that dispatch's
// output layout, `capacityRows` of them. `pos` / `weights` are (tokens, topk): pos[t, j] is the row
// of my dispatch input that carried token t's choice j (-1: not sent). out row t =
// round(sum over j with pos[t, j] >= 0, in order, of weights[t, j] * float(row)), each step a
// correctly rounded fp32 multiply and add, starting from +0. The source pulls its rows, so nothing
// but `out` is written. Registered expertOut: read in place; plain: each rank stages its rows
// through its pool, which caps the capacity. Rows must be a multiple of 16 bytes, expertOut and
// out 16-byte aligned and disjoint, 1 <= topk <= 32. Errors found on the device (splits, a pos
// out of range, arguments that differ between ranks, an overflowing holder) are raised like
// alltoallvDev's, and no rank writes its out. Null `weights`: every weight is 1 (the unweighted
// sum, the backward of the top-k dispatch), byte for byte a call with a tensor of ones.
void alltoallvDevCombineTopk(PeerContext& pc, void* out, size_t tokens, int topk, const int64_t* pos,
                             const float* weights, const int64_t* splits, const MoeOut& expertOut, size_t capacityRows,
                             size_t rowBytes, DataType dt, int experts, int align, cudaStream_t stream);
// Backward of alltoallvDevCombineTopk, in one kernel, with its arguments and `gradOut` (dy, tokens
// rows of dt). For each routed choice (t, j): gradWeights[t, j] = sum over h of float(dy[t, h]) ·
// float(row[h]), in fp32 (+0 where pos = -1), and the holder's gradExpertOut row (same layout and
// capacity as expertOut) = round(weights[t, j] · float(dy[t])), one correctly rounded multiply. Each
// holder writes +0 to every gradExpertOut row outside its receive segments. expertOut and
// gradExpertOut are both registered (zero copy) or both plain (staged: each rank's pool then holds
// both, which caps the capacity at half that of the combine). gradExpertOut must not overlap
// expertOut, gradOut or gradWeights. pos must name each dispatch-input row at most once. Errors
// found on the device are raised like the combine's, and no rank writes gradExpertOut or
// gradWeights.
void alltoallvDevCombineTopkBackward(PeerContext& pc, const MoeOut& gradExpertOut, float* gradWeights,
                                     const void* gradOut, const MoeOut& expertOut, size_t tokens, int topk,
                                     const int64_t* pos, const float* weights, const int64_t* splits,
                                     size_t capacityRows, size_t rowBytes, DataType dt, int experts, int align,
                                     cudaStream_t stream);
// Low-latency top-k MoE exchange for decoding (moe_kernels.cu): fixed per-(expert, source) slots in a
// buffer every rank allocates with the same arguments, one signal round each way, no barrier, static
// shapes. The layout of that buffer for P ranks, E experts per rank, max_tokens tokens per rank, top-k
// and rows of `hidden` elements of `elemBytes` (fp8: bf16 in, e4m3 codes + fp32 scales per 128 in the
// slots, bf16 combine rows). Every region starts at a multiple of 16 bytes:
//   E·P·max_tokens dispatch rows of rowBytes, their scales (fp8) and int32 tags; E·P 64-bit dispatch
//   words; max_tokens·k combine rows; P 64-bit combine words; max_tokens·k int32 choice marks; 16
//   bytes of call count and ticket.
// Limits: 1 <= E <= 32, 1 <= k <= 32, max_tokens >= 1, max_tokens·k <= 2^31 - 1, rows a positive
// multiple of 16 bytes (fp8: hidden a multiple of 128).
MoeLLLayout moeLLLayout(int nranks, int experts, int maxTokens, int topk, size_t hidden, size_t elemBytes, bool fp8);
// Dispatch on the buffer at `offset` of `buf` (symmetric, layout `l`): x (tokens <= max_tokens rows;
// fp8: bf16), topkIdx int64 (tokens, k); out / outScales plain (E, P·max_tokens, ...) and outSplits
// int64 (E·P). Expert e's rows land in out[e, 0 : sum_s outSplits[e·P + s]] in source order, then
// by token and choice: the bytes of expert e's segment from alltoallvDevTopk. Rows past it are not
// written. A (source, expert) group above max_tokens rows sends nothing and is raised on the source
// and the holder at the next host call.
void alltoallvLLTopk(PeerContext& pc, const PeerBuffer& buf, size_t offset, const MoeLLLayout& l, const void* x,
                     size_t tokens, const int64_t* topkIdx, void* out, float* outScales, int64_t* outSplits,
                     cudaStream_t stream);
// Combine on the same buffer after its dispatch: expertOut (E, P·max_tokens, H) of dt in the
// dispatch's out layout; y (tokens, H) of dt; weights float32 (tokens, k) or null (weight 1). y
// equals alltoallvDevCombineTopk's on the same expert rows byte for byte.
void alltoallvLLCombineTopk(PeerContext& pc, const PeerBuffer& buf, size_t offset, const MoeLLLayout& l, void* y,
                            size_t tokens, const void* expertOut, const float* weights, DataType dt,
                            cudaStream_t stream);
// Fixed-size alltoall: every chunk is `bytes` long on every rank (this is known to all
// ranks, so the small-message LL kernel and size-dependent grids are safe here).
void alltoall(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset, size_t bytes,
              cudaStream_t stream);
void alltoall(PeerContext& pc, const void* in, void* out, size_t bytes, cudaStream_t stream);
// Root's input holds P chunks of `bytes`; chunk j lands in rank j's out.
void scatter(PeerContext& pc, const void* in, const PeerBuffer& out, size_t outOffset, size_t bytes, int root,
             cudaStream_t stream);
void scatter(PeerContext& pc, const void* in, void* out, size_t bytes, int root, cudaStream_t stream);

// Rank r gets elements [prefix(counts, r), +counts[r]) of the reduction in `out`.
void reduce_scatter(PeerContext& pc, const PeerBuffer& in, size_t inOffset, void* out,
                    const std::vector<size_t>& counts, DataType dt, ReduceOp op, cudaStream_t stream,
                    double scale = 1.0);
void reduce_scatter(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& counts, DataType dt,
                    ReduceOp op, cudaStream_t stream, double scale = 1.0);
// The cast form (docs/cuda.md, "Cast reduce-scatter / allgather"): dt float16 / bfloat16, outDt
// float32, op SUM. out[i] = fp32(sum over ranks of float(in_q[off_r + i])) * fp32(scale): the
// sum is accumulated in fp32 and never rounded to 16 bits. outDt == dt is the call above. Every
// path of that call runs (registered, staged, pipelined; one local kernel at P = 1), never LL or
// NVLS; one launch per call at P > 1. Another pair, another op, an `out` that overlaps the input
// or an input range beyond the registered buffer raises InputException before any launch.
void reduce_scatter(PeerContext& pc, const PeerBuffer& in, size_t inOffset, void* out, const std::vector<size_t>& counts,
                    DataType dt, DataType outDt, ReduceOp op, cudaStream_t stream, double scale = 1.0);
void reduce_scatter(PeerContext& pc, const void* in, void* out, const std::vector<size_t>& counts, DataType dt,
                    DataType outDt, ReduceOp op, cudaStream_t stream, double scale = 1.0);
// Reduction of every rank's `in` delivered to root's `out` (both registered).
void reduce(PeerContext& pc, const PeerBuffer& in, size_t inOffset, const PeerBuffer& out, size_t outOffset,
            size_t count, DataType dt, ReduceOp op, int root, cudaStream_t stream);
void reduce(PeerContext& pc, const void* in, void* out, size_t count, DataType dt, ReduceOp op, int root,
            cudaStream_t stream);

// ---- point to point ----------------------------------------------------------------------------
// Device buffers between two ranks over NVLink (p2p_kernels.cu). Sends and receives between
// a pair of ranks match in posting order. sendrecv posts both directions in ONE kernel, the
// right call for ring / pipeline exchanges (a separate send and recv on one stream would
// serialise and, for messages larger than the mailbox ring, wait for each other).
void send(PeerContext& pc, const void* ptr, size_t bytes, int dst, cudaStream_t stream);
void recv(PeerContext& pc, void* ptr, size_t bytes, int src, cudaStream_t stream);
void sendrecv(PeerContext& pc, const void* sendPtr, size_t sendBytes, int dst, void* recvPtr, size_t recvBytes,
              int src, cudaStream_t stream);
// One-sided on registered memory: my [local, local+bytes) <-> rank `peer`'s copy of `remote`
// at remoteOffset. Completion is stream order on the initiator; the target learns about it
// through a later collective / barrier / message (RDMA semantics, as
// gloo/transport/unbound_buffer.h:128-152).
// Zero-copy sendrecv for a peer-mapped receive buffer that every rank uses at the same offset
// (ring attention's K/V double buffer, a pipeline stage's activation slot): my `sendBytes` are
// written straight into recvBuf on `dst` at recvOffset, `src` writes into mine. One kernel, one
// pass over the data, one flag round trip per call. After it completes on `stream`, my
// recvBuf[recvOffset, +recvBytes) holds src's payload; my sendPtr may be reused. The receive
// range must not be read or written by work queued behind the PREVIOUS exchange's consumer
// until this call is enqueued (the kernel start is the "ready to be overwritten" signal).
void exchange(PeerContext& pc, const void* sendPtr, size_t sendBytes, int dst, const PeerBuffer& recvBuf,
              size_t recvOffset, size_t recvBytes, int src, cudaStream_t stream);
void put(PeerContext& pc, const void* local, const PeerBuffer& remote, size_t remoteOffset, size_t bytes, int peer,
         cudaStream_t stream);
void get(PeerContext& pc, void* local, const PeerBuffer& remote, size_t remoteOffset, size_t bytes, int peer,
         cudaStream_t stream);

}  // namespace cuda
}  // namespace glb
