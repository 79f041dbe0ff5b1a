// Host-callable launchers for the device kernels (implemented in the .cu files).
#pragma once

#include <cuda_runtime.h>

#include "glb/cuda/comm_types.h"
#include "glb/types.h"

namespace glb {
namespace cuda {

// Force-load all kernels of the library on the current device (idempotent, cheap).
void preloadAllreduceKernels();
void preloadCollectiveKernels();
void preloadMoeKernels();
void preloadScheduleKernels();
void preloadLocalKernels();
void preloadPipelineKernels();
void preloadP2pKernels();
void preloadAllreduceNormKernels();

// allreduce_kernels.cu ---------------------------------------------------------------------
void launchBarrier(const CommArgs& a, cudaStream_t stream);
// Flag-in-data one-shot (no barrier). `ll.p[r]` = LL region of rank r's pool.
void launchLLAllreduce(const CommArgs& a, const void* in, void* out, size_t count, DataType dt, DataType outDt,
                       ReduceOp op, float scale, const PeerPtrs& ll, size_t srcStride, size_t parityStride,
                       const LocalPtrs& extra, int blocks, int threads, cudaStream_t stream);
// Small reduce_scatter (equal shares of `perRank` elements), flag-in-data, no barrier.
void launchLLReduceScatter(const CommArgs& a, const void* in, void* out, size_t perRank, DataType dt, ReduceOp op,
                           float scale, const PeerPtrs& ll, size_t srcStride, size_t parityStride, int blocks, int threads,
                           cudaStream_t stream);
void launchOneShotAllreduce(const CommArgs& a, const void* in, void* out, size_t count, DataType dt, ReduceOp op,
                            float scale, const PeerPtrs& stage, size_t halfBytes, const LocalPtrs& extra, int blocks,
                            cudaStream_t stream);
void launchTwoShotAllreduce(const CommArgs& a, const PeerPtrs& bufs, size_t count, DataType dt, ReduceOp op,
                            float scale, bool vectorOk, const LocalPtrs& extra, const LaunchCfg& cfg,
                            cudaStream_t stream);
bool nvlsSupports(DataType dt, ReduceOp op);
void setOneShotPush(bool on);  // tuning / A-B testing of the push flavour of one-shot
bool oneShotPushEnabled();
void launchNvlsAllreduce(const CommArgs& a, void* mcPtr, const PeerPtrs& bufs, size_t count, DataType dt, float scale,
                         const LocalPtrs& extra, const LaunchCfg& cfg, cudaStream_t stream);
// NVLS on the first part of the vector + peer-to-peer two-shot on the rest, concurrently
// (P = 4 or 8, sum of f32 / f16 / bf16, multicast-bound buffer).
const void* hybridKernelFor(DataType dt, int nranks);
void launchHybridAllreduce(const CommArgs& a, void* mcPtr, const PeerPtrs& bufs, size_t count, DataType dt, float scale,
                           int blocks, int nvlsBlocks, unsigned p2pPermille, cudaStream_t stream);
// Output dtype != input dtype (f32 <-> f16/bf16): out-of-place on registered buffers.
bool castSupported(DataType in, DataType out);
void launchCastAllreduce(const CommArgs& a, const PeerPtrs& ins, void* mcIn, const PeerPtrs& outs, size_t count,
                         DataType dt, DataType outDt, ReduceOp op, float scale, bool vectorOk, int blocks,
                         cudaStream_t stream);
// Kernel entry points (for occupancy queries: grids must stay co-resident).
const void* twoShotKernelFor(DataType dt, int nranks, int unroll);
const void* nvlsKernelFor(DataType dt, int unroll);
const void* castKernelFor(DataType in, DataType out);

// allreduce_norm_kernels.cu — allreduce fused with bias, residual add and RMSNorm / LayerNorm ------
// Widest row (elements) of the fused operation: a CTA holds a whole row in registers.
constexpr int kMaxNormHidden = 16384;
enum NormKind : int { kNormNone = 0, kNormRms = 1, kNormLayer = 2 };
// The exchange of the partials: LL lines, one-shot pool halves, row-sharded two-shot through the
// pool's bulk region, or none (one rank). kNormScatter is the reduce-scatter form (sequence
// parallelism): each rank keeps the rows of its own token shard, out optionally gathered.
enum NormVariant : int { kNormLL = 0, kNormOneShot = 1, kNormTwoShot = 2, kNormLocal = 3, kNormScatter = 4 };
// One (rows, hidden) problem: contiguous rows of hidden elements, 16-byte aligned. bias / gamma /
// beta may be null (none, 1, 0); out is unused without a norm. outScales set (the quantising form,
// with a norm, hidden a multiple of 16): out holds e4m3 codes (rows, hidden) and outScales one
// fp32 scale per row.
struct NormArgs {
  const void* partial;
  const void* residual;
  void* residualOut;
  void* out;
  const void* bias;
  const void* gamma;
  const void* beta;
  unsigned long long rows;
  unsigned long long hidden;
  float eps;
  float* outScales = nullptr;
};
// Where the partials travel. LL: peers.p[r] = rank r's LL region, mine = mine, srcStride and
// parityStride its layout. One-shot: rank r's pool halves, parityStride = one half. Two-shot: rank
// r's 2 x rows rows of the bulk region. Reduce-scatter: rank r's bulk region (P x rows staged rows,
// then P x rows gathered out rows when `gather`); shardRows = rows between the shards of the
// user's partial and gathered out (NormArgs::rows is the chunk of every shard). The quantising
// form's out in the pool is its rows of hidden code bytes, then one fp32 scale per row.
struct NormXchg {
  PeerPtrs peers;
  void* mine;
  unsigned long long srcStride;
  unsigned long long parityStride;
  unsigned long long shardRows;
  int gather;
};
bool normSupports(DataType dt);
const void* allreduceNormKernelFor(DataType dt, int norm, int variant, bool quant = false);
void launchAllreduceNorm(const CommArgs& a, const NormArgs& n, const NormXchg& x, DataType dt, int norm, int variant,
                         int blocks, cudaStream_t stream);
// The backward of the reduce-scatter form with a norm, one chunk of `rows` rows of every shard
// (kNormScatter; the NormXchg as in the forward, with the pool rows of docs/cuda.md) or of the
// one rank's rows (kNormLocal). s / gradS / gradResidual are this rank's shard rows; gradOut is
// its shard, or with x.gather P shards x.shardRows apart; gradPartial is P shards x.shardRows
// apart. gradS / gradResidual / gamma may be null. ws: per-CTA fp32 column sums, [CTA][vectors]
// [hidden]; vecWeight / vecNormBias / vecBias index the vectors (-1: not asked for). `first`: the
// first chunk starts the sums from zero, later chunks from ws.
// The allreduce forms (kNormOneShot: x as the forward's one-shot; kNormTwoShot: x.peers the bulk
// regions) take `rows` rows of s, gradS, gradOut (this rank's partial) and gradPartial; gradResidual
// is unused.
struct NormBwdArgs {
  const void* gradOut;
  const void* s;
  const void* gradS;
  void* gradResidual;
  void* gradPartial;
  const void* gamma;
  float* ws;
  unsigned long long rows;
  unsigned long long hidden;
  float eps;
  int vectors;
  int vecWeight;
  int vecNormBias;
  int vecBias;
  int first;
};
const void* normBackwardKernelFor(DataType dt, int norm, int variant);
// Dynamic shared memory of that kernel: the CTA's fp32 column sums (none without vectors).
size_t normBackwardSmemBytes(int vectors);
void launchNormBackward(const CommArgs& a, const NormBwdArgs& n, const NormXchg& x, DataType dt, int norm, int variant,
                        int blocks, cudaStream_t stream);
// out_v[c] = round(sum over slots b < `slots` in order of ws[b][v][c]) for each vector v whose
// out is non-null (outs in the order of ws's vectors).
void launchNormBackwardFinish(const float* ws, int slots, int vectors, size_t hidden, void* const (&outs)[3],
                              DataType dt, cudaStream_t stream);
// The same for the two-shot allreduce backward, whose slots hold this rank's rows only: a collective
// that stages this rank's fp32 sums at pool.p[rank] (vectors x hidden floats), sums the P staged
// vectors in rank order and rounds once, the same bytes on every rank. Every rank launches the same
// co-resident grid of normBackwardFinishThreads() threads per CTA.
const void* normBackwardFinishAllreduceKernelFor(DataType dt);
int normBackwardFinishThreads();
void launchNormBackwardFinishAllreduce(const CommArgs& a, const float* ws, int slots, int vectors, size_t hidden,
                                       void* const (&outs)[3], const PeerPtrs& pool, DataType dt, int blocks,
                                       cudaStream_t stream);

// pipeline_kernels.cu — arbitrary pointers through the pool, in-kernel pipelines (allreduce:
// 3 stages).
const void* pipelinedKernelFor(DataType dt, bool mc, int nranks);
void launchPipelinedAllreduce(const CommArgs& a, const void* in, void* out, size_t count, DataType dt, ReduceOp op,
                              float scale, const PeerPtrs& stage, void* mcStage, int tileVecs, int exchangeThreads,
                              const LocalPtrs& extra, int blocks, cudaStream_t stream);
// allgather(v) / gather(v) of plain pointers of any size, two-stage pipeline through two pool
// slots of G x tileVecs 16-byte groups. Rank r's block (lens[r] bytes) lands at offs[r] of the
// output of every rank, or of rank onlyDst only (>= 0: gather; nothing else writes its out).
const void* pipelinedAllgatherKernelPtr();
void launchPipelinedAllgather(const CommArgs& a, const void* in, void* out, const size_t* offs, const size_t* lens,
                              int onlyDst, const PeerPtrs& stage, int tileVecs, int exchangeThreads, int blocks,
                              cudaStream_t stream);
// reduce_scatter of plain pointers of any size: rank r's share is elemLen[r] elements at
// elemOff[r] of `in`; `out` receives my share, reduced over all ranks and scaled.
const void* pipelinedReduceScatterKernelFor(DataType dt, int nranks);
void launchPipelinedReduceScatter(const CommArgs& a, const void* in, void* out, const size_t* elemOff,
                                  const size_t* elemLen, DataType dt, ReduceOp op, float scale, const PeerPtrs& stage,
                                  int tileVecs, int exchangeThreads, int blocks, cudaStream_t stream);
// The cast forms of the two (docs/cuda.md, "Cast reduce-scatter / allgather"). reduce_scatter:
// 16-bit `in` (dt float16 / bfloat16), float32 `out`, SUM, accumulated, scaled and stored in fp32.
// allgather(v): float32 `in` rounded to outDt (float16 / bfloat16) in the copy-in stage; offs /
// lens in outDt bytes, so the slots and the pulls move outDt bytes only.
const void* castPipelinedReduceScatterKernelFor(DataType dt, int nranks);
void launchCastPipelinedReduceScatter(const CommArgs& a, const void* in, float* out, const size_t* elemOff,
                                      const size_t* elemLen, DataType dt, float scale, const PeerPtrs& stage,
                                      int tileVecs, int exchangeThreads, int blocks, cudaStream_t stream);
const void* castPipelinedAllgatherKernelFor(DataType outDt);
void launchCastPipelinedAllgather(const CommArgs& a, const void* in, void* out, DataType outDt, const size_t* offs,
                                  const size_t* lens, const PeerPtrs& stage, int tileVecs, int exchangeThreads,
                                  int blocks, cudaStream_t stream);
// reduce to `root` of plain pointers of any size: `count` elements cut into the shares of
// reduce_scatter (elemOff / elemLen); only the root writes `out` (null elsewhere is fine).
const void* pipelinedReduceKernelFor(DataType dt, int nranks);
void launchPipelinedReduce(const CommArgs& a, const void* in, void* out, const size_t* elemOff, const size_t* elemLen,
                           int root, DataType dt, ReduceOp op, const PeerPtrs& stage, int tileVecs, int exchangeThreads,
                           int blocks, cudaStream_t stream);
// alltoall(v) / scatter of plain pointers of any size: my block for rank j is sendLen[j] bytes at
// sendOff[j] of `in`; the block from rank q lands at recvOff[q] of `out` (recvLen[q] bytes). The
// lengths may differ between ranks: the kernel agrees on the step count on the device. Scatter:
// only the root sends, and every rank receives from the root only.
const void* pipelinedAlltoallKernelPtr();
void launchPipelinedAlltoall(const CommArgs& a, const void* in, void* out, const size_t* sendOff, const size_t* sendLen,
                             const size_t* recvOff, const size_t* recvLen, const PeerPtrs& stage, int tileVecs,
                             int exchangeThreads, int blocks, cudaStream_t stream);

// collective_kernels.cu -----------------------------------------------------------------------
void launchBroadcast(const CommArgs& a, const PeerPtrs& bufs, void* mc, size_t bytes, int root, int mode, bool vec,
                     int blocks, int tile, cudaStream_t stream);
void launchGatherPush(const CommArgs& a, const void* in, const PeerPtrs& outs, void* mcOut, const size_t* offs,
                      const size_t* lens, int onlyDst, bool vec, int blocks, cudaStream_t stream);
void launchAlltoallPush(const CommArgs& a, const void* in, const PeerPtrs& outs, const size_t* sendOff,
                        const size_t* sendLen, const size_t* dstOff, const size_t* recvOffTable, int onlySrc,
                        bool vec, int blocks, cudaStream_t stream);
void launchReducePull(const CommArgs& a, const PeerPtrs& ins, void* mcIn, void* out, const size_t* elemOff,
                      const size_t* elemLen, DataType dt, ReduceOp op, float scale, bool vec, bool useMc, int blocks,
                      cudaStream_t stream);
// The cast forms (docs/cuda.md, "Cast reduce-scatter / allgather"). Reduce-pull: 16-bit inputs
// (dt float16 / bfloat16), SUM, rank r's share accumulated in fp32, scaled and stored as float32
// to `out`. Gather push: float32 `in`, rounded once to outDt (float16 / bfloat16) on the source;
// offs / counts in outDt elements; `vec`: `in` and the outputs are 16-byte aligned.
void launchCastReducePull(const CommArgs& a, const PeerPtrs& ins, float* out, const size_t* elemOff,
                          const size_t* elemLen, DataType dt, float scale, bool vec, int blocks, cudaStream_t stream);
void launchCastGatherPush(const CommArgs& a, const void* in, const PeerPtrs& outs, DataType outDt, const size_t* offs,
                          const size_t* counts, bool vec, int blocks, cudaStream_t stream);
// One rank's form of both: out = outDt(float(in) * scale) for (float16 / bfloat16 -> float32) and
// (float32 -> float16 / bfloat16).
void launchCastScale(const void* in, DataType inDt, void* out, DataType outDt, size_t count, float scale, int blocks,
                     cudaStream_t stream);
const void* castReducePullKernelPtr(DataType dt, int nranks);
const void* castGatherPushKernelPtr(DataType outDt);
// Entry points, for occupancy queries (every CTA of a collective kernel must be resident).
const void* broadcastKernelPtr();
const void* gatherPushKernelPtr();
const void* alltoallPushKernelPtr();
const void* reducePullKernelPtr(DataType dt, int nranks);
// Flag-in-data exchange for small messages (no barrier): mode 0 = allgather (my block to
// everyone), 1 = alltoall (block j of my input to rank j). `bytes` per block, uniform.
void launchLLExchange(const CommArgs& a, const void* in, void* out, size_t bytes, int mode, const PeerPtrs& ll,
                      size_t srcStride, size_t parityStride, int blocks, int threads, cudaStream_t stream);

// moe_kernels.cu — device-split MoE exchange ----------------------------------------------------
// What every form shares. `peers.p[r]` (the launchers' `outs` / `srcs`) is rank r's output
// (dispatch) or expert_out (combine) in place, or its staging area when `plain` is set: my plain
// output `staged` is then copied out of my staging area after the last push (dispatch), or my
// plain expert_out into it before the first pull (combine).
struct MoeArgs {
  unsigned long long rowBytes;  // of an output row; quantising: H codes
  char* staged;                 // null = zero copy (or an empty plain output)
  InputStatus* status;          // host-mapped
  uint32_t capRows;             // rows this rank's output can hold
  int experts;
  int align;
  int plain;                    // the rows go through the staging areas: set even when `staged` is null
};
// The quantising dispatches' extension: each destination receives e4m3 codes and one fp32 scale
// per 128-element block, rank r's in `scales.p[r]` (rows x H / 128), or, when `plain` is set, in
// its staging area after capRows rows of codes; my plain out_scales `stagedScales` is copied from
// there like `staged`. Which of the two a destination uses follows `plain`, never these pointers:
// a plain tensor with no rows has a null data pointer.
struct MoeScales {
  PeerPtrs scales;      // zero copy only
  float* stagedScales;  // plain only (null if it is empty)
};
struct MoeQuantArgs : MoeArgs, MoeScales {};

// Device-split all-to-all-v: row counts come from device arrays (int64, P·E entries) and are
// exchanged inside the kernel; see moe_kernels.cu for the two layouts. `scales` set: the
// quantising forward form, `in` holding bf16 rows of rowBytes elements (a multiple of 128).
void launchAlltoallvDev(const CommArgs& a, const PeerPtrs& outs, const MoeArgs& d, const MoeScales* scales,
                        const void* in, size_t inRows, const long long* inSplits, const long long* inOffsets,
                        long long* outSplits, long long* outOffsets, bool inverse, int blocks, cudaStream_t stream);
// Top-k MoE combine, the mirror of the forward form: for each of `tokens` tokens, out row t =
// sum over j < topk with pos[t, j] >= 0, in order, of weights[t, j] * (row pos[t, j] of my dispatch
// input, as it lies on the rank holding its expert), in fp32, rounded to dt (float, bfloat16 or
// float16). `splits` is my dispatch in_splits.
// Null `weights`: every routed choice has weight 1 (the backward of the top-k dispatch).
void launchMoeCombineTopk(const CommArgs& a, const PeerPtrs& srcs, const MoeArgs& d, void* out, size_t tokens,
                          int topk, const long long* pos, const float* weights, const long long* splits, DataType dt,
                          int blocks, cudaStream_t stream);
// Its backward, run by the source with the combine's arguments and dy (tokens rows): for each routed
// choice, gradWeights[t, j] = <dy[t], its expert row> in fp32 (+0 where pos = -1), and
// round(weights[t, j] · dy[t]) pushed to the same row of the holder's grad_expert_out: `grads.p[r]`,
// or, when `plain` is set, rank r's staging area after its capRows rows of staged expert_out, copied
// out to my plain `stagedGrad` at the end. Each holder zeroes the rows of its grad_expert_out
// (capacityRows) outside its receive segments.
void launchMoeCombineTopkBackward(const CommArgs& a, const PeerPtrs& srcs, const PeerPtrs& grads, const MoeArgs& d,
                                  void* stagedGrad, size_t capacityRows, const void* dy, float* gradWeights,
                                  size_t tokens, int topk, const long long* pos, const float* weights,
                                  const long long* splits, DataType dt, int blocks, cudaStream_t stream);
// Top-k MoE dispatch: route x's `tokens` rows by `idx` ((tokens, topk) int64; entry j·E + e =
// local expert e of rank j, anything outside 0..P·E-1 is not routed) and push each to every
// choice. Writes `splits` (P·E) and `pos` (tokens, topk) as route() does; out, outSplits and
// outOffsets are those of the forward launchAlltoallvDev on route()'s rows. Rows are a multiple
// of 16 bytes, x 16-byte aligned. `scales` set: the quantising form, each token quantised once.
void launchMoeDispatchTopk(const CommArgs& a, const PeerPtrs& outs, const MoeArgs& d, const MoeScales* scales,
                           const void* x, size_t tokens, int topk, const long long* idx, long long* splits,
                           long long* pos, long long* outSplits, long long* outOffsets, int blocks, cudaStream_t stream);
// Low-latency top-k exchange for decoding: fixed per-(expert, source) slots instead of a layout agreed
// at a barrier. Every rank owns one buffer of the same layout (symmetric memory); offsets are bytes
// from its start, each a multiple of 16. See moe_kernels.cu for the protocol.
struct MoeLLLayout {
  unsigned long long rowBytes;         // a dispatch slot row: H elements, or H e4m3 codes (fp8)
  unsigned long long scaleBytes;       // its fp32 scales: H / 128 · 4 (fp8), else 0
  unsigned long long combineRowBytes;  // a combine slot row, and a row of y
  unsigned long long slots;            // E · P · maxTokens dispatch rows, [e][s][r]
  unsigned long long scales;           // their scales (fp8)
  unsigned long long tags;             // int32 t·k + j of each dispatch row
  unsigned long long dispatchSig;      // E · P 64-bit words, [e][s]
  unsigned long long combineSlots;     // maxTokens · topk combine rows, by t·k + j
  unsigned long long combineSig;       // P 64-bit words, [holder]
  unsigned long long choices;          // int32 per (t, j) of my last dispatch: routed and sent (>= 0) or -1
  unsigned long long ctrl;             // uint32 call count, uint32 completion ticket
  unsigned long long bytes;            // the whole buffer
  int experts, maxTokens, topk, fp8;
};
struct MoeLLArgs {
  PeerPtrs bufs;        // rank r's buffer
  MoeLLLayout l;
  InputStatus* status;  // host-mapped
};
// The signal word a rank stores for call `seq` (the buffer's call count + 1) of `form` with `count`
// rows; exposed for the loopback self-test, which stands in for the virtual peers.
enum MoeLLForm : uint32_t { kMoeLLDispatch = 1, kMoeLLDispatchFp8 = 2, kMoeLLCombine = 3 };
unsigned long long moeLLSignal(uint32_t seq, uint32_t form, uint32_t count);
// Low-latency dispatch: route x's `tokens` rows by idx ((tokens, topk) int64) and push each routed
// choice to slot (e, me, r) of rank j, r its rank in its group in (token, choice) order; then receive
// and pack expert e's rows into out[e, 0 : n] (out: E · P · maxTokens rows of rowBytes, plain), in
// source order, writing outSplits[e·P + s] (int64). fp8: x is bf16, out holds codes and outScales
// the fp32 scales.
void launchMoeLLDispatch(const CommArgs& a, const MoeLLArgs& L, const void* x, size_t tokens, const long long* idx,
                         void* out, float* outScales, long long* outSplits, int blocks, cudaStream_t stream);
// Low-latency combine: every packed row of my experts (expertOut, the dispatch's out layout, dt)
// goes back to its source's combine slot; then y[t] = round(sum over my routed, sent choices j of
// weights[t, j] · float(row)), as launchMoeCombineTopk (null weights: 1).
void launchMoeLLCombine(const CommArgs& a, const MoeLLArgs& L, const void* expertOut, const float* weights, void* y,
                        size_t tokens, DataType dt, int blocks, cudaStream_t stream);
const void* moeLLDispatchKernelPtr(bool fp8);
const void* moeLLCombineKernelPtr(DataType dt);
const void* alltoallvDevKernelPtr(bool fp8 = false);
const void* moeCombineTopkKernelPtr(DataType dt);
const void* moeCombineTopkBackwardKernelPtr(DataType dt);
const void* moeDispatchTopkKernelPtr(bool fp8);

// p2p_kernels.cu — point-to-point between two ranks through the receiver's mailbox ring.
// sendBytes == 0 / recvBytes == 0 disables that role; both set = fused send+recv (one launch).
void launchP2p(const CommArgs& a, const void* sendPtr, size_t sendBytes, int dst, void* recvPtr, size_t recvBytes,
               int src, const PeerPtrs& mailbox, size_t boxStride, size_t slotBytes, int nslots, int lanes,
               cudaStream_t stream);
// One-sided copy between my memory and a peer-mapped pointer (put / get), whole grid.
// tma: stream through shared memory with cp.async.bulk (one issuing thread per CTA) when the
// pointers are 16-byte aligned; LDG/STG otherwise.
void launchPeerCopy(void* dst, const void* src, size_t bytes, int blocks, cudaStream_t stream, bool tma = false);
// Zero-copy neighbour exchange: write `sendBytes` straight into `remote` (the peer mapping of
// dst's receive buffer) once dst has signalled ready, and wait for src's data to have landed in
// my own buffer. `blocks` must be the same on both ends of a transfer.
void launchExchange(const CommArgs& a, const void* sendPtr, size_t sendBytes, int dst, void* remote, size_t recvBytes,
                    int src, int blocks, bool tma, cudaStream_t stream);

// reduce_kernels.cu — local element-wise ops: dst = dst (op) src, and
// multi-source reduce / broadcast between buffers visible to one device.
void launchLocalReduce(void* dst, const void* src, size_t count, DataType dt, ReduceOp op, cudaStream_t stream);
void launchLocalReduceMany(void* dst, const void* const* srcs, int nsrc, size_t count, DataType dt, ReduceOp op,
                           cudaStream_t stream);
void launchLocalBroadcast(void* const* dsts, int ndst, const void* src, size_t bytes, cudaStream_t stream);
// Every buffer := scale * reduce(all buffers) in one pass (fused reduce + broadcast).
// tileCounter: a device word on the launching device that is zero when the launch runs; the
// bulk-copy kernel hands out its tiles through it and leaves it zero again. Launches that share
// a counter must run one after the other on the device (one stream, or ordered by events).
void launchLocalAllreduceMany(void* const* bufs, int n, size_t count, DataType dt, ReduceOp op, float scale,
                              unsigned int* tileCounter, cudaStream_t stream);
// Owns a zeroed tile counter for launchLocalAllreduceMany on `device`.
class TileCounter {
 public:
  explicit TileCounter(int device);
  ~TileCounter();
  TileCounter(const TileCounter&) = delete;
  TileCounter& operator=(const TileCounter&) = delete;
  unsigned int* get() const { return p_; }

 private:
  unsigned int* p_ = nullptr;
};
// Whether launchLocalAllreduceMany runs the TMA bulk-copy kernel for these arguments (at least
// 1 MB per buffer, every pointer 16-byte aligned, n small enough for its shared-memory stages)
// rather than the LDG/STG kernel. An explicit setLocalAllreduceShape() overrides it.
bool localAllreduceUsesBulk(void* const* bufs, int n, size_t count, DataType dt);
void launchFill(void* dst, size_t count, DataType dt, double start, double stride, cudaStream_t stream);
// Device-side check of buf[i] == start + stride*i; deviceResult = {mismatch count, min(bad index + 1)}
// (initialise to {0, ~0ull}).
void launchVerify(const void* buf, size_t count, DataType dt, double start, double stride, double rtol, double atol,
                  unsigned long long* deviceResult, cudaStream_t stream);
void launchSpin(long long cycles, cudaStream_t stream);
// Launch shape of the single-rank fused step's LDG/STG kernel (localAllreduceManyKernel): CTAs
// per SM, packs per thread and trip, contiguous tile per CTA or grid stride. Setting a shape
// (here or through GLB_LOCAL_SHAPE) makes every call run that kernel with it, to measure or test
// it; ctasPerSm = 0 restores the default shape and the choice by size and alignment.
void setLocalAllreduceShape(int ctasPerSm, int unroll, bool tiled);

}  // namespace cuda
}  // namespace glb
