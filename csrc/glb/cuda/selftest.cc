// Single-GPU, single-process self-test of the collective kernels ("virtual-rank loopback").
//
// Nsight Compute serialises kernels, so two ranks whose kernels wait for each other can
// never be profiled together — and a box with one GPU cannot host two real ranks at full
// speed. PeerContext::loopbackComm(P) builds kernel arguments with which ONE launch plays
// rank 0 of P ranks (the flags it posts for its peers are the ones it waits for); the
// "peer" buffers are P distinct local allocations. Every hot kernel — including the
// P = 2 / 4 / 8 specialisations and, where the driver allows a one-device multicast object,
// the multimem (NVLS) kernels — runs exactly the code it runs across GPUs, and rank 0's
// part of the result has a closed form that is checked here on the host.
#include "glb/cuda/selftest.h"

#include <cmath>
#include <cstring>
#include <numeric>
#include <sstream>

#include "glb/common/utils.h"
#include "glb/cuda/collectives.h"
#include "glb/cuda/kernels.h"
#include "glb/cuda/local_ops.h"
#include "glb/cuda/schedules.h"

namespace glb {
namespace cuda {

namespace {

struct DevBuf {
  void* p = nullptr;
  size_t bytes = 0;
  explicit DevBuf(size_t n) : bytes(n) { GLB_CUDA_CHECK(cudaMalloc(&p, std::max<size_t>(n, 16))); }
  ~DevBuf() { cudaFree(p); }
  DevBuf(const DevBuf&) = delete;
};

MoeArgs moeArgs(size_t rowBytes, size_t cap, int experts, int align, InputStatus* status) {
  MoeArgs d{};
  d.rowBytes = rowBytes;
  d.status = status;
  d.capRows = static_cast<uint32_t>(cap);
  d.experts = experts;
  d.align = align;
  return d;
}

void shareOfHost(size_t n, int parts, int r, size_t& b, size_t& e) {
  const size_t base = n / parts, rem = n % parts;
  b = r * base + std::min<size_t>(r, rem);
  e = b + base + (static_cast<size_t>(r) < rem ? 1 : 0);
}

std::vector<float> download(const void* dev, size_t count, cudaStream_t s) {
  std::vector<float> h(count);
  GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), dev, count * 4, cudaMemcpyDeviceToHost, s));
  GLB_CUDA_CHECK(cudaStreamSynchronize(s));
  return h;
}

bool close(float a, double want) { return std::fabs(static_cast<double>(a) - want) <= 1e-5 * std::fabs(want) + 1e-6; }

float bf16ToFloat(uint16_t h) {
  uint32_t w = static_cast<uint32_t>(h) << 16;
  float f;
  std::memcpy(&f, &w, 4);
  return f;
}

// Round to nearest even (finite, non-NaN x).
uint16_t floatToBf16(float x) {
  uint32_t w;
  std::memcpy(&w, &x, 4);
  return static_cast<uint16_t>((w + 0x7fffu + ((w >> 16) & 1u)) >> 16);
}

// Fused allreduce + residual + norm in loopback: rank 0's partial row i, element j is 1 + i * H + j,
// the residual 0.5 * (i * H + j), the bias j, gamma 1 + j / H and beta -j / H, all exact in fp32.
// Every virtual peer's partial is rank 0's (their staging aliases mine), so row i reduces to
// P * partial + bias + residual. Checks row i of residual_out (r) and, with a norm, out (o).
std::string checkNormRow(const float* r, const float* o, size_t i, int P, size_t H, int norm) {
  std::vector<double> v(H);
  double mean = 0, sq = 0;
  for (size_t j = 0; j < H; j++) {
    const double e = static_cast<double>(i * H + j);
    v[j] = P * (1.0 + e) + 0.5 * e + static_cast<double>(j);
    if (r[j] != static_cast<float>(v[j])) return strcat_all("residual_out[", i, ", ", j, "]: got ", r[j], " want ", v[j]);
    mean += v[j] / H;
  }
  if (norm == kNormNone) return "";
  for (size_t j = 0; j < H; j++) sq += (norm == kNormLayer ? (v[j] - mean) * (v[j] - mean) : v[j] * v[j]) / H;
  for (size_t j = 0; j < H; j++) {
    const double g = 1.0 + static_cast<double>(j) / H, b = -static_cast<double>(j) / H;
    const double want = norm == kNormLayer ? (v[j] - mean) / std::sqrt(sq + 1e-5) * g + b : v[j] / std::sqrt(sq + 1e-5) * g;
    if (std::fabs(o[j] - want) > 1e-5 * std::fabs(want) + 1e-5) return strcat_all("out[", i, ", ", j, "]: got ", o[j], " want ", want);
  }
  return "";
}

// The arguments of checkNormRow's problem over buffers of `rows` rows of H floats.
NormArgs fillNormProblem(const DevBuf& partial, const DevBuf& residual, const DevBuf& resOut, const DevBuf& out,
                         const DevBuf& vec, size_t partialRows, size_t rows, size_t H, cudaStream_t s) {
  launchFill(partial.p, partialRows * H, DataType::FLOAT32, 1.0, 1.0, s);
  launchFill(residual.p, rows * H, DataType::FLOAT32, 0.0, 0.5, s);
  launchFill(vec.p, H, DataType::FLOAT32, 0.0, 1.0, s);
  launchFill(static_cast<float*>(vec.p) + H, H, DataType::FLOAT32, 1.0, 1.0 / H, s);
  launchFill(static_cast<float*>(vec.p) + 2 * H, H, DataType::FLOAT32, 0.0, -1.0 / H, s);
  NormArgs a;
  a.partial = partial.p;
  a.residual = residual.p;
  a.residualOut = resOut.p;
  a.out = out.p;
  a.bias = vec.p;
  a.gamma = static_cast<float*>(vec.p) + H;
  a.beta = static_cast<float*>(vec.p) + 2 * H;
  a.rows = rows;
  a.hidden = H;
  a.eps = 1e-5f;
  return a;
}

// `rows` says which rows rank 0 computes (the two-shot: its share).
std::string checkAllreduceNorm(const CommArgs& ca, const NormXchg& x, int variant, int norm, size_t rows, size_t H,
                               size_t rowsBegin, size_t rowsEnd, int blocks, cudaStream_t s) {
  DevBuf partial(rows * H * 4), residual(rows * H * 4), resOut(rows * H * 4), out(rows * H * 4), vec(3 * H * 4);
  const NormArgs a = fillNormProblem(partial, residual, resOut, out, vec, rows, rows, H, s);
  launchAllreduceNorm(ca, a, x, DataType::FLOAT32, norm, variant, blocks, s);
  noteLaunch();
  auto r = download(resOut.p, rows * H, s);
  auto o = download(out.p, rows * H, s);
  for (size_t i = rowsBegin; i < rowsEnd; i++) {
    std::string why = checkNormRow(&r[i * H], &o[i * H], i, ca.nranks, H, norm);
    if (!why.empty()) return why;
  }
  return "";
}

// The reduce-scatter form as one chunk of `rows` rows of shards of x.shardRows rows: rank 0 owns the
// chunk's rows of shard 0, and a gathered out holds them at the same rows (the other shards come
// from virtual peers that do not run).
std::string checkScatterNorm(const CommArgs& ca, const NormXchg& x, int norm, size_t rows, size_t H, int blocks,
                             cudaStream_t s) {
  const size_t all = ca.nranks * x.shardRows, outRows = x.gather ? all : rows;
  DevBuf partial(all * H * 4), residual(rows * H * 4), resOut(rows * H * 4), out(outRows * H * 4), vec(3 * H * 4);
  const NormArgs a = fillNormProblem(partial, residual, resOut, out, vec, all, rows, H, s);
  launchAllreduceNorm(ca, a, x, DataType::FLOAT32, norm, kNormScatter, blocks, s);
  noteLaunch();
  auto r = download(resOut.p, rows * H, s);
  auto o = download(out.p, outRows * H, s);
  for (size_t i = 0; i < rows; i++) {
    std::string why = checkNormRow(&r[i * H], &o[i * H], i, ca.nranks, H, norm);
    if (!why.empty()) return why;
  }
  return "";
}

// The backward of the reduce-scatter norm as one chunk of `rows` rows (shards of x.shardRows rows;
// kNormLocal: the one rank's rows): s[i, j] = 1 + i + j / H, grad_out 0.5 - k / (4 H) at flat index
// k, grad_s 0.25 + k / (2 H), gamma 1 + j / H, all exact in fp32. Rank 0 owns the chunk's rows of
// shard 0; with a gather its virtual peers staged the same grad_out rows, so g = P grad_out. Checks
// grad_residual, rank 0's rows of grad_partial and the weight, norm bias and bias column sums
// against a CPU double-precision row.
// The allreduce forms (kNormOneShot / kNormTwoShot) take `rows` rows of every tensor, and their
// virtual peers staged the same grad_out, so g = P grad_out; they write grad_partial only. The
// one-shot computes every row and sums; the two-shot rank 0's share of the rows, and its collective
// finish sums P staged copies of rank 0's column sums.
std::string checkNormBackward(const CommArgs& ca, const NormXchg& x, int variant, int norm, size_t rows, size_t H,
                              int blocks, cudaStream_t st) {
  const bool scatter = variant == kNormScatter, tp = variant == kNormOneShot || variant == kNormTwoShot;
  const size_t all = scatter ? ca.nranks * x.shardRows : rows, outRows = scatter && x.gather ? all : rows;
  const int vectors = norm == kNormLayer ? 3 : 2;
  DevBuf gradOut(outRows * H * 4), sv(rows * H * 4), gs(rows * H * 4), gr(rows * H * 4), gp(all * H * 4),
      gamma(H * 4), vecs(3 * H * 4), ws(static_cast<size_t>(blocks) * vectors * H * 4);
  launchFill(gradOut.p, outRows * H, DataType::FLOAT32, 0.5, -0.25 / H, st);
  launchFill(sv.p, rows * H, DataType::FLOAT32, 1.0, 1.0 / H, st);
  launchFill(gs.p, rows * H, DataType::FLOAT32, 0.25, 0.5 / H, st);
  launchFill(gamma.p, H, DataType::FLOAT32, 1.0, 1.0 / H, st);
  NormBwdArgs a;
  a.gradOut = gradOut.p;
  a.s = sv.p;
  a.gradS = gs.p;
  a.gradResidual = tp ? nullptr : gr.p;
  a.gradPartial = gp.p;
  a.gamma = gamma.p;
  a.ws = static_cast<float*>(ws.p);
  a.rows = rows;
  a.hidden = H;
  a.eps = 1e-5f;
  a.vectors = vectors;
  a.vecWeight = 0;
  a.vecNormBias = norm == kNormLayer ? 1 : -1;
  a.vecBias = vectors - 1;
  a.first = 1;
  launchNormBackward(ca, a, x, DataType::FLOAT32, norm, variant, blocks, st);
  float* v = static_cast<float*>(vecs.p);
  void* const outs[3] = {v, norm == kNormLayer ? v + H : nullptr, v + 2 * H};
  void* const packed[3] = {outs[0], outs[1] != nullptr ? outs[1] : outs[2], outs[1] != nullptr ? outs[2] : nullptr};
  if (variant == kNormTwoShot) {
    launchNormBackwardFinishAllreduce(ca, a.ws, blocks, vectors, H, packed, x.peers, DataType::FLOAT32, 2, st);
  } else {
    launchNormBackwardFinish(a.ws, blocks, vectors, H, packed, DataType::FLOAT32, st);
  }
  noteLaunch(2);
  const auto p = download(gp.p, all * H, st), go = download(gradOut.p, outRows * H, st);
  const auto r = tp ? p : download(gr.p, rows * H, st);
  const auto vw = download(v, H, st), vnb = download(v + H, H, st), vb = download(v + 2 * H, H, st);
  const double mult = (scatter && x.gather) || tp ? ca.nranks : 1;
  const double vmult = variant == kNormTwoShot ? ca.nranks : 1;
  size_t rb = 0, re = rows;
  if (variant == kNormTwoShot) shareOfHost(rows, ca.nranks, 0, rb, re);
  std::vector<double> sw(H, 0), snb(H, 0), sb(H, 0), aw(H, 0), anb(H, 0), ab(H, 0);
  for (size_t i = rb; i < re; i++) {
    std::vector<double> xs(H), g(H);
    double mean = 0, sq = 0, mg = 0, mgx = 0, scale = 0;
    for (size_t j = 0; j < H; j++) {
      xs[j] = 1.0 + static_cast<double>(i) + static_cast<double>(j) / H;
      g[j] = mult * go[i * H + j];
      mean += xs[j] / H;
    }
    if (norm == kNormRms) mean = 0;
    for (size_t j = 0; j < H; j++) sq += (xs[j] - mean) * (xs[j] - mean) / H;
    const double rinv = 1.0 / std::sqrt(sq + 1e-5);
    for (size_t j = 0; j < H; j++) {
      xs[j] = (xs[j] - mean) * rinv;
      const double gg = g[j] * (1.0 + static_cast<double>(j) / H);
      mg += gg / H;
      mgx += gg * xs[j] / H;
      sw[j] += g[j] * xs[j];
      snb[j] += g[j];
      aw[j] += std::fabs(g[j] * xs[j]);
      anb[j] += std::fabs(g[j]);
    }
    if (norm == kNormRms) mg = 0;
    std::vector<double> want(H);
    for (size_t j = 0; j < H; j++) {
      const double gg = g[j] * (1.0 + static_cast<double>(j) / H);
      want[j] = 0.25 + static_cast<double>(i * H + j) * 0.5 / H + rinv * (gg - mg - xs[j] * mgx);
      scale = std::max(scale, std::fabs(want[j]));
    }
    for (size_t j = 0; j < H; j++) {
      if (std::fabs(r[i * H + j] - want[j]) > 1e-4 * scale + 1e-6) {
        return strcat_all("grad_residual[", i, ", ", j, "]: got ", r[i * H + j], " want ", want[j]);
      }
      if (p[i * H + j] != r[i * H + j]) return strcat_all("grad_partial[", i, ", ", j, "] differs from grad_residual");
      sb[j] += r[i * H + j];
      ab[j] += std::fabs(r[i * H + j]);
    }
  }
  for (auto* acc : {&sw, &snb, &sb, &aw, &anb, &ab}) {
    for (double& e : *acc) e *= vmult;
  }
  for (size_t j = 0; j < H; j++) {
    if (std::fabs(vw[j] - sw[j]) > 1e-4 * aw[j] + 1e-6) return strcat_all("grad_weight[", j, "]: got ", vw[j], " want ", sw[j]);
    if (norm == kNormLayer && std::fabs(vnb[j] - snb[j]) > 1e-4 * anb[j] + 1e-6) {
      return strcat_all("grad_norm_bias[", j, "]: got ", vnb[j], " want ", snb[j]);
    }
    if (std::fabs(vb[j] - sb[j]) > 1e-5 * ab[j] + 1e-6) return strcat_all("grad_bias[", j, "]: got ", vb[j], " want ", sb[j]);
  }
  return "";
}

class Runner {
 public:
  Runner(PeerContext& pc, cudaStream_t s) : pc_(pc), s_(s) {}
  std::vector<SelfTestResult> results;

  template <typename F>
  void run(const std::string& name, F&& body) {
    SelfTestResult r;
    r.name = name;
    try {
      std::string why = body();
      GLB_CUDA_CHECK(cudaStreamSynchronize(s_));
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) why = cudaGetErrorString(e);
      r.ok = why.empty();
      r.detail = why;
    } catch (const std::exception& e) {
      r.ok = false;
      r.detail = e.what();
    }
    if (r.detail.rfind("skipped", 0) == 0) {
      r.ok = true;
      r.skipped = true;
    }
    results.push_back(r);
  }

 private:
  PeerContext& pc_;
  cudaStream_t s_;
};

}  // namespace

std::vector<SelfTestResult> loopbackSelfTest(PeerContext& pc, cudaStream_t stream, size_t count) {
  GLB_ENFORCE(count >= 4096, "loopbackSelfTest: count too small");
  DeviceGuard g(pc.device);
  pc.checkHealth();
  GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
  Runner R(pc, stream);
  const int dtF = static_cast<int>(DataType::FLOAT32);
  (void)dtF;
  const size_t n = count / 4 * 4 + 3;  // not a multiple of the pack width: exercises the tails
  const PeerPtrs poolStage = pc.stagePtrs(0);
  char* myStage = static_cast<char*>(poolStage.p[pc.rank]);
  const size_t half = std::min<size_t>(roundUp(std::max<size_t>(tuning().oneShotMaxBytes, 4096), 4096), pc.stageBytes() / 4);

  for (int P : {2, 4, 8}) {
    const CommArgs ca = pc.loopbackComm(P);
    std::vector<std::unique_ptr<DevBuf>> bufs;
    PeerPtrs pp;
    std::memset(&pp, 0, sizeof(pp));
    for (int r = 0; r < P; r++) {
      bufs.emplace_back(new DevBuf(n * 4));
      pp.p[r] = bufs[r]->p;
    }
    auto fillAll = [&] {
      for (int r = 0; r < P; r++) launchFill(pp.p[r], n, DataType::FLOAT32, r, P, stream);  // value = i*P + r
    };
    const double tri = P * (P - 1) / 2.0;
    const size_t nvec = n / 4;
    size_t vb, ve;
    shareOfHost(nvec, P, 0, vb, ve);
    size_t tb, te;
    shareOfHost(n - nvec * 4, P, 0, tb, te);

    // ---- two-shot, every unroll of this P ------------------------------------------------
    for (int unroll : {1, 2, 4, 8}) {
      if ((P == 2 && unroll == 1) || (P == 4 && unroll == 8) || (P == 8 && unroll > 2)) continue;
      R.run(strcat_all("twoShotAllreduceKernel<float,", P, ",", unroll, ">"), [&]() -> std::string {
        fillAll();
        LaunchCfg cfg;
        cfg.blocks = std::min(pc.coResidentBlocks(twoShotKernelFor(DataType::FLOAT32, P, unroll)), 32);
        cfg.unroll = unroll;
        launchTwoShotAllreduce(ca, pp, n, DataType::FLOAT32, ReduceOp::SUM, 0.5f, true, LocalPtrs(), cfg, stream);
        noteLaunch();
        auto last = download(pp.p[P - 1], n, stream);
        for (size_t i = 0; i < n; i++) {
          const bool mine = (i / 4 >= vb && i / 4 < ve && i < nvec * 4) || (i >= nvec * 4 + tb && i < nvec * 4 + te);
          const double want = mine ? 0.5 * (static_cast<double>(i) * P * P + tri) : static_cast<double>(i) * P + (P - 1);
          if (!close(last[i], want)) return strcat_all("element ", i, ": got ", last[i], " want ", want);
        }
        return "";
      });
    }

    // ---- two-shot on e4m3 (16 lanes per pack, fp32 accumulate, one saturating rounding) ------
    if (P == 4) {
      R.run("twoShotAllreduceKernel<e4m3,4>", [&]() -> std::string {
        for (int r = 0; r < P; r++) launchFill(pp.p[r], n, DataType::FLOAT8_E4M3, r + 1, 0.0, stream);
        LaunchCfg cfg;
        cfg.blocks = std::min(pc.coResidentBlocks(twoShotKernelFor(DataType::FLOAT8_E4M3, P, 2)), 32);
        cfg.unroll = 2;
        launchTwoShotAllreduce(ca, pp, n, DataType::FLOAT8_E4M3, ReduceOp::SUM, 0.5f, true, LocalPtrs(), cfg, stream);
        noteLaunch();
        std::vector<uint8_t> h(n);
        GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), pp.p[P - 1], n, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        const size_t nv8 = n / 16;
        size_t b8, e8, t8b, t8e;
        shareOfHost(nv8, P, 0, b8, e8);
        shareOfHost(n - nv8 * 16, P, 0, t8b, t8e);
        for (size_t i = 0; i < n; i++) {
          const bool mine = (i / 16 >= b8 && i / 16 < e8 && i < nv8 * 16) || (i >= nv8 * 16 + t8b && i < nv8 * 16 + t8e);
          const float want = mine ? 5.0f : static_cast<float>(P);  // 0.5 * (1 + 2 + 3 + 4), else rank P-1's input
          const float got = float8_e4m3::toFloat(h[i]);
          if (got != want) return strcat_all("element ", i, ": got ", got, " want ", want);
        }
        return "";
      });
    }

    // ---- reduce-scatter / reduce pull -----------------------------------------------------
    R.run(strcat_all("reducePullKernel<float,", P, ">"), [&]() -> std::string {
      fillAll();
      std::vector<size_t> off(P + 1, 0), len(P, 0);
      for (int r = 0; r < P; r++) {
        len[r] = n / P + (static_cast<size_t>(r) < n % P ? 1 : 0);
        off[r + 1] = off[r] + len[r];
      }
      DevBuf out(len[0] * 4);
      launchReducePull(ca, pp, nullptr, out.p, off.data(), len.data(), DataType::FLOAT32, ReduceOp::SUM, 1.0f, true, false,
                       std::min(pc.maxBlocks(), 16), stream);
      noteLaunch();
      auto h = download(out.p, len[0], stream);
      for (size_t i = 0; i < len[0]; i++) {
        if (!close(h[i], static_cast<double>(i) * P * P + tri)) return strcat_all("element ", i, ": got ", h[i]);
      }
      return "";
    });

    // ---- cast reduce-scatter (16-bit in, f32 out): peer 0 holds 256, the others 1, so the share
    // sums to 256 + P - 1, which fp32 holds and bf16 / f16 (P = 4: 259 needs 9 bits) would round.
    R.run(strcat_all("castReducePullKernel<", P == 4 ? "f16," : "bf16,", P, ">"), [&]() -> std::string {
      const DataType dt = P == 4 ? DataType::FLOAT16 : DataType::BFLOAT16;
      for (int r = 0; r < P; r++) launchFill(pp.p[r], n, dt, r == 0 ? 256.0 : 1.0, 0.0, stream);
      std::vector<size_t> off(P + 1, 0), len(P, 0);
      for (int r = 0; r < P; r++) {
        len[r] = n / P + (static_cast<size_t>(r) < n % P ? 1 : 0);
        off[r + 1] = off[r] + len[r];
      }
      DevBuf out(len[0] * 4);
      launchCastReducePull(ca, pp, static_cast<float*>(out.p), off.data(), len.data(), dt, 0.5f, true,
                           std::min(pc.maxBlocks(), 16), stream);
      noteLaunch();
      auto h = download(out.p, len[0], stream);
      const float want = 0.5f * static_cast<float>(256 + P - 1);
      for (size_t i = 0; i < len[0]; i++) {
        if (h[i] != want) return strcat_all("element ", i, ": got ", h[i], " want ", want);
      }
      return "";
    });

    // ---- cast epilogue (f32 in, bf16 out) -----------------------------------------------------
    R.run(strcat_all("castAllreduceKernel<float,bf16> P=", P), [&]() -> std::string {
      for (int r = 0; r < P; r++) launchFill(pp.p[r], n, DataType::FLOAT32, r % 3, 0.0, stream);  // small exact values
      std::vector<std::unique_ptr<DevBuf>> outs;
      PeerPtrs po;
      std::memset(&po, 0, sizeof(po));
      for (int r = 0; r < P; r++) {
        outs.emplace_back(new DevBuf(n * 2));
        GLB_CUDA_CHECK(cudaMemsetAsync(outs[r]->p, 0, n * 2, stream));
        po.p[r] = outs[r]->p;
      }
      launchCastAllreduce(ca, pp, nullptr, po, n, DataType::FLOAT32, DataType::BFLOAT16, ReduceOp::SUM, 2.0f, true,
                          std::min(pc.maxBlocks(), 16), stream);
      noteLaunch();
      std::vector<uint16_t> h(n);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), po.p[P - 1], n * 2, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      double sum = 0;
      for (int r = 0; r < P; r++) sum += r % 3;
      size_t ib, ie, xb, xe;
      shareOfHost(n / 8, P, 0, ib, ie);
      shareOfHost(n - n / 8 * 8, P, 0, xb, xe);
      for (size_t i = 0; i < n; i++) {
        const bool mine = (i / 8 >= ib && i / 8 < ie && i < n / 8 * 8) || (i >= n / 8 * 8 + xb && i < n / 8 * 8 + xe);
        const double want = mine ? 2.0 * sum : 0.0;
        if (std::fabs(bf16ToFloat(h[i]) - want) > 1e-2 * std::fabs(want) + 1e-6) {
          return strcat_all("element ", i, ": got ", bf16ToFloat(h[i]), " want ", want);
        }
      }
      return "";
    });

    // ---- one-shot (pull + push) through the pool; every virtual peer aliases my pool --------
    R.run(strcat_all("oneShotAllreduceKernel<float> P=", P), [&]() -> std::string {
      const size_t m = std::min<size_t>(n, half / 4 / P) / 4 * 4 - 1;
      PeerPtrs alias;
      std::memset(&alias, 0, sizeof(alias));
      for (int r = 0; r < P; r++) alias.p[r] = myStage;
      GLB_CUDA_CHECK(cudaMemsetAsync(myStage, 0, 2 * half, stream));
      launchFill(pp.p[0], m, DataType::FLOAT32, 1.0, 1.0, stream);
      setOneShotPush(false);
      launchOneShotAllreduce(ca, pp.p[0], pp.p[1], m, DataType::FLOAT32, ReduceOp::SUM, 1.0f, alias, half, LocalPtrs(), 2, stream);
      noteLaunch();
      auto pull = download(pp.p[1], m, stream);  // P reads of my own staged copy
      setOneShotPush(true);
      GLB_CUDA_CHECK(cudaMemsetAsync(myStage, 0, 2 * half, stream));
      launchOneShotAllreduce(ca, pp.p[0], pp.p[1], m, DataType::FLOAT32, ReduceOp::SUM, 1.0f, alias, half, LocalPtrs(), 2, stream);
      noteLaunch();
      auto push = download(pp.p[1], m, stream);  // slot 0 holds my data, the other slots are zero
      for (size_t i = 0; i < m; i++) {
        if (!close(pull[i], P * (1.0 + i))) return strcat_all("pull: element ", i, ": got ", pull[i]);
        if (!close(push[i], 1.0 + i)) return strcat_all("push: element ", i, ": got ", push[i]);
      }
      return "";
    });

    // ---- allreduce + residual + norm: LL, one-shot and row-sharded two-shot ----------------------
    {
      const size_t rows = 5, H = 1024;  // 20 KB: one LL slot of every virtual peer holds it at P = 8
      const char* norms[] = {"none", "rms", "layer"};
      for (int variant : {kNormLL, kNormOneShot, kNormTwoShot}) {
        for (int norm : {kNormNone, kNormRms, kNormLayer}) {
          R.run(strcat_all("allreduceNormKernel<float,", norms[norm], ",", normVariantName(variant), "> P=", P),
                [&]() -> std::string {
            NormXchg x{};
            size_t rb = 0, re = rows;
            if (variant == kNormLL) {
              // Virtual peer r's region is mine shifted by r source slots: my store for "peer r" lands
              // in the slot I poll for rank r. The slots shrink to fit P of them in my region.
              const size_t region = pc.llParityStride() * 2;
              x.srcStride = region / 2 / P / 16 * 16;
              x.parityStride = x.srcStride * P;
              if (rows * H * 4 * 2 > x.srcStride) return "skipped: LL region too small";
              char* myLL = static_cast<char*>(pc.llPtrs().p[pc.rank]);
              for (int r = 0; r < P; r++) x.peers.p[r] = myLL + r * x.srcStride;
            } else if (variant == kNormOneShot) {
              for (int r = 0; r < P; r++) x.peers.p[r] = myStage;
              x.parityStride = half;
            } else {
              for (int r = 0; r < P; r++) x.peers.p[r] = myStage + 2 * half;
              shareOfHost(rows, P, 0, rb, re);
            }
            x.mine = x.peers.p[0];
            return checkAllreduceNorm(ca, x, variant, norm, rows, H, rb, re, 3, stream);
          });
        }
      }
      // the reduce-scatter form: a chunk of 3 rows of shards of 5, out gathered or not
      for (int gather : {0, 1}) {
        for (int norm : {kNormNone, kNormRms, kNormLayer}) {
          R.run(strcat_all("allreduceNormKernel<float,", norms[norm], ",reduce_scatter> P=", P, gather ? " gather" : ""),
                [&]() -> std::string {
            NormXchg x{};
            for (int r = 0; r < P; r++) x.peers.p[r] = myStage + 2 * half;
            x.mine = x.peers.p[0];
            x.shardRows = 5;
            x.gather = gather;
            return checkScatterNorm(ca, x, norm, 3, H, 3, stream);
          });
        }
      }
      // its backward: the same chunk, grad_out gathered or not, and the one-rank form
      for (int gather : {0, 1}) {
        for (int norm : {kNormRms, kNormLayer}) {
          R.run(strcat_all("normBackwardKernel<float,", norms[norm], ",reduce_scatter> P=", P, gather ? " gather" : ""),
                [&]() -> std::string {
            NormXchg x{};
            for (int r = 0; r < P; r++) x.peers.p[r] = myStage + 2 * half;
            x.mine = x.peers.p[0];
            x.shardRows = 5;
            x.gather = gather;
            return checkNormBackward(ca, x, kNormScatter, norm, 3, H, 3, stream);
          });
        }
      }
      // the allreduce form's backward (tensor parallelism): one-shot and row-sharded two-shot
      for (int variant : {kNormOneShot, kNormTwoShot}) {
        for (int norm : {kNormRms, kNormLayer}) {
          R.run(strcat_all("normBackwardKernel<float,", norms[norm], ",", normVariantName(variant), "> P=", P),
                [&]() -> std::string {
            NormXchg x{};
            for (int r = 0; r < P; r++) x.peers.p[r] = myStage + (variant == kNormOneShot ? 0 : 2 * half);
            x.mine = x.peers.p[0];
            x.parityStride = half;
            return checkNormBackward(ca, x, variant, norm, rows, H, 3, stream);
          });
        }
      }
      if (P == 2) {
        for (int norm : {kNormRms, kNormLayer}) {
          R.run(strcat_all("normBackwardKernel<float,", norms[norm], ",local>"), [&]() -> std::string {
            return checkNormBackward(ca, NormXchg{}, kNormLocal, norm, 5, H, 3, stream);
          });
        }
      }
    }

    // ---- data movement ---------------------------------------------------------------------
    R.run(strcat_all("broadcastKernel(direct) P=", P), [&]() -> std::string {
      fillAll();
      launchBroadcast(ca, pp, nullptr, n * 4, 0, 0, true, std::min(2 * pc.maxBlocks(), 32), 0, stream);
      noteLaunch();
      auto h = download(pp.p[P - 1], n, stream);
      for (size_t i = 0; i < n; i++) {
        if (!close(h[i], static_cast<double>(i) * P)) return strcat_all("element ", i, ": got ", h[i]);
      }
      return "";
    });
    R.run(strcat_all("gatherPushKernel(allgather) P=", P), [&]() -> std::string {
      const size_t per = n / P;
      std::vector<size_t> off(P), len(P, per * 4);
      for (int r = 0; r < P; r++) off[r] = r * per * 4;
      DevBuf in(per * 4);
      launchFill(in.p, per, DataType::FLOAT32, 7.0, 1.0, stream);
      for (int r = 0; r < P; r++) GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0, n * 4, stream));
      launchGatherPush(ca, in.p, pp, nullptr, off.data(), len.data(), -1, true, std::min(2 * pc.maxBlocks(), 32), stream);
      noteLaunch();
      auto h = download(pp.p[P - 1], n, stream);
      for (size_t i = 0; i < per; i++) {
        if (!close(h[i], 7.0 + i)) return strcat_all("element ", i, ": got ", h[i]);
      }
      return h[per] == 0.0f ? "" : "wrote outside my block";
    });
    R.run(strcat_all("castGatherPushKernel<bf16> (allgather, f32 in) P=", P), [&]() -> std::string {
      const size_t per = n / P;
      std::vector<size_t> off(P), len(P, per);
      for (int r = 0; r < P; r++) off[r] = r * per;
      DevBuf in(per * 4);
      launchFill(in.p, per, DataType::FLOAT32, 7.0, 1.0 / 3.0, stream);  // most need rounding
      for (int r = 0; r < P; r++) GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0, n * 2, stream));
      launchCastGatherPush(ca, in.p, pp, DataType::BFLOAT16, off.data(), len.data(), true,
                           std::min(2 * pc.maxBlocks(), 32), stream);
      noteLaunch();
      auto x = download(in.p, per, stream);
      std::vector<uint16_t> h(n);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), pp.p[P - 1], n * 2, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < per; i++) {
        if (h[i] != floatToBf16(x[i])) return strcat_all("element ", i, ": got ", bf16ToFloat(h[i]), " for ", x[i]);
      }
      return h[per] == 0 ? "" : "wrote outside my block";
    });
    R.run(strcat_all("alltoallPushKernel P=", P), [&]() -> std::string {
      const size_t per = n / P / 4 * 4;
      std::vector<size_t> soff(P), slen(P, per * 4), doff(P, 0);
      for (int r = 0; r < P; r++) soff[r] = r * per * 4;
      DevBuf in(per * 4 * P);
      launchFill(in.p, per * P, DataType::FLOAT32, 0.0, 1.0, stream);
      for (int r = 0; r < P; r++) GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0, n * 4, stream));
      launchAlltoallPush(ca, in.p, pp, soff.data(), slen.data(), doff.data(), nullptr, -1, true,
                         std::min(2 * pc.maxBlocks(), 32), stream);
      noteLaunch();
      auto h = download(pp.p[P - 1], per, stream);  // chunk P-1 of my input lands in slot 0 of rank P-1
      for (size_t i = 0; i < per; i++) {
        if (!close(h[i], static_cast<double>((P - 1) * per + i))) return strcat_all("element ", i, ": got ", h[i]);
      }
      return "";
    });
    // Device-split all-to-all-v. Rank 0 writes its counts into column j of the tables for virtual
    // peer j, which is column j of its own pad: every virtual rank holds rank 0's splits. Rank 0's
    // segments then have a closed form: on rank j, expert e's segment starts at
    // base_e = sum over e' < e of roundUp(P * split(j, e'), align), and rank 0's rows come first.
    R.run(strcat_all("alltoallvDevKernel (dispatch + combine, E=3, align=8, 12-byte rows) P=", P), [&]() -> std::string {
      const int E = 3, A = 8, K = P * E;
      const size_t rb = 12, cap = n * 4 / rb;
      std::vector<int64_t> sp(K), pre(K + 1, 0);
      for (int k = 0; k < K; k++) {
        sp[k] = (k * 7 + 3) % 11;
        pre[k + 1] = pre[k] + sp[k];
      }
      auto base = [&](int j, int e) {
        int64_t b = 0;
        for (int x = 0; x < e; x++) b = (b + P * sp[j * E + x] + A - 1) / A * A;
        return b;
      };
      DevBuf in(pre[K] * rb), splits(K * 8), outSplits(K * 8), outOffsets(K * 8);
      launchFill(in.p, pre[K] * 3, DataType::FLOAT32, 0.0, 1.0, stream);  // row r = {3r, 3r+1, 3r+2}
      GLB_CUDA_CHECK(cudaMemcpyAsync(splits.p, sp.data(), K * 8, cudaMemcpyHostToDevice, stream));
      for (int r = 0; r < P; r++) GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0xff, n * 4, stream));
      const int blocks = std::min(pc.coResidentBlocks(alltoallvDevKernelPtr()), 16);
      launchAlltoallvDev(ca, pp, moeArgs(rb, cap, E, A, pc.inputStatusDevice()), nullptr, in.p, pre[K],
                         static_cast<const long long*>(splits.p), nullptr, static_cast<long long*>(outSplits.p),
                         static_cast<long long*>(outOffsets.p), false, blocks, stream);
      noteLaunch();
      std::vector<int64_t> os(K), oo(K);
      GLB_CUDA_CHECK(cudaMemcpyAsync(os.data(), outSplits.p, K * 8, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaMemcpyAsync(oo.data(), outOffsets.p, K * 8, cudaMemcpyDeviceToHost, stream));
      for (int j = 0; j < P; j++) {
        auto h = download(pp.p[j], n, stream);
        for (int e = 0; e < E; e++) {
          const int k = j * E + e;
          const int64_t at = base(j, e);
          for (int64_t r = 0; r < sp[k]; r++) {
            for (int c = 0; c < 3; c++) {
              const float got = h[(at + r) * 3 + c];
              if (!close(got, 3.0 * (pre[k] + r) + c)) return strcat_all("dispatch dst ", j, " expert ", e, " row ", r, ": got ", got);
            }
          }
          // Virtual rank 1's rows follow (never written). An empty segment has no such row: the
          // next expert's segment starts at the same place.
          if (sp[k] > 0 && !std::isnan(h[(at + sp[k]) * 3])) {
            return strcat_all("dispatch dst ", j, ": wrote past rank 0's segment");
          }
        }
      }
      for (int e = 0; e < E; e++) {
        for (int s = 0; s < P; s++) {
          if (os[e * P + s] != sp[e] || oo[e * P + s] != base(0, e) + s * sp[e]) {
            return strcat_all("out_splits/out_offsets[", e * P + s, "] = ", os[e * P + s], "/", oo[e * P + s]);
          }
        }
      }
      // Combine from rank 0's dispatch output: its own rows come back to where they were.
      DevBuf back(n * 4);
      PeerPtrs bp = pp;
      bp.p[0] = back.p;
      GLB_CUDA_CHECK(cudaMemsetAsync(back.p, 0, n * 4, stream));
      launchAlltoallvDev(ca, bp, moeArgs(rb, cap, E, 1, pc.inputStatusDevice()), nullptr, pp.p[0], cap,
                         static_cast<const long long*>(outSplits.p), static_cast<const long long*>(outOffsets.p),
                         nullptr, nullptr, true, blocks, stream);
      noteLaunch();
      auto h = download(back.p, n, stream);
      for (int64_t i = 0; i < pre[E] * 3; i++) {
        if (!close(h[i], static_cast<double>(i))) return strcat_all("combine element ", i, ": got ", h[i]);
      }
      if (h[pre[E] * 3] != 0.0f) return "combine wrote past its rows";
      return "";
    });
    // Its quantising form (bf16 -> e4m3 codes + one fp32 scale per 128 elements). Every block holds
    // small integers and one element of magnitude 448, so its scale is exactly 1 and its codes are
    // the e4m3 encodings of the inputs. The layout has the closed form of the case above.
    if (P == 2 || P == 8) {
      R.run(strcat_all("alltoallvDevKernel<fp8> (dispatch, E=2, align=4, H=256) P=", P), [&]() -> std::string {
        const int E = 2, A = 4, K = P * E, H = 256, nb = H / kFp8Block;
        const size_t cap = 512;
        std::vector<int64_t> sp(K), pre(K + 1, 0);
        for (int k = 0; k < K; k++) {
          sp[k] = (k * 5 + 1) % 4;
          pre[k + 1] = pre[k] + sp[k];
        }
        auto base = [&](int j, int e) {
          int64_t b = 0;
          for (int x = 0; x < e; x++) b = (b + P * sp[j * E + x] + A - 1) / A * A;
          return b;
        };
        auto value = [&](int64_t r, int i) -> float {
          const int b = i / kFp8Block, pos = i % kFp8Block;
          if (pos == (r * 3 + b * 5) % kFp8Block) return (r + b) % 2 ? -448.0f : 448.0f;
          return static_cast<float>((r * 7 + i * 3) % 33 - 16);
        };
        std::vector<uint16_t> rows(pre[K] * H);
        for (int64_t r = 0; r < pre[K]; r++) {
          for (int i = 0; i < H; i++) {
            const float f = value(r, i);
            uint32_t w;
            std::memcpy(&w, &f, 4);
            rows[r * H + i] = static_cast<uint16_t>(w >> 16);  // exact: small integers and 448
          }
        }
        DevBuf in(rows.size() * 2), splits(K * 8), outSplits(K * 8), outOffsets(K * 8);
        std::vector<std::unique_ptr<DevBuf>> scaleBufs;
        PeerPtrs sc;
        std::memset(&sc, 0, sizeof(sc));
        for (int r = 0; r < P; r++) {
          scaleBufs.emplace_back(new DevBuf(cap * nb * 4));
          sc.p[r] = scaleBufs[r]->p;
          GLB_CUDA_CHECK(cudaMemsetAsync(sc.p[r], 0xff, cap * nb * 4, stream));
          GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0xff, cap * H, stream));
        }
        GLB_CUDA_CHECK(cudaMemcpyAsync(in.p, rows.data(), rows.size() * 2, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(splits.p, sp.data(), K * 8, cudaMemcpyHostToDevice, stream));
        const int blocks = std::min(pc.coResidentBlocks(alltoallvDevKernelPtr(true)), 16);
        const MoeScales scales{sc, nullptr};
        launchAlltoallvDev(ca, pp, moeArgs(H, cap, E, A, pc.inputStatusDevice()), &scales, in.p, pre[K],
                           static_cast<const long long*>(splits.p), nullptr, static_cast<long long*>(outSplits.p),
                           static_cast<long long*>(outOffsets.p), false, blocks, stream);
        noteLaunch();
        std::vector<int64_t> os(K), oo(K);
        GLB_CUDA_CHECK(cudaMemcpyAsync(os.data(), outSplits.p, K * 8, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(oo.data(), outOffsets.p, K * 8, cudaMemcpyDeviceToHost, stream));
        for (int j = 0; j < P; j++) {
          std::vector<uint8_t> codes(cap * H);
          std::vector<float> scales(cap * nb);
          GLB_CUDA_CHECK(cudaMemcpyAsync(codes.data(), pp.p[j], codes.size(), cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaMemcpyAsync(scales.data(), sc.p[j], scales.size() * 4, cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
          for (int e = 0; e < E; e++) {
            const int k = j * E + e;
            const int64_t at = base(j, e);
            for (int64_t r = 0; r < sp[k]; r++) {
              for (int i = 0; i < H; i++) {
                const uint8_t want = float8_e4m3::fromFloat(value(pre[k] + r, i));
                if (codes[(at + r) * H + i] != want) {
                  return strcat_all("dst ", j, " expert ", e, " row ", r, " element ", i, ": code ",
                                    static_cast<int>(codes[(at + r) * H + i]), ", want ", static_cast<int>(want));
                }
              }
              for (int b = 0; b < nb; b++) {
                if (scales[(at + r) * nb + b] != 1.0f) {
                  return strcat_all("dst ", j, " expert ", e, " row ", r, " scale ", b, ": ", scales[(at + r) * nb + b]);
                }
              }
            }
            // Virtual rank 1's rows follow and are never written, in either tensor.
            if (sp[k] > 0 && (codes[(at + sp[k]) * H] != 0xff || !std::isnan(scales[(at + sp[k]) * nb]))) {
              return strcat_all("dispatch dst ", j, ": wrote past rank 0's segment");
            }
          }
        }
        for (int e = 0; e < E; e++) {
          for (int s = 0; s < P; s++) {
            if (os[e * P + s] != sp[e] || oo[e * P + s] != base(0, e) + s * sp[e]) {
              return strcat_all("out_splits/out_offsets[", e * P + s, "] = ", os[e * P + s], "/", oo[e * P + s]);
            }
          }
        }
        return "";
      });
      // The top-k dispatch, both forms, zero copy. Every virtual rank holds rank 0's splits, so rank
      // 0's rows for expert e of rank j start at base(j, e) (as above) and go by token, then choice.
      // The host routes the indices itself (entries -1 and >= P·E are not routed, some tokens pick an
      // expert twice) and checks splits, pos, out_splits / out_offsets and every pushed row.
      for (const bool fp8 : {false, true}) {
        const char* what = fp8 ? "moeDispatchTopkKernel<fp8> (E=2, align=4, k=3, H=256) P="
                               : "moeDispatchTopkKernel (E=3, align=8, k=4, 32-byte rows) P=";
        R.run(strcat_all(what, P), [&, fp8]() -> std::string {
          const int E = fp8 ? 2 : 3, A = fp8 ? 4 : 8, K = P * E, topk = fp8 ? 3 : 4, H = fp8 ? 256 : 8, nb = H / kFp8Block;
          const size_t T = 45, rb = fp8 ? H : H * 4, cap = 512;
          std::vector<int64_t> idx(T * topk), sp(K, 0), pos(T * topk, -1), pre(K + 1, 0);
          for (size_t i = 0; i < T * topk; i++) idx[i] = static_cast<int64_t>((i * 7 + i / topk * 3) % (K + 2)) - 1;
          for (size_t i = 0; i < T * topk; i++) if (idx[i] >= 0 && idx[i] < K) sp[idx[i]]++;
          for (int g = 0; g < K; g++) pre[g + 1] = pre[g] + sp[g];
          std::vector<int64_t> seen(K, 0);
          for (size_t i = 0; i < T * topk; i++) if (idx[i] >= 0 && idx[i] < K) pos[i] = pre[idx[i]] + seen[idx[i]]++;
          auto base = [&](int j, int e) {
            int64_t b = 0;
            for (int x = 0; x < e; x++) b = (b + P * sp[j * E + x] + A - 1) / A * A;
            return b;
          };
          // fp8: small integers and one +-448 per block (scale 1, codes exact); else row t = 8t .. 8t + 7.
          auto value = [&](int64_t r, int i) -> float {
            if (!fp8) return static_cast<float>(r * H + i);
            const int b = i / kFp8Block, at = i % kFp8Block;
            if (at == (r * 3 + b * 5) % kFp8Block) return (r + b) % 2 ? -448.0f : 448.0f;
            return static_cast<float>((r * 7 + i * 3) % 33 - 16);
          };
          DevBuf x(T * H * 4), idxDev(idx.size() * 8), splits(K * 8), posDev(pos.size() * 8), outSplits(K * 8),
              outOffsets(K * 8);
          if (fp8) {
            std::vector<uint16_t> rows(T * H);
            for (size_t r = 0; r < T; r++) {
              for (int i = 0; i < H; i++) {
                const float f = value(r, i);
                uint32_t w;
                std::memcpy(&w, &f, 4);
                rows[r * H + i] = static_cast<uint16_t>(w >> 16);  // exact
              }
            }
            GLB_CUDA_CHECK(cudaMemcpyAsync(x.p, rows.data(), rows.size() * 2, cudaMemcpyHostToDevice, stream));
          } else {
            launchFill(x.p, T * H, DataType::FLOAT32, 0.0, 1.0, stream);
          }
          GLB_CUDA_CHECK(cudaMemcpyAsync(idxDev.p, idx.data(), idx.size() * 8, cudaMemcpyHostToDevice, stream));
          std::vector<std::unique_ptr<DevBuf>> scaleBufs;
          PeerPtrs sc;
          std::memset(&sc, 0, sizeof(sc));
          for (int r = 0; r < P; r++) {
            scaleBufs.emplace_back(new DevBuf(cap * 4 * 4));
            sc.p[r] = scaleBufs[r]->p;
            GLB_CUDA_CHECK(cudaMemsetAsync(sc.p[r], 0xff, cap * 4 * 4, stream));
            GLB_CUDA_CHECK(cudaMemsetAsync(pp.p[r], 0xff, cap * rb, stream));
          }
          const int blocks = std::min(pc.coResidentBlocks(moeDispatchTopkKernelPtr(fp8)), 16);
          auto ll = [](DevBuf& b) { return static_cast<long long*>(b.p); };
          const MoeScales scales{sc, nullptr};
          launchMoeDispatchTopk(ca, pp, moeArgs(rb, cap, E, A, pc.inputStatusDevice()),
                                fp8 ? &scales : nullptr, x.p, T, topk, ll(idxDev), ll(splits), ll(posDev),
                                ll(outSplits), ll(outOffsets), blocks, stream);
          noteLaunch();
          std::vector<int64_t> gs(K), gp(T * topk), os(K), oo(K);
          GLB_CUDA_CHECK(cudaMemcpyAsync(gs.data(), splits.p, K * 8, cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaMemcpyAsync(gp.data(), posDev.p, gp.size() * 8, cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaMemcpyAsync(os.data(), outSplits.p, K * 8, cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaMemcpyAsync(oo.data(), outOffsets.p, K * 8, cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
          if (gs != sp) return "splits differ from the host routing";
          if (gp != pos) return "pos differs from the host routing";
          for (int e = 0; e < E; e++) {
            for (int s = 0; s < P; s++) {
              if (os[e * P + s] != sp[e] || oo[e * P + s] != base(0, e) + s * sp[e]) {
                return strcat_all("out_splits/out_offsets[", e * P + s, "] = ", os[e * P + s], "/", oo[e * P + s]);
              }
            }
          }
          for (int j = 0; j < P; j++) {
            std::vector<uint8_t> out(cap * rb);
            std::vector<float> scales(cap * 4);
            GLB_CUDA_CHECK(cudaMemcpyAsync(out.data(), pp.p[j], out.size(), cudaMemcpyDeviceToHost, stream));
            GLB_CUDA_CHECK(cudaMemcpyAsync(scales.data(), sc.p[j], scales.size() * 4, cudaMemcpyDeviceToHost, stream));
            GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
            for (size_t i = 0; i < T * topk; i++) {
              if (pos[i] < 0 || idx[i] / E != j) continue;
              const int g = static_cast<int>(idx[i]);
              const int64_t row = base(j, g % E) + (pos[i] - pre[g]), tok = static_cast<int64_t>(i / topk);
              for (int c = 0; c < H; c++) {
                bool ok;
                if (fp8) {
                  ok = out[row * rb + c] == float8_e4m3::fromFloat(value(tok, c));
                } else {
                  float f;
                  std::memcpy(&f, &out[row * rb + c * 4], 4);
                  ok = f == value(tok, c);
                }
                if (!ok) return strcat_all("dst ", j, " row ", row, " (token ", tok, ") element ", c, " differs");
              }
              for (int b = 0; fp8 && b < nb; b++) {
                if (scales[row * nb + b] != 1.0f) return strcat_all("dst ", j, " row ", row, " scale ", b, " differs");
              }
            }
            // Virtual rank 1's rows follow rank 0's in each segment and are never written.
            for (int e = 0; e < E; e++) {
              const int64_t end = base(j, e) + sp[j * E + e];
              if (sp[j * E + e] > 0 && out[end * rb] != 0xff) return strcat_all("dst ", j, ": wrote past rank 0's rows");
            }
          }
          return "";
        });
      }
      // The top-k combine, zero copy, with the closed-form layout of the dispatch case above: rank 0's
      // chunk k = j·E + e lies on virtual holder j from row base(j, e) on. Holder j's expert_out
      // (pp.p[j]) holds bf16 halves of small integers; the host sums in the kernel's fp32 order.
      R.run(strcat_all("moeCombineTopkKernel<bf16> (E=2, align=4, k=3, 64-element rows) P=", P), [&]() -> std::string {
        const int E = 2, A = 4, K = P * E, H = 64, topk = 3;
        const size_t rb = H * 2, cap = n * 4 / rb, T = 37;
        std::vector<int64_t> sp(K), pre(K + 1, 0);
        for (int k = 0; k < K; k++) {
          sp[k] = (k * 5 + 2) % 4;
          pre[k + 1] = pre[k] + sp[k];
        }
        auto base = [&](int j, int e) {
          int64_t b = 0;
          for (int x = 0; x < e; x++) b = (b + P * sp[j * E + x] + A - 1) / A * A;
          return b;
        };
        auto value = [](int j, int64_t row, int c) { return static_cast<float>((j * 7 + row * 3 + c) % 17 - 8) * 0.5f; };
        std::vector<int64_t> pos(T * topk);
        std::vector<float> w(T * topk);
        for (size_t t = 0; t < T; t++) {
          for (int c = 0; c < topk; c++) {
            pos[t * topk + c] = (t * c) % 5 == 1 || t == 4 ? -1 : static_cast<int64_t>((t * 7 + c * 11) % pre[K]);
            w[t * topk + c] = static_cast<float>((t * 5 + c * 3) % 9) * 0.3f - 1.1f;
          }
        }
        for (int j = 0; j < P; j++) {
          std::vector<uint16_t> rows(cap * H);
          for (size_t r = 0; r < cap; r++) {
            for (int c = 0; c < H; c++) {
              const float f = value(j, r, c);
              uint32_t u;
              std::memcpy(&u, &f, 4);
              rows[r * H + c] = static_cast<uint16_t>(u >> 16);  // exact: halves of small integers
            }
          }
          GLB_CUDA_CHECK(cudaMemcpyAsync(pp.p[j], rows.data(), rows.size() * 2, cudaMemcpyHostToDevice, stream));
          GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        }
        DevBuf splits(K * 8), posDev(pos.size() * 8), wDev(w.size() * 4), out(T * rb);
        GLB_CUDA_CHECK(cudaMemcpyAsync(splits.p, sp.data(), K * 8, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(posDev.p, pos.data(), pos.size() * 8, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(wDev.p, w.data(), w.size() * 4, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0xff, T * rb, stream));
        const int blocks = std::min(pc.coResidentBlocks(moeCombineTopkKernelPtr(DataType::BFLOAT16)), 16);
        launchMoeCombineTopk(ca, pp, moeArgs(rb, cap, E, A, pc.inputStatusDevice()), out.p, T, topk,
                             static_cast<const long long*>(posDev.p), static_cast<const float*>(wDev.p),
                             static_cast<const long long*>(splits.p), DataType::BFLOAT16, blocks, stream);
        noteLaunch();
        std::vector<uint16_t> got(T * H);
        GLB_CUDA_CHECK(cudaMemcpyAsync(got.data(), out.p, T * rb, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (size_t t = 0; t < T; t++) {
          for (int c = 0; c < H; c++) {
            float acc = 0.0f;
            for (int x = 0; x < topk; x++) {
              const int64_t p = pos[t * topk + x];
              if (p < 0) continue;
              int k = 0;
              while (pre[k + 1] <= p) k++;
              const float prod = w[t * topk + x] * value(k / E, base(k / E, k % E) + (p - pre[k]), c);
              acc = acc + prod;
            }
            uint32_t u;
            std::memcpy(&u, &acc, 4);
            const uint16_t want = static_cast<uint16_t>((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);  // round to nearest even
            if (got[t * H + c] != want) {
              return strcat_all("token ", t, " element ", c, ": got bf16 bits ", static_cast<int>(got[t * H + c]),
                                ", want ", static_cast<int>(want));
            }
          }
        }
        return "";
      });
    }
    // The top-k combine's backward, zero copy, with the combine case's closed-form layout. pos names
    // every routed row of rank 0's dispatch input at most once. dy holds quarters and expert_out halves
    // of small integers, so every product and partial sum of the dot is exact in fp32 and grad_w is
    // the exact dot product. Holder j's gradient rows of rank 0 must be bf16(w · dy); holder 0 (rank 0
    // itself) zeroes its alignment gaps and tail; a guard row after the capacity stays untouched.
    R.run(strcat_all("moeCombineTopkBackwardKernel<bf16> (E=2, align=4, k=3, 64-element rows) P=", P),
          [&]() -> std::string {
      const int E = 2, A = 4, K = P * E, H = 64, topk = 3;
      const size_t rb = H * 2, cap = n * 4 / rb - 1, T = 37;
      std::vector<int64_t> sp(K), pre(K + 1, 0);
      for (int k = 0; k < K; k++) {
        sp[k] = (k * 5 + 2) % 4;
        pre[k + 1] = pre[k] + sp[k];
      }
      auto base = [&](int j, int e) {
        int64_t b = 0;
        for (int x = 0; x < e; x++) b = (b + P * sp[j * E + x] + A - 1) / A * A;
        return b;
      };
      auto value = [](int j, int64_t row, int c) { return static_cast<float>((j * 7 + row * 3 + c) % 17 - 8) * 0.5f; };
      auto dyv = [](size_t t, int c) { return static_cast<float>(static_cast<int>((t * 5 + c * 3) % 9) - 4) * 0.25f; };
      auto bf16 = [](float f) {
        uint32_t u;
        std::memcpy(&u, &f, 4);
        return static_cast<uint16_t>((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);  // round to nearest even
      };
      // pos: a stride permutation of the routed rows, dealt to the choices that are not dropped.
      const int64_t N = pre[K];
      int64_t stride = 7;
      while (std::gcd(stride, N) != 1) stride++;
      std::vector<int64_t> pos(T * topk, -1);
      std::vector<float> w(T * topk);
      int64_t next = 0;
      for (size_t t = 0; t < T; t++) {
        for (int c = 0; c < topk; c++) {
          const bool dropped = (t * c) % 5 == 1 || t == 4;
          if (!dropped && next < N) pos[t * topk + c] = (next++ * stride) % N;
          w[t * topk + c] = static_cast<float>((t * 5 + c * 3) % 9) * 0.3f - 1.1f;
        }
      }
      std::vector<uint16_t> dyHost(T * H);
      for (size_t t = 0; t < T; t++) {
        for (int c = 0; c < H; c++) dyHost[t * H + c] = bf16(dyv(t, c));
      }
      std::vector<std::unique_ptr<DevBuf>> gradBufs;
      PeerPtrs gp;
      std::memset(&gp, 0, sizeof(gp));
      for (int j = 0; j < P; j++) {
        std::vector<uint16_t> rows(cap * H);
        for (size_t r = 0; r < cap; r++) {
          for (int c = 0; c < H; c++) rows[r * H + c] = bf16(value(j, r, c));  // exact
        }
        GLB_CUDA_CHECK(cudaMemcpyAsync(pp.p[j], rows.data(), rows.size() * 2, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        gradBufs.emplace_back(new DevBuf((cap + 1) * rb));  // + a guard row
        gp.p[j] = gradBufs[j]->p;
        GLB_CUDA_CHECK(cudaMemsetAsync(gp.p[j], 0xff, (cap + 1) * rb, stream));
      }
      DevBuf splits(K * 8), posDev(pos.size() * 8), wDev(w.size() * 4), dy(T * rb), gw(T * topk * 4);
      GLB_CUDA_CHECK(cudaMemcpyAsync(splits.p, sp.data(), K * 8, cudaMemcpyHostToDevice, stream));
      GLB_CUDA_CHECK(cudaMemcpyAsync(posDev.p, pos.data(), pos.size() * 8, cudaMemcpyHostToDevice, stream));
      GLB_CUDA_CHECK(cudaMemcpyAsync(wDev.p, w.data(), w.size() * 4, cudaMemcpyHostToDevice, stream));
      GLB_CUDA_CHECK(cudaMemcpyAsync(dy.p, dyHost.data(), T * rb, cudaMemcpyHostToDevice, stream));
      GLB_CUDA_CHECK(cudaMemsetAsync(gw.p, 0xff, T * topk * 4, stream));
      const int blocks = std::min(pc.coResidentBlocks(moeCombineTopkBackwardKernelPtr(DataType::BFLOAT16)), 16);
      launchMoeCombineTopkBackward(ca, pp, gp, moeArgs(rb, cap, E, A, pc.inputStatusDevice()), nullptr, cap, dy.p,
                                   static_cast<float*>(gw.p), T, topk, static_cast<const long long*>(posDev.p),
                                   static_cast<const float*>(wDev.p), static_cast<const long long*>(splits.p),
                                   DataType::BFLOAT16, blocks, stream);
      noteLaunch();
      std::vector<float> gotW(T * topk);
      GLB_CUDA_CHECK(cudaMemcpyAsync(gotW.data(), gw.p, gotW.size() * 4, cudaMemcpyDeviceToHost, stream));
      std::vector<std::vector<uint16_t>> grads(P, std::vector<uint16_t>((cap + 1) * H));
      for (int j = 0; j < P; j++) {
        GLB_CUDA_CHECK(cudaMemcpyAsync(grads[j].data(), gp.p[j], (cap + 1) * rb, cudaMemcpyDeviceToHost, stream));
      }
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < T * topk; i++) {
        const size_t t = i / topk;
        const int64_t p = pos[i];
        if (p < 0) {
          uint32_t u;
          std::memcpy(&u, &gotW[i], 4);
          if (u != 0u) return strcat_all("token ", t, " choice ", i % topk, ": grad_w of a dropped choice is not +0");
          continue;
        }
        int k = 0;
        while (pre[k + 1] <= p) k++;
        const int j = k / E;
        const int64_t row = base(j, k % E) + (p - pre[k]);
        double dot = 0.0;
        for (int c = 0; c < H; c++) {
          dot += static_cast<double>(dyv(t, c)) * value(j, row, c);
          const uint16_t want = bf16(w[i] * bf16ToFloat(dyHost[t * H + c]));
          if (grads[j][row * H + c] != want) {
            return strcat_all("holder ", j, " row ", row, " element ", c, ": got bf16 bits ",
                              static_cast<int>(grads[j][row * H + c]), ", want ", static_cast<int>(want));
          }
        }
        if (static_cast<double>(gotW[i]) != dot) {
          return strcat_all("token ", t, " choice ", i % topk, ": grad_w ", gotW[i], ", want ", dot);
        }
      }
      // Holder 0's rows outside its segments (every source sends rank 0's splits): zero.
      for (int e = 0; e < E; e++) {
        const int64_t lo = base(0, e) + P * sp[e], hi = e + 1 < E ? base(0, e + 1) : static_cast<int64_t>(cap);
        for (int64_t r = lo; r < hi; r++) {
          for (int c = 0; c < H; c++) {
            if (grads[0][r * H + c] != 0) return strcat_all("holder 0 row ", r, " (outside its segments) is not zero");
          }
        }
      }
      for (int j = 0; j < P; j++) {
        for (int c = 0; c < H; c++) {
          if (grads[j][cap * H + c] != 0xffffu) return strcat_all("holder ", j, ": wrote past its capacity");
        }
      }
      return "";
    });
    // The low-latency dispatch and combine, both forms, at P = 2 and 8. Virtual rank 0 pushes to slot
    // (e, 0, r) of every virtual holder and packs its own experts' rows; the host stands in for the
    // other sources by storing their signal words (no rows) into rank 0's buffer. The combine pushes
    // rank 0's packed rows back to its own combine slots; the slots of choices held by the virtual
    // holders are filled by the host. bf16 values are halves / quarters of small integers, FP8 rows
    // small integers with one +-448 per block (scale 1, codes exact), so every sum is exact in order.
    for (const bool fp8 : {false, true}) {
      if (P != 2 && P != 8) break;
      const char* what = fp8 ? "moeLLDispatchKernel<fp8> + moeLLCombineKernel<bf16> (E=2, k=3, H=256) P="
                             : "moeLLDispatchKernel + moeLLCombineKernel<bf16> (E=2, k=3, H=64) P=";
      R.run(strcat_all(what, P), [&, fp8]() -> std::string {
        const int E = 2, K = P * E, topk = 3, H = fp8 ? 256 : 64, T = 13, M = T * topk, nb = H / kFp8Block;
        const MoeLLLayout l = moeLLLayout(P, E, M, topk, H, 2, fp8);
        const uint32_t form = fp8 ? kMoeLLDispatchFp8 : kMoeLLDispatch;
        std::vector<std::unique_ptr<DevBuf>> bufs;
        MoeLLArgs L{};
        for (int r = 0; r < P; r++) {
          bufs.emplace_back(new DevBuf(l.bytes));
          L.bufs.p[r] = bufs[r]->p;
          GLB_CUDA_CHECK(cudaMemsetAsync(L.bufs.p[r], 0, l.bytes, stream));
        }
        L.l = l;
        L.status = pc.inputStatusDevice();
        char* b0 = static_cast<char*>(L.bufs.p[0]);
        auto bf16 = [](float f) {
          uint32_t u;
          std::memcpy(&u, &f, 4);
          return static_cast<uint16_t>(u >> 16);  // exact for the values used here
        };
        auto value = [&](int t, int c) -> float {
          if (!fp8) return static_cast<float>((t * 3 + c) % 17 - 8) * 0.5f;
          const int b = c / kFp8Block;
          if (c % kFp8Block == (t * 3 + b * 5) % kFp8Block) return (t + b) % 2 ? -448.0f : 448.0f;
          return static_cast<float>((t * 7 + c * 3) % 33 - 16);
        };
        std::vector<int64_t> idx(T * topk);
        std::vector<int> rank(T * topk, -1), cnt(K, 0);
        for (int i = 0; i < T * topk; i++) {
          idx[i] = static_cast<int64_t>((i * 5 + i / topk * 3) % (K + 2)) - 1;
          if (idx[i] >= 0 && idx[i] < K) rank[i] = cnt[idx[i]]++;
        }
        std::vector<uint16_t> xh(T * H);
        for (int t = 0; t < T; t++) for (int c = 0; c < H; c++) xh[t * H + c] = bf16(value(t, c));
        const size_t rb = l.rowBytes, slotsRows = static_cast<size_t>(E) * P * M;
        DevBuf x(xh.size() * 2), idxDev(idx.size() * 8), out(slotsRows * rb), outScales(slotsRows * nb * 4 + 16),
            outSplits(K * 8);
        GLB_CUDA_CHECK(cudaMemcpyAsync(x.p, xh.data(), xh.size() * 2, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(idxDev.p, idx.data(), idx.size() * 8, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0xff, out.bytes, stream));
        std::vector<unsigned long long> words(K, 0ull);
        for (int e = 0; e < E; e++) for (int s2 = 1; s2 < P; s2++) words[e * P + s2] = moeLLSignal(1, form, 0);
        GLB_CUDA_CHECK(cudaMemcpyAsync(b0 + l.dispatchSig, words.data(), K * 8, cudaMemcpyHostToDevice, stream));
        const int blocks = std::min(pc.coResidentBlocks(moeLLDispatchKernelPtr(fp8)), 16);
        launchMoeLLDispatch(ca, L, x.p, T, static_cast<const long long*>(idxDev.p), out.p,
                            static_cast<float*>(outScales.p), static_cast<long long*>(outSplits.p), blocks, stream);
        noteLaunch();
        std::vector<int64_t> os(K);
        std::vector<uint8_t> outH(out.bytes);
        std::vector<float> scH(slotsRows * nb);
        GLB_CUDA_CHECK(cudaMemcpyAsync(os.data(), outSplits.p, K * 8, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(outH.data(), out.p, out.bytes, cudaMemcpyDeviceToHost, stream));
        if (fp8) GLB_CUDA_CHECK(cudaMemcpyAsync(scH.data(), outScales.p, scH.size() * 4, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (int e = 0; e < E; e++) {
          for (int s2 = 0; s2 < P; s2++) {
            if (os[e * P + s2] != (s2 == 0 ? cnt[e] : 0)) return strcat_all("out_splits[", e * P + s2, "] = ", os[e * P + s2]);
          }
        }
        // Every routed choice: its slot row and tag on its holder; rank 0's own experts: the packed row.
        auto rowOk = [&](const uint8_t* row, int t) {
          for (int c = 0; c < H; c++) {
            if (fp8 ? row[c] != float8_e4m3::fromFloat(value(t, c))
                    : std::memcmp(row + 2 * c, &xh[t * H + c], 2) != 0) return false;
          }
          return true;
        };
        for (int j = 0; j < P; j++) {
          std::vector<uint8_t> slots(l.tags - l.slots);
          std::vector<int32_t> tags(slotsRows);
          GLB_CUDA_CHECK(cudaMemcpyAsync(slots.data(), static_cast<char*>(L.bufs.p[j]) + l.slots, slots.size(),
                                         cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaMemcpyAsync(tags.data(), static_cast<char*>(L.bufs.p[j]) + l.tags, tags.size() * 4,
                                         cudaMemcpyDeviceToHost, stream));
          GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
          for (int i = 0; i < T * topk; i++) {
            if (rank[i] < 0 || idx[i] / E != j) continue;
            const int e = static_cast<int>(idx[i] % E), t = i / topk;
            const size_t slot = static_cast<size_t>(e) * P * M + rank[i];  // (e, source 0, r)
            if (tags[slot] != i) return strcat_all("holder ", j, " slot ", slot, ": tag ", tags[slot], ", want ", i);
            if (!rowOk(&slots[slot * rb], t)) return strcat_all("holder ", j, " slot ", slot, " (token ", t, ") differs");
            if (j == 0) {
              const size_t row = static_cast<size_t>(e) * P * M + rank[i];
              if (!rowOk(&outH[row * rb], t)) return strcat_all("out[", e, ", ", rank[i], "] (token ", t, ") differs");
              for (int b = 0; fp8 && b < nb; b++) {
                if (scH[row * nb + b] != 1.0f) return strcat_all("out_scales[", e, ", ", rank[i], "] differs");
              }
            }
          }
        }
        for (int e = 0; e < E; e++) {
          if (outH[(static_cast<size_t>(e) * P * M + cnt[e]) * rb] != 0xff) return strcat_all("wrote past expert ", e);
        }

        // ---- combine ----
        const size_t crb = l.combineRowBytes;
        auto eoValue = [](int e, size_t q, int c) { return static_cast<float>((e * 5 + q * 3 + c) % 13 - 6) * 0.5f; };
        auto preValue = [](int i, int c) { return static_cast<float>((i * 7 + c) % 11 - 5) * 0.25f; };
        std::vector<uint16_t> eo(slotsRows * H), pre(static_cast<size_t>(T) * topk * H);
        for (int e = 0; e < E; e++) {
          for (size_t q = 0; q < static_cast<size_t>(P) * M; q++) {
            for (int c = 0; c < H; c++) eo[(e * P * M + q) * H + c] = bf16(eoValue(e, q, c));
          }
        }
        for (int i = 0; i < T * topk; i++) for (int c = 0; c < H; c++) pre[i * H + c] = bf16(preValue(i, c));
        std::vector<float> w(T * topk);
        for (int i = 0; i < T * topk; i++) w[i] = static_cast<float>((i * 5) % 9) * 0.25f - 1.0f;
        DevBuf eoDev(eo.size() * 2), wDev(w.size() * 4), y(static_cast<size_t>(T) * crb);
        GLB_CUDA_CHECK(cudaMemcpyAsync(eoDev.p, eo.data(), eo.size() * 2, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(wDev.p, w.data(), w.size() * 4, cudaMemcpyHostToDevice, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(b0 + l.combineSlots, pre.data(), pre.size() * 2, cudaMemcpyHostToDevice, stream));
        std::vector<unsigned long long> cw(P, moeLLSignal(2, kMoeLLCombine, 0));
        GLB_CUDA_CHECK(cudaMemcpyAsync(b0 + l.combineSig + 8, cw.data(), (P - 1) * 8, cudaMemcpyHostToDevice, stream));
        launchMoeLLCombine(ca, L, eoDev.p, static_cast<const float*>(wDev.p), y.p, T, DataType::BFLOAT16,
                           std::min(pc.coResidentBlocks(moeLLCombineKernelPtr(DataType::BFLOAT16)), 16), stream);
        noteLaunch();
        std::vector<uint16_t> got(static_cast<size_t>(T) * H);
        GLB_CUDA_CHECK(cudaMemcpyAsync(got.data(), y.p, got.size() * 2, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (int t = 0; t < T; t++) {
          for (int c = 0; c < H; c++) {
            float acc = 0.0f;
            for (int x2 = 0; x2 < topk; x2++) {
              const int i = t * topk + x2;
              if (rank[i] < 0) continue;
              const float row = idx[i] / E == 0 ? bf16ToFloat(bf16(eoValue(static_cast<int>(idx[i] % E), rank[i], c)))
                                                : bf16ToFloat(pre[i * H + c]);
              const float prod = w[i] * row;
              acc = acc + prod;
            }
            uint32_t u;
            std::memcpy(&u, &acc, 4);
            const uint16_t want = static_cast<uint16_t>((u + 0x7fffu + ((u >> 16) & 1u)) >> 16);
            if (got[t * H + c] != want) {
              return strcat_all("y token ", t, " element ", c, ": got bf16 bits ", static_cast<int>(got[t * H + c]),
                                ", want ", static_cast<int>(want));
            }
          }
        }
        return "";
      });
    }

    // ---- literal schedule executor (halving-doubling, plain and pipelined) -------------------
    R.run(strcat_all("scheduleKernel<float>(halving_doubling) P=", P), [&]() -> std::string {
      fillAll();
      for (int pipelined = 0; pipelined < 2; pipelined++) {
        Schedule sc = pipelined ? buildHalvingDoublingPipelinedSchedule(0, P, n, 4, 2) : buildHalvingDoublingSchedule(0, P, n, 4);
        DevBuf table(sc.steps.size() * sizeof(SchedStep));
        GLB_CUDA_CHECK(cudaMemcpyAsync(table.p, sc.steps.data(), sc.steps.size() * sizeof(SchedStep), cudaMemcpyHostToDevice, stream));
        PeerPtrs st = pc.stagePtrs(pc.stageBytes() / 2);
        launchSchedule(ca, pp, st, static_cast<const SchedStep*>(table.p), static_cast<int>(sc.steps.size()), scheduleBarriers(sc),
                       DataType::FLOAT32, ReduceOp::SUM, 1.0f, n, true, std::min(pc.maxBlocks(), 16), stream);
        noteLaunch();
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      }
      return "";  // rank 0's partial view has no closed form here; completion without a hang is the check
    });
  }

  // ---- flag-in-data kernels: one rank (no peers to hear from), fused scale + cast -------------
  {
    const CommArgs one = pc.loopbackComm(1);
    R.run("allreduceNormKernel<float,layer,local>", [&]() -> std::string {
      return checkAllreduceNorm(one, NormXchg{}, kNormLocal, kNormLayer, 7, 4096, 0, 7, 4, stream);
    });
    R.run("llAllreduceKernel<float,float>", [&]() -> std::string {
      const size_t m = std::min<size_t>(pc.llMaxBytes() / 4, 4099);
      DevBuf in(m * 4), out(m * 4);
      launchFill(in.p, m, DataType::FLOAT32, 1.0, 1.0, stream);
      launchLLAllreduce(one, in.p, out.p, m, DataType::FLOAT32, DataType::FLOAT32, ReduceOp::SUM, 0.25f, pc.llPtrs(),
                        pc.llSrcStride(), pc.llParityStride(), LocalPtrs(), 4, 256, stream);
      noteLaunch();
      auto h = download(out.p, m, stream);
      for (size_t i = 0; i < m; i++) {
        if (!close(h[i], 0.25 * (1.0 + i))) return strcat_all("element ", i, ": got ", h[i]);
      }
      return "";
    });
    R.run("llAllreduceKernel<float,bf16> (cast epilogue)", [&]() -> std::string {
      const size_t m = 1001;
      DevBuf in(m * 4), out(m * 2);
      launchFill(in.p, m, DataType::FLOAT32, 3.0, 0.0, stream);
      launchLLAllreduce(one, in.p, out.p, m, DataType::FLOAT32, DataType::BFLOAT16, ReduceOp::SUM, 1.0f, pc.llPtrs(),
                        pc.llSrcStride(), pc.llParityStride(), LocalPtrs(), 1, 256, stream);
      noteLaunch();
      std::vector<uint16_t> h(m);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), out.p, m * 2, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < m; i++) {
        if (bf16ToFloat(h[i]) != 3.0f) return strcat_all("element ", i, ": got ", bf16ToFloat(h[i]));
      }
      return "";
    });
    R.run("llAllreduceKernel<e4m3,e4m3>", [&]() -> std::string {
      const size_t m = 1001;
      DevBuf in(m), out(m);
      launchFill(in.p, m, DataType::FLOAT8_E4M3, 1.5, 0.0, stream);
      launchLLAllreduce(one, in.p, out.p, m, DataType::FLOAT8_E4M3, DataType::FLOAT8_E4M3, ReduceOp::SUM, 0.25f,
                        pc.llPtrs(), pc.llSrcStride(), pc.llParityStride(), LocalPtrs(), 1, 256, stream);
      noteLaunch();
      std::vector<uint8_t> h(m);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), out.p, m, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < m; i++) {
        if (float8_e4m3::toFloat(h[i]) != 0.375f) return strcat_all("element ", i, ": got ", float8_e4m3::toFloat(h[i]));
      }
      return "";
    });
    R.run("llExchangeKernel", [&]() -> std::string {
      const size_t bytes = 1000;
      DevBuf in(bytes), out(bytes);
      GLB_CUDA_CHECK(cudaMemsetAsync(in.p, 0x5a, bytes, stream));
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, bytes, stream));
      launchLLExchange(one, in.p, out.p, bytes, 0, pc.llPtrs(), pc.llSrcStride(), pc.llParityStride(), 1, 128, stream);
      noteLaunch();
      std::vector<unsigned char> h(bytes);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), out.p, bytes, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (size_t i = 0; i < bytes; i++) {
        if (h[i] != 0x5a) return strcat_all("byte ", i, " wrong");
      }
      return "";
    });
  }

  // ---- pipelined kernel for plain pointers (P virtual ranks alias my pool) ---------------------
  for (int P : {2, 8}) {
    R.run(strcat_all("pipelinedAllreduceKernel<float,false,", P, ">"), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const size_t bulkOff = 2 * half;
      PeerPtrs st;
      std::memset(&st, 0, sizeof(st));
      for (int r = 0; r < P; r++) st.p[r] = myStage + bulkOff;
      const int blocks = std::min(pc.coResidentBlocks(pipelinedKernelFor(DataType::FLOAT32, false, P)), 8), tile = 64;
      const size_t chunkVecs = static_cast<size_t>(P) * blocks * tile;
      GLB_ENFORCE_LE(3 * chunkVecs * 16, pc.stageBytes() - bulkOff, "pool too small for the pipelined self-test");
      DevBuf in(n * 4), out(n * 4);
      launchFill(in.p, n, DataType::FLOAT32, 1.0, 0.0, stream);
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, n * 4, stream));
      launchPipelinedAllreduce(ca, in.p, out.p, n, DataType::FLOAT32, ReduceOp::SUM, 1.0f, st, nullptr, tile, 256, LocalPtrs(),
                               blocks, stream);
      noteLaunch();
      auto h = download(out.p, n, stream);
      // Rank 0 reduces share 0 of every chunk (P reads of its own copy -> P x 1); the other
      // shares pass through the pool untouched.
      for (size_t i = 0; i < n; i++) {
        const size_t w = (i / 4) % chunkVecs;
        const double want = w < static_cast<size_t>(blocks) * tile ? P : 1.0;
        if (!close(h[i], want)) return strcat_all("element ", i, ": got ", h[i], " want ", want);
      }
      return "";
    });
  }

  // ---- pipelined allgather / reduce_scatter for plain pointers (same aliasing) -----------------
  // Every virtual rank's slot is my slot, so every block rank 0 pulls is its own input, and the
  // share it reduces is P copies of share 0 of its input.
  auto aliasedBulk = [&](int P) {
    PeerPtrs st;
    std::memset(&st, 0, sizeof(st));
    for (int r = 0; r < P; r++) st.p[r] = myStage + 2 * half;
    return st;
  };
  for (int P : {2, 8}) {
    for (size_t shift : {size_t(0), size_t(1)}) {
      R.run(strcat_all("pipelinedAllgatherKernel P=", P, shift ? " (out 1 byte off)" : ""), [&]() -> std::string {
        const CommArgs ca = pc.loopbackComm(P);
        const int blocks = std::min(pc.coResidentBlocks(pipelinedAllgatherKernelPtr()), 8), tile = 64;
        const size_t C = static_cast<size_t>(blocks) * tile * 16;
        GLB_ENFORCE_LE(2 * C, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
        const size_t bytes = 5 * C + 36;  // five whole chunks and a part that is not a whole 16-byte group
        std::vector<size_t> offs(P), lens(P, bytes);
        for (int r = 0; r < P; r++) offs[r] = r * bytes;
        DevBuf in(bytes), out(P * bytes + shift);
        launchFill(in.p, bytes / 4, DataType::FLOAT32, 1.0, 1.0, stream);
        GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
        launchPipelinedAllgather(ca, in.p, static_cast<char*>(out.p) + shift, offs.data(), lens.data(), -1, aliasedBulk(P),
                                 tile, 256, blocks, stream);
        noteLaunch();
        std::vector<char> hin(bytes), hout(out.bytes);
        GLB_CUDA_CHECK(cudaMemcpyAsync(hin.data(), in.p, bytes, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaMemcpyAsync(hout.data(), out.p, out.bytes, cudaMemcpyDeviceToHost, stream));
        GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
        for (int r = 0; r < P; r++) {
          if (std::memcmp(hout.data() + shift + offs[r], hin.data(), bytes) != 0) return strcat_all("block ", r, " differs");
        }
        return "";
      });
    }
  }
  // P = 3 runs the generic-P instantiation; P = 8 has uneven shares and an output one element off.
  for (int P : {2, 8, 3}) {
    R.run(strcat_all("pipelinedReduceScatterKernel<float,", P == 3 ? 0 : P, "> P=", P), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const void* k = pipelinedReduceScatterKernelFor(DataType::FLOAT32, P);
      const int blocks = std::min(pc.coResidentBlocks(k), 8), tile = 32;
      const size_t chunkElems = static_cast<size_t>(blocks) * tile * 4;
      GLB_ENFORCE_LE(2 * P * chunkElems * 4, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
      std::vector<size_t> counts(P), off(P + 1, 0);
      for (int r = 0; r < P; r++) {
        counts[r] = 3 * chunkElems + (P == 2 ? 0 : 7 + 5 * r);
        off[r + 1] = off[r] + counts[r];
      }
      const size_t shift = P == 8 ? 1 : 0;
      DevBuf in(off[P] * 4), out((counts[0] + shift) * 4);
      launchFill(in.p, off[P], DataType::FLOAT32, 0.0, 1.0, stream);  // share 0 = 0, 1, 2, ...
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
      launchPipelinedReduceScatter(ca, in.p, static_cast<float*>(out.p) + shift, off.data(), counts.data(),
                                   DataType::FLOAT32, ReduceOp::SUM, 0.5f, aliasedBulk(P), tile, 256, blocks, stream);
      noteLaunch();
      auto h = download(out.p, counts[0] + shift, stream);
      for (size_t i = 0; i < counts[0]; i++) {
        const double want = 0.5 * P * static_cast<double>(i);
        if (!close(h[i + shift], want)) return strcat_all("element ", i, ": got ", h[i + shift], " want ", want);
      }
      return "";
    });
  }
  // The cast forms of the two. Allgather: f32 in, bf16 blocks rounded on the copy-in, every block
  // rank 0's. Reduce-scatter: share 0 of the bf16 input is 0, 1, 2, ... (bf16-rounded), the fp32
  // result P x 0.5 x that, exact in fp32 (P = 3 needs more than bf16's 8 bits above 256).
  for (int P : {2, 8}) {
    R.run(strcat_all("castPipelinedAllgatherKernel<bf16> P=", P), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const int blocks = std::min(pc.coResidentBlocks(castPipelinedAllgatherKernelFor(DataType::BFLOAT16)), 8), tile = 64;
      const size_t C = static_cast<size_t>(blocks) * tile * 16;
      GLB_ENFORCE_LE(2 * C, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
      const size_t count = (5 * C + 36) / 2;  // five whole chunks and a part that is not a whole 16-byte group
      std::vector<size_t> offs(P), lens(P, count * 2);
      for (int r = 0; r < P; r++) offs[r] = r * count * 2;
      DevBuf in(count * 4), out(P * count * 2);
      launchFill(in.p, count, DataType::FLOAT32, 1.0, 1.0 / 3.0, stream);
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
      launchCastPipelinedAllgather(ca, in.p, out.p, DataType::BFLOAT16, offs.data(), lens.data(), aliasedBulk(P), tile,
                                   256, blocks, stream);
      noteLaunch();
      auto x = download(in.p, count, stream);
      std::vector<uint16_t> h(P * count);
      GLB_CUDA_CHECK(cudaMemcpyAsync(h.data(), out.p, out.bytes, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (int r = 0; r < P; r++) {
        for (size_t i = 0; i < count; i++) {
          if (h[r * count + i] != floatToBf16(x[i])) return strcat_all("block ", r, " element ", i, " differs");
        }
      }
      return "";
    });
  }
  for (int P : {2, 8, 3}) {
    R.run(strcat_all("castPipelinedReduceScatterKernel<bf16,", P == 3 ? 0 : P, "> P=", P), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const void* k = castPipelinedReduceScatterKernelFor(DataType::BFLOAT16, P);
      const int blocks = std::min(pc.coResidentBlocks(k), 8), tile = 32;
      const size_t chunkElems = static_cast<size_t>(blocks) * tile * 8;
      GLB_ENFORCE_LE(2 * P * chunkElems * 2, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
      std::vector<size_t> counts(P), off(P + 1, 0);
      for (int r = 0; r < P; r++) {
        counts[r] = 3 * chunkElems + (P == 2 ? 0 : 7 + 5 * r);
        off[r + 1] = off[r] + counts[r];
      }
      const size_t shift = P == 8 ? 1 : 0;
      DevBuf in(off[P] * 2), out((counts[0] + shift) * 4);
      launchFill(in.p, off[P], DataType::BFLOAT16, 0.0, 1.0, stream);
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
      launchCastPipelinedReduceScatter(ca, in.p, static_cast<float*>(out.p) + shift, off.data(), counts.data(),
                                       DataType::BFLOAT16, 0.5f, aliasedBulk(P), tile, 256, blocks, stream);
      noteLaunch();
      std::vector<uint16_t> x(counts[0]);
      GLB_CUDA_CHECK(cudaMemcpyAsync(x.data(), in.p, counts[0] * 2, cudaMemcpyDeviceToHost, stream));
      auto h = download(out.p, counts[0] + shift, stream);
      for (size_t i = 0; i < counts[0]; i++) {
        const double want = 0.5 * P * static_cast<double>(bf16ToFloat(x[i]));
        if (h[i + shift] != want) return strcat_all("element ", i, ": got ", h[i + shift], " want ", want);
      }
      return "";
    });
  }
  // One rank's form: f16 -> f32 scaled, and f32 -> bf16.
  R.run("castScaleKernel<f16,float> / <float,bf16>", [&]() -> std::string {
    const size_t count = 200 * 8 + 5;
    DevBuf a(count * 2), b(count * 4), c(count * 2);
    launchFill(a.p, count, DataType::FLOAT16, -100.0, 0.125, stream);  // exact in f16
    launchCastScale(a.p, DataType::FLOAT16, b.p, DataType::FLOAT32, count, 3.0f, 16, stream);
    launchCastScale(b.p, DataType::FLOAT32, c.p, DataType::BFLOAT16, count, 1.0f, 16, stream);
    noteLaunch(2);
    auto h = download(b.p, count, stream);
    std::vector<uint16_t> hc(count);
    GLB_CUDA_CHECK(cudaMemcpyAsync(hc.data(), c.p, count * 2, cudaMemcpyDeviceToHost, stream));
    GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
    for (size_t i = 0; i < count; i++) {
      const float want = 3.0f * static_cast<float>(-100.0 + 0.125 * static_cast<double>(i));
      if (h[i] != want) return strcat_all("f32 element ", i, ": got ", h[i], " want ", want);
      if (hc[i] != floatToBf16(want)) return strcat_all("bf16 element ", i, " differs");
    }
    return "";
  });
  // reduce to root 0 with every virtual rank's slots aliasing mine: rank 0 stores P copies of share 0
  // of its input as its own share, and pulls every other share from "peer q's" result slot, which is
  // its own, which a root never writes: zero, as cleared here. The output starts filled with NaN.
  // P = 2 has even shares; P = 8 uneven ones and an output one element off; P = 3 is generic.
  for (int P : {2, 8, 3}) {
    R.run(strcat_all("pipelinedReduceKernel<float,", P == 3 ? 0 : P, "> P=", P), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const int blocks = std::min(pc.coResidentBlocks(pipelinedReduceKernelFor(DataType::FLOAT32, P)), 8), tile = 32;
      const size_t chunkElems = static_cast<size_t>(blocks) * tile * 4, C = chunkElems * 4;
      GLB_ENFORCE_LE((2 * P + 2) * C, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
      const size_t count = P * 3 * chunkElems + (P == 2 ? 0 : 5);
      std::vector<size_t> counts(P), off(P + 1, 0);
      for (int r = 0; r < P; r++) {
        counts[r] = count / P + (static_cast<size_t>(r) < count % P ? 1 : 0);
        off[r + 1] = off[r] + counts[r];
      }
      const size_t shift = P == 8 ? 1 : 0;
      DevBuf in(count * 4), out((count + shift) * 4);
      launchFill(in.p, count, DataType::FLOAT32, 0.0, 1.0, stream);
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0xff, out.bytes, stream));
      GLB_CUDA_CHECK(cudaMemsetAsync(myStage + 2 * half + 2 * P * C, 0, 2 * C, stream));
      launchPipelinedReduce(ca, in.p, static_cast<float*>(out.p) + shift, off.data(), counts.data(), 0, DataType::FLOAT32,
                            ReduceOp::SUM, aliasedBulk(P), tile, 256, blocks, stream);
      noteLaunch();
      auto h = download(out.p, count + shift, stream);
      for (size_t i = 0; i < count; i++) {
        const double want = i < counts[0] ? static_cast<double>(P) * i : 0.0;
        if (!close(h[i + shift], want)) return strcat_all("element ", i, ": got ", h[i + shift], " want ", want);
      }
      return "";
    });
  }
  // alltoall(v): virtual peer q's pool is my pool shifted by q sub-slots, so sub-slot 0 of its slot
  // is sub-slot q of mine and rank 0 pulls back its own block for destination q. Blocks are uneven
  // (some empty, some several chunks), received in the reverse order, into an output one byte off.
  for (int P : {2, 8}) {
    R.run(strcat_all("pipelinedAlltoallKernel P=", P, " (uneven blocks, out 1 byte off)"), [&]() -> std::string {
      const CommArgs ca = pc.loopbackComm(P);
      const int blocks = std::min(pc.coResidentBlocks(pipelinedAlltoallKernelPtr()), 8), tile = 64;
      const size_t C = static_cast<size_t>(blocks) * tile * 16;
      GLB_ENFORCE_LE(2 * P * C, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
      std::vector<size_t> len(P), soff(P, 0), roff(P, 0);
      for (int j = 0; j < P; j++) len[j] = j % 3 == 2 ? 0 : (j % 4 + 1) * C + 13 * j + 3;
      for (int j = 1; j < P; j++) soff[j] = soff[j - 1] + len[j - 1];
      for (int j = P - 2; j >= 0; j--) roff[j] = roff[j + 1] + len[j + 1];
      const size_t total = soff[P - 1] + len[P - 1];
      PeerPtrs st;
      std::memset(&st, 0, sizeof(st));
      for (int q = 0; q < P; q++) st.p[q] = myStage + 2 * half + q * C;
      DevBuf in(total), out(total + 1);
      launchFill(in.p, total / 4, DataType::FLOAT32, 1.0, 1.0, stream);
      GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
      launchPipelinedAlltoall(ca, in.p, static_cast<char*>(out.p) + 1, soff.data(), len.data(), roff.data(), len.data(),
                              st, tile, 256, blocks, stream);
      noteLaunch();
      std::vector<char> hin(total), hout(out.bytes);
      GLB_CUDA_CHECK(cudaMemcpyAsync(hin.data(), in.p, total, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaMemcpyAsync(hout.data(), out.p, out.bytes, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      for (int j = 0; j < P; j++) {
        if (std::memcmp(hout.data() + 1 + roff[j], hin.data() + soff[j], len[j]) != 0) return strcat_all("block ", j, " differs");
      }
      return hout[0] == 0 ? "" : "wrote before the output";
    });
  }
  // The scatter form at root 0, the root's path: it stages the blocks for the other ranks and copies
  // its own block straight to its output; it receives from nobody else.
  R.run("pipelinedAlltoallKernel (scatter, root 0) P=4", [&]() -> std::string {
    const int P = 4;
    const CommArgs ca = pc.loopbackComm(P);
    const int blocks = std::min(pc.coResidentBlocks(pipelinedAlltoallKernelPtr()), 8), tile = 64;
    const size_t C = static_cast<size_t>(blocks) * tile * 16, bytes = 3 * C + 20;
    GLB_ENFORCE_LE(2 * P * C, pc.stageBytes() - 2 * half, "pool too small for the pipelined self-test");
    std::vector<size_t> slen(P, bytes), soff(P), rlen(P, 0), roff(P, 0);
    for (int j = 0; j < P; j++) soff[j] = j * bytes;
    rlen[0] = bytes;
    DevBuf in(P * bytes), out(bytes + 16);
    launchFill(in.p, P * bytes / 4, DataType::FLOAT32, 0.0, 1.0, stream);
    GLB_CUDA_CHECK(cudaMemsetAsync(out.p, 0, out.bytes, stream));
    launchPipelinedAlltoall(ca, in.p, out.p, soff.data(), slen.data(), roff.data(), rlen.data(), aliasedBulk(P), tile, 256,
                            blocks, stream);
    noteLaunch();
    std::vector<char> hin(bytes), hout(out.bytes);
    GLB_CUDA_CHECK(cudaMemcpyAsync(hin.data(), in.p, bytes, cudaMemcpyDeviceToHost, stream));
    GLB_CUDA_CHECK(cudaMemcpyAsync(hout.data(), out.p, out.bytes, cudaMemcpyDeviceToHost, stream));
    GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
    if (std::memcmp(hout.data(), hin.data(), bytes) != 0) return "block 0 differs";
    for (size_t i = bytes; i < out.bytes; i++) {
      if (hout[i] != 0) return "wrote past the output";
    }
    return "";
  });

  // ---- point to point: fused send + recv through my own mailbox --------------------------------
  R.run("p2pKernel(sendrecv)", [&]() -> std::string {
    const CommArgs ca = pc.loopbackComm(2);
    const auto& o = pc.options();
    PeerPtrs mb = pc.mailboxPtrs();
    char* base = static_cast<char*>(mb.p[pc.rank]);
    // "rank 1"'s box for source 0 is my box for source 1.
    mb.p[0] = base;
    mb.p[1] = base + pc.mailboxStride();
    const size_t bytes = 3 * o.p2pSlotBytes * o.p2pSlots / 2 + 20;  // more than the ring holds: must stream
    DevBuf src(bytes), dst(bytes);
    launchFill(src.p, bytes / 4, DataType::FLOAT32, 0.0, 1.0, stream);
    GLB_CUDA_CHECK(cudaMemsetAsync(dst.p, 0, bytes, stream));
    launchP2p(ca, src.p, bytes / 4 * 4, 1, dst.p, bytes / 4 * 4, 1, mb, pc.mailboxStride(), o.p2pSlotBytes, o.p2pSlots,
              std::min(o.p2pLanes, std::max(1, pc.maxBlocks() / 2)), stream);
    noteLaunch();
    auto h = download(dst.p, bytes / 4, stream);
    for (size_t i = 0; i < bytes / 4; i++) {
      if (!close(h[i], static_cast<double>(i))) return strcat_all("element ", i, ": got ", h[i]);
    }
    return "";
  });

  for (bool tma : {false, true}) {
    R.run(tma ? "exchangeKernel<true> (zero-copy sendrecv, TMA)" : "exchangeKernel<false> (zero-copy sendrecv)",
          [&]() -> std::string {
            const CommArgs ca = pc.loopbackComm(2);
            const size_t bytes = (5u << 20) + 16 + 4;
            DevBuf src(bytes), dst(bytes);
            for (int round = 0; round < 2; round++) {  // twice: the counters must carry over
              launchFill(src.p, bytes / 4, DataType::FLOAT32, 0.0, 1.0 + round, stream);
              GLB_CUDA_CHECK(cudaMemsetAsync(dst.p, 0, bytes, stream));
              launchExchange(ca, src.p, bytes, 1, dst.p, bytes, 1, std::min(pc.maxBlocks(), 24), tma, stream);
              noteLaunch();
              auto h = download(dst.p, bytes / 4, stream);
              for (size_t i = 0; i < bytes / 4; i++) {
                if (!close(h[i], static_cast<double>(i) * (1.0 + round))) return strcat_all("round ", round, " element ", i, ": got ", h[i]);
              }
            }
            return "";
          });
  }

  R.run("peerBulkCopyKernel (put / get, TMA)", [&]() -> std::string {
    const size_t bytes = (3u << 20) + 48 + 5;  // 16-byte body + a byte tail
    DevBuf src(bytes), dst(bytes);
    launchFill(src.p, bytes / 4, DataType::FLOAT32, 0.0, 1.0, stream);
    GLB_CUDA_CHECK(cudaMemsetAsync(dst.p, 0, bytes, stream));
    launchPeerCopy(dst.p, src.p, bytes, 24, stream, /*tma=*/true);
    noteLaunch();
    auto h = download(dst.p, bytes / 4, stream);
    for (size_t i = 0; i < bytes / 4; i++) {
      if (!close(h[i], static_cast<double>(i))) return strcat_all("element ", i, ": got ", h[i]);
    }
    return "";
  });

  // ---- NVLS kernels on a one-device multicast object (when the driver allows it) ----------------
  R.run("nvlsAllreduceKernel<float,4> (1-device multicast)", [&]() -> std::string {
    std::string why;
    auto mcbuf = pc.tryAllocMulticastLoopback(n * 4, &why);
    if (!mcbuf) return "skipped: " + why;
    const CommArgs ca = pc.loopbackComm(4);
    PeerPtrs pp;
    std::memset(&pp, 0, sizeof(pp));
    for (int r = 0; r < 4; r++) pp.p[r] = mcbuf->local;
    launchFill(mcbuf->local, n, DataType::FLOAT32, 1.0, 1.0, stream);
    LaunchCfg cfg;
    cfg.blocks = std::min(pc.maxBlocks(), 32);
    cfg.unroll = 4;
    launchNvlsAllreduce(ca, mcbuf->mc, pp, n / 4 * 4, DataType::FLOAT32, 3.0f, LocalPtrs(), cfg, stream);
    noteLaunch();
    auto h = download(mcbuf->local, n / 4 * 4, stream);
    size_t vb, ve;
    shareOfHost(n / 4, 4, 0, vb, ve);
    for (size_t i = 0; i < n / 4 * 4; i++) {
      const double want = (i / 4 >= vb && i / 4 < ve) ? 3.0 * (1.0 + i) : 1.0 + i;
      if (!close(h[i], want)) return strcat_all("element ", i, ": got ", h[i], " want ", want);
    }
    return "";
  });

  // ---- local kernels ------------------------------------------------------------------------------
  R.run("localAllreduceManyKernel<float>", [&]() -> std::string {
    DevBuf a(n * 4), b(n * 4), c(n * 4);
    launchFill(a.p, n, DataType::FLOAT32, 0.0, 3.0, stream);
    launchFill(b.p, n, DataType::FLOAT32, 1.0, 3.0, stream);
    launchFill(c.p, n, DataType::FLOAT32, 2.0, 3.0, stream);
    void* all[3] = {a.p, b.p, c.p};
    TileCounter tiles(pc.device);
    launchLocalAllreduceMany(all, 3, n, DataType::FLOAT32, ReduceOp::SUM, 1.0f, tiles.get(), stream);
    noteLaunch();
    DevBuf res(16);
    unsigned long long init[2] = {0ull, ~0ull};
    GLB_CUDA_CHECK(cudaMemcpyAsync(res.p, init, 16, cudaMemcpyHostToDevice, stream));
    launchVerify(c.p, n, DataType::FLOAT32, 3.0, 9.0, 1e-5, 1e-6, static_cast<unsigned long long*>(res.p), stream);
    unsigned long long got[2];
    GLB_CUDA_CHECK(cudaMemcpyAsync(got, res.p, 16, cudaMemcpyDeviceToHost, stream));
    GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
    return got[0] == 0 ? "" : strcat_all(got[0], " mismatches, first at ", got[1] - 1);
  });
  R.run("localAllreduceManyBulkKernel<float>", [&]() -> std::string {
    const size_t m = (size_t(1) << 20) + 5;  // 4 MB: whole tiles, then packs, then single elements
    DevBuf a(m * 4), b(m * 4);
    launchFill(a.p, m, DataType::FLOAT32, 0.0, 2.0, stream);
    launchFill(b.p, m, DataType::FLOAT32, 1.0, 2.0, stream);
    void* all[2] = {a.p, b.p};
    if (!localAllreduceUsesBulk(all, 2, m, DataType::FLOAT32)) return "the size no longer selects the bulk kernel";
    TileCounter tiles(pc.device);
    launchLocalAllreduceMany(all, 2, m, DataType::FLOAT32, ReduceOp::SUM, 0.5f, tiles.get(), stream);
    noteLaunch();
    DevBuf res(16);
    unsigned long long init[2] = {0ull, ~0ull};
    unsigned long long got[2];
    for (void* p : all) {
      GLB_CUDA_CHECK(cudaMemcpyAsync(res.p, init, 16, cudaMemcpyHostToDevice, stream));
      launchVerify(p, m, DataType::FLOAT32, 0.5, 2.0, 1e-6, 0.0, static_cast<unsigned long long*>(res.p), stream);
      GLB_CUDA_CHECK(cudaMemcpyAsync(got, res.p, 16, cudaMemcpyDeviceToHost, stream));
      GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
      if (got[0] != 0) return strcat_all(got[0], " mismatches, first at ", got[1] - 1);
    }
    return "";
  });

  GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
  pc.checkHealth();
  return R.results;
}

// A barrier whose only peer never shows up: the kernel must give up after the timeout,
// leave the GPU usable and poison the context (the caller sees IoException).
bool loopbackTimeoutTest(PeerContext& pc, cudaStream_t stream, int timeoutMs, double* elapsedMs) {
  DeviceGuard g(pc.device);
  CommArgs ca = pc.loopbackComm(2);
  // Virtual rank 1's pad lives elsewhere: my flag for it lands there, its flag for me never comes.
  DevBuf lonely(sizeof(SignalPad));
  GLB_CUDA_CHECK(cudaMemsetAsync(lonely.p, 0, sizeof(SignalPad), stream));
  ca.sig[1] = static_cast<SignalPad*>(lonely.p);  // (ca.self stays my real pad)
  ca.timeoutNs = static_cast<unsigned long long>(timeoutMs) * 1000000ull;
  cudaEvent_t a, b;
  GLB_CUDA_CHECK(cudaEventCreate(&a));
  GLB_CUDA_CHECK(cudaEventCreate(&b));
  GLB_CUDA_CHECK(cudaEventRecord(a, stream));
  launchBarrier(ca, stream);
  GLB_CUDA_CHECK(cudaEventRecord(b, stream));
  GLB_CUDA_CHECK(cudaStreamSynchronize(stream));
  float ms = 0;
  cudaEventElapsedTime(&ms, a, b);
  cudaEventDestroy(a);
  cudaEventDestroy(b);
  if (elapsedMs != nullptr) *elapsedMs = ms;
  try {
    pc.checkHealth();
  } catch (const IoException&) {
    return true;
  }
  return false;
}

// LocalOp classes (cuda/local_ops.h) on one device: memcpy, native / host reduce and
// broadcast, and the dispatchers. The NCCL flavours need one GPU per pointer and are
// exercised when `devices` names several.
std::vector<SelfTestResult> localOpsSelfTest(const std::vector<int>& devices, size_t count) {
  std::vector<SelfTestResult> out;
  auto run = [&](const std::string& name, auto&& body) {
    SelfTestResult r;
    r.name = name;
    try {
      r.detail = body();
      r.ok = r.detail.empty();
    } catch (const std::exception& e) {
      r.detail = e.what();
    }
    out.push_back(r);
  };
  const int n = static_cast<int>(devices.size());
  GLB_ENFORCE_GE(n, 1);
  std::vector<CudaDevicePointer<float>> ptrs;
  std::vector<CudaStream> streams;
  const int nptr = n >= 2 ? n : 3;  // several devices: one pointer each (what the NCCL flavours need)
  for (int i = 0; i < nptr; i++) {
    const int dev = devices[i % n];
    DeviceGuard g(dev);
    ptrs.push_back(CudaDevicePointer<float>::alloc(count));
    streams.emplace_back(dev);
  }
  auto fill = [&] {
    for (int i = 0; i < nptr; i++) {
      DeviceGuard g(ptrs[i].getDeviceID());
      launchFill(*ptrs[i], count, DataType::FLOAT32, i, nptr, *streams[i]);
    }
  };
  const double tri = nptr * (nptr - 1) / 2.0;
  auto check = [&](const float* host, double start, double stride) -> std::string {
    for (size_t i = 0; i < count; i++) {
      if (!close(host[i], start + stride * static_cast<double>(i))) return strcat_all("element ", i, ": got ", host[i]);
    }
    return "";
  };
  auto host = CudaHostPointer<float>::alloc(count);

  run("CudaLocalMemcpy (device -> host)", [&]() -> std::string {
    fill();
    CudaLocalMemcpy<float, CudaDevicePointer<float>, CudaHostPointer<float>> cp(streams[0], ptrs[0], host, 0, count);
    cp.run();
    return check(*host, 0, nptr);
  });
  run("cudaDeviceReduce + cudaDeviceBroadcast", [&]() -> std::string {
    fill();
    auto red = cudaDeviceReduce<float>(streams, ptrs, ptrs[0], CudaReductionFunction<float>::sum, 0, count);
    red->run();
    auto bc = cudaDeviceBroadcast<float>(streams, ptrs, ptrs[0], 0, count);
    bc->run();
    CudaLocalMemcpy<float, CudaDevicePointer<float>, CudaHostPointer<float>> cp(streams[nptr - 1], ptrs[nptr - 1], host, 0, count);
    cp.run();
    return check(*host, tri, static_cast<double>(nptr) * nptr);
  });
  run("cudaHostReduce (device fold) + cudaHostBroadcast", [&]() -> std::string {
    fill();
    auto red = cudaHostReduce<float>(streams, ptrs, host, CudaReductionFunction<float>::sum, 0, count);
    red->run();
    std::string why = check(*host, tri, static_cast<double>(nptr) * nptr);
    if (!why.empty()) return why;
    auto bc = cudaHostBroadcast<float>(streams, ptrs, host, 0, count);
    bc->run();
    auto back = CudaHostPointer<float>::alloc(count);
    CudaLocalMemcpy<float, CudaDevicePointer<float>, CudaHostPointer<float>> cp(streams[1], ptrs[1], back, 0, count);
    cp.run();
    return check(*back, tri, static_cast<double>(nptr) * nptr);
  });
  run("CudaLocalHostReduce (CPU fold)", [&]() -> std::string {
    fill();
    CudaLocalHostReduce<float> red(streams, ptrs, host, CudaReductionFunction<float>::sum, 0, count);
    red.run();
    return check(*host, tri, static_cast<double>(nptr) * nptr);
  });
  if (n >= 2 && n == nptr && ncclAvailable()) {
    run("CudaLocalNCCLReduce + CudaLocalNCCLBroadcast", [&]() -> std::string {
      fill();
      CudaLocalNCCLReduce<float> red(streams, ptrs, ptrs[0], CudaReductionFunction<float>::sum, 0, count);
      red.run();
      CudaLocalNCCLBroadcast<float> bc(streams, ptrs, ptrs[0], 0, count);
      bc.run();
      CudaLocalMemcpy<float, CudaDevicePointer<float>, CudaHostPointer<float>> cp(streams[n - 1], ptrs[n - 1], host, 0, count);
      cp.run();
      return check(*host, tri, static_cast<double>(nptr) * nptr);
    });
  }
  return out;
}

}  // namespace cuda
}  // namespace glb
