"""The FP8 form of the fused residual norm: `out` as e4m3 codes with one fp32 scale per row.

The contract is exact: the FP8 call's `residual_out` is the unquantised call's, byte for byte, and
its codes and scales are `strategies.fp8_rows` (the torch quantisation) of the unquantised call's
`out`, byte for byte. Every GPU check runs both calls on the same inputs and compares bytes; the
unquantised `out` itself is checked against fp64 in test_allreduce_norm.py and
test_sequence_parallel_norm.py.

Ranks are threads sharing cuda:0, as in the other GPU tests; each rank's thread checks its own
results and returns digests, which must be equal on every rank.
"""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.models import DenseBlock, TPBlock
from gloo_b200.ops import cuda as gcu
from gloo_b200.parallel import SequenceParallel, TensorParallel
from gloo_b200.parallel.strategies import fp8_rows
from test_allreduce_norm import EPS, MAIN, _digest, _guarded, _guards_intact, _kind, _launches
from test_reduce_numerics import _gen

E4M3 = torch.float8_e4m3fn
NORMS = ("rms", "layer")
ALGOS = ("auto", "ll", "one_shot", "two_shot")
# (T, H): every T with every H at decode sizes; prefill-sized T at the narrower rows
SHAPES = [(t, h) for t in (1, 3, 17) for h in (16, 4096, 7168, 16384)] + [(1000, 16), (1000, 4096)]


def _bytes(t):
    return t.contiguous().view(torch.uint8)


def _spawn(P, fn, stage_bytes=64 << 20):
    def body(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=stage_bytes)
        cc.set_timeout(120000)
        return fn(ctx, cc)

    return gb.spawn_threads(P, body, cuda_device=0, timeout_ms=600000)


def _problem(key, rank, T, H, dtype, norm, with_bias=True, Tres=None):
    """This rank's partial (T, H) and the shared residual (Tres rows), bias, weight and norm_bias."""
    g, g0 = _gen(key, rank), _gen(key, 0)
    partial = (3 * torch.randn(T, H, generator=g)).to(dtype).cuda()
    residual = torch.randn(T if Tres is None else Tres, H, generator=g0).to(dtype).cuda()
    bias = torch.randn(H, generator=g0).to(dtype).cuda() if with_bias else None
    w = (0.5 + torch.rand(H, generator=g0)).to(dtype).cuda()
    nb = torch.randn(H, generator=g0).to(dtype).cuda() if norm == "layer" else None
    return partial, residual, bias, w, nb


def _plan_tp(cc, T, H, dtype, norm, algo, fp8):
    return gb._C.cuda.plan_residual_norm(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)), _kind(norm),
                                         gcu._algo(algo), fp8)


def _plan_sp(cc, T, H, dtype, norm, gather, fp8):
    return gb._C.cuda.plan_reduce_scatter_norm(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)), _kind(norm), gather,
                                               fp8)


def _fp8_outputs(rows, H, dtype):
    """Guarded residual_out (rows, H) of dtype, codes (rows, H) and scales (rows, 1)."""
    rraw, rout = _guarded((rows, H), dtype)
    craw, codes = _guarded((rows, H), E4M3)
    sraw, scales = _guarded((rows, 1), torch.float32)
    return (rraw, craw, sraw), rout, codes, scales


def _check_fp8(what, want_r, want_o, rout, codes, scales, raws):
    """The FP8 call's outputs against the unquantised call's: failures."""
    bad = []
    want_c, want_s = fp8_rows(want_o)
    if not torch.equal(_bytes(rout), _bytes(want_r)):
        bad.append(f"{what}: residual_out differs from the unquantised call's")
    if not torch.equal(_bytes(codes), _bytes(want_c)):
        n = int((_bytes(codes) != _bytes(want_c)).sum())
        bad.append(f"{what}: {n} codes differ from the torch quantisation")
    if not torch.equal(_bytes(scales), _bytes(want_s)):
        bad.append(f"{what}: scales differ from the torch quantisation")
    for raw, name in zip(raws, ("residual_out", "codes", "scales")):
        if not _guards_intact(raw):
            bad.append(f"{what}: wrote outside {name}")
    return bad


def _tp_cases(P):
    out, i = [], 0
    for dtype in MAIN:
        for norm in NORMS:
            for with_bias in (True, False):
                for algo in ALGOS:
                    T, H = SHAPES[(i + 3 * P) % len(SHAPES)]
                    out.append((dtype, norm, with_bias, algo, T, H))
                    i += 1
    return out


def _run_tp_case(cc, P, rank, case):
    dtype, norm, with_bias, algo, T, H = case
    partial, res, b, w, nb = _problem(("tp", case), rank, T, H, dtype, norm, with_bias)
    inputs = [t for t in (partial, res, b, w, nb) if t is not None]
    kept = [t.clone() for t in inputs]
    want_r, want_o = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b,
                                                residual_out=torch.empty_like(res), algo=algo)
    raws, rout, codes, scales = _fp8_outputs(T, H, dtype)
    plan = _plan_tp(cc, T, H, dtype, norm, algo, True)
    got = {}

    def call():
        got["r"] = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b, residual_out=rout,
                                              out=codes, algo=algo, out_scales=scales)

    n = _launches(cc, call)
    bad = _check_fp8(f"rank {rank} {case}", want_r, want_o, rout, codes, scales, raws)
    if got["r"][0] is not rout or got["r"][1] is not codes:
        bad.append(f"rank {rank} {case}: returned other tensors than (residual_out, out)")
    if n != P * plan["launches"] or plan["launches"] != -(-T // plan["chunk_rows"]):
        bad.append(f"rank {rank} {case}: {n} launches over {P} ranks, plan {plan}")
    if not all(torch.equal(t, k) for t, k in zip(inputs, kept)):
        bad.append(f"rank {rank} {case}: an input changed")
    return bad, (_digest(rout), _digest(codes), _digest(scales))


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_allreduce_fp8_equals_torch_quantisation(P):
    """Every dtype x norm x bias x algo over T in {1, 3, 17, 1000} and H in {16, 4096, 7168, 16384}:
    residual_out and the codes and scales byte for byte, the same bytes on every rank, guard bands,
    inputs and one launch per chunk."""
    cases = _tp_cases(P)

    def fn(ctx, cc):
        bad, digests = [], []
        for case in cases:
            b, d = _run_tp_case(cc, P, ctx.rank, case)
            bad += b
            digests.append(d)
        return bad, digests

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    assert not bad, "\n".join(bad[:40])
    assert len({tuple(d) for _, d in results}) == 1, "ranks got different bytes"


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3, 4, 8])
def test_reduce_scatter_fp8_equals_allreduce_rows(P):
    """The SP form's codes and scales (gathered or this rank's shard) equal the matching rows of the
    TP FP8 form, and residual_out its rows; guard bands, launches and identical gathered bytes."""
    cases = [(dtype, norm, Ts, H) for dtype in MAIN for norm in NORMS for Ts, H in ((1, 16), (3, 7168), (40, 4096))]

    def fn(ctx, cc):
        bad, digests = [], []
        for dtype, norm, Ts, H in cases:
            T = P * Ts
            partial, res, b, w, nb = _problem(("sp", dtype, norm, Ts, H), ctx.rank, T, H, dtype, norm)
            full_s = torch.empty(T, 1, dtype=torch.float32, device="cuda")
            full_r, full_c = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b,
                                                        residual_out=torch.empty_like(res), out_scales=full_s)
            rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
            for gather in (True, False):
                what = f"rank {ctx.rank} {dtype} {norm} Ts={Ts} H={H} gather={gather}"
                raws, rout, codes, scales = _fp8_outputs(T if gather else Ts, H, dtype)
                rraw, rout = _guarded((Ts, H), dtype)
                raws = (rraw,) + raws[1:]
                plan = _plan_sp(cc, T, H, dtype, norm, gather, True)

                def call():
                    cc.reduce_scatter_residual_norm(partial, res[rows].clone(), w, nb, norm=norm, eps=EPS, bias=b,
                                                    residual_out=rout, out=codes, gather_out=gather,
                                                    out_scales=scales)

                n = _launches(cc, call)
                if n != P * plan["launches"]:
                    bad.append(f"{what}: {n} launches over {P} ranks, plan {plan}")
                want = slice(None) if gather else rows
                if not torch.equal(_bytes(rout), _bytes(full_r[rows])):
                    bad.append(f"{what}: residual_out differs")
                if not torch.equal(_bytes(codes), _bytes(full_c[want])):
                    bad.append(f"{what}: codes differ from the TP FP8 rows")
                if not torch.equal(_bytes(scales), _bytes(full_s[want])):
                    bad.append(f"{what}: scales differ from the TP FP8 rows")
                bad += [f"{what}: wrote outside an output" for raw in raws if not _guards_intact(raw)]
                if gather:
                    digests.append((_digest(codes), _digest(scales)))
        cc.synchronize()
        return bad, digests

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    assert not bad, "\n".join(bad[:40])
    assert len({tuple(d) for _, d in results}) == 1, "ranks gathered different codes or scales"


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3])
def test_fp8_chunked(P):
    """A 1 MiB pool: the FP8 two-shot and the gathered SP form run as chunks, one launch each, each
    exact; their out rows in the pool are H code bytes and a scale, so a chunk holds more rows than
    the bfloat16 form's."""
    stage = 1 << 20
    dtype, H = torch.bfloat16, 4096

    def fn(ctx, cc):
        t = gb._C.cuda.get_tuning()
        half = min(-(-max(t["one_shot_max_bytes"], 4096) // 4096) * 4096, stage // 4)
        bulk = stage - 2 * half
        rb = H * 2
        bad = []
        for norm in NORMS:
            T = 500
            p16, p8 = (_plan_tp(cc, T, H, dtype, norm, "two_shot", f) for f in (False, True))
            if p8["chunk_rows"] != bulk // (rb + H + 4) or p16["chunk_rows"] != bulk // (2 * rb):
                bad.append(f"two-shot {norm}: plans {p16} / {p8}, bulk {bulk}")
            if not p8["chunk_rows"] > p16["chunk_rows"] or p8["launches"] < 2:
                bad.append(f"two-shot {norm}: the FP8 plan {p8} holds no more rows than {p16}")
            bad += _run_tp_case(cc, P, ctx.rank, (dtype, norm, True, "two_shot", T, H))[0]
            Ts = 60
            s16, s8 = (_plan_sp(cc, P * Ts, H, dtype, norm, True, f) for f in (False, True))
            if s8["chunk_rows"] != bulk // (P * (rb + H + 4)) or s16["chunk_rows"] != bulk // (P * 2 * rb):
                bad.append(f"SP {norm}: plans {s16} / {s8}, bulk {bulk}")
            if not s8["chunk_rows"] > s16["chunk_rows"] or s8["launches"] < 2:
                bad.append(f"SP {norm}: the FP8 plan {s8} holds no more rows than {s16}")
            T = P * Ts
            partial, res, b, w, nb = _problem(("chunk", norm), ctx.rank, T, H, dtype, norm)
            rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
            full_r, full_o = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b,
                                                        residual_out=torch.empty_like(res))
            for gather in (True, False):
                raws, _, codes, scales = _fp8_outputs(T if gather else Ts, H, dtype)
                rraw, rout = _guarded((Ts, H), dtype)
                plan = _plan_sp(cc, T, H, dtype, norm, gather, True)
                n = _launches(cc, lambda: cc.reduce_scatter_residual_norm(
                    partial, res[rows].clone(), w, nb, norm=norm, eps=EPS, bias=b, residual_out=rout, out=codes,
                    gather_out=gather, out_scales=scales))
                if n != P * plan["launches"] or plan["launches"] < 2:
                    bad.append(f"SP {norm} gather={gather}: {n} launches, plan {plan}")
                bad += _check_fp8(f"SP {norm} gather={gather}", full_r[rows], full_o if gather else full_o[rows],
                                  rout, codes, scales, (rraw,) + raws[1:])
        return [f"rank {ctx.rank} {x}" for x in bad]

    bad = [x for b in _spawn(P, fn, stage_bytes=stage) for x in b]
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2])
def test_fp8_edge_rows(P):
    """An all-zero out (weight 0) gives scale 1e-4 / 448 and zero codes; a constant row under
    LayerNorm gives out = norm_bias, quantised like any other row."""
    H = 4096

    def fn(ctx, cc):
        bad = []
        for dtype in MAIN:
            for algo in ALGOS:
                T = 5
                partial, res, b, w, nb = _problem(("edge", dtype, algo), ctx.rank, T, H, dtype, "layer")
                for norm, weight in (("rms", torch.zeros_like(w)), ("layer", torch.zeros_like(w))):
                    s = torch.empty(T, 1, dtype=torch.float32, device="cuda")
                    _, codes = cc.allreduce_residual_norm(partial, res, weight, None, norm=norm, eps=EPS, bias=b,
                                                          residual_out=torch.empty_like(res), algo=algo, out_scales=s)
                    want = torch.tensor(1e-4, dtype=torch.float32) / torch.tensor(448.0)
                    if not bool((s.cpu() == want).all()) or not bool((codes.float() == 0).all()):
                        bad.append(f"{dtype} {algo} {norm}: zero out gave scales {s.flatten()[:3].tolist()}")
                # constant rows: every partial 0, the residual row r holds the value r - 2
                zero = torch.zeros_like(partial)
                const = (torch.arange(T, device="cuda", dtype=torch.float32) - 2).to(dtype)[:, None].expand(T, H)
                const = const.contiguous()
                want_r, want_o = cc.allreduce_residual_norm(zero, const, w, nb, norm="layer", eps=EPS,
                                                            residual_out=torch.empty_like(const), algo=algo)
                raws, rout, codes, scales = _fp8_outputs(T, H, dtype)
                cc.allreduce_residual_norm(zero, const, w, nb, norm="layer", eps=EPS, residual_out=rout, out=codes,
                                           algo=algo, out_scales=scales)
                if not torch.equal(want_o, nb.expand(T, H)):
                    bad.append(f"{dtype} {algo}: LayerNorm of a constant row is not norm_bias")
                bad += _check_fp8(f"{dtype} {algo} constant rows", want_r, want_o, rout, codes, scales, raws)
        cc.synchronize()
        return [f"rank {ctx.rank} {x}" for x in bad]

    bad = [x for b in _spawn(P, fn) for x in b]
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
def test_fp8_back_to_back(P):
    """120 calls on one context alternating the FP8 and bfloat16 forms, every algo and the SP form
    (pool parity and epochs), each exact."""
    dtype, norm, H = torch.bfloat16, "rms", 4096

    def fn(ctx, cc):
        probs = {}
        for T in (P * 2, P * 50):
            partial, res, b, w, nb = _problem(("b2b", T), ctx.rank, T, H, dtype, norm)
            r, o = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, bias=b, residual_out=torch.empty_like(res))
            probs[T] = (partial, res, b, w, r.clone(), o.clone(), fp8_rows(o))
        bad = []
        for i in range(120):
            T = P * 2 if i % 3 else P * 50
            partial, res, b, w, want_r, want_o, (want_c, want_s) = probs[T]
            fp8, algo = i % 2 == 1, ALGOS[(i // 2) % 4]
            if i % 5 == 4:
                Ts = T // P
                rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
                s = torch.empty(T, 1, dtype=torch.float32, device="cuda") if fp8 else None
                r, o = cc.reduce_scatter_residual_norm(partial, res[rows].clone(), w, None, norm=norm, bias=b,
                                                       out_scales=s)
                ok = torch.equal(r, want_r[rows]) and (
                    torch.equal(_bytes(o), _bytes(want_c)) and torch.equal(s, want_s) if fp8 else torch.equal(o, want_o))
            else:
                s = torch.empty(T, 1, dtype=torch.float32, device="cuda") if fp8 else None
                r, o = cc.allreduce_residual_norm(partial, res, w, None, norm=norm, bias=b,
                                                  residual_out=torch.empty_like(res), algo=algo, out_scales=s)
                ok = torch.equal(r, want_r) and (
                    torch.equal(_bytes(o), _bytes(want_c)) and torch.equal(s, want_s) if fp8 else torch.equal(o, want_o))
            if not ok:
                bad.append(f"rank {ctx.rank} call {i} (T={T} fp8={fp8} algo={algo}) differs")
        cc.synchronize()
        return bad

    bad = [x for b in _spawn(P, fn) for x in b]
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
def test_fp8_malformed_calls():
    """Each malformed FP8 call raises ValueError and launches nothing."""
    P, T, H = 2, 4, 64
    dtype = torch.bfloat16

    def fn(ctx, cc):
        partial, res, b, w, nb = _problem(("bad",), ctx.rank, T, H, dtype, "layer")
        s = lambda rows=T: torch.empty(rows, 1, dtype=torch.float32, device="cuda")  # noqa: E731
        buf = torch.zeros(4096, dtype=torch.uint8, device="cuda")
        TP = cc.allreduce_residual_norm
        SP = cc.reduce_scatter_residual_norm
        cases = {
            "fp8 out without out_scales": lambda: TP(partial, res, w, norm="rms",
                                                     out=torch.empty(T, H, dtype=E4M3, device="cuda")),
            "e5m2 out": lambda: TP(partial, res, w, norm="rms", out=torch.empty(T, H, dtype=torch.float8_e5m2,
                                                                               device="cuda"), out_scales=s()),
            "bf16 out with out_scales": lambda: TP(partial, res, w, norm="rms", out=torch.empty_like(partial),
                                                   out_scales=s()),
            "out_scales (T,)": lambda: TP(partial, res, w, norm="rms", out_scales=torch.empty(T, device="cuda")),
            "out_scales bf16": lambda: TP(partial, res, w, norm="rms", out_scales=s().to(dtype)),
            "out_scales not contiguous": lambda: TP(partial, res, w, norm="rms",
                                                    out_scales=torch.empty(T, 2, device="cuda")[:, :1]),
            "codes wrong shape": lambda: TP(partial, res, w, norm="rms", out=torch.empty(T, H // 2, dtype=E4M3,
                                                                                         device="cuda"),
                                            out_scales=s()),
            "no norm": lambda: TP(partial, res, norm=None, out_scales=s()),
            "H % 16": lambda: TP(partial[:, :8].contiguous(), res[:, :8].contiguous(), w[:8].contiguous(), norm="rms",
                                 out_scales=s()),
            "scales overlap residual_out": lambda: TP(partial, res, w, norm="rms",
                                                      residual_out=buf[:T * H * 2].view(dtype).view(T, H),
                                                      out_scales=buf[:T * 4].view(torch.float32).view(T, 1)),
            "codes overlap partial": lambda: TP(partial, res, w, norm="rms",
                                                out=partial.view(-1).view(E4M3)[:T * H].view(T, H), out_scales=s()),
            "scales misaligned": lambda: TP(partial, res, w, norm="rms",
                                            out_scales=buf[4:4 + T * 4].view(torch.float32).view(T, 1)),
            "SP gathered scales of a shard": lambda: SP(partial, res[:T // P].clone(), w, norm="rms",
                                                        out_scales=s(T // P)),
            "SP shard scales of all rows": lambda: SP(partial, res[:T // P].clone(), w, norm="rms", gather_out=False,
                                                      out_scales=s()),
        }
        bad = []
        for name, call in cases.items():
            def expect():
                with pytest.raises(ValueError):
                    call()

            try:
                n = _launches(cc, expect)
            except BaseException as e:  # noqa: BLE001 - reported, not raised, so every rank goes on
                bad.append(f"rank {ctx.rank} {name}: {type(e).__name__} {e}")
                continue
            if n:
                bad.append(f"rank {ctx.rank} {name}: {n} launches")
        return bad

    bad = [x for b in _spawn(P, fn) for x in b]
    assert not bad, "\n".join(bad)


def _ref_tp_block(blk, x):
    """TPBlock's CUDA forward with ln2's out taken unquantised from the fused step and quantised
    with torch (fp8_rows), the weight likewise, and the same scaled_mm."""
    F, tp = torch.nn.functional, blk.tp
    B, S, E = x.shape
    hd = E // blk.n_heads
    h = blk.ln1(x)
    q, k, v = (F.linear(h, lin.weight, lin.bias).view(B, S, blk.local_heads, hd).transpose(1, 2)
               for lin in (blk.q, blk.k, blk.v))
    a = F.scaled_dot_product_attention(q, k, v, is_causal=True).transpose(1, 2).reshape(B, S, -1)
    x, o = tp.reduce_residual_norm(F.linear(a, blk.proj.weight), x, blk.ln2, blk.proj.bias)
    p = F.linear(F.gelu(_ref_up(blk, o)), blk.down.weight)
    return tp.reduce_residual_norm(p, x, None, blk.down.bias)


def _ref_sp_block(blk, x):
    F, sp = torch.nn.functional, blk.sp
    h = sp.gather_from_sequence(blk.ln1(x))
    S, B, _ = h.shape
    hd = blk.d_model // blk.n_heads
    q, k, v = (F.linear(h, lin.weight, lin.bias).view(S, B, blk.local_heads, hd).permute(1, 2, 0, 3)
               for lin in (blk.q, blk.k, blk.v))
    a = F.scaled_dot_product_attention(q, k, v, is_causal=True).permute(2, 0, 1, 3).reshape(S, B, -1)
    x, o = sp.reduce_scatter_residual_norm(F.linear(a, blk.proj.weight), x, blk.ln2, blk.proj.bias)
    p = F.linear(F.gelu(_ref_up(blk, o)), blk.down.weight)
    return sp.reduce_scatter_residual_norm(p, x, None, blk.down.bias, gather_out=False)


def _ref_up(blk, o):
    codes, scales = fp8_rows(o)
    wc, ws = fp8_rows(blk.up.weight)
    E = blk.d_model
    h = torch._scaled_mm(codes.reshape(-1, E), wc.t(), scale_a=scales.reshape(-1, 1), scale_b=ws.reshape(1, -1),
                         out_dtype=torch.bfloat16)
    return (h + blk.up.bias).view(*o.shape[:-1], -1)


# The FP8 block against the bfloat16 DenseBlock: ||y_fp8 - y_dense|| / ||mlp_dense|| <= REL_BOUND,
# where mlp_dense = down(gelu(up(ln2(.)))) is the branch the FP8 GEMM feeds.
REL_BOUND = 0.125


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("sequence_parallel", [False, True])
def test_tp_block_fp8(P, sequence_parallel):
    """TPBlock.enable_fp8() under no_grad: the output equals, exactly, a torch reference that
    quantises ln2's unquantised fused output and the up weight with fp8_rows and calls the same
    scaled_mm. Against the bfloat16 DenseBlock its error relative to the MLP branch is at most
    REL_BOUND = 2^-3: e4m3 keeps 3 mantissa bits, so each of the GEMM's two operands carries a
    relative rounding error of at most 2^-4 and a product of the two at most about 2 * 2^-4 = 2^-3.
    Summed over the K = d_model products with independent errors, the GEMM's error relative to its
    output is about the RMS of the per-product error (~0.05) and stays below that worst case; gelu
    and the down projection do not amplify a relative error of the branch, and the bfloat16
    differences between the two blocks are two orders smaller. Measured on an H100: about 0.04. In
    grad mode the forward raises."""
    B, S, E, heads, d_ff = 2, 16, 128, 4, 512
    # built once here: the ranks' threads share torch's global generator
    torch.manual_seed(23)
    dense = DenseBlock(d_model=E, n_heads=heads, d_ff=d_ff).cuda().to(torch.bfloat16)
    x = torch.randn(B, S, E, device="cuda").to(torch.bfloat16)

    def fn(ctx, cc):
        tp = TensorParallel(ctx, cc)
        blk = TPBlock(tp, d_model=E, n_heads=heads, d_ff=d_ff, device="cuda", dtype=torch.bfloat16,
                      sequence_parallel=sequence_parallel)
        blk.load_dense(dense)
        blk.enable_fp8()
        lo, hi = S // P * ctx.rank, S // P * (ctx.rank + 1)
        xi = x.transpose(0, 1)[lo:hi].contiguous() if sequence_parallel else x
        bad = []
        with pytest.raises(ValueError):
            blk(xi)
        with torch.no_grad():
            y = blk(xi)
            want = (_ref_sp_block if sequence_parallel else _ref_tp_block)(blk, xi)
            y_dense = dense(x)
            x1 = x + dense.proj(_dense_attention(dense, x))
            mlp = dense.down(torch.nn.functional.gelu(dense.up(dense.ln2(x1))))
        if sequence_parallel:
            y_dense, mlp = y_dense.transpose(0, 1)[lo:hi], mlp.transpose(0, 1)[lo:hi]
        if not torch.equal(y, want):
            bad.append(f"rank {ctx.rank}: block output differs from the torch FP8 reference "
                       f"(max {float((y.float() - want.float()).abs().max())})")
        rel = float((y.float() - y_dense.float()).norm() / mlp.float().norm())
        if not rel <= REL_BOUND:
            bad.append(f"rank {ctx.rank}: relative error {rel:.4f} against DenseBlock beyond {REL_BOUND}")
        cc.synchronize()
        return bad, rel

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    assert not bad, "\n".join(bad)
    print(f"relative error against DenseBlock: {max(r for _, r in results):.4f}")


def _dense_attention(dense, x):
    B, S, E = x.shape
    q, k, v = dense.qkv(dense.ln1(x)).view(B, S, 3, dense.n_heads, E // dense.n_heads).unbind(2)
    a = torch.nn.functional.scaled_dot_product_attention(q.transpose(1, 2), k.transpose(1, 2), v.transpose(1, 2),
                                                         is_causal=True)
    return a.transpose(1, 2).reshape(B, S, E)


def test_fp8_fallback_on_cpu():
    """On CPU tensors, TensorParallel / SequenceParallel's fp8=True run the unfused composition and
    fp8_rows, byte for byte; in grad mode with parameters that require grad, fp8 raises."""
    P, T, H = 2, 6, 32

    def body(ctx):
        g = torch.Generator().manual_seed(5)
        parts = [torch.randn(T, H, generator=g) for _ in range(P)]
        residual = torch.randn(T, H, generator=g)
        bias = torch.randn(H, generator=g)
        ln = torch.nn.LayerNorm(H)
        rms = torch.nn.RMSNorm(H, eps=1e-6)
        bad = []
        tp, sp = TensorParallel(ctx), SequenceParallel(ctx)
        with torch.no_grad():
            for norm in (ln, rms):
                s_want = parts[0] + parts[1] + bias + residual
                o_want = norm(s_want)
                s, (codes, scales) = tp.reduce_residual_norm(parts[ctx.rank].clone(), residual, norm, bias, fp8=True)
                c, sc = fp8_rows(o_want)
                if not (torch.equal(s, s_want) and torch.equal(_bytes(codes), _bytes(c)) and torch.equal(scales, sc)):
                    bad.append(f"rank {ctx.rank} TP {type(norm).__name__}")
                if codes.dtype != E4M3 or tuple(scales.shape) != (T, 1):
                    bad.append(f"rank {ctx.rank} TP: codes {codes.dtype}, scales {tuple(scales.shape)}")
                Ts = T // P
                rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
                for gather in (True, False):
                    s, (codes, scales) = sp.reduce_scatter_residual_norm(parts[ctx.rank].clone(), residual[rows], norm,
                                                                         bias, gather_out=gather, fp8=True)
                    want = slice(None) if gather else rows
                    if not (torch.equal(s, s_want[rows]) and torch.equal(_bytes(codes), _bytes(c[want])) and
                            torch.equal(scales, sc[want])):
                        bad.append(f"rank {ctx.rank} SP {type(norm).__name__} gather={gather}")
        for call in (lambda: tp.reduce_residual_norm(parts[ctx.rank].clone(), residual, ln, bias, fp8=True),
                     lambda: sp.reduce_scatter_residual_norm(parts[ctx.rank].clone(), residual[:T // P], ln, fp8=True),
                     lambda: tp.reduce_residual_norm(parts[ctx.rank].clone(), residual, None, bias, fp8=True)):
            try:
                call()
                bad.append(f"rank {ctx.rank}: a grad-mode / no-norm fp8 call did not raise")
            except ValueError:
                pass
        return bad

    bad = [x for b in gb.spawn_threads(P, body, timeout_ms=60000) for x in b]
    assert not bad, bad


def test_fp8_rows_matches_the_documented_rule():
    """fp8_rows is amax / 448 per row with the 1e-4 floor, codes round to nearest even and saturate."""
    o = torch.tensor([[0.0, -0.0, 0.0, 0.0], [1.0, -2.0, 0.5, 448.0], [3.0, -3.0, 1.5, 0.001]])
    codes, scales = fp8_rows(o)
    assert torch.equal(scales, torch.tensor([[1e-4], [448.0], [3.0]]) / torch.tensor(448.0))
    assert torch.equal(codes.float()[1], torch.tensor([1.0, -2.0, 0.5, 448.0]))
    assert torch.equal(codes.float()[2, :3], torch.tensor([448.0, -448.0, 224.0]))
    assert float(codes.float()[0].abs().max()) == 0.0
