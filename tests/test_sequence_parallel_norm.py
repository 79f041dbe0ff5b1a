"""Sequence parallelism: the reduce-scatter form of the fused residual norm and its autograd.

`CudaContext.reduce_scatter_residual_norm` is checked against an fp64 reference on the order-free
inputs of test_allreduce_norm.py (`residual_out` byte for byte, `out` within one ulp), and, on
random inputs, byte for byte against the matching rows of `allreduce_residual_norm`, which sums in
the same order. `SequenceParallel`'s operators and `models.TPBlock(sequence_parallel=True)` are
checked against dense compositions: on CPU tensors here, on CUDA in sp_block_worker.py.

Ranks are threads sharing cuda:0, as in the other GPU tests; every rank's thread returns its outputs
to the test, which builds the reference once per case.
"""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.models import DenseBlock, TPBlock
from gloo_b200.ops import cuda as gcu
from gloo_b200.parallel import SequenceParallel, TensorParallel
from test_allreduce_norm import (EPS, MAIN, NORMS, _close, _digest, _guarded, _guards_intact, _hidden, _inputs, _kind,
                                 _launches, _norm_module, _reference)
from test_reduce_numerics import _gen, _mismatch

# (Ts, H): every shard size with every H, the largest shard at the narrower rows
SHAPES = [(t, h) for t in (1, 3, 17) for h in ("min", 4096, 7168, 16384)] + [(125, "min"), (125, 4096), (125, 7168)]


def _plan(cc, T, H, dtype, norm, gather):
    return gb._C.cuda.plan_reduce_scatter_norm(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)), _kind(norm), gather)


def _cases(P):
    out, i = [], 0
    for dtype in MAIN:
        for norm in NORMS:
            for with_bias in (True, False):
                for gather in (True, False):
                    Ts, h = SHAPES[(i + 5 * P) % len(SHAPES)]
                    out.append((dtype, norm, with_bias, gather, P * Ts, _hidden(h, dtype), i % 3 == 0))
                    i += 1
    return out


def _run_case(cc, P, rank, case):
    """One fused call of this rank on the order-free inputs of `case`; returns (failures, results)."""
    dtype, norm, with_bias, gather, T, H, in_place = case
    Ts = T // P
    bad = []
    parts, residual, bias, weight, norm_bias = _inputs(case, P, T, H, dtype, [rank])
    bias = bias if with_bias else None
    weight = weight if norm is not None else None
    norm_bias = norm_bias if norm == "layer" else None
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    partial, res = parts[rank].cuda(), residual[rank * Ts:(rank + 1) * Ts].cuda()
    b, w, nb = dev(bias), dev(weight), dev(norm_bias)
    inputs = [t for t in (partial, None if in_place else res, b, w, nb) if t is not None]
    kept = [t.clone() for t in inputs]
    rraw, rout = (None, None) if in_place else _guarded((Ts, H), dtype)
    oraw, out = _guarded((T if gather else Ts, H), dtype) if norm is not None else (None, None)
    plan = _plan(cc, T, H, dtype, norm, gather)
    got = {}

    def call():
        got["r"] = cc.reduce_scatter_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b, residual_out=rout,
                                                   out=out, gather_out=gather)

    n = _launches(cc, call)
    want_variant = "local" if P == 1 else "reduce_scatter"
    if plan["variant"] != want_variant or plan["launches"] != -(-Ts // plan["chunk_rows"]):
        bad.append(f"{case}: plan {plan}")
    if n != P * plan["launches"]:
        bad.append(f"{case}: {n} launches over {P} ranks, planned {plan['launches']} each")
    res_out = res if in_place else rout
    r = got["r"]
    if norm is None:
        if r is not res_out:
            bad.append(f"{case}: returned another tensor than residual_out")
    elif r[0] is not res_out or r[1] is not out:
        bad.append(f"{case}: returned other tensors than (residual_out, out)")
    for raw, what in ((rraw, "residual_out"), (oraw, "out")):
        if raw is not None and not _guards_intact(raw):
            bad.append(f"{case}: wrote outside {what}")
    if not all(torch.equal(t, k) for t, k in zip(inputs, kept)):
        bad.append(f"{case}: an input changed")
    return bad, (res_out.cpu(), None if out is None else out.cpu(), plan["launches"])


def _check_reference(case, P, results):
    """`results[r]` = rank r's (residual_out, out): against the fp64 reference of the whole problem."""
    dtype, norm, with_bias, gather, T, H, _ = case
    Ts = T // P
    parts, residual, bias, weight, norm_bias = _inputs(case, P, T, H, dtype, range(P))
    want_r, want_o = _reference([parts[q] for q in range(P)], residual, bias if with_bias else None, weight, norm_bias,
                                norm, dtype)
    bad = []
    for rank, (r, o) in enumerate(results):
        rows = slice(rank * Ts, (rank + 1) * Ts)
        m = _mismatch(r.reshape(-1), want_r[rows].reshape(-1))
        if m is not None:
            bad.append(f"{case} rank {rank}: residual_out {m}")
        if norm is not None:
            m = _close(o, want_o if gather else want_o[rows], dtype)
            if m is not None:
                bad.append(f"{case} rank {rank}: out {m}")
    if norm is not None and gather and len({_digest(o) for _, o in results}) != 1:
        bad.append(f"{case}: ranks gathered different out")
    return bad


def _spawn(P, fn, stage_bytes=64 << 20):
    def body(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=stage_bytes)
        cc.set_timeout(120000)
        return fn(ctx, cc)

    return gb.spawn_threads(P, body, cuda_device=0, timeout_ms=600000)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_reduce_scatter_residual_norm(P):
    """Every dtype x norm x bias x gather_out, over Ts in {1, 3, 17, 125} and H in {min, 4096, 7168,
    16384}, against fp64; guard bands, inputs, in-place residual_out and launch counts."""
    cases = _cases(P)

    def fn(ctx, cc):
        bad, outs = [], []
        for case in cases:
            b, o = _run_case(cc, P, ctx.rank, case)
            bad += [f"rank {ctx.rank} {x}" for x in b]
            outs.append(o)
        return bad, outs

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    for i, case in enumerate(cases):
        bad += _check_reference(case, P, [outs[i][:2] for _, outs in results])
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3, 4, 8])
def test_equals_allreduce_rows_on_random_inputs(P):
    """Random inputs, whose sums depend on the order: the shard and the gathered out equal the rows
    of allreduce_residual_norm's outputs byte for byte, and every rank gathers the same bytes."""
    cases = [(dtype, norm, Ts, H) for dtype in MAIN for norm in NORMS for Ts, H in ((3, 4096), (40, 1024))]

    def fn(ctx, cc):
        bad, digests = [], []
        for dtype, norm, Ts, H in cases:
            T = P * Ts
            g = _gen(("random", str(dtype), norm, Ts), ctx.rank)
            g0 = _gen(("random", str(dtype), norm, Ts), 0)
            partial = (3 * torch.randn(T, H, generator=g)).to(dtype).cuda()
            residual = torch.randn(T, H, generator=g0).to(dtype).cuda()
            bias = torch.randn(H, generator=g0).to(dtype).cuda()
            w = (0.5 + torch.rand(H, generator=g0)).to(dtype).cuda() if norm else None
            nb = torch.randn(H, generator=g0).to(dtype).cuda() if norm == "layer" else None
            full = cc.allreduce_residual_norm(partial, residual, w, nb, norm=norm, bias=bias,
                                              residual_out=torch.empty_like(residual))
            rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
            for gather in (True, False):
                got = cc.reduce_scatter_residual_norm(partial, residual[rows].clone(), w, nb, norm=norm, bias=bias,
                                                      gather_out=gather)
                want_r, want_o = (full, None) if norm is None else full
                r, o = (got, None) if norm is None else got
                if not torch.equal(r, want_r[rows]):
                    bad.append(f"rank {ctx.rank} {dtype} {norm} Ts={Ts} gather={gather}: residual_out differs")
                if norm is not None and not torch.equal(o, want_o if gather else want_o[rows]):
                    bad.append(f"rank {ctx.rank} {dtype} {norm} Ts={Ts} gather={gather}: out differs")
                if norm is not None and gather:
                    digests.append(_digest(o))
        cc.synchronize()
        return bad, digests

    results = _spawn(P, fn)
    assert not [x for b, _ in results for x in b], [x for b, _ in results for x in b][:20]
    assert len({tuple(d) for _, d in results}) == 1, "ranks gathered different out"


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3])
def test_chunked(P):
    """A 1 MiB pool: every shard runs as ceil(Ts / chunk rows) chunks, one launch each, each exact."""
    stage = 1 << 20
    dtype, Ts, H = torch.bfloat16, 250, 4096

    def fn(ctx, cc):
        t = gb._C.cuda.get_tuning()
        half = min(-(-max(t["one_shot_max_bytes"], 4096) // 4096) * 4096, stage // 4)
        bulk = stage - 2 * half
        bad, outs = [], []
        for norm, gather in (("layer", True), ("rms", False), (None, True)):
            case = (dtype, norm, True, gather, P * Ts, H, False)
            plan = _plan(cc, P * Ts, H, dtype, norm, gather)
            chunk = bulk // (P * (2 if norm and gather else 1) * H * 2)
            if plan["chunk_rows"] != chunk or plan["launches"] != -(-Ts // chunk) or plan["launches"] < 2:
                bad.append(f"plan {plan}, want chunks of {chunk} rows")
            b, o = _run_case(cc, P, ctx.rank, case)
            bad += b
            outs.append((case, o))
        return bad, outs

    results = _spawn(P, fn, stage_bytes=stage)
    bad = [x for b, _ in results for x in b]
    for i, (case, _) in enumerate(results[0][1]):
        bad += _check_reference(case, P, [outs[i][1][:2] for _, outs in results])
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
def test_back_to_back_calls(P):
    """200 calls on one context with no host synchronisation between them, gathered and not, with
    and without a norm, over 4 input sets: each result equals the allreduce form's rows. A rank
    that restaged its pool while a peer still read it would corrupt a later call."""
    Ts, H, dtype = 8, 1024, torch.bfloat16
    T = P * Ts
    kinds = [("rms", True), ("layer", False), (None, True), ("rms", False)]

    def fn(ctx, cc):
        rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
        sets = []
        for k in range(4):
            g, g0 = _gen(("b2b", k), ctx.rank), _gen(("b2b", k), 0)
            partial = torch.randn(T, H, generator=g).to(dtype).cuda()
            residual = torch.randn(T, H, generator=g0).to(dtype).cuda()
            bias, w = torch.randn(H, generator=g0).to(dtype).cuda(), (0.5 + torch.rand(H, generator=g0)).to(dtype).cuda()
            norm, gather = kinds[k]
            nb = torch.randn(H, generator=g0).to(dtype).cuda() if norm == "layer" else None
            want = cc.allreduce_residual_norm(partial, residual, w if norm else None, nb, norm=norm, bias=bias,
                                              residual_out=torch.empty_like(residual))
            want_r, want_o = (want, None) if norm is None else want
            want_o = None if want_o is None else (want_o if gather else want_o[rows])
            sets.append((partial, residual[rows].contiguous(), bias, w if norm else None, nb, norm, gather,
                         want_r[rows], want_o))
        cc.synchronize()
        cc.pc.host_barrier()
        got = []
        for i in range(200):
            partial, res, bias, w, nb, norm, gather, _, _ = sets[i % 4]
            got.append(cc.reduce_scatter_residual_norm(partial, res, w, nb, norm=norm, bias=bias,
                                                       residual_out=torch.empty_like(res), gather_out=gather))
        cc.synchronize()
        bad = []
        for i, g in enumerate(got):
            *_, norm, gather, want_r, want_o = sets[i % 4]
            r, o = (g, None) if norm is None else g
            if not torch.equal(r, want_r) or (o is not None and not torch.equal(o, want_o)):
                bad.append(f"rank {ctx.rank} call {i}: differs")
        return bad

    for bad in _spawn(P, fn, stage_bytes=16 << 20):
        assert not bad, bad[:10]


@pytest.mark.gpu
def test_malformed_calls_raise_and_launch_nothing():
    P = 2

    def fn(ctx, cc):
        bf = torch.bfloat16
        p = torch.ones(4, 64, dtype=bf, device="cuda")
        r = torch.ones(2, 64, dtype=bf, device="cuda")
        w = torch.ones(64, dtype=bf, device="cuda")
        raw = torch.ones(4 * 64 + 8, dtype=bf, device="cuda")
        odd = torch.ones(4, 12, dtype=bf, device="cuda")  # 24-byte rows
        wide = torch.ones(2, 16384 + 8, dtype=bf, device="cuda")
        full_out = torch.empty(4, 64, dtype=bf, device="cuda")
        dt = int(gb.DataType.BFLOAT16)
        calls = {
            "T not divisible by P": lambda: cc.reduce_scatter_residual_norm(p[:3], r, w),
            "T not divisible by P (native)": lambda: gb._C.cuda.reduce_scatter_residual_norm(
                cc.pc, p.data_ptr(), r.data_ptr(), r.data_ptr(), full_out.data_ptr(), 0, w.data_ptr(), 0, 3, 64, dt, 1,
                1e-6, True),
            "residual of every row": lambda: cc.reduce_scatter_residual_norm(p, p.clone(), w),
            "residual of one row": lambda: cc.reduce_scatter_residual_norm(p, r[:1], w),
            "shard out with gather_out": lambda: cc.reduce_scatter_residual_norm(p, r, w, out=r.clone()),
            "gathered out without gather_out": lambda: cc.reduce_scatter_residual_norm(p, r, w, out=full_out,
                                                                                        gather_out=False),
            "dtype mix": lambda: cc.reduce_scatter_residual_norm(p, r.float(), w),
            "weight dtype": lambda: cc.reduce_scatter_residual_norm(p, r, w.half()),
            "float64": lambda: cc.reduce_scatter_residual_norm(p.double(), r.double(), w.double()),
            "H not 16 bytes": lambda: cc.reduce_scatter_residual_norm(odd, odd[:2].clone(), None),
            "H over the limit": lambda: cc.reduce_scatter_residual_norm(wide, wide[:1].clone(), None),
            "unaligned view": lambda: cc.reduce_scatter_residual_norm(raw[1:1 + 256].view(4, 64), r, w),
            "out is partial": lambda: cc.reduce_scatter_residual_norm(p, r, w, out=p),
            "residual_out in partial": lambda: cc.reduce_scatter_residual_norm(p, r, w, residual_out=p[2:]),
            "residual_out overlaps residual": lambda: cc.reduce_scatter_residual_norm(
                p, raw[:128].view(2, 64), w, residual_out=raw[8:8 + 128].view(2, 64)),
            "out overlaps residual_out": lambda: cc.reduce_scatter_residual_norm(p, r, w, out=r, gather_out=False),
            "bad norm": lambda: cc.reduce_scatter_residual_norm(p, r, w, norm="batch"),
        }
        bad = []
        for name, call in calls.items():
            raised = []

            def go():
                try:
                    call()
                except ValueError:
                    raised.append(True)

            if _launches(cc, go) != 0 or not raised:
                bad.append(f"{name}: raised {bool(raised)}")
        return bad

    for bad in _spawn(P, fn, stage_bytes=16 << 20):
        assert not bad, bad


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sp_block_worker.py")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_sp_block_cuda_matches_dense(size):
    """models.TPBlock(sequence_parallel=True) on CUDA == DenseBlock: output shard, input gradient,
    weight-shard gradients and, after allreduce_sequence_parallel_grads, ln1 / ln2 / bias gradients;
    a forward is three collective launches. One process per rank (sp_block_worker.py)."""
    d = tempfile.mkdtemp(prefix="glb_sp_block_")
    procs = [subprocess.Popen([sys.executable, WORKER, d, str(r), str(size)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(size)]
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=300)
        except subprocess.TimeoutExpired:
            p.kill()
            o, _ = p.communicate()
        outs.append(o)
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"WORKER {r} OK" in o, f"rank {r} failed:\n{o[-3000:]}"


# ---- CPU: the operators and the block on the host collectives ----------------------------------
# (On CUDA the backward's collectives run on the device's autograd thread, which ranks sharing one
# process cannot share: sp_block_worker.py checks the CUDA autograd one process per rank.)


def _check_sp_autograd(P, kind, gather):
    """reduce_scatter_residual_norm's forward and the gradients of partial, residual, bias, weight and
    norm_bias (the last three summed over ranks) against the dense composition in one process."""
    Ts, H = 3, 64
    T = P * Ts
    f64 = lambda key, r, *shape: torch.randn(*shape, generator=_gen((key, kind, gather), r),  # noqa: E731
                                             dtype=torch.float64).float()
    parts = [f64("part", r, T, H) for r in range(P)]
    residual, bias = f64("res", 0, T, H), f64("bias", 0, H)
    g_r, g_o = f64("gr", 0, T, H), f64("go", 0, T, H)

    dp = [p.clone().requires_grad_(True) for p in parts]
    dres, dbias = residual.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    dnorm = _norm_module(kind, H)
    s = sum(dp) + dbias + dres
    loss = (s * g_r).sum()
    if dnorm is not None:
        y = dnorm(s)
        loss = loss + (y * g_o).sum()
    loss.backward()

    def fn(ctx):
        sp = SequenceParallel(ctx)
        rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
        p = parts[ctx.rank].clone().requires_grad_(True)
        res = residual[rows].clone().requires_grad_(True)
        b = bias.clone().requires_grad_(True)
        norm = _norm_module(kind, H)
        got = sp.reduce_scatter_residual_norm(p, res, norm, b, gather_out=gather)
        s_, y_ = (got, None) if norm is None else got
        loss = (s_ * g_r[rows]).sum()
        if y_ is not None:
            # a gathered out is replicated: each rank's loss takes its own rows of it
            loss = loss + ((y_[rows] if gather else y_) * g_o[rows]).sum()
        loss.backward()
        shared = [b] + ([] if norm is None else list(norm.parameters()))
        sp.allreduce_sequence_parallel_grads(shared)
        grads = [p.grad.cpu(), res.grad.cpu()] + [t.grad.cpu() for t in shared]
        return s_.detach().cpu(), None if y_ is None else y_.detach().cpu(), grads

    for rank, (s_, y_, grads) in enumerate(gb.spawn_threads(P, fn)):
        rows = slice(rank * Ts, (rank + 1) * Ts)
        torch.testing.assert_close(s_, s.detach()[rows], rtol=1e-5, atol=1e-5)
        if dnorm is not None:
            torch.testing.assert_close(y_, y.detach() if gather else y.detach()[rows], rtol=1e-5, atol=1e-5)
        want = [dp[rank].grad, dres.grad[rows], dbias.grad] + ([] if dnorm is None else
                                                               [t.grad for t in dnorm.parameters()])
        assert len(grads) == len(want)
        for g, w in zip(grads, want):
            torch.testing.assert_close(g, w, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("kind", ["layer", "rms", None])
@pytest.mark.parametrize("gather", [True, False])
def test_reduce_scatter_residual_norm_autograd_cpu(kind, gather):
    """CPU tensors run reduce_scatter_to_sequence, + bias, + residual, the module and
    gather_from_sequence, with the same gradients as the dense composition."""
    _check_sp_autograd(2, kind, gather)


def test_gather_and_scatter_operators_cpu():
    """gather_from_sequence and reduce_scatter_to_sequence against the dense composition: the
    gathered tensor is the concatenation of the shards and its gradient the sum over ranks of the
    shard's rows; the scattered tensor is the shard's rows of the sum and its gradient the gathered
    gradient."""
    P, Ts, H = 3, 2, 8
    xs = [torch.randn(Ts, 4, H, generator=_gen("shard", r)) for r in range(P)]
    parts = [torch.randn(P * Ts, 4, H, generator=_gen("full", r)) for r in range(P)]
    g_gather = [torch.randn(P * Ts, 4, H, generator=_gen("gg", r)) for r in range(P)]
    g_scatter = [torch.randn(Ts, 4, H, generator=_gen("gs", r)) for r in range(P)]

    def fn(ctx):
        sp = SequenceParallel(ctx)
        x = xs[ctx.rank].clone().requires_grad_(True)
        full = sp.gather_from_sequence(x)
        p = parts[ctx.rank].clone().requires_grad_(True)
        shard = sp.reduce_scatter_to_sequence(p)
        ((full * g_gather[ctx.rank]).sum() + (shard * g_scatter[ctx.rank]).sum()).backward()
        return full.detach(), shard.detach(), x.grad, p.grad

    want_full = torch.cat(xs)
    want_sum = sum(parts)
    want_xgrad = sum(g_gather)
    for r, (full, shard, xg, pg) in enumerate(gb.spawn_threads(P, fn)):
        rows = slice(r * Ts, (r + 1) * Ts)
        torch.testing.assert_close(full, want_full)
        torch.testing.assert_close(shard, want_sum[rows])
        torch.testing.assert_close(xg, want_xgrad[rows])
        torch.testing.assert_close(pg, torch.cat(g_scatter))


@pytest.mark.parametrize("P", [2, 4])
def test_sp_block_cpu_matches_dense(P):
    """models.TPBlock(sequence_parallel=True) on CPU tensors == DenseBlock, at the tolerances of
    sp_block_worker.py."""
    torch.manual_seed(19)
    B, S, E = 2, 12, 32
    dense = DenseBlock(d_model=E, n_heads=4, d_ff=64)
    x = torch.randn(B, S, E, requires_grad=True)
    out_d = dense(x)
    out_d.square().mean().backward()
    shard_of = lambda t, r: t.detach().transpose(0, 1)[S // P * r:S // P * (r + 1)]  # noqa: E731

    def fn(ctx):
        blk = TPBlock(TensorParallel(ctx), d_model=E, n_heads=4, d_ff=64, sequence_parallel=True)
        blk.load_dense(dense)
        xi = shard_of(x, ctx.rank).contiguous().requires_grad_(True)
        out = blk(xi)
        (out.square().sum() / (B * S * E)).backward()
        blk.sp.allreduce_sequence_parallel_grads(blk.sequence_parallel_parameters())
        return blk, out.detach(), xi.grad

    close = torch.testing.assert_close
    for r, (blk, out, xg) in enumerate(gb.spawn_threads(P, fn)):
        close(out, shard_of(out_d, r), rtol=1e-4, atol=1e-5)
        close(xg, shard_of(x.grad, r), rtol=1e-3, atol=1e-6)
        close(blk.up.weight.grad, dense.up.weight.grad[blk.up.lo:blk.up.hi], rtol=1e-3, atol=1e-6)
        close(blk.v.weight.grad, dense.qkv.weight.grad[2 * E + blk.v.lo:2 * E + blk.v.hi], rtol=1e-3, atol=1e-6)
        close(blk.proj.weight.grad, dense.proj.weight.grad[:, blk.proj.lo:blk.proj.hi], rtol=1e-3, atol=1e-6)
        for mine, want in ((blk.ln1, dense.ln1), (blk.ln2, dense.ln2)):
            close(mine.weight.grad, want.weight.grad, rtol=1e-3, atol=1e-6)
            close(mine.bias.grad, want.bias.grad, rtol=1e-3, atol=1e-6)
        close(blk.proj.bias.grad, dense.proj.bias.grad, rtol=1e-3, atol=1e-6)
        close(blk.down.bias.grad, dense.down.bias.grad, rtol=1e-3, atol=1e-6)
