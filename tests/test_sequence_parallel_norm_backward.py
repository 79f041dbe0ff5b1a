"""The fused backward of the sequence-parallel residual norm.

`CudaContext.reduce_scatter_residual_norm_backward` is checked against an fp64 reference built from
the rounded saved shard `s`: g = the exact sum of every rank's grad_out rows, the norm's statistics
and input gradient in fp64, plus grad_s. The tolerance of an element is one unit in the last place
of the dtype at the reference's magnitude plus an fp32 accumulation bound at the row's scale,
4 (H + P) 2^-24 times rinv (max|g|w| + max|x̂| mean|g|w x̂|) + max|grad_s| 2^-24, where |g| is the
sum of the summands' magnitudes (the fp32 sum over ranks errs in proportion to it, not to g); the
column sums get one ulp plus 4 (Ts + H + P) 2^-24 times the sum of their terms' magnitudes, with
|g| again (grad_bias: of the kernel's own rounded rows, 4 Ts 2^-24). Beyond that: every rank's
grad_partial has the same bytes,
grad_residual equals the rank's rows of it, guard bands and inputs are intact, a second identical
call gives identical bits, chunked runs give the same rows, launches equal the plan, malformed
calls raise and launch nothing.

Ranks are threads sharing cuda:0; sp_norm_backward_worker.py checks SequenceParallel's autograd with
one process per rank.
"""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu
from test_allreduce_norm import EPS, MAIN, _digest, _guarded, _guards_intact, _hidden, _launches
from test_reduce_numerics import _gen

# (Ts, H): every shard size with every H, the largest shard at the narrower rows
SHAPES = [(t, h) for t in (1, 3, 17) for h in ("min", 4096, 7168, 16384)] + [(125, "min"), (125, 4096), (125, 7168)]
NORMS = ("rms", "layer")
U = 2.0 ** -24


def _plan(cc, T, H, dtype, norm, gather, vectors):
    return gb._C.cuda.plan_reduce_scatter_norm_backward(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)),
                                                        {"rms": 1, "layer": 2}[norm], gather, vectors)


def _inputs(case, P, rank):
    """Rank `rank`'s grad_out, and the shards s / grad_s of every rank plus the weight (shared)."""
    dtype, norm, gather, with_gs, with_w, T, H = case[:7]
    Ts = T // P
    g_out = (torch.randn(T if gather else Ts, H, generator=_gen((case, "go"), rank), dtype=torch.float64)).to(dtype)
    s = (1.5 * torch.randn(T, H, generator=_gen((case, "s"), 0), dtype=torch.float64) + 0.25).to(dtype)
    gs = torch.randn(T, H, generator=_gen((case, "gs"), 0), dtype=torch.float64).to(dtype) if with_gs else None
    w = (0.5 + torch.rand(H, generator=_gen((case, "w"), 0), dtype=torch.float64)).to(dtype) if with_w else None
    return g_out, s, gs, w


def _ulp(ref, dtype):
    mant, emin = {torch.float32: (23, -126), torch.bfloat16: (7, -126), torch.float16: (10, -14)}[dtype]
    return torch.pow(2.0, torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin))) - mant)


def _reference(case, P):
    """fp64: (grad_residual of all T rows, per-rank column sums [(weight, norm_bias, |.| sums)], row bound)."""
    dtype, norm, gather, with_gs, with_w, T, H = case[:7]
    Ts = T // P
    outs = [_inputs(case, P, r)[0].double() for r in range(P)]
    _, s, gs, w = _inputs(case, P, 0)
    if gather:
        g, gabs = sum(outs), sum(o.abs() for o in outs)
    else:
        g = torch.cat(outs)  # rank r's grad_out is its own shard
        gabs = g.abs()
    x = s.double()
    mean = x.mean(-1, keepdim=True) if norm == "layer" else torch.zeros_like(x[:, :1])
    rinv = 1.0 / torch.sqrt((x - mean).square().mean(-1, keepdim=True) + EPS)
    xh = (x - mean) * rinv
    gg = g * (w.double() if w is not None else 1.0)
    mgg = gg.mean(-1, keepdim=True) if norm == "layer" else 0.0
    mggx = (gg * xh).mean(-1, keepdim=True)
    dx = rinv * (gg - mgg - xh * mggx)
    ref = dx + (gs.double() if gs is not None else 0.0)
    wabs = w.double().abs() if w is not None else 1.0
    scale = rinv * ((gabs * wabs).amax(-1, keepdim=True) +
                    xh.abs().amax(-1, keepdim=True) * (gabs * wabs * xh.abs()).mean(-1, keepdim=True))
    bound = _ulp(ref, dtype) + 4 * (H + P) * U * scale
    if gs is not None:
        bound = bound + U * gs.double().abs().amax(-1, keepdim=True)
    sums = []
    for r in range(P):
        rows = slice(r * Ts, (r + 1) * Ts)
        gx = g[rows] * xh[rows]
        sums.append((gx.sum(0), (gabs[rows] * xh[rows].abs()).sum(0), g[rows].sum(0), gabs[rows].sum(0)))
    return ref, sums, bound


def _vec_bad(got, want, mag, n_terms, dtype):
    got = got.cpu().double()
    tol = _ulp(want, dtype) + 4 * n_terms * U * mag
    bad = (got - want).abs() > tol
    if not bool(bad.any()):
        return None
    i = int(bad.nonzero()[0])
    return f"{int(bad.sum())} beyond tolerance, first {i}: got {got[i].item()!r} want {want[i].item()!r}"


def _run_case(cc, P, rank, case, repeat=False):
    """One call of this rank; returns (failures, (grad_partial, grad_residual, gw, gnb, gb) on the CPU)."""
    dtype, norm, gather, with_gs, with_w, T, H, in_place = case
    Ts = T // P
    bad = []
    g_out, s, gs, w = _inputs(case, P, rank)
    rows = slice(rank * Ts, (rank + 1) * Ts)
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    g_out, s_, gs_, w_ = dev(g_out), s[rows].cuda(), dev(None if gs is None else gs[rows]), dev(w)
    in_place = in_place and gs_ is not None
    inputs = [t for t in (g_out, s_, None if in_place else gs_, w_) if t is not None]
    kept = [t.clone() for t in inputs]
    praw, gp = _guarded((T, H), dtype)
    rraw, gr = (None, gs_) if in_place else _guarded((Ts, H), dtype)
    vraw = [_guarded((H,), dtype) for _ in range(3)]
    # without grad_s and weight, no column sums either: the launch without them (a frozen norm, no bias)
    sums = with_gs or with_w
    gw = vraw[0][1] if with_w else None
    gnb = vraw[1][1] if norm == "layer" and sums else None
    gb_ = vraw[2][1] if sums else None
    vectors = sum(t is not None for t in (gw, gnb, gb_))
    plan = _plan(cc, T, H, dtype, norm, gather, vectors)

    def call():
        got = cc.reduce_scatter_residual_norm_backward(g_out, s_, gs_, w_, norm=norm, eps=EPS, gather_out=gather,
                                                       grad_partial=gp, grad_residual=gr, grad_weight=gw,
                                                       grad_norm_bias=gnb, grad_bias=gb_)
        if got[0] is not gp or got[1] is not gr or got[2] is not gw or got[3] is not gnb or got[4] is not gb_:
            bad.append(f"{case}: returned other tensors than the outputs given")

    n = _launches(cc, call)
    want_variant = "local" if P == 1 else "reduce_scatter"
    chunks = -(-Ts // plan["chunk_rows"]) if Ts else 0
    if plan["variant"] != want_variant or plan["launches"] != chunks + (1 if vectors and Ts else 0):
        bad.append(f"{case}: plan {plan}")
    if n != P * plan["launches"]:
        bad.append(f"{case}: {n} launches over {P} ranks, planned {plan['launches']} each")
    for raw, what in [(praw, "grad_partial"), (rraw, "grad_residual")] + [(r, f"vector {k}") for k, (r, _) in enumerate(vraw)]:
        if raw is not None and not _guards_intact(raw):
            bad.append(f"{case}: wrote outside {what}")
    if not all(torch.equal(t, k) for t, k in zip(inputs, kept)):
        bad.append(f"{case}: an input changed")
    if not torch.equal(gr, gp[rows]):
        bad.append(f"{case}: grad_residual differs from the rank's rows of grad_partial")
    result = tuple(None if t is None else t.cpu().clone() for t in (gp, gr, gw, gnb, gb_))
    if repeat and not in_place:
        # the same call again: identical bits in every output
        call()
        cc.synchronize()
        again = tuple(None if t is None else t.cpu() for t in (gp, gr, gw, gnb, gb_))
        if any(a is not None and not torch.equal(a.view(torch.uint8), b.view(torch.uint8)) for a, b in zip(result, again)):
            bad.append(f"{case}: a second identical call gave other bits")
    return bad, result


def _check_reference(case, P, results):
    dtype, norm, gather, with_gs, with_w, T, H, _ = case
    Ts = T // P
    ref, sums, bound = _reference(case, P)
    bad = []
    for rank, (gp, gr, gw, gnb, gb_) in enumerate(results):
        over = (gp.double() - ref).abs() > bound
        if bool(over.any()):
            i = tuple(int(v) for v in over.nonzero()[0])
            bad.append(f"{case} rank {rank}: grad_partial {int(over.sum())} beyond tolerance, first {i}: "
                       f"got {gp.double()[i].item()!r} want {ref[i].item()!r} tol {bound[i].item()!r}")
        sw, aw, snb, anb = sums[rank]
        checks = [(gw, sw, aw, "grad_weight"), (gnb, snb, anb, "grad_norm_bias")]
        for got, want, mag, what in checks:
            if got is not None:
                m = _vec_bad(got, want, mag, Ts + H + P, dtype)
                if m:
                    bad.append(f"{case} rank {rank}: {what} {m}")
        own = gr.double()
        m = None if gb_ is None else _vec_bad(gb_, own.sum(0), own.abs().sum(0), Ts, dtype)
        if m:
            bad.append(f"{case} rank {rank}: grad_bias {m}")
    if len({_digest(gp) for gp, *_ in results}) != 1:
        bad.append(f"{case}: ranks hold different grad_partial bytes")
    return bad


def _cases(P):
    out, i = [], 0
    for dtype in MAIN:
        for norm in NORMS:
            for gather in (True, False):
                for with_gs, with_w in ((True, True), (False, False), (True, False), (False, True)):
                    Ts, h = SHAPES[(i + 5 * P) % len(SHAPES)]
                    out.append((dtype, norm, gather, with_gs, with_w, P * Ts, _hidden(h, dtype), i % 3 == 0))
                    i += 1
    return out


def _spawn(P, fn, stage_bytes=64 << 20):
    def body(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=stage_bytes)
        cc.set_timeout(120000)
        return fn(ctx, cc)

    return gb.spawn_threads(P, body, cuda_device=0, timeout_ms=600000)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_reduce_scatter_residual_norm_backward(P):
    """Every dtype x norm x gather_out x (grad_s, weight) over Ts in {1, 3, 17, 125} and H in {min,
    4096, 7168, 16384} against fp64; ranks agree, guard bands, inputs, in place, repeat, launches."""
    cases = _cases(P)

    def fn(ctx, cc):
        bad, outs = [], []
        for i, case in enumerate(cases):
            b, o = _run_case(cc, P, ctx.rank, case, repeat=i % 4 == 1)
            bad += [f"rank {ctx.rank} {x}" for x in b]
            outs.append(o)
        return bad, outs

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    for i, case in enumerate(cases):
        bad += _check_reference(case, P, [outs[i] for _, outs in results])
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3])
def test_chunked_equals_one_launch(P):
    """A 1 MiB pool: each shard runs as several chunks; the rows equal the one-launch run's bytes and
    the column sums (carried across chunks per CTA) agree within the tolerance."""
    Ts, H = 250, 4096
    cases = [(torch.bfloat16, "layer", True, True, True, P * Ts, H, False),
             (torch.float32, "rms", False, True, True, P * Ts, 1024, False)]

    def run(stage):
        def fn(ctx, cc):
            bad, outs = [], []
            for case in cases:
                plan = _plan(cc, case[5], case[6], case[0], case[1], case[2], 3 if case[1] == "layer" else 2)
                if stage < (64 << 20) and plan["launches"] < 3:
                    bad.append(f"{case}: plan {plan} does not chunk")
                b, o = _run_case(cc, P, ctx.rank, case)
                bad += b
                outs.append(o)
            return bad, outs

        return _spawn(P, fn, stage_bytes=stage)

    small, big = run(1 << 20), run(64 << 20)
    bad = [x for b, _ in small + big for x in b]
    for i, case in enumerate(cases):
        for rank in range(P):
            a, b = small[rank][1][i], big[rank][1][i]
            if not (torch.equal(a[0].view(torch.uint8), b[0].view(torch.uint8)) and torch.equal(a[1], b[1])):
                bad.append(f"{case} rank {rank}: chunked rows differ from the one-launch rows")
        bad += _check_reference(case, P, [outs[i] for _, outs in small])
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2])
def test_side_stream(P):
    """stream= a side stream: the workspace of the column sums belongs to that stream, so memory the
    current stream takes right after the call cannot be it; the results equal the current-stream
    call's bits."""
    Ts, H, dtype = 512, 8192, torch.bfloat16
    T = P * Ts

    def fn(ctx, cc):
        g = _gen("side-stream", ctx.rank)
        g_out = torch.randn(T, H, generator=g).to(dtype).cuda()
        s = torch.randn(Ts, H, generator=g).to(dtype).cuda()
        g_s = torch.randn(Ts, H, generator=g).to(dtype).cuda()
        w = (0.5 + torch.rand(H, generator=g)).to(dtype).cuda()
        ws_bytes = _plan(cc, T, H, dtype, "layer", True, 3)["workspace_bytes"]

        def outs():
            return {"grad_partial": torch.empty(T, H, dtype=dtype, device="cuda"),
                    "grad_residual": torch.empty(Ts, H, dtype=dtype, device="cuda"),
                    **{k: torch.empty(H, dtype=dtype, device="cuda") for k in ("grad_weight", "grad_norm_bias",
                                                                             "grad_bias")}}

        want = outs()
        cc.reduce_scatter_residual_norm_backward(g_out, s, g_s, w, norm="layer", **want)
        got = outs()
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        cc.reduce_scatter_residual_norm_backward(g_out, s, g_s, w, norm="layer", stream=side, **got)
        # the current stream at once writes memory of the workspace's size
        junk = [torch.empty(ws_bytes, dtype=torch.uint8, device="cuda").fill_(0xFF) for _ in range(4)]
        side.synchronize()
        torch.cuda.synchronize()
        del junk
        return [k for k in want if not torch.equal(want[k].view(torch.uint8), got[k].view(torch.uint8))]

    for bad in _spawn(P, fn):
        assert not bad, f"differ on the side stream: {bad}"


@pytest.mark.gpu
def test_empty_shard_zeroes_vectors():
    """Ts = 0: no launch, the requested column sums are zero."""
    P = 2

    def fn(ctx, cc):
        e = torch.empty(0, 64, dtype=torch.bfloat16, device="cuda")
        vecs = [torch.full((64,), 3.0, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
        n = _launches(cc, lambda: cc.reduce_scatter_residual_norm_backward(
            e, e, None, vecs[0].clone(), norm="layer", grad_weight=vecs[0], grad_norm_bias=vecs[1], grad_bias=vecs[2]))
        return n, [bool((v == 0).all()) for v in vecs]

    for n, zero in _spawn(P, fn, stage_bytes=16 << 20):
        assert n == 0 and all(zero)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
def test_back_to_back_forward_backward(P):
    """200 forward + backward pairs with no host synchronisation, gathered and not: each backward
    equals the one computed alone before."""
    Ts, H, dtype = 8, 1024, torch.bfloat16
    T = P * Ts
    kinds = [("rms", True), ("layer", False), ("layer", True), ("rms", False)]

    def fn(ctx, cc):
        rows = slice(ctx.rank * Ts, (ctx.rank + 1) * Ts)
        sets = []
        for k, (norm, gather) in enumerate(kinds):
            g, g0 = _gen(("b2b-bwd", k), ctx.rank), _gen(("b2b-bwd", k), 0)
            partial = torch.randn(T, H, generator=g).to(dtype).cuda()
            res = torch.randn(T, H, generator=g0).to(dtype)[rows].contiguous().cuda()
            w = (0.5 + torch.rand(H, generator=g0)).to(dtype).cuda()
            nb = torch.randn(H, generator=g0).to(dtype).cuda() if norm == "layer" else None
            g_out = torch.randn(T if gather else Ts, H, generator=g).to(dtype).cuda()
            g_s = torch.randn(Ts, H, generator=g).to(dtype).cuda()
            s, _ = cc.reduce_scatter_residual_norm(partial, res, w, nb, norm=norm, residual_out=torch.empty_like(res),
                                                   gather_out=gather)
            want = cc.reduce_scatter_residual_norm_backward(g_out, s, g_s, w, norm=norm, gather_out=gather,
                                                            grad_weight=torch.empty_like(w))
            sets.append((partial, res, w, nb, norm, gather, g_out, g_s, [t.clone() for t in want if t is not None]))
        cc.synchronize()
        cc.pc.host_barrier()
        got = []
        for i in range(200):
            partial, res, w, nb, norm, gather, g_out, g_s, _ = sets[i % 4]
            s, _ = cc.reduce_scatter_residual_norm(partial, res, w, nb, norm=norm, residual_out=torch.empty_like(res),
                                                   gather_out=gather)
            got.append(cc.reduce_scatter_residual_norm_backward(g_out, s, g_s, w, norm=norm, gather_out=gather,
                                                                grad_weight=torch.empty_like(w)))
        cc.synchronize()
        bad = []
        for i, g in enumerate(got):
            want = sets[i % 4][-1]
            if not all(torch.equal(a, b) for a, b in zip([t for t in g if t is not None], want)):
                bad.append(f"rank {ctx.rank} call {i}: differs")
        return bad

    for bad in _spawn(P, fn, stage_bytes=16 << 20):
        assert not bad, bad[:10]


@pytest.mark.gpu
def test_malformed_calls_raise_and_launch_nothing():
    P = 2

    def fn(ctx, cc):
        bf = torch.bfloat16
        go = torch.ones(4, 64, dtype=bf, device="cuda")
        s = torch.ones(2, 64, dtype=bf, device="cuda")
        w = torch.ones(64, dtype=bf, device="cuda")
        raw = torch.ones(4 * 64 + 8, dtype=bf, device="cuda")
        odd = torch.ones(2, 12, dtype=bf, device="cuda")  # 24-byte rows
        wide = torch.ones(1, 16384 + 8, dtype=bf, device="cuda")
        gp = torch.empty(4, 64, dtype=bf, device="cuda")
        dt = int(gb.DataType.BFLOAT16)
        bwd = cc.reduce_scatter_residual_norm_backward
        calls = {
            "no norm": lambda: bwd(go, s, None, w, norm=None),
            "bad norm": lambda: bwd(go, s, None, w, norm="batch"),
            "no norm (native)": lambda: gb._C.cuda.reduce_scatter_residual_norm_backward(
                cc.pc, go.data_ptr(), s.data_ptr(), 0, 0, gp.data_ptr(), 0, 0, 0, 0, 0, 0, 4, 64, dt, 0, 1e-6, True),
            "rows not divisible by P (native)": lambda: gb._C.cuda.reduce_scatter_residual_norm_backward(
                cc.pc, go.data_ptr(), s.data_ptr(), 0, 0, gp.data_ptr(), 0, 0, 0, 0, 0, 0, 3, 64, dt, 1, 1e-6, True),
            "workspace too small (native)": lambda: gb._C.cuda.reduce_scatter_residual_norm_backward(
                cc.pc, go.data_ptr(), s.data_ptr(), 0, 0, gp.data_ptr(), 0, w.clone().data_ptr(), 0, 0, 0, 0, 4, 64,
                dt, 1, 1e-6, True),
            "grad_norm_bias with rms": lambda: bwd(go, s, None, w, norm="rms", grad_norm_bias=torch.empty_like(w)),
            "shard grad_out with gather_out": lambda: bwd(s.clone(), s, None, w, norm="rms"),
            "gathered grad_out without gather_out": lambda: bwd(go, s, None, w, norm="rms", gather_out=False),
            "dtype mix": lambda: bwd(go.float(), s, None, w, norm="rms"),
            "weight dtype": lambda: bwd(go, s, None, w.half(), norm="rms"),
            "float64": lambda: bwd(go.double(), s.double(), None, w.double(), norm="rms"),
            "H not 16 bytes": lambda: bwd(torch.ones(4, 12, dtype=bf, device="cuda"), odd, None, None, norm="rms"),
            "H over the limit": lambda: bwd(torch.ones(2, 16384 + 8, dtype=bf, device="cuda"), wide, None, None,
                                            norm="rms"),
            "unaligned view": lambda: bwd(raw[1:1 + 256].view(4, 64), s, None, w, norm="rms"),
            "grad_partial is grad_out": lambda: bwd(go, s, None, w, norm="rms", grad_partial=go),
            "grad_residual in grad_partial": lambda: bwd(go, s, None, w, norm="rms", grad_partial=gp,
                                                         grad_residual=gp[2:]),
            "grad_residual is residual_out": lambda: bwd(go, s, None, w, norm="rms", grad_residual=s),
            "grad_residual overlaps grad_residual_out": lambda: bwd(
                go, s, raw[:128].view(2, 64), w, norm="rms", grad_residual=raw[8:8 + 128].view(2, 64)),
            "grad_weight is weight": lambda: bwd(go, s, None, w, norm="rms", grad_weight=w),
            "grad_bias is grad_weight": lambda: bwd(go, s, None, w, norm="rms", grad_weight=gp[0], grad_bias=gp[0]),
        }
        bad = []
        for name, call in calls.items():
            raised = []

            def go_():
                try:
                    call()
                except ValueError:
                    raised.append(True)

            if _launches(cc, go_) != 0 or not raised:
                bad.append(f"{name}: raised {bool(raised)}")
        return bad

    for bad in _spawn(P, fn, stage_bytes=16 << 20):
        assert not bad, bad


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sp_norm_backward_worker.py")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_sequence_parallel_autograd_fused_backward(size):
    """SequenceParallel.reduce_scatter_residual_norm's gradients on CUDA against the dense composition
    for rms and layer, gathered and not; the backward makes exactly the planned launches and no
    reduce_scatter or allgather of its own. One process per rank (sp_norm_backward_worker.py)."""
    d = tempfile.mkdtemp(prefix="glb_sp_bwd_")
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
