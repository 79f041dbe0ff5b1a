"""The fused backward of the tensor-parallel residual norm.

`CudaContext.allreduce_residual_norm_backward` is checked against an fp64 reference built from the
rounded saved `s`: g = the exact sum of every rank's grad_out rows, the norm's statistics and input
gradient in fp64, plus grad_s, with the per-element and column-sum bounds of
test_sequence_parallel_norm_backward.py (the column sums now over all T rows). Beyond that:
grad_partial has the same bytes on every rank, for one_shot, two_shot and auto, and as the
gathered grad_partial of the reduce-scatter backward given the same partials; the column sums have
the same bytes on every rank and on a repeated call; guard bands and inputs are intact; an in-place
call gives the same bytes; chunked runs give the same rows; launches equal the plan; malformed calls
raise and launch nothing.

Ranks are threads sharing cuda:0; tp_norm_backward_worker.py checks TensorParallel's autograd and
TPBlock with one process per rank.
"""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu
from gloo_b200.parallel import TensorParallel
from test_allreduce_norm import EPS, MAIN, _digest, _guarded, _guards_intact, _hidden, _launches
from test_reduce_numerics import _gen
from test_sequence_parallel_norm_backward import U, _spawn, _ulp, _vec_bad

# (T, H): every row count with every H, the most rows at the narrower rows
SHAPES = [(t, h) for t in (1, 3, 17) for h in ("min", 4096, 7168, 16384)] + [(250, "min"), (250, 4096), (120, 7168)]
NORMS = ("rms", "layer")
ALGOS = ("one_shot", "two_shot", "auto")


def _plan(cc, T, H, dtype, norm, vectors, algo="auto"):
    return gb._C.cuda.plan_residual_norm_backward(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)),
                                                  {"rms": 1, "layer": 2}[norm], vectors, gcu.ALGOS[algo])


def _inputs(case, rank):
    """Rank `rank`'s grad_out partial, and s / grad_s / weight (the same on every rank)."""
    case = case[:6]  # the problem: the same inputs under every algo
    dtype, norm, with_gs, with_w, T, H = case
    g_out = torch.randn(T, H, generator=_gen((case, "go"), rank), dtype=torch.float64).to(dtype)
    s = (1.5 * torch.randn(T, H, generator=_gen((case, "s"), 0), dtype=torch.float64) + 0.25).to(dtype)
    gs = torch.randn(T, H, generator=_gen((case, "gs"), 0), dtype=torch.float64).to(dtype) if with_gs else None
    w = (0.5 + torch.rand(H, generator=_gen((case, "w"), 0), dtype=torch.float64)).to(dtype) if with_w else None
    return g_out, s, gs, w


def _reference(case, P):
    """fp64: (grad_partial, (weight sum, |.|, norm-bias sum, |.|) over all rows, per-element bound)."""
    dtype, norm, with_gs, with_w, T, H = case[:6]
    outs = [_inputs(case, r)[0].double() for r in range(P)]
    _, s, gs, w = _inputs(case, 0)
    g, gabs = sum(outs), sum(o.abs() for o in outs)
    x = s.double()
    mean = x.mean(-1, keepdim=True) if norm == "layer" else torch.zeros_like(x[:, :1])
    rinv = 1.0 / torch.sqrt((x - mean).square().mean(-1, keepdim=True) + EPS)
    xh = (x - mean) * rinv
    gg = g * (w.double() if w is not None else 1.0)
    mgg = gg.mean(-1, keepdim=True) if norm == "layer" else 0.0
    dx = rinv * (gg - mgg - xh * (gg * xh).mean(-1, keepdim=True))
    ref = dx + (gs.double() if gs is not None else 0.0)
    wabs = w.double().abs() if w is not None else 1.0
    scale = rinv * ((gabs * wabs).amax(-1, keepdim=True) +
                    xh.abs().amax(-1, keepdim=True) * (gabs * wabs * xh.abs()).mean(-1, keepdim=True))
    bound = _ulp(ref, dtype) + 4 * (H + P) * U * scale
    if gs is not None:
        bound = bound + U * gs.double().abs().amax(-1, keepdim=True)
    sums = ((g * xh).sum(0), (gabs * xh.abs()).sum(0), g.sum(0), gabs.sum(0))
    return ref, sums, bound


def _raw(t):
    return None if t is None else t.view(torch.uint8)


def _run_case(cc, P, rank, case, repeat=False):
    """One call of this rank; returns (failures, (grad_partial, gw, gnb, gb) on the CPU)."""
    dtype, norm, with_gs, with_w, T, H, algo, in_place = case
    bad = []
    g_out, s, gs, w = _inputs(case, rank)
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    g_out, s_, gs_, w_ = dev(g_out), s.cuda(), dev(gs), dev(w)
    in_place = in_place and gs_ is not None
    inputs = [t for t in (g_out, s_, None if in_place else gs_, w_) if t is not None]
    kept = [t.clone() for t in inputs]
    want_inplace = gs_.clone() if in_place else None
    praw, gp = (None, gs_) if in_place else _guarded((T, H), dtype)
    vraw = [_guarded((H,), dtype) for _ in range(3)]
    # without grad_s and weight, no column sums either: the launch of a frozen norm without bias
    sums = with_gs or with_w
    gw = vraw[0][1] if with_w else None
    gnb = vraw[1][1] if norm == "layer" and sums else None
    gb_ = vraw[2][1] if sums else None
    vectors = sum(t is not None for t in (gw, gnb, gb_))
    plan = _plan(cc, T, H, dtype, norm, vectors, algo)

    def call():
        got = cc.allreduce_residual_norm_backward(g_out, s_, gs_, w_, norm=norm, eps=EPS, grad_partial=gp,
                                                  grad_weight=gw, grad_norm_bias=gnb, grad_bias=gb_, algo=algo)
        if got[0] is not gp or got[1] is not gw or got[2] is not gnb or got[3] is not gb_:
            bad.append(f"{case}: returned other tensors than the outputs given")

    n = _launches(cc, call)
    want_variant = {"one_shot": "one_shot", "two_shot": "two_shot"}.get(algo) if P > 1 else "local"
    if (want_variant and plan["variant"] != want_variant and
            not (algo == "one_shot" and plan["variant"] == "two_shot")) or plan["variant"] == "ll":
        bad.append(f"{case}: plan {plan}")
    if plan["launches"] != -(-T // plan["chunk_rows"]) + (1 if vectors else 0):
        bad.append(f"{case}: plan {plan}")
    if n != P * plan["launches"]:
        bad.append(f"{case}: {n} launches over {P} ranks, planned {plan['launches']} each")
    for raw, what in [(praw, "grad_partial")] + [(r, f"vector {k}") for k, (r, _) in enumerate(vraw)]:
        if raw is not None and not _guards_intact(raw):
            bad.append(f"{case}: wrote outside {what}")
    if not all(torch.equal(t, k) for t, k in zip(inputs, kept)):
        bad.append(f"{case}: an input changed")
    result = tuple(None if t is None else t.cpu().clone() for t in (gp, gw, gnb, gb_))
    if in_place:
        # the same call out of place: the same bytes
        again = cc.allreduce_residual_norm_backward(g_out, s_, want_inplace, w_, norm=norm, eps=EPS, algo=algo)[0]
        if not torch.equal(_raw(again.cpu()), _raw(result[0])):
            bad.append(f"{case}: the in-place call differs from the out-of-place one")
    elif repeat:
        call()
        cc.synchronize()
        again = tuple(None if t is None else t.cpu() for t in (gp, gw, gnb, gb_))
        if any(a is not None and not torch.equal(_raw(a), _raw(b)) for a, b in zip(result, again)):
            bad.append(f"{case}: a second identical call gave other bits")
    return bad, (result, plan["variant"])


def _check_reference(case, P, results):
    dtype, norm, with_gs, with_w, T, H, algo, _ = case
    ref, (sw, aw, snb, anb), bound = _reference(case, P)
    bad = []
    gp, gw, gnb, gb_ = results[0]
    over = (gp.double() - ref).abs() > bound
    if bool(over.any()):
        i = tuple(int(v) for v in over.nonzero()[0])
        bad.append(f"{case}: grad_partial {int(over.sum())} beyond tolerance, first {i}: "
                   f"got {gp.double()[i].item()!r} want {ref[i].item()!r} tol {bound[i].item()!r}")
    for got, want, mag, what in [(gw, sw, aw, "grad_weight"), (gnb, snb, anb, "grad_norm_bias")]:
        m = None if got is None else _vec_bad(got, want, mag, T + H + P, dtype)
        if m:
            bad.append(f"{case}: {what} {m}")
    own = gp.double()
    m = None if gb_ is None else _vec_bad(gb_, own.sum(0), own.abs().sum(0), T, dtype)
    if m:
        bad.append(f"{case}: grad_bias {m}")
    for k, what in enumerate(("grad_partial", "grad_weight", "grad_norm_bias", "grad_bias")):
        if len({_digest(r[k]) for r in results if r[k] is not None}) > 1:
            bad.append(f"{case}: ranks hold different {what} bytes")
    return bad


def _cases(P):
    """Each (dtype, norm, grad_s / weight) problem under every algo, consecutively."""
    out, i = [], 0
    for dtype in MAIN:
        for norm in NORMS:
            for with_gs, with_w in ((True, True), (False, False), (True, False), (False, True)):
                T, h = SHAPES[(i + 5 * P) % len(SHAPES)]
                for algo in ALGOS:
                    out.append((dtype, norm, with_gs, with_w, T, _hidden(h, dtype), algo, algo == "auto" and i % 3 == 0))
                i += 1
    return out


def _scatter_rows(cc, P, rank, case):
    """grad_partial of reduce_scatter_residual_norm_backward(gather_out=True) on the same partials and
    this rank's shards of s / grad_s."""
    dtype, norm, with_gs, with_w, T, H = case[:6]
    g_out, s, gs, w = _inputs(case, rank)
    rows = slice(rank * (T // P), (rank + 1) * (T // P))
    got = cc.reduce_scatter_residual_norm_backward(g_out.cuda(), s[rows].contiguous().cuda(),
                                                   None if gs is None else gs[rows].contiguous().cuda(),
                                                   None if w is None else w.cuda(), norm=norm, eps=EPS)
    return got[0].cpu()


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_allreduce_residual_norm_backward(P):
    """Every dtype x norm x (grad_s, weight) x algo over T in {1, 3, 17, 120, 250} and H in {min, 4096,
    7168, 16384} against fp64; ranks and variants agree, and match the reduce-scatter backward's
    rows; guard bands, inputs, in place, repeat, launches."""
    cases = _cases(P)

    def fn(ctx, cc):
        bad, outs = [], []
        for i, case in enumerate(cases):
            b, o = _run_case(cc, P, ctx.rank, case, repeat=i % 4 == 1)
            bad += [f"rank {ctx.rank} {x}" for x in b]
            sp = _scatter_rows(cc, P, ctx.rank, case) if case[4] % P == 0 and case[6] == "auto" else None
            outs.append((o, sp))
        return bad, outs

    results = _spawn(P, fn)
    bad = [x for b, _ in results for x in b]
    for i, case in enumerate(cases):
        per_rank = [outs[i][0][0] for _, outs in results]
        bad += _check_reference(case, P, per_rank)
        if case[6] == "auto":
            # the three algos of one problem are consecutive: the same rows
            first = cases.index(case[:6] + ("one_shot", False))
            for j in range(first, i + 1):
                if not torch.equal(_raw(results[0][1][j][0][0][0]), _raw(per_rank[0][0])):
                    bad.append(f"{cases[j]}: grad_partial differs from {case}")
            sp = results[0][1][i][1]
            if sp is not None and not torch.equal(_raw(sp), _raw(per_rank[0][0])):
                bad.append(f"{case}: grad_partial differs from the reduce-scatter backward's")
    assert not bad, "\n".join(bad[:40])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3])
def test_chunked_two_shot_equals_one_launch(P):
    """A 1 MiB pool: the two-shot runs as several chunks; the rows equal the one-launch run's bytes
    and the column sums (carried across chunks per CTA) agree within the tolerance."""
    cases = [(torch.bfloat16, "layer", True, True, 500, 4096, "two_shot", False),
             (torch.float32, "rms", False, True, 333, 1024, "two_shot", False)]

    def run(stage):
        def fn(ctx, cc):
            bad, outs = [], []
            for case in cases:
                plan = _plan(cc, case[4], case[5], case[0], case[1], 3 if case[1] == "layer" else 2, "two_shot")
                if stage < (64 << 20) and plan["launches"] < 3:
                    bad.append(f"{case}: plan {plan} does not chunk")
                b, (o, _) = _run_case(cc, P, ctx.rank, case)
                bad += b
                outs.append(o)
            return bad, outs

        return _spawn(P, fn, stage_bytes=stage)

    small, big = run(1 << 20), run(64 << 20)
    bad = [x for b, _ in small + big for x in b]
    for i, case in enumerate(cases):
        for rank in range(P):
            if not torch.equal(_raw(small[rank][1][i][0]), _raw(big[rank][1][i][0])):
                bad.append(f"{case} rank {rank}: chunked rows differ from the one-launch rows")
        bad += _check_reference(case, P, [outs[i] for _, outs in small])
    assert not bad, "\n".join(bad[:20])


@pytest.mark.gpu
def test_empty_rows_zeroes_vectors():
    """rows = 0: no launch, the requested column sums are zero."""
    P = 2

    def fn(ctx, cc):
        e = torch.empty(0, 64, dtype=torch.bfloat16, device="cuda")
        vecs = [torch.full((64,), 3.0, dtype=torch.bfloat16, device="cuda") for _ in range(3)]
        n = _launches(cc, lambda: cc.allreduce_residual_norm_backward(
            e, e, None, vecs[0].clone(), norm="layer", grad_weight=vecs[0], grad_norm_bias=vecs[1], grad_bias=vecs[2]))
        return n, [bool((v == 0).all()) for v in vecs]

    for n, zero in _spawn(P, fn, stage_bytes=16 << 20):
        assert n == 0 and all(zero)


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
def test_back_to_back_with_forward_and_allreduce(P):
    """200 backward calls with no host synchronisation, alternating one_shot and two_shot, each after
    a forward and a plain cc.allreduce on the same pool: each equals the call made alone before."""
    T, H, dtype = 24, 1024, torch.bfloat16
    kinds = [("rms", "one_shot"), ("layer", "two_shot"), ("layer", "one_shot"), ("rms", "two_shot")]

    def fn(ctx, cc):
        sets = []
        for k, (norm, algo) in enumerate(kinds):
            g, g0 = _gen(("b2b-ar-bwd", k), ctx.rank), _gen(("b2b-ar-bwd", k), 0)
            partial = torch.randn(T, H, generator=g).to(dtype).cuda()
            res = torch.randn(T, H, generator=g0).to(dtype).cuda()
            w = (0.5 + torch.rand(H, generator=g0)).to(dtype).cuda()
            nb = torch.randn(H, generator=g0).to(dtype).cuda() if norm == "layer" else None
            g_out = torch.randn(T, H, generator=g).to(dtype).cuda()
            g_s = torch.randn(T, H, generator=g0).to(dtype).cuda()
            flat = torch.randn(5000, generator=g).cuda()
            s, _ = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, residual_out=torch.empty_like(res),
                                              algo=algo)
            want = cc.allreduce_residual_norm_backward(g_out, s, g_s, w, norm=norm, algo=algo,
                                                       grad_weight=torch.empty_like(w), grad_bias=torch.empty_like(w))
            sets.append((partial, res, w, nb, norm, algo, g_out, g_s, flat, [t.clone() for t in want if t is not None]))
        cc.synchronize()
        cc.pc.host_barrier()
        got = []
        for i in range(200):
            partial, res, w, nb, norm, algo, g_out, g_s, flat, _ = sets[i % 4]
            s, _ = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, residual_out=torch.empty_like(res),
                                              algo=algo)
            cc.allreduce(flat.clone())
            got.append(cc.allreduce_residual_norm_backward(g_out, s, g_s, w, norm=norm, algo=algo,
                                                           grad_weight=torch.empty_like(w),
                                                           grad_bias=torch.empty_like(w)))
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
        s = torch.ones(4, 64, dtype=bf, device="cuda")
        w = torch.ones(64, dtype=bf, device="cuda")
        raw = torch.ones(4 * 64 + 8, dtype=bf, device="cuda")
        gp = torch.empty(4, 64, dtype=bf, device="cuda")
        dt = int(gb.DataType.BFLOAT16)
        bwd = cc.allreduce_residual_norm_backward
        native = gb._C.cuda.allreduce_residual_norm_backward
        calls = {
            "no norm": lambda: bwd(go, s, None, w, norm=None),
            "bad norm": lambda: bwd(go, s, None, w, norm="batch"),
            "bad algo": lambda: bwd(go, s, None, w, norm="rms", algo="ll"),
            "bad algo (native)": lambda: native(cc.pc, go.data_ptr(), s.data_ptr(), 0, gp.data_ptr(), 0, 0, 0, 0, 0, 0,
                                                4, 64, dt, 1, 1e-6, gcu.ALGOS["pipelined"]),
            "no norm (native)": lambda: native(cc.pc, go.data_ptr(), s.data_ptr(), 0, gp.data_ptr(), 0, 0, 0, 0, 0, 0,
                                               4, 64, dt, 0, 1e-6),
            "workspace too small (native)": lambda: native(cc.pc, go.data_ptr(), s.data_ptr(), 0, gp.data_ptr(), 0,
                                                           w.clone().data_ptr(), 0, 0, 0, 0, 4, 64, dt, 1, 1e-6),
            "grad_norm_bias with rms": lambda: bwd(go, s, None, w, norm="rms", grad_norm_bias=torch.empty_like(w)),
            "grad_norm_bias with rms (native)": lambda: native(cc.pc, go.data_ptr(), s.data_ptr(), 0, gp.data_ptr(), 0,
                                                               0, w.clone().data_ptr(), 0, 0, 0, 4, 64, dt, 1, 1e-6),
            "grad_out shape": lambda: bwd(go[:2].clone(), s, None, w, norm="rms"),
            "dtype mix": lambda: bwd(go.float(), s, None, w, norm="rms"),
            "weight dtype": lambda: bwd(go, s, None, w.half(), norm="rms"),
            "float64": lambda: bwd(go.double(), s.double(), None, w.double(), norm="rms"),
            "H not 16 bytes": lambda: bwd(torch.ones(2, 12, dtype=bf, device="cuda"),
                                          torch.ones(2, 12, dtype=bf, device="cuda"), None, None, norm="rms"),
            "H over the limit": lambda: bwd(torch.ones(1, 16384 + 8, dtype=bf, device="cuda"),
                                            torch.ones(1, 16384 + 8, dtype=bf, device="cuda"), None, None, norm="rms"),
            "unaligned view": lambda: bwd(raw[1:1 + 256].view(4, 64), s, None, w, norm="rms"),
            "unaligned view (native)": lambda: native(cc.pc, raw.data_ptr() + 2, s.data_ptr(), 0, gp.data_ptr(), 0, 0,
                                                      0, 0, 0, 0, 4, 64, dt, 1, 1e-6),
            "grad_partial is grad_out": lambda: bwd(go, s, None, w, norm="rms", grad_partial=go),
            "grad_partial is residual_out": lambda: bwd(go, s, None, w, norm="rms", grad_partial=s),
            "grad_partial overlaps grad_residual_out": lambda: bwd(
                go, s, raw[:256].view(4, 64), w, norm="rms", grad_partial=raw[8:8 + 256].view(4, 64)),
            "grad_weight is weight": lambda: bwd(go, s, None, w, norm="rms", grad_weight=w),
            "grad_weight in grad_partial": lambda: bwd(go, s, None, w, norm="rms", grad_partial=gp, grad_weight=gp[0]),
            "grad_bias is grad_weight": lambda: bwd(go, s, None, w, norm="rms", grad_weight=raw[:64],
                                                    grad_bias=raw[:64]),
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


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tp_norm_backward_worker.py")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_tensor_parallel_autograd_fused_backward(size):
    """TensorParallel.reduce_residual_norm(copy_out=True) and TPBlock on CUDA against the dense
    compositions: the backward calls the fused entry once, no allreduce of its own, makes the planned
    launches, and gives every rank the same bytes of the norm and bias gradients. One process per
    rank (tp_norm_backward_worker.py)."""
    d = tempfile.mkdtemp(prefix="glb_tp_bwd_")
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


# ---- CPU ----------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["layer", "rms"])
def test_copy_out_cpu_is_copy_to_region_of_the_norm(kind):
    """On CPU tensors, reduce_residual_norm(copy_out=True) gives the values and gradients of
    copy_to_region(norm_module(s)) after the unfused sequence."""
    P, T, H = 2, 3, 16
    parts = [torch.randn(T, H, generator=_gen(("cpu-copy", kind), r)) for r in range(P)]
    residual, bias = torch.randn(T, H, generator=_gen(("cpu-res", kind), 0)), torch.randn(H)
    g_s, g_o = torch.randn(T, H), [torch.randn(T, H, generator=_gen(("cpu-go", kind), r)) for r in range(P)]

    def norm_module():
        m = torch.nn.LayerNorm(H) if kind == "layer" else torch.nn.RMSNorm(H, eps=1e-6)
        with torch.no_grad():
            m.weight.copy_(0.5 + torch.rand(H, generator=_gen(("cpu-w", kind), 0)))
        return m

    def fn(ctx):
        tp = TensorParallel(ctx)
        got = []
        for copy_out in (True, False):
            p = parts[ctx.rank].clone().requires_grad_(True)
            res, b = residual.clone().requires_grad_(True), bias.clone().requires_grad_(True)
            m = norm_module()
            if copy_out:
                s, y = tp.reduce_residual_norm(p, res, m, b, copy_out=True)
            else:
                y_ = tp.reduce_from_region(p) + b
                s = y_ + res
                y = tp.copy_to_region(m(s))
            ((s * g_s).sum() + (y * g_o[ctx.rank]).sum()).backward()
            got.append([s.detach(), y.detach(), p.grad, res.grad, b.grad] + [t.grad for t in m.parameters()])
        return got

    for fused, plain in gb.spawn_threads(P, fn):
        assert len(fused) == len(plain)
        for a, b in zip(fused, plain):
            torch.testing.assert_close(a, b)


def test_copy_out_needs_a_norm():
    def fn(ctx):
        with pytest.raises(ValueError):
            TensorParallel(ctx).reduce_residual_norm(torch.ones(2, 16), torch.ones(2, 16), None, copy_out=True)
        return True

    assert all(gb.spawn_threads(2, fn))
