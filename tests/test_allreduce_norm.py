"""The tensor-parallel allreduce fused with bias, residual add and RMSNorm / LayerNorm.

`CudaContext.allreduce_residual_norm` against an fp64 reference, `TensorParallel.reduce_residual_norm`
against the unfused composition under autograd, and `models.TPBlock` on CUDA against `DenseBlock`.

The inputs of the sum come from the order-free generators of test_reduce_numerics.py: the exact
value of `sum_r partial_r + bias + residual` (at most 10 terms) is an fp32 value whatever the
order, so `residual_out` has exactly one correct byte pattern. `out` is checked against an fp64 norm
of that `residual_out`: within one unit in the last place of a 16-bit output, or a relative 2e-6 in
fp32, plus 1e-6 of the row's largest |out| for the elements the mean subtraction of LayerNorm
brings near zero (fp32 statistics have an absolute error there, not a relative one).

Ranks are threads sharing cuda:0, as in the other GPU tests. Rank 0 computes the reference; every
rank returns digests of its outputs, which must be the same on every rank.
"""
import hashlib
import math
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu
from gloo_b200.parallel import TensorParallel
from test_reduce_numerics import _gen, _mismatch, _sum_values

MAIN = (torch.float32, torch.bfloat16, torch.float16)
NORMS = ("rms", "layer", None)
ALGOS = ("auto", "ll", "one_shot", "two_shot")
# (T, H): every T with every H at decode sizes; prefill-sized T at the narrower rows
SHAPES = [(t, h) for t in (1, 3, 17) for h in ("min", 4096, 7168, 16384)] + [(1000, "min"), (1000, 4096)]
PAD = 256  # bytes of sentinel on each side of an output
SENTINEL = 0xA5
EPS = 1e-6


def _es(dtype):
    return torch.empty((), dtype=dtype).element_size()


def _hidden(h, dtype):
    return 16 // _es(dtype) if h == "min" else h


def _inputs(case, P, T, H, dtype, ranks):
    """Partials of `ranks`, and the shared residual, bias, weight and norm_bias."""
    parts = {r: _sum_values(dtype, T * H, _gen((case, "p"), r)).view(T, H) for r in ranks}
    residual = _sum_values(dtype, T * H, _gen((case, "res"), 0)).view(T, H)
    bias = _sum_values(dtype, H, _gen((case, "b"), 0))
    weight = (0.5 + torch.rand(H, generator=_gen((case, "w"), 0), dtype=torch.float64)).to(dtype)
    norm_bias = (0.25 * torch.randn(H, generator=_gen((case, "nb"), 0), dtype=torch.float64)).to(dtype)
    return parts, residual, bias, weight, norm_bias


def _reference(parts, residual, bias, weight, norm_bias, norm, dtype):
    exact = sum(p.double() for p in parts) + residual.double()
    if bias is not None:
        exact = exact + bias.double()
    res_out = exact.to(torch.float32).to(dtype)  # exact in fp32, rounded once
    if norm is None:
        return res_out, None
    x = res_out.double()
    if norm == "rms":
        y = x / torch.sqrt(x.square().mean(-1, keepdim=True) + EPS) * weight.double()
    else:
        m = x.mean(-1, keepdim=True)
        y = (x - m) / torch.sqrt((x - m).square().mean(-1, keepdim=True) + EPS) * weight.double() + norm_bias.double()
    return res_out, y


def _close(got, ref, dtype):
    """None if `got` is within the tolerance of the fp64 `ref` (module docstring), else a message."""
    got = got.cpu().double()
    scale = ref.abs().amax(-1, keepdim=True)
    if dtype == torch.float32:
        tol = 2e-6 * ref.abs()
    else:
        mant, emin = {torch.bfloat16: (7, -126), torch.float16: (10, -14)}[dtype]
        e = torch.floor(torch.log2(ref.abs().clamp_min(2.0 ** emin)))
        tol = torch.pow(2.0, e - mant)
    bad = (got - ref).abs() > tol + 1e-6 * scale
    if not bool(bad.any()):
        return None
    i = tuple(int(v) for v in bad.nonzero()[0])
    return f"{int(bad.sum())} of {got.numel()} beyond tolerance, first {i}: got {got[i].item()!r} want {ref[i].item()!r}"


def _kind(norm):
    return {None: 0, "rms": 1, "layer": 2}[norm]


def _guarded(shape, dtype):
    """An output with PAD sentinel bytes on each side: (backing bytes, view)."""
    n = math.prod(shape) * _es(dtype)
    raw = torch.full((n + 2 * PAD,), SENTINEL, dtype=torch.uint8, device="cuda")
    return raw, raw[PAD:PAD + n].view(dtype).view(shape)


def _guards_intact(raw):
    return bool((raw[:PAD] == SENTINEL).all()) and bool((raw[-PAD:] == SENTINEL).all())


def _digest(t):
    return hashlib.sha1(t.contiguous().view(torch.uint8).cpu().numpy().tobytes()).hexdigest()


def _launches(cc, fn):
    """Launches of every rank during fn(), which every rank calls at the same point."""
    cc.pc.host_barrier()
    before = gb._C.cuda.launch_count()
    cc.pc.host_barrier()
    try:
        fn()
    finally:
        cc.synchronize()
        cc.pc.host_barrier()
        after = gb._C.cuda.launch_count()
        cc.pc.host_barrier()
    return after - before


def _cases(P):
    out = []
    i = 0
    for dtype in MAIN:
        for norm in NORMS:
            for with_bias in (True, False):
                for algo in ALGOS:
                    T, h = SHAPES[(i + 3 * P) % len(SHAPES)]
                    out.append((dtype, norm, with_bias, algo, T, _hidden(h, dtype), i % 2 == 0))
                    i += 1
    return out


def _run_case(cc, P, rank, case):
    """One fused call; returns (failures seen by this rank, digests of its outputs)."""
    dtype, norm, with_bias, algo, T, H, in_place = case
    bad = []
    parts, residual, bias, weight, norm_bias = _inputs(case, P, T, H, dtype, range(P) if rank == 0 else [rank])
    bias = bias if with_bias else None
    weight = weight if norm is not None else None
    norm_bias = norm_bias if norm == "layer" else None
    dev = lambda t: None if t is None else t.cuda()  # noqa: E731
    partial, res, b, w, nb = dev(parts[rank]), dev(residual), dev(bias), dev(weight), dev(norm_bias)
    inputs = [t for t in (partial, None if in_place else res, b, w, nb) if t is not None]
    kept = [t.clone() for t in inputs]
    rraw, rout = (None, None) if in_place else _guarded((T, H), dtype)
    oraw, out = _guarded((T, H), dtype) if norm is not None else (None, None)
    plan = gb._C.cuda.plan_residual_norm(cc.pc, T, H, int(gcu._torch_dtype_to_glb(dtype)), _kind(norm), gcu.ALGOS[algo])
    got = {}

    def call():
        got["r"] = cc.allreduce_residual_norm(partial, res, w, nb, norm=norm, eps=EPS, bias=b, residual_out=rout,
                                              out=out, algo=algo)

    n = _launches(cc, call)
    if plan["launches"] != 1 and not (plan["variant"] == "two_shot" and plan["launches"] == -(-T // plan["chunk_rows"])):
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
    if rank == 0:
        want_r, want_o = _reference([parts[q] for q in range(P)], residual, bias, weight, norm_bias, norm, dtype)
        m = _mismatch(res_out.reshape(-1), want_r.reshape(-1))
        if m is not None:
            bad.append(f"{case}: residual_out {m}")
        if norm is not None:
            m = _close(out, want_o, dtype)
            if m is not None:
                bad.append(f"{case}: out {m}")
    for raw, what in ((rraw, "residual_out"), (oraw, "out")):
        if raw is not None and not _guards_intact(raw):
            bad.append(f"{case}: wrote outside {what}")
    if not all(torch.equal(t, k) for t, k in zip(inputs, kept)):
        bad.append(f"{case}: an input changed")
    return bad, (_digest(res_out), None if out is None else _digest(out), plan["variant"])


@pytest.mark.gpu
@pytest.mark.parametrize("P", [1, 2, 3, 4, 8])
def test_allreduce_residual_norm(P):
    """Every dtype x norm x bias x algo, over T in {1, 3, 17, 1000} and H in {min, 4096, 7168, 16384}."""
    cases = _cases(P)

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=64 << 20)
        cc.set_timeout(120000)
        bad, digests = [], []
        for case in cases:
            b, d = _run_case(cc, P, ctx.rank, case)
            bad += [f"rank {ctx.rank} {x}" for x in b]
            digests.append(d)
        return bad, digests

    results = gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=600000)
    bad = [x for b, _ in results for x in b]
    for i, case in enumerate(cases):
        seen = {d[i][:2] for _, d in results}
        if len(seen) != 1:
            bad.append(f"{case}: ranks differ")
    variants = {d[i][2] for _, d in results for i in range(len(cases))}
    assert not bad, "\n".join(bad[:40])
    assert variants == ({"local"} if P == 1 else {"ll", "one_shot", "two_shot"}), variants


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 3])
def test_chunked_two_shot(P):
    """A 1 MiB pool: the row-sharded two-shot runs as ceil(rows / chunk rows) launches, each exact."""
    stage = 1 << 20
    dtype, T, H = torch.bfloat16, 1000, 4096

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=stage)
        cc.set_timeout(120000)
        t = gb._C.cuda.get_tuning()
        half = min(-(-max(t["one_shot_max_bytes"], 4096) // 4096) * 4096, stage // 4)
        bulk = stage - 2 * half
        bad = []
        for norm in ("layer", None):
            case = (dtype, norm, True, "two_shot", T, H, False)
            plan = gb._C.cuda.plan_residual_norm(cc.pc, T, H, int(gb.DataType.BFLOAT16), _kind(norm), gcu.ALGOS["two_shot"])
            chunk = bulk // ((2 if norm else 1) * H * 2)
            if plan["chunk_rows"] != chunk or plan["launches"] != -(-T // chunk) or plan["launches"] < 2:
                bad.append(f"plan {plan}, want chunks of {chunk} rows")
            b, d = _run_case(cc, P, ctx.rank, case)
            bad += b
        return bad, d

    results = gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=600000)
    assert not [x for b, _ in results for x in b], results[0][0]
    assert len({d[:2] for _, d in results}) == 1


@pytest.mark.gpu
def test_malformed_calls_raise_and_launch_nothing():
    P = 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        cc.set_timeout(60000)
        bf = torch.bfloat16
        p = torch.ones(4, 64, dtype=bf, device="cuda")
        r = torch.ones(4, 64, dtype=bf, device="cuda")
        w = torch.ones(64, dtype=bf, device="cuda")
        raw = torch.ones(4 * 64 + 8, dtype=bf, device="cuda")
        odd = torch.ones(4, 12, dtype=bf, device="cuda")  # 24-byte rows
        wide = torch.ones(1, 16384 + 8, dtype=bf, device="cuda")
        calls = {
            "dtype mix": lambda: cc.allreduce_residual_norm(p, r.float(), w),
            "weight dtype": lambda: cc.allreduce_residual_norm(p, r, w.half()),
            "float64": lambda: cc.allreduce_residual_norm(p.double(), r.double(), w.double()),
            "H not 16 bytes": lambda: cc.allreduce_residual_norm(odd, odd.clone(), None),
            "H over the limit": lambda: cc.allreduce_residual_norm(wide, wide.clone(), None),
            "unaligned view": lambda: cc.allreduce_residual_norm(raw[1:1 + 256].view(4, 64), r, w),
            "out is partial": lambda: cc.allreduce_residual_norm(p, r, w, out=p),
            "residual_out is partial": lambda: cc.allreduce_residual_norm(p, r, w, residual_out=p),
            "residual_out overlaps residual": lambda: cc.allreduce_residual_norm(
                p, raw[:256].view(4, 64), w, residual_out=raw[8:8 + 256].view(4, 64)),
            "out is residual_out": lambda: cc.allreduce_residual_norm(p, r, w, out=r),
            "out is weight": lambda: cc.allreduce_residual_norm(p[:1], r[:1], w, out=w.view(1, 64)),
            "bad norm": lambda: cc.allreduce_residual_norm(p, r, w, norm="batch"),
            "bad algo": lambda: cc.allreduce_residual_norm(p, r, w, algo="nvls"),
            "shape": lambda: cc.allreduce_residual_norm(p, r[:2], w),
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

    for bad in gb.spawn_threads(P, fn, cuda_device=0):
        assert not bad, bad


# ---- autograd ---------------------------------------------------------------------------------


def _norm_module(kind, H):
    if kind == "layer":
        m = torch.nn.LayerNorm(H)
    elif kind == "rms":
        m = torch.nn.RMSNorm(H, eps=1e-5)
    else:
        return None
    with torch.no_grad():
        m.weight.copy_(0.5 + torch.rand(H, generator=_gen(("w", kind), 0)))
        if getattr(m, "bias", None) is not None:
            m.bias.copy_(0.1 * torch.randn(H, generator=_gen(("nb", kind), 0)))
    return m


@pytest.mark.gpu
@pytest.mark.parametrize("P", [2, 4])
@pytest.mark.parametrize("kind", ["layer", "rms", None])
def test_reduce_residual_norm_autograd(P, kind):
    """Forward and the gradients of partial, residual, bias, weight and norm_bias against the unfused
    composition run densely in one process."""
    T, H = 6, 256
    parts = [torch.randn(T, H, generator=_gen(("part", kind), r), dtype=torch.float64).float() for r in range(P)]
    residual = torch.randn(T, H, generator=_gen(("res", kind), 0), dtype=torch.float64).float()
    bias = torch.randn(H, generator=_gen(("bias", kind), 0), dtype=torch.float64).float()
    g_r = torch.randn(T, H, generator=_gen(("gr", kind), 0), dtype=torch.float64).float()
    g_o = torch.randn(T, H, generator=_gen(("go", kind), 0), dtype=torch.float64).float()

    # dense: every partial is a leaf, the sum is what g computes
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
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        cc.set_timeout(60000)
        tp = TensorParallel(ctx, cc)
        p = parts[ctx.rank].cuda().requires_grad_(True)
        res = residual.cuda().requires_grad_(True)
        b = bias.cuda().requires_grad_(True)
        norm = _norm_module(kind, H)
        norm = norm.cuda() if norm is not None else None
        got = tp.reduce_residual_norm(p, res, norm, b)
        s_, y_ = (got, None) if norm is None else got
        loss = (s_ * g_r.cuda()).sum()
        if y_ is not None:
            loss = loss + (y_ * g_o.cuda()).sum()
        loss.backward()
        grads = [t.grad.cpu() for t in (p, res, b)]
        if norm is not None:
            grads += [norm.weight.grad.cpu()] + ([norm.bias.grad.cpu()] if getattr(norm, "bias", None) is not None else [])
        return s_.detach().cpu(), None if y_ is None else y_.detach().cpu(), grads

    for s_, y_, grads in gb.spawn_threads(P, fn, cuda_device=0):
        torch.testing.assert_close(s_, s.detach(), rtol=1e-5, atol=1e-5)
        if dnorm is not None:
            torch.testing.assert_close(y_, y.detach(), rtol=1e-5, atol=1e-5)
        want = [dp[0].grad, dres.grad, dbias.grad]
        if dnorm is not None:
            want += [dnorm.weight.grad] + ([dnorm.bias.grad] if getattr(dnorm, "bias", None) is not None else [])
        assert len(grads) == len(want)
        for g, w in zip(grads, want):
            torch.testing.assert_close(g, w, rtol=1e-4, atol=1e-4)


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "tp_block_worker.py")


@pytest.mark.gpu
def test_tp_block_cuda_matches_dense():
    """models.TPBlock on CUDA at P = 2 (each row-parallel output fused with bias, residual and ln2) ==
    DenseBlock: output, input gradient and shard gradients, at the tolerances of
    test_tensor_parallel_transformer_block_matches_dense; a forward is two collective launches. One
    process per rank (tp_block_worker.py): the backward's allreduces cannot share an autograd thread."""
    size = 2
    d = tempfile.mkdtemp(prefix="glb_tp_block_")
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


# ---- CPU: the reference and the unfused path ---------------------------------------------------


def test_reference_residual_is_exact():
    """The inputs make `sum partials + bias + residual` exact in fp32 in any order."""
    for dtype in MAIN:
        case = ("cpu", str(dtype))
        parts, residual, bias, _, _ = _inputs(case, 8, 3, 64, dtype, range(8))
        terms = [parts[r].float() for r in range(8)] + [bias.float().expand(3, 64), residual.float()]
        exact = sum(t.double() for t in terms)
        for order in (range(10), reversed(range(10)), [9, 0, 8, 1, 7, 2, 6, 3, 5, 4]):
            acc = torch.zeros(3, 64)
            for i in order:
                acc = acc + terms[i]
            assert torch.equal(acc.double(), exact)


def test_reduce_residual_norm_cpu_is_the_unfused_sequence():
    """CPU tensors run reduce_from_region, + bias, + residual and the module."""
    P, T, H = 2, 3, 16
    parts = [torch.randn(T, H, generator=_gen("cpu", r)) for r in range(P)]
    residual, bias = torch.randn(T, H), torch.randn(H)
    norm = torch.nn.LayerNorm(H)

    def fn(ctx):
        tp = TensorParallel(ctx)
        s, y = tp.reduce_residual_norm(parts[ctx.rank].clone(), residual, norm, bias)
        return s, y.detach()

    s_want = sum(parts) + bias + residual
    for s, y in gb.spawn_threads(P, fn):
        torch.testing.assert_close(s, s_want)
        torch.testing.assert_close(y, norm(s_want).detach())
