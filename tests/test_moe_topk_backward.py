"""The top-k MoE combine's backward (CudaContext.alltoallv_dev_combine_topk_backward), the unweighted
top-k combine (the dispatch's backward) and MoEDispatcher's autograd operators built on them. Ranks
are threads sharing cuda:0, each on its own stream, except for the autograd test: autograd runs the
backward of every thread of a process on one device thread, where a collective would wait for
itself, so it runs one process per rank (moe_autograd_worker.py)."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_combine_topk import DTYPES, H, _fresh_out, _pools, _problem, _reference, _route
from test_moe_dev import SENTINEL, _bytes, _layout

KINDS = ("symmetric", "registered", "plain")
GUARD = 2  # sentinel rows after each gradient tensor


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _exact_rows(n, dtype, seed, step):
    """n rows of H small integers times `step`: every product of two such values (steps 0.5 and
    0.25) and every partial sum of H of them is exact in fp32, so any summation order gives the
    same bits."""
    g = torch.Generator().manual_seed(seed)
    return (torch.randint(-8, 9, (n, H), generator=g).float() * step).to(dtype)


def _grad_rows(dy, pos, w, dtype):
    """The pushed gradient rows in dispatch-input order: row pos[t, j] = w[t, j] * dy[t], one fp32
    multiply rounded to dtype. Rows no choice names stay None."""
    n = int(pos.max()) + 1 if pos.numel() else 0
    rows = [None] * n
    for t in range(pos.shape[0]):
        for j in range(pos.shape[1]):
            p = int(pos[t, j])
            if p >= 0:
                rows[p] = (w[t, j, None] * dy[t].float()).to(dtype)
    return rows


def _grad_w_exact(dy, rows, pos):
    """grad_w with inputs whose every product and partial sum is exact: the dot in float64, then
    float32 (exact), +0.0 where pos = -1."""
    T, k = pos.shape
    out = torch.zeros(T, k)
    for t in range(T):
        for j in range(k):
            p = int(pos[t, j])
            if p >= 0:
                out[t, j] = float((dy[t].double() * rows[p].double()).sum())
    return out


def _holder_grad(per, d, P, E, align, cap, dtype):
    """Holder d's expected grad_expert_out: every source's gradient rows in the dispatch layout, +0
    in the gaps and the tail."""
    sp = [p["splits"].tolist() for p in per]
    osp, ooff, _ = _layout(sp, P, E, align, d)
    out = torch.zeros(cap, H, dtype=dtype)
    for e in range(E):
        for s in range(P):
            k = d * E + e
            src = sum(sp[s][:k])
            for r in range(sp[s][k]):
                out[ooff[e * P + s] + r] = per[s]["grad_rows"][src + r]
    return out


def _setup(P, E, k, dtype, seed, align, idle_last=True):
    """Every rank's routing, exact dispatch-input rows (expert outputs), dy and gate weights, the
    expected gradients, and each rank's need in rows."""
    per = []
    for s, (x, idx, w) in enumerate(_problem(P, E, k, dtype, seed, idle_last)):
        _, splits, pos = _route(P, x, idx, E)
        n = int(splits.sum())
        rows = _exact_rows(n, dtype, seed * 31 + s, 0.5)
        dy = _exact_rows(x.shape[0], dtype, seed * 37 + s, 0.25)
        per.append(dict(rows=rows, splits=splits, pos=pos, w=w, dy=dy, grad_rows=_grad_rows(dy, pos, w, dtype),
                        grad_w=_grad_w_exact(dy, rows, pos)))
    sp = [p["splits"].tolist() for p in per]
    needs = [_layout(sp, P, E, align, d)[2] for d in range(P)]
    return per, needs


def _tensors(kind, pools, cap, dtype, second=False):
    """A (cap + GUARD, H) sentinel-filled tensor and its first cap rows: a view of a symmetric or
    registered pool (its second half for `second`), or a plain tensor."""
    nbytes = (cap + GUARD) * H * torch.empty((), dtype=dtype).element_size()
    if kind == "plain":
        full = torch.empty((cap + GUARD, H), dtype=dtype, device="cuda")
    else:
        pool = pools[kind]
        at = pool.numel() // 2 if second else 0
        full = pool[at:at + nbytes].view(dtype).view(cap + GUARD, H)
    full.view(torch.uint8).fill_(SENTINEL)
    return full, full[:cap]


def _grad_w_tensor(T, k):
    full = torch.empty(T * k + 4, device="cuda")
    full.view(torch.uint8).fill_(SENTINEL)
    return full, full[:T * k].view(T, k)


def _dispatch(cc, eo, rank_data, E, align):
    osp = torch.empty(cc.size * E, dtype=torch.int64, device="cuda")
    cc.alltoallv_dev(eo, rank_data["rows"].cuda(), rank_data["splits"].cuda(), osp, torch.empty_like(osp), experts=E,
                     align=align)


def _backward(cc, geo, gw, eo, d, E, align, pos=None):
    cc.alltoallv_dev_combine_topk_backward(geo, gw, d["dy"].cuda(), eo, d["splits"].cuda(),
                                           (d["pos"] if pos is None else pos).cuda(), d["w"].cuda(), experts=E,
                                           align=align)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_backward_layouts(size):
    """Every (dtype, E, align, k, symmetric / registered / plain) at this P: grad_expert_out equals
    the reference at every named row and is +0 in every gap and tail row, the guard rows after it
    and after grad_w keep the sentinel, expert_out keeps every byte and grad_w equals the
    order-free reference bit for bit (+0.0 for dropped choices)."""
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        pools = _pools(cc, 2 << 20)
        me = ctx.rank
        case = 0
        for dtype in DTYPES:
            for E in (1, 2, 4):
                for align in (1, 8):
                    for k in (1, 2, 8):
                        case += 1
                        per, needs = _setup(P, E, k, dtype, 900 * case + P, align)
                        d = per[me]
                        T = d["pos"].shape[0]
                        cap = max(needs) + 3
                        want_geo = _bytes(_holder_grad(per, me, P, E, align, cap, dtype))
                        want_gw = _bytes(d["grad_w"])
                        for kind in KINDS:
                            _, eo = _tensors(kind, pools, cap, dtype)
                            geo_full, geo = _tensors(kind, pools, cap, dtype, second=True)
                            gw_full, gw = _grad_w_tensor(T, k)
                            _dispatch(cc, eo, d, E, align)
                            cc.synchronize()
                            before = _bytes(eo)
                            _backward(cc, geo, gw, eo, d, E, align)
                            cc.synchronize()
                            tag = (str(dtype), E, align, k, kind)
                            assert torch.equal(_bytes(geo), want_geo), tag
                            assert bool((_bytes(geo_full[cap:]) == SENTINEL).all()), tag
                            assert torch.equal(_bytes(gw), want_gw), tag
                            assert bool((_bytes(gw_full[T * k:]) == SENTINEL).all()), tag
                            assert torch.equal(_bytes(eo), before), tag
                            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=240000))


@pytest.mark.gpu
@pytest.mark.parametrize("size,kind", [(2, "plain"), (4, "symmetric")])
def test_backward_random(size, kind):
    """Random bf16 data, 256-element rows: grad_w is within n·2^-23·Σ|dy·x| of the fp64 dot (the
    bound of any fp32 summation of n = 256 terms), the pushed rows equal torch's bytes, and a second
    call gives identical bytes."""
    gcu = _cuda()
    P, E, k, align, Hd = size, 2, 4, 8, 256
    dtype = torch.bfloat16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        g = torch.Generator().manual_seed(77 + me)
        T = 40
        idx = torch.randint(0, P * E, (T, k), generator=g)
        x = torch.zeros(T, Hd)
        _, splits, pos = _route(P, x, idx, E)
        n = int(splits.sum())
        rows = torch.randn(n, Hd, generator=g).to(dtype)
        dy = torch.randn(T, Hd, generator=g).to(dtype)
        w = torch.rand(T, k, generator=g)
        cap = P * T * k + E * align
        mk = (lambda: cc.empty((cap, Hd), dtype)) if kind == "symmetric" else (
            lambda: torch.empty((cap, Hd), dtype=dtype, device="cuda"))
        eo, geo = mk(), mk()
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        cc.alltoallv_dev(eo, rows.cuda(), splits.cuda(), osp, ooff, experts=E, align=align)
        results = []
        for _ in range(2):
            geo.view(torch.uint8).fill_(SENTINEL)
            gw = torch.empty((T, k), device="cuda")
            cc.alltoallv_dev_combine_topk_backward(geo, gw, dy.cuda(), eo, splits.cuda(), pos.cuda(), w.cuda(),
                                                   experts=E, align=align)
            cc.synchronize()
            results.append((_bytes(geo), _bytes(gw)))
            cc.pc.host_barrier()
        assert torch.equal(results[0][0], results[1][0]) and torch.equal(results[0][1], results[1][1])
        got = gw.cpu().double()
        terms = dy.double()[:, None, :] * rows.double()[pos.clamp(min=0)]
        ref = terms.sum(-1)
        bound = Hd * 2.0 ** -23 * terms.abs().sum(-1)
        ok = pos >= 0
        assert bool(((got - ref).abs() <= bound)[ok].all())
        assert bool((got[~ok] == 0).all())
        # the rows this rank pushed, pulled back through the inverse exchange
        back = torch.empty((n, Hd), dtype=dtype, device="cuda")
        cc.alltoallv_dev_combine(back, geo, osp, ooff, experts=E)
        cc.synchronize()
        want = torch.empty(n, Hd, dtype=dtype)
        for t in range(T):
            for j in range(k):
                want[int(pos[t, j])] = (w[t, j, None] * dy[t].float()).to(dtype)
        assert torch.equal(_bytes(back), _bytes(want))
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 3])
def test_unweighted_combine(size):
    """weights=None gives the bytes of weights=ones for every dtype and kind of expert_out."""
    gcu = _cuda()
    P, E, k, align = size, 2, 3, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        pools = _pools(cc, 2 << 20)
        me = ctx.rank
        for i, dtype in enumerate(DTYPES):
            per, needs = _setup(P, E, k, dtype, 40 + i, align)
            d = per[me]
            T = d["pos"].shape[0]
            for kind in KINDS:
                _, eo = _tensors(kind, pools, max(needs) + 1, dtype)
                _dispatch(cc, eo, d, E, align)
                outs = []
                for w in (None, torch.ones(T, k, device="cuda")):
                    out = _fresh_out(T, dtype)
                    cc.alltoallv_dev_combine_topk(out, eo, d["splits"].cuda(), d["pos"].cuda(), w, experts=E,
                                                  align=align)
                    outs.append(out)
                cc.synchronize()
                tag = (str(dtype), kind)
                assert torch.equal(_bytes(outs[0]), _bytes(outs[1])), tag
                assert torch.equal(_bytes(outs[0]), _bytes(_reference(d["rows"], d["pos"], torch.ones(T, k), dtype))), tag
                cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (4, False)])
def test_graph_capture_replays(size, symmetric):
    """route, dispatch_dev and the backward captured once per rank; three replays with new routing,
    weights, rows and dy give the eager bytes."""
    gcu = _cuda()
    P, E, T, k, align = size, 2, 16, 2, 4
    G = P * E
    dtype = torch.float32

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        cap = P * (T * k + E * align)
        mk = (lambda: cc.empty((cap, H), dtype)) if symmetric else (lambda: torch.empty((cap, H), device="cuda"))
        got, geo, geo_eager = mk(), mk(), mk()
        x = torch.zeros((T, H), device="cuda")
        dy = torch.zeros((T, H), device="cuda")
        idx = torch.zeros((T, k), dtype=torch.int64, device="cuda")
        w = torch.zeros((T, k), device="cuda")
        gw, gw_eager = torch.empty((T, k), device="cuda"), torch.empty((T, k), device="cuda")

        def load(seed):
            g = torch.Generator().manual_seed(seed * 10 + me)
            i = torch.randint(0, G, (T, k), generator=g)
            i[torch.rand(T, k, generator=g) < 0.2] = -1
            x.copy_(torch.randn(T, H, generator=g))
            dy.copy_(torch.randn(T, H, generator=g))
            idx.copy_(i)
            w.copy_(torch.rand(T, k, generator=g))

        def step(geo_t, gw_t):
            rows, splits, pos = moe.route(x, idx, E)
            moe.dispatch_dev(rows, splits, got, experts=E, align=align)
            moe.combine_dev_topk_backward(dy, got, splits, pos, w, geo_t, gw_t, experts=E, align=align)

        stream = torch.cuda.current_stream()
        load(1)
        step(geo, gw)  # warm-up outside the graph
        cc.synchronize()
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            step(geo, gw)
        cc.pc.host_barrier()
        for seed in (2, 3, 4):
            load(seed)
            stream.synchronize()
            cc.pc.host_barrier()
            g.replay()
            cc.synchronize()
            cc.pc.host_barrier()
            step(geo_eager, gw_eager)
            cc.synchronize()
            assert torch.equal(_bytes(gw), _bytes(gw_eager)), seed
            assert torch.equal(_bytes(geo[:cap]), _bytes(geo_eager[:cap])), seed
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_no_host_sync(symmetric):
    """route, dispatch_dev and the backward run under torch's sync debug mode "error"."""
    gcu = _cuda()
    P, E, k, align = 2, 2, 2, 4
    dtype = torch.bfloat16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        per, needs = _setup(P, E, k, dtype, 42, align)
        d = per[ctx.rank]
        T = d["pos"].shape[0]
        cap = 64
        mk = (lambda: cc.empty((cap, H), dtype)) if symmetric else (
            lambda: torch.empty((cap, H), dtype=dtype, device="cuda"))
        eo, geo = mk(), mk()
        gw = torch.empty((T, k), device="cuda")
        rows, splits, pos, w, dy = (d[n].cuda() for n in ("rows", "splits", "pos", "w", "dy"))
        torch.cuda.current_stream().synchronize()
        cc.pc.host_barrier()
        if ctx.rank == 0:
            torch.cuda.set_sync_debug_mode("error")
        cc.pc.host_barrier()
        try:
            moe.dispatch_dev(rows, splits, eo, experts=E, align=align)
            moe.combine_dev_topk_backward(dy, eo, splits, pos, w, geo, gw, experts=E, align=align)
        finally:
            cc.pc.host_barrier()
            if ctx.rank == 0:
                torch.cuda.set_sync_debug_mode("default")
            cc.pc.host_barrier()
        cc.synchronize()
        assert torch.equal(_bytes(gw), _bytes(d["grad_w"]))
        assert torch.equal(_bytes(geo), _bytes(_holder_grad(per, ctx.rank, P, E, align, cap, dtype)))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
def test_host_errors():
    """Every malformed call raises ValueError before launch, alike on every rank; a correct call
    afterwards works, so none of them launched."""
    gcu = _cuda()
    P, E, k, align = 2, 1, 2, 1
    dtype = torch.float32

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        per, needs = _setup(P, E, k, dtype, 11, align, idle_last=False)
        d = per[ctx.rank]
        T = d["pos"].shape[0]
        cap = max(needs) + 2
        eo = cc.empty((cap, H), dtype)
        geo = cc.empty((cap, H), dtype)
        big = cc.empty((2 * cap + 2, H), dtype)
        _dispatch(cc, eo, d, E, align)
        cs, cp, cw, dy = d["splits"].cuda(), d["pos"].cuda(), d["w"].cuda(), d["dy"].cuda()
        gw = torch.empty((T, k), device="cuda")
        plain = torch.empty((cap, H), device="cuda")
        odd = torch.empty(T * H + 4, device="cuda")[1:T * H + 1].view(T, H)
        wide = cc.empty((cap, H + 1), dtype)
        ok = (geo, gw, dy, eo, cs, cp, cw)

        def sub(**kw):
            names = ("geo", "gw", "dy", "eo", "cs", "cp", "cw")
            return tuple(kw.get(n, v) for n, v in zip(names, ok))

        bad = {
            "float64 rows": sub(geo=geo.double(), dy=dy.double(), eo=eo.double()),
            "grad_out dtype differs": sub(dy=dy.half()),
            "grad_expert_out dtype differs": sub(geo=cc.empty((cap, H), torch.float16)),
            "grad_expert_out shape differs": sub(geo=geo[:-1]),
            "grad_weights bf16": sub(gw=gw.bfloat16()),
            "grad_weights shape": sub(gw=gw[:, :1].contiguous()),
            "pos int32": sub(cp=cp.int()),
            "weights bf16": sub(cw=cw.bfloat16()),
            "weights shape": sub(cw=cw[:, :1].contiguous()),
            "grad_out rows != T": sub(dy=torch.empty((T + 1, H), device="cuda")),
            "non-contiguous pos": sub(cp=torch.stack([cp, cp], 1)[:, 0]),
            "non-contiguous grad_out": sub(dy=torch.empty((H, T), device="cuda").t()),
            "rows not a multiple of 16 bytes": sub(geo=cc.empty((cap, H + 1), dtype), eo=wide,
                                                   dy=torch.empty((T, H + 1), device="cuda")),
            "grad_out not 16-byte aligned": sub(dy=odd),
            "k = 0": sub(gw=gw[:, :0], cp=cp[:, :0], cw=cw[:, :0]),
            "k = 33": sub(gw=gw[:, :1].repeat(1, 33), cp=cp[:, :1].repeat(1, 33), cw=cw[:, :1].repeat(1, 33)),
            "splits too short": sub(cs=cs[:-1]),
            "registered expert_out, plain grad_expert_out": sub(geo=plain),
            "plain expert_out, registered grad_expert_out": sub(eo=plain),
            "grad_expert_out overlaps expert_out": sub(geo=big[1:cap + 1], eo=big[:cap]),
            "grad_expert_out overlaps grad_out": sub(geo=big[:cap], dy=big[cap - T // 2:cap - T // 2 + T]),
            "grad_expert_out overlaps grad_weights": sub(geo=big[:cap], gw=big.view(-1)[:T * k].view(T, k)),
            "pos on the host": sub(cp=d["pos"]),
        }
        for why, args in bad.items():
            with pytest.raises(ValueError):
                cc.alltoallv_dev_combine_topk_backward(*args, experts=E, align=align)
                pytest.fail(why)
        cc.pc.host_barrier()
        cc.alltoallv_dev_combine_topk_backward(*ok, experts=E, align=align)
        cc.synchronize()
        assert torch.equal(_bytes(gw), _bytes(d["grad_w"]))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["symmetric", "plain"])
def test_device_errors(kind):
    """A bad pos on one rank, a capacity one row too small on one rank, and one rank running the
    forward combine while its peers run the backward each raise ValueError on every rank at
    synchronize(), with every grad_expert_out, grad_weights (and the combine's out) untouched and
    the context usable; a correct call right after works."""
    gcu = _cuda()
    P, E, k, align = 3, 2, 2, 4
    dtype = torch.bfloat16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        pools = _pools(cc, 2 << 20)
        me = ctx.rank
        per, needs = _setup(P, E, k, dtype, 23, align)
        d = per[me]
        T = d["pos"].shape[0]
        cap = max(needs) + 1
        small = 1
        assert needs[small] > 0
        _, eo = _tensors(kind, pools, cap, dtype)
        _dispatch(cc, eo, d, E, align)
        cc.synchronize()
        cc.pc.host_barrier()

        def fresh():
            geo_full, geo = _tensors(kind, pools, cap, dtype, second=True)
            gw_full, gw = _grad_w_tensor(T, k)
            return geo_full, geo, gw_full, gw

        def untouched(*ts):
            return all(bool((_bytes(t) == SENTINEL).all()) for t in ts)

        # a pos entry past the dispatch input on rank 0 (rank 2 has no tokens)
        bad_pos = d["pos"].clone()
        if me == 0:
            bad_pos[1, 0] = int(d["splits"].sum())
        geo_full, geo, gw_full, gw = fresh()
        _backward(cc, geo, gw, eo, d, E, align, pos=bad_pos)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        assert untouched(geo_full, gw_full)
        assert not cc.pc.poisoned()
        cc.pc.host_barrier()

        # one row too few on rank `small`
        geo_full, geo, gw_full, gw = fresh()
        n = needs[me] - 1 if me == small else cap
        _backward(cc, geo[:n], gw, eo[:n], d, E, align)
        with pytest.raises(ValueError, match=f"rank {small} needs {needs[small]} output rows but has room for "
                                             f"{needs[small] - 1}"):
            cc.synchronize()
        assert untouched(geo_full, gw_full)
        cc.pc.host_barrier()

        # rank 0 runs the forward combine, its peers the backward
        geo_full, geo, gw_full, gw = fresh()
        out = _fresh_out(T, dtype)
        if me == 0:
            cc.alltoallv_dev_combine_topk(out, eo, d["splits"].cuda(), d["pos"].cuda(), d["w"].cuda(), experts=E,
                                          align=align)
        else:
            _backward(cc, geo, gw, eo, d, E, align)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        assert untouched(geo_full, gw_full, out)
        cc.pc.host_barrier()

        geo_full, geo, gw_full, gw = fresh()
        _backward(cc, geo, gw, eo, d, E, align)
        cc.synchronize()
        assert torch.equal(_bytes(gw), _bytes(d["grad_w"]))
        assert torch.equal(_bytes(geo), _bytes(_holder_grad(per, me, P, E, align, cap, dtype)))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


def test_references_cpu():
    """The CPU references: pushed rows are w * dy rounded once, the exact dot is order-free (the
    same bits summed forwards and backwards in fp32), and the holder layout puts every source's
    rows where the dispatch puts them."""
    P, E, k, align = 3, 2, 3, 4
    per, needs = _setup(P, E, k, torch.bfloat16, 5, align)
    for d in per:
        for t in range(d["pos"].shape[0]):
            for j in range(k):
                p = int(d["pos"][t, j])
                if p < 0:
                    assert d["grad_w"][t, j].item() == 0.0
                    continue
                prod = d["dy"][t].float() * d["rows"][p].float()
                fwd, bwd = torch.zeros(()), torch.zeros(())
                for h in range(H):
                    fwd = fwd + prod[h]
                    bwd = bwd + prod[H - 1 - h]
                assert fwd.item() == bwd.item() == d["grad_w"][t, j].item()
    for dst in range(P):
        g = _holder_grad(per, dst, P, E, align, needs[dst] + 2, torch.bfloat16)
        assert bool((g[needs[dst]:] == 0).all())


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "moe_autograd_worker.py")


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_autograd_layer_processes(size):
    """One process per rank (rank % device_count, so ranks may share a GPU): a gate, the
    differentiable top-k dispatch, per-expert Linear + SiLU, the differentiable combine and a
    weighted-sum loss. x.grad, the gate's and every expert's weight gradients match a dense
    single-process CPU reference over all ranks' tokens, in fp32 and, looser, in bf16."""
    d = tempfile.mkdtemp(prefix="glb_moe_autograd_")
    procs = [subprocess.Popen([sys.executable, WORKER, d, str(r), str(size)], stdout=subprocess.PIPE,
                              stderr=subprocess.STDOUT, text=True) for r in range(size)]
    outs = []
    for p in procs:
        try:
            o, _ = p.communicate(timeout=600)
        except subprocess.TimeoutExpired:
            p.kill()
            o, _ = p.communicate()
        outs.append(o)
    for r, (p, o) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"WORKER {r} OK" in o, f"rank {r} failed:\n{o[-3000:]}"
