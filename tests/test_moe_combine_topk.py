"""The top-k MoE combine: CudaContext.alltoallv_dev_combine_topk, and MoEDispatcher.route /
combine_dev_topk built around it. Ranks are threads sharing cuda:0, each on its own stream. References
are computed on the CPU, in the kernel's fp32 order."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_dev import SENTINEL, _bytes, _layout
from test_moe_fp8_dispatch import _dequant

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
H = 24  # row bytes: 96 (float32), 48 (16-bit types)


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


class _Ranks:
    """route() needs only the group size."""

    def __init__(self, size):
        self.size = size


def _route(P, x, idx, E):
    return MoEDispatcher.route(_Ranks(P), x, idx, E)


def _reference(rows, pos, w, dtype):
    """The documented CPU expression: byte for byte what the kernel computes."""
    T, k = pos.shape
    acc = torch.zeros(T, rows.shape[1])
    for j in range(k):
        m = pos[:, j] >= 0
        acc[m] = acc[m] + w[m, j, None] * rows[pos[m, j]].float()
    return acc.to(dtype)


def _chunk_of(splits, n):
    """The chunk (global expert) of each of the first n dispatch input rows."""
    return torch.repeat_interleave(torch.arange(splits.numel()), splits)[:n]


def _expert(rows, chunks, dtype):
    """A per-row 'expert' that depends on its global expert, computed on the CPU."""
    c = chunks.float()[:, None]
    return (rows.float() * (1 + 0.125 * c) - 0.5 * c).to(dtype)


def _problem(P, E, k, dtype, seed, idle_last=True):
    """Every rank's tokens, top-k indices (-1 entries, a token with every choice dropped, and an
    idle last rank) and gate weights."""
    g = torch.Generator().manual_seed(seed)
    G = P * E
    out = []
    for s in range(P):
        T = 0 if (idle_last and P > 1 and s == P - 1) else int(torch.randint(3, 20, (1,), generator=g))
        x = torch.randn(T, H, generator=g).to(dtype)
        idx = torch.randint(0, G, (T, k), generator=g)
        idx[torch.rand(T, k, generator=g) < 0.2] = -1
        if T > 0:
            idx[0] = -1
        w = torch.rand(T, k, generator=g) * 2 - 0.5
        out.append((x, idx, w))
    return out


def _setup(P, E, k, dtype, seed, align, idle_last=True):
    """Per rank: (dispatch input rows of expert outputs, splits, pos, weights) and each rank's need."""
    per = []
    for x, idx, w in _problem(P, E, k, dtype, seed, idle_last):
        rows, splits, pos = _route(P, x, idx, E)
        n = int(splits.sum())
        y = _expert(rows[:n], _chunk_of(splits, n), dtype)
        per.append((y, splits, pos, w))
    sp = [p[1].tolist() for p in per]
    needs = [_layout(sp, P, E, align, d)[2] for d in range(P)]
    return per, needs


def _expert_out(cc, kind, pools, cap, dtype):
    """An expert_out of `cap` rows filled with the sentinel: a view of a symmetric or a registered
    buffer, or a plain tensor."""
    nbytes = cap * H * torch.empty((), dtype=dtype).element_size()
    if kind == "plain":
        t = torch.empty((cap, H), dtype=dtype, device="cuda")
    else:
        t = pools[kind][:nbytes].view(dtype).view(cap, H)
    t.view(torch.uint8).fill_(SENTINEL)
    return t


def _fresh_out(T, dtype):
    out = torch.empty((T, H), dtype=dtype, device="cuda")
    out.view(torch.uint8).fill_(SENTINEL)
    return out


def _pools(cc, nbytes):
    reg = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    cc.register(reg)
    return {"symmetric": cc.empty(nbytes, torch.uint8), "registered": reg}


def _run_case(cc, me, per, needs, E, align, dtype, kind, pools):
    """Dispatch rank me's expert rows into expert_out, then the top-k combine. Returns
    (out, expert_out bytes before the combine, expert_out)."""
    y, splits, pos, w = per[me]
    cap = max(needs) + 3
    eo = _expert_out(cc, kind, pools, cap, dtype)
    osp = torch.empty(cc.size * E, dtype=torch.int64, device="cuda")
    ooff = torch.empty_like(osp)
    cc.alltoallv_dev(eo, y.cuda(), splits.cuda(), osp, ooff, experts=E, align=align)
    cc.synchronize()
    before = _bytes(eo)
    out = _fresh_out(pos.shape[0], dtype)
    cc.alltoallv_dev_combine_topk(out, eo, splits.cuda(), pos.cuda(), w.cuda(), experts=E, align=align)
    return out, before, eo


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_combine_topk_layouts(size):
    """Every (dtype, E, align, k, symmetric / registered / plain expert_out) at this P: out equals the
    CPU reference bit for bit and expert_out keeps every byte."""
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        pools = _pools(cc, 1 << 20)
        me = ctx.rank
        case = 0
        for dtype in DTYPES:
            for E in (1, 2, 4):
                for align in (1, 8):
                    for k in (1, 2, 8):
                        case += 1
                        per, needs = _setup(P, E, k, dtype, 500 * case + P, align)
                        y, splits, pos, w = per[me]
                        want = _bytes(_reference(y, pos, w, dtype))
                        for kind in ("symmetric", "registered", "plain"):
                            out, before, eo = _run_case(cc, me, per, needs, E, align, dtype, kind, pools)
                            cc.synchronize()
                            tag = (str(dtype), E, align, k, kind)
                            assert torch.equal(_bytes(out), want), tag
                            assert torch.equal(_bytes(eo), before), tag
                            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=240000))


def _moe_expert(x, e_global):
    a = 0.5 + 0.125 * e_global
    return (torch.nn.functional.silu(x * a) * (1.0 - 0.0625 * e_global)).to(x.dtype)


def _weighted_sum(back, pos, w, dtype):
    """The composed path's last step on the device, in the same order as the kernel."""
    acc = torch.zeros(pos.shape[0], back.shape[1], device=back.device)
    for j in range(pos.shape[1]):
        m = pos[:, j] >= 0
        term = acc + w[:, j, None] * back[pos[:, j].clamp(min=0)].float()
        acc = torch.where(m[:, None], term, acc)
    return acc.to(dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("size,fp8", [(2, False), (4, False), (2, True), (4, True)])
def test_moe_layer_end_to_end(size, fp8):
    """route -> dispatch_dev (or dispatch_dev_fp8) -> experts -> combine_dev_topk equals the composed
    path (combine_dev, un-permute, weighted sum) byte for byte, and the dense layer within tolerance."""
    gcu = _cuda()
    P, E, T, Hd, k = size, 2, 24, 256, 3
    G = P * E

    def routed(rank):
        g = torch.Generator().manual_seed(700 + rank)
        x = torch.randn(T, Hd, generator=g).to(torch.bfloat16)
        w, idx = torch.topk(torch.softmax(torch.randn(T, G, generator=g), dim=-1), k, dim=-1)
        idx[5, 1] = -1  # a dropped choice (capacity)
        return x, w / w.sum(-1, keepdim=True), idx

    def dense(rank):
        x, w, idx = routed(rank)
        y = torch.zeros(T, Hd)
        for t in range(T):
            for j in range(k):
                if int(idx[t, j]) >= 0:
                    y[t] += w[t, j] * _moe_expert(x[t:t + 1], int(idx[t, j]))[0].float()
        return y

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        x, w, idx = (t.cuda() for t in routed(me))
        rows, splits, pos = moe.route(x, idx, E)
        cap = T * k * P
        if fp8:
            codes = cc.empty((cap, Hd), torch.float8_e4m3fn)
            scales = cc.empty((cap, Hd // 128), torch.float32)
            _, _, osp, ooff = moe.dispatch_dev_fp8(rows, splits, codes, scales, experts=E)
            got = _dequant(codes, scales)
        else:
            got = cc.empty((cap, Hd), torch.bfloat16)
            _, osp, ooff = moe.dispatch_dev(rows, splits, got, experts=E)
        expert_out = cc.empty((cap, Hd), torch.bfloat16)
        expert_out.zero_()
        osp_h, ooff_h = osp.tolist(), ooff.tolist()
        for e in range(E):
            lo, hi = ooff_h[e * P], ooff_h[e * P + P - 1] + osp_h[e * P + P - 1]
            expert_out[lo:hi] = _moe_expert(got[lo:hi], me * E + e)
        y = torch.empty((T, Hd), dtype=torch.bfloat16, device="cuda")
        moe.combine_dev_topk(expert_out, splits, pos, w, y, experts=E)
        back = torch.empty_like(rows)
        moe.combine_dev(expert_out, osp, ooff, back, experts=E)
        y_comp = _weighted_sum(back, pos, w, torch.bfloat16)
        cc.synchronize()
        assert torch.equal(_bytes(y), _bytes(y_comp))
        tol = dict(rtol=0.05, atol=0.15) if fp8 else dict(rtol=2e-2, atol=2e-2)
        torch.testing.assert_close(y.float().cpu(), dense(me), **tol)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (4, False)])
def test_graph_capture_replays(size, symmetric):
    """route, dispatch_dev, the experts and combine_dev_topk captured once per rank; three replays
    with new routing, weights and tokens are all correct."""
    gcu = _cuda()
    P, E, T, k, align = size, 2, 16, 2, 4
    G = P * E

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        cap = P * (T * k + E * align)
        got = cc.empty((cap, H), torch.float32) if symmetric else torch.empty((cap, H), device="cuda")
        expert_out = cc.empty((cap, H), torch.float32) if symmetric else torch.empty((cap, H), device="cuda")
        x = torch.zeros((T, H), device="cuda")
        idx = torch.zeros((T, k), dtype=torch.int64, device="cuda")
        w = torch.zeros((T, k), device="cuda")
        y = torch.empty((T, H), device="cuda")

        def load(seed):
            g = torch.Generator().manual_seed(seed * 10 + me)
            i = torch.randint(0, G, (T, k), generator=g)
            i[torch.rand(T, k, generator=g) < 0.2] = -1
            x.copy_(torch.randn(T, H, generator=g))
            idx.copy_(i)
            w.copy_(torch.rand(T, k, generator=g))

        def step():
            rows, splits, pos = moe.route(x, idx, E)
            moe.dispatch_dev(rows, splits, got, experts=E, align=align)
            torch.mul(got, 0.75, out=expert_out)  # the experts: a row-wise map, so gaps do not matter
            moe.combine_dev_topk(expert_out, splits, pos, w, y, experts=E, align=align)

        stream = torch.cuda.current_stream()
        load(1)
        step()  # warm-up outside the graph
        cc.synchronize()
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            step()
        cc.pc.host_barrier()
        for seed in (2, 3, 4):
            load(seed)
            stream.synchronize()
            cc.pc.host_barrier()
            g.replay()
            cc.synchronize()
            rows, _, pos = _route(P, x.cpu(), idx.cpu(), E)
            want = _reference(rows * 0.75, pos, w.cpu(), torch.float32)
            assert torch.equal(_bytes(y), _bytes(want)), seed
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_no_host_sync(symmetric):
    """route, dispatch_dev and combine_dev_topk run under torch's sync debug mode "error"."""
    gcu = _cuda()
    P, E, T, k = 2, 2, 12, 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        per = _problem(P, E, k, torch.bfloat16, 42)
        x, idx, w = per[ctx.rank]
        x, idx, w = x.cuda(), idx.cuda(), w.cuda()
        cap = 64
        got = cc.empty((cap, H), torch.bfloat16) if symmetric else torch.empty((cap, H), dtype=torch.bfloat16,
                                                                             device="cuda")
        y = torch.empty((x.shape[0], H), dtype=torch.bfloat16, device="cuda")
        torch.cuda.current_stream().synchronize()
        cc.pc.host_barrier()
        if ctx.rank == 0:
            torch.cuda.set_sync_debug_mode("error")
        cc.pc.host_barrier()
        try:
            rows, splits, pos = moe.route(x, idx, E)
            moe.dispatch_dev(rows, splits, got, experts=E, align=4)
            moe.combine_dev_topk(got, splits, pos, w, y, experts=E, align=4)
        finally:
            cc.pc.host_barrier()
            if ctx.rank == 0:
                torch.cuda.set_sync_debug_mode("default")
            cc.pc.host_barrier()
        cc.synchronize()
        rows, _, pos = _route(P, x.cpu(), idx.cpu(), E)
        assert torch.equal(_bytes(y), _bytes(_reference(rows, pos, w.cpu(), torch.bfloat16)))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
def test_host_errors():
    """Every malformed call raises ValueError before launch, alike on every rank; a correct call
    afterwards works, so none of them launched."""
    gcu = _cuda()
    P, E, k = 2, 1, 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        per, needs = _setup(P, E, k, torch.float32, 11, 1, idle_last=False)  # non-contiguous needs rows
        y, splits, pos, w = per[ctx.rank]
        T = pos.shape[0]
        eo = cc.empty((max(needs) + 2, H), torch.float32)
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        cc.alltoallv_dev(eo, y.cuda(), splits.cuda(), osp, torch.empty_like(osp), experts=E)
        cs, cp, cw = splits.cuda(), pos.cuda(), w.cuda()
        out = torch.empty((T, H), device="cuda")
        odd = torch.empty(T * H + 4, device="cuda")[1:T * H + 1].view(T, H)
        wide = torch.empty((eo.shape[0], H + 1), device="cuda")
        bad = {
            "float64 rows": (out.double(), eo.double(), cs, cp, cw),
            "out dtype differs": (out.half(), eo, cs, cp, cw),
            "pos int32": (out, eo, cs, cp.int(), cw),
            "weights bf16": (out, eo, cs, cp, cw.bfloat16()),
            "weights shape": (out, eo, cs, cp, cw[:, :1].contiguous()),
            "out rows != T": (torch.empty((T + 1, H), device="cuda"), eo, cs, cp, cw),
            "out row width": (torch.empty((T, H * 2), device="cuda"), eo, cs, cp, cw),
            "1-D expert_out": (torch.empty(T, device="cuda"), eo.view(-1), cs, cp, cw),
            "non-contiguous pos": (out, eo, cs, torch.stack([cp, cp], 1)[:, 0], cw),
            "non-contiguous expert_out": (out, eo.t().contiguous().t(), cs, cp, cw),
            "rows not a multiple of 16 bytes": (torch.empty((T, H + 1), device="cuda"), wide, cs, cp, cw),
            "out not 16-byte aligned": (odd, eo, cs, cp, cw),
            "k = 0": (out, eo, cs, cp[:, :0], cw[:, :0]),
            "k = 33": (out, eo, cs, cp[:, :1].repeat(1, 33), cw[:, :1].repeat(1, 33)),
            "splits too short": (out, eo, cs[:-1], cp, cw),
            "out overlaps expert_out": (eo[:T], eo, cs, cp, cw),
            "pos on the host": (out, eo, cs, pos, cw),
        }
        for why, args in bad.items():
            with pytest.raises(ValueError):
                cc.alltoallv_dev_combine_topk(*args, experts=E)
                pytest.fail(why)
        cc.pc.host_barrier()
        cc.alltoallv_dev_combine_topk(out, eo, cs, cp, cw, experts=E)
        cc.synchronize()
        assert torch.equal(_bytes(out), _bytes(_reference(y, pos, w, torch.float32)))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["symmetric", "plain"])
def test_device_errors(kind):
    """An out-of-range pos on one rank, an expert_out one row too small on one rank, and mixed
    symmetric / plain expert_out each raise on every rank at synchronize() with every out untouched
    and the context usable; a correct call right after works."""
    gcu = _cuda()
    P, E, k, align = 3, 2, 2, 4
    dtype = torch.bfloat16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        pools = _pools(cc, 1 << 18)
        me = ctx.rank
        per, needs = _setup(P, E, k, dtype, 23, align)
        y, splits, pos, w = per[me]
        want = _bytes(_reference(y, pos, w, dtype))
        small = 1
        untouched = _bytes(torch.full((pos.shape[0], H * 2), SENTINEL, dtype=torch.uint8))
        assert needs[small] > 0

        def attempt(**change):
            eo = change.get("eo")
            if eo is None:
                out, _, _ = _run_case(cc, me, per, needs, E, align, dtype, kind, pools)
                return out
            out = _fresh_out(pos.shape[0], dtype)
            cc.alltoallv_dev_combine_topk(out, eo, splits.cuda(), change.get("pos", pos).cuda(), w.cuda(), experts=E,
                                          align=align)
            return out

        # a pos entry past the dispatch input on rank 0 (rank 2 has no tokens)
        bad_pos = pos.clone()
        if me == 0:
            bad_pos[1, 0] = int(splits.sum())
        out, _, eo = _run_case(cc, me, per, needs, E, align, dtype, kind, pools)
        cc.synchronize()
        cc.pc.host_barrier()
        out = attempt(eo=eo, pos=bad_pos)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        assert torch.equal(_bytes(out), untouched)
        assert not cc.pc.poisoned()
        cc.pc.host_barrier()

        # one row too few on rank `small`
        out = attempt(eo=eo[:needs[me] - 1] if me == small else eo)
        with pytest.raises(ValueError, match=f"rank {small} needs {needs[small]} output rows but has room for "
                                             f"{needs[small] - 1}"):
            cc.synchronize()
        assert torch.equal(_bytes(out), untouched)
        cc.pc.host_barrier()

        # rank 0 passes the other kind of expert_out
        other = eo.clone() if kind == "symmetric" else pools["symmetric"][:eo.numel() * 2].view(dtype).view(eo.shape)
        if kind != "symmetric":
            other.copy_(eo)
        out = attempt(eo=other if me == 0 else eo)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        assert torch.equal(_bytes(out), untouched)
        cc.pc.host_barrier()

        out = attempt()
        cc.synchronize()
        assert torch.equal(_bytes(out), want)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


def test_route_cpu():
    """route() on CPU tensors: splits count the routed choices per (rank, expert), rows are the tokens
    in (rank, expert) order, stable by token, and pos inverts that order with -1 for the rest."""
    P, E, T, k = 3, 2, 9, 3
    G = P * E
    g = torch.Generator().manual_seed(3)
    x = torch.randn(T, 4, generator=g)
    idx = torch.randint(0, G, (T, k), generator=g)
    idx[0] = -1
    idx[2, 1] = G  # outside 0..G-1: not routed
    rows, splits, pos = _route(P, x, idx, E)
    assert rows.shape == (T * k, 4) and splits.dtype == torch.int64 and pos.shape == (T, k)
    flat = idx.reshape(-1)
    ok = (flat >= 0) & (flat < G)
    assert splits.tolist() == [int(((flat == e) & ok).sum()) for e in range(G)]
    expect = []
    for e in range(G):
        for i in range(T * k):
            if int(flat[i]) == e:
                expect.append(i)
    assert len(expect) == int(splits.sum())
    for r, i in enumerate(expect):
        assert int(pos.view(-1)[i]) == r and torch.equal(rows[r], x[i // k])
    assert int((pos < 0).sum()) == T * k - len(expect)
    assert bool((pos.view(-1)[~ok] == -1).all())


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "moe_topk_worker.py")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_combine_topk_all_gpus():
    """One rank per GPU: the weighted combine over NVLink equals the CPU reference, with symmetric
    and plain expert_out."""
    n = torch.cuda.device_count()
    size = 8 if n >= 8 else (4 if n >= 4 else 2)
    d = tempfile.mkdtemp(prefix="glb_topk_mp_")
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
