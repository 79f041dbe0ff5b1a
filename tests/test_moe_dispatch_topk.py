"""The top-k MoE dispatch: CudaContext.alltoallv_dev_topk and MoEDispatcher.dispatch_dev_topk. Ranks
are threads sharing cuda:0, each on its own stream. The reference is route() followed by
alltoallv_dev on the same inputs, which the fused kernel must match byte for byte."""
import os
import subprocess
import sys
import tempfile

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_combine_topk import _chunk_of, _expert, _pools, _reference, _route
from test_moe_dev import SENTINEL, _bytes, _layout, _ref_dispatch
from test_moe_fp8_dispatch import _dequant

# (dtype, elements per row): rows of 16, 48, 16 and 32 bytes
ROWS = [(torch.float32, 4), (torch.bfloat16, 24), (torch.float16, 8), (torch.uint8, 32)]
KINDS = ["symmetric", "registered", "plain"]
DEFAULT_ALLTOALLV_BLOCKS = 64  # Tuning::alltoallvBlocks


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _x(T, dtype, width, g):
    if dtype == torch.uint8:
        return torch.randint(0, 256, (T, width), generator=g, dtype=torch.uint8)
    return torch.randn(T, width, generator=g).to(dtype)


def _problem(P, E, k, dtype, width, seed, tmax=30):
    """Every rank's (x, topk_idx): -1 entries, entries below -1 and at or past P * E (not routed),
    an idle rank when P > 2."""
    g = torch.Generator().manual_seed(seed)
    G = P * E
    out = []
    for s in range(P):
        T = 0 if (P > 2 and s == 1) else int(torch.randint(1, tmax, (1,), generator=g))
        idx = torch.randint(0, G, (T, k), generator=g)
        r = torch.rand(T, k, generator=g)
        idx[r < 0.15] = -1
        idx[(r >= 0.15) & (r < 0.2)] = G + 3
        idx[(r >= 0.2) & (r < 0.22)] = -5
        out.append((_x(T, dtype, width, g), idx))
    return out


def _needs(per, P, E, align):
    sp = [_route(P, x, idx, E)[1].tolist() for x, idx in per]
    return [_layout(sp, P, E, align, d)[2] for d in range(P)]


def _out(kind, pools, half, cap, dtype, width):
    """A sentinel-filled out of `cap` rows: half `half` of a symmetric / registered pool, or plain."""
    es = torch.empty((), dtype=dtype).element_size()
    nbytes = cap * width * es
    if kind == "plain":
        t = torch.empty((cap, width), dtype=dtype, device="cuda")
    else:
        pool = pools[kind]
        n = pool.numel() // 2
        assert nbytes <= n
        t = pool[half * n:half * n + nbytes].view(dtype).view(cap, width)
    t.view(torch.uint8).fill_(SENTINEL)
    return t


def _index(cc, n):
    return torch.full((n,), -7, dtype=torch.int64, device="cuda")


def _fused(cc, out, x, idx, E, align, out_scales=None):
    P = cc.size
    splits, osp, ooff = _index(cc, P * E), _index(cc, P * E), _index(cc, P * E)
    pos = torch.full(tuple(idx.shape), -7, dtype=torch.int64, device="cuda")
    cc.alltoallv_dev_topk(out, x, idx, splits, pos, osp, ooff, experts=E, align=align, out_scales=out_scales)
    return splits, pos, osp, ooff


def _composed(cc, moe, out, x, idx, E, align, out_scales=None):
    rows, splits, pos = moe.route(x, idx, E)
    osp, ooff = _index(cc, cc.size * E), _index(cc, cc.size * E)
    cc.alltoallv_dev(out, rows, splits, osp, ooff, experts=E, align=align, out_scales=out_scales)
    return splits, pos, osp, ooff


def _check(cc, moe, per, E, align, kind, pools, tag):
    """Rank me's fused call against route() + alltoallv_dev on the same inputs, into the same kind."""
    me = cc.rank
    x, idx = per[me]
    dtype, width = x.dtype, x.shape[1]
    cap = max(_needs(per, cc.size, E, align)) + 5
    xc, ic = x.cuda(), idx.cuda()
    got, want = _out(kind, pools, 0, cap, dtype, width), _out(kind, pools, 1, cap, dtype, width)
    a = _fused(cc, got, xc, ic, E, align)
    b = _composed(cc, moe, want, xc, ic, E, align)
    cc.synchronize()
    assert torch.equal(_bytes(got), _bytes(want)), tag
    for name, u, v in zip(("splits", "pos", "out_splits", "out_offsets"), a, b):
        assert torch.equal(u.cpu(), v.cpu()), (name, tag)
    assert torch.equal(_bytes(xc), _bytes(x)), tag
    need = _needs(per, cc.size, E, align)[me]
    assert bool((_bytes(got[need:]) == SENTINEL).all()), tag  # the tail
    cc.pc.host_barrier()


def _layout_cases(slow):
    Es, As, Ks = (1, 3, 32), (1, 8), (1, 2, 8, 32)
    if slow:
        return [(E, A, k, r, kind) for E in Es for A in As for k in Ks for r in ROWS for kind in KINDS]
    return [(Es[c % 3], As[c % 2], Ks[c % 4], ROWS[c % 4], KINDS[c % 3]) for c in range(12)]


def _run_layouts(size, slow):
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        moe = MoEDispatcher(ctx, cc)
        pools = _pools(cc, 4 << 20)
        for c, (E, align, k, (dtype, width), kind) in enumerate(_layout_cases(slow)):
            per = _problem(P, E, k, dtype, width, 1000 * P + c)
            _check(cc, moe, per, E, align, kind, pools, (E, align, k, str(dtype), kind))
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=600000))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_dispatch_topk_layouts(size):
    """A spread of (E, align, k, row dtype, symmetric / registered / plain out) at this P: out, splits,
    pos, out_splits and out_offsets equal route() + alltoallv_dev byte for byte, x is unchanged and
    the tail of out keeps the sentinel."""
    _run_layouts(size, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_dispatch_topk_layouts_sweep(size):
    """The whole cross product E x align x k x row dtype x kind of out at this P."""
    _run_layouts(size, slow=True)


def _fixed(P, E, k, idx_of, T_of, seed, dtype=torch.float32, width=4):
    g = torch.Generator().manual_seed(seed)
    return [(_x(T_of(s), dtype, width, g), idx_of(s, T_of(s))) for s in range(P)]


@pytest.mark.gpu
def test_routing_edge_cases():
    """No tokens on a rank, every choice -1, entries below -1 and past P * E, the same expert twice in
    a row, every token on one expert, and many tokens whose groups straddle CTA slices at grids of
    1, 3 and 64 CTAs. Two calls give identical bytes."""
    gcu = _cuda()
    P, E, k = 3, 2, 4
    G = P * E

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=64 << 20)
        moe = MoEDispatcher(ctx, cc)
        pools = _pools(cc, 8 << 20)
        T = lambda s: 7 + 3 * s  # noqa: E731
        cases = {
            "T = 0 on rank 1, all -1 on rank 2": _fixed(
                P, E, k, lambda s, t: torch.full((t, k), -1, dtype=torch.int64) if s == 2
                else torch.arange(t * k).view(t, k) % G, lambda s: 0 if s == 1 else T(s), 1),
            "out of range": _fixed(
                P, E, k, lambda s, t: torch.tensor([-3, G, G + 100, -2**40, 2**40, 0, G - 1, -1] * t)[:t * k].view(t, k),
                T, 2),
            "same expert twice": _fixed(
                P, E, k, lambda s, t: (torch.arange(t * k).view(t, k) // 2 + s) % G, T, 3),
            "all on one expert": _fixed(P, E, k, lambda s, t: torch.full((t, k), 4, dtype=torch.int64), T, 4),
        }
        for why, per in cases.items():
            for kind in KINDS:
                _check(cc, moe, per, E, 8, kind, pools, (why, kind))

        # Thousands of tokens: every group straddles CTA slices.
        big = _problem(P, E, 8, torch.bfloat16, 8, 77, tmax=6000)
        for n in (1, 3, 64):
            cc.pc.host_barrier()
            if ctx.rank == 0:
                gb._C.cuda.set_tuning({"alltoallv_blocks": n})
            cc.pc.host_barrier()
            try:
                for kind in ("symmetric", "plain"):
                    _check(cc, moe, big, E, 4, kind, pools, (n, kind))
            finally:
                cc.pc.host_barrier()
                if ctx.rank == 0:
                    gb._C.cuda.set_tuning({"alltoallv_blocks": DEFAULT_ALLTOALLV_BLOCKS})
                cc.pc.host_barrier()

        # Determinism: two calls, identical bytes.
        x, idx = (t.cuda() for t in big[ctx.rank])
        cap = max(_needs(big, P, E, 4)) + 1
        outs = [_out("symmetric", pools, h, cap, x.dtype, x.shape[1]) for h in (0, 1)]
        res = [_fused(cc, o, x, idx, E, 4) for o in outs]
        cc.synchronize()
        assert torch.equal(_bytes(outs[0]), _bytes(outs[1]))
        for u, v in zip(*res):
            assert torch.equal(u, v)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (2, False), (4, True), (4, False)])
def test_fp8_dispatch_topk(size, symmetric):
    """The quantising form: codes, scales, splits, pos and the layout equal route() + the FP8
    alltoallv_dev byte for byte, and the received rows dequantise to x within e4m3 rounding."""
    gcu = _cuda()
    P, E, k, align, Hd = size, 3, 4, 4, 384

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        per = _problem(P, E, k, torch.bfloat16, Hd, 300 + P)
        for x, _ in per:
            if x.shape[0] > 2:
                x[1] *= 1e-6  # a block whose amax is below the 1e-4 floor
                x[2, :128] = 0
        me = ctx.rank
        x, idx = per[me]
        cap = max(_needs(per, P, E, align)) + 3

        def outs():
            if symmetric:
                o, s = cc.empty((cap, Hd), torch.float8_e4m3fn), cc.empty((cap, Hd // 128), torch.float32)
            else:
                o = torch.empty((cap, Hd), dtype=torch.float8_e4m3fn, device="cuda")
                s = torch.empty((cap, Hd // 128), dtype=torch.float32, device="cuda")
            o.view(torch.uint8).fill_(SENTINEL)
            s.view(torch.uint8).fill_(SENTINEL)
            return o, s

        (go, gs), (wo, ws) = outs(), outs()
        xc, ic = x.cuda(), idx.cuda()
        a = _fused(cc, go, xc, ic, E, align, out_scales=gs)
        b = _composed(cc, moe, wo, xc, ic, E, align, out_scales=ws)
        cc.synchronize()
        assert torch.equal(_bytes(go), _bytes(wo)) and torch.equal(_bytes(gs), _bytes(ws))
        for u, v in zip(a, b):
            assert torch.equal(u.cpu(), v.cpu())
        # Dequantised segment rows against the bf16 rows route() would have sent.
        routed = [_route(P, x_, i_, E) for x_, i_ in per]
        sp = [r[1].tolist() for r in routed]
        ref, osp, ooff = _ref_dispatch([r[0] for r in routed], sp, P, E, align, me, cap)
        ref = ref.view(torch.bfloat16).view(cap, Hd)
        rows = torch.cat([torch.arange(o, o + n) for o, n in zip(ooff, osp)]).long()
        deq, want = _dequant(go.cpu(), gs.cpu())[rows].float(), ref[rows].float()
        scale = gs.cpu()[rows].repeat_interleave(128, dim=1)
        # e4m3 keeps 3 mantissa bits (half an ulp: 2^-4 relative, 2^-10 of the scale at the bottom of
        # its subnormals); _dequant rounds once more to bf16.
        assert bool(((deq - want).abs() <= want.abs() * (2**-4 + 2**-8) + scale * 2**-9).all())
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size,kind", [(2, "symmetric"), (3, "plain"), (4, "registered")])
def test_layer_round_trip(size, kind):
    """dispatch_dev_topk -> a per-expert transform -> combine_dev_topk equals the documented combine
    reference bit for bit."""
    gcu = _cuda()
    P, E, k, align, W = size, 2, 3, 8, 24

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        moe = MoEDispatcher(ctx, cc)
        pools = _pools(cc, 1 << 20)
        me = ctx.rank
        per = _problem(P, E, k, torch.bfloat16, W, 50 + P)
        g = torch.Generator().manual_seed(9 + me)
        x, idx = per[me]
        w = torch.rand(idx.shape, generator=g) * 2 - 0.5
        cap = max(_needs(per, P, E, align)) + 2
        got = _out(kind, pools, 0, cap, torch.bfloat16, W)
        expert_out = _out(kind, pools, 1, cap, torch.bfloat16, W)
        _, osp, ooff, splits, pos = moe.dispatch_dev_topk(x.cuda(), idx.cuda(), got, experts=E, align=align)
        osp_h, ooff_h = osp.tolist(), ooff.tolist()
        for e in range(E):
            lo, hi = ooff_h[e * P], ooff_h[e * P + P - 1] + osp_h[e * P + P - 1]
            c = float(me * E + e)
            expert_out[lo:hi] = (got[lo:hi].float() * (1 + 0.125 * c) - 0.5 * c).to(torch.bfloat16)
        y = torch.empty((x.shape[0], W), dtype=torch.bfloat16, device="cuda")
        moe.combine_dev_topk(expert_out, splits, pos, w.cuda(), y, experts=E, align=align)
        cc.synchronize()
        rows, rs, rp = _route(P, x, idx, E)
        n = int(rs.sum())
        want = _reference(_expert(rows[:n], _chunk_of(rs, n), torch.bfloat16), rp, w, torch.bfloat16)
        assert torch.equal(_bytes(y), _bytes(want))
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (4, False)])
def test_graph_capture_replays(size, symmetric):
    """dispatch_dev_topk, the experts and combine_dev_topk captured once per rank; three replays with
    new tokens, routing and weights written into the captured tensors are all correct."""
    gcu = _cuda()
    P, E, T, k, align, W = size, 2, 16, 2, 4, 8
    G = P * E

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        cap = P * (T * k + E * align)
        got = cc.empty((cap, W), torch.float32) if symmetric else torch.empty((cap, W), device="cuda")
        expert_out = cc.empty((cap, W), torch.float32) if symmetric else torch.empty((cap, W), device="cuda")
        x = torch.zeros((T, W), device="cuda")
        idx = torch.zeros((T, k), dtype=torch.int64, device="cuda")
        w = torch.zeros((T, k), device="cuda")
        y = torch.empty((T, W), device="cuda")

        def load(seed):
            g = torch.Generator().manual_seed(seed * 10 + me)
            i = torch.randint(0, G, (T, k), generator=g)
            i[torch.rand(T, k, generator=g) < 0.2] = -1
            x.copy_(torch.randn(T, W, generator=g))
            idx.copy_(i)
            w.copy_(torch.rand(T, k, generator=g))

        def step():
            _, _, _, splits, pos = moe.dispatch_dev_topk(x, idx, got, experts=E, align=align)
            torch.mul(got, 0.75, out=expert_out)
            moe.combine_dev_topk(expert_out, splits, pos, w, y, experts=E, align=align)

        stream = torch.cuda.current_stream()
        load(1)
        step()
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
    """dispatch_dev_topk (both forms) runs under torch's sync debug mode "error"."""
    gcu = _cuda()
    P, E, k, Hd = 2, 2, 2, 256

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        per = _problem(P, E, k, torch.bfloat16, Hd, 42)
        x, idx = (t.cuda() for t in per[ctx.rank])
        cap = 128
        if symmetric:
            got, codes, scales = (cc.empty((cap, Hd), torch.bfloat16), cc.empty((cap, Hd), torch.float8_e4m3fn),
                                  cc.empty((cap, Hd // 128), torch.float32))
        else:
            got = torch.empty((cap, Hd), dtype=torch.bfloat16, device="cuda")
            codes = torch.empty((cap, Hd), dtype=torch.float8_e4m3fn, device="cuda")
            scales = torch.empty((cap, Hd // 128), dtype=torch.float32, device="cuda")
        torch.cuda.current_stream().synchronize()
        cc.pc.host_barrier()
        if ctx.rank == 0:
            torch.cuda.set_sync_debug_mode("error")
        cc.pc.host_barrier()
        try:
            moe.dispatch_dev_topk(x, idx, got, experts=E, align=4)
            moe.dispatch_dev_topk(x, idx, codes, experts=E, align=4, out_scales=scales)
        finally:
            cc.pc.host_barrier()
            if ctx.rank == 0:
                torch.cuda.set_sync_debug_mode("default")
            cc.pc.host_barrier()
        cc.synchronize()
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_empty_plain_out(fp8):
    """Every rank passes a plain out and rank 1's has no rows (a null data pointer), as no token
    chooses one of its experts; rank 1 still sends its own tokens. The call is valid and rank 0
    receives route()'s rows. The copying form then combines from those outputs, rank 1's
    expert_out still empty, and each rank gets the reference sum."""
    from test_moe_fp8_dispatch import _ref as _fp8_ref

    gcu = _cuda()
    P, E, k, T, W, H = 2, 2, 2, 9, 4, 256

    def problem(s):
        g = torch.Generator().manual_seed(60 + s)
        idx = torch.randint(0, E, (T, k), generator=g)  # experts of rank 0 only
        idx[0, 1] = -1
        x = torch.randn(T, H, generator=g).to(torch.bfloat16) if fp8 else torch.randn(T, W, generator=g)
        w = torch.rand(T, k, generator=g)
        return x, idx, w

    probs = [problem(s) for s in range(P)]
    routed = [_route(P, x, idx, E) for x, idx, _ in probs]
    sp = [[int(c) for c in splits] for _, splits, _ in routed]
    cap0 = _layout(sp, P, E, 1, 0)[2] + 3

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        cap = cap0 if me == 0 else 0
        x, idx, w = (t.cuda() for t in probs[me])
        out = torch.empty((cap, H if fp8 else W), dtype=torch.float8_e4m3fn if fp8 else torch.float32, device="cuda")
        out.view(torch.uint8).fill_(SENTINEL)
        scales = None
        if fp8:
            scales = torch.empty((cap, H // 128), dtype=torch.float32, device="cuda")
            scales.view(torch.uint8).fill_(SENTINEL)
        splits = torch.empty(P * E, dtype=torch.int64, device="cuda")
        pos = torch.empty((T, k), dtype=torch.int64, device="cuda")
        osp, ooff = torch.empty_like(splits), torch.empty_like(splits)
        cc.alltoallv_dev_topk(out, x, idx, splits, pos, osp, ooff, experts=E, out_scales=scales)
        cc.synchronize()
        assert splits.tolist() == sp[me] and torch.equal(pos.cpu(), routed[me][2])
        rows = [r for r, _, _ in routed]
        if me == 0 and fp8:
            want_codes, want_scales, _, _ = _fp8_ref(rows, sp, P, E, 1, 0, cap)
            assert torch.equal(_bytes(out), want_codes) and torch.equal(_bytes(scales), want_scales)
        elif me == 0:
            assert torch.equal(_bytes(out), _ref_dispatch(rows, sp, P, E, 1, 0, cap)[0])
        if not fp8:
            res = torch.empty((T, W), device="cuda")
            cc.alltoallv_dev_combine_topk(res, out, splits, pos, w, experts=E)
            cc.synchronize()
            assert torch.equal(res.cpu(), _reference(rows[me], routed[me][2], probs[me][2], torch.float32))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
def test_host_errors():
    """Every malformed call raises ValueError before launch, alike on every rank; a correct call
    afterwards works, so none of them launched."""
    gcu = _cuda()
    P, E, k, W = 2, 2, 2, 8

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        per = _fixed(P, E, k, lambda s, t: torch.arange(t * k).view(t, k) % (P * E), lambda s: 6, 5, width=W)
        x, idx = (t.cuda() for t in per[ctx.rank])
        T = x.shape[0]
        out = cc.empty((64, W), torch.float32)
        sp, osp, ooff = _index(cc, P * E), _index(cc, P * E), _index(cc, P * E)
        pos = torch.empty((T, k), dtype=torch.int64, device="cuda")
        odd = torch.empty(T * W + 4, device="cuda")[1:T * W + 1].view(T, W)
        xb = x.bfloat16()
        codes = cc.empty((64, 256), torch.float8_e4m3fn)
        scales = cc.empty((64, 2), torch.float32)
        xq = torch.zeros((T, 256), dtype=torch.bfloat16, device="cuda")
        bad = {
            "int32 topk_idx": dict(topk_idx=idx.int()),
            "topk_idx 1-D": dict(topk_idx=idx.view(-1)),
            "topk_idx rows != T": dict(topk_idx=idx[:-1].contiguous()),
            "non-contiguous topk_idx": dict(topk_idx=torch.stack([idx, idx], 2)[..., 0]),
            "topk_idx on the host": dict(topk_idx=idx.cpu()),
            "k = 0": dict(topk_idx=idx[:, :0].contiguous(), pos=pos[:, :0].contiguous()),
            "k = 33": dict(topk_idx=idx[:, :1].repeat(1, 33), pos=pos[:, :1].repeat(1, 33)),
            "pos int32": dict(pos=pos.int()),
            "pos shape": dict(pos=pos[:, :1].contiguous()),
            "splits too short": dict(splits=sp[:-1]),
            "splits float": dict(splits=sp.double()),
            "out_offsets on the host": dict(out_offsets=ooff.cpu()),
            "out dtype differs": dict(out=out.double()),
            "out row width": dict(out=cc.empty((64, W * 2), torch.float32)),
            "rows not a multiple of 16 bytes": dict(x=x[:, :3].contiguous(), out=out[:, :3].contiguous()),
            "non-contiguous x": dict(x=torch.empty((T, W * 2), device="cuda")[:, :W]),
            "x not 16-byte aligned": dict(x=odd),
            "out overlaps x": dict(x=out[:T]),
            "experts = 0": dict(experts=0),
            "experts = 33": dict(experts=33),
            "align = 0": dict(align=0),
            "fp8 without out_scales": dict(x=xq, out=codes),
            "fp8 from float32": dict(x=xq.float(), out=codes, out_scales=scales),
            "fp8 scales shape": dict(x=xq, out=codes, out_scales=cc.empty((64, 3), torch.float32)),
            "fp8 row not a multiple of 128": dict(x=xq[:, :192].contiguous(), out=codes[:, :192].contiguous(),
                                                  out_scales=scales[:, :1].contiguous()),
            "fp8 symmetric out, plain scales": dict(x=xq, out=codes, out_scales=torch.empty((64, 2), device="cuda")),
            "bf16 input for a float32 out": dict(x=xb),
        }
        args = dict(out=out, x=x, topk_idx=idx, splits=sp, pos=pos, out_splits=osp, out_offsets=ooff, experts=E,
                    align=1)
        for why, change in bad.items():
            with pytest.raises(ValueError):
                cc.alltoallv_dev_topk(**{**args, **change})
                pytest.fail(why)
        # T * k = 2^31, checked from the shapes before anything is read: broadcast views stand in
        # for 16 GB of indices.
        T2 = 2**26
        huge = dict(x=x[:1].expand(T2, W), topk_idx=idx[:1, :1].expand(T2, 32), pos=pos[:1, :1].expand(T2, 32))
        with pytest.raises(ValueError, match="2\\^31"):
            cc.alltoallv_dev_topk(**{**args, **huge})
        cc.pc.host_barrier()
        got, want = cc.empty((64, W), torch.float32), cc.empty((64, W), torch.float32)
        got.zero_()
        want.zero_()
        a = _fused(cc, got, x, idx, E, 1)
        b = _composed(cc, moe, want, x, idx, E, 1)
        cc.synchronize()
        assert torch.equal(_bytes(got), _bytes(want)) and all(torch.equal(u, v) for u, v in zip(a, b))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["symmetric", "plain"])
def test_device_errors(kind):
    """One row too few on one rank: every rank raises at synchronize(), the overflowing rank receives
    nothing and the others are served. A rank calling alltoallv_dev against alltoallv_dev_topk, and
    ranks disagreeing on align, each raise "invalid" on every rank. splits and pos are written in
    every case, and a correct call right after works."""
    gcu = _cuda()
    P, E, k, align = 3, 2, 3, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        pools = _pools(cc, 1 << 20)
        me = ctx.rank
        per = _problem(P, E, k, torch.float32, 8, 31, tmax=20)
        x, idx = (t.cuda() for t in per[me])
        needs = _needs(per, P, E, align)
        small = 2
        assert needs[small] > 0
        cap = max(needs) + 2
        want = _out(kind, pools, 1, cap, torch.float32, 8)
        ref = _composed(cc, moe, want, x, idx, E, align)
        cc.synchronize()
        cc.pc.host_barrier()

        def check_meta(res):
            assert torch.equal(res[0], ref[0]) and torch.equal(res[1], ref[1])

        # overflow on rank `small`
        got = _out(kind, pools, 0, cap, torch.float32, 8)
        res = _fused(cc, got[:needs[me] - 1] if me == small else got, x, idx, E, align)
        with pytest.raises(ValueError, match=f"rank {small} needs {needs[small]} output rows but has room for "
                                             f"{needs[small] - 1}"):
            cc.synchronize()
        check_meta(res)
        if me == small:
            assert bool((_bytes(got) == SENTINEL).all())
        else:
            assert torch.equal(_bytes(got), _bytes(want))
        assert not cc.pc.poisoned()
        cc.pc.host_barrier()

        # rank 0 runs the plain dispatch, the others the top-k form
        got = _out(kind, pools, 0, cap, torch.float32, 8)
        if me == 0:
            _composed(cc, moe, got, x, idx, E, align)
        else:
            res = _fused(cc, got, x, idx, E, align)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        if me != 0:
            check_meta(res)
        assert bool((_bytes(got) == SENTINEL).all())
        cc.pc.host_barrier()

        # rank 1 passes another align
        got = _out(kind, pools, 0, cap, torch.float32, 8)
        res = _fused(cc, got, x, idx, E, 1 if me == 1 else align)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        check_meta(res)
        assert bool((_bytes(got) == SENTINEL).all())
        cc.pc.host_barrier()

        got = _out(kind, pools, 0, cap, torch.float32, 8)
        res = _fused(cc, got, x, idx, E, align)
        cc.synchronize()
        assert torch.equal(_bytes(got), _bytes(want))
        check_meta(res)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


WORKER = os.path.join(os.path.dirname(os.path.abspath(__file__)), "moe_dispatch_topk_worker.py")


@pytest.mark.gpu
@pytest.mark.multigpu
@pytest.mark.skipif(not torch.cuda.is_available() or torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_dispatch_topk_all_gpus():
    """One rank per GPU: the top-k dispatch over NVLink equals route() + alltoallv_dev, bf16 and FP8,
    with symmetric and plain outputs."""
    n = torch.cuda.device_count()
    size = 8 if n >= 8 else (4 if n >= 4 else 2)
    d = tempfile.mkdtemp(prefix="glb_dispatch_topk_mp_")
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
