"""Device-split all-to-all-v (CudaContext.alltoallv_dev / alltoallv_dev_combine) and the
MoEDispatcher paths built on it. Ranks are threads sharing cuda:0, each on its own stream."""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher

SENTINEL = 0xA5
# (dtype, row width): byte sizes 16, 12, 6 (the byte path), 16, 5 and 16
KINDS = [(torch.float32, 4), (torch.float32, 3), (torch.bfloat16, 3), (torch.float8_e4m3fn, 16),
         (torch.float8_e4m3fn, 5), (torch.int64, 2)]


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _bytes(t):
    return t.contiguous().view(-1).view(torch.uint8).cpu()


def _splits(P, E, seed):
    """Every rank's in_splits (P lists of P*E row counts), seeded; zeros included and the last rank
    of a multi-rank job sends nothing."""
    g = torch.Generator().manual_seed(seed)
    sp = []
    for s in range(P):
        row = torch.randint(0, 6, (P * E,), generator=g)
        row[torch.rand(P * E, generator=g) < 0.25] = 0
        if P > 1 and s == P - 1:
            row.zero_()
        sp.append([int(x) for x in row])
    return sp


def _rows(dtype, width, n, seed):
    g = torch.Generator().manual_seed(seed)
    raw = torch.randint(0, 256, (n * width * torch.empty((), dtype=dtype).element_size(),), dtype=torch.uint8,
                        generator=g)
    return raw.view(dtype).view(n, width)


def _layout(sp, P, E, align, d):
    """Forward layout on rank d: (out_splits, out_offsets) indexed e*P+s, and rows needed."""
    osp, ooff = [0] * (P * E), [0] * (P * E)
    base = 0
    for e in range(E):
        off = base
        for s in range(P):
            osp[e * P + s] = sp[s][d * E + e]
            ooff[e * P + s] = off
            off += sp[s][d * E + e]
        base = off if e == E - 1 else -(-off // align) * align
    return osp, ooff, base


def _ref_dispatch(inputs, sp, P, E, align, d, cap):
    """Pure-torch CPU reference of rank d's output bytes (sentinel outside the segments)."""
    osp, ooff, _ = _layout(sp, P, E, align, d)
    width = inputs[0].shape[1]
    out = torch.full((cap * width * inputs[0].element_size(),), SENTINEL, dtype=torch.uint8)
    out = out.view(inputs[0].dtype).view(cap, width)
    for e in range(E):
        for s in range(P):
            k = d * E + e
            src = sum(sp[s][:k])
            n = sp[s][k]
            out[ooff[e * P + s]:ooff[e * P + s] + n] = inputs[s][src:src + n]
    return _bytes(out), osp, ooff


def _alloc(cc, sym_bytes, rows, width, dtype, symmetric):
    es = torch.empty((), dtype=dtype).element_size()
    if symmetric:
        t = sym_bytes[: rows * width * es].view(dtype).view(rows, width)
    else:
        t = torch.empty((rows, width), dtype=dtype, device="cuda")
    t.view(-1).view(torch.uint8).fill_(SENTINEL)
    return t


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_dispatch_combine_layouts(size):
    """Every (dtype, row width, E, align, symmetric / plain out) at this P: out, out_splits and
    out_offsets equal the CPU reference bit for bit, rows outside the segments keep the sentinel,
    combine(dispatch(x)) == x, and with E = 1, align = 1 the result equals cc.alltoallv."""
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        sym = cc.empty(1 << 20, torch.uint8)
        sym2 = cc.empty(1 << 20, torch.uint8)
        me = ctx.rank
        case = 0
        for dtype, width in KINDS:
            for E in (1, 2, 4):
                for align in (1, 8):
                    for symmetric in (True, False):
                        case += 1
                        seed = 1000 * case + 7 * P
                        sp = _splits(P, E, seed)
                        inputs = [_rows(dtype, width, sum(sp[s]), seed + 1 + s) for s in range(P)]
                        cap = max(_layout(sp, P, E, align, d)[2] for d in range(P)) + 3
                        want, wsp, woff = _ref_dispatch(inputs, sp, P, E, align, me, cap)
                        inp = inputs[me].cuda()
                        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
                        out = _alloc(cc, sym, cap, width, dtype, symmetric)
                        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
                        ooff = torch.empty_like(osp)
                        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align)
                        back = _alloc(cc, sym2, inp.shape[0] + 2, width, dtype, symmetric)
                        cc.alltoallv_dev_combine(back, out, osp, ooff, experts=E)
                        cc.synchronize()
                        tag = (str(dtype), width, E, align, symmetric)
                        assert torch.equal(_bytes(out), want), tag
                        assert osp.tolist() == wsp and ooff.tolist() == woff, tag
                        got = _bytes(back)
                        nb = _bytes(inp).numel()
                        assert torch.equal(got[:nb], _bytes(inp)), tag
                        assert bool((got[nb:] == SENTINEL).all()), tag
                        if E == 1 and align == 1:
                            recv = [sp[s][me] * width for s in range(P)]
                            ref = torch.empty_like(out)
                            ref.view(-1).view(torch.uint8).fill_(SENTINEL)
                            cc.alltoallv(ref, recv, inp, [c * width for c in sp[me]])
                            cc.synchronize()
                            assert torch.equal(_bytes(ref), _bytes(out)), tag
                        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=120000))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [False, True])
def test_back_to_back_imbalanced(symmetric):
    """Dispatch and combine issued back to back, several rounds, no synchronisation in between,
    with routing so uneven that rank 0 receives megabytes while the other ranks receive a few rows.
    The light ranks finish each call long before rank 0 has copied its rows out of staging and start
    the next one at once (which publishes new counts into rank 0's pad): every output must still
    match the reference, alignment gaps and all."""
    gcu = _cuda()
    P, E, width, align, rounds = 4, 4, 16, 8, 4

    def splits_for(seed):
        g = torch.Generator().manual_seed(seed)
        sp = []
        for s in range(P):
            row = torch.randint(0, 4, (P * E,), generator=g)
            row[:E] = torch.randint(1500, 2500, (E,), generator=g)  # everything heavy goes to rank 0
            sp.append([int(x) for x in row])
        return sp

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        me = ctx.rank
        cases = []
        for r in range(rounds):
            sp = splits_for(900 + r)
            inputs = [_rows(torch.float32, width, sum(sp[s]), 910 + 10 * r + s) for s in range(P)]
            cap = _layout(sp, P, E, align, me)[2] + 5
            cases.append((sp, inputs, cap))
        big = max(c[2] for c in cases)
        sym = cc.empty(big * width * 4, torch.uint8) if symmetric else None
        sym_back = cc.empty(max(c[1][me].shape[0] for c in cases) * width * 4 + 64, torch.uint8) if symmetric else None
        outs, backs, metas, inps = [], [], [], []
        cc.synchronize()
        cc.pc.host_barrier()
        for r, (sp, inputs, cap) in enumerate(cases):
            if symmetric and r > 0:
                break  # one symmetric buffer: one round (its pushes are zero copy, nothing is staged)
            inp = inputs[me].cuda()
            splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
            out = _alloc(cc, sym, cap, width, torch.float32, symmetric)
            back = _alloc(cc, sym_back, inp.shape[0] + 1, width, torch.float32, symmetric)
            osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
            ooff = torch.empty_like(osp)
            cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align)
            cc.alltoallv_dev_combine(back, out, osp, ooff, experts=E)
            outs.append(out), backs.append(back), metas.append((osp, ooff)), inps.append(inp)
        cc.synchronize()
        for r, (out, back, (osp, ooff), inp) in enumerate(zip(outs, backs, metas, inps)):
            sp, inputs, cap = cases[r]
            want, wsp, woff = _ref_dispatch(inputs, sp, P, E, align, me, cap)
            assert torch.equal(_bytes(out), want), r
            assert osp.tolist() == wsp and ooff.tolist() == woff, r
            got, nb = _bytes(back), _bytes(inp).numel()
            assert torch.equal(got[:nb], _bytes(inp)), r
            assert bool((got[nb:] == SENTINEL).all()), r
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_no_host_sync(symmetric):
    """dispatch_dev + combine_dev run under torch's sync debug mode "error"."""
    gcu = _cuda()
    P, E = 2, 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        sym = cc.empty(1 << 16, torch.uint8)
        sp = _splits(P, E, 5)
        inputs = [_rows(torch.bfloat16, 8, sum(sp[s]), 50 + s) for s in range(P)]
        inp = inputs[ctx.rank].cuda()
        splits = torch.tensor(sp[ctx.rank], dtype=torch.int64, device="cuda")
        out = _alloc(cc, sym, 64, 8, torch.bfloat16, symmetric)
        back = torch.empty_like(inp)
        torch.cuda.current_stream().synchronize()
        cc.pc.host_barrier()
        if ctx.rank == 0:
            torch.cuda.set_sync_debug_mode("error")
        cc.pc.host_barrier()
        try:
            _, osp, ooff = moe.dispatch_dev(inp, splits, out, experts=E, align=4)
            moe.combine_dev(out, osp, ooff, back, experts=E)
        finally:
            cc.pc.host_barrier()
            if ctx.rank == 0:
                torch.cuda.set_sync_debug_mode("default")
            cc.pc.host_barrier()
        cc.synchronize()
        assert torch.equal(_bytes(back), _bytes(inp))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_graph_capture_replays(size):
    """dispatch + combine captured once per rank; between three replays both the splits and the
    input data change, and every replay gives the right result."""
    gcu = _cuda()
    P, E, width, align = size, 2, 8, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        max_rows = 5 * P * E  # _splits draws 0..5 rows per entry
        cap = P * (max_rows + E * align)
        out = cc.empty((cap, width), torch.float32)
        inp = torch.zeros((max_rows, width), dtype=torch.float32, device="cuda")
        back = torch.empty_like(inp)
        splits = torch.zeros(P * E, dtype=torch.int64, device="cuda")

        def load(seed):
            sp = _splits(P, E, seed)
            inputs = [_rows(torch.float32, width, max_rows, seed + 1 + s) for s in range(P)]
            splits.copy_(torch.tensor(sp[me], dtype=torch.int64))
            inp.copy_(inputs[me])
            out.view(-1).view(torch.uint8).fill_(SENTINEL)
            return sp, inputs

        def check(sp, inputs, osp, ooff):
            used = [sum(sp[s]) for s in range(P)]
            trimmed = [x[:n] for x, n in zip(inputs, used)]
            want, wsp, woff = _ref_dispatch(trimmed, sp, P, E, align, me, cap)
            assert torch.equal(_bytes(out), want)
            assert osp.tolist() == wsp and ooff.tolist() == woff
            assert torch.equal(_bytes(back[:used[me]]), _bytes(inputs[me][:used[me]]))

        stream = torch.cuda.current_stream()
        load(11)
        moe.dispatch_dev(inp, splits, out, experts=E, align=align)  # warm-up outside the graph
        cc.synchronize()
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            _, osp, ooff = moe.dispatch_dev(inp, splits, out, experts=E, align=align)
            moe.combine_dev(out, osp, ooff, back, experts=E)
        cc.pc.host_barrier()
        for seed in (21, 31, 41):
            sp, inputs = load(seed)
            stream.synchronize()
            cc.pc.host_barrier()
            g.replay()
            cc.synchronize()
            check(sp, inputs, osp, ooff)
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_overflow_and_invalid_input(symmetric):
    """An out one row too small: that rank's out keeps every byte and the next host call raises
    ValueError (with both row counts) on every rank; a correct call right after works. A negative
    split: every rank raises and the context stays usable. Both are data checks in the kernel."""
    gcu = _cuda()
    P, E, width, align = 3, 2, 4, 1

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        sym = cc.empty(1 << 16, torch.uint8)
        sp = [[2, 1, 3, 0, 1, 2], [1, 1, 1, 1, 1, 1], [0, 2, 2, 0, 3, 1]]
        inputs = [_rows(torch.float32, width, sum(sp[s]), 70 + s) for s in range(P)]
        needs = [_layout(sp, P, E, align, d)[2] for d in range(P)]
        small = 1  # rank 1 gets one row less than it needs
        cap = needs[me] - 1 if me == small else needs[me] + 2
        inp = inputs[me].cuda()
        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)

        out = _alloc(cc, sym, cap, width, torch.float32, symmetric)
        before = _bytes(out)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align)
        with pytest.raises(ValueError, match=f"rank {small} needs {needs[small]} output rows but has room for "
                                             f"{needs[small] - 1}"):
            cc.synchronize()
        if me == small:
            assert torch.equal(_bytes(out), before)
            assert osp.tolist() == _layout(sp, P, E, align, me)[0]  # true values even so
        else:
            assert torch.equal(_bytes(out), _ref_dispatch(inputs, sp, P, E, align, me, cap)[0])
        cc.check_health()  # raised once, cleared
        cc.pc.host_barrier()

        out = _alloc(cc, sym, needs[me] + 2, width, torch.float32, symmetric)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align)
        cc.synchronize()
        assert torch.equal(_bytes(out), _ref_dispatch(inputs, sp, P, E, align, me, needs[me] + 2)[0])
        cc.pc.host_barrier()

        bad = torch.tensor([-1 if (me == 0 and k == 2) else v for k, v in enumerate(sp[me])], dtype=torch.int64,
                           device="cuda")
        out = _alloc(cc, sym, needs[me] + 2, width, torch.float32, symmetric)
        before = _bytes(out)
        cc.alltoallv_dev(out, inp, bad, osp, ooff, experts=E, align=align)
        with pytest.raises(ValueError, match="invalid splits"):
            cc.synchronize()
        assert torch.equal(_bytes(out), before)
        assert not cc.pc.poisoned()
        cc.pc.host_barrier()

        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align)
        cc.synchronize()
        assert torch.equal(_bytes(out), _ref_dispatch(inputs, sp, P, E, align, me, needs[me] + 2)[0])
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_mixed_registered_and_plain_out(fp8):
    """Rank 0 passes a plain out (and out_scales) while its peer passes symmetric ones: the ranks
    would push into different places, so the call is invalid input on every rank, nothing moves,
    and a correct call on the same context right after works."""
    from test_moe_fp8_dispatch import _ref as _fp8_ref, _rows as _bf16_rows

    gcu = _cuda()
    P, E, align, H = 2, 2, 4, 256
    sp = [[2, 1, 3, 0], [1, 0, 2, 2]]
    caps = [_layout(sp, P, E, align, d)[2] + 3 for d in range(P)]

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        cap = caps[me]
        sym = cc.empty(1 << 16, torch.uint8)
        sym_scales = cc.empty(1 << 14, torch.uint8)
        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        if fp8:
            inputs = [_bf16_rows(sum(sp[s]), H, 40 + s) for s in range(P)]
            want_codes, want_scales, _, _ = _fp8_ref(inputs, sp, P, E, align, me, cap)
        else:
            inputs = [_rows(torch.float32, 4, sum(sp[s]), 40 + s) for s in range(P)]
            want_codes = _ref_dispatch(inputs, sp, P, E, align, me, cap)[0]
        inp = inputs[me].cuda()

        def outputs(symmetric):
            if not fp8:
                return _alloc(cc, sym, cap, 4, torch.float32, symmetric), None
            out = _alloc(cc, sym, cap, H, torch.float8_e4m3fn, symmetric)
            scales = _alloc(cc, sym_scales, cap, H // 128, torch.float32, symmetric)
            return out, scales

        out, scales = outputs(symmetric=me != 0)
        before = [_bytes(t) for t in (out, scales) if t is not None]
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
        with pytest.raises(ValueError, match="invalid"):
            cc.synchronize()
        assert all(torch.equal(b, _bytes(t)) for b, t in zip(before, (out, scales)))
        cc.pc.host_barrier()

        out, scales = outputs(symmetric=True)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
        cc.synchronize()
        assert torch.equal(_bytes(out), want_codes)
        if fp8:
            assert torch.equal(_bytes(scales), want_scales)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fp8", [False, True])
def test_empty_plain_out(fp8):
    """Both ranks pass plain outputs and rank 1's has no rows (a null data pointer): nobody sends
    it anything, while it still sends its own rows to rank 0. The call is valid and rank 0 gets
    every row, with its scales in the quantising form."""
    from test_moe_fp8_dispatch import _ref as _fp8_ref, _rows as _bf16_rows

    gcu = _cuda()
    P, E, H = 2, 2, 256
    sp = [[2, 3, 0, 0], [1, 2, 0, 0]]
    cap0 = _layout(sp, P, E, 1, 0)[2] + 3

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        cap = cap0 if me == 0 else 0
        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        scales = None
        if fp8:
            inputs = [_bf16_rows(sum(sp[s]), H, 80 + s) for s in range(P)]
            out = _alloc(cc, None, cap, H, torch.float8_e4m3fn, False)
            scales = _alloc(cc, None, cap, H // 128, torch.float32, False)
        else:
            inputs = [_rows(torch.float32, 4, sum(sp[s]), 80 + s) for s in range(P)]
            out = _alloc(cc, None, cap, 4, torch.float32, False)
        cc.alltoallv_dev(out, inputs[me].cuda(), splits, osp, ooff, experts=E, out_scales=scales)
        cc.synchronize()
        assert osp.tolist() == _layout(sp, P, E, 1, me)[0]
        if me == 0 and fp8:
            want_codes, want_scales, _, _ = _fp8_ref(inputs, sp, P, E, 1, 0, cap)
            assert torch.equal(_bytes(out), want_codes) and torch.equal(_bytes(scales), want_scales)
        elif me == 0:
            assert torch.equal(_bytes(out), _ref_dispatch(inputs, sp, P, E, 1, 0, cap)[0])
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


def _moe_expert(x, e_global):
    """A per-row expert (elementwise, so its result does not depend on how rows are batched)."""
    a = 0.5 + 0.125 * e_global
    return (torch.nn.functional.silu(x * a) * (1.0 - 0.0625 * e_global)).to(x.dtype)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_moe_layer_end_to_end(size):
    """A top-2 MoE layer, 2 experts per rank: dispatch_dev, experts over each segment found through
    out_offsets, combine_dev, weighted sum. Matches the dense single-process computation within
    bf16 tolerance, and the host-count dispatch / combine path exactly."""
    gcu = _cuda()
    P, E, T, H = size, 2, 24, 64
    G = P * E

    def routed(rank):
        g = torch.Generator().manual_seed(300 + rank)
        x = torch.randn(T, H, generator=g).to(torch.bfloat16)
        logits = torch.randn(T, G, generator=g)
        w, idx = torch.topk(torch.softmax(logits, dim=-1), 2, dim=-1)
        return x, w / w.sum(-1, keepdim=True), idx

    def dense(rank):
        x, w, idx = routed(rank)
        y = torch.zeros(T, H)
        for t in range(T):
            for slot in range(2):
                y[t] += w[t, slot] * _moe_expert(x[t:t + 1], int(idx[t, slot]))[0].float()
        return y

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        x, w, idx = routed(me)
        x, w, idx = x.cuda(), w.cuda(), idx.cuda()
        flat = idx.reshape(-1)                      # pair p = token * 2 + slot
        order = torch.argsort(flat, stable=True)    # pairs grouped by (rank, expert)
        tokens = x[order // 2]
        splits = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, flat, torch.ones_like(flat))
        cap = T * 2 * P

        def finish(rows_back):
            y_pairs = torch.empty_like(rows_back)
            y_pairs[order] = rows_back
            y_pairs = y_pairs.view(T, 2, H).float()
            return y_pairs[:, 0] * w[:, :1] + y_pairs[:, 1] * w[:, 1:]

        # device-split path
        out = cc.empty((cap, H), torch.bfloat16)
        out, osp, ooff = moe.dispatch_dev(tokens, splits, out, experts=E)
        expert_out = torch.empty_like(out)
        osp_h, ooff_h = osp.tolist(), ooff.tolist()
        for e in range(E):
            lo = ooff_h[e * P]
            hi = ooff_h[e * P + P - 1] + osp_h[e * P + P - 1]
            expert_out[lo:hi] = _moe_expert(out[lo:hi], me * E + e)
        back = torch.empty_like(tokens)
        moe.combine_dev(expert_out, osp, ooff, back, experts=E)
        y_dev = finish(back)

        # host-count path: per-(source, expert) counts through the host alltoall
        import numpy as np

        sp_h = splits.tolist()
        per_expert = moe.exchange_counts(sp_h)      # entry s*E + e: rows from s for my expert e
        send = [sum(sp_h[j * E:(j + 1) * E]) for j in range(P)]
        recv = [sum(per_expert[s * E:(s + 1) * E]) for s in range(P)]
        out_h = torch.empty((sum(recv), H), dtype=torch.bfloat16, device="cuda")
        moe.dispatch(tokens, send, out_h, recv)
        expert_h = torch.empty_like(out_h)
        row = 0
        for s in range(P):
            for e in range(E):
                n = per_expert[s * E + e]
                expert_h[row:row + n] = _moe_expert(out_h[row:row + n], me * E + e)
                row += n
        back_h = torch.empty_like(tokens)
        moe.combine(expert_h, recv, back_h, send)
        y_host = finish(back_h)
        cc.synchronize()
        assert np.array_equal(_bytes(y_dev).numpy(), _bytes(y_host).numpy())
        torch.testing.assert_close(y_dev.cpu(), dense(me), rtol=2e-2, atol=2e-2)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))
