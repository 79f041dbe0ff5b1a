"""The quantising device-split all-to-all-v: CudaContext.alltoallv_dev with bf16 input, e4m3 out and
fp32 out_scales (one per 1x128 block), and MoEDispatcher.dispatch_dev_fp8 built on it. Ranks are
threads sharing cuda:0, each on its own stream. References are computed on the CPU."""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_dev import SENTINEL, _bytes, _layout, _moe_expert, _splits

E4M3 = torch.float8_e4m3fn


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _quant(x):
    """The 1x128 per-token-group recipe, bit for bit what the kernel computes, on either device.
    The scale divides by a tensor: on CUDA, torch divides by a Python scalar by multiplying with
    its rounded reciprocal, which is not ``amax / 448`` correctly rounded (on the CPU both agree)."""
    n, H = x.shape
    xf = x.float().view(n, H // 128, 128)
    amax = xf.abs().amax(-1).clamp(min=1e-4)
    codes = (xf * (448.0 / amax)[..., None]).to(E4M3).view(n, H)
    return codes, amax / torch.full_like(amax, 448.0)


def _dequant(codes, scales):
    n, H = codes.shape
    return (codes.float().view(n, H // 128, 128) * scales[..., None]).view(n, H).to(torch.bfloat16)


def _rows(n, H, seed):
    """bf16 rows whose magnitude varies from row to row (and so does every block scale)."""
    g = torch.Generator().manual_seed(seed)
    mag = torch.exp(torch.randn(n, 1, generator=g) * 3)
    return (torch.randn(n, H, generator=g) * mag).to(torch.bfloat16)


def _ref(inputs, sp, P, E, align, d, cap):
    """Rank d's codes and scales as bytes, sentinel outside the segments, and its layout."""
    osp, ooff, _ = _layout(sp, P, E, align, d)
    H = inputs[0].shape[1]
    codes = torch.full((cap, H), SENTINEL, dtype=torch.uint8)
    scales = torch.full((cap, H // 128 * 4), SENTINEL, dtype=torch.uint8)
    for e in range(E):
        for s in range(P):
            k = d * E + e
            src, n = sum(sp[s][:k]), sp[s][k]
            if n == 0:
                continue
            c, sc = _quant(inputs[s][src:src + n])
            at = ooff[e * P + s]
            codes[at:at + n] = c.view(torch.uint8)
            scales[at:at + n] = sc.contiguous().view(torch.uint8).view(n, H // 128 * 4)
    return codes.view(-1), scales.view(-1), osp, ooff


def _outs(cc, sym, cap, H, symmetric):
    """(out, out_scales) filled with the sentinel: views of two symmetric byte buffers, or plain."""
    nb = H // 128
    if symmetric:
        out = sym[0][: cap * H].view(E4M3).view(cap, H)
        scales = sym[1][: cap * nb * 4].view(torch.float32).view(cap, nb)
    else:
        out = torch.empty((cap, H), dtype=E4M3, device="cuda")
        scales = torch.empty((cap, nb), dtype=torch.float32, device="cuda")
    out.view(torch.uint8).fill_(SENTINEL)
    scales.view(torch.uint8).fill_(SENTINEL)
    return out, scales


def _composed(cc, out, out_scales, inp, splits, osp, ooff, E, align):
    """Quantise with torch ops on the device, then two alltoallv_dev calls (codes, scale rows)."""
    codes, sc = _quant(inp)
    cc.alltoallv_dev(out, codes, splits, osp, ooff, experts=E, align=align)
    cc.alltoallv_dev(out_scales, sc.contiguous(), splits, torch.empty_like(osp), torch.empty_like(ooff),
                     experts=E, align=align)


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_fp8_dispatch_layouts(size):
    """Every (E, align, H, symmetric / plain out) at this P, with seeded splits that include zeros
    and an idle last rank: codes and scales equal the CPU reference byte for byte, rows outside the
    segments keep the sentinel in both tensors, and out_splits / out_offsets equal those of the
    bf16 alltoallv_dev of the same rows."""
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        sym = (cc.empty(4 << 20, torch.uint8), cc.empty(1 << 20, torch.uint8))
        me = ctx.rank
        case = 0
        for E in (1, 3):
            for align in (1, 16):
                for H in (128, 384, 7168):
                    for symmetric in (True, False):
                        case += 1
                        seed = 1000 * case + 7 * P
                        sp = _splits(P, E, seed)
                        inputs = [_rows(sum(sp[s]), H, seed + 1 + s) for s in range(P)]
                        cap = max(_layout(sp, P, E, align, d)[2] for d in range(P)) + 3
                        assert cap * H <= sym[0].numel() and cap * H // 32 <= sym[1].numel()
                        want_c, want_s, wsp, woff = _ref(inputs, sp, P, E, align, me, cap)
                        inp = inputs[me].cuda()
                        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
                        out, scales = _outs(cc, sym, cap, H, symmetric)
                        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
                        ooff = torch.empty_like(osp)
                        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
                        ref = torch.empty((cap, H), dtype=torch.bfloat16, device="cuda")
                        rsp, roff = torch.empty_like(osp), torch.empty_like(ooff)
                        cc.alltoallv_dev(ref, inp, splits, rsp, roff, experts=E, align=align)
                        cc.synchronize()
                        tag = (E, align, H, symmetric)
                        assert torch.equal(_bytes(out), want_c), tag
                        assert torch.equal(_bytes(scales), want_s), tag
                        assert osp.tolist() == wsp and ooff.tolist() == woff, tag
                        assert osp.tolist() == rsp.tolist() and ooff.tolist() == roff.tolist(), tag
                        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=120000))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (4, False), (3, True)])
def test_fused_equals_composed(size, symmetric):
    """Torch quantisation followed by two alltoallv_dev calls gives the fused call's bytes."""
    gcu = _cuda()
    P, E, align, H = size, 2, 8, 1024

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        sym = (cc.empty(1 << 20, torch.uint8), cc.empty(1 << 16, torch.uint8))
        sym2 = (cc.empty(1 << 20, torch.uint8), cc.empty(1 << 16, torch.uint8))
        me = ctx.rank
        sp = _splits(P, E, 77)
        inputs = [_rows(sum(sp[s]), H, 78 + s) for s in range(P)]
        cap = max(_layout(sp, P, E, align, d)[2] for d in range(P)) + 2
        inp = inputs[me].cuda()
        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
        out, scales = _outs(cc, sym, cap, H, symmetric)
        out2, scales2 = _outs(cc, sym2, cap, H, symmetric)
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        osp2, ooff2 = torch.empty_like(osp), torch.empty_like(osp)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
        _composed(cc, out2, scales2, inp, splits, osp2, ooff2, E, align)
        cc.synchronize()
        assert torch.equal(_bytes(out), _bytes(out2))
        assert torch.equal(_bytes(scales), _bytes(scales2))
        assert osp.tolist() == osp2.tolist() and ooff.tolist() == ooff2.tolist()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def _special_rows():
    """One row set of 8-block rows: all zeros, all -0.0, amax below 1e-4, bf16 subnormals, a block
    holding +-bf16 max, a block whose amax element sits at an odd position, and two random blocks."""
    g = torch.Generator().manual_seed(5)
    n, H = 6, 8 * 128
    x = torch.randn(n, H, generator=g).to(torch.bfloat16)
    blk = x.view(n, 8, 128)
    blk[:, 0] = 0.0
    blk[:, 1] = -0.0
    blk[:, 2] = (torch.randn(n, 128, generator=g) * 2e-5).to(torch.bfloat16)
    sub = torch.randint(1, 0x80, (n, 128), generator=g, dtype=torch.int16)
    sub[:, 1::2] |= -0x8000  # negative subnormals too
    blk[:, 3] = sub.view(torch.bfloat16)
    bmax = torch.finfo(torch.bfloat16).max
    blk[:, 4, 10] = bmax
    blk[:, 4, 11] = -bmax
    for r in range(n):
        blk[r, 5, 2 * r + 77] = -9.5 - r  # amax at an odd position
    return x


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_special_blocks(symmetric):
    gcu = _cuda()
    P, E, align = 2, 1, 1

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        sym = (cc.empty(1 << 16, torch.uint8), cc.empty(1 << 12, torch.uint8))
        x = _special_rows()
        sp = [[3, 3], [2, 4]]
        inputs = [x, x.flip(0)]
        cap = 8
        out, scales = _outs(cc, sym, cap, x.shape[1], symmetric)
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        cc.alltoallv_dev(out, inputs[ctx.rank].cuda(), torch.tensor(sp[ctx.rank], device="cuda"), osp, ooff,
                         out_scales=scales)
        cc.synchronize()
        want_c, want_s, _, _ = _ref(inputs, sp, P, E, align, ctx.rank, cap)
        assert torch.equal(_bytes(out), want_c)
        assert torch.equal(_bytes(scales), want_s)
        # The documented special values: zero blocks give codes 0 (0x80 for -0.0) and 1e-4 / 448.
        c, s = _quant(x)
        assert bool((c.view(torch.uint8).view(6, 8, 128)[:, 0] == 0).all())
        assert bool((c.view(torch.uint8).view(6, 8, 128)[:, 1] == 0x80).all())
        assert bool((s[:, :2] == torch.tensor(1e-4, dtype=torch.float32) / 448.0).all())
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_fp8_moe_layer_end_to_end(size):
    """A top-2 MoE layer, 2 experts per rank: dispatch_dev_fp8, experts on the dequantised rows,
    combine_dev, weighted sum. Equals the same layer on the composed path exactly, and the dense
    bf16 computation within FP8 tolerance."""
    gcu = _cuda()
    P, E, T, H = size, 2, 24, 256
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
        flat = idx.reshape(-1)
        order = torch.argsort(flat, stable=True)
        tokens = x[order // 2]
        splits = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, flat, torch.ones_like(flat))
        cap = T * 2 * P

        def layer(out, scales, osp, ooff):
            deq = _dequant(out, scales)
            expert_out = torch.zeros_like(deq)
            osp_h, ooff_h = osp.tolist(), ooff.tolist()
            for e in range(E):
                lo = ooff_h[e * P]
                hi = ooff_h[e * P + P - 1] + osp_h[e * P + P - 1]
                expert_out[lo:hi] = _moe_expert(deq[lo:hi], me * E + e)
            back = torch.empty_like(tokens)
            moe.combine_dev(expert_out, osp, ooff, back, experts=E)
            y_pairs = torch.empty_like(back)
            y_pairs[order] = back
            y_pairs = y_pairs.view(T, 2, H).float()
            return y_pairs[:, 0] * w[:, :1] + y_pairs[:, 1] * w[:, 1:]

        out = cc.empty((cap, H), E4M3)
        scales = cc.empty((cap, H // 128), torch.float32)
        out, scales, osp, ooff = moe.dispatch_dev_fp8(tokens, splits, out, scales, experts=E)
        y_fused = layer(out, scales, osp, ooff)

        out2 = torch.zeros((cap, H), dtype=E4M3, device="cuda")
        scales2 = torch.zeros((cap, H // 128), dtype=torch.float32, device="cuda")
        osp2, ooff2 = torch.empty_like(osp), torch.empty_like(ooff)
        _composed(cc, out2, scales2, tokens, splits, osp2, ooff2, E, 1)
        y_comp = layer(out2, scales2, osp2, ooff2)
        cc.synchronize()
        assert torch.equal(_bytes(y_fused), _bytes(y_comp))
        torch.testing.assert_close(y_fused.cpu(), dense(me), rtol=0.05, atol=0.15)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size,symmetric", [(2, True), (4, False)])
def test_fp8_graph_capture_replays(size, symmetric):
    """dispatch_dev_fp8 + dequantise + combine_dev captured once per rank; between three replays
    the splits and the data change, and every replay gives the right codes, scales and rows back."""
    gcu = _cuda()
    P, E, H, align = size, 2, 256, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = ctx.rank
        max_rows = 5 * P * E
        cap = P * (max_rows + E * align)
        sym = (cc.empty(cap * H, torch.uint8), cc.empty(cap * H // 32, torch.uint8))
        out, scales = _outs(cc, sym, cap, H, symmetric)
        inp = torch.zeros((max_rows, H), dtype=torch.bfloat16, device="cuda")
        back = torch.empty_like(inp)
        splits = torch.zeros(P * E, dtype=torch.int64, device="cuda")

        def load(seed):
            sp = _splits(P, E, seed)
            inputs = [_rows(max_rows, H, seed + 1 + s) for s in range(P)]
            splits.copy_(torch.tensor(sp[me], dtype=torch.int64))
            inp.copy_(inputs[me])
            out.view(torch.uint8).fill_(SENTINEL)
            scales.view(torch.uint8).fill_(SENTINEL)
            return sp, inputs

        def step():
            _, _, osp, ooff = moe.dispatch_dev_fp8(inp, splits, out, scales, experts=E, align=align)
            moe.combine_dev(_dequant(out, scales), osp, ooff, back, experts=E)
            return osp, ooff

        stream = torch.cuda.current_stream()
        load(11)
        step()  # warm-up outside the graph
        cc.synchronize()
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            osp, ooff = step()
        cc.pc.host_barrier()
        for seed in (21, 31, 41):
            sp, inputs = load(seed)
            stream.synchronize()
            cc.pc.host_barrier()
            g.replay()
            cc.synchronize()
            used = [sum(sp[s]) for s in range(P)]
            want_c, want_s, wsp, woff = _ref([x[:n] for x, n in zip(inputs, used)], sp, P, E, align, me, cap)
            assert torch.equal(_bytes(out), want_c), seed
            assert torch.equal(_bytes(scales), want_s), seed
            assert osp.tolist() == wsp and ooff.tolist() == woff, seed
            mine = inputs[me][:used[me]]
            assert torch.equal(_bytes(back[:used[me]]), _bytes(_dequant(*_quant(mine)))), seed
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_fp8_no_host_sync(symmetric):
    """dispatch_dev_fp8 runs under torch's sync debug mode "error"."""
    gcu = _cuda()
    P, E, H = 2, 2, 256

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        sym = (cc.empty(1 << 16, torch.uint8), cc.empty(1 << 12, torch.uint8))
        sp = _splits(P, E, 5)
        inputs = [_rows(sum(sp[s]), H, 50 + s) for s in range(P)]
        inp = inputs[ctx.rank].cuda()
        splits = torch.tensor(sp[ctx.rank], dtype=torch.int64, device="cuda")
        cap = 64
        out, scales = _outs(cc, sym, cap, H, symmetric)
        torch.cuda.current_stream().synchronize()
        cc.pc.host_barrier()
        if ctx.rank == 0:
            torch.cuda.set_sync_debug_mode("error")
        cc.pc.host_barrier()
        try:
            moe.dispatch_dev_fp8(inp, splits, out, scales, experts=E, align=4)
        finally:
            cc.pc.host_barrier()
            if ctx.rank == 0:
                torch.cuda.set_sync_debug_mode("default")
            cc.pc.host_barrier()
        cc.synchronize()
        want_c, want_s, _, _ = _ref(inputs, sp, P, E, 4, ctx.rank, cap)
        assert torch.equal(_bytes(out), want_c) and torch.equal(_bytes(scales), want_s)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("symmetric", [True, False])
def test_fp8_overflow(symmetric):
    """An out one row too small: every rank raises the overflow ValueError, that rank's codes and
    scales keep every byte, the others are right, and the next call works."""
    gcu = _cuda()
    P, E, align, H = 3, 2, 1, 256

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        me = ctx.rank
        sym = (cc.empty(1 << 16, torch.uint8), cc.empty(1 << 12, torch.uint8))
        sp = [[2, 1, 3, 0, 1, 2], [1, 1, 1, 1, 1, 1], [0, 2, 2, 0, 3, 1]]
        inputs = [_rows(sum(sp[s]), H, 70 + s) for s in range(P)]
        needs = [_layout(sp, P, E, align, d)[2] for d in range(P)]
        small = 1
        cap = needs[me] - 1 if me == small else needs[me] + 2
        inp = inputs[me].cuda()
        splits = torch.tensor(sp[me], dtype=torch.int64, device="cuda")
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        out, scales = _outs(cc, sym, cap, H, symmetric)
        before = (_bytes(out), _bytes(scales))
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
        with pytest.raises(ValueError, match=f"rank {small} needs {needs[small]} output rows but has room for "
                                             f"{needs[small] - 1}"):
            cc.synchronize()
        if me == small:
            assert torch.equal(_bytes(out), before[0]) and torch.equal(_bytes(scales), before[1])
        else:
            want_c, want_s, _, _ = _ref(inputs, sp, P, E, align, me, cap)
            assert torch.equal(_bytes(out), want_c) and torch.equal(_bytes(scales), want_s)
        cc.check_health()
        cc.pc.host_barrier()

        out, scales = _outs(cc, sym, needs[me] + 2, H, symmetric)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, experts=E, align=align, out_scales=scales)
        cc.synchronize()
        want_c, want_s, _, _ = _ref(inputs, sp, P, E, align, me, needs[me] + 2)
        assert torch.equal(_bytes(out), want_c) and torch.equal(_bytes(scales), want_s)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))


@pytest.mark.gpu
def test_fp8_host_errors():
    """Every malformed quantising call raises ValueError before launch, alike on every rank; a
    correct call afterwards works, so none of them launched."""
    gcu = _cuda()
    P, E, H, cap = 2, 1, 256, 16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        sym = (cc.empty(1 << 16, torch.uint8), cc.empty(1 << 12, torch.uint8))
        sp = [[2, 3], [1, 4]]
        inp = _rows(5, H, 90 + ctx.rank).cuda()
        splits = torch.tensor(sp[ctx.rank], dtype=torch.int64, device="cuda")
        osp = torch.empty(P * E, dtype=torch.int64, device="cuda")
        ooff = torch.empty_like(osp)
        out = torch.empty((cap, H), dtype=E4M3, device="cuda")
        scales = torch.empty((cap, H // 128), dtype=torch.float32, device="cuda")
        sym_out, sym_scales = _outs(cc, sym, cap, H, True)
        odd_in = torch.empty(5 * H + 8, dtype=torch.bfloat16, device="cuda")[1:5 * H + 1].view(5, H)
        odd_out = torch.empty(cap * H + 16, dtype=E4M3, device="cuda")[1:cap * H + 1].view(cap, H)
        bad = {
            "H not a multiple of 128": (torch.empty((cap, 192), dtype=E4M3, device="cuda"),
                                        inp[:, :192].contiguous(), torch.empty((cap, 1), device="cuda")),
            "out_scales missing": (out, inp, None),
            "out_scales for a copy": (torch.empty((cap, H), dtype=torch.bfloat16, device="cuda"), inp, scales),
            "fp16 input": (out, inp.half(), scales),
            "fp32 input": (out, inp.float(), scales),
            "e5m2 out": (torch.empty((cap, H), dtype=torch.float8_e5m2, device="cuda"), inp, scales),
            "fp16 scales": (out, inp, scales.half()),
            "scales too wide": (out, inp, torch.empty((cap, H // 128 + 1), device="cuda")),
            "scales rows != cap": (out, inp, torch.empty((cap - 1, H // 128), device="cuda")),
            "scales on the host": (out, inp, torch.empty((cap, H // 128))),
            "1-D input": (out, inp.view(-1), scales),
            "input not 16-byte aligned": (out, odd_in, scales),
            "out not 16-byte aligned": (odd_out, inp, scales),
            "registered out, plain scales": (sym_out, inp, scales),
            "plain out, registered scales": (out, inp, sym_scales),
        }
        for why, (o, i, s) in bad.items():
            with pytest.raises(ValueError):
                cc.alltoallv_dev(o, i, splits, osp, ooff, out_scales=s)
                pytest.fail(why)
        cc.pc.host_barrier()
        out.view(torch.uint8).fill_(SENTINEL)
        scales.view(torch.uint8).fill_(SENTINEL)
        cc.alltoallv_dev(out, inp, splits, osp, ooff, out_scales=scales)
        cc.synchronize()
        inputs = [_rows(5, H, 90 + s) for s in range(P)]
        want_c, want_s, _, _ = _ref(inputs, sp, P, E, 1, ctx.rank, cap)
        assert torch.equal(_bytes(out), want_c) and torch.equal(_bytes(scales), want_s)
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0))
