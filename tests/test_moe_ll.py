"""The low-latency top-k MoE exchange: CudaContext.moe_ll_buffer, alltoallv_ll_topk and
alltoallv_ll_combine_topk, and MoEDispatcher.dispatch_ll / combine_ll. Ranks are threads sharing
cuda:0, each on its own stream. The reference is the device-split top-k exchange on the same inputs:
alltoallv_dev_topk (align 1) for the dispatch, combine_dev_topk for the combine, byte for byte."""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_combine_topk import _reference
from test_moe_dev import SENTINEL, _bytes
from test_moe_dispatch_topk import ROWS, _x

COMBINE_DTYPES = [torch.float32, torch.bfloat16, torch.float16]


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _problem(P, E, k, dtype, width, M, seed, distinct=False):
    """Every rank's (x, topk_idx) with T <= M: -1 and out-of-range entries, an idle rank when P > 2 and
    T = M on rank 0. `distinct`: no token picks an expert twice, so no group can overflow."""
    g = torch.Generator().manual_seed(seed)
    G = P * E
    out = []
    for s in range(P):
        T = M if s == 0 else (0 if (P > 2 and s == 1) else int(torch.randint(1, M + 1, (1,), generator=g)))
        if distinct:
            idx = torch.stack([torch.randperm(max(G, k), generator=g)[:k] for _ in range(T)]) if T else \
                torch.empty(0, k, dtype=torch.int64)
            idx = torch.where(idx < G, idx, torch.full_like(idx, -1))
        else:
            idx = torch.randint(0, G, (T, k), generator=g)
        r = torch.rand(T, k, generator=g)
        idx[r < 0.15] = -1
        idx[(r >= 0.15) & (r < 0.2)] = G + 3
        out.append((_x(T, dtype, width, g), idx))
    return out


def _sentinel(shape, dtype, symmetric, cc):
    t = cc.empty(shape, dtype) if symmetric else torch.empty(shape, dtype=dtype, device="cuda")
    t.view(torch.uint8).fill_(SENTINEL)
    return t


def _ref_dispatch(cc, moe, x, idx, E, tmax, out_scales=False):
    """alltoallv_dev_topk (align 1) into a symmetric out big enough for any layout of up to `tmax`
    tokens per rank."""
    P = cc.size
    cap = P * tmax * idx.shape[1] + 1
    if out_scales:
        o = cc.empty((cap, x.shape[1]), torch.float8_e4m3fn)
        sc = cc.empty((cap, x.shape[1] // 128), torch.float32)
        res = moe.dispatch_dev_topk(x, idx, o, experts=E, align=1, out_scales=sc)
        return res[0], res[2], res[3], res[4], res[5], res[1]
    o = cc.empty((cap, x.shape[1]), x.dtype)
    out, osp, ooff, splits, pos = moe.dispatch_dev_topk(x, idx, o, experts=E, align=1)
    return out, osp, ooff, splits, pos, None


def _check_dispatch(cc, out, osp, ref, E, tag, out_scales=None, skip_experts=()):
    """out[e, :count] against expert e's segment of the reference, out_splits, the sentinel tail."""
    P = cc.size
    rout, rsp, roff = ref[0], ref[1].cpu(), ref[2].cpu()
    got_sp = osp.cpu()
    for e in range(E):
        if e in skip_experts:
            continue
        assert torch.equal(got_sp[e * P:(e + 1) * P], rsp[e * P:(e + 1) * P]), (tag, e)
        n, o = int(rsp[e * P:(e + 1) * P].sum()), int(roff[e * P])
        assert torch.equal(_bytes(out[e, :n]), _bytes(rout[o:o + n])), (tag, e)
        assert bool((_bytes(out[e, n:]) == SENTINEL).all()), (tag, e)
        if out_scales is not None:
            assert torch.equal(_bytes(out_scales[e, :n]), _bytes(ref[5][o:o + n])), (tag, e)
            assert bool((_bytes(out_scales[e, n:]) == SENTINEL).all()), (tag, e)


def _cases(P):
    Es, Ks = (1, 3, 32), (1, 2, 8, 32)
    return [(Es[c % 3], Ks[c % 4], ROWS[c % 4], c % 2 == 0) for c in range(12)]


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_ll_dispatch_identity(size):
    """A spread of (E, k, row dtype, symmetric / plain out) at this P: every expert's packed rows and
    out_splits equal alltoallv_dev_topk's segment byte for byte, rows past the count keep the
    sentinel and x is unchanged; combine_ll over those rows equals the CPU combine. Inputs have -1 and
    out-of-range entries, an idle rank, T = max_tokens and tokens that pick an expert twice (max_tokens
    is large enough that no group overflows)."""
    gcu = _cuda()
    P = size

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        for c, (E, k, (dtype, width), symmetric) in enumerate(_cases(P)):
            T = 9
            M = T * k  # a group may take every choice of every token
            per = _problem(P, E, k, dtype, width, T, 500 * P + c)
            x, idx = (t.cuda() for t in per[cc.rank])
            buf = cc.moe_ll_buffer(E, M, k, width, dtype=dtype)
            out = _sentinel((E, P * M, width), dtype, symmetric, cc)
            x0 = _bytes(x)
            got, osp = moe.dispatch_ll(x, idx, buf, out)
            ref = _ref_dispatch(cc, moe, x, idx, E, T)
            cc.synchronize()
            _check_dispatch(cc, got, osp, ref, E, (E, k, str(dtype), symmetric))
            assert torch.equal(_bytes(x), x0)
            if dtype in COMBINE_DTYPES:  # rows of other dtypes have no combine; the buffer is dropped
                y = torch.empty((x.shape[0], width), dtype=dtype, device="cuda")
                moe.combine_ll(out, None, buf, y)
                # out holds each routed choice's own token row, and no group overflows: the CPU
                # combine of row t * k + j = x[t] over every routed choice
                T = x.shape[0]
                flat = idx.cpu().reshape(-1)
                pos = torch.where((flat >= 0) & (flat < P * E), torch.arange(T * k), -1).view(T, k)
                want = _reference(x.cpu().repeat_interleave(k, 0), pos, torch.ones(T, k), dtype)
                cc.synchronize()
                assert torch.equal(_bytes(y), _bytes(want)), (E, k, str(dtype), symmetric)
            cc.synchronize()
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_ll_fp8_identity(size):
    """The FP8 form: codes and scales equal the FP8 alltoallv_dev_topk's byte for byte, and the bf16
    combine of the dequantised rows equals combine_dev_topk's."""
    gcu = _cuda()
    P, E, k, H, M = size, 3, 4, 384, 8

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        per = _problem(P, E, k, torch.bfloat16, H, M, 70 + P, distinct=True)
        x, idx = (t.cuda() for t in per[cc.rank])
        if x.shape[0] > 2:
            x[1] *= 1e-6  # a block whose amax is below the 1e-4 floor
        buf = cc.moe_ll_buffer(E, M, k, H, fp8=True)
        out = _sentinel((E, P * M, H), torch.float8_e4m3fn, False, cc)
        sc = _sentinel((E, P * M, H // 128), torch.float32, False, cc)
        got, gsc, osp = moe.dispatch_ll(x, idx, buf, out, out_scales=sc)
        ref = _ref_dispatch(cc, moe, x, idx, E, M, out_scales=True)
        cc.synchronize()
        _check_dispatch(cc, got, osp, ref, E, "fp8", out_scales=gsc)
        deq = (got.float().view(E, P * M, H // 128, 128) * gsc.unsqueeze(-1)).view(E, P * M, H).to(torch.bfloat16)
        y = torch.empty((x.shape[0], H), dtype=torch.bfloat16, device="cuda")
        moe.combine_ll(deq, None, buf, y)
        rdeq = (ref[0].float().view(-1, H // 128, 128) * ref[5].unsqueeze(-1)).view(-1, H).to(torch.bfloat16)
        want = torch.empty_like(y)
        moe.combine_dev_topk(rdeq.contiguous(), ref[3], ref[4], None, want, experts=E, align=1)
        cc.synchronize()
        assert torch.equal(_bytes(y), _bytes(want))
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=300000))


def _expert_fn(e, rows):
    """A deterministic per-expert row function, applied alike to both layouts."""
    return (rows.float() * (0.5 + 0.25 * e) + (e - 1.0)).to(rows.dtype)


def _ll_layer(cc, moe, buf, x, idx, w, out, eo, y):
    E = buf.experts
    moe.dispatch_ll(x, idx, buf, out)
    for e in range(E):
        eo[e].copy_(_expert_fn(e, out[e]))
    return moe.combine_ll(eo, w, buf, y)


def _dev_layer(cc, moe, x, idx, w, E, tmax):
    out, osp, ooff, splits, pos, _ = _ref_dispatch(cc, moe, x, idx, E, tmax)
    eo = torch.zeros_like(out)
    sp, off = osp.cpu(), ooff.cpu()
    P = cc.size
    for e in range(E):
        n, o = int(sp[e * P:(e + 1) * P].sum()), int(off[e * P])
        eo[o:o + n] = _expert_fn(e, out[o:o + n])
    y = torch.empty_like(x)
    moe.combine_dev_topk(eo, splits, pos, w, y, experts=E, align=1)
    return y


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 4, 8])
def test_ll_combine_identity(size):
    """Dispatch, a per-expert row function, combine: y equals combine_dev_topk's on the same expert
    rows byte for byte, for float32, bfloat16 and float16, with weights and with None."""
    gcu = _cuda()
    P, E, k, H, M = size, 3, 4, 64, 16

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        for c, dtype in enumerate(COMBINE_DTYPES):
            buf = cc.moe_ll_buffer(E, M, k, H, dtype=dtype)
            out = torch.empty((E, P * M, H), dtype=dtype, device="cuda")
            eo = torch.zeros_like(out)
            for weighted in (True, False):
                per = _problem(P, E, k, dtype, H, M, 900 + 10 * P + c, distinct=True)
                x, idx = (t.cuda() for t in per[cc.rank])
                w = torch.randn(x.shape[0], k, generator=torch.Generator().manual_seed(c)).cuda() if weighted else None
                y = _ll_layer(cc, moe, buf, x, idx, w, out, eo, torch.empty_like(x))
                want = _dev_layer(cc, moe, x, idx, w, E, M)
                cc.synchronize()
                assert torch.equal(_bytes(y), _bytes(want)), (dtype, weighted)
                cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
def test_ll_reuse_200_calls():
    """200 alternating dispatch / combine calls on one buffer with fresh inputs, each checked."""
    gcu = _cuda()
    P, E, k, H, M = 3, 2, 3, 32, 12

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        buf = cc.moe_ll_buffer(E, M, k, H)
        out = torch.empty((E, P * M, H), dtype=torch.bfloat16, device="cuda")
        eo = torch.zeros_like(out)
        for it in range(200):
            per = _problem(P, E, k, torch.bfloat16, H, M, 10_000 + it, distinct=True)
            x, idx = (t.cuda() for t in per[cc.rank])
            w = torch.rand(x.shape[0], k, generator=torch.Generator().manual_seed(it)).cuda()
            y = _ll_layer(cc, moe, buf, x, idx, w, out, eo, torch.empty_like(x))
            want = _dev_layer(cc, moe, x, idx, w, E, M)
            cc.synchronize()
            assert torch.equal(_bytes(y), _bytes(want)), it
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
def test_ll_cuda_graph_replay():
    """dispatch_ll -> experts -> combine_ll captured once in a CUDA graph and replayed with new contents
    in the static x and topk_idx: each replay equals the eager device-split layer."""
    gcu = _cuda()
    P, E, k, H, M = 2, 4, 4, 128, 8

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        buf = cc.moe_ll_buffer(E, M, k, H)
        out = torch.empty((E, P * M, H), dtype=torch.bfloat16, device="cuda")
        eo = torch.zeros_like(out)
        x = torch.empty((M, H), dtype=torch.bfloat16, device="cuda")
        idx = torch.full((M, k), -1, dtype=torch.int64, device="cuda")
        w = torch.ones((M, k), dtype=torch.float32, device="cuda")
        y = torch.empty_like(x)
        _ll_layer(cc, moe, buf, x, idx, w, out, eo, y)  # warm up every kernel outside the capture
        cc.synchronize()
        cc.pc.host_barrier()
        # Captured on this rank's own stream, thread-local, and without torch.cuda.graph's device-wide
        # synchronize: the other rank's thread may be capturing already.
        g = torch.cuda.CUDAGraph()
        g.capture_begin(capture_error_mode="thread_local")
        _ll_layer(cc, moe, buf, x, idx, w, out, eo, y)
        g.capture_end()
        cc.pc.host_barrier()
        for it in range(20):
            per = _problem(P, E, k, torch.bfloat16, H, M, 300 + it, distinct=True)
            xs, ids = per[cc.rank]
            T = xs.shape[0]
            x.zero_()
            idx.fill_(-1)
            x[:T].copy_(xs)
            idx[:T].copy_(ids)
            w.copy_(torch.rand(M, k, generator=torch.Generator().manual_seed(it)))
            g.replay()
            want = _dev_layer(cc, moe, x, idx, w, E, M)
            cc.synchronize()
            assert torch.equal(_bytes(y), _bytes(want)), it
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
def test_ll_slot_overflow():
    """Rank 0 sends more than max_tokens rows to expert 0 of rank 1 (its tokens pick it twice): both
    ranks raise ValueError at synchronize(), every other group is served and checked, the combine
    leaves the overflowed choices out, and the next layer succeeds."""
    gcu = _cuda()
    P, E, k, H, M = 2, 2, 2, 32, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        buf = cc.moe_ll_buffer(E, M, k, H)
        out = _sentinel((E, P * M, H), torch.bfloat16, False, cc)
        g = torch.Generator().manual_seed(5)
        x = torch.randn(M, H, generator=g).to(torch.bfloat16).cuda()
        if cc.rank == 0:
            idx = torch.tensor([[2, 2], [2, 2], [2, 1], [0, 3]], dtype=torch.int64).cuda()  # 5 rows for expert 2
        else:
            idx = torch.tensor([[0, 2], [1, 3], [3, -1], [2, 0]], dtype=torch.int64).cuda()
        _, osp = moe.dispatch_ll(x, idx, buf, out)
        with pytest.raises(ValueError, match="max_tokens"):
            cc.synchronize()
        ref = _ref_dispatch(cc, moe, x, idx, E, M)
        # Rank 1's expert 0 lost rank 0's group; everything else matches.
        skip = (0,) if cc.rank == 1 else ()
        _check_dispatch(cc, out, osp, ref, E, "overflow", skip_experts=skip)
        if cc.rank == 1:
            assert int(osp[0]) == 0 and int(osp[1]) == int(ref[1][1])
            n0 = int(ref[1][1])
            o = int(ref[2][1])
            assert torch.equal(_bytes(out[0, :n0]), _bytes(ref[0][o:o + n0]))
        eo = torch.zeros_like(out)
        for e in range(E):
            eo[e].copy_(_expert_fn(e, out[e]))
        w = torch.rand(M, k, generator=g).cuda()
        y = moe.combine_ll(eo, w, buf, torch.empty_like(x))
        # The reference combine with the overflowed choices unrouted.
        pos = ref[4].clone()
        if cc.rank == 0:
            pos[idx == 2] = -1
        rout, rsp, roff = ref[0], ref[1].cpu(), ref[2].cpu()
        reo = torch.zeros_like(rout)
        for e in range(E):
            n, o = int(rsp[e * P:(e + 1) * P].sum()), int(roff[e * P])
            reo[o:o + n] = _expert_fn(e, rout[o:o + n])
        want = torch.empty_like(x)
        moe.combine_dev_topk(reo, ref[3], pos, w, want, experts=E, align=1)
        cc.synchronize()
        assert torch.equal(_bytes(y), _bytes(want))
        # The next layer succeeds.
        ok = idx.clone()
        ok[:, 1] = (ok[:, 0] + 1) % (P * E)
        y2 = _ll_layer(cc, moe, buf, x, ok, w, torch.empty_like(out), torch.zeros_like(out), torch.empty_like(x))
        want2 = _dev_layer(cc, moe, x, ok, w, E, M)
        cc.synchronize()
        assert torch.equal(_bytes(y2), _bytes(want2))
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=300000))


@pytest.mark.gpu
def test_ll_host_checks():
    """Every malformed call raises ValueError before launch and leaves the buffer usable; buffer
    arguments that differ between ranks raise on every rank."""
    gcu = _cuda()
    P, E, k, H, M = 2, 2, 2, 64, 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        with pytest.raises(ValueError, match="differ between ranks"):
            cc.moe_ll_buffer(E, M + cc.rank, k, H)
        for bad in ((0, M, k, H), (33, M, k, H), (E, M, 0, H), (E, M, 33, H), (E, 0, k, H), (E, M, k, 4)):
            with pytest.raises(ValueError):
                cc.moe_ll_buffer(*bad)
        with pytest.raises(ValueError):
            cc.moe_ll_buffer(E, M, k, 100, fp8=True)
        buf = cc.moe_ll_buffer(E, M, k, H)
        bf = torch.bfloat16
        x = torch.randn(M, H, device="cuda").to(bf)
        idx = torch.tensor([[0, 1]] * M, dtype=torch.int64, device="cuda")  # no group above max_tokens
        out = torch.empty((E, P * M, H), dtype=bf, device="cuda")
        sp = torch.empty(E * P, dtype=torch.int64, device="cuda")
        y = torch.empty_like(x)
        with pytest.raises(ValueError, match="no dispatch"):
            cc.alltoallv_ll_combine_topk(buf, y, out, None)
        bad_dispatch = [
            dict(x=x.float()),                                                       # dtype
            dict(x=torch.randn(M + 1, H, device="cuda").to(bf),                      # T > max_tokens
                 topk_idx=torch.zeros(M + 1, k, dtype=torch.int64, device="cuda")),
            dict(topk_idx=torch.zeros(M, k + 1, dtype=torch.int64, device="cuda")),  # k
            dict(topk_idx=idx.int()),                                                # int32 indices
            dict(out=torch.empty((E, P * M - 1, H), dtype=bf, device="cuda")),       # shape
            dict(out=torch.empty((E, H, P * M), dtype=bf, device="cuda").transpose(1, 2)),  # contiguity
            dict(x=torch.empty(M * H + 1, dtype=bf, device="cuda")[1:].view(M, H)),  # alignment
            dict(out_splits=torch.empty(E * P, dtype=torch.int32, device="cuda")),
            dict(out=buf.tensor[:E * P * M * H * 2].view(bf).view(E, P * M, H)),    # overlaps the buffer
            dict(out_scales=torch.empty((E, P * M, H // 128), device="cuda")),       # not an FP8 buffer
        ]
        shared = torch.empty(M * H + E * P * M * H, dtype=bf, device="cuda")
        bad_dispatch.append(dict(x=shared[:M * H].view(M, H), out=shared[:E * P * M * H].view(E, P * M, H)))
        for kw in bad_dispatch:
            args = dict(x=x, topk_idx=idx, out=out, out_splits=sp)
            args.update(kw)
            with pytest.raises(ValueError):
                cc.alltoallv_ll_topk(buf, args["out"], args["x"], args["topk_idx"], args["out_splits"],
                                     out_scales=args.get("out_scales"))
        moe.dispatch_ll(x, idx, buf, out)
        with pytest.raises(ValueError, match="not been combined"):
            moe.dispatch_ll(x, idx, buf, out)
        bad_combine = [
            dict(y=torch.empty((M - 1, H), dtype=bf, device="cuda")),        # T of the dispatch
            dict(y=y.float()),
            dict(eo=out.float()),
            dict(w=torch.ones(M, k + 1, device="cuda")),
            dict(w=torch.ones(M, k, device="cuda", dtype=torch.float64)),
            dict(y=out[0, :M]),                                              # overlaps expert_out
        ]
        for kw in bad_combine:
            with pytest.raises(ValueError):
                cc.alltoallv_ll_combine_topk(buf, kw.get("y", y), kw.get("eo", out), kw.get("w"))
        moe.combine_ll(out, None, buf, y)
        cc.synchronize()
        return True

    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=300000))
