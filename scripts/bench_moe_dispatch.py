"""MoE dispatch + combine: host-count alltoallv against the device-split alltoallv_dev.

One rank per visible GPU. With a single GPU the ranks are threads sharing it (--ranks, default 2):
those figures show what removing the ``.tolist()`` sync and the TCP count exchange saves, not
what NVLink bandwidth looks like, and are labelled as such.

Per dispatch + combine pair it times:
  host   splits.tolist() + TCP alltoall of the counts + cc.alltoallv, and the inverse alltoallv
  dev    MoEDispatcher.dispatch_dev + combine_dev (no host sync)
  graph  the same two calls captured once in a CUDA graph and replayed

Rows: --tokens x top-k routed to --experts local experts per rank, rows of --hidden elements, in
bf16 and FP8 e4m3. Outputs are symmetric (zero copy) for every path.

A second table times the FP8 dispatch of bf16 rows (dispatch only, median per call, rank 0):
  bf16      MoEDispatcher.dispatch_dev of the bf16 rows
  composed  torch 1x128 quantisation, then alltoallv_dev of the codes and of the scale rows
  fused     MoEDispatcher.dispatch_dev_fp8 (quantises inside the dispatch kernel)
The three outputs are checked against each other before timing.

A third table times the top-k combine, the end of a MoE layer (median per call, rank 0), with the
experts' output symmetric (read in place) and plain (staged through each rank's pool):
  composed  MoEDispatcher.combine_dev, un-permute, and the gate-weighted sum over k in torch (fp32)
  topk      MoEDispatcher.combine_dev_topk (pulls each token's k rows and sums them in one kernel)
Both arms' outputs are checked equal byte for byte before timing. MB/rank counts the expert rows
that reach this rank plus its (tokens, hidden) result, from the shapes.

A fourth table times the top-k dispatch, the start of a MoE layer (median per call, rank 0, the two
arms alternating), with symmetric outputs:
  dispatch  route() + dispatch_dev (bf16) or + dispatch_dev_fp8 (fp8), against dispatch_dev_topk
  layer     route() + dispatch_dev + identity experts + combine_dev_topk, against
            dispatch_dev_topk + identity experts + combine_dev_topk
Both arms' outputs are checked equal byte for byte before timing. "MB avoided" is route()'s copy of
the T x k rows, written once and read back by the dispatch, from the shapes.

A fifth table times the top-k combine's backward (median per call, rank 0, the two arms
alternating), with expert_out and grad_expert_out symmetric and plain, at the combine table's sizes:
  composed  MoEDispatcher.combine_dev of expert_out, un-permute, the fp32 dot with dy per choice in
            torch, w * dy permuted into route order, then dispatch_dev into grad_expert_out
  fused     MoEDispatcher.combine_dev_topk_backward (one kernel: pull, dot and push)
Before timing, grad_expert_out is checked equal byte for byte between the arms, and grad_w within
n * 2^-23 * sum |dy * x| of each other (n = hidden: the bound of any fp32 summation order of n
terms; the two arms sum in different orders). MB/rank is the T x k expert rows read plus the T x k
gradient rows written, from the shapes.

A sixth table (--tables ll) times a decode-sized MoE layer with identity experts (median per layer,
rank 0), each arm captured once in a CUDA graph and replayed, the arms alternating, CUDA events around
each replay, at T = 1, 32 and 128 tokens per rank, bf16 and FP8:
  dev  dispatch_dev_topk + combine_dev_topk (the variable layout agreed at barriers)
  ll   dispatch_ll + combine_ll on a buffer of max_tokens = 128 (fixed slots, one signal round each way)
Before timing, every expert's rows (FP8: codes and scales) and the layer outputs are checked equal byte
for byte between the arms. The FP8 arms combine bf16 rows dequantised once from each arm's codes.

    python scripts/bench_moe_dispatch.py [--ranks 2] [--iters 20] [--tables pairs,fp8,combine,dispatch,backward,ll]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
# Ranks may be threads sharing one GPU: a rank loading a torch kernel for the first time must not
# block behind another rank's collective kernel that waits for it.
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel.strategies import MoEDispatcher  # noqa: E402


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else torch.cuda.get_device_name(0)
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def run_rank(ctx, args, dtype, shared):
    if shared:  # spawn_threads already gave this rank cuda:0 and a stream of its own
        return measure(ctx, args, dtype, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure(ctx, args, dtype, ctx.rank)


def measure(ctx, args, dtype, dev):
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    moe = MoEDispatcher(ctx, cc)
    P, E, H = ctx.size, args.experts, args.hidden
    G = P * E
    k = min(args.topk, G)
    rows = args.tokens * k
    g = torch.Generator(device="cuda").manual_seed(1234 + ctx.rank)
    logits = torch.randn(args.tokens, G, device="cuda", generator=g)
    flat = torch.topk(logits, k, dim=-1).indices.reshape(-1)
    splits = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, flat, torch.ones_like(flat))
    tokens = torch.randn(rows, H, device="cuda", generator=g).to(dtype)
    cap = P * rows
    out = cc.empty((cap, H), dtype)
    back = cc.empty((rows, H), dtype)
    stream = torch.cuda.current_stream()

    def host_pair():
        sp = splits.tolist()
        per = moe.exchange_counts(sp)
        send = [sum(sp[j * E:(j + 1) * E]) * H for j in range(P)]
        recv = [sum(per[s * E:(s + 1) * E]) * H for s in range(P)]
        cc.alltoallv(out, recv, tokens, send)
        cc.alltoallv(back, send, out, recv)

    def dev_pair():
        _, osp, ooff = moe.dispatch_dev(tokens, splits, out, experts=E)
        moe.combine_dev(out, osp, ooff, back, experts=E)

    graph = torch.cuda.CUDAGraph()

    def timed(fn):
        fn()
        cc.synchronize()
        times = []
        for _ in range(args.iters):
            cc.pc.host_barrier()
            t0 = time.perf_counter()
            fn()
            cc.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(times)

    res = {"host": timed(host_pair), "dev": timed(dev_pair)}
    cc.pc.host_barrier()
    with torch.cuda.graph(graph, stream=stream, capture_error_mode="thread_local"):
        dev_pair()
    cc.pc.host_barrier()
    res["graph"] = timed(graph.replay)
    res["bytes_per_rank"] = 2 * rows * H * tokens.element_size()
    return res


def quantise(x):
    """The 1x128 per-token-group recipe with torch ops (what the fused kernel computes). The scale
    divides by a tensor: torch's CUDA division by a Python scalar multiplies by its reciprocal."""
    n, H = x.shape
    xf = x.float().view(n, H // 128, 128)
    amax = xf.abs().amax(-1).clamp(min=1e-4)
    codes = (xf * (448.0 / amax)[..., None]).to(torch.float8_e4m3fn).view(n, H)
    return codes, amax / torch.full_like(amax, 448.0)


def run_rank_fp8(ctx, args, shared):
    if shared:
        return measure_fp8(ctx, args, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure_fp8(ctx, args, ctx.rank)


def measure_fp8(ctx, args, dev):
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    moe = MoEDispatcher(ctx, cc)
    P, E, H = ctx.size, args.experts, args.hidden
    G = P * E
    k = min(args.topk, G)
    rows = args.tokens * k
    g = torch.Generator(device="cuda").manual_seed(4321 + ctx.rank)
    flat = torch.topk(torch.randn(args.tokens, G, device="cuda", generator=g), k, dim=-1).indices.reshape(-1)
    splits = torch.zeros(G, dtype=torch.int64, device="cuda").index_add_(0, flat, torch.ones_like(flat))
    tokens = torch.randn(rows, H, device="cuda", generator=g).to(torch.bfloat16)
    cap = P * rows
    out_bf16 = cc.empty((cap, H), torch.bfloat16)
    codes = [cc.empty((cap, H), torch.float8_e4m3fn) for _ in range(2)]
    scales = [cc.empty((cap, H // 128), torch.float32) for _ in range(2)]
    osp = torch.empty(G, dtype=torch.int64, device="cuda")
    ooff, osp2, ooff2 = torch.empty_like(osp), torch.empty_like(osp), torch.empty_like(osp)

    def bf16():
        moe.dispatch_dev(tokens, splits, out_bf16, experts=E)

    def composed():
        c, s = quantise(tokens)
        cc.alltoallv_dev(codes[0], c, splits, osp, ooff, experts=E)
        cc.alltoallv_dev(scales[0], s, splits, osp2, ooff2, experts=E)

    def fused():
        moe.dispatch_dev_fp8(tokens, splits, codes[1], scales[1], experts=E)

    quantise(tokens)  # this rank's torch kernels and allocations, before any peer waits on it
    cc.synchronize()
    cc.pc.host_barrier()
    for fn in (bf16, composed, fused):
        fn()
    cc.synchronize()
    # Every received row: fused == composed byte for byte, and both dequantise to the bf16 rows.
    n = int(osp.sum())
    lo = int(ooff.min()) if n else 0
    assert torch.equal(codes[0].view(torch.uint8)[lo:lo + n], codes[1].view(torch.uint8)[lo:lo + n])
    assert torch.equal(scales[0].view(torch.int32)[lo:lo + n], scales[1].view(torch.int32)[lo:lo + n])
    deq = (codes[1][lo:lo + n].float().view(n, H // 128, 128) * scales[1][lo:lo + n, :, None]).view(n, H)
    ref = out_bf16[lo:lo + n].float()
    assert bool(((deq - ref).abs() <= ref.abs().view(n, H // 128, 128).amax(-1).repeat_interleave(128, -1)
                 / 16 + 1e-30).all()), "fp8 dispatch is not within e4m3 rounding of the bf16 dispatch"

    def timed(fn):
        fn()
        cc.synchronize()
        times = []
        for _ in range(args.iters):
            cc.pc.host_barrier()
            t0 = time.perf_counter()
            fn()
            cc.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(times)

    res = {"bf16": timed(bf16), "composed": timed(composed), "fused": timed(fused)}
    # Bytes this rank sends (its own rows included): bf16 rows, or e4m3 codes + fp32 scales.
    res["bytes_bf16"] = rows * H * 2
    res["bytes_fp8"] = rows * (H + H // 128 * 4)
    return res


def run_rank_topk(ctx, args, shared):
    if shared:
        return measure_topk(ctx, args, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure_topk(ctx, args, ctx.rank)


def measure_topk(ctx, args, dev):
    P, E, H, T = ctx.size, args.experts, args.hidden, args.tokens
    G = P * E
    k = min(args.topk, G)
    rows = T * k
    cap = P * rows
    rb = H * 2
    # A plain expert_out is staged through the pool, and so is combine_dev's plain output: room for
    # a holder that receives every row.
    cc = gcu.CudaContext(ctx, dev, stage_bytes=(cap + 1024) * rb)
    moe = MoEDispatcher(ctx, cc)
    g = torch.Generator(device="cuda").manual_seed(777 + ctx.rank)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    w, idx = torch.topk(torch.softmax(torch.randn(T, G, device="cuda", generator=g), -1), k, dim=-1)
    tokens, splits, pos = moe.route(x, idx, E)
    eo = {"symmetric": cc.empty((cap, H), torch.bfloat16)}
    _, osp, ooff = moe.dispatch_dev(tokens, splits, eo["symmetric"], experts=E)  # identity experts
    eo["plain"] = eo["symmetric"].clone()
    backs = {"symmetric": cc.empty((rows, H), torch.bfloat16),
             "plain": torch.empty((rows, H), dtype=torch.bfloat16, device="cuda")}
    outs = {kind: [torch.empty((T, H), dtype=torch.bfloat16, device="cuda") for _ in range(2)] for kind in eo}

    def composed(kind):
        back = backs[kind]
        moe.combine_dev(eo[kind], osp, ooff, back, experts=E)
        acc = torch.zeros((T, H), device="cuda")
        for j in range(k):  # the kernel's order: acc + w * x, one rounding each
            acc = acc + w[:, j, None] * back.index_select(0, pos[:, j]).float()
        outs[kind][0].copy_(acc)

    def topk(kind):
        moe.combine_dev_topk(eo[kind], splits, pos, w, outs[kind][1], experts=E)

    def timed(fn):
        fn()
        cc.synchronize()
        times = []
        for _ in range(args.iters):
            cc.pc.host_barrier()
            t0 = time.perf_counter()
            fn()
            cc.synchronize()
            times.append((time.perf_counter() - t0) * 1e3)
        return statistics.median(times)

    res = {}
    for kind in eo:
        composed(kind)
        topk(kind)
        cc.synchronize()
        assert torch.equal(outs[kind][0].view(torch.int16), outs[kind][1].view(torch.int16)), kind
        res[f"composed_{kind}"] = timed(lambda: composed(kind))
        res[f"topk_{kind}"] = timed(lambda: topk(kind))
        cc.pc.host_barrier()
    res["bytes"] = (rows + T) * rb
    return res


def run_rank_backward(ctx, args, shared):
    if shared:
        return measure_backward(ctx, args, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure_backward(ctx, args, ctx.rank)


def measure_backward(ctx, args, dev):
    P, E, H, T = ctx.size, args.experts, args.hidden, args.tokens
    G = P * E
    k = min(args.topk, G)
    rows = T * k
    cap = P * rows
    rb = H * 2
    # Plain, the backward stages expert_out and the gradient rows: room for two holders' worth.
    cc = gcu.CudaContext(ctx, dev, stage_bytes=(2 * cap + 2048) * rb)
    moe = MoEDispatcher(ctx, cc)
    g = torch.Generator(device="cuda").manual_seed(991 + ctx.rank)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    dy = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    w, idx = torch.topk(torch.softmax(torch.randn(T, G, device="cuda", generator=g), -1), k, dim=-1)
    tokens, splits, pos = moe.route(x, idx, E)  # every choice is routed: pos is a permutation
    eo = {"symmetric": cc.empty((cap, H), torch.bfloat16)}
    _, osp, ooff = moe.dispatch_dev(tokens, splits, eo["symmetric"], experts=E)  # identity experts
    eo["plain"] = eo["symmetric"].clone()
    mk = {"symmetric": lambda shape: cc.empty(shape, torch.bfloat16),
          "plain": lambda shape: torch.empty(shape, dtype=torch.bfloat16, device="cuda")}
    backs = {kind: mk[kind]((rows, H)) for kind in eo}
    gins = {kind: mk[kind]((rows, H)) for kind in eo}
    geos = {kind: [mk[kind]((cap, H)).zero_() for _ in range(2)] for kind in eo}
    gws = {kind: [torch.empty((T, k), device="cuda") for _ in range(2)] for kind in eo}
    flat = pos.view(-1)

    def composed(kind):
        back = backs[kind]
        moe.combine_dev(eo[kind], osp, ooff, back, experts=E)
        xr = back.index_select(0, flat).view(T, k, H)
        gws[kind][0].copy_((xr.float() * dy.float()[:, None, :]).sum(-1))
        scaled = (w[:, :, None] * dy.float()[:, None, :]).to(torch.bfloat16)
        gins[kind].index_copy_(0, flat, scaled.view(rows, H))
        moe.dispatch_dev(gins[kind], splits, geos[kind][0], experts=E)

    def fused(kind):
        moe.combine_dev_topk_backward(dy, eo[kind], splits, pos, w, geos[kind][1], gws[kind][1], experts=E)

    res = {}
    for kind in eo:
        composed(kind)
        fused(kind)
        cc.synchronize()
        assert torch.equal(geos[kind][0].view(torch.int16), geos[kind][1].view(torch.int16)), kind
        xr = backs[kind].index_select(0, flat).view(T, k, H).float()
        bound = H * 2.0 ** -23 * (xr.abs() * dy.float().abs()[:, None, :]).sum(-1)
        assert bool(((gws[kind][0] - gws[kind][1]).abs() <= bound).all()), kind
        times = {"composed": [], "fused": []}
        for _ in range(args.iters):
            for arm, fn in (("composed", composed), ("fused", fused)):
                cc.pc.host_barrier()
                t0 = time.perf_counter()
                fn(kind)
                cc.synchronize()
                times[arm].append((time.perf_counter() - t0) * 1e3)
        res[f"composed_{kind}"] = statistics.median(times["composed"])
        res[f"fused_{kind}"] = statistics.median(times["fused"])
        cc.pc.host_barrier()
    res["bytes"] = 2 * rows * rb
    return res


def run_rank_dispatch_topk(ctx, args, shared):
    if shared:
        return measure_dispatch_topk(ctx, args, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure_dispatch_topk(ctx, args, ctx.rank)


def measure_dispatch_topk(ctx, args, dev):
    P, E, H, T = ctx.size, args.experts, args.hidden, args.tokens
    G = P * E
    k = min(args.topk, G)
    cap = P * T * k
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    moe = MoEDispatcher(ctx, cc)
    g = torch.Generator(device="cuda").manual_seed(999 + ctx.rank)
    x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
    w, idx = torch.topk(torch.softmax(torch.randn(T, G, device="cuda", generator=g), -1), k, dim=-1)
    outs = [cc.empty((cap, H), torch.bfloat16) for _ in range(2)]
    codes = [cc.empty((cap, H), torch.float8_e4m3fn) for _ in range(2)]
    scales = [cc.empty((cap, H // 128), torch.float32) for _ in range(2)]
    ys = [torch.empty((T, H), dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    for t in outs + codes + scales:
        t.view(torch.uint8).zero_()
    got = {}

    def composed_bf16(i=0):
        rows, splits, pos = moe.route(x, idx, E)
        moe.dispatch_dev(rows, splits, outs[i], experts=E)
        return splits, pos

    def fused_bf16(i=1):
        return moe.dispatch_dev_topk(x, idx, outs[i], experts=E)[3:]

    def composed_fp8():
        rows, splits, _ = moe.route(x, idx, E)
        moe.dispatch_dev_fp8(rows, splits, codes[0], scales[0], experts=E)

    def fused_fp8():
        moe.dispatch_dev_topk(x, idx, codes[1], experts=E, out_scales=scales[1])

    def layer(dispatch, i):
        def fn():
            splits, pos = dispatch(i)
            moe.combine_dev_topk(outs[i], splits, pos, w, ys[i], experts=E)  # identity experts
        return fn

    arms = {
        "dispatch_bf16": (composed_bf16, fused_bf16, lambda: (outs[0], outs[1])),
        "dispatch_fp8": (composed_fp8, fused_fp8, lambda: (torch.cat([codes[0].view(torch.uint8).view(-1),
                                                                       scales[0].view(torch.uint8).view(-1)]),
                                                            torch.cat([codes[1].view(torch.uint8).view(-1),
                                                                       scales[1].view(torch.uint8).view(-1)]))),
        "layer_bf16": (layer(composed_bf16, 0), layer(fused_bf16, 1), lambda: (ys[0], ys[1])),
    }
    for name, (a, b, results) in arms.items():
        a()
        b()
        cc.synchronize()
        u, v = results()
        assert torch.equal(u.view(torch.uint8), v.view(torch.uint8)), name
        ta, tb = [], []
        for _ in range(args.iters):
            for fn, times in ((a, ta), (b, tb)):
                cc.pc.host_barrier()
                t0 = time.perf_counter()
                fn()
                cc.synchronize()
                times.append((time.perf_counter() - t0) * 1e3)
        got[f"{name}_composed"] = statistics.median(ta)
        got[f"{name}_topk"] = statistics.median(tb)
        cc.pc.host_barrier()
    got["bytes_avoided"] = 2 * T * k * H * 2
    return got


def run_rank_ll(ctx, args, shared):
    if shared:
        return measure_ll(ctx, args, 0)
    torch.cuda.set_device(ctx.rank)
    with torch.cuda.stream(gcu.new_stream(ctx.rank)):
        return measure_ll(ctx, args, ctx.rank)


def measure_ll(ctx, args, dev):
    P, E, H, M = ctx.size, args.experts, args.hidden, 128
    G = P * E
    k = min(args.topk, G)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    moe = MoEDispatcher(ctx, cc)
    got = {}
    for fp8 in (False, True):
        buf = cc.moe_ll_buffer(E, M, k, H, fp8=fp8)
        cap = P * M * k
        dt = torch.float8_e4m3fn if fp8 else torch.bfloat16
        dout, lout = cc.empty((cap, H), dt), torch.empty((E, P * M, H), dtype=dt, device="cuda")
        dsc = cc.empty((cap, H // 128), torch.float32) if fp8 else None
        lsc = torch.empty((E, P * M, H // 128), dtype=torch.float32, device="cuda") if fp8 else None
        for T in (1, 32, 128):
            g = torch.Generator(device="cuda").manual_seed(77 + 1000 * T + ctx.rank)
            x = torch.randn(T, H, device="cuda", generator=g).to(torch.bfloat16)
            w, idx = torch.topk(torch.softmax(torch.randn(T, G, device="cuda", generator=g), -1), k, dim=-1)
            ys = [torch.empty((T, H), dtype=torch.bfloat16, device="cuda") for _ in range(2)]
            # Identity experts: the bf16 rows each arm's combine reads are its dispatch output (FP8:
            # dequantised once, below, outside the timed layer).
            res = moe.dispatch_dev_topk(x, idx, dout, experts=E, out_scales=dsc)
            osp, ooff, splits, pos = res[-4:]
            lres = moe.dispatch_ll(x, idx, buf, lout, out_scales=lsc)
            lsp = lres[-1]
            cc.synchronize()
            assert torch.equal(osp, lsp), "out_splits"
            sp, off = osp.cpu(), ooff.cpu()
            for e in range(E):
                n, o = int(sp[e * P:(e + 1) * P].sum()), int(off[e * P])
                assert torch.equal(dout[o:o + n].view(torch.uint8), lout[e, :n].view(torch.uint8)), ("rows", e)
                if fp8:
                    assert torch.equal(dsc[o:o + n], lsc[e, :n]), ("scales", e)
            if fp8:
                deo = (dout.float().view(cap, H // 128, 128) * dsc.unsqueeze(-1)).view(cap, H).to(torch.bfloat16)
                leo = (lout.float().view(E, P * M, H // 128, 128) * lsc.unsqueeze(-1)).view(E, P * M, H)
                leo = leo.to(torch.bfloat16)
            else:
                deo, leo = dout, lout
            moe.combine_ll(leo, w, buf, ys[1])

            def dev_layer():
                r = moe.dispatch_dev_topk(x, idx, dout, experts=E, out_scales=dsc)
                moe.combine_dev_topk(deo, r[-2], r[-1], w, ys[0], experts=E)

            def ll_layer():
                moe.dispatch_ll(x, idx, buf, lout, out_scales=lsc)
                moe.combine_ll(leo, w, buf, ys[1])

            dev_layer()
            cc.synchronize()
            assert torch.equal(ys[0].view(torch.uint8), ys[1].view(torch.uint8)), "y"
            graphs = []
            for fn in (dev_layer, ll_layer):
                cc.pc.host_barrier()
                # On this rank's stream, without torch.cuda.graph's device-wide synchronize: the other
                # ranks' threads may be capturing already.
                gr = torch.cuda.CUDAGraph()
                gr.capture_begin(capture_error_mode="thread_local")
                fn()
                gr.capture_end()
                graphs.append(gr)
            cc.pc.host_barrier()
            times = ([], [])
            for it in range(args.iters + 3):
                for gr, tl in zip(graphs, times):
                    cc.pc.host_barrier()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    gr.replay()
                    e1.record()
                    cc.synchronize()
                    if it >= 3:  # warm-up replays
                        tl.append(e0.elapsed_time(e1))
            name = f"{'fp8' if fp8 else 'bf16'}_T{T}"
            got[f"{name}_dev"] = statistics.median(times[0])
            got[f"{name}_ll"] = statistics.median(times[1])
            cc.pc.host_barrier()
            del graphs
        got[f"{'fp8' if fp8 else 'bf16'}_buffer_bytes"] = buf.nbytes
    return got


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--ranks", type=int, default=2, help="threads sharing the GPU when only one is visible")
    ap.add_argument("--tokens", type=int, default=4096)
    ap.add_argument("--topk", type=int, default=8)
    ap.add_argument("--hidden", type=int, default=7168)
    ap.add_argument("--experts", type=int, default=8, help="local experts per rank")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--tables", default="pairs,fp8,combine,dispatch,backward", help="comma-separated tables to run")
    args = ap.parse_args()
    tables = set(args.tables.split(","))
    assert torch.cuda.is_available(), "needs a GPU"
    ngpu = torch.cuda.device_count()
    shared = ngpu == 1
    P = args.ranks if shared else ngpu
    label = f"{P} threads as ranks sharing one GPU" if shared else f"{P} GPUs, one rank each"
    print(f"# card: {card()}", flush=True)
    print(f"# ranks: {label}; {args.tokens} tokens x top-{args.topk}, hidden {args.hidden}, "
          f"{args.experts} experts per rank; median of {args.iters} dispatch + combine pairs (rank 0)", flush=True)
    if "pairs" in tables:
        print(f"{'dtype':>14} {'host ms':>9} {'dev ms':>9} {'graph ms':>9} {'host/dev':>9} {'MB/rank':>9}")
    for dtype in (torch.bfloat16, torch.float8_e4m3fn) if "pairs" in tables else ():
        if shared:
            r = gb.spawn_threads(P, run_rank, args, dtype, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank, args, dtype, False, timeout_ms=300000)[0]
        print(f"{str(dtype).replace('torch.', ''):>14} {r['host']:9.3f} {r['dev']:9.3f} {r['graph']:9.3f} "
              f"{r['host'] / r['dev']:9.2f} {r['bytes_per_rank'] / 1e6:9.1f}", flush=True)
        print(json.dumps({"dtype": str(dtype), "ranks": P, "shared_gpu": shared, **r}), flush=True)

    if "fp8" in tables:
        print(f"# FP8 dispatch of bf16 rows ({label}); median of {args.iters} dispatch calls (rank 0)", flush=True)
        if shared:
            r = gb.spawn_threads(P, run_rank_fp8, args, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank_fp8, args, False, timeout_ms=300000)[0]
        print(f"{'arm':>10} {'ms':>9} {'MB/rank':>9}")
        for arm, nbytes in (("bf16", r["bytes_bf16"]), ("composed", r["bytes_fp8"]), ("fused", r["bytes_fp8"])):
            print(f"{arm:>10} {r[arm]:9.3f} {nbytes / 1e6:9.1f}", flush=True)
        print(json.dumps({"table": "fp8_dispatch", "ranks": P, "shared_gpu": shared, **r}), flush=True)

    note = "; ranks share one GPU: local-HBM savings, not NVLink" if shared else ""
    if "combine" in tables:
        print(f"# top-k combine, bf16 ({label}{note}); median of {args.iters} calls (rank 0), outputs checked equal",
              flush=True)
        if shared:
            r = gb.spawn_threads(P, run_rank_topk, args, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank_topk, args, False, timeout_ms=300000)[0]
        print(f"{'expert_out':>10} {'composed ms':>12} {'topk ms':>9} {'speed-up':>9} {'MB/rank':>9}")
        for kind in ("symmetric", "plain"):
            c, t = r[f"composed_{kind}"], r[f"topk_{kind}"]
            print(f"{kind:>10} {c:12.3f} {t:9.3f} {c / t:9.2f} {r['bytes'] / 1e6:9.1f}", flush=True)
        print(json.dumps({"table": "topk_combine", "ranks": P, "shared_gpu": shared, **r}), flush=True)

    if "dispatch" in tables:
        print(f"# top-k dispatch ({label}{note}); median of {args.iters} calls (rank 0), arms alternating, "
              "outputs checked equal", flush=True)
        if shared:
            r = gb.spawn_threads(P, run_rank_dispatch_topk, args, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank_dispatch_topk, args, False, timeout_ms=300000)[0]
        print(f"{'arm':>14} {'composed ms':>12} {'topk ms':>9} {'speed-up':>9} {'MB avoided':>11}")
        for arm in ("dispatch_bf16", "dispatch_fp8", "layer_bf16"):
            c, t = r[f"{arm}_composed"], r[f"{arm}_topk"]
            print(f"{arm:>14} {c:12.3f} {t:9.3f} {c / t:9.2f} {r['bytes_avoided'] / 1e6:11.1f}", flush=True)
        print(json.dumps({"table": "topk_dispatch", "ranks": P, "shared_gpu": shared, **r}), flush=True)

    if "ll" in tables:
        print(f"# decode MoE layer, top-{args.topk}, hidden {args.hidden}, {args.experts} experts per rank ({label}{note}); "
              f"median of {args.iters} graph replays (rank 0, CUDA events), arms alternating, outputs checked equal",
              flush=True)
        if shared:
            r = gb.spawn_threads(P, run_rank_ll, args, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank_ll, args, False, timeout_ms=300000)[0]
        print(f"{'form':>6} {'T':>5} {'dev ms':>9} {'ll ms':>9} {'dev/ll':>8}")
        for form in ("bf16", "fp8"):
            for T in (1, 32, 128):
                d, ll = r[f"{form}_T{T}_dev"], r[f"{form}_T{T}_ll"]
                print(f"{form:>6} {T:>5} {d:9.3f} {ll:9.3f} {d / ll:8.2f}", flush=True)
        print(json.dumps({"table": "ll_layer", "ranks": P, "shared_gpu": shared, **r}), flush=True)

    if "backward" in tables:
        print(f"# top-k combine backward, bf16 ({label}{note}); median of {args.iters} calls (rank 0), arms "
              "alternating, grad_expert_out checked equal, grad_w within the fp32 summation bound", flush=True)
        if shared:
            r = gb.spawn_threads(P, run_rank_backward, args, True, cuda_device=0, timeout_ms=300000)[0]
        else:
            r = gb.spawn_threads(P, run_rank_backward, args, False, timeout_ms=300000)[0]
        print(f"{'tensors':>10} {'composed ms':>12} {'fused ms':>9} {'speed-up':>9} {'MB/rank':>9}")
        for kind in ("symmetric", "plain"):
            c, t = r[f"composed_{kind}"], r[f"fused_{kind}"]
            print(f"{kind:>10} {c:12.3f} {t:9.3f} {c / t:9.2f} {r['bytes'] / 1e6:9.1f}", flush=True)
        print(json.dumps({"table": "topk_combine_backward", "ranks": P, "shared_gpu": shared, **r}), flush=True)


if __name__ == "__main__":
    main()
