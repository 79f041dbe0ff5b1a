"""The top-k MoE kernels at the row widths, k and layer shapes they were written for, against CPU
references: the device-split top-k dispatch (copying and FP8), the top-k combine and its backward,
and the low-latency (LL) dispatch and combine. Ranks are threads sharing cuda:0, each on its own
stream. Every reference is computed on the CPU from the documented semantics and calls no kernel of
this project, so a bug in a device helper that the kernels share cannot cancel out.

Row widths are counted in 16-byte packs (PACKS) so that each kernel loop reaches its second unroll
slot, its second trip and a partial last trip: the copy push holds 4 packs per lane (128 per warp
step), the combine 2 (64 per step), the backward's dot and the LL combine 1 (32 per step). The FP8
push quantises 8 blocks of 128 elements per warp step (FP8_H: 1, 8, 9, 15 and 56 blocks)."""
from itertools import product

import numpy as np
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.parallel.strategies import MoEDispatcher
from test_moe_combine_topk import _pools, _reference, _route
from test_moe_dev import SENTINEL, _bytes, _layout, _ref_dispatch
from test_moe_dispatch_topk import DEFAULT_ALLTOALLV_BLOCKS, _fused, _out, _x
from test_moe_fp8_dispatch import _dequant, _quant, _ref as _fp8_ref_dispatch
from test_moe_topk_backward import GUARD, _grad_rows, _grad_w_tensor

PACKS = [1, 32, 33, 64, 65, 129, 256, 896, 897]  # 8 ... 7176 elements of a 16-bit type
FP8_H = [128, 1024, 1152, 1920, 7168]
KS = [1, 3, 4, 5, 8, 9, 31, 32]
K_PACKS = [33, 896]  # every k runs at these widths: 264 and 7168 elements of a 16-bit type
COMBINE_DTYPES = [torch.float32, torch.bfloat16, torch.float16]
ROW_DTYPES = COMBINE_DTYPES + [torch.uint8]
KINDS = ("symmetric", "registered", "plain")
POOL = 64 << 20  # bytes of each symmetric / registered pool per rank, and of the staging pool


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


def _width(dtype, packs):
    return packs * 16 // torch.empty((), dtype=dtype).element_size()


def _spawn(P, fn):
    assert all(gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=900000))


# ---- CPU references --------------------------------------------------------------------------
def fma32(a, b, c):
    """fp32 a * b + c with one rounding: the exact product in float64, the sum rounded to odd, then
    rounded once to fp32."""
    a, b, c = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a * b  # exact: 24 + 24 bits
    s = p + c
    bb = s - p
    err = (p - (s - bb)) + (c - bb)  # TwoSum: s + err == p + c exactly
    fix = (err != 0) & ((s.view(np.int64) & 1) == 0)
    s = np.where(fix, np.nextafter(s, np.where(err > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


def _grad_w_order(dy, rows, pos):
    """The backward's grad_w in its documented order, bit for bit: lane l of 32 runs fp32 fused
    multiply-adds over the elements of 16-byte packs l, l + 32, ... of dy[t] and the expert row
    rows[pos[t, j]] (each pack's elements in order), then a butterfly over lane distances 16, 8, 4,
    2, 1 adds the lanes and lane 0 holds the result; +0.0 where pos = -1."""
    T, k = pos.shape
    out = np.zeros((T, k), np.float32)
    ti, ji = (pos >= 0).nonzero(as_tuple=True)
    if ti.numel() == 0:
        return torch.from_numpy(out)
    per = 16 // dy.element_size()
    npk = dy.shape[1] // per
    trips = -(-npk // 32)
    pad = trips * 32 * per - dy.shape[1]
    a = torch.nn.functional.pad(dy.float()[ti], (0, pad)).numpy().reshape(-1, trips, 32, per)
    b = torch.nn.functional.pad(rows.float()[pos[ti, ji]], (0, pad)).numpy().reshape(-1, trips, 32, per)
    lanes = np.arange(32)
    part = np.zeros((a.shape[0], 32), np.float32)
    for v in range(trips):
        live = v * 32 + lanes < npk
        for i in range(per):
            part = np.where(live, fma32(a[:, v, :, i], b[:, v, :, i], part), part)
    for o in (16, 8, 4, 2, 1):
        part = part + part[:, lanes ^ o]
    out[ti.numpy(), ji.numpy()] = part[:, 0]
    return torch.from_numpy(out)


def _holder(inputs, sp, P, E, align, d, cap, fill):
    """Rank d's rows in the forward dispatch layout of every source's `inputs` (rows in (rank,
    expert) order, sp[s] their counts); `fill` in the alignment gaps and the tail."""
    osp, ooff, _ = _layout(sp, P, E, align, d)
    out = torch.full((cap, inputs[0].shape[1]), fill, dtype=inputs[0].dtype)
    for e in range(E):
        for s in range(P):
            c = d * E + e
            src, n = sum(sp[s][:c]), sp[s][c]
            out[ooff[e * P + s]:ooff[e * P + s] + n] = inputs[s][src:src + n]
    return out


def _ll_layout(idxs, P, E, M, j):
    """Holder j's LL dispatch from every source's topk_idx alone: for each local expert e, the
    (source, flat choice indices) whose rows fill out[e] in that order (source order, then token and
    choice), and out_splits (entry e * P + s). A (source, group) of more than M rows sends nothing
    and counts 0."""
    groups = [[] for _ in range(E)]
    osp = [0] * (E * P)
    for e in range(E):
        for s in range(P):
            chosen = (idxs[s].reshape(-1) == j * E + e).nonzero().flatten()
            if 0 < chosen.numel() <= M:
                osp[e * P + s] = chosen.numel()
                groups[e].append((s, chosen))
    return groups, osp


def _ll_sent(idx, G, M):
    """The choices of a source that the LL dispatch sends: routed, in a group of at most M rows."""
    flat = idx.reshape(-1)
    routed = (flat >= 0) & (flat < G)
    g = torch.where(routed, flat, torch.full_like(flat, G))
    counts = torch.bincount(g, minlength=G + 1)
    return (routed & (counts[g] <= M)).view(idx.shape)


def _expert_rows(g, rows):
    """A per-group 'expert', the same CPU expression for the holder's rows and for the reference:
    g is a group (rank * experts + e) or a column of groups."""
    g = torch.as_tensor(g, dtype=torch.float32)
    if g.dim():
        g = g[:, None]
    return (rows.float() * (0.75 + g / 32) - g / 16).to(rows.dtype)


def _ll_combine_ref(choice_rows, idx, sent, w, dtype):
    """y of the LL combine: _reference over each choice's expert row (row t * k + j of
    `choice_rows`) with pos restricted to the choices that were sent."""
    T, k = idx.shape
    pos = torch.where(sent, torch.arange(T * k).view(T, k), torch.full((T, k), -1))
    return _reference(choice_rows, pos, torch.ones(T, k) if w is None else w, dtype)


def _routing(P, E, k, seed, tmax):
    """Every rank's topk_idx: T in 2..tmax, -1 and out-of-range entries, token 0 with every choice
    unrouted and, for k >= 2, token 1 picking one expert twice (k > P * E forces more)."""
    g = torch.Generator().manual_seed(seed)
    G = P * E
    out = []
    for s in range(P):
        T = int(torch.randint(2, tmax + 1, (1,), generator=g))
        idx = torch.randint(0, G, (T, k), generator=g)
        r = torch.rand(T, k, generator=g)
        idx[r < 0.1] = -1
        idx[(r >= 0.1) & (r < 0.15)] = G + 2
        idx[0] = -1
        if k >= 2:
            idx[1, :2] = s % G
        out.append(idx)
    return out


def _fp8_x(T, H, g):
    """bf16 rows whose magnitude varies from row to row, so every block scale differs."""
    mag = torch.exp(torch.randn(T, 1, generator=g) * 3)
    return (torch.randn(T, H, generator=g) * mag).to(torch.bfloat16)


def _sentinel_out(T, width, dtype):
    y = torch.empty((T, width), dtype=dtype, device="cuda")
    y.view(torch.uint8).fill_(SENTINEL)
    return y


def _assert_zero_row(y, t, tag):
    """Token t has no routed choice: its row is +0 in every element."""
    assert bool((_bytes(y[t]) == 0).all()), tag


# ---- the device-split top-k dispatch -----------------------------------------------------------
def _dispatch_case(cc, pools, E, k, dtype, width, kind, seed, align=8, tmax=8):
    """alltoallv_dev_topk, copying: out against the CPU layout of route()'s rows (sentinel in the gaps
    and past the end), splits, pos, out_splits and out_offsets."""
    P, me = cc.size, cc.rank
    g = torch.Generator().manual_seed(seed)
    per = [(_x(i.shape[0], dtype, width, g), i) for i in _routing(P, E, k, seed, tmax)]
    routed = [_route(P, x, i, E) for x, i in per]
    sp = [r[1].tolist() for r in routed]
    cap = _layout(sp, P, E, align, me)[2] + 5
    x, idx = per[me]
    out = _out(kind, pools, 0, cap, dtype, width)
    splits, pos, osp, ooff = _fused(cc, out, x.cuda(), idx.cuda(), E, align)
    want, wsp, woff = _ref_dispatch([r[0] for r in routed], sp, P, E, align, me, cap)
    cc.synchronize()
    tag = (str(dtype), width, k, kind)
    assert torch.equal(_bytes(out), want), tag
    assert splits.tolist() == sp[me] and torch.equal(pos.cpu(), routed[me][2]), tag
    assert osp.tolist() == wsp and ooff.tolist() == woff, tag
    cc.pc.host_barrier()


def _dispatch_cases(slow):
    if slow:
        return [(dt, p, kind) for dt in ROW_DTYPES for p in PACKS for kind in KINDS]
    cases = [(torch.bfloat16, p, KINDS[c % 3]) for c, p in enumerate(PACKS)]
    cases += [(torch.float32, p, KINDS[c % 3]) for c, p in enumerate((33, 129, 897))]
    cases += [(torch.float16, 65, "plain"), (torch.float16, 256, "symmetric")]
    cases += [(torch.uint8, 33, "registered"), (torch.uint8, 897, "plain")]
    return cases


def _run_dispatch(P, slow):
    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=POOL)
        pools = _pools(cc, POOL)
        for c, (dtype, packs, kind) in enumerate(_dispatch_cases(slow)):
            _dispatch_case(cc, pools, 3, KS[c % len(KS)], dtype, _width(dtype, packs), kind, 1000 * P + c)
        return True

    _spawn(P, fn)


@pytest.mark.gpu
def test_dispatch_topk_widths():
    """The copying top-k dispatch at 1 to 897 packs a row (bfloat16 at every width, the other row
    types at a few), k cycling through 1..32, every kind of out."""
    _run_dispatch(2, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_dispatch_topk_widths_sweep(size):
    """Every row type x width x kind of out."""
    _run_dispatch(size, slow=True)


def _fp8_dispatch_case(cc, pools, E, k, H, kind, seed, align=4, tmax=8):
    """alltoallv_dev_topk, quantising: codes and scales against _quant of the routed rows in the CPU
    layout, byte for byte, and the index outputs."""
    P, me = cc.size, cc.rank
    g = torch.Generator().manual_seed(seed)
    per = [(_fp8_x(i.shape[0], H, g), i) for i in _routing(P, E, k, seed, tmax)]
    routed = [_route(P, x, i, E) for x, i in per]
    sp = [r[1].tolist() for r in routed]
    cap = _layout(sp, P, E, align, me)[2] + 3
    x, idx = per[me]
    codes = _out(kind, pools, 0, cap, torch.float8_e4m3fn, H)
    scales = _out(kind, pools, 1, cap, torch.float32, H // 128)
    splits, pos, osp, ooff = _fused(cc, codes, x.cuda(), idx.cuda(), E, align, out_scales=scales)
    wc, ws, wsp, woff = _fp8_ref_dispatch([r[0] for r in routed], sp, P, E, align, me, cap)
    cc.synchronize()
    tag = (H, k, kind)
    assert torch.equal(_bytes(codes), wc) and torch.equal(_bytes(scales), ws), tag
    assert splits.tolist() == sp[me] and torch.equal(pos.cpu(), routed[me][2]), tag
    assert osp.tolist() == wsp and ooff.tolist() == woff, tag
    cc.pc.host_barrier()


def _run_fp8_dispatch(P, slow):
    cases = [(H, kind) for H in FP8_H for kind in KINDS] if slow else \
        [(H, KINDS[c % 3]) for c, H in enumerate(FP8_H)]

    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=POOL)
        pools = _pools(cc, POOL)
        for c, (H, kind) in enumerate(cases):
            _fp8_dispatch_case(cc, pools, 3, KS[(c + 3) % len(KS)], H, kind, 2000 * P + c)
        return True

    _spawn(P, fn)


@pytest.mark.gpu
def test_fp8_dispatch_topk_widths():
    """The quantising top-k dispatch at 1, 8, 9, 15 and 56 blocks a row."""
    _run_fp8_dispatch(2, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_fp8_dispatch_topk_widths_sweep(size):
    """Every FP8 width x kind of out."""
    _run_fp8_dispatch(size, slow=True)


# ---- the device-split top-k combine and its backward ----------------------------------------------
def _pull_setup(P, E, k, dtype, width, seed, tmax=8):
    """Every rank's routing (route() on the CPU), dispatch-input rows (the expert outputs), gate
    weights (negative ones included) and dy."""
    g = torch.Generator().manual_seed(seed)
    per = []
    for idx in _routing(P, E, k, seed, tmax):
        T = idx.shape[0]
        _, splits, pos = _route(P, torch.zeros(T, 1), idx, E)
        n = int(splits.sum())
        per.append(dict(splits=splits, pos=pos, rows=_x(n, dtype, width, g), w=torch.rand(T, k, generator=g) * 2 - 0.5,
                        dy=_x(T, dtype, width, g)))
    return per


def _expert_out(cc, kind, pools, half, per, E, align, extra):
    """This rank's expert_out in the dispatch layout of every rank's rows, NaN in every row that no
    choice names (the alignment gaps and `extra` rows of tail). Returns (tensor, cap, CPU copy)."""
    P, me = cc.size, cc.rank
    sp = [p["splits"].tolist() for p in per]
    cap = _layout(sp, P, E, align, me)[2] + extra
    rows = [p["rows"] for p in per]
    want = _holder(rows, sp, P, E, align, me, cap, float("nan"))
    eo = _out(kind, pools, half, cap, want.dtype, want.shape[1])
    eo.copy_(want.cuda())
    return eo, cap, want


def _combine_case(cc, pools, E, k, dtype, width, kind, weighted, seed, align=8):
    """alltoallv_dev_combine_topk against _reference; NaN in every expert_out row that no choice
    names, which must not reach out."""
    me = cc.rank
    per = _pull_setup(cc.size, E, k, dtype, width, seed)
    d = per[me]
    T = d["pos"].shape[0]
    eo, _, eo_cpu = _expert_out(cc, kind, pools, 0, per, E, align, 3)
    out = _sentinel_out(T, width, dtype)
    w = d["w"] if weighted else None
    cc.alltoallv_dev_combine_topk(out, eo, d["splits"].cuda(), d["pos"].cuda(), None if w is None else w.cuda(),
                                  experts=E, align=align)
    want = _reference(d["rows"], d["pos"], torch.ones(T, k) if w is None else w, dtype)
    cc.synchronize()
    tag = (str(dtype), width, k, kind, weighted)
    assert torch.equal(_bytes(out), _bytes(want)), tag
    assert not bool(out.isnan().any()), tag
    _assert_zero_row(out, 0, tag)
    assert torch.equal(_bytes(eo), _bytes(eo_cpu)), tag
    cc.pc.host_barrier()


def _pull_cases(slow):
    """(dtype, packs, k, kind, weighted): every width, then every k at the K_PACKS widths."""
    if slow:
        cases = [(dt, p, KS[c % len(KS)], kind, wt) for c, (dt, p, kind, wt) in
                 enumerate(product(COMBINE_DTYPES, PACKS, KINDS, (True, False)))]
        return cases + [(dt, p, k, KINDS[c % 3], c % 2 == 0) for c, (dt, p, k) in
                        enumerate(product(COMBINE_DTYPES, K_PACKS, KS))]
    cases = [(torch.bfloat16, p, 8, KINDS[c % 3], c % 2 == 0) for c, p in enumerate(PACKS)]
    cases += [(dt, p, 4, KINDS[c % 3], c % 2 == 1) for c, (dt, p) in
              enumerate(product((torch.float32, torch.float16), (33, 65, 129, 897)))]
    return cases + [(torch.bfloat16, p, k, KINDS[c % 3], c % 2 == 0) for c, (p, k) in
                    enumerate(product(K_PACKS, KS))]


def _run_combine(P, slow):
    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=POOL)
        pools = _pools(cc, POOL)
        for c, (dtype, packs, k, kind, weighted) in enumerate(_pull_cases(slow)):
            _combine_case(cc, pools, 3, k, dtype, _width(dtype, packs), kind, weighted, 3000 * P + c)
        return True

    _spawn(P, fn)


@pytest.mark.gpu
def test_combine_topk_widths():
    """The top-k combine at 1 to 897 packs a row and every k at 264 and 7168 bfloat16 elements, with
    weights and with None, every kind of expert_out."""
    _run_combine(2, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_combine_topk_widths_sweep(size):
    """Every dtype x width x kind x weights, and every k at both K_PACKS widths for every dtype."""
    _run_combine(size, slow=True)


def _backward_case(cc, pools, E, k, dtype, width, kind, seed, align=8, exact=False):
    """alltoallv_dev_combine_topk_backward: grad_w bit for bit against its documented order (random
    inputs) or the exact dot (inputs whose every partial sum is exact), grad_expert_out against the
    pushed rows in the holder layout (+0 in the gaps and the tail), guard rows untouched, NaN in
    every expert_out row that no choice names."""
    P, me = cc.size, cc.rank
    per = _pull_setup(P, E, k, dtype, width, seed)
    if exact:
        g = torch.Generator().manual_seed(seed + 1)
        for p in per:
            p["rows"] = (torch.randint(-8, 9, p["rows"].shape, generator=g).float() * 0.5).to(dtype)
            p["dy"] = (torch.randint(-8, 9, p["dy"].shape, generator=g).float() * 0.25).to(dtype)
    for p in per:
        n = p["rows"].shape[0]
        gr = _grad_rows(p["dy"], p["pos"], p["w"], dtype)
        assert len(gr) == n and all(r is not None for r in gr)
        p["grad_rows"] = torch.stack(gr) if n else torch.empty(0, width, dtype=dtype)
    d = per[me]
    T = d["pos"].shape[0]
    eo, cap, eo_cpu = _expert_out(cc, kind, pools, 0, per, E, align, 2)
    geo_full = _out(kind, pools, 1, cap + GUARD, dtype, width)
    geo = geo_full[:cap]
    gw_full, gw = _grad_w_tensor(T, k)
    cc.alltoallv_dev_combine_topk_backward(geo, gw, d["dy"].cuda(), eo, d["splits"].cuda(), d["pos"].cuda(),
                                           d["w"].cuda(), experts=E, align=align)
    sp = [p["splits"].tolist() for p in per]
    want_geo = _holder([p["grad_rows"] for p in per], sp, P, E, align, me, cap, 0.0)
    want_gw = _grad_w_order(d["dy"], d["rows"], d["pos"])
    if exact:
        m = d["pos"] >= 0
        dots = (d["dy"].double()[:, None, :] * d["rows"].double()[d["pos"].clamp(min=0)]).sum(-1)
        assert torch.equal(want_gw[m], dots[m].float())
    cc.synchronize()
    tag = (str(dtype), width, k, kind, exact)
    assert torch.equal(_bytes(geo), _bytes(want_geo)), tag
    assert bool((_bytes(geo_full[cap:]) == SENTINEL).all()), tag
    assert torch.equal(_bytes(gw), _bytes(want_gw)), tag
    assert bool((_bytes(gw_full[T * k:]) == SENTINEL).all()), tag
    assert torch.equal(_bytes(eo), _bytes(eo_cpu)), tag
    cc.pc.host_barrier()


def _run_backward(P, slow):
    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=POOL)
        pools = _pools(cc, POOL)
        for c, (dtype, packs, k, kind, _) in enumerate(_pull_cases(slow)):
            _backward_case(cc, pools, 3, k, dtype, _width(dtype, packs), kind, 4000 * P + c)
        _backward_case(cc, pools, 3, 8, torch.bfloat16, _width(torch.bfloat16, 897), "symmetric", 4999, exact=True)
        return True

    _spawn(P, fn)


@pytest.mark.gpu
def test_combine_topk_backward_widths():
    """The combine's backward at 1 to 897 packs a row and every k at 264 and 7168 bfloat16 elements,
    every kind of expert_out, random inputs against the emulated order, and one exact-input case."""
    _run_backward(2, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_combine_topk_backward_widths_sweep(size):
    """Every dtype x width x kind, and every k at both K_PACKS widths for every dtype."""
    _run_backward(size, slow=True)


# ---- the low-latency dispatch and combine -------------------------------------------------------------
class _LLRef:
    """Everything one rank expects of an LL dispatch + combine, from every rank's x and topk_idx."""

    def __init__(self, xs, idxs, P, E, M, me, fp8):
        k = idxs[me].shape[1]
        groups, self.osp = _ll_layout(idxs, P, E, M, me)
        self.counts = [sum(self.osp[e * P:(e + 1) * P]) for e in range(E)]
        # what each source sends, and what its experts see
        if fp8:
            q = [_quant(x) for x in xs]
            seen = [_dequant(c, s) for c, s in q]
        else:
            seen = xs
        self.out = [torch.cat([(q[s][0] if fp8 else xs[s])[ch // k] for s, ch in groups[e]])
                    if groups[e] else None for e in range(E)]
        self.scales = [torch.cat([q[s][1][ch // k] for s, ch in groups[e]]) if fp8 and groups[e] else None
                       for e in range(E)]
        self.expert = [_expert_rows(me * E + e, torch.cat([seen[s][ch // k] for s, ch in groups[e]]))
                       if groups[e] else None for e in range(E)]
        idx = idxs[me]
        self.sent = _ll_sent(idx, P * E, M)
        flat = idx.reshape(-1)
        self.choice_rows = _expert_rows(torch.where(self.sent.reshape(-1), flat, torch.zeros_like(flat)),
                                        seen[me].repeat_interleave(k, 0))

    def want_bytes(self, E, rows, width, dtype, parts):
        """The expected (E, rows, width) tensor as bytes on the device: `parts[e]` then the sentinel."""
        es = torch.empty((), dtype=dtype).element_size()
        want = torch.full((E, rows, width * es), SENTINEL, dtype=torch.uint8, device="cuda")
        for e in range(E):
            if parts[e] is not None:
                want[e, :parts[e].shape[0]] = parts[e].contiguous().view(torch.uint8).view(-1, width * es).cuda()
        return want


def _ll_run(cc, moe, buf, ref, x, idx, w, out, scales, tag, raises=None):
    """One LL dispatch + combine on `buf`, checked against `ref`: out (and scales) byte for byte with
    the sentinel past each count, out_splits, x unchanged, then y from an expert_out whose rows past
    each count are NaN."""
    E, M, H, P = buf.experts, buf.max_tokens, buf.hidden, cc.size
    x0 = _bytes(x)
    out.view(torch.uint8).fill_(SENTINEL)
    if scales is not None:
        scales.view(torch.uint8).fill_(SENTINEL)
        _, _, osp = moe.dispatch_ll(x, idx, buf, out, out_scales=scales)
    else:
        _, osp = moe.dispatch_ll(x, idx, buf, out)
    if raises is not None:
        with pytest.raises(ValueError, match=raises):
            cc.synchronize()
    cc.synchronize()
    assert torch.equal(out.view(torch.uint8), ref.want_bytes(E, P * M, H, out.dtype, ref.out)), tag
    if scales is not None:
        assert torch.equal(scales.view(torch.uint8), ref.want_bytes(E, P * M, H // 128, torch.float32, ref.scales)), tag
    assert osp.tolist() == ref.osp, tag
    assert torch.equal(_bytes(x), x0), tag
    cdt = torch.bfloat16 if buf.fp8 else buf.dtype
    if cdt not in COMBINE_DTYPES:
        return
    eo = torch.full((E, P * M, H), float("nan"), dtype=cdt, device="cuda")
    for e in range(E):
        if ref.expert[e] is not None:
            eo[e, :ref.counts[e]] = ref.expert[e].cuda()
    y = _sentinel_out(x.shape[0], H, cdt)
    moe.combine_ll(eo, None if w is None else w.cuda(), buf, y)
    want = _ll_combine_ref(ref.choice_rows, idx.cpu(), ref.sent, w, cdt)
    cc.synchronize()
    assert torch.equal(_bytes(y), _bytes(want)), tag
    assert not bool(y.isnan().any()), tag
    return y


def _ll_case(cc, moe, pools, E, k, dtype, width, fp8, kind, weighted, seed, tmax=8):
    """An LL layer at one width: max_tokens is the fullest (source, group) or the most tokens, so
    some group fills its slots exactly."""
    P, me = cc.size, cc.rank
    G = P * E
    g = torch.Generator().manual_seed(seed)
    idxs = _routing(P, E, k, seed, tmax)
    xs = [_fp8_x(i.shape[0], width, g) if fp8 else _x(i.shape[0], dtype, width, g) for i in idxs]
    fullest = max(int(torch.bincount(torch.where((i >= 0) & (i < G), i, G).reshape(-1), minlength=G + 1)[:G].max())
                  for i in idxs)
    M = max(max(i.shape[0] for i in idxs), fullest)
    buf = cc.moe_ll_buffer(E, M, k, width, dtype=dtype, fp8=fp8)
    odt = torch.float8_e4m3fn if fp8 else dtype
    out = _out(kind, pools, 0, E * P * M, odt, width).view(E, P * M, width)
    scales = _out(kind, pools, 1, E * P * M, torch.float32, width // 128).view(E, P * M, width // 128) if fp8 else None
    ref = _LLRef(xs, idxs, P, E, M, me, fp8)
    w = torch.rand(idxs[me].shape, generator=torch.Generator().manual_seed(seed + me)) * 2 - 0.5 if weighted else None
    tag = (str(dtype), width, k, fp8, kind, weighted)
    y = _ll_run(cc, moe, buf, ref, xs[me].cuda(), idxs[me].cuda(), w, out, scales, tag)
    if y is not None:
        _assert_zero_row(y, 0, tag)
    cc.synchronize()
    cc.pc.host_barrier()


def _ll_cases(slow):
    """(dtype, packs or FP8 H, k, fp8, kind, weighted)."""
    if slow:
        cases = [(dt, p, KS[c % len(KS)], False, kind, c % 2 == 0) for c, (dt, p, kind) in
                 enumerate(product(ROW_DTYPES, PACKS, KINDS))]
        cases += [(dt, p, k, False, KINDS[c % 3], c % 2 == 0) for c, (dt, p, k) in
                  enumerate(product(COMBINE_DTYPES, K_PACKS, KS))]
        return cases + [(torch.bfloat16, H, k, True, KINDS[c % 3], c % 2 == 0) for c, (H, k) in
                        enumerate(product(FP8_H, (1, 8, 32)))]
    cases = [(torch.bfloat16, p, 4, False, KINDS[c % 3], c % 2 == 0) for c, p in enumerate(PACKS)]
    cases += [(dt, p, 3, False, KINDS[c % 3], c % 2 == 1) for c, (dt, p) in
              enumerate(product((torch.float32, torch.float16), (33, 129, 897)))]
    cases += [(torch.uint8, 33, 5, False, "plain", False), (torch.uint8, 897, 9, False, "symmetric", False)]
    cases += [(torch.bfloat16, p, k, False, KINDS[c % 3], c % 2 == 0) for c, (p, k) in
              enumerate(product(K_PACKS, KS))]
    return cases + [(torch.bfloat16, H, KS[c + 2], True, KINDS[c % 3], c % 2 == 0) for c, H in enumerate(FP8_H)]


def _run_ll(P, slow):
    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=32 << 20)
        moe = MoEDispatcher(ctx, cc)
        pools = _pools(cc, POOL)
        for c, (dtype, packs, k, fp8, kind, weighted) in enumerate(_ll_cases(slow)):
            width = packs if fp8 else _width(dtype, packs)
            _ll_case(cc, moe, pools, 3, k, dtype, width, fp8, kind, weighted, 5000 * P + c)
        return True

    _spawn(P, fn)


@pytest.mark.gpu
def test_ll_widths():
    """The LL dispatch (copying and FP8) and combine at 1 to 897 packs a row, every k at 264 and 7168
    bfloat16 elements and the FP8 widths, against the CPU layout built from topk_idx alone and the
    CPU combine; out symmetric, registered or plain."""
    _run_ll(2, slow=False)


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", [2, 3, 4])
def test_ll_widths_sweep(size):
    """Every row type x width x kind of out, every k at both K_PACKS widths for every combine dtype,
    and the FP8 widths at k = 1, 8 and 32."""
    _run_ll(size, slow=True)


def _decode_routing(case, P, E, k, M, seed):
    """Every rank's topk_idx for one decode case, and the (source, group) that overflows, if any.
      random      T = M, random groups (repeats included), -1 entries, token 0 unrouted
      full        T = M, every token picks the same k distinct groups: each holds exactly M rows
      duplicates  T = M / 2, every token picks one group twice and never otherwise: exactly M rows
      overflow    as full on the last rank; rank 0 sends M + 1 rows to the last group, whose
                  holder also receives exactly M rows from the last rank"""
    g = torch.Generator().manual_seed(seed)
    G = P * E
    out = []
    for s in range(P):
        if case == "random":
            idx = torch.randint(0, G, (M, k), generator=g)
            idx[torch.rand(M, k, generator=g) < 0.1] = -1
            idx[0] = -1
        elif case == "full" or (case == "overflow" and s == P - 1):
            picks = (torch.arange(k) * (G // k) + s) % G if case == "full" else (torch.arange(k) + G - k) % G
            idx = picks.repeat(M, 1)
        elif case == "duplicates":
            g0 = (3 * s + 1) % G
            idx = torch.randint(0, G - 1, (M // 2, k), generator=g)
            idx = idx + (idx >= g0).long()
            idx[:, :2] = g0
        else:  # overflow, rank < P - 1
            idx = torch.randint(0, G - 1, (M, k), generator=g)
            if s == 0:
                idx[:, 0] = G - 1
                idx[0, 1] = G - 1
        out.append(idx)
    return out, ((0, G - 1) if case == "overflow" else None)


@pytest.mark.gpu
@pytest.mark.parametrize("P,E", [(2, 32), (8, 4)])
def test_ll_decode_layer(P, E):
    """A decode-sized LL layer, T = max_tokens = 128, k = 8, H = 7168, bfloat16 and FP8, at grids of 1,
    3 and 64 CTAs (tokens straddle CTA slices): random routing, groups filled to exactly max_tokens
    (by T = max_tokens and by repeated picks) and max_tokens + 1 rows, which raises on the source and
    on the holder while every other group is served. Every grid gives the CPU reference's bytes."""
    M, k, H = 128, 8, 7168
    G = P * E

    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=8 << 20)
        moe = MoEDispatcher(ctx, cc)
        me = cc.rank
        try:
            for fp8 in (False, True):
                buf = cc.moe_ll_buffer(E, M, k, H, fp8=fp8)
                out = torch.empty((E, P * M, H), dtype=torch.float8_e4m3fn if fp8 else torch.bfloat16, device="cuda")
                scales = torch.empty((E, P * M, H // 128), device="cuda") if fp8 else None
                for c, case in enumerate(("random", "full", "duplicates", "overflow")):
                    idxs, over = _decode_routing(case, P, E, k, M, 60 + c)
                    g = torch.Generator().manual_seed(70 + c)
                    xs = [_fp8_x(i.shape[0], H, g) for i in idxs]
                    ref = _LLRef(xs, idxs, P, E, M, me, fp8)
                    w = torch.rand(idxs[me].shape, generator=torch.Generator().manual_seed(80 + me)) * 2 - 0.5
                    raises = None
                    if over is not None and me in (over[0], over[1] // E):
                        raises = f"source rank {over[0]} routed {M + 1} rows to expert {over[1]} .*max_tokens = {M}"
                    x, idx = xs[me].cuda(), idxs[me].cuda()
                    for n in (1, 3, 64):
                        cc.pc.host_barrier()
                        if me == 0:
                            gb._C.cuda.set_tuning({"alltoallv_blocks": n})
                        cc.pc.host_barrier()
                        y = _ll_run(cc, moe, buf, ref, x, idx, w, out, scales, (fp8, case, n), raises=raises)
                        if case == "random":
                            _assert_zero_row(y, 0, (fp8, case, n))
                del buf
                cc.synchronize()
                cc.pc.host_barrier()
        finally:
            cc.pc.host_barrier()
            if me == 0:
                gb._C.cuda.set_tuning({"alltoallv_blocks": DEFAULT_ALLTOALLV_BLOCKS})
            cc.pc.host_barrier()
        return True

    _spawn(P, fn)


# ---- 16-bit value edges in both combines ----------------------------------------------------------
def _edge_x(T, width, g):
    """float16 rows mixing subnormals, values near the top of the range, signed zeros and ordinary
    values; row 1 negative, rows 2 and 3 at +-60000 (their weighted sums overflow to +-inf)."""
    pick = torch.randint(0, 5, (T, width), generator=g)
    base = torch.randn(T, width, generator=g)
    sub = torch.randint(-1023, 1024, (T, width), generator=g).float() * 2.0 ** -24
    big = torch.where(base >= 0, 60000.0, -60000.0)
    zero = torch.where(base >= 0, 0.0, -0.0)
    x = torch.where(pick == 0, sub, torch.where(pick == 1, big, torch.where(pick == 2, zero, base)))
    x[1] = -(x[1].abs() + 2.0 ** -20)
    x[2] = 60000.0
    x[3] = -60000.0
    return x.to(torch.float16)


def _edge_weights(T, k, g):
    """Negative, +-0 and ordinary weights; token 1 weighs every choice 0, tokens 2 and 3 use 2."""
    choices = torch.tensor([-1.0, 0.0, -0.0, 0.5, 2.0, -2.0, 1.5, 0.25])
    w = choices[torch.randint(0, len(choices), (T, k), generator=g)]
    w[1] = torch.tensor([0.0, -0.0] * (k // 2))
    w[2:4] = 2.0
    return w


@pytest.mark.gpu
def test_combine_fp16_value_edges():
    """float16 rows with subnormals, sums that overflow to +-inf, negative and zero weights, zero
    weights times negative rows (+0 out): the device-split combine (rows no choice names are NaN)
    and the LL combine (identity experts, rows past each count NaN) equal the CPU reference."""
    P, E, k, T, align = 2, 2, 4, 12, 8
    width = _width(torch.float16, 65)
    dtype = torch.float16
    G = P * E

    def fn(ctx):
        cc = _cuda().CudaContext(ctx, 0, stage_bytes=POOL)
        moe = MoEDispatcher(ctx, cc)
        me = cc.rank
        per = []
        for s in range(P):
            g = torch.Generator().manual_seed(90 + s)
            idx = torch.randint(0, G, (T, k), generator=g)
            idx[4:][torch.rand(T - 4, k, generator=g) < 0.2] = -1
            idx[0] = -1
            per.append((_edge_x(T, width, g), idx, _edge_weights(T, k, g)))
        x, idx, w = per[me]

        def check(y, want, tag):
            assert torch.equal(_bytes(y), _bytes(want)), tag
            assert not bool(y.isnan().any()), tag
            assert bool(y[2].isinf().any()) and bool(y[3].isinf().any()), tag
            yc = y.cpu().float()
            assert bool(((yc != 0) & (yc.abs() < 2.0 ** -14)).any()), tag  # subnormal results
            _assert_zero_row(y, 0, tag)
            _assert_zero_row(y, 1, tag)

        # device-split: the routed rows are the expert outputs
        routed = [_route(P, xs, i, E) for xs, i, _ in per]
        sp = [r[1].tolist() for r in routed]
        cap = _layout(sp, P, E, align, me)[2] + 3
        eo = _holder([r[0] for r in routed], sp, P, E, align, me, cap, float("nan")).cuda()
        y = _sentinel_out(T, width, dtype)
        moe.combine_dev_topk(eo, routed[me][1].cuda(), routed[me][2].cuda(), w.cuda(), y, experts=E, align=align)
        want = _reference(routed[me][0], routed[me][2], w, dtype)
        cc.synchronize()
        check(y, want, "device-split")
        cc.pc.host_barrier()

        # LL: the dispatched rows are the expert outputs
        buf = cc.moe_ll_buffer(E, T * k, k, width, dtype=dtype)
        out = torch.empty((E, P * T * k, width), dtype=dtype, device="cuda")
        moe.dispatch_ll(x.cuda(), idx.cuda(), buf, out)
        cc.synchronize()
        counts = [sum(_ll_layout([i for _, i, _ in per], P, E, T * k, me)[1][e * P:(e + 1) * P]) for e in range(E)]
        eo = torch.full_like(out, float("nan"))
        for e in range(E):
            eo[e, :counts[e]] = out[e, :counts[e]]
        y = _sentinel_out(T, width, dtype)
        moe.combine_ll(eo, w.cuda(), buf, y)
        want = _ll_combine_ref(x.repeat_interleave(k, 0), idx, _ll_sent(idx, G, T * k), w, dtype)
        cc.synchronize()
        check(y, want, "LL")
        cc.pc.host_barrier()
        return True

    _spawn(P, fn)


# ---- the references themselves, on the CPU ------------------------------------------------------------
def test_references_cpu():
    """fma32 is a correctly rounded fp32 fused multiply-add (against exact rational arithmetic, with
    cancelling triples); the emulated backward order equals the exact dot on exact inputs and, on
    random ones, differs from a plain sequential fp32 sum, so a different order cannot pass; the LL
    layout built from topk_idx alone equals route()'s layout at align 1 when no group overflows, and
    drops exactly the overflowing groups when one does."""
    from fractions import Fraction

    rng = np.random.default_rng(7)
    a = (rng.standard_normal(4000) * np.exp2(rng.integers(-20, 20, 4000))).astype(np.float32)
    b = (rng.standard_normal(4000) * np.exp2(rng.integers(-20, 20, 4000))).astype(np.float32)
    c = (rng.standard_normal(4000) * np.exp2(rng.integers(-40, 40, 4000))).astype(np.float32)
    c[::4] = -(a[::4].astype(np.float64) * b[::4]).astype(np.float32)  # cancellation
    got = fma32(a, b, c)
    for i in range(len(a)):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        lo = np.float32(float(exact))
        # the correctly rounded fp32 value: the nearer of the two fp32 neighbours of `exact`, even on a tie
        cands = [np.nextafter(lo, np.float32(-np.inf)), lo, np.nextafter(lo, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, (a[i], b[i], c[i])

    g = torch.Generator().manual_seed(3)
    T, k, W = 6, 3, _width(torch.bfloat16, 897)
    pos = torch.tensor([[0, -1, 1], [2, 3, 4], [-1, -1, -1], [5, 6, 7], [8, 9, 10], [11, 12, 13]])
    dy = (torch.randint(-8, 9, (T, W), generator=g).float() * 0.25).to(torch.bfloat16)
    rows = (torch.randint(-8, 9, (14, W), generator=g).float() * 0.5).to(torch.bfloat16)
    gw = _grad_w_order(dy, rows, pos)
    dots = (dy.double()[:, None, :] * rows.double()[pos.clamp(min=0)]).sum(-1).float()
    assert torch.equal(gw[pos >= 0], dots[pos >= 0]) and bool((gw[pos < 0] == 0).all())
    dy, rows = torch.randn(T, W, generator=g).to(torch.bfloat16), torch.randn(14, W, generator=g).to(torch.bfloat16)
    gw = _grad_w_order(dy, rows, pos)
    seq = torch.zeros(T, k)
    prod = dy.float()[:, None, :] * rows.float()[pos.clamp(min=0)]
    for h in range(W):
        seq = seq + prod[:, :, h]
    assert not torch.equal(gw[pos >= 0], seq[pos >= 0])

    P, E, kk, M = 3, 2, 4, 40
    idxs = _routing(P, E, kk, 11, 10)
    for j in range(P):
        groups, osp = _ll_layout(idxs, P, E, M, j)
        sp = [_route(P, torch.zeros(i.shape[0], 1), i, E)[1].tolist() for i in idxs]
        assert osp == _layout(sp, P, E, 1, j)[0]
        for e in range(E):
            for s, ch in groups[e]:
                assert bool((idxs[s].reshape(-1)[ch] == j * E + e).all())
    for s in range(P):
        r = _route(P, torch.zeros(idxs[s].shape[0], 1), idxs[s], E)[2]
        assert torch.equal(_ll_sent(idxs[s], P * E, M), r >= 0)
    over = [i.clone() for i in idxs]
    over[0][:, 0] = 1  # rank 0 sends at least T rows to group 1
    M = int((over[0] == 1).sum()) - 1
    groups, osp = _ll_layout(over, P, E, M, 0)
    assert osp[1 * P + 0] == 0 and all(s != 0 for s, _ in groups[1])
    sent = _ll_sent(over[0], P * E, M)
    assert not bool(sent[over[0] == 1].any())
