"""Bit-exact checks of every reducing kernel against an order-free reference.

The contract (DESIGN.md, docs/cuda.md): 16-bit and FP8 buffers accumulate in fp32, the scale is
applied to the fp32 accumulator and the result is rounded once; every rank holds the same bytes.
A tolerance cannot tell one rounding from one per combine, so the inputs here are chosen such that
their exact sum (or product, min, max) is representable in fp32 for every summation order. The
contract then gives exactly one answer, which the reference computes from an fp64 reduction
without copying any kernel's summation order, and results are compared byte for byte.

Every rank draws every rank's input from CPU generators seeded by (case, rank), so each rank
computes the whole reference itself. Ranks are threads sharing cuda:0, as in the other GPU tests.
Cases are collected per rank and reported together, so one run lists every path that fails.
"""
import itertools
import math
import zlib

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu

E4M3, E5M2 = torch.float8_e4m3fn, torch.float8_e5m2
FP8 = (E4M3, E5M2)
HALF = (torch.bfloat16, torch.float16)
MAIN = (torch.float32, torch.bfloat16, torch.float16)  # the full product runs on these
OTHER = (E4M3, E5M2, torch.float64, torch.int32, torch.int64, torch.uint8, torch.int8)
SIZES = [2, 3, 4, 5, 8]  # 2 / 4 / 8 take the P-specialised instantiations, 3 / 5 the generic ones
OPS = {"sum": gb.ReduceOp.SUM, "prod": gb.ReduceOp.PRODUCT, "min": gb.ReduceOp.MIN, "max": gb.ReduceOp.MAX}
# 1 MiB pool (bulk region ~512 KiB): the multi-CTA counts of the plain reduce_scatter and reduce
# stream through the pipelined kernels, smaller ones are staged whole
STAGE = 1 << 20
BIG = 300_001  # a multi-CTA count, odd


def _es(dtype):
    return torch.empty((), dtype=dtype).element_size()


def _floating(dtype):
    return dtype.is_floating_point


# ---- order-free inputs ---------------------------------------------------------------------------

# SUM values are m * 2^e with |m| < 2^bits and e in [elo, 0]. The exact sum of up to 16 of them
# (8 ranks x 2 local pointers) needs at most bits + 4 - elo + 1 significant bits: 19 (bf16), 21
# (f16) and 24 (f32) -- always exact in fp32, whatever the order, yet far more than the 8 / 11
# significant bits of bf16 / f16, so a kernel that rounds after each combine gives other bytes.
_SUM_SHAPE = {torch.bfloat16: (7, -7), torch.float16: (10, -6), torch.float32: (15, -4), torch.float64: (15, -4)}


def _gen(case, r):
    return torch.Generator().manual_seed(zlib.crc32(repr(case).encode()) * 64 + r)


def _sum_values(dtype, n, g):
    if dtype in _SUM_SHAPE:
        bits, elo = _SUM_SHAPE[dtype]
        m = torch.randint(-(1 << bits) + 1, 1 << bits, (n,), generator=g, dtype=torch.float64)
        e = torch.randint(elo, 1, (n,), generator=g, dtype=torch.float64)
        return (m * torch.pow(2.0, e)).to(dtype)
    if dtype == E4M3:
        # any finite code: fp32 holds any sum of up to 16 e4m3 values (exponents 2^-9 .. 2^8)
        codes = torch.randint(0, 255, (n,), generator=g, dtype=torch.int64)
        codes = torch.where(codes == 0x7F, torch.zeros_like(codes), codes)  # 0x7f / 0xff are NaN
        return codes.to(torch.uint8).view(E4M3)
    if dtype == E5M2:
        # zero or +-{1, 1.25, 1.5, 1.75} * 2^e, e in [-6, 10] (docs/cuda.md, "FP8 numerics")
        m = torch.randint(4, 8, (n,), generator=g, dtype=torch.float64) / 4
        e = torch.randint(-6, 11, (n,), generator=g, dtype=torch.float64)
        s = torch.randint(0, 2, (n,), generator=g, dtype=torch.float64) * 2 - 1
        z = torch.randint(0, 8, (n,), generator=g) == 0
        return torch.where(z, torch.zeros(n, dtype=torch.float64), s * m * torch.pow(2.0, e)).to(E5M2)
    if dtype == torch.int32:
        return torch.randint(-(1 << 26), 1 << 26, (n,), generator=g, dtype=torch.int32)
    if dtype == torch.int64:
        # near 2^59 / 16: exact in int64, not in a double (53 bits)
        return (1 << 55) + torch.randint(-(1 << 20), 1 << 20, (n,), generator=g, dtype=torch.int64)
    if dtype == torch.uint8:
        return torch.randint(0, 256, (n,), generator=g, dtype=torch.uint8)  # the sum wraps mod 256
    if dtype == torch.int8:
        return torch.randint(-8, 8, (n,), generator=g, dtype=torch.int8)
    raise AssertionError(dtype)


def _values(op, dtype, n, g):
    if op == "prod":
        # +-2^k * {1, 1.25, 1.5, 1.75}, |k| <= 2: any product of up to 8 is exact in fp32
        m = torch.randint(4, 8, (n,), generator=g, dtype=torch.float64) / 4
        k = torch.randint(-2, 3, (n,), generator=g, dtype=torch.float64)
        s = torch.randint(0, 2, (n,), generator=g, dtype=torch.float64) * 2 - 1
        return (s * m * torch.pow(2.0, k)).to(dtype)
    x = _sum_values(dtype, n, g)
    if op in ("min", "max") and _floating(dtype):
        # no +-0: which zero MIN / MAX return is order dependent
        x = torch.where(x.double() == 0, torch.ones((), dtype=dtype), x)
    return x


def _combine(xs, op):
    """The exact reduction of the rank inputs: fp64 for floating types, int64 for integers."""
    wide = [x.double() if _floating(x.dtype) else x.long() for x in xs]
    acc = wide[0].clone()
    for w in wide[1:]:
        acc = {"sum": torch.add, "prod": torch.mul, "min": torch.minimum, "max": torch.maximum}[op](acc, w)
    return acc


def _finish(exact, dtype, scale=1.0):
    """The contract's single rounding: fp32 value of the exact result, times fp32(scale) in fp32,
    one conversion to `dtype` (fp64 keeps the fp64 value; FP8 saturates to +-max, NaN stays)."""
    if not _floating(dtype):
        if dtype == torch.uint8:
            return (exact % 256).to(torch.uint8)
        return exact.to(dtype)
    if dtype == torch.float64:
        return exact * float(torch.tensor(scale, dtype=torch.float32)) if scale != 1.0 else exact.clone()
    v = exact.to(torch.float32)
    if scale != 1.0:
        v = v * torch.tensor(scale, dtype=torch.float32)
    if dtype in FP8:
        m = torch.finfo(dtype).max
        v = torch.where(v.isnan(), v, v.clamp(-m, m))
    return v.to(dtype)


def _bits(t):
    return t.contiguous().view({1: torch.uint8, 2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


def _mismatch(got, want):
    """None if `got` has `want`'s bytes (any NaN matches any NaN), else the first bad index."""
    got = got.cpu()
    if got.shape != want.shape:
        return f"shape {tuple(got.shape)} != {tuple(want.shape)}"
    gb_, wb = _bits(got), _bits(want)
    same = gb_ == wb
    if _floating(want.dtype):
        same |= got.float().isnan() & want.float().isnan()
    if bool(same.all()):
        return None
    i = int((~same).nonzero()[0])
    return f"[{i}] got {got[i].item()!r} want {want[i].item()!r} ({int((~same).sum())} of {got.numel()} differ)"


# ---- CPU checks of the inputs and the reference (no GPU needed) ------------------------------------


@pytest.mark.parametrize("dtype,op", [(d, "sum") for d in MAIN + FP8 + (torch.float64,)] +
                         [(d, "prod") for d in MAIN])
def test_inputs_are_order_free(dtype, op):
    """Every permutation of a sampled column reduces to the same fp32 value (and to the exact one)."""
    for n in (3, 5, 8, 16):
        if op == "prod" and n > 8:
            continue
        cols = torch.stack([_values(op, dtype, 64, _gen(("free", str(dtype), op, n), r)) for r in range(n)])
        exact = _combine(list(cols), op)
        perms = list(itertools.permutations(range(n))) if n <= 5 else [torch.randperm(n, generator=_gen("p", k)).tolist()
                                                                         for k in range(200)]
        for perm in perms:
            acc = cols[perm[0]].float()
            for r in perm[1:]:
                acc = acc + cols[r].float() if op == "sum" else acc * cols[r].float()
            assert torch.equal(acc.double(), exact), (n, perm)


def test_reference_rounding_rules():
    """The reference applies the documented rules on known values."""
    f32, bf16, f16 = torch.float32, torch.bfloat16, torch.float16
    t = lambda *v: torch.tensor(v, dtype=torch.float64)  # noqa: E731
    # one rounding of the exact sum: 256 + 1 + 1 is 258 (a bf16 value); per combine it would be 256
    assert _finish(t(258.0), bf16).item() == 258.0
    assert _finish(t(257.0), bf16).item() == 256.0  # tie, to even
    assert _finish(t(259.0), bf16).item() == 260.0  # tie, to even
    # f16: 40000 + 40000 - 40000 is 40000, not inf
    assert _finish(_combine([t(40000.0), t(40000.0), t(-40000.0)], "sum"), f16).item() == 40000.0
    # the scale multiplies the fp32 value in fp32, then the result is rounded once
    s = 0.3
    want = (torch.tensor(3.0, dtype=f32) * torch.tensor(s, dtype=f32)).to(bf16)
    assert torch.equal(_finish(t(3.0), bf16, s), want.reshape(1))
    assert _finish(t(1.0), f32, 0.3).item() == float(torch.tensor(0.3, dtype=f32))
    # FP8 saturates to +-max where torch's own cast gives NaN / inf; NaN stays NaN
    assert _finish(t(448.0 * 3), E4M3).float().item() == 448.0
    assert _finish(t(-1e9), E4M3).float().item() == -448.0
    assert _finish(t(60000.0 * 2), E5M2).float().item() == 57344.0
    assert math.isnan(_finish(t(float("nan")), E4M3).float().item())
    assert _finish(t(448.0 * 3), E4M3, 0.25).float().item() == 320.0  # 1344 * 0.25 = 336 -> 320
    # subnormals survive (no flush to zero)
    assert _finish(t(2.0 ** -24 * 3), f16).item() == 2.0 ** -24 * 3
    assert _finish(t(2.0 ** -130), bf16).item() == 2.0 ** -130
    # integers: u8 wraps, i64 keeps all 64 bits
    assert _finish(torch.tensor([300]), torch.uint8).item() == 44
    assert _finish(torch.tensor([(1 << 60) + 1]), torch.int64).item() == (1 << 60) + 1
    # the comparison: any NaN matches any NaN, +0 and -0 differ
    assert _mismatch(torch.tensor([float("nan")]), torch.tensor([-float("nan")])) is None
    assert _mismatch(torch.tensor([0.0]), torch.tensor([-0.0])) is not None


# ---- GPU helpers ----------------------------------------------------------------------------------


def _cc(ctx):
    cc = gcu.CudaContext(ctx, 0, stage_bytes=STAGE)
    cc.set_timeout(120000)
    return cc


def _limits(cc):
    """Byte limits of this context: what the LL kernel and a one-shot half take, where `plan()`
    switches from LL and from one-shot, and the pool's bulk region (collectives.cc, layoutOf)."""
    t = gb._C.cuda.get_tuning()
    half = min(-(-max(t["one_shot_max_bytes"], 4096) // 4096) * 4096, STAGE // 4)
    return {"ll": cc.pc.ll_max_bytes(), "half": half, "plan_ll": min(t["ll_max_bytes"], cc.pc.ll_max_bytes()),
            "plan_one": t["one_shot_max_bytes"] // cc.size, "bulk": STAGE - 2 * half}


def _fits(algo, count, dtype, lim):
    """Whether an explicit `algo` runs as named for a plain tensor of `count` elements (a larger
    one is served by the pipelined kernel)."""
    nbytes = count * _es(dtype)
    if algo == "ll":
        return nbytes <= lim["ll"]
    if algo == "one_shot":
        return -(-nbytes // 16) * 16 <= lim["half"]
    return True


def _auto_algo(count, dtype, lim):
    """What plan() picks for a plain tensor without a tuning-table entry (collectives.cc)."""
    nbytes = count * _es(dtype)
    if nbytes <= lim["plan_ll"]:
        return "ll"
    if nbytes <= lim["plan_one"] and _fits("one_shot", count, dtype, lim):
        return "one_shot"
    return "pipelined"


def _counts(dtype, P, thorough):
    K = 16 // _es(dtype)
    base = [1, K - 1, K, K + 1, P * K - 1, P * K + 1, (3 * P + 1) * K + 3, BIG]
    if not thorough:
        base = [K - 1, K + 1, P * K + 1, (3 * P + 1) * K + 3, BIG]
    return sorted({c for c in base if c > 0})


class Checker:
    """Collects mismatches of one rank instead of raising, so that the ranks stay in step."""

    def __init__(self, rank):
        self.rank, self.bad, self.n = rank, [], 0

    def __call__(self, what, got, want):
        self.n += 1
        m = _mismatch(got, want)
        if m is not None:
            self.bad.append(f"rank {self.rank} {what}: {m}")


def _report(results):
    bad = [b for r in results for b in r[0]]
    assert sum(r[1] for r in results) > 0
    assert not bad, f"{len(bad)} mismatches:\n" + "\n".join(bad[:60])


def _sync(cc):
    cc.synchronize()


class Buffers:
    """Per-dtype registered and symmetric buffers, registered once (registration is collective)."""

    def __init__(self, cc):
        self.cc, self.reg, self.sym = cc, {}, {}

    def view(self, kind, dtype, count, off):
        if kind == "plain":
            return torch.empty(count + off, dtype=dtype, device="cuda")[off:]
        n = BIG + 64
        if kind == "reg":
            if dtype not in self.reg:
                self.reg[dtype] = torch.empty(n, dtype=dtype, device="cuda")
                self.cc.register(self.reg[dtype])
            return self.reg[dtype][off:off + count]
        if dtype not in self.sym:
            self.sym[dtype] = self.cc.empty(n, dtype)
        return self.sym[dtype][off:off + count]


# ---- allreduce -----------------------------------------------------------------------------------

# (name, algo, buffer kind)
PATHS = [("ll", "ll", "plain"), ("one_shot", "one_shot", "plain"), ("two_shot_reg", "two_shot", "reg"),
         ("two_shot_sym", "two_shot", "sym"), ("pipelined", "pipelined", "plain"), ("auto", "auto", "plain")]


def _scales(dtype, thorough):
    if not _floating(dtype):
        return [1.0]
    return [1.0, "avg", 0.3] if thorough else [1.0, 0.3]


def _allreduce_cases(cc, dtype, thorough):
    P, es = cc.size, _es(dtype)
    K = 16 // es
    lim = _limits(cc)
    counts = _counts(dtype, P, thorough)
    for name, algo, kind in PATHS:
        cs = list(counts)
        if name == "auto":  # both sides of plan()'s LL and one-shot thresholds
            cs += [lim["plan_ll"] // es, lim["plan_ll"] // es + 1, lim["plan_one"] // es, lim["plan_one"] // es + 1]
        for count in sorted(set(cs)):
            if kind == "plain" and not _fits(algo, count, dtype, lim):
                continue
            # view offsets: none, one element, one element short of 16 bytes
            for off in (sorted({0, 1, K - 1}) if thorough else [0, 1]):
                for scale in _scales(dtype, thorough):
                    yield name, algo, kind, count, off, scale


def _allreduce_worker(ctx, dtypes, ops, thorough):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bufs = Buffers(cc)
    lim = _limits(cc)
    for dtype in dtypes:
        K = 16 // _es(dtype)
        for op in ops:
            full = thorough and op == "sum"  # the other ops run a thinner product
            n = max(BIG, lim["plan_one"] // _es(dtype), lim["plan_ll"] // _es(dtype)) + 64
            xs = [_values(op, dtype, n, _gen(("ar", str(dtype), op), r)) for r in range(P)]
            exact = _combine(xs, op)
            mine = xs[me].cuda()
            for name, algo, kind, count, off, scale in _allreduce_cases(cc, dtype, full):
                if name == "auto":
                    plan = cc.plan(mine[:count], OPS[op])
                    if not plan["from_table"] and plan["algo"] != _auto_algo(count, dtype, lim):
                        chk.bad.append(f"rank {me} plan {dtype} count={count}: {plan['algo']}, expected "
                                       f"{_auto_algo(count, dtype, lim)}")
                s = 1.0 / P if scale == "avg" else scale
                want = _finish(exact[:count], dtype, s)
                # twice: both LL / stage parities; plain tensors the second time out of place
                for rep in range(2 if full else 1):
                    t = bufs.view(kind, dtype, count, off)
                    t.copy_(mine[:count])
                    kw = {"average": True} if scale == "avg" else {"scale": scale}
                    if name == "pipelined":
                        kw.update(tile=16, blocks=2)
                    if kind == "plain" and (rep == 1 or not full and off == 1):
                        dst = bufs.view("plain", dtype, count, (off + 3) % K if K > 1 else 0)
                        cc.allreduce(t, op=OPS[op], algo=algo, out=dst, **kw)
                        t = dst
                    else:
                        cc.allreduce(t, op=OPS[op], algo=algo, **kw)
                    _sync(cc)
                    chk(f"allreduce {name} {dtype} {op} count={count} off={off} scale={scale} rep={rep}", t, want)
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("dtype", MAIN)
def test_allreduce_exact(size, dtype):
    _report(gb.spawn_threads(size, _allreduce_worker, [dtype], ["sum", "prod", "min", "max"], True, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_allreduce_exact_other_dtypes(size):
    _report(gb.spawn_threads(size, _allreduce_worker, list(OTHER), ["sum"], False, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", SIZES)
@pytest.mark.parametrize("dtype", OTHER)
def test_allreduce_exact_sweep(size, dtype):
    ops = ["sum", "min", "max"] + (["prod"] if _floating(dtype) and dtype not in FP8 else [])
    _report(gb.spawn_threads(size, _allreduce_worker, [dtype], ops, True, cuda_device=0))


def _edge_inputs(dtype, P, r):
    """Small vectors of the edge values: NaN, +-inf, f16 intermediate overflow, subnormals, ties."""
    f = torch.finfo(dtype)
    cols = []
    # inf on rank 0, -inf on rank 1: NaN; inf with finite values: inf; NaN on the last rank: NaN
    cols.append([float("inf") if q == 0 else (-float("inf") if q == 1 else 1.0) for q in range(P)])
    cols.append([float("inf") if q == 0 else 2.0 for q in range(P)])
    cols.append([float("nan") if q == P - 1 else 1.0 for q in range(P)])
    # x + x - x: fine in fp32, inf if rounded to f16 after the first add (near fp32's own range
    # the sum would depend on the order, so the other types add small values)
    big = 40000.0 if dtype == torch.float16 else 1.0
    cols.append([big if q < 2 else (-big if q == 2 else 0.0) for q in range(P)])
    # subnormals (no flush to zero) and a subnormal result
    tiny = f.smallest_normal
    cols.append([tiny / 8 * (q + 1) for q in range(P)])
    cols.append([tiny / 16 if q % 2 == 0 else -tiny / 64 for q in range(P)])
    # round to nearest even: 256 + 1 [+ 1 ...] in bf16 (8 bits), 2048 + 1 ... in f16 (11 bits)
    top = 256.0 if dtype == torch.bfloat16 else 2048.0
    for k in (1, 3):
        cols.append([top if q == 0 else (k if q == 1 else 1.0) for q in range(P)])
        cols.append([-top if q == 0 else (-k if q == 1 else -1.0) for q in range(P)])
    x = torch.tensor(cols, dtype=torch.float64)[:, r]
    return x.to(dtype)


def _edge_worker(ctx, dtypes):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bufs = Buffers(cc)
    for dtype in dtypes:
        col = [_edge_inputs(dtype, P, r) for r in range(P)]
        m = col[0].numel()
        # tile the columns, with a pack-sized tail, so they land in packs and in scalar tails
        reps = 40
        xs = [c.repeat(reps) for c in col]
        exact = _combine(xs, "sum")
        mine = xs[me].cuda()
        for count in (m, m * reps - 1, m * 3 + 1):
            for name, algo, kind in PATHS:
                for off in (0, 1):
                    t = bufs.view(kind, dtype, count, off)
                    t.copy_(mine[:count])
                    cc.allreduce(t, algo=algo)
                    _sync(cc)
                    chk(f"edge allreduce {name} {dtype} count={count} off={off}", t, _finish(exact[:count], dtype))
            # reduce_scatter of the same values, registered and staged
            counts = [count // P + (1 if q < count % P else 0) for q in range(P)]
            lo = sum(counts[:me])
            for kind in ("reg", "plain"):
                src = bufs.view(kind, dtype, count, 1)
                src.copy_(mine[:count])
                out = torch.empty(counts[me], dtype=dtype, device="cuda")
                cc.reduce_scatter(out, src, counts)
                _sync(cc)
                chk(f"edge reduce_scatter {kind} {dtype} count={count}", out, _finish(exact[lo:lo + counts[me]], dtype))
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 3, 8])
def test_edge_values(size):
    _report(gb.spawn_threads(size, _edge_worker, [torch.float32, torch.bfloat16, torch.float16], cuda_device=0))


# ---- cast epilogue and extra local pointers ------------------------------------------------------


def _cast_worker(ctx):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bufs = Buffers(cc)
    ll = cc.pc.ll_max_bytes()
    for idt, odt in ((torch.float32, torch.bfloat16), (torch.float32, torch.float16), (torch.bfloat16, torch.float32),
                     (torch.float16, torch.float32)):
        n = BIG + 64
        # f32 inputs: values whose sum is exact in fp32, so the one rounding is to the output dtype
        xs = [_sum_values(idt, n, _gen(("cast", str(idt), str(odt)), r)) for r in range(P)]
        exact = _combine(xs, "sum")
        mine = xs[me].cuda()
        ie, oe = _es(idt), _es(odt)
        for count in (1, 7, 9, 8 * P + 5, 4099, BIG):
            for scale in (1.0, "avg", 0.3):
                s = 1.0 / P if scale == "avg" else scale
                kw = {"average": True} if scale == "avg" else {"scale": scale}
                want = _finish(exact[:count], odt, s)
                # registered in and out (castAllreduceKernel); 16 bytes in is 32-byte misaligned
                for off_bytes in (0, 16):
                    a = bufs.view("sym", idt, count, off_bytes // ie)
                    o = bufs.view("sym", odt, count, off_bytes // oe)
                    a.copy_(mine[:count])
                    cc.allreduce(a, out=o, **kw)
                    _sync(cc)
                    chk(f"cast registered {idt}->{odt} count={count} off={off_bytes}B scale={scale}", o, want)
                # plain tensors (LL)
                if count * ie <= ll:
                    a = bufs.view("plain", idt, count, 1)
                    o = bufs.view("plain", odt, count, 0)
                    a.copy_(mine[:count])
                    cc.allreduce(a, out=o, **kw)
                    _sync(cc)
                    chk(f"cast plain {idt}->{odt} count={count} scale={scale}", o, want)
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_cast_epilogue_exact(size):
    _report(gb.spawn_threads(size, _cast_worker, cuda_device=0))


def _extra_worker(ctx, size):
    """Two local pointers per rank. Under every documented rule the result is
    round(scale * sum_r round(a_r + b_r)) (one pointer fold per rank, rounded), and at one rank
    the fused local step's round(scale * (a + b))."""
    cc = _cc(ctx)
    P, me = size, ctx.rank
    chk = Checker(me)
    bufs = Buffers(cc)
    lim = _limits(cc)
    for dtype in MAIN:
        n = BIG + 64
        a = [_sum_values(dtype, n, _gen(("xa", str(dtype)), r)) for r in range(P)]
        b = [_sum_values(dtype, n, _gen(("xb", str(dtype)), r)) for r in range(P)]
        folded = [_finish(_combine([x, y], "sum"), dtype) for x, y in zip(a, b)] if P > 1 else None
        exact = _combine(folded, "sum") if P > 1 else _combine([a[0], b[0]], "sum")
        ma, mb = a[me].cuda(), b[me].cuda()
        K = 16 // _es(dtype)
        # one rank: the fused local step (local_allreduce_many)
        paths = [("local", "auto", "plain")] if P == 1 else [p for p in PATHS if p[0] != "two_shot_sym"]
        for name, algo, kind in paths:
            for count in (1, K - 1, K + 1, P * K + 1, (3 * P + 1) * K + 3, BIG):
                if kind == "plain" and not _fits(algo, count, dtype, lim):
                    continue
                for off in (0, 1):
                    for scale in (1.0, 0.3):
                        t = bufs.view(kind, dtype, count, off)
                        u = torch.empty(count + 1, dtype=dtype, device="cuda")[1 - off:][:count]
                        t.copy_(ma[:count])
                        u.copy_(mb[:count])
                        cc.allreduce(t, algo=algo, extra=[u], scale=scale)
                        _sync(cc)
                        want = _finish(exact[:count], dtype, scale)
                        chk(f"extra {name} {dtype} count={count} off={off} scale={scale} (main)", t, want)
                        chk(f"extra {name} {dtype} count={count} off={off} scale={scale} (extra)", u, want)
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
def test_extra_pointers_exact(size):
    _report(gb.spawn_threads(size, _extra_worker, size, cuda_device=0))


# ---- reduce_scatter and reduce ---------------------------------------------------------------------


def _rs_counts(P, K, kind, bulk):
    if kind == "ll":  # equal and small
        return [[3] * P, [K + 1] * P, [4 * K - 1] * P]
    # uneven: shares start off the 16-byte grid on several ranks, one rank gets nothing
    small = [(5 * q + 3) % (2 * K + 1) + K * (q % 3) + 1 for q in range(P)]
    small[P // 2] = 0
    large = [bulk // 2 // P // (16 // K) + 7 * q + 1 for q in range(P)]  # staged whole: fits the bulk region
    large[-1] = 0
    if kind == "pipelined":  # larger than the pool's bulk region
        large = [(3 * STAGE // P) // (16 // K) + 7 * q + 1 for q in range(P)]
        large[1] = 0
        return [large]
    return [small, large]


def _rs_worker(ctx, dtypes):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bufs, outs = Buffers(cc), Buffers(cc)
    bulk = _limits(cc)["bulk"]
    for dtype in dtypes:
        K = 16 // _es(dtype)
        n = 3 * STAGE // _es(dtype) + 64 * P + 64
        xs = [_sum_values(dtype, n, _gen(("rs", str(dtype)), r)) for r in range(P)]
        exact = _combine(xs, "sum")
        mine = xs[me].cuda()
        for kind in ("ll", "reg", "staged", "pipelined"):
            for counts in _rs_counts(P, K, kind, bulk):
                total = sum(counts)
                lo = sum(counts[:me])
                for scale in (_scales(dtype, True)):
                    s = 1.0 / P if scale == "avg" else scale
                    for off in (0, 1):
                        src = bufs.view("reg" if kind == "reg" else "plain", dtype, total, off)
                        src.copy_(mine[:total])
                        out = torch.empty(counts[me] + off, dtype=dtype, device="cuda")[off:]
                        cc.reduce_scatter(out, src, counts, scale=s)
                        _sync(cc)
                        chk(f"reduce_scatter {kind} {dtype} counts={counts} off={off} scale={scale}", out,
                            _finish(exact[lo:lo + counts[me]], dtype, s))
        # reduce: registered and plain, roots 0 and P - 1, count % (8 P) != 0
        for count in (8 * P + 3, 1000 * P + 5, 100_003):
            for root in sorted({0, P - 1}):
                for kind in ("sym", "plain"):
                    for off in (0, 1):
                        src = bufs.view(kind, dtype, count, off)
                        src.copy_(mine[:count])
                        dst = outs.view(kind, dtype, count, off)
                        cc.reduce(dst, src, root=root)
                        _sync(cc)
                        if me == root:
                            chk(f"reduce {kind} {dtype} count={count} root={root} off={off}", dst,
                                _finish(exact[:count], dtype))
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_reduce_scatter_and_reduce_exact(size):
    _report(gb.spawn_threads(size, _rs_worker, [torch.float32, torch.bfloat16, torch.float16, E4M3], cuda_device=0))


@pytest.mark.gpu
@pytest.mark.slow
@pytest.mark.parametrize("size", SIZES)
def test_reduce_scatter_and_reduce_exact_sweep(size):
    _report(gb.spawn_threads(size, _rs_worker, [E5M2, torch.float64, torch.int32, torch.int64, torch.uint8],
                             cuda_device=0))


# ---- single rank: the fused local step and the local reductions -------------------------------------

_DT = {torch.float32: gb.DataType.FLOAT32, torch.float16: gb.DataType.FLOAT16, torch.bfloat16: gb.DataType.BFLOAT16,
       E4M3: gb.DataType.FLOAT8_E4M3, E5M2: gb.DataType.FLOAT8_E5M2}


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", MAIN + (E4M3,))
def test_local_steps_exact(dtype):
    cu = gb._C.cuda
    stream = torch.cuda.current_stream().cuda_stream
    es = _es(dtype)
    bad = []
    big = (1 << 20) // es // 8 * 8 + 8 * 17  # above the bulk kernel's size threshold
    for n in (2, 3, 4, 5):
        xs = [_sum_values(dtype, big + 8, _gen(("local", str(dtype)), i)) for i in range(n)]
        exact = _combine(xs, "sum")
        for count in (big, big + 3, big + 7, 8 * 5 + 3, 7):
            for misalign in (0, 1):
                for scale in (1.0, 0.3):
                    for shape in ("bulk", "ldg"):
                        bufs = []
                        for i, x in enumerate(xs):
                            pad = misalign if i == n - 1 else 0
                            t = torch.empty(count + pad, dtype=dtype, device="cuda")[pad:]
                            t.copy_(x[:count])
                            bufs.append(t)
                        ptrs = [t.data_ptr() for t in bufs]
                        try:
                            cu.set_local_shape(*((0, 0, False) if shape == "bulk" else (2, 2, False)))
                            uses_bulk = cu.local_allreduce_many_uses_bulk(ptrs, count, int(_DT[dtype]))
                            if shape == "bulk" and count >= big and not misalign and n <= 4:
                                assert uses_bulk, (n, count)
                            cu.local_allreduce_many(ptrs, count, int(_DT[dtype]), 1, scale, stream)
                            torch.cuda.synchronize()
                        finally:
                            cu.set_local_shape(0, 0, False)
                        want = _finish(exact[:count], dtype, scale)
                        for i, t in enumerate(bufs):
                            m = _mismatch(t, want)
                            if m:
                                bad.append(f"local_allreduce_many {shape} n={n} count={count} misalign={misalign} "
                                           f"scale={scale} buffer {i}: {m}")
            # local_reduce_many: dst := sum of the sources, one rounding
            for misalign in (0, 1):
                srcs = []
                for i, x in enumerate(xs):
                    t = torch.empty(count + misalign, dtype=dtype, device="cuda")[misalign:]
                    t.copy_(x[:count])
                    srcs.append(t)
                dst = torch.empty(count, dtype=dtype, device="cuda")
                cu.local_reduce_many(dst.data_ptr(), [t.data_ptr() for t in srcs], count, int(_DT[dtype]), 1, stream)
                torch.cuda.synchronize()
                m = _mismatch(dst, _finish(exact[:count], dtype))
                if m:
                    bad.append(f"local_reduce_many n={n} count={count} misalign={misalign}: {m}")
    # local_reduce: dst := dst + src
    xs = [_sum_values(dtype, big + 8, _gen(("local2", str(dtype)), i)) for i in range(2)]
    exact = _combine(xs, "sum")
    for count in (big + 3, 8 * 3 + 7, 5):
        for misalign in (0, 1):
            d = torch.empty(count + misalign, dtype=dtype, device="cuda")[misalign:]
            s = torch.empty(count, dtype=dtype, device="cuda")
            d.copy_(xs[0][:count])
            s.copy_(xs[1][:count])
            cu.local_reduce(d.data_ptr(), s.data_ptr(), count, int(_DT[dtype]), 1, stream)
            torch.cuda.synchronize()
            m = _mismatch(d, _finish(exact[:count], dtype))
            if m:
                bad.append(f"local_reduce count={count} misalign={misalign}: {m}")
    assert not bad, f"{len(bad)} mismatches:\n" + "\n".join(bad[:60])


# ---- random inputs: order matters, so bound the error and compare ranks ------------------------------


def _randn_worker(ctx):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    bufs = Buffers(cc)
    out = {}
    bad = []
    for dtype in (torch.float32, torch.bfloat16):
        K = 16 // _es(dtype)
        n = BIG + 64
        xs = [torch.randn(n, generator=_gen(("randn", str(dtype)), r), dtype=torch.float64).to(dtype) for r in range(P)]
        mine = xs[me].cuda()
        exact = _combine(xs, "sum")
        absum = sum(x.double().abs() for x in xs)
        # left-to-right fp32 sum in rank order: what LL and one-shot document
        ordered = xs[0].float()
        for x in xs[1:]:
            ordered = ordered + x.float()
        lim = _limits(cc)
        u_out = 2.0 ** -24 if dtype == torch.float32 else 2.0 ** -8
        for name, algo, kind in PATHS:
            for count in (K + 1, P * K + 1, 4099, BIG):
                if kind == "plain" and not _fits(algo, count, dtype, lim):
                    continue
                for scale in (1.0, 0.3):
                    t = bufs.view(kind, dtype, count, 0)
                    t.copy_(mine[:count])
                    cc.allreduce(t, algo=algo, scale=scale)
                    _sync(cc)
                    got = t.cpu()
                    out[(str(dtype), name, count, scale)] = _bits(got).clone()
                    s32 = float(torch.tensor(scale, dtype=torch.float32))
                    err = (got.double() - exact[:count] * s32).abs()
                    # P - 1 fp32 adds, the fp32 multiply by the scale (when there is one), one rounding
                    # to the output type
                    mag = (exact[:count] * s32).abs()
                    bound = (abs(s32) * (P - 1) * 2.0 ** -24 * absum[:count] + (scale != 1.0) * 2.0 ** -24 * mag) * (
                        1 + u_out) + u_out * mag + 1e-30
                    if not bool((err <= bound).all()):
                        i = int((err > bound).nonzero()[0])
                        bad.append(f"randn {name} {dtype} count={count} scale={scale}: [{i}] error {err[i]} > {bound[i]}")
                    if algo in ("ll", "one_shot"):
                        v = ordered[:count]
                        if scale != 1.0:
                            v = v * torch.tensor(scale, dtype=torch.float32)
                        m = _mismatch(got, v.to(dtype))
                        if m:
                            bad.append(f"randn {name} {dtype} count={count} scale={scale} not the rank-order sum: {m}")
    cc.pc.host_barrier()
    return bad, out


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_random_inputs_bounded_and_identical(size):
    res = gb.spawn_threads(size, _randn_worker, cuda_device=0)
    bad = [b for r in res for b in r[0]]
    for key, bits in res[0][1].items():
        for r in range(1, size):
            if not torch.equal(res[r][1][key], bits):
                bad.append(f"rank {r} differs from rank 0: {key}")
    assert not bad, f"{len(bad)} failures:\n" + "\n".join(bad[:60])
