"""fp32 master weights for ZeRO-1 with 16-bit parameters, and the cast collectives under it.

The cast reduce-scatter takes bfloat16 / float16 gradients and writes a float32 shard: the sum is
accumulated in fp32, scaled in fp32 and never rounded to 16 bits. The cast allgather takes a float32
shard and writes it into every rank's 16-bit output, rounded once on the sender (torch's ``.to()``).
Both are checked byte for byte against torch on every path a same-dtype call takes, with guard bands
around each output, using the order-free inputs of test_reduce_numerics.py so that the fp32 answer is
unique whatever the summation order. ``ZeroOptimizer(master_dtype=torch.float32)`` is then checked
byte for byte against one fp32 master tensor stepped by the same torch AdamW.

Ranks are threads sharing cuda:0, as in the other GPU tests; each rank builds every rank's inputs from
seeded CPU generators and so computes the whole reference itself.
"""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.models import DDPMLP
from gloo_b200.ops import cuda as gcu
from gloo_b200.parallel import ZeroOptimizer, ZeroShard
from test_reduce_numerics import STAGE, Checker, _combine, _finish, _gen, _limits, _mismatch, _report, _sum_values

HALF = (torch.bfloat16, torch.float16)
SIZES = [1, 2, 3, 4, 5, 8]  # 2 / 4 / 8 take the P-specialised instantiations, 3 / 5 the generic ones
GUARD = 40  # elements of sentinel on each side of every output (a multiple of 16 bytes)


def _cc(ctx):
    cc = gcu.CudaContext(ctx, 0, stage_bytes=STAGE)  # 1 MiB: larger plain calls run the pipelined kernels
    cc.set_timeout(120000)
    return cc


def _guarded(dtype, count, reg=None, shift=0):
    """(whole, view): `count` elements between two guard bands of 0x5a bytes, in `reg` (a registered
    uint8 tensor) when it is given, `shift` elements in (1: off the 16-byte grid)."""
    es = torch.empty((), dtype=dtype).element_size()
    nbytes = (count + 2 * GUARD) * es
    if reg is None:
        whole = torch.empty(nbytes, dtype=torch.uint8, device="cuda")
    else:
        assert nbytes + 16 <= reg.numel()
        whole = reg[shift * es:shift * es + nbytes]
    whole.fill_(0x5A)
    return whole, whole.view(dtype)[GUARD:GUARD + count]


def _guards_ok(whole, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    band = whole.cpu()
    return bool((band[:GUARD * es] == 0x5A).all()) and bool((band[band.numel() - GUARD * es:] == 0x5A).all())


def _launches(cc, fn):
    """Kernel launches of every rank while fn() runs on each (barriers keep other work out)."""
    cc.synchronize()
    cc.pc.host_barrier()
    c0 = gb._C.cuda.launch_count()
    cc.pc.host_barrier()
    fn()
    cc.synchronize()
    cc.pc.host_barrier()
    c1 = gb._C.cuda.launch_count()
    cc.pc.host_barrier()
    return c1 - c0


# ---- cast reduce-scatter ---------------------------------------------------------------------------


def _rs_cases(P, bulk, es):
    """(kind, counts): registered (aligned and one element off the 16-byte grid), plain staged whole,
    plain pipelined (larger than the pool's bulk region). Counts 1 and 7, uneven shares with a zero,
    odd multi-CTA shares."""
    small = [[1] * P, [7] * P, [(5 * q + 3) % 17 + 8 * (q % 3) + 1 for q in range(P)]]
    small[-1][P // 2] = 0
    staged = [bulk // 4 // P // es + 2 * q + 1 for q in range(P)]  # a quarter of the bulk region
    staged[-1] = 0
    piped = [(3 * STAGE // P) // es + 7 * q + 1 for q in range(P)]
    piped[P // 2] = 0
    for counts in small + [staged]:
        for kind in ("reg", "reg_off", "plain"):
            yield kind, counts
    yield "reg", piped
    yield "plain", piped


def _rs_worker(ctx):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bulk = _limits(cc)["bulk"] if P > 1 else STAGE
    reg = torch.empty(4 * STAGE + 4096, dtype=torch.uint8, device="cuda")
    cc.register(reg)
    rounded_somewhere = 0
    for dtype in HALF:
        es = 2
        for kind, counts in _rs_cases(P, bulk, es):
            total, lo, mine = sum(counts), sum(counts[:me]), counts[me]
            if kind != "plain" and (total + 8) * es > reg.numel():
                continue
            case = ("rs", str(dtype), kind, tuple(counts))
            xs = [_sum_values(dtype, total, _gen(case, r)) for r in range(P)]
            exact = _combine(xs, "sum")[lo:lo + mine]
            rounded_somewhere += int((_finish(exact, dtype).float() != _finish(exact, torch.float32)).sum())
            if kind == "plain":
                src = torch.empty(total + 1, dtype=dtype, device="cuda")[1:]  # 2 bytes off the 16-byte grid
            else:
                src = reg[(16 if kind == "reg" else 16 + es):][:total * es].view(dtype)
            src.copy_(xs[me].cuda())
            for scale in (1.0, 1.0 / P, 0.3):
                whole, out = _guarded(torch.float32, mine)
                cc.reduce_scatter(out, src, counts, scale=scale)
                cc.synchronize()
                what = f"reduce_scatter {dtype}->f32 {kind} counts={counts} scale={scale}"
                chk(what, out, _finish(exact, torch.float32, scale))
                if not _guards_ok(whole, torch.float32):
                    chk.bad.append(f"rank {me} {what}: guard band written")
    # the inputs are meant to need more than 8 / 11 significant bits: with two or more ranks, an answer
    # rounded to 16 bits anywhere would differ from the reference
    assert rounded_somewhere > 0 or P == 1
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_cast_reduce_scatter_exact(size):
    _report(gb.spawn_threads(size, _rs_worker, cuda_device=0))


# ---- cast allgather(v) -----------------------------------------------------------------------------


def _special(dtype):
    """fp32 values where the cast to `dtype` has to get the rule right."""
    f32 = torch.float32
    one = [1.0, -1.0, 0.0, -0.0]
    if dtype == torch.bfloat16:
        ties = [1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 2.0 ** 100 * (1 + 2.0 ** -8)]
        sub = [2.0 ** -130, 3 * 2.0 ** -135, -(2.0 ** -140) * 1.5, 2.0 ** -149]
        big = [3.4e38, -3.4e38, float(torch.finfo(f32).max), 3.3895e38]
    else:
        ties = [1 + 2.0 ** -11, 1 + 3 * 2.0 ** -11, 2048 + 1.0, -(2048 + 3.0)]
        sub = [2.0 ** -20, 3 * 2.0 ** -25, 2.0 ** -24 * 1.5, 2.0 ** -26, -(2.0 ** -15)]
        big = [65504.0, 65519.0, 65520.0, 1e5, -1e6, 3e38]
    return torch.tensor(one + ties + sub + big + [float("inf"), float("-inf"), float("nan")], dtype=f32)


def _ag_input(dtype, case, r, n):
    g = _gen(case, r)
    x = torch.randn(n, generator=g) * torch.pow(2.0, torch.randint(-20, 20, (n,), generator=g).float())
    sp = _special(dtype)
    k = min(n, sp.numel())
    if k:
        x[torch.randperm(n, generator=g)[:k]] = sp[torch.randperm(sp.numel(), generator=g)[:k]]
    return x


def _ag_cases(P, bulk):
    """(kind, counts): registered output, plain output staged whole, plain pipelined."""
    even = [[1] * P, [513] * P]
    uneven = [(7 * q + 5) % 19 + 16 * (q % 2) for q in range(P)]
    uneven[-1] = 0
    staged = [bulk // 4 // P // 2 + 3 * q + 1 for q in range(P)]
    staged[P // 2] = 0
    piped = [(3 * STAGE // P) // 2 + 5 * q + 3 for q in range(P)]
    piped[0] = 0
    for counts in even + [uneven, staged]:
        for kind in ("reg", "reg_off", "plain"):
            yield kind, counts
    yield "reg", piped
    yield "plain", piped


def _ag_worker(ctx):
    cc = _cc(ctx)
    P, me = cc.size, cc.rank
    chk = Checker(me)
    bulk = _limits(cc)["bulk"] if P > 1 else STAGE
    reg = torch.empty(4 * STAGE + 4096, dtype=torch.uint8, device="cuda")
    cc.register(reg)
    for dtype in HALF:
        for kind, counts in _ag_cases(P, bulk):
            case = ("ag", str(dtype), kind, tuple(counts))
            xs = [_ag_input(dtype, case, r, counts[r]) for r in range(P)]
            want = torch.cat([x.to(dtype) for x in xs])
            total = sum(counts)
            if kind != "plain" and (total + 2 * GUARD) * 2 + 16 > reg.numel():
                continue
            whole, out = _guarded(dtype, total, reg if kind != "plain" else None, 1 if kind == "reg_off" else 0)
            mine = xs[me].cuda()
            cc.allgatherv(out, mine, counts)
            cc.synchronize()
            what = f"allgatherv f32->{dtype} {kind} counts={counts}"
            chk(what, out, want)
            if not _guards_ok(whole, dtype):
                chk.bad.append(f"rank {me} {what}: guard band written")
            if len(set(counts)) == 1 and kind == "plain":
                whole, out = _guarded(dtype, total)
                cc.allgather(out, mine)
                cc.synchronize()
                chk(f"allgather f32->{dtype} counts={counts}", out, want)
    cc.pc.host_barrier()
    return chk.bad, chk.n


@pytest.mark.gpu
@pytest.mark.parametrize("size", SIZES)
def test_cast_allgather_exact(size):
    _report(gb.spawn_threads(size, _ag_worker, cuda_device=0))


def test_cast_reference_rules():
    """The reference of the allgather is torch's cast: ties to even, subnormals kept, overflow to
    +-inf, NaN stays NaN (no GPU needed)."""
    bf, f16 = torch.bfloat16, torch.float16
    t = lambda *v: torch.tensor(v, dtype=torch.float32)  # noqa: E731
    assert t(1 + 2.0 ** -8).to(bf).item() == 1.0 and t(1 + 3 * 2.0 ** -8).to(bf).item() == 1 + 2.0 ** -6
    assert t(2.0 ** -130).to(bf).item() == 2.0 ** -130
    assert t(3.4e38).to(bf).item() == float("inf") and t(65520.0).to(f16).item() == float("inf")
    assert t(65519.0).to(f16).item() == 65504.0 and t(2.0 ** -24 * 1.5).to(f16).item() == 2.0 ** -23
    assert torch.isnan(t(float("nan")).to(f16)).all()
    assert _mismatch(t(1.0).to(bf), t(1.0 + 2.0 ** -7).to(bf)) is not None


# ---- launches and malformed calls -------------------------------------------------------------------


def _calls_worker(ctx):
    cc = _cc(ctx)
    P = cc.size
    bf, f32 = torch.bfloat16, torch.float32
    counts = [1000 + q for q in range(P)]
    total, mine = sum(counts), counts[cc.rank]
    reg = torch.zeros(total * 4 + 64, dtype=torch.uint8, device="cuda")
    cc.register(reg)
    reg_in = reg[:total * 2].view(bf)
    reg_out = reg[:total * 2].view(bf)
    plain_in, plain_out = torch.zeros(total, dtype=bf, device="cuda"), torch.zeros(total, dtype=bf, device="cuda")
    shard32, shard16 = torch.zeros(mine, device="cuda"), torch.zeros(mine, dtype=bf, device="cuda")
    big = torch.zeros(3 * STAGE, dtype=bf, device="cuda")
    big_counts = [3 * STAGE // P] * P
    big_shard = torch.zeros(big_counts[0], device="cuda")
    # one launch per cast call, on every path
    calls = [lambda: cc.reduce_scatter(shard32, reg_in, counts), lambda: cc.reduce_scatter(shard32, plain_in, counts),
             lambda: cc.reduce_scatter(big_shard, big[:sum(big_counts)], big_counts, scale=0.5),
             lambda: cc.allgatherv(reg_out, shard32, counts), lambda: cc.allgatherv(plain_out, shard32, counts),
             lambda: cc.allgatherv(big[:sum(big_counts)], big_shard, big_counts)]
    got = [_launches(cc, f) for f in calls]
    want = [P] * len(calls)  # one kernel on each rank (one local kernel at P = 1)
    # malformed: no launch, ValueError on every rank
    raw = torch.zeros(total * 4, dtype=torch.uint8, device="cuda")
    F32, BF16, F16, F64 = (int(d) for d in (gb.DataType.FLOAT32, gb.DataType.BFLOAT16, gb.DataType.FLOAT16,
                                            gb.DataType.FLOAT64))
    s = torch.cuda.current_stream().cuda_stream
    buf, off = cc.lookup(reg)
    bad = [lambda: cc.reduce_scatter(shard16, plain_in.float(), counts),            # f32 -> bf16: not a pair
           lambda: cc.reduce_scatter(torch.zeros(mine, dtype=torch.float16, device="cuda"), plain_in, counts),
           lambda: cc.reduce_scatter(shard32.double(), plain_in, counts),            # bf16 -> f64
           lambda: cc.reduce_scatter(shard32, plain_in, counts, op=gb.ReduceOp.MAX),  # not SUM
           lambda: cc.reduce_scatter(shard32, reg_in, counts, op=gb.ReduceOp.MAX),
           lambda: cc.reduce_scatter(raw[:mine * 4].view(f32), raw[:total * 2].view(bf), counts),  # overlap
           lambda: cc.reduce_scatter(reg[:mine * 4].view(f32), reg_in, counts),                     # overlap, registered
           lambda: gb._C.cuda.reduce_scatter_reg(cc.pc, buf, off + reg.numel() - 2, shard32.data_ptr(), counts, BF16, 1, s,
                                                 1.0, F32),  # input beyond the registered buffer
           lambda: cc.allgatherv(plain_out.float(), shard16, counts),                # bf16 -> f32: not a pair
           lambda: cc.allgatherv(plain_out.to(torch.float16), shard32.double(), counts),
           lambda: cc.allgatherv(raw[:total * 2].view(bf), raw[:mine * 4].view(f32), counts),  # overlap
           lambda: cc.allgatherv(reg_out, reg[:mine * 4].view(f32), counts),                     # overlap, registered
           lambda: gb._C.cuda.allgatherv_cast_reg(cc.pc, shard32.data_ptr(), F32, buf, off + reg.numel() - 2, counts, BF16,
                                                  s),  # output beyond the registered buffer
           lambda: gb._C.cuda.allgatherv_cast(cc.pc, shard32.data_ptr(), F32, plain_out.data_ptr(), counts, F64, s),
           lambda: gb._C.cuda.allgatherv_cast(cc.pc, shard32.data_ptr(), F32, plain_out.data_ptr(), counts + [1], F16, s)]
    raised = []

    def run_bad():
        for f in bad:
            try:
                f()
                raised.append(False)
            except ValueError:
                raised.append(True)

    n_bad = _launches(cc, run_bad)
    cc.pc.host_barrier()
    return got, want, raised, n_bad


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4])
def test_cast_calls_launch_once_and_reject_malformed(size):
    for got, want, raised, n_bad in gb.spawn_threads(size, _calls_worker, cuda_device=0):
        assert got == want
        assert all(raised), [i for i, r in enumerate(raised) if not r]
        assert n_bad == 0


# ---- ZeroOptimizer master mode -----------------------------------------------------------------------

SHAPES = [(37,), (5, 13), (1000,), (3,)]


def _params(dtype, device, g):
    return [torch.nn.Parameter((torch.randn(s, generator=g) * 0.5).to(dtype).to(device)) for s in SHAPES]


def _master_worker(ctx, cuda, opt_kw, dtype, steps):
    cc = _cc(ctx) if cuda else None
    P, me = ctx.size, ctx.rank
    device = "cuda" if cuda else "cpu"
    params = _params(dtype, device, torch.Generator().manual_seed(3))
    zo = ZeroOptimizer(ctx, cc, params, torch.optim.AdamW, master_dtype=torch.float32, lr=1e-3, weight_decay=0.01,
                       **opt_kw)
    n = zo.flat_param.numel()
    ref = torch.nn.Parameter(zo.flat_param.detach().float().clone())
    ref_opt = torch.optim.AdamW([ref], lr=1e-3, weight_decay=0.01, **opt_kw)
    bad, launches = [], []
    for k in range(steps):
        flats = []
        for r in range(P):
            flat = torch.zeros(n, dtype=dtype)
            for p, off in zip(params, zo._offs):
                flat[off:off + p.numel()] = _sum_values(dtype, p.numel(), _gen(("zero", k, off), r))
            flats.append(flat)
        for p, off in zip(params, zo._offs):
            p.grad.copy_(flats[me][off:off + p.numel()].view_as(p))
        if cuda:
            launches.append(_launches(cc, zo.step))
        else:
            zo.step()
        ref.grad = _finish(_combine(flats, "sum"), torch.float32, 1.0 / P).to(device)
        ref_opt.step()
        want = ref.detach().to(dtype)
        m = _mismatch(zo.flat_param, want.cpu())
        if m is not None:
            bad.append(f"rank {me} step {k} flat_param: {m}")
        m = _mismatch(zo.shard.detach(), ref.detach()[zo.start:zo.start + zo.counts[me]].cpu())
        if m is not None:
            bad.append(f"rank {me} step {k} master shard: {m}")
        zo.zero_grad()
    assert zo.shard.dtype == torch.float32 and zo.flat_param.dtype == dtype and zo.flat_grad.dtype == dtype
    assert zo.state_bytes() >= 3 * zo.counts[me] * 4  # master, exp_avg, exp_avg_sq
    if cuda:
        cc.pc.host_barrier()
    return bad, launches


@pytest.mark.gpu
@pytest.mark.parametrize("size", [1, 2, 3, 4])
@pytest.mark.parametrize("opt_kw", [{"foreach": False}, {"foreach": True}, {"fused": True}], ids=["single", "foreach", "fused"])
def test_zero_master_matches_fp32_adamw(size, opt_kw):
    for dtype in HALF:
        for bad, launches in gb.spawn_threads(size, _master_worker, True, opt_kw, dtype, 4, cuda_device=0):
            assert not bad, "\n".join(bad[:20])
            assert launches == [2 * size] * 4  # two collective kernels per rank and step


def test_zero_master_cpu_matches_fp32_adamw():
    """The CPU-tensor path: torch casts around the host collectives give the same bytes."""
    for dtype in HALF:
        for bad, _ in gb.spawn_threads(3, _master_worker, False, {"foreach": False}, dtype, 3):
            assert not bad, "\n".join(bad[:20])


def test_zero_master_dtype_rules():
    def fn(ctx):
        ps = [torch.nn.Parameter(torch.randn(10))]
        zo = ZeroOptimizer(ctx, None, ps, torch.optim.SGD, master_dtype=torch.float32, lr=0.1)
        assert not zo.master and zo.shard.dtype == torch.float32  # fp32 parameters: nothing changes
        for bad_dtype in (torch.float16, torch.bfloat16, torch.float64, "float32"):
            with pytest.raises(ValueError):
                ZeroOptimizer(ctx, None, [torch.nn.Parameter(torch.randn(4).bfloat16())], torch.optim.SGD,
                              master_dtype=bad_dtype, lr=0.1)
        zb = ZeroOptimizer(ctx, None, [torch.nn.Parameter(torch.randn(16).bfloat16())], torch.optim.SGD, lr=0.1)
        zm = ZeroOptimizer(ctx, None, [torch.nn.Parameter(torch.randn(16).bfloat16())], torch.optim.SGD,
                           master_dtype=torch.float32, lr=0.1)
        assert zb.shard.dtype == torch.bfloat16 and zm.shard.dtype == torch.float32
        assert zm.state_bytes() == zm.shard.numel() * 4 and zb.state_bytes() == 0
        return True

    assert all(gb.spawn_threads(2, fn))


def test_zero_shard_cast_cpu():
    """ZeroShard on CPU tensors: a float32 shard of a bfloat16 flat buffer."""
    size = 3

    def fn(ctx):
        z = ZeroShard(ctx)
        n = 999
        start, cnt, counts = z.shard_range(n)
        xs = [_sum_values(torch.bfloat16, n, _gen("zs", r)) for r in range(size)]
        shard = torch.zeros(cnt)
        z.reduce_scatter_gradients(xs[ctx.rank], shard, average=True)
        want = _finish(_combine(xs, "sum")[start:start + cnt], torch.float32, 1.0 / size)
        assert _mismatch(shard, want) is None
        full = torch.zeros(n, dtype=torch.bfloat16)
        z.allgather_parameters(full, shard + ctx.rank)
        return full

    outs = gb.spawn_threads(size, fn)
    assert all(torch.equal(o, outs[0]) for o in outs)


# ---- a real model -----------------------------------------------------------------------------------


def _model_worker(ctx, xs, ys, state, lr, steps):
    cc = _cc(ctx)
    m = DDPMLP().to(torch.bfloat16).cuda()
    m.load_state_dict(state)
    zo = ZeroOptimizer(ctx, cc, m.parameters(), torch.optim.AdamW, master_dtype=torch.float32, lr=lr)
    b = xs.shape[0] // ctx.size
    for _ in range(steps):
        x, y = xs[ctx.rank * b:(ctx.rank + 1) * b].cuda(), ys[ctx.rank * b:(ctx.rank + 1) * b].cuda()
        torch.nn.functional.mse_loss(m(x).float(), y.float()).backward()
        zo.step()
        zo.zero_grad()
    cc.pc.host_barrier()
    return [p.detach().cpu() for p in m.parameters()]


@pytest.mark.gpu
@pytest.mark.parametrize("size", [2, 4])
def test_zero_master_trains_like_single_process(size):
    """A bf16 DDPMLP trained with master mode on per-rank batches stays within 2 x steps x lr (plus
    one bf16 step of the weight) of one process training the same bf16 model on the whole batch with
    fp32-master AdamW: AdamW moves each weight by at most about lr per step, so gradients that differ
    only in summation order and rounding can separate the two by at most that much."""
    lr, steps = 1e-3, 4
    g = torch.Generator().manual_seed(21)
    torch.manual_seed(21)
    ref = DDPMLP().to(torch.bfloat16)
    xs, ys = torch.randn(8 * size, 64, generator=g).bfloat16(), torch.randn(8 * size, 8, generator=g).bfloat16()
    single = DDPMLP().to(torch.bfloat16).cuda()
    single.load_state_dict(ref.state_dict())
    master = [p.detach().float().clone().requires_grad_(True) for p in single.parameters()]
    opt = torch.optim.AdamW(master, lr=lr)
    for _ in range(steps):
        single.zero_grad()
        torch.nn.functional.mse_loss(single(xs.cuda()).float(), ys.cuda().float()).backward()
        for mp, p in zip(master, single.parameters()):
            mp.grad = p.grad.float()
        opt.step()
        with torch.no_grad():
            for mp, p in zip(master, single.parameters()):
                p.copy_(mp)
    want = [p.detach().cpu() for p in single.parameters()]
    for params in gb.spawn_threads(size, _model_worker, xs, ys, ref.state_dict(), lr, steps, cuda_device=0):
        for p, w, p0 in zip(params, want, ref.parameters()):
            ulp = w.float().abs() * 2.0 ** -7
            assert bool(((p.float() - w.float()).abs() <= 2 * steps * lr + ulp).all())
            assert not torch.equal(p, p0.detach())  # it trained


def _small_lr_worker(ctx, master_dtype, steps):
    cc = _cc(ctx)
    m = DDPMLP().to(torch.bfloat16).cuda()
    with torch.no_grad():
        for p in m.parameters():
            p.fill_(1.0)  # bf16 spacing below 1.0 is 2^-8: an update of 1e-3 rounds away
    zo = ZeroOptimizer(ctx, cc, m.parameters(), torch.optim.AdamW, master_dtype=master_dtype, lr=1e-3,
                       weight_decay=0.0)
    for _ in range(steps):
        for p in m.parameters():
            p.grad.fill_(1.0)  # AdamW then moves every weight by lr each step
        zo.step()
        zo.zero_grad()
    cc.pc.host_barrier()
    shard = zo.shard.detach().cpu()
    return torch.cat([p.detach().reshape(-1) for p in m.parameters()]).cpu(), shard[shard != 0]  # not the padding


@pytest.mark.gpu
def test_zero_master_keeps_small_updates():
    """Without master weights every update smaller than half a bf16 step of the weight is lost; with
    them the fp32 master accumulates the updates and the bf16 weights follow."""
    steps = 5
    for flat, shard in gb.spawn_threads(2, _small_lr_worker, None, steps, cuda_device=0):
        assert bool((flat.float() == 1.0).all()) and bool((shard.float() == 1.0).all())
    for flat, shard in gb.spawn_threads(2, _small_lr_worker, torch.float32, steps, cuda_device=0):
        assert shard.dtype == torch.float32
        torch.testing.assert_close(shard, torch.full_like(shard, 1.0 - steps * 1e-3), rtol=0, atol=1e-6)
        assert bool((flat == torch.tensor(1.0 - steps * 1e-3).bfloat16()).all()) and bool((flat.float() < 1.0).all())
