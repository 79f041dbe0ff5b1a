"""FP8 (e4m3 / e5m2) buffers in every collective.

Numerical contract (docs/cuda.md): the kernels widen FP8 to fp32, reduce in fp32, apply the
scale in fp32 and round once, to nearest even, saturating to +-max finite. The host CPU
collectives round after every step. Every FP8 input below is chosen so that fp32 holds its
sums exactly, so the expected result is bit-predictable: satfinite(float32(sum) * float32(scale)).
"""
import math
import os
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import torch

import gloo_b200 as gb
from gloo_b200 import _C
from gloo_b200.ops import algorithms as alg

FMTS = [torch.float8_e4m3fn, torch.float8_e5m2]
GLB = {torch.float8_e4m3fn: gb.DataType.FLOAT8_E4M3, torch.float8_e5m2: gb.DataType.FLOAT8_E5M2}
# small integers whose partial sums stay exact in the format (host collectives round per step)
SMALL = {torch.float8_e4m3fn: 16, torch.float8_e5m2: 8}


def _max(fmt):
    return torch.finfo(fmt).max


def _sat(x, fmt):
    """float32 -> fmt, round to nearest even, saturating (torch's .to() would give NaN / inf)."""
    x = x.float()
    return torch.where(torch.isnan(x), x, torch.clamp(x, -_max(fmt), _max(fmt))).to(fmt)


def _bits(t):
    return t.view(torch.uint8)


def _random_codes(fmt, count, seed):
    """FP8 values whose sums of up to 8 are exact in fp32: every finite e4m3 value, and e5m2
    values of magnitude 2^-6 ... 2^10 (or zero)."""
    g = torch.Generator().manual_seed(seed)
    b = torch.randint(0, 256, (count,), generator=g, dtype=torch.int32)
    if fmt == torch.float8_e4m3fn:
        b = torch.where((b & 0x7F) == 0x7F, b & 0x80, b)  # NaN codes -> (signed) zero
    else:
        exp = torch.randint(9, 25, (count,), generator=g, dtype=torch.int32)  # 2^-6 ... 2^9 * 1.75
        b = (b & 0x83) | (exp << 2)
    return b.to(torch.uint8).view(fmt)


def _reduce_ref(inputs, fmt, scale=1.0):
    # added one input at a time from the first, like the kernels: torch's sum() starts from +0
    # and would turn an all-negative-zero column into +0
    s = inputs[0].float()
    for x in inputs[1:]:
        s = s + x.float()
    return _sat(s * torch.tensor(scale, dtype=torch.float32), fmt)


def _float_grid():
    """float32 values over the whole FP8 range: a dense grid, every midpoint between adjacent
    values of both formats with its +-1-ulp neighbours, subnormals, and overflow."""
    parts = [torch.linspace(-70000.0, 70000.0, 200_001), torch.linspace(-500.0, 500.0, 100_001),
             torch.linspace(-2.0 ** -5, 2.0 ** -5, 20_001)]
    for fmt in FMTS:
        v = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(fmt).float()
        v = torch.sort(v[torch.isfinite(v)].unique()).values
        mid = (v[1:] + v[:-1]) / 2  # exact in float32
        parts += [mid, torch.nextafter(mid, torch.full_like(mid, math.inf)),
                  torch.nextafter(mid, torch.full_like(mid, -math.inf)), v]
    return torch.cat(parts).float()


# ---- host conversion ---------------------------------------------------------------------------

@pytest.mark.parametrize("fmt", FMTS)
def test_decode_all_codes(fmt):
    want = torch.arange(256, dtype=torch.int32).to(torch.uint8).view(fmt).float()
    for c in range(256):
        got = _C.fp8_bits_to_float(c, int(GLB[fmt]))
        w = float(want[c])
        assert (math.isnan(got) and math.isnan(w)) or got == w, (c, got, w)


@pytest.mark.parametrize("fmt", FMTS)
def test_encode_matches_clamped_torch(fmt):
    x = _float_grid()
    want = _bits(_sat(x, fmt))
    got = torch.tensor([_C.float_to_fp8_bits(float(v), int(GLB[fmt])) for v in x.tolist()], dtype=torch.uint8)
    bad = (got != want).nonzero()
    assert bad.numel() == 0, [(float(x[i]), int(got[i]), int(want[i])) for i in bad[:5, 0]]
    m = _max(fmt)
    for v in (m * 1.01, m * 2, 1e30, math.inf):
        assert _C.fp8_bits_to_float(_C.float_to_fp8_bits(v, int(GLB[fmt])), int(GLB[fmt])) == m
        assert _C.fp8_bits_to_float(_C.float_to_fp8_bits(-v, int(GLB[fmt])), int(GLB[fmt])) == -m
    assert math.isnan(_C.fp8_bits_to_float(_C.float_to_fp8_bits(math.nan, int(GLB[fmt])), int(GLB[fmt])))


def test_describe_fp8_and_rejects_other_8bit_floats():
    assert gb.types.describe(torch.zeros(3, dtype=torch.float8_e4m3fn))[2] == gb.DataType.FLOAT8_E4M3
    assert gb.types.describe(torch.zeros(3, dtype=torch.float8_e5m2))[2] == gb.DataType.FLOAT8_E5M2
    assert _C.element_size(int(gb.DataType.FLOAT8_E4M3)) == 1
    for name in ("float8_e4m3fnuz", "float8_e5m2fnuz", "float8_e8m0fnu"):
        dt = getattr(torch, name, None)
        if dt is None:
            continue
        with pytest.raises(TypeError, match=name):
            gb.types.describe(torch.zeros(3, dtype=dt))


# ---- host collectives ----------------------------------------------------------------------------

def _small(fmt, rank, count, size):
    """Small integers: every partial sum of `size` of them is exact in `fmt`."""
    lim = SMALL[fmt] // size
    j = torch.arange(count)
    return (((j * 7 + rank * 3) % (2 * lim + 1)) - lim).to(fmt) if lim > 0 else torch.zeros(count).to(fmt)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [1, 2, 3, 4, 7])
def test_host_collectives(fmt, size):
    def fn(ctx):
        r = ctx.rank
        count = 37
        ins = [_small(fmt, q, count, size) for q in range(size)]
        # allreduce: sum / max / min, and product of +-1 / 2 values
        for op, f in ((gb.ReduceOp.SUM, None), (gb.ReduceOp.MAX, torch.maximum), (gb.ReduceOp.MIN, torch.minimum)):
            t = ins[r].clone()
            gb.allreduce(ctx, t, op=op)
            if f is None:
                want = _reduce_ref(ins, fmt)
            else:
                want = ins[0].float()
                for x in ins[1:]:
                    want = f(want, x.float())
                want = want.to(fmt)
            assert torch.equal(_bits(t), _bits(want)), (op, t.float(), want.float())
        pins = [torch.where(torch.arange(count) % (q + 2) == 0, -1.0, 1.0).to(fmt) for q in range(size)]
        t = pins[r].clone()
        gb.allreduce(ctx, t, op=gb.ReduceOp.PRODUCT)
        want = torch.stack([p.float() for p in pins]).prod(0).to(fmt)
        assert torch.equal(_bits(t), _bits(want))
        # reduce_scatter / reduce
        base, rem = divmod(count, size)
        counts = [base + (1 if q < rem else 0) for q in range(size)]
        off = np.cumsum([0] + counts)
        out = torch.zeros(counts[r]).to(fmt)
        gb.reduce_scatter(ctx, out, ins[r].clone())
        assert torch.equal(_bits(out), _bits(_reduce_ref(ins, fmt)[off[r]:off[r + 1]]))
        out = torch.zeros(count).to(fmt)
        gb.reduce(ctx, out, ins[r].clone(), root=size - 1)
        if r == size - 1:
            assert torch.equal(_bits(out), _bits(_reduce_ref(ins, fmt)))
        # data movement: the bytes come back unchanged
        out = torch.zeros(count * size).to(fmt)
        gb.allgather(ctx, out, ins[r])
        assert torch.equal(_bits(out), _bits(torch.cat(ins)))
        t = ins[r].clone()
        gb.broadcast(ctx, t, root=0)
        assert torch.equal(_bits(t), _bits(ins[0]))
        a2a_in = torch.cat([ins[r][:5]] * size)
        out = torch.zeros(5 * size).to(fmt)
        gb.alltoall(ctx, out, a2a_in)
        assert torch.equal(_bits(out), _bits(torch.cat([ins[q][:5] for q in range(size)])))
        # an old-style host allreduce class
        t = ins[r].clone()
        alg.AllreduceRing(ctx, [t]).run()
        assert torch.equal(_bits(t), _bits(_reduce_ref(ins, fmt)))
        return True

    assert all(gb.spawn_threads(size, fn))


def _pg_run(worker_args, size, timeout=240):
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pg_fp8_worker.py")
    init = os.path.join(tempfile.mkdtemp(prefix="glb_pg_fp8_"), "init")
    procs = [subprocess.Popen([sys.executable, worker, init, str(r), str(size)] + worker_args, stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(size)]
    outs = [p.communicate(timeout=timeout) for p in procs]
    for r, (p, (out, err)) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r} ok" in out, (r, p.returncode, out[-500:], err[-2000:])


@pytest.mark.parametrize("size", [1, 2, 3])
def test_process_group_cpu(size):
    _pg_run(["cpu"], size)


# ---- CUDA ------------------------------------------------------------------------------------

ALGOS = ["auto", "one_shot", "two_shot", "ll", "pipelined"]
COUNTS = [1, 15, 17, 4099, 300001]


def _cuda():
    from gloo_b200.ops import cuda as gcu

    return gcu


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_device_encoding_equals_host(fmt):
    """f32 -> FP8 through the cast epilogue at one rank (the LL kernel), bit for bit against torch's
    clamped .to(). test_encode_matches_clamped_torch holds the host encoder to the same reference
    over the same grid, so device and host encodings are equal."""
    gcu = _cuda()
    x = _float_grid()
    want = _bits(_sat(x, fmt))

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        xs = x.cuda()
        out = torch.empty(x.numel(), dtype=fmt, device="cuda")
        step = 50_000
        for lo in range(0, x.numel(), step):
            cc.allreduce(xs[lo:lo + step], out=out[lo:lo + step])
        torch.cuda.synchronize()
        return _bits(out.cpu())

    got = gb.spawn_threads(1, fn, cuda_device=0)[0]
    bad = (got != want).nonzero()
    assert bad.numel() == 0, [(float(x[i]), int(got[i]), int(want[i])) for i in bad[:5, 0]]


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("registered", [True, False])
def test_allreduce_bit_exact(fmt, size, registered):
    gcu = _cuda()

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        sym = cc.empty(max(COUNTS), fmt) if registered else None
        for count in COUNTS:
            ins = [_random_codes(fmt, count, 1000 * count + q) for q in range(size)]
            for algo in ALGOS:
                if registered and algo in ("ll", "one_shot") and count > 65536:
                    continue  # registered LL / one-shot take messages up to their limits only
                for scale, avg in ((1.0, False), (0.25, False), (1.0, True)):
                    if size == 1 and scale == 1.0:
                        continue  # one rank, nothing to scale: no kernel runs
                    t = sym[:count] if registered else torch.empty(count, dtype=fmt, device="cuda")
                    t.copy_(ins[ctx.rank].cuda())
                    cc.allreduce(t, algo=algo, scale=scale, average=avg)
                    torch.cuda.current_stream().synchronize()
                    want = _reduce_ref(ins, fmt, 1.0 / size if avg else scale)
                    got = _bits(t.cpu())
                    assert torch.equal(got, _bits(want)), (algo, count, scale, avg,
                                                           (got != _bits(want)).nonzero()[:5].tolist())
                    cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [2, 3, 4])
def test_literal_schedules(fmt, size):
    gcu = _cuda()
    classes = [gcu.CudaAllreduceRing, gcu.CudaAllreduceRingChunked, gcu.CudaAllreduceHalvingDoubling,
               gcu.CudaAllreduceBcube]

    def fn(ctx):
        for cls in classes:
            for count in (1, 17, 4099, 300001):
                ins = [_small(fmt, q, count, size) for q in range(size)]
                t = ins[ctx.rank].cuda()
                cls(ctx, t, literal=True).run()
                torch.cuda.synchronize()
                assert torch.equal(_bits(t.cpu()), _bits(_reduce_ref(ins, fmt))), (cls, count)
        gcu._cu.peer_context_for(ctx, 0).host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [2, 3, 4])
def test_reduce_scatter_reduce_and_byte_movers(fmt, size):
    gcu = _cuda()

    def fn(ctx):
        r = ctx.rank
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for count in (17, 4099, 300001):
            ins = [_random_codes(fmt, count, 7 * count + q) for q in range(size)]
            full = _reduce_ref(ins, fmt, 0.25)
            base, rem = divmod(count, size)
            counts = [base + (1 if q < rem else 0) for q in range(size)]
            off = np.cumsum([0] + counts)
            out = torch.empty(counts[r], dtype=fmt, device="cuda")
            cc.reduce_scatter(out, ins[r].cuda(), scale=0.25)
            torch.cuda.synchronize()
            assert torch.equal(_bits(out.cpu()), _bits(full[off[r]:off[r + 1]])), ("reduce_scatter", count)
            out = torch.empty(count, dtype=fmt, device="cuda")
            cc.reduce(out, ins[r].cuda(), root=size - 1)
            torch.cuda.synchronize()
            if r == size - 1:
                assert torch.equal(_bits(out.cpu()), _bits(_reduce_ref(ins, fmt))), ("reduce", count)
            # byte movers
            mine = ins[r].cuda()
            t = mine.clone()
            cc.broadcast(t, root=0)
            torch.cuda.synchronize()
            assert torch.equal(_bits(t.cpu()), _bits(ins[0]))
            out = torch.empty(count * size, dtype=fmt, device="cuda")
            cc.allgather(out, mine)
            torch.cuda.synchronize()
            assert torch.equal(_bits(out.cpu()), _bits(torch.cat(ins)))
            vc = [count - q for q in range(size)]
            out = torch.empty(sum(vc), dtype=fmt, device="cuda")
            cc.allgatherv(out, mine[:vc[r]], vc)
            torch.cuda.synchronize()
            assert torch.equal(_bits(out.cpu()), _bits(torch.cat([ins[q][:vc[q]] for q in range(size)])))
            per = count // size
            out = torch.empty(per * size, dtype=fmt, device="cuda")
            cc.alltoall(out, mine[:per * size])
            torch.cuda.synchronize()
            assert torch.equal(_bits(out.cpu()), _bits(torch.cat([ins[q][r * per:(r + 1) * per] for q in range(size)])))
            sc = [1 + q for q in range(size)]  # rank r sends q + 1 elements to rank q
            oc = [r + 1] * size
            out = torch.empty(sum(oc), dtype=fmt, device="cuda")
            cc.alltoallv(out, oc, mine[:sum(sc)], sc)
            torch.cuda.synchronize()
            soff = np.cumsum([0] + sc)
            assert torch.equal(_bits(out.cpu()), _bits(torch.cat([ins[q][soff[r]:soff[r + 1]] for q in range(size)])))
            out = torch.empty(count * size, dtype=fmt, device="cuda")
            cc.gather(out, mine, root=0)
            torch.cuda.synchronize()
            if r == 0:
                assert torch.equal(_bits(out.cpu()), _bits(torch.cat(ins)))
            out = torch.empty(per, dtype=fmt, device="cuda")
            cc.scatter(out, ins[0][:per * size].cuda() if r == 0 else None, root=0)
            torch.cuda.synchronize()
            assert torch.equal(_bits(out.cpu()), _bits(ins[0][r * per:(r + 1) * per]))
            # point to point, and the zero-copy exchange around the ring
            dst, src = (r + 1) % size, (r - 1) % size
            if r % 2 == 0 and r + 1 < size:
                cc.send(mine, r + 1)
            elif r % 2 == 1:
                got = torch.empty(count, dtype=fmt, device="cuda")
                cc.recv(got, r - 1)
                torch.cuda.synchronize()
                assert torch.equal(_bits(got.cpu()), _bits(ins[r - 1]))
            sym = cc.empty(count, fmt)
            cc.exchange(mine, dst, sym, src)
            torch.cuda.synchronize()
            assert torch.equal(_bits(sym.cpu()), _bits(ins[src]))
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("size", [1, 2, 4])
def test_cast_epilogue(fmt, size):
    """FP8 -> f32 / bf16 and f32 / bf16 -> FP8, on registered (castAllreduceKernel) and plain
    (LL) tensors."""
    gcu = _cuda()

    def fn(ctx):
        r = ctx.rank
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for registered, count in ((True, 100_003), (False, 4099)):
            for wide in (torch.float32, torch.bfloat16):
                # FP8 in, wide out
                ins = [_random_codes(fmt, count, 11 * count + q) for q in range(size)]
                src = cc.empty(count, fmt) if registered else torch.empty(count, dtype=fmt, device="cuda")
                dst = cc.empty(count, wide) if registered else torch.empty(count, dtype=wide, device="cuda")
                src.copy_(ins[r].cuda())
                cc.allreduce(src, out=dst, scale=0.5)
                torch.cuda.synchronize()
                want = (_reduce_ref(ins, torch.float32) * 0.5).to(wide)
                assert torch.equal(dst.cpu(), want), ("fp8->wide", registered, wide)
                # wide in, FP8 out: small integers * 1/16 (exact in bf16 and in the sum)
                wins = [((torch.arange(count) * (q + 3)) % 33 - 16).to(wide) / 16 for q in range(size)]
                src = cc.empty(count, wide) if registered else torch.empty(count, dtype=wide, device="cuda")
                dst = cc.empty(count, fmt) if registered else torch.empty(count, dtype=fmt, device="cuda")
                src.copy_(wins[r].cuda())
                cc.allreduce(src, out=dst, scale=3.0)
                torch.cuda.synchronize()
                assert torch.equal(_bits(dst.cpu()), _bits(_reduce_ref(wins, fmt, 3.0))), ("wide->fp8", registered, wide)
                cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("n", [2, 3, 4, 5])
def test_local_fused_step_bulk_and_ldg_stg(fmt, n):
    cu = _C.cuda
    count = 24_000_000 + 16 + 3  # whole tiles, then packs, then single elements
    host = [_random_codes(fmt, count, 99 + k) for k in range(n)]
    want = _bits(_reduce_ref(host, fmt, 0.25))
    stream = torch.cuda.current_stream().cuda_stream
    dev = [h.cuda() for h in host]
    ptrs = [t.data_ptr() for t in dev]
    try:
        cu.set_local_shape(0, 0, False)
        assert cu.local_allreduce_many_uses_bulk(ptrs, count, int(GLB[fmt])) == (n <= 4)
        cu.local_allreduce_many(ptrs, count, int(GLB[fmt]), 1, 0.25, stream)
        torch.cuda.synchronize()
        bulk = [_bits(t.cpu()) for t in dev]
        for b in bulk:
            assert torch.equal(b, want)
        for t, h in zip(dev, host):
            t.copy_(h)
        cu.set_local_shape(2, 2, False)  # pins the LDG/STG kernel
        cu.local_allreduce_many(ptrs, count, int(GLB[fmt]), 1, 0.25, stream)
        torch.cuda.synchronize()
        for t, b in zip(dev, bulk):
            assert torch.equal(_bits(t.cpu()), b)
    finally:
        cu.set_local_shape(0, 0, False)
    one_m = [torch.empty(1 << 20, dtype=fmt, device="cuda") for _ in range(2)]
    assert cu.local_allreduce_many_uses_bulk([t.data_ptr() for t in one_m], 1 << 20, int(GLB[fmt]))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_saturation_and_nan(fmt):
    gcu = _cuda()
    size = 2
    m = _max(fmt)

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for algo in ("ll", "one_shot", "two_shot", "pipelined"):
            vals = torch.tensor([m, -m, m / 2 + m / 4, 1.0, math.nan] + [m] * 20).to(fmt)
            t = cc.empty(vals.numel(), fmt) if algo == "two_shot" else torch.empty(vals.numel(), dtype=fmt, device="cuda")
            t.copy_(vals.cuda())
            cc.allreduce(t, algo=algo)
            torch.cuda.synchronize()
            got = t.cpu().float()
            assert got[0] == m and got[1] == -m and got[2] == m and got[3] == 2.0, (algo, got[:4])
            assert math.isnan(got[4]) and bool((got[5:] == m).all()), algo
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FMTS)
def test_plan_never_nvls_and_explicit_nvls_raises(fmt):
    gcu = _cuda()
    size = 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for kind in (0, 1, 2):
            for nbytes in (1 << 10, 1 << 20, 1 << 26, 1 << 30):
                p = gcu._cu.plan_allreduce(cc.pc, nbytes, int(GLB[fmt]), int(gb.ReduceOp.SUM), kind)
                assert p["algo"] not in ("nvls", "hybrid"), (kind, nbytes, p)
        sym = cc.empty(4096, fmt)
        plain = torch.zeros(4096, dtype=fmt, device="cuda")
        for t in (sym, plain):
            assert cc.plan(t)["algo"] not in ("nvls", "hybrid")
            for algo in ("nvls", "hybrid"):
                with pytest.raises(Exception, match="no float8"):
                    cc.allreduce(t, algo=algo)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.gpu
def test_process_group_cuda():
    _pg_run(["cuda"], min(torch.cuda.device_count(), 2))
