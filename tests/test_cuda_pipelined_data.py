"""allgather(v), gather(v) and reduce_scatter of plain CUDA tensors larger than the staging pool.

Every rank's context has a 1 MiB pool, so its bulk region is 512 KiB and the payloads below (a
few MB) run the pipelined kernels of pipeline_kernels.cu instead of the staged copy. Ranks are
threads on cuda:0, each on its own stream; expected values come from torch on the CPU.
"""
import os
import subprocess
import sys
import tempfile
import threading
from datetime import timedelta

import pytest
import torch

import gloo_b200 as gb
from gloo_b200 import ReduceOp
from gloo_b200.ops import cuda as gcu

pytestmark = pytest.mark.gpu

STAGE = 1 << 20
BULK = STAGE // 2  # the pool minus its two one-shot halves (a quarter each at this size)
SIZES = [2, 3, 4, 8]
E4M3 = torch.float8_e4m3fn


def _cc(ctx):
    cc = gcu.CudaContext(ctx, 0, stage_bytes=STAGE)
    cc.set_timeout(60000)
    return cc


def _bytes(t):
    return t.contiguous().view(torch.uint8).cpu()


def _random(n, dtype, seed):
    """n elements of arbitrary bit patterns (NaN codes included: results are compared as bytes)."""
    g = torch.Generator().manual_seed(seed)
    es = torch.empty((), dtype=dtype).element_size()
    return torch.randint(0, 256, (n * es,), generator=g, dtype=torch.uint8).view(dtype)


def _view(n, dtype, shift, fill=0):
    """A CUDA tensor of n elements that starts `shift` elements into its allocation."""
    base = torch.full((n + shift,), fill, dtype=torch.uint8 if dtype == E4M3 else dtype, device="cuda")
    return base.view(dtype)[shift:shift + n] if dtype == E4M3 else base[shift:shift + n]


# ---- allgather / allgatherv -------------------------------------------------------------------


def _ag_counts(P, es, kind):
    if kind == "equal":
        return [(3 << 20) // P // es + 3] * P
    # rank 0 sends nothing, rank 1 much more than the others
    return [0 if r == 0 else ((1536 << 10) + 5 if r == 1 else (96 << 10) + 7 * r) // es for r in range(P)]


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bfloat16, torch.float32, E4M3])
@pytest.mark.parametrize("size", SIZES)
def test_allgather(size, dtype):
    es = torch.empty((), dtype=dtype).element_size()

    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        for kind in ("equal", "uneven"):
            counts = _ag_counts(size, es, kind)
            assert sum(counts) * es > BULK
            ins = [_random(c, dtype, 100 * r + c) for r, c in enumerate(counts)]
            want = _bytes(torch.cat(ins))
            offs = [sum(counts[:r]) for r in range(size)]
            for mode in ("aligned", "offset", "in_place"):
                shift = 1 if mode == "offset" else 0
                out = _view(sum(counts), dtype, shift, fill=7)
                if mode == "in_place":
                    out[offs[me]:offs[me] + counts[me]].copy_(ins[me])
                    inp = out[offs[me]:offs[me] + counts[me]]
                else:
                    inp = _view(counts[me], dtype, shift)
                    inp.copy_(ins[me])
                if kind == "equal":
                    cc.allgather(out, inp)
                else:
                    cc.allgatherv(out, inp, counts)
                cc.synchronize()
                assert torch.equal(_bytes(out), want), (kind, mode)
            # the same call into a registered output (zero copy) gives the same bytes
            sym = cc.empty(sum(counts), dtype)
            inp = _view(counts[me], dtype, 0)
            inp.copy_(ins[me])
            cc.allgatherv(sym, inp, counts)
            cc.synchronize()
            assert torch.equal(_bytes(sym), want), kind
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", SIZES)
def test_gather(size):
    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        for counts in ([(1 << 20) // size + 1] * size, [(700 << 10) if r == size - 1 else 3 * r for r in range(size)]):
            ins = [_random(c, torch.uint8, 7 * r + c) for r, c in enumerate(counts)]
            for root in (0, size - 1):
                out = torch.full((sum(counts),), 0xA5, dtype=torch.uint8, device="cuda")
                inp = ins[me].cuda()
                cc.gatherv(out, inp, counts, root=root)
                cc.synchronize()
                if me == root:
                    assert torch.equal(out.cpu(), torch.cat(ins)), root
                else:
                    assert bool((out == 0xA5).all()), "a non-root rank's output was written"
                cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- reduce_scatter ------------------------------------------------------------------------------

OPS = {"sum": ReduceOp.SUM, "max": ReduceOp.MAX, "min": ReduceOp.MIN, "product": ReduceOp.PRODUCT}
TOL = {torch.float32: (1e-5, 1e-5), torch.bfloat16: (8e-3, 1e-2), torch.float16: (1e-3, 1e-3)}


def _rs_counts(P, es, kind):
    per = (1536 << 10) // P // es
    if kind == "even":
        return [per] * P
    return [0 if r == P - 1 else per + 37 * r + 1 for r in range(P)]  # one empty share


def _ints(n, op, seed):
    """Small integers whose reduction over up to 8 ranks is exact in every dtype tested."""
    g = torch.Generator().manual_seed(seed)
    if op == "product":
        return torch.tensor([-1.0, 1.0, 2.0])[torch.randint(0, 3, (n,), generator=g)]
    return torch.randint(-8, 9, (n,), generator=g).double()


def _reduce(xs, op):
    r = xs[0].clone()
    for x in xs[1:]:
        r = {"sum": torch.add, "max": torch.maximum, "min": torch.minimum, "product": torch.mul}[op](r, x)
    return r


def _e4m3_codes(n, seed):
    """Every finite e4m3 value (sums of up to 8 are exact in fp32)."""
    g = torch.Generator().manual_seed(seed)
    b = torch.randint(0, 256, (n,), generator=g, dtype=torch.int32)
    b = torch.where((b & 0x7F) == 0x7F, b & 0x80, b)
    return b.to(torch.uint8).view(E4M3)


def _sat_e4m3(x):
    m = torch.finfo(E4M3).max
    return torch.clamp(x.float(), -m, m).to(E4M3)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.int32, E4M3])
@pytest.mark.parametrize("size", SIZES)
def test_reduce_scatter(size, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    floating = dtype != torch.int32

    def run(cc, full, counts, op, scale, mode):
        """reduce_scatter of this rank's `full` input; returns my share of the result (CPU)."""
        me = cc.rank
        off = sum(counts[:me])
        shift = 1 if mode == "offset" else 0
        inp = _view(full.numel(), dtype, shift)
        inp.copy_(full.to(dtype) if dtype != E4M3 else full)
        if mode == "in_place":
            out = inp[off:off + counts[me]]
        else:
            out = _view(counts[me], dtype, shift)
        cc.reduce_scatter(out, inp, counts, op=OPS[op], scale=scale)
        cc.synchronize()
        return out.cpu()

    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        for kind in ("even", "uneven"):
            counts = _rs_counts(size, es, kind)
            n = sum(counts)
            assert n * es > BULK
            off = sum(counts[:me])
            mine = slice(off, off + counts[me])
            # integer-valued data: exact for every op
            for op in OPS:
                for mode in ("aligned", "offset", "in_place"):
                    xs = [_ints(n, op, 1000 * r + len(op)) for r in range(size)]
                    if dtype == E4M3:
                        xs = [x.to(E4M3) for x in xs]
                        got = run(cc, xs[me], counts, op, 1.0, mode)
                        want = _sat_e4m3(_reduce([x.float() for x in xs], op)[mine])
                        assert torch.equal(_bytes(got), _bytes(want)), (kind, op, mode)
                    else:
                        got = run(cc, xs[me], counts, op, 1.0, mode)
                        want = _reduce(xs, op)[mine].to(dtype)
                        assert torch.equal(got, want), (kind, op, mode)
            if not floating:
                continue
            # random data, averaged: scale = 1/P inside the kernel, one rounding
            scale = 1.0 / size
            for mode in ("aligned", "offset", "in_place"):
                if dtype == E4M3:
                    xs = [_e4m3_codes(n, 17 * r + 3) for r in range(size)]
                    got = run(cc, xs[me], counts, "sum", scale, mode)
                    s = _reduce([x.float() for x in xs], "sum")[mine]
                    want = _sat_e4m3(s * torch.tensor(scale, dtype=torch.float32))
                    assert torch.equal(_bytes(got), _bytes(want)), (kind, mode)
                else:
                    g = torch.Generator().manual_seed(5)
                    xs = [torch.randn(n, generator=g, dtype=torch.float64).to(dtype) for _ in range(size)]
                    got = run(cc, xs[me], counts, "sum", scale, mode)
                    want = _reduce([x.double() for x in xs], "sum")[mine] * scale
                    rtol, atol = TOL[dtype]
                    torch.testing.assert_close(got.double(), want, rtol=rtol, atol=atol)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- the pool rules: the new calls between the other users of the pool -----------------------


@pytest.mark.parametrize("size", [2, 4])
def test_mixed_sequence(size):
    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        big = (768 << 10) // 4      # floats per rank: allgather output and reduce_scatter input > pool
        for rnd in range(20):
            base = float(rnd * 10)
            step = rnd % 5
            if step == 0:            # pipelined allgather
                out = torch.empty(big * size, device="cuda")
                cc.allgather(out, torch.full((big,), base + me, device="cuda"))
                cc.synchronize()
                want = torch.cat([torch.full((big,), base + r) for r in range(size)])
                assert torch.equal(out.cpu(), want), rnd
            elif step == 1:          # pipelined reduce_scatter
                inp = torch.arange(big * size, dtype=torch.float32, device="cuda") % 64 + base + me
                out = torch.empty(big, device="cuda")
                cc.reduce_scatter(out, inp)
                cc.synchronize()
                full = (torch.arange(big * size, dtype=torch.float32) % 64 + base) * size + size * (size - 1) / 2
                assert torch.equal(out.cpu(), full[me * big:(me + 1) * big]), rnd
            elif step == 2:          # LL allreduce, then the pipelined allreduce
                for n, algo in ((1000, "ll"), (1 << 20, "pipelined")):
                    t = torch.full((n,), base + me, device="cuda")
                    cc.allreduce(t, algo=algo)
                    cc.synchronize()
                    assert bool((t.cpu() == base * size + size * (size - 1) / 2).all()), (rnd, algo)
            elif step == 3:          # staged broadcast (cut into pool-sized pieces)
                t = torch.full((300000,), base + me, device="cuda")
                cc.broadcast(t, root=size - 1)
                cc.synchronize()
                assert bool((t.cpu() == base + size - 1).all()), rnd
            else:                    # staged allgatherv that fits the pool
                counts = [1000 + 3 * r for r in range(size)]
                out = torch.empty(sum(counts), device="cuda")
                cc.allgatherv(out, torch.full((counts[me],), base + me, device="cuda"), counts)
                cc.synchronize()
                want = torch.cat([torch.full((c,), base + r) for r, c in enumerate(counts)])
                assert torch.equal(out.cpu(), want), rnd
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- CUDA graph ------------------------------------------------------------------------------------


@pytest.mark.parametrize("size", [2, 3])
def test_cuda_graph(size):
    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        n = (640 << 10) // 4
        ag_in, ag_out = torch.empty(n, device="cuda"), torch.empty(n * size, device="cuda")
        rs_in, rs_out = torch.empty(n * size, device="cuda"), torch.empty(n, device="cuda")

        def load(seed):
            ag_in.copy_(torch.arange(n, dtype=torch.float32) + seed * 100 + me)
            rs_in.copy_(torch.arange(n * size, dtype=torch.float32) % 128 + seed + me)

        def check(seed):
            want = torch.cat([torch.arange(n, dtype=torch.float32) + seed * 100 + r for r in range(size)])
            assert torch.equal(ag_out.cpu(), want), seed
            full = (torch.arange(n * size, dtype=torch.float32) % 128 + seed) * size + size * (size - 1) / 2
            assert torch.equal(rs_out.cpu(), full[me * n:(me + 1) * n]), seed

        stream = torch.cuda.current_stream()
        load(1)
        cc.allgather(ag_out, ag_in)  # warm-up outside the graph
        cc.reduce_scatter(rs_out, rs_in)
        cc.synchronize()
        check(1)
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            cc.allgather(ag_out, ag_in)
            cc.reduce_scatter(rs_out, rs_in)
        cc.pc.host_barrier()
        for seed in (2, 3, 4):
            load(seed)
            stream.synchronize()
            cc.pc.host_barrier()
            g.replay()
            cc.synchronize()
            check(seed)
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- torch.distributed backend ------------------------------------------------------------------


def _pg_collectives(all_gather, reduce_scatter_avg, rank, size, dev):
    """all_gather_into_tensor and reduce_scatter_tensor (AVG) beyond a 1 MiB pool."""
    n = (400 << 10) // 2 + 3                       # bf16 elements per rank
    inp = (torch.arange(n, dtype=torch.float32) % 100 + rank).to(torch.bfloat16).to(dev)
    out = torch.empty(n * size, dtype=torch.bfloat16, device=dev)
    all_gather(out, inp)
    want = torch.cat([(torch.arange(n, dtype=torch.float32) % 100 + r).to(torch.bfloat16) for r in range(size)])
    assert torch.equal(out.cpu(), want)
    full = torch.arange(n * size, dtype=torch.float32) % 50 * size + rank * size
    res = torch.empty(n, dtype=torch.float32, device=dev)
    reduce_scatter_avg(res, full.to(dev))
    # mean over ranks of (i % 50) * size + r * size = (i % 50) * size + size * (size - 1) / 2
    want = (torch.arange(n * size, dtype=torch.float32) % 50 * size + size * (size - 1) / 2)[rank * n:(rank + 1) * n]
    torch.testing.assert_close(res.cpu(), want, rtol=1e-6, atol=1e-5)


@pytest.mark.parametrize("size", [2, 4])
def test_process_group_threads(size, monkeypatch):
    """GlbProcessGroup built directly by threads over one HashStore, every rank on cuda:0 with
    its own current stream."""
    import torch.distributed as dist
    from torch._C._distributed_c10d import ReduceScatterOptions

    from gloo_b200.parallel.process_group import GlbProcessGroup

    monkeypatch.setenv("GLB_PG_STAGE_MB", "1")
    store = dist.HashStore()
    errors = [None] * size

    def run(rank):
        try:
            torch.cuda.set_device(0)
            with torch.cuda.stream(gcu.new_stream(0)):
                pg = GlbProcessGroup(store, rank, size, timedelta(seconds=60))
                opts = ReduceScatterOptions()
                opts.reduceOp = dist.ReduceOp.AVG
                _pg_collectives(lambda o, i: pg._allgather_base(o, i).wait(),
                                lambda o, i: pg._reduce_scatter_base(o, i, opts).wait(), rank, size,
                                torch.device("cuda", 0))
                torch.cuda.current_stream().synchronize()
                pg._cc(torch.empty(1, device="cuda")).pc.host_barrier()
        except BaseException as e:  # noqa: BLE001
            errors[rank] = e

    threads = [threading.Thread(target=run, args=(r,)) for r in range(size)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=240)
    assert not any(t.is_alive() for t in threads), "a rank did not finish"
    for e in errors:
        if e is not None:
            raise e


_WORKER = """
import os, sys
sys.path.insert(0, {root!r})
sys.path.insert(0, {tests!r})
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")
os.environ["GLB_PG_STAGE_MB"] = "1"
import torch, torch.distributed as dist
import gloo_b200.parallel.process_group  # registers "glb"
from test_cuda_pipelined_data import _pg_collectives
rank, size = int(sys.argv[1]), int(sys.argv[2])
torch.cuda.set_device(rank)
dist.init_process_group("glb", init_method="file://" + {init!r}, rank=rank, world_size=size)
_pg_collectives(dist.all_gather_into_tensor,
                lambda o, i: dist.reduce_scatter_tensor(o, i, op=dist.ReduceOp.AVG), rank, size,
                torch.device("cuda", rank))
torch.cuda.synchronize()
dist.barrier()
dist.destroy_process_group()
print("rank", rank, "ok", flush=True)
"""


def test_process_group_multiprocess():
    """One process per GPU (never two processes on one GPU: their kernels would time-slice)."""
    size = min(torch.cuda.device_count(), 4)
    if size < 2:
        pytest.skip("needs at least 2 GPUs")
    here = os.path.dirname(os.path.abspath(__file__))
    init = os.path.join(tempfile.mkdtemp(prefix="glb_pg_pipe_"), "init")
    code = _WORKER.format(root=os.path.dirname(here), tests=here, init=init)
    procs = [subprocess.Popen([sys.executable, "-c", code, str(r), str(size)], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(size)]
    outs = [p.communicate(timeout=300) for p in procs]
    for r, (p, (out, err)) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r} ok" in out, (r, p.returncode, out[-500:], err[-2000:])
