"""alltoall(v), scatter and reduce of plain CUDA tensors larger than the staging pool.

Every rank's context has a 1 MiB pool, so its bulk region is 512 KiB and the payloads below (a
few MB) run the pipelined kernels of pipeline_kernels.cu instead of the staged copy. The plain
alltoallv always runs the pipelined kernel. Ranks are threads on cuda:0, each on its own stream;
expected values come from torch on the CPU.
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
from gloo_b200.ops import cuda as gcu
from test_cuda_pipelined_data import BULK, E4M3, OPS, SIZES, TOL, _bytes, _cc, _e4m3_codes, _ints, _random, \
    _reduce, _sat_e4m3, _view

pytestmark = pytest.mark.gpu


# ---- alltoall / alltoallv -----------------------------------------------------------------------


@pytest.mark.parametrize("dtype", [torch.uint8, torch.bfloat16, torch.float32, E4M3])
@pytest.mark.parametrize("size", SIZES)
def test_alltoall(size, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    per = (1 << 20) // size // es + 3  # elements per block: the whole exchange is > the bulk region

    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        ins = [_random(per * size, dtype, 31 * r + size) for r in range(size)]
        want = _bytes(torch.cat([ins[q][me * per:(me + 1) * per] for q in range(size)]))
        assert per * size * es > BULK
        for shift in (0, 1):
            inp = _view(per * size, dtype, shift)
            inp.copy_(ins[me])
            out = _view(per * size, dtype, shift, fill=7)
            cc.alltoall(out, inp)
            cc.synchronize()
            assert torch.equal(_bytes(out), want), shift
        # the same call into a registered output (zero copy) gives the same bytes
        sym = cc.empty(per * size, dtype)
        inp = _view(per * size, dtype, 0)
        inp.copy_(ins[me])
        cc.alltoall(sym, inp)
        cc.synchronize()
        assert torch.equal(_bytes(sym), want)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def _run_alltoallv(cc, split, seed):
    """alltoallv of uint8 blocks: split[s][d] bytes from rank s to rank d. Returns (got, want)."""
    me, size = cc.rank, len(split)
    blocks = [[_random(split[s][d], torch.uint8, seed + 97 * s + d) for d in range(size)] for s in range(size)]
    inp = torch.cat(blocks[me]).cuda()
    recv = [split[s][me] for s in range(size)]
    out = torch.full((sum(recv),), 0xA5, dtype=torch.uint8, device="cuda")
    cc.alltoallv(out, recv, inp, split[me])
    cc.synchronize()
    return out.cpu(), torch.cat([blocks[s][me] for s in range(size)])


@pytest.mark.parametrize("size", SIZES)
def test_alltoallv(size):
    big = BULK + 4099  # one block larger than the whole bulk region

    def fn(ctx):
        cc = _cc(ctx)
        # uneven, with empty blocks (and an empty diagonal entry on rank 1)
        uneven = [[0 if (s + 2 * d) % 3 == 1 else (s + 1) * 7919 + d * 131 for d in range(size)] for s in range(size)]
        uneven[0][size - 1] = big
        # small: the whole exchange fits the pool (the path that replaced the staged one)
        small = [[(s * size + d) % 5 * 33 + 1 for d in range(size)] for s in range(size)]
        # receive totals on both sides of the bulk size: rank 0 receives more than the bulk region,
        # every other rank much less
        skew = [[(BULK // size + 1000 if d == 0 else 100 + s) for d in range(size)] for s in range(size)]
        for name, split in (("uneven", uneven), ("small", small), ("skew", skew)):
            got, want = _run_alltoallv(cc, split, len(name))
            assert torch.equal(got, want), name
        assert sum(skew[s][0] for s in range(size)) > BULK > sum(skew[s][1] for s in range(size))
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", [2, 3])
def test_alltoall_overlap_raises(size):
    """Overlapping input and output raise ValueError on every rank, so no rank launches."""
    def fn(ctx):
        cc = _cc(ctx)
        n = BULK  # per block: past the staged path
        buf = torch.zeros(n * size + 16, dtype=torch.uint8, device="cuda")
        with pytest.raises(ValueError):
            cc.alltoall(buf[16:], buf[:n * size])
        with pytest.raises(ValueError):
            cc.alltoallv(buf[8:8 + 64 * size], [64] * size, buf[:64 * size], [64] * size)
        # the context is still usable
        got, want = _run_alltoallv(cc, [[1000 + s + d for d in range(size)] for s in range(size)], 3)
        assert torch.equal(got, want)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- scatter --------------------------------------------------------------------------------------


@pytest.mark.parametrize("size", SIZES)
def test_scatter(size):
    per = BULK + 333  # bytes per rank: more than the bulk region

    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        for root in (0, size - 1):
            full = _random(per * size, torch.uint8, 5 * root + size)
            for shift in (0, 1):
                inp = None
                if me == root:
                    inp = _view(per * size, torch.uint8, shift)
                    inp.copy_(full)
                out = _view(per, torch.uint8, shift, fill=7)
                cc.scatter(out, inp, root=root)
                cc.synchronize()
                assert torch.equal(out.cpu(), full[me * per:(me + 1) * per]), (root, shift)
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- reduce ---------------------------------------------------------------------------------------


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16, torch.int32, E4M3])
@pytest.mark.parametrize("size", SIZES)
def test_reduce(size, dtype):
    es = torch.empty((), dtype=dtype).element_size()
    n = (1536 << 10) // es + 2 * size + 1  # > half the bulk region, not a multiple of P

    def run(cc, x, op, root, none_out=False):
        inp = _view(n, dtype, 1)
        inp.copy_(x.to(dtype) if dtype != E4M3 else x)
        if cc.rank != root and none_out:
            cc.reduce(None, inp, root=root, op=OPS[op])
            cc.synchronize()
            return None
        out = _view(n, dtype, 1, fill=0x5B)
        sentinel = _bytes(out)
        cc.reduce(out, inp, root=root, op=OPS[op])
        cc.synchronize()
        if cc.rank != root:
            assert torch.equal(_bytes(out), sentinel), "a non-root rank's output was written"
        return out.cpu()

    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        assert n * es > BULK // 2
        for root in (0, size - 1):
            # integer-valued data: exact for every op
            for op in OPS:
                xs = [_ints(n, op, 1000 * r + len(op)) for r in range(size)]
                if dtype == E4M3:
                    xs = [x.to(E4M3) for x in xs]
                    got = run(cc, xs[me], op, root)
                    if me == root:
                        assert torch.equal(_bytes(got), _bytes(_sat_e4m3(_reduce([x.float() for x in xs], op)))), op
                else:
                    got = run(cc, xs[me], op, root, none_out=op == "max")
                    if me == root:
                        assert torch.equal(got, _reduce(xs, op).to(dtype)), (root, op)
            if dtype == torch.int32:
                continue
            # random data
            if dtype == E4M3:
                xs = [_e4m3_codes(n, 17 * r + 3) for r in range(size)]
                got = run(cc, xs[me], "sum", root)
                if me == root:
                    assert torch.equal(_bytes(got), _bytes(_sat_e4m3(_reduce([x.float() for x in xs], "sum"))))
            else:
                g = torch.Generator().manual_seed(5)
                xs = [torch.randn(n, generator=g, dtype=torch.float64).to(dtype) for _ in range(size)]
                got = run(cc, xs[me], "sum", root)
                if me == root:
                    rtol, atol = TOL[dtype]
                    torch.testing.assert_close(got.double(), _reduce([x.double() for x in xs], "sum"), rtol=rtol,
                                               atol=atol * size)
            cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- the pool rules: the new calls between the other users of the pool -----------------------


@pytest.mark.parametrize("size", [2, 4])
def test_mixed_sequence(size):
    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        big = (768 << 10) // 4  # floats per rank: more than the pool
        for rnd in range(20):
            base = float(rnd * 10)
            step = rnd % 5
            if step == 0:  # all-empty alltoallv directly followed by a pipelined alltoall, then staged allgather
                empty = torch.empty(0, device="cuda")
                cc.alltoallv(empty, [0] * size, torch.empty(0, device="cuda"), [0] * size)
                inp = torch.arange(big, dtype=torch.float32, device="cuda") + base + 1000 * me
                out = torch.empty(big, device="cuda")
                cc.alltoall(out, inp)
                per = big // size
                want = torch.cat([torch.arange(me * per, (me + 1) * per, dtype=torch.float32) + base + 1000 * q
                                  for q in range(size)])
                small = 30000  # staged: more than the LL limit, the whole output fits the pool
                ag = torch.empty(small * size, device="cuda")
                cc.allgather(ag, torch.full((small,), base + me, device="cuda"))
                cc.synchronize()
                assert torch.equal(out.cpu(), want), rnd
                assert torch.equal(ag.cpu(), torch.cat([torch.full((small,), base + r) for r in range(size)])), rnd
            elif step == 1:  # pipelined reduce, then LL allreduce
                inp = torch.arange(big, dtype=torch.float32, device="cuda") % 64 + base + me
                out = torch.empty(big, device="cuda")
                cc.reduce(out, inp, root=rnd % size)
                t = torch.full((1000,), base + me, device="cuda")
                cc.allreduce(t, algo="ll")
                cc.synchronize()
                if me == rnd % size:
                    want = (torch.arange(big, dtype=torch.float32) % 64 + base) * size + size * (size - 1) / 2
                    assert torch.equal(out.cpu(), want), rnd
                assert bool((t.cpu() == base * size + size * (size - 1) / 2).all()), rnd
            elif step == 2:  # pipelined scatter, then pipelined reduce_scatter
                full = torch.arange(big * size, dtype=torch.float32, device="cuda") + base if me == 0 else None
                out = torch.empty(big, device="cuda")
                cc.scatter(out, full, root=0)
                rs_in = torch.arange(big * size, dtype=torch.float32, device="cuda") % 64 + base + me
                rs_out = torch.empty(big, device="cuda")
                cc.reduce_scatter(rs_out, rs_in)
                cc.synchronize()
                assert torch.equal(out.cpu(), torch.arange(me * big, (me + 1) * big, dtype=torch.float32) + base), rnd
                full_rs = (torch.arange(big * size, dtype=torch.float32) % 64 + base) * size + size * (size - 1) / 2
                assert torch.equal(rs_out.cpu(), full_rs[me * big:(me + 1) * big]), rnd
            elif step == 3:  # staged broadcast, then a small alltoallv
                t = torch.full((300000,), base + me, device="cuda")
                cc.broadcast(t, root=size - 1)
                got, want = _run_alltoallv(cc, [[500 + 3 * s + d for d in range(size)] for s in range(size)], rnd)
                assert bool((t.cpu() == base + size - 1).all()), rnd
                assert torch.equal(got, want), rnd
            else:  # pipelined alltoallv with uneven blocks
                split = [[(s + d + rnd) % 3 * 200000 for d in range(size)] for s in range(size)]
                got, want = _run_alltoallv(cc, split, rnd)
                assert torch.equal(got, want), rnd
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- CUDA graph ------------------------------------------------------------------------------------


@pytest.mark.parametrize("size", [2, 3])
def test_cuda_graph(size):
    def fn(ctx):
        cc = _cc(ctx)
        me = ctx.rank
        n = (640 << 10) // 4 // size * size
        a_in, a_out = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")
        r_in, r_out = torch.empty(n, device="cuda"), torch.empty(n, device="cuda")

        def load(seed):
            a_in.copy_(torch.arange(n, dtype=torch.float32) + seed * 100 + 1000 * me)
            r_in.copy_(torch.arange(n, dtype=torch.float32) % 128 + seed + me)

        def check(seed):
            per = n // size
            want = torch.cat([torch.arange(me * per, (me + 1) * per, dtype=torch.float32) + seed * 100 + 1000 * q
                              for q in range(size)])
            assert torch.equal(a_out.cpu(), want), seed
            if me == 0:
                want = (torch.arange(n, dtype=torch.float32) % 128 + seed) * size + size * (size - 1) / 2
                assert torch.equal(r_out.cpu(), want), seed

        stream = torch.cuda.current_stream()
        load(1)
        cc.alltoall(a_out, a_in)  # warm-up outside the graph
        cc.reduce(r_out, r_in, root=0)
        cc.synchronize()
        check(1)
        cc.pc.host_barrier()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=stream, capture_error_mode="thread_local"):
            cc.alltoall(a_out, a_in)
            cc.reduce(r_out, r_in, root=0)
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


def _pg_exchange(all_to_all_single, all_to_all, scatter, reduce, rank, size, dev):
    """all_to_all_single (with and without splits), all_to_all, scatter and reduce (SUM, AVG)
    beyond a 1 MiB pool."""
    per = (600 << 10) // 4 // size  # floats per block
    inp = torch.arange(per * size, dtype=torch.float32).to(dev) + 10000 * rank
    out = torch.empty(per * size, device=dev)
    all_to_all_single(out, inp, None, None)
    want = torch.cat([torch.arange(rank * per, (rank + 1) * per, dtype=torch.float32) + 10000 * q for q in range(size)])
    assert torch.equal(out.cpu(), want)
    # splits: rank s sends (s + d + 1) * per // 2 elements to rank d
    send = [(rank + d + 1) * per // 2 for d in range(size)]
    recv = [(s + rank + 1) * per // 2 for s in range(size)]
    inp = torch.cat([torch.full((send[d],), float(100 * rank + d)) for d in range(size)]).to(dev)
    out = torch.empty(sum(recv), device=dev)
    all_to_all_single(out, inp, recv, send)
    assert torch.equal(out.cpu(), torch.cat([torch.full((recv[s],), float(100 * s + rank)) for s in range(size)]))
    ins = [torch.full((per * (d + 1),), float(100 * rank + d), device=dev) for d in range(size)]
    outs = [torch.empty(per * (rank + 1), device=dev) for _ in range(size)]
    all_to_all(outs, ins)
    for s in range(size):
        assert bool((outs[s].cpu() == 100 * s + rank).all())
    root = size - 1
    n = 3 * per * size
    parts = [torch.arange(n, dtype=torch.float32).to(dev) + 7 * r for r in range(size)] if rank == root else None
    got = torch.empty(n, device=dev)
    scatter(got, parts, root)
    assert torch.equal(got.cpu(), torch.arange(n, dtype=torch.float32) + 7 * rank)
    for op, div in (("sum", 1), ("avg", size)):
        t = (torch.arange(n, dtype=torch.float32) % 50 * size + rank * size).to(dev)
        reduce(t, root, op)
        if rank == root:
            want = (torch.arange(n, dtype=torch.float32) % 50 * size * size + size * size * (size - 1) / 2) / div
            torch.testing.assert_close(t.cpu(), want, rtol=1e-6, atol=1e-4)


def _dist_ops(pg=None):
    import torch.distributed as dist

    def a2a_single(o, i, osp, isp):
        if pg is None:
            dist.all_to_all_single(o, i, osp, isp)
        else:
            pg.alltoall_base(o, i, osp or [], isp or []).wait()

    def a2a(outs, ins):
        if pg is None:
            dist.all_to_all(outs, ins)
        else:
            pg.alltoall(outs, ins).wait()

    def scatter(o, parts, root):
        if pg is None:
            dist.scatter(o, parts, src=root)
        else:
            from torch._C._distributed_c10d import ScatterOptions
            opts = ScatterOptions()
            opts.rootRank = root
            pg.scatter([o], [parts] if parts is not None else [], opts).wait()

    def reduce(t, root, op):
        rop = dist.ReduceOp.SUM if op == "sum" else dist.ReduceOp.AVG
        if pg is None:
            dist.reduce(t, dst=root, op=rop)
        else:
            from torch._C._distributed_c10d import ReduceOptions
            opts = ReduceOptions()
            opts.rootRank = root
            opts.reduceOp = rop
            pg.reduce([t], opts).wait()

    return a2a_single, a2a, scatter, reduce


@pytest.mark.parametrize("size", [2, 4])
def test_process_group_threads(size, monkeypatch):
    """GlbProcessGroup built directly by threads over one HashStore, every rank on cuda:0 with
    its own current stream."""
    import torch.distributed as dist

    from gloo_b200.parallel.process_group import GlbProcessGroup

    monkeypatch.setenv("GLB_PG_STAGE_MB", "1")
    store = dist.HashStore()
    errors = [None] * size

    def run(rank):
        try:
            torch.cuda.set_device(0)
            with torch.cuda.stream(gcu.new_stream(0)):
                pg = GlbProcessGroup(store, rank, size, timedelta(seconds=60))
                _pg_exchange(*_dist_ops(pg), rank, size, torch.device("cuda", 0))
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
from test_cuda_pipelined_exchange import _dist_ops, _pg_exchange
rank, size = int(sys.argv[1]), int(sys.argv[2])
torch.cuda.set_device(rank)
dist.init_process_group("glb", init_method="file://" + {init!r}, rank=rank, world_size=size)
_pg_exchange(*_dist_ops(), rank, size, torch.device("cuda", rank))
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
    init = os.path.join(tempfile.mkdtemp(prefix="glb_pg_a2a_"), "init")
    code = _WORKER.format(root=os.path.dirname(here), tests=here, init=init)
    procs = [subprocess.Popen([sys.executable, "-c", code, str(r), str(size)], stdout=subprocess.PIPE,
                              stderr=subprocess.PIPE, text=True) for r in range(size)]
    outs = [p.communicate(timeout=300) for p in procs]
    for r, (p, (out, err)) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r} ok" in out, (r, p.returncode, out[-500:], err[-2000:])
