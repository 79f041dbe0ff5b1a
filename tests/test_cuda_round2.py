"""GPU tests for the fused epilogues, the flag-in-data (LL) kernels, the pipelined
plain-pointer allreduce, point-to-point transfers, device-side failure detection and the
virtual-rank loopback self-test. Numerics are compared against a plain PyTorch fp32/fp64
reference of the same operation. Ranks are threads sharing cuda:0 (see test_cuda_allreduce.py)."""
import os

import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu

pytestmark = pytest.mark.gpu


def _inp(rank, size, count, dtype=torch.float32):
    return (torch.arange(count, dtype=torch.float64) % 61 * size + rank).to(dtype).cuda()


def _exp(size, count):
    return (torch.arange(count, dtype=torch.float64) % 61) * size * size + size * (size - 1) / 2


def _sync():
    torch.cuda.current_stream().synchronize()


# ---- loopback self-test + failure detection (single rank, profiler safe) ---------------------

def test_loopback_selftest_covers_hot_kernels():
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=64 << 20)
        return cc.pc.loopback_selftest(torch.cuda.current_stream().cuda_stream, 1 << 16)

    (res,) = gb.spawn_threads(1, fn, cuda_device=0)
    names = " ".join(r["name"] for r in res)
    for frag in ("twoShotAllreduceKernel<float,8,2>", "twoShotAllreduceKernel<float,2,4>", "reducePullKernel",
                 "oneShotAllreduceKernel", "llAllreduceKernel", "pipelinedAllreduceKernel", "p2pKernel",
                 "broadcastKernel", "gatherPushKernel", "alltoallPushKernel", "castAllreduceKernel", "scheduleKernel"):
        assert frag in names
    bad = [r for r in res if not r["ok"]]
    assert not bad, bad


def test_device_timeout_poisons_context_and_gpu_survives():
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        raised, ms = cc.pc.loopback_timeout_test(torch.cuda.current_stream().cuda_stream, 300)
        assert raised, "the abandoned barrier did not poison the context"
        assert 250 <= ms <= 1500, ms
        assert cc.pc.poisoned()
        with pytest.raises(gb.IoError):
            cc.allreduce(torch.ones(8, device="cuda"))
        # the GPU is still usable
        x = torch.arange(10, device="cuda").float().sum().item()
        assert x == 45.0
        return True

    assert gb.spawn_threads(1, fn, cuda_device=0) == [True]


# ---- LL one-shot -----------------------------------------------------------------------------

@pytest.mark.parametrize("size", [2, 3, 4, 8])
def test_ll_allreduce_sizes_and_dtypes(size):
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for dtype, tol in ((torch.float32, 1e-6), (torch.float16, 1e-2), (torch.bfloat16, 3e-2), (torch.int32, 0),
                           (torch.float64, 1e-12), (torch.int64, 0), (torch.uint8, 0)):
            for count in (1, 2, 3, 5, 257, 4099):
                small = 3 if dtype == torch.uint8 else 61
                base = (torch.arange(count, dtype=torch.float64) % small)
                t = (base + ctx.rank).to(dtype).cuda()
                exp = sum((base + r).to(dtype).double() for r in range(size))
                for rep in range(3):  # parity halves are reused every other launch
                    u = t.clone()
                    cc.allreduce(u, algo="ll")
                    _sync()
                    torch.testing.assert_close(u.double().cpu(), exp.to(dtype).double(), rtol=tol, atol=tol)
        # unaligned input / output views
        big = _inp(ctx.rank, size, 1001)
        v = big[1:]
        cc.allreduce(v, algo="ll")
        _sync()
        torch.testing.assert_close(v.double().cpu(), _exp(size, 1001)[1:], rtol=1e-6, atol=0)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def test_auto_picks_ll_for_tiny_and_matches_reference():
    size = 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        t = _inp(ctx.rank, size, 100)
        assert cc.plan(t)["algo"] == "ll"
        cc.allreduce(t)
        _sync()
        torch.testing.assert_close(t.double().cpu(), _exp(size, 100), rtol=1e-6, atol=0)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- fused scale / cast epilogue ------------------------------------------------------------------

@pytest.mark.parametrize("algo", ["ll", "one_shot", "two_shot", "pipelined"])
def test_scale_epilogue_every_variant(algo):
    size = 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        for count in (1000, 70001) if algo not in ("ll",) else (1000, 4000):
            if algo == "one_shot" and count * 4 > 64 * 1024:
                continue
            t = _inp(ctx.rank, size, count)
            if algo == "two_shot":
                cc.register(t)
            cc.allreduce(t, algo=algo, average=True)
            _sync()
            torch.testing.assert_close(t.double().cpu(), _exp(size, count) / size, rtol=1e-6, atol=1e-6)
            for dtype in (torch.bfloat16, torch.float16):
                h = ((torch.arange(count) % 7) + ctx.rank).to(dtype).cuda()
                if algo == "two_shot":
                    cc.register(h)
                cc.allreduce(h, algo=algo, scale=0.5)
                _sync()
                want = sum(((torch.arange(count) % 7) + r).float() for r in range(size)) * 0.5
                torch.testing.assert_close(h.float().cpu(), want.to(dtype).float(), rtol=2e-2, atol=2e-2)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def test_cast_epilogue_registered_and_ll():
    size = 4

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        for count in (8, 1000, 100003):
            src = torch.randn(count, generator=torch.Generator().manual_seed(ctx.rank)).cuda()
            ref = sum(torch.randn(count, generator=torch.Generator().manual_seed(r)) for r in range(size)) / size
            # registered buffers, any size: fp32 in, bf16 / fp16 out, averaged, ONE rounding
            for odt in (torch.bfloat16, torch.float16):
                a = cc.empty(count, torch.float32)
                o = cc.empty(count, odt)
                a.copy_(src)
                cc.allreduce(a, out=o, average=True)
                _sync()
                torch.testing.assert_close(o.float().cpu(), ref.to(odt).float(), rtol=1e-2, atol=1e-2)
            # 16-bit in, fp32 out
            h = cc.empty(count, torch.bfloat16)
            o32 = cc.empty(count, torch.float32)
            h.copy_(src.to(torch.bfloat16))
            cc.allreduce(h, out=o32)
            _sync()
            ref16 = sum(torch.randn(count, generator=torch.Generator().manual_seed(r)).to(torch.bfloat16).float()
                        for r in range(size))
            torch.testing.assert_close(o32.cpu(), ref16, rtol=1e-5, atol=1e-5)
        # plain tensors below the LL limit
        p = torch.full((777,), float(ctx.rank + 1), device="cuda")
        q = torch.empty(777, dtype=torch.bfloat16, device="cuda")
        cc.allreduce(p, out=q)
        _sync()
        assert float(q[5]) == size * (size + 1) / 2
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- pipelined plain-pointer allreduce ---------------------------------------------------------------

@pytest.mark.parametrize("size", [2, 4])
def test_pipelined_allreduce_plain_pointers(size):
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        for count in (70001, 1 << 20, 3_000_003):
            t = _inp(ctx.rank, size, count)
            assert cc.plan(t)["algo"] == "pipelined"
            cc.allreduce(t)
            _sync()
            torch.testing.assert_close(t.double().cpu(), _exp(size, count), rtol=1e-6, atol=0)
            # out of place, unaligned views, small tiles (many pipeline steps)
            src = _inp(ctx.rank, size, count + 1)[1:]
            dst = torch.zeros(count + 3, device="cuda")[3:]
            cc.allreduce(src, out=dst, algo="pipelined", tile=16, blocks=4)
            _sync()
            torch.testing.assert_close(dst.double().cpu(), _exp(size, count + 1)[1:], rtol=1e-6, atol=0)
        for dtype in (torch.bfloat16, torch.int32, torch.float64):
            t = ((torch.arange(500001) % 5) + ctx.rank).to(dtype).cuda()
            cc.allreduce(t, algo="pipelined")
            _sync()
            want = sum(((torch.arange(500001) % 5) + r).to(dtype).double() for r in range(size))
            torch.testing.assert_close(t.double().cpu(), want, rtol=1e-2, atol=1e-2)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- multi-pointer fold inside the collective kernel -----------------------------------------------------

@pytest.mark.parametrize("size", [1, 2, 4])
def test_multi_pointer_is_one_launch(size):
    def fn(ctx):
        ptrs = 3
        stride = size * ptrs
        for count in (100, 4099, 300000):
            for symmetric in (False, True):
                if symmetric and size == 1:
                    continue
                cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20) if size > 1 else None
                ts = []
                for i in range(ptrs):
                    t = cc.empty(count, torch.float32) if (symmetric and i == 0) else torch.empty(count, device="cuda")
                    t.copy_((torch.arange(count, dtype=torch.float64) * stride + ctx.rank * ptrs + i).float())
                    ts.append(t)
                algo = gcu.CudaAllreduceRingChunked(ctx, ts)
                assert algo.launches_per_run() == 1
                before = gb._C.cuda.launch_count()
                algo.set_scale(0.5)
                algo.run()
                exp = 0.5 * (torch.arange(count, dtype=torch.float64) * stride * stride + stride * (stride - 1) / 2)
                for t in ts:
                    torch.testing.assert_close(t.double().cpu(), exp, rtol=1e-6, atol=0)
                if size == 1:
                    assert gb._C.cuda.launch_count() - before == 1
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- uneven / divergent tables (advisor findings) -------------------------------------------------------------

def test_skewed_counts_allgatherv_gatherv_reduce_scatter():
    size = 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=32 << 20)
        counts = [256, 1 << 20]  # 1 KiB vs 4 MiB: the grid must not depend on the local share
        mine = torch.full((counts[ctx.rank],), float(ctx.rank + 1), device="cuda")
        out = torch.zeros(sum(counts), device="cuda")
        cc.allgatherv(out, mine, counts)
        _sync()
        assert float(out[0]) == 1.0 and float(out[255]) == 1.0 and float(out[256]) == 2.0 and float(out[-1]) == 2.0
        g = torch.zeros(sum(counts), device="cuda")
        cc.gatherv(g, mine, counts, root=1)
        _sync()
        if ctx.rank == 1:
            assert float(g[0]) == 1.0 and float(g[-1]) == 2.0
        full = _inp(ctx.rank, size, sum(counts))
        rs = torch.zeros(counts[ctx.rank], device="cuda")
        cc.reduce_scatter(rs, full, counts)
        _sync()
        off = sum(counts[: ctx.rank])
        torch.testing.assert_close(rs.double().cpu(), _exp(size, sum(counts))[off:off + counts[ctx.rank]], rtol=1e-6, atol=0)
        # boundary size from the report: 4103 floats at P=2 -> 513 vs 512 vectors per rank
        t = _inp(ctx.rank, size, 4103)
        r = torch.zeros(4103, device="cuda")
        cc.reduce(r, t, root=0)
        _sync()
        if ctx.rank == 0:
            torch.testing.assert_close(r.double().cpu(), _exp(size, 4103), rtol=1e-6, atol=0)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def test_alltoallv_tables_that_look_uniform_on_one_rank_only():
    size = 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        # rank 0: send = recv = [4, 4]; rank 1: send = [4, 6], recv = [4, 6]
        send = [[4, 4], [4, 6]][ctx.rank]
        recv = [[4, 4], [4, 6]][ctx.rank]
        inp = torch.cat([torch.full((n,), float(ctx.rank * 10 + j)) for j, n in enumerate(send)]).cuda()
        out = torch.full((sum(recv),), -1.0, device="cuda")
        cc.alltoallv(out, recv, inp, send)
        _sync()
        exp = torch.cat([torch.full((n,), float(j * 10 + ctx.rank)) for j, n in enumerate(recv)])
        torch.testing.assert_close(out.cpu(), exp)
        # skewed byte counts and offsets that are only 4-byte aligned
        send = [[3, 100001], [70003, 5]][ctx.rank]
        recv = [[3, 70003], [100001, 5]][ctx.rank]
        inp = torch.cat([torch.full((n,), float(ctx.rank * 10 + j)) for j, n in enumerate(send)]).cuda()
        out = torch.full((sum(recv),), -1.0, device="cuda")
        cc.alltoallv(out, recv, inp, send)
        _sync()
        exp = torch.cat([torch.full((n,), float(j * 10 + ctx.rank)) for j, n in enumerate(recv)])
        torch.testing.assert_close(out.cpu(), exp)
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", [2, 4])
def test_small_allgather_alltoall_use_flag_in_data(size):
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        for n in (1, 3, 250, 2048):
            for dtype in (torch.float32, torch.uint8):
                out = torch.zeros(n * size, dtype=dtype, device="cuda")
                cc.allgather(out, torch.full((n,), ctx.rank + 1, dtype=dtype, device="cuda"))
                a_in = torch.cat([torch.full((n,), ctx.rank * 10 + j, dtype=dtype) for j in range(size)]).cuda()
                a_out = torch.zeros(n * size, dtype=dtype, device="cuda")
                cc.alltoall(a_out, a_in)
                _sync()
                torch.testing.assert_close(out.cpu(), torch.arange(1, size + 1).repeat_interleave(n).to(dtype))
                torch.testing.assert_close(a_out.cpu(), torch.cat([torch.full((n,), j * 10 + ctx.rank, dtype=dtype)
                                                                   for j in range(size)]))
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- point to point ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("size", [2, 4])
def test_p2p_ring_sendrecv_put_get(size):
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        right, left = (ctx.rank + 1) % size, (ctx.rank - 1) % size
        bufs = []
        for n in (1, 1000, 300001, 3_000_000):  # the last one is larger than the mailbox ring
            bufs.append((torch.full((n,), float(ctx.rank), device="cuda"), torch.zeros(n, device="cuda")))
        cc.pc.host_barrier()  # all allocations done before kernels that wait for a peer
        for s, r in bufs:
            cc.sendrecv(s, right, r, left)
        _sync()
        for s, r in bufs:
            assert float(r[0]) == left and float(r[-1]) == left
        if size == 2:
            # separate send / recv kernels on separate streams, both directions at once
            s1, s2 = gcu.new_stream(0), gcu.new_stream(0)
            a = torch.full((2_000_000,), float(ctx.rank + 5), device="cuda")
            b = torch.zeros(2_000_000, device="cuda")
            _sync()
            cc.pc.host_barrier()
            cc.send(a, 1 - ctx.rank, stream=s1)
            cc.recv(b, 1 - ctx.rank, stream=s2)
            s1.synchronize()
            s2.synchronize()
            assert float(b[-1]) == (1 - ctx.rank) + 5
        # one-sided
        win = cc.empty(4096, torch.float32)
        win.fill_(-1.0)
        _sync()
        cc.pc.host_barrier()
        cc.put(torch.full((16,), float(ctx.rank), device="cuda"), win, right, remote_offset=16 * ctx.rank)
        _sync()
        cc.barrier()
        _sync()
        assert float(win[16 * left]) == left
        got = torch.zeros(16, device="cuda")
        cc.get(got, win, left, remote_offset=16 * ((left - 1) % size))
        _sync()
        assert float(got[0]) == (left - 1) % size
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", [2, 3, 4])
def test_zero_copy_exchange_ring(size):
    """exchange(): the sender writes straight into the neighbour's symmetric buffer; counters carry over
    from call to call, every payload size (sub-16-byte tail, TMA and LDG/STG variants)."""
    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        right, left = (ctx.rank + 1) % size, (ctx.rank - 1) % size
        for n in (1, 1001, 70_001, 2_000_003):
            kv = cc.empty(2 * n + 8, torch.float32)
            halves = [kv[:n], kv[n + (-n) % 4:2 * n + (-n) % 4]]   # both 16-byte aligned
            halves[0].fill_(float(ctx.rank))
            _sync()
            cc.pc.host_barrier()
            for step in range(size + 1):
                cur, nxt = halves[step % 2], halves[(step + 1) % 2]
                cc.exchange(cur, right, nxt, left)
                _sync()
                want = float((ctx.rank - step - 1) % size)
                assert float(nxt[0]) == want and float(nxt[-1]) == want and float(nxt[n // 2]) == want, (n, step)
            cc.pc.host_barrier()
        # unregistered receive tensor: falls back to the mailbox path
        r = torch.zeros(5000, device="cuda")
        cc.exchange(torch.full((5000,), float(ctx.rank), device="cuda"), right, r, left)
        _sync()
        assert float(r[-1]) == left
        cc.check_health()
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", [3, 4])
def test_relay_broadcast(size, monkeypatch):
    """Chunk-pipelined relay broadcast (mode 3): every root, sizes with partial tiles / chunks and a byte tail,
    registered buffers and plain pointers (staged)."""
    monkeypatch.setenv("GLB_CUDA_BCAST_MODE", "3")

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        for n, tile in ((5, 0), (4099, 0), (300_001, 64), (2_500_003, 256), (2_500_003, 0)):
            os.environ["GLB_CUDA_BCAST_TILE"] = str(tile)
            for root in range(size):
                t = cc.empty(n, torch.float32)
                t.fill_(-1.0)
                if ctx.rank == root:
                    t.copy_(torch.arange(n, dtype=torch.float32, device="cuda") * 0.5 + root)
                cc.broadcast(t, root=root)
                _sync()
                want = torch.arange(n, dtype=torch.float64) * 0.5 + root
                torch.testing.assert_close(t.double().cpu(), want)
                cc.pc.host_barrier()
        u = torch.full((1_000_003,), float(ctx.rank), dtype=torch.uint8, device="cuda")[3:]  # misaligned plain pointer
        cc.broadcast(u, root=size - 1)
        _sync()
        assert int(u[0]) == size - 1 and int(u[-1]) == size - 1
        cc.check_health()
        cc.pc.host_barrier()
        return True

    try:
        assert all(gb.spawn_threads(size, fn, cuda_device=0))
    finally:
        os.environ.pop("GLB_CUDA_BCAST_TILE", None)


def test_local_allreduce_many_launch_shapes():
    """Every launch shape of the single-rank fused step gives the same result (odd count: vector body + tail)."""
    cu = gb._C.cuda
    n = 1_000_003
    want = None
    try:
        for tiled in (False, True):
            for ctas in (1, 4, 8):
                for unroll in (1, 2, 4):
                    cu.set_local_shape(ctas, unroll, tiled)
                    ts = [torch.arange(n, dtype=torch.float32, device="cuda") * (i + 1) for i in range(3)]
                    cu.local_allreduce_many([t.data_ptr() for t in ts], n, int(gb.DataType.FLOAT32), 1, 0.25,
                                            torch.cuda.current_stream().cuda_stream)
                    _sync()
                    if want is None:
                        want = (torch.arange(n, dtype=torch.float64) * 6 * 0.25).float()
                    for t in ts:
                        torch.testing.assert_close(t.cpu(), want, rtol=1e-6, atol=0)
    finally:
        cu.set_local_shape(4, 1, False)


# ---- ordering across streams, literal pipelined schedule ------------------------------------------------------------

def test_collectives_on_two_streams_are_ordered():
    size = 2

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        s1, s2 = gcu.new_stream(0), gcu.new_stream(0)
        a, b = _inp(ctx.rank, size, 200000), _inp(ctx.rank, size, 200000)
        cc.register(a)
        cc.register(b)
        _sync()
        for _ in range(5):
            cc.allreduce(a, algo="two_shot", stream=s1, scale=0.5)
            cc.allreduce(b, algo="two_shot", stream=s2, scale=0.5)
        s1.synchronize()
        s2.synchronize()
        cc.check_health()
        cc.pc.host_barrier()
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


@pytest.mark.parametrize("size", [2, 3, 4, 6, 8])
def test_halving_doubling_pipelined_literal(size):
    def fn(ctx):
        for count in (1000, 300001):
            t = _inp(ctx.rank, size, count)
            algo = gcu.CudaAllreduceHalvingDoublingPipelined(ctx, t, literal=True)
            assert algo.resolved_algo() == "halving_doubling_pipelined"
            algo.run()
            torch.testing.assert_close(t.double().cpu(), _exp(size, count), rtol=1e-6, atol=0)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


def test_host_workspace_chunked_overlap():
    size = 2

    def fn(ctx):
        t = _inp(ctx.rank, size, 3_000_001)
        algo = gcu.CudaAllreduceRingChunked(ctx, t, host_workspace=True)
        assert not algo.uses_peer_memory()
        algo.set_scale(0.25)
        algo.run()
        torch.testing.assert_close(t.double().cpu(), 0.25 * _exp(size, 3_000_001), rtol=1e-6, atol=0)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0))


# ---- the NVLink data plane behind the transport API (mirrors gloo/test/remote_key_test.cc) ------------

def test_nvl_transport_device_buffers_send_recv_put_get():
    size = 2

    def fn(ctx):
        assert "nvl(" in str(ctx.device()) and ctx.device().has_gpu_direct()
        peer = 1 - ctx.rank
        n = 1_000_000
        mine = torch.full((n,), float(ctx.rank + 1), device="cuda")
        inbox = torch.zeros(n, device="cuda")
        window = torch.full((4096,), -1.0, device="cuda")
        torch.cuda.synchronize()
        gb.barrier(ctx)
        sb = ctx.create_unbound_buffer(mine.data_ptr(), n * 4)
        rb = ctx.create_unbound_buffer(inbox.data_ptr(), n * 4)
        # two-sided: every rank posts the send first, then the receive (larger than the mailbox ring)
        sb.send(peer, 7)
        rb.recv(peer, 7)
        assert rb.wait_recv() == peer
        assert sb.wait_send() == peer
        assert float(inbox[0]) == peer + 1 and float(inbox[-1]) == peer + 1
        # one-sided through a remote key that travels over the host collectives
        wb = ctx.create_unbound_buffer(window.data_ptr(), 4096 * 4)
        key = wb.get_remote_key()
        import numpy as np
        raw = np.frombuffer(key.encode().ljust(512, b" "), dtype=np.uint8).copy()
        allk = np.zeros(512 * size, dtype=np.uint8)
        gb.allgather(ctx, allk, raw)
        peer_key = bytes(allk[512 * peer:512 * (peer + 1)]).decode().strip()
        src = ctx.create_unbound_buffer(mine.data_ptr(), 64 * 4)
        src.put(ctx, peer_key, 1, 0, 16 * 4 * (ctx.rank + 1), 64 * 4)  # local offset 0 -> remote offset
        src.wait_send()
        gb.barrier(ctx)
        torch.cuda.synchronize()
        lo = 16 * (peer + 1)
        assert float(window[lo]) == peer + 1 and float(window[lo + 63]) == peer + 1 and float(window[0]) == -1.0
        got = torch.zeros(64, device="cuda")
        gbuf = ctx.create_unbound_buffer(got.data_ptr(), 64 * 4)
        gbuf.get(ctx, peer_key, 2, 0, 16 * 4 * (ctx.rank + 1), 64 * 4)  # what I just put there
        gbuf.wait_recv()
        assert float(got[0]) == ctx.rank + 1
        # bounds are checked against the key
        with pytest.raises(gb.GlbError):
            src.put(ctx, peer_key, 3, 0, 4096 * 4 - 8, 64 * 4)
        # host memory still goes through the control-plane transport
        h = np.full(1000, float(ctx.rank), dtype=np.float32)
        gb.allreduce(ctx, h)
        assert h[0] == 1.0
        gb.barrier(ctx)
        return True

    assert all(gb.spawn_threads(size, fn, cuda_device=0, nvl=True))


def test_local_op_classes():
    res = gb._C.cuda.local_ops_selftest([0], 100003)
    assert len(res) >= 4
    assert all(r["ok"] for r in res), res
    if torch.cuda.device_count() >= 2:
        res = gb._C.cuda.local_ops_selftest(list(range(min(4, torch.cuda.device_count()))), 100003)
        assert all(r["ok"] for r in res), res
        assert any("NCCL" in r["name"] for r in res)


# ---- consumers: gradients living in symmetric buckets (kept last in the file) ----------------------------------

@pytest.mark.parametrize("size", [2, 3])
def test_gradient_bucketer_cuda(size):
    """GradientBucketer on CUDA: p.grad is a view into a symmetric bucket, buckets are averaged by the fused
    kernel on a side stream while backward is still running; result == full-batch gradient."""
    from gloo_b200.models import DDPMLP
    from gloo_b200.parallel import GradientBucketer

    torch.manual_seed(3)
    ref = DDPMLP()
    x, y = torch.randn(size * 4, 64), torch.randn(size * 4, 8)
    single = DDPMLP()
    single.load_state_dict(ref.state_dict())
    torch.nn.functional.mse_loss(single(x), y).backward()
    want = [p.grad.clone() for p in single.parameters()]

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=8 << 20)
        m = DDPMLP().cuda()
        m.load_state_dict(ref.state_dict())
        gbk = GradientBucketer(ctx, cc, m.parameters(), bucket_bytes=8 << 10)
        assert len(gbk.buckets) > 1 and all(cc.lookup(b["flat"])[0] is not None for b in gbk.buckets)
        xs, ys = x[ctx.rank * 4:(ctx.rank + 1) * 4].cuda(), y[ctx.rank * 4:(ctx.rank + 1) * 4].cuda()
        _sync()
        cc.pc.host_barrier()
        out = []
        for _ in range(2):
            torch.nn.functional.mse_loss(m(xs), ys).backward()
            gbk.finish()
            _sync()
            out.append([p.grad.detach().cpu().clone() for p in m.parameters()])
            gbk.zero_grad()
        cc.check_health()
        cc.pc.host_barrier()
        return out

    for steps in gb.spawn_threads(size, fn, cuda_device=0):
        for grads in steps:
            for g, w in zip(grads, want):
                torch.testing.assert_close(g, w, rtol=1e-4, atol=1e-5)
