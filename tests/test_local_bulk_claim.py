"""GPU tests for how localAllreduceManyBulkKernel deals its tiles: each CTA's first two tiles are
static and every later one is claimed from a counter that its owner keeps across calls and that
each launch leaves at zero. Every result is compared byte for byte with the same sum in torch,
and the buffers carry guard bands that must come back untouched."""
import pytest
import torch

import gloo_b200 as gb
from gloo_b200.ops import cuda as gcu

pytestmark = pytest.mark.gpu

cu = gb._C.cuda
F32 = int(gb.DataType.FLOAT32)
BF16 = int(gb.DataType.BFLOAT16)
DT = {torch.float32: F32, torch.bfloat16: BF16}
TILE = 16 * 1024  # bytes of one buffer per tile (reduce_kernels.cu)
STATIC = 2  # tiles per CTA before the first claim: the pipeline's stages - 1
GUARD = 4096  # elements on each side of every buffer
SENTINEL = -12345.0


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _buffers(n, count, dtype, seed):
    """n guarded buffers of `count` random elements: (whole tensors, the views the step runs on, inputs)."""
    g = torch.Generator().manual_seed(seed)
    whole, views, inputs = [], [], []
    for _ in range(n):
        w = torch.full((count + 2 * GUARD,), SENTINEL, dtype=dtype, device="cuda")
        x = torch.randn(count, generator=g, dtype=torch.float32).to(dtype).cuda()
        w[GUARD:GUARD + count].copy_(x)
        whole.append(w)
        views.append(w[GUARD:GUARD + count])
        inputs.append(x)
    return whole, views, inputs


def _expected(inputs, scale):
    """The kernel's arithmetic: sum in buffer order in fp32, then the scale, one rounding."""
    acc = inputs[0].float().clone()
    for x in inputs[1:]:
        acc += x.float()
    if scale != 1.0:
        acc *= scale
    return acc.to(inputs[0].dtype)


def _check(whole, count, want):
    for w in whole:
        assert torch.equal(w[GUARD:GUARD + count], want)
        assert bool((w[:GUARD] == SENTINEL).all()) and bool((w[GUARD + count:] == SENTINEL).all())


def _tile_counts():
    sms = _sms()
    return {
        "below_grid": 64,  # the smallest bulk call: fewer tiles than SMs, one CTA per tile
        "equal_grid": sms,  # one static tile per CTA, the first claim of every CTA comes back empty
        "all_static": STATIC * sms,  # the last whole tile is static: nothing to claim
        "one_claimed": STATIC * sms + 1,
        "far_above": 40 * sms + 7,
    }


@pytest.mark.parametrize("n", [1, 2, 3, 16])
@pytest.mark.parametrize("case", ["below_grid", "equal_grid", "all_static", "one_claimed", "far_above"])
@pytest.mark.parametrize("tail", [False, True])
def test_tile_counts(n, case, tail):
    tiles = _tile_counts()[case]
    count = tiles * TILE // 4 + ((TILE // 4 - 8) + 3 if tail else 0)  # tail: a partial tile of packs, then 3 elements
    scale = 0.5 if n != 2 else 1.0
    whole, views, inputs = _buffers(n, count, torch.float32, seed=n * 100 + tiles)
    ptrs = [v.data_ptr() for v in views]
    assert cu.local_allreduce_many_uses_bulk(ptrs, count, F32) == (n <= 4)
    cu.local_allreduce_many(ptrs, count, F32, 1, scale, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _check(whole, count, _expected(inputs, scale))


@pytest.mark.parametrize("case", ["equal_grid", "one_claimed", "far_above"])
def test_tile_counts_bfloat16(case):
    count = _tile_counts()[case] * TILE // 2 + 13
    whole, views, inputs = _buffers(3, count, torch.bfloat16, seed=7)
    ptrs = [v.data_ptr() for v in views]
    assert cu.local_allreduce_many_uses_bulk(ptrs, count, BF16)
    cu.local_allreduce_many(ptrs, count, BF16, 1, 0.25, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    _check(whole, count, _expected(inputs, 0.25))


def _one_rank(fn):
    assert all(gb.spawn_threads(1, fn, cuda_device=0))


def test_back_to_back_calls_one_algorithm():
    """200 runs of one fused step on one stream, new inputs before each: every run claims through
    the same counter, so a launch that did not leave it at zero would skip or repeat tiles in the next."""
    count = (STATIC * _sms() + 300) * TILE // 4 + 1001

    def fn(ctx):
        stream = torch.cuda.Stream()
        whole, views, _ = _buffers(2, count, torch.float32, seed=11)
        pool = [_buffers(2, count, torch.float32, seed=20 + k)[2] for k in range(3)]
        wants = [_expected(p, 1.0) for p in pool]
        algo = gcu.CudaAllreduceRingChunked(ctx, views, streams=[stream, stream])
        assert algo.launches_per_run() == 1
        bad = torch.zeros((), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            for k in range(200):
                for v, x in zip(views, pool[k % 3]):
                    v.copy_(x)
                algo.run()
                for v in views:
                    bad += (v.view(torch.int32) != wants[k % 3].view(torch.int32)).sum()
        stream.synchronize()
        assert int(bad) == 0
        _check(whole, count, wants[199 % 3])
        return True

    _one_rank(fn)


def test_back_to_back_calls_mixed_sizes_one_context():
    """200 calls through one CudaContext on one stream, alternating sizes (and so the number of
    claims per launch) and the registered and plain-pointer entries, which share its counter."""
    sms = _sms()
    counts = [64 * TILE // 4, (STATIC * sms + 1) * TILE // 4 + 5, (9 * sms + 3) * TILE // 4 + 777, STATIC * sms * TILE // 4]

    def fn(ctx):
        cc = gcu.CudaContext(ctx, 0, stage_bytes=16 << 20)
        stream = torch.cuda.Stream()
        cases = []
        for i, count in enumerate(counts):
            whole, views, inputs = _buffers(2, count, torch.float32, seed=40 + i)
            if i % 2:  # the first buffer from the context's own allocator: the registered entry
                sym = cc.empty(count, torch.float32)
                sym.copy_(inputs[0])
                views[0], whole[0] = sym, None
            cases.append((whole, views, inputs, _expected(inputs, 0.5)))
        bad = torch.zeros((), dtype=torch.int64, device="cuda")
        torch.cuda.synchronize()
        with torch.cuda.stream(stream):
            for k in range(200):
                _, views, inputs, want = cases[k % len(cases)]
                for v, x in zip(views, inputs):
                    v.copy_(x)
                cc.allreduce(views[0], extra=views[1:], scale=0.5, stream=stream)
                for v in views:
                    bad += (v.view(torch.int32) != want.view(torch.int32)).sum()
        stream.synchronize()
        assert int(bad) == 0
        for whole, views, _, want in cases:
            _check([w for w in whole if w is not None], views[1].numel(), want)
            assert torch.equal(views[0], want)
        return True

    _one_rank(fn)


def test_two_owners_on_two_streams():
    """Two fused steps, each with its own counter, launched alternately on two streams so that
    their kernels can run at the same time; and the same for two direct calls."""
    sms = _sms()
    counts = [(30 * sms + 5) * TILE // 4 + 9, (STATIC * sms + 17) * TILE // 4]

    def fn(ctx):
        streams = [torch.cuda.Stream(), torch.cuda.Stream()]
        owners = []
        for i, count in enumerate(counts):
            whole, views, inputs = _buffers(2, count, torch.float32, seed=60 + i)
            algo = gcu.CudaAllreduceRingChunked(ctx, views, streams=[streams[i]] * 2)
            algo.set_scale(0.5)
            owners.append((algo, whole, views, inputs, _expected(inputs, 0.5)))
        bad = [torch.zeros((), dtype=torch.int64, device="cuda") for _ in owners]
        torch.cuda.synchronize()
        for k in range(50):
            for i, (algo, _, views, inputs, want) in enumerate(owners):
                with torch.cuda.stream(streams[i]):
                    for v, x in zip(views, inputs):
                        v.copy_(x)
                    algo.run()
                    for v in views:
                        bad[i] += (v.view(torch.int32) != want.view(torch.int32)).sum()
        torch.cuda.synchronize()
        assert [int(b) for b in bad] == [0, 0]
        for _, whole, views, _, want in owners:
            _check(whole, views[0].numel(), want)

        direct = [_buffers(3, count, torch.float32, seed=80 + i) for i, count in enumerate(counts)]
        for k in range(20):
            for i, (_, views, inputs) in enumerate(direct):
                with torch.cuda.stream(streams[i]):
                    for v, x in zip(views, inputs):
                        v.copy_(x)
                    cu.local_allreduce_many([v.data_ptr() for v in views], views[0].numel(), F32, 1, 1.0,
                                            streams[i].cuda_stream)
        torch.cuda.synchronize()
        for whole, views, inputs in direct:
            _check(whole, views[0].numel(), _expected(inputs, 1.0))
        return True

    _one_rank(fn)
