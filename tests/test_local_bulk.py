"""GPU tests for the single-rank fused step's two kernels: localAllreduceManyBulkKernel (TMA
bulk-copy pipeline, taken for large 16-byte-aligned calls) and localAllreduceManyKernel (LDG/STG).
Results are checked against a float64 host reference and must be bit-identical between the two."""
import pytest
import torch

import gloo_b200 as gb

pytestmark = pytest.mark.gpu

cu = gb._C.cuda
DT = {torch.float32: gb.DataType.FLOAT32, torch.float16: gb.DataType.FLOAT16, torch.bfloat16: gb.DataType.BFLOAT16}
# (rtol, atol): one rounding of the fp32-accumulated result
TOL = {torch.float32: (1e-6, 1e-6), torch.float16: (1e-3, 5e-3), torch.bfloat16: (8e-3, 4e-2)}
# Largest number of buffers whose pipeline stages fit in an H100's shared memory (reduce_kernels.cu:
# 3 stages of 16 KB per buffer): one more buffer runs the LDG/STG kernel.
BULK_MAX_N = 4
# Above the size threshold for every dtype; odd, so the call ends in whole tiles, then packs,
# then single elements.
COUNT_BYTES = 24_000_000


def _inputs(n, count, dtype, offset_elems=0):
    g = torch.Generator().manual_seed(1234 + n)
    host = [torch.randn(count, generator=g, dtype=torch.float64).to(dtype) for _ in range(n)]
    dev = []
    for i, h in enumerate(host):
        pad = offset_elems if i == n - 1 else 0
        t = torch.empty(count + pad, dtype=dtype, device="cuda")[pad:]
        t.copy_(h)
        dev.append(t)
    return host, dev


def _run(dev, dtype, scale):
    """One fused step over `dev`; returns whether its size and pointers select the bulk kernel."""
    ptrs, count = [t.data_ptr() for t in dev], dev[0].numel()
    cu.local_allreduce_many(ptrs, count, int(DT[dtype]), 1, scale, torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    return cu.local_allreduce_many_uses_bulk(ptrs, count, int(DT[dtype]))


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("n", sorted({2, 3, BULK_MAX_N, BULK_MAX_N + 1}))
@pytest.mark.parametrize("scale", [1.0, 0.25])
def test_bulk_step_matches_reference_and_ldg_stg(dtype, n, scale):
    esize = torch.tensor([], dtype=dtype).element_size()
    count = COUNT_BYTES // esize + 8 + 3
    host, dev = _inputs(n, count, dtype)
    want = sum(h.double() for h in host) * scale
    try:
        cu.set_local_shape(0, 0, False)
        assert _run(dev, dtype, scale) == (n <= BULK_MAX_N)
        bulk = [t.cpu() for t in dev]
        for t in bulk:
            torch.testing.assert_close(t.double(), want, rtol=TOL[dtype][0], atol=TOL[dtype][1])
            assert torch.equal(t, bulk[0])
        # the same inputs through the LDG/STG kernel: the same bits
        for t, h in zip(dev, host):
            t.copy_(h)
        cu.set_local_shape(2, 2, False)  # pins the LDG/STG kernel
        _run(dev, dtype, scale)
        for t, b in zip(dev, bulk):
            assert torch.equal(t.cpu(), b)
    finally:
        cu.set_local_shape(0, 0, False)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
def test_unaligned_pointer_takes_ldg_stg_kernel(dtype):
    esize = torch.tensor([], dtype=dtype).element_size()
    count = COUNT_BYTES // esize + 5
    host, dev = _inputs(2, count, dtype, offset_elems=4 // esize)
    assert dev[-1].data_ptr() % 16 == 4
    cu.set_local_shape(0, 0, False)
    assert not _run(dev, dtype, 0.25)
    assert cu.local_allreduce_many_uses_bulk([t.data_ptr() for t in dev[:1]], count, int(DT[dtype]))
    want = (host[0].double() + host[1].double()) * 0.25
    for t in dev:
        torch.testing.assert_close(t.cpu().double(), want, rtol=TOL[dtype][0], atol=TOL[dtype][1])
