#!/usr/bin/env python
"""Target for Nsight Compute (one GPU, one process): the N=1 flagship step on the benchmark's
400 MB buffers and the virtual-rank loopback of the collective kernels on 64 MB buffers, so
that `ncu --set full -k regex:...` captures the hot kernels at a realistic size.

  ncu --set full --clock-control none --import-source on -k regex:'localAllreduceMany|twoShotAllreduce|pipelinedAllreduce|peerBulkCopy' \
      -c 8 -o gpurun_out/prof_r2 python scripts/ncu_target.py
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
os.environ.setdefault("CUDA_MODULE_LOADING", "EAGER")

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402


def fn(ctx):
    cc = gcu.CudaContext(ctx, 0, stage_bytes=256 << 20)
    n = 100_000_000
    a, b = torch.ones(n, device="cuda"), torch.ones(n, device="cuda")
    step = gcu.CudaAllreduceRingChunked(ctx, [a, b])
    for _ in range(3):
        step.run()
    del a, b, step
    torch.cuda.synchronize()
    res = cc.pc.loopback_selftest(torch.cuda.current_stream().cuda_stream, int(os.environ.get("GLB_NCU_COUNT", 1 << 24)))
    bad = [r for r in res if not r["ok"]]
    assert not bad, bad
    return len(res)


if __name__ == "__main__":
    print(gb.spawn_threads(1, fn, cuda_device=0))
