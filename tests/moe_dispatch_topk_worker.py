"""One process per GPU: the top-k MoE dispatch over the cross-process peer-memory path.
usage: moe_dispatch_topk_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel.strategies import MoEDispatcher  # noqa: E402
from test_moe_dev import SENTINEL, _bytes  # noqa: E402
from test_moe_dispatch_topk import _composed, _fused, _needs, _problem  # noqa: E402


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=32 << 20)
    moe = MoEDispatcher(ctx, cc)
    E, align, H = 2, 8, 256
    for k in (1, 8):
        per = _problem(size, E, k, torch.bfloat16, H, 40 + k)
        x, idx = (t.cuda() for t in per[rank])
        cap = max(_needs(per, size, E, align)) + 1
        for symmetric in (True, False):
            for fp8 in (False, True):
                dt = torch.float8_e4m3fn if fp8 else torch.bfloat16
                outs = []
                for _ in range(2):
                    o = cc.empty((cap, H), dt) if symmetric else torch.empty((cap, H), dtype=dt, device="cuda")
                    s = None
                    if fp8:
                        s = (cc.empty((cap, H // 128), torch.float32) if symmetric
                             else torch.empty((cap, H // 128), device="cuda"))
                        s.view(torch.uint8).fill_(SENTINEL)
                    o.view(torch.uint8).fill_(SENTINEL)
                    outs.append((o, s))
                a = _fused(cc, outs[0][0], x, idx, E, align, out_scales=outs[0][1])
                b = _composed(cc, moe, outs[1][0], x, idx, E, align, out_scales=outs[1][1])
                cc.synchronize()
                tag = (k, symmetric, fp8)
                assert torch.equal(_bytes(outs[0][0]), _bytes(outs[1][0])), tag
                if fp8:
                    assert torch.equal(_bytes(outs[0][1]), _bytes(outs[1][1])), tag
                assert all(torch.equal(u, v) for u, v in zip(a, b)), tag
                cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
