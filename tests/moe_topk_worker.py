"""One process per GPU: the top-k MoE combine over the cross-process peer-memory path.
usage: moe_topk_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from test_moe_combine_topk import _bytes, _expert_out, _reference, _setup  # noqa: E402


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=32 << 20)
    pools = {"symmetric": cc.empty(1 << 20, torch.uint8)}
    E, align = 2, 8
    for case, dtype in enumerate((torch.float32, torch.bfloat16, torch.float16)):
        for k in (1, 8):
            per, needs = _setup(size, E, k, dtype, 90 + 10 * case + k, align)
            y, splits, pos, w = per[rank]
            for kind in ("symmetric", "plain"):
                eo = _expert_out(cc, kind, pools, max(needs) + 1, dtype)
                osp = torch.empty(size * E, dtype=torch.int64, device="cuda")
                cc.alltoallv_dev(eo, y.cuda(), splits.cuda(), osp, torch.empty_like(osp), experts=E, align=align)
                out = torch.empty((pos.shape[0], y.shape[1]), dtype=dtype, device="cuda")
                cc.alltoallv_dev_combine_topk(out, eo, splits.cuda(), pos.cuda(), w.cuda(), experts=E, align=align)
                cc.synchronize()
                assert torch.equal(_bytes(out), _bytes(_reference(y, pos, w, dtype))), (str(dtype), k, kind)
                cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
