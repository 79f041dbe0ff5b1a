"""One process per rank: models.TPBlock(sequence_parallel=True) on CUDA against DenseBlock on the CPU.
The block takes and returns this rank's shard of a sequence-first input; its backward has
collectives on the autograd thread of each device, which ranks sharing one process cannot run,
hence processes.
usage: sp_block_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.models import DenseBlock, TPBlock  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel import TensorParallel  # noqa: E402


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    # the problem and tolerances of tp_block_worker.py, with a sequence that splits over 2 and 4 ranks
    torch.manual_seed(19)
    B, S, E = 2, 12, 32
    dense = DenseBlock(d_model=E, n_heads=4, d_ff=64)
    x = torch.randn(B, S, E, requires_grad=True)
    out_d = dense(x)
    out_d.square().mean().backward()

    tp = TensorParallel(ctx, cc)
    blk = TPBlock(tp, d_model=E, n_heads=4, d_ff=64, sequence_parallel=True).cuda()
    blk.load_dense(dense)
    lo, hi = S // size * rank, S // size * (rank + 1)
    shard = lambda t: t.detach().transpose(0, 1)[lo:hi]  # noqa: E731  [B, S, E] -> this rank's [S/P, B, E]
    xi = shard(x).contiguous().cuda().requires_grad_(True)
    torch.cuda.synchronize()
    before = gb._C.cuda.launch_count()
    out = blk(xi)
    torch.cuda.synchronize()
    launches = gb._C.cuda.launch_count() - before
    assert launches == 3, f"{launches} collective launches in a forward"
    (out.square().sum() / (B * S * E)).backward()  # this rank's share of the mean
    blk.sp.allreduce_sequence_parallel_grads(blk.sequence_parallel_parameters())
    torch.cuda.synchronize()
    close = torch.testing.assert_close
    close(out.detach().cpu(), shard(out_d), rtol=1e-4, atol=1e-5)
    close(xi.grad.cpu(), shard(x.grad), rtol=1e-3, atol=1e-6)
    close(blk.up.weight.grad.cpu(), dense.up.weight.grad[blk.up.lo:blk.up.hi], rtol=1e-3, atol=1e-6)
    close(blk.q.weight.grad.cpu(), dense.qkv.weight.grad[blk.q.lo:blk.q.hi], rtol=1e-3, atol=1e-6)
    close(blk.proj.weight.grad.cpu(), dense.proj.weight.grad[:, blk.proj.lo:blk.proj.hi], rtol=1e-3, atol=1e-6)
    close(blk.down.weight.grad.cpu(), dense.down.weight.grad[:, blk.down.lo:blk.down.hi], rtol=1e-3, atol=1e-6)
    for mine, want in ((blk.ln1, dense.ln1), (blk.ln2, dense.ln2)):
        close(mine.weight.grad.cpu(), want.weight.grad, rtol=1e-3, atol=1e-6)
        close(mine.bias.grad.cpu(), want.bias.grad, rtol=1e-3, atol=1e-6)
    close(blk.proj.bias.grad.cpu(), dense.proj.bias.grad, rtol=1e-3, atol=1e-6)
    close(blk.down.bias.grad.cpu(), dense.down.bias.grad, rtol=1e-3, atol=1e-6)
    cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
