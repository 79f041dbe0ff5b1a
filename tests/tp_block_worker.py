"""One process per rank: models.TPBlock on CUDA (each row-parallel output fused with bias, residual
add and, after the attention, ln2) against DenseBlock on the CPU. The backward of the column-parallel
layers allreduces, which ranks sharing one process's autograd thread cannot do, hence processes.
usage: tp_block_worker.py STORE_DIR RANK SIZE"""
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
    # the tolerances and problem of test_parallel.py::test_tensor_parallel_transformer_block_matches_dense
    torch.manual_seed(19)
    dense = DenseBlock(d_model=32, n_heads=4, d_ff=64)
    x = torch.randn(2, 10, 32, requires_grad=True)
    out_d = dense(x)
    out_d.square().mean().backward()

    tp = TensorParallel(ctx, cc)
    blk = TPBlock(tp, d_model=32, n_heads=4, d_ff=64).cuda()
    blk.load_dense(dense)
    xi = x.detach().clone().cuda().requires_grad_(True)
    torch.cuda.synchronize()
    before = gb._C.cuda.launch_count()
    out = blk(xi)
    torch.cuda.synchronize()
    launches = gb._C.cuda.launch_count() - before
    assert launches == 2, f"{launches} collective launches in a forward"
    out.square().mean().backward()
    torch.cuda.synchronize()
    close = torch.testing.assert_close
    close(out.detach().cpu(), out_d.detach(), rtol=1e-4, atol=1e-5)
    close(xi.grad.cpu(), x.grad, rtol=1e-3, atol=1e-6)
    close(blk.up.weight.grad.cpu(), dense.up.weight.grad[blk.up.lo:blk.up.hi], rtol=1e-3, atol=1e-6)
    close(blk.proj.weight.grad.cpu(), dense.proj.weight.grad[:, blk.proj.lo:blk.proj.hi], rtol=1e-3, atol=1e-6)
    close(blk.ln1.weight.grad.cpu(), dense.ln1.weight.grad, rtol=1e-3, atol=1e-6)
    close(blk.ln2.weight.grad.cpu(), dense.ln2.weight.grad, rtol=1e-3, atol=1e-6)
    close(blk.down.bias.grad.cpu(), dense.down.bias.grad, rtol=1e-3, atol=1e-6)
    cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
