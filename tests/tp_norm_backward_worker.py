"""One process per rank: TensorParallel.reduce_residual_norm(copy_out=True) on CUDA, whose backward is
the fused kernel, against the dense composition on the CPU, for rms and layer norms and for a frozen
norm without bias (no column sums); then models.TPBlock on CUDA against DenseBlock. The backward must
call the fused entry point once and no allreduce of its own, and every rank must get the same bytes
of the norm and bias gradients. The backward's collectives run on each device's autograd thread,
which ranks sharing one process cannot run, hence processes.
usage: tp_norm_backward_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.models import DenseBlock, TPBlock  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel import TensorParallel  # noqa: E402


def _norm(kind, H):
    if kind == "layer":
        m = torch.nn.LayerNorm(H)
    else:
        m = torch.nn.RMSNorm(H, eps=1e-6)
    with torch.no_grad():
        m.weight.copy_(0.5 + torch.rand(H))
        if kind == "layer":
            m.bias.copy_(0.25 * torch.randn(H))
    return m


class Counted:
    """Counts the calls of the fused backward and of cc.allreduce while active."""

    def __init__(self, cc):
        self.cc, self.calls = cc, {"fused": 0, "allreduce": 0}

    def __enter__(self):
        for name, attr in (("fused", "allreduce_residual_norm_backward"), ("allreduce", "allreduce")):
            fn = getattr(self.cc, attr)

            def wrapper(*args, _fn=fn, _name=name, **kwargs):
                self.calls[_name] += 1
                return _fn(*args, **kwargs)

            setattr(self.cc, attr, wrapper)
        torch.cuda.synchronize()
        self.before = gb._C.cuda.launch_count()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self.launches = gb._C.cuda.launch_count() - self.before
        for attr in ("allreduce_residual_norm_backward", "allreduce"):
            vars(self.cc).pop(attr, None)


def same_on_every_rank(cc, size, tensors, what):
    """Every rank's bytes of each (fp32) tensor equal rank 0's."""
    for t in tensors:
        mine = t.detach().contiguous().reshape(-1)
        all_ = torch.empty(size * mine.numel(), dtype=mine.dtype, device=mine.device)
        cc.allgather(all_, mine)
        torch.cuda.synchronize()
        rows = all_.view(torch.int32).view(size, -1)
        assert all(torch.equal(rows[0], rows[r]) for r in range(size)), f"{what}: ranks differ"


def check_op(tp, cc, rank, size, kind, frozen=False):
    """frozen: the norm's parameters need no gradient and there is no bias: no column sums."""
    T, B, H = 5, 2, 64
    torch.manual_seed(11)
    parts = [torch.randn(T, B, H) for _ in range(size)]
    residual, bias = torch.randn(T, B, H), torch.randn(H)
    g_r, g_o = torch.randn(T, B, H), [torch.randn(T, B, H) for _ in range(size)]
    norm_d = _norm(kind, H)
    norm_c = _norm(kind, H).cuda()
    norm_c.load_state_dict(norm_d.state_dict())
    for m in (norm_d, norm_c):
        m.requires_grad_(not frozen)

    # dense: s is replicated, so it enters the loss once; out feeds every rank's next layer, so its
    # gradient is the sum of theirs
    dp = [p.clone().requires_grad_(True) for p in parts]
    dres, dbias = residual.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    s = sum(dp) + dres + (0 if frozen else dbias)
    y = norm_d(s)
    ((s * g_r).sum() + sum((y * g).sum() for g in g_o)).backward()

    p = parts[rank].cuda().requires_grad_(True)
    res = residual.cuda().requires_grad_(True)
    b = None if frozen else bias.cuda().requires_grad_(True)
    s_, y_ = tp.reduce_residual_norm(p, res, norm_c, b, copy_out=True)
    loss = (s_ * g_r.cuda()).sum() + (y_ * g_o[rank].cuda()).sum()
    vectors = 0 if frozen else len(list(norm_c.parameters())) + 1
    plan = gb._C.cuda.plan_residual_norm_backward(cc.pc, T * B, H, int(gb.DataType.FLOAT32),
                                                  {"rms": 1, "layer": 2}[kind], vectors)
    with Counted(cc) as c:
        loss.backward()
    what = f"{kind} frozen={frozen}"
    assert c.calls == {"fused": 1, "allreduce": 0}, f"{what}: backward calls {c.calls}"
    assert c.launches == plan["launches"], f"{what}: {c.launches} launches in the backward, plan {plan}"
    close = torch.testing.assert_close
    close(s_.detach().cpu(), s.detach(), rtol=1e-5, atol=1e-5)
    close(y_.detach().cpu(), y.detach(), rtol=1e-5, atol=1e-5)
    close(p.grad.cpu(), dp[rank].grad, rtol=1e-4, atol=1e-5)
    close(res.grad.cpu(), dres.grad, rtol=1e-4, atol=1e-5)
    same_on_every_rank(cc, size, [p.grad], what)
    if frozen:
        assert all(t.grad is None for t in norm_c.parameters())
        return
    close(b.grad.cpu(), dbias.grad, rtol=1e-4, atol=1e-4)
    for mine, want in zip(norm_c.parameters(), norm_d.parameters()):
        close(mine.grad.cpu(), want.grad, rtol=1e-4, atol=1e-4)
    same_on_every_rank(cc, size, [b.grad] + [t.grad for t in norm_c.parameters()], what)


def check_block(tp, cc, rank, size):
    """TPBlock against DenseBlock at tp_block_worker.py's tolerances; ln2's backward is the fused call."""
    torch.manual_seed(19)
    dense = DenseBlock(d_model=32, n_heads=4, d_ff=64)
    x = torch.randn(2, 10, 32, requires_grad=True)
    dense(x).square().mean().backward()
    blk = TPBlock(tp, d_model=32, n_heads=4, d_ff=64).cuda()
    blk.load_dense(dense)
    xi = x.detach().clone().cuda().requires_grad_(True)
    out = blk(xi)
    with Counted(cc) as c:
        out.square().mean().backward()
    # ln2's backward is the fused call; the allreduces left are ln1's copy_to_region of q, k and v
    assert c.calls["fused"] == 1, f"block backward calls {c.calls}"
    assert c.calls["allreduce"] == 3, f"block backward calls {c.calls}"
    close = torch.testing.assert_close
    close(xi.grad.cpu(), x.grad, rtol=1e-3, atol=1e-6)
    close(blk.up.weight.grad.cpu(), dense.up.weight.grad[blk.up.lo:blk.up.hi], rtol=1e-3, atol=1e-6)
    close(blk.up.bias.grad.cpu(), dense.up.bias.grad[blk.up.lo:blk.up.hi], rtol=1e-3, atol=1e-6)
    close(blk.proj.weight.grad.cpu(), dense.proj.weight.grad[:, blk.proj.lo:blk.proj.hi], rtol=1e-3, atol=1e-6)
    close(blk.proj.bias.grad.cpu(), dense.proj.bias.grad, rtol=1e-3, atol=1e-6)
    close(blk.ln1.weight.grad.cpu(), dense.ln1.weight.grad, rtol=1e-3, atol=1e-6)
    close(blk.ln2.weight.grad.cpu(), dense.ln2.weight.grad, rtol=1e-3, atol=1e-6)
    close(blk.ln2.bias.grad.cpu(), dense.ln2.bias.grad, rtol=1e-3, atol=1e-6)
    same_on_every_rank(cc, size, [blk.ln2.weight.grad, blk.ln2.bias.grad, blk.proj.bias.grad], "block")


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    tp = TensorParallel(ctx, cc)
    for kind in ("rms", "layer"):
        check_op(tp, cc, rank, size, kind)
        cc.pc.host_barrier()
        check_op(tp, cc, rank, size, kind, frozen=True)
        cc.pc.host_barrier()
    check_block(tp, cc, rank, size)
    cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
