"""One process per rank: SequenceParallel.reduce_scatter_residual_norm's autograd on CUDA, whose
backward is the fused kernel, against the dense composition on the CPU, for rms and layer norms with
out gathered and not, and with a frozen norm and no bias (no column sums). The backward must call
the fused entry point once and no reduce_scatter or allgather. The backward's collectives run on
each device's autograd thread, which ranks sharing one process cannot run, hence processes.
usage: sp_norm_backward_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel import SequenceParallel  # noqa: E402


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


def check(sp, cc, rank, size, kind, gather, frozen=False):
    """frozen: the norm's parameters need no gradient and there is no bias, so the backward computes
    no column sums."""
    Ts, B, H = 3, 2, 64
    T = size * Ts
    torch.manual_seed(7)
    parts = [torch.randn(T, B, H) for _ in range(size)]
    residual, bias = torch.randn(T, B, H), torch.randn(H)
    g_r, g_o = torch.randn(T, B, H), torch.randn(T, B, H)
    norm_d = _norm(kind, H)
    norm_c = _norm(kind, H).cuda()
    norm_c.load_state_dict(norm_d.state_dict())
    for m in (norm_d, norm_c):
        m.requires_grad_(not frozen)

    # the dense composition: every rank's partial, the full sequence, one process
    dp = [p.clone().requires_grad_(True) for p in parts]
    dres, dbias = residual.clone().requires_grad_(True), bias.clone().requires_grad_(True)
    s = sum(dp) + dres + (0 if frozen else dbias)
    y = norm_d(s)
    ((s * g_r).sum() + (y * g_o).sum()).backward()

    rows = slice(rank * Ts, (rank + 1) * Ts)
    p = parts[rank].cuda().requires_grad_(True)
    res = residual[rows].contiguous().cuda().requires_grad_(True)
    b = None if frozen else bias.cuda().requires_grad_(True)
    s_, y_ = sp.reduce_scatter_residual_norm(p, res, norm_c, b, gather_out=gather)
    # a gathered out is replicated: each rank's loss takes its own rows of it
    loss = (s_ * g_r[rows].cuda()).sum() + ((y_[rows] if gather else y_) * g_o[rows].cuda()).sum()
    vectors = 0 if frozen else len(list(norm_c.parameters())) + 1
    plan = gb._C.cuda.plan_reduce_scatter_norm_backward(cc.pc, T * B, H, int(gb.DataType.FLOAT32),
                                                        {"rms": 1, "layer": 2}[kind], gather, vectors)
    # The backward must be the fused entry point, with no reduce_scatter or allgather of its own.
    calls = {"fused": 0, "reduce_scatter": 0, "allgather": 0}
    fused = cc.reduce_scatter_residual_norm_backward

    def counting(name, fn):
        def wrapper(*args, **kwargs):
            calls[name] += 1
            return fn(*args, **kwargs)
        return wrapper

    cc.reduce_scatter_residual_norm_backward = counting("fused", fused)
    cc.reduce_scatter = counting("reduce_scatter", cc.reduce_scatter)
    cc.allgather = counting("allgather", cc.allgather)
    torch.cuda.synchronize()
    before = gb._C.cuda.launch_count()
    try:
        loss.backward()
        torch.cuda.synchronize()
    finally:
        for name in calls:
            vars(cc).pop(name if name != "fused" else "reduce_scatter_residual_norm_backward", None)
    launches = gb._C.cuda.launch_count() - before
    what = f"{kind} gather={gather} frozen={frozen}"
    assert calls == {"fused": 1, "reduce_scatter": 0, "allgather": 0}, f"{what}: backward calls {calls}"
    assert launches == plan["launches"], f"{what}: {launches} launches in the backward, plan {plan}"
    shared = ([] if frozen else [b] + list(norm_c.parameters()))
    sp.allreduce_sequence_parallel_grads(shared)
    torch.cuda.synchronize()
    close = torch.testing.assert_close
    close(s_.detach().cpu(), s.detach()[rows], rtol=1e-5, atol=1e-5)
    close(p.grad.cpu(), dp[rank].grad, rtol=1e-4, atol=1e-5)
    close(res.grad.cpu(), dres.grad[rows], rtol=1e-4, atol=1e-5)
    if frozen:
        assert all(t.grad is None for t in norm_c.parameters())
        return
    close(b.grad.cpu(), dbias.grad, rtol=1e-4, atol=1e-4)
    for mine, want in zip(norm_c.parameters(), norm_d.parameters()):
        close(mine.grad.cpu(), want.grad, rtol=1e-4, atol=1e-4)


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=16 << 20)
    sp = SequenceParallel(ctx, cc)
    for kind in ("rms", "layer"):
        for gather in (True, False):
            check(sp, cc, rank, size, kind, gather)
            cc.pc.host_barrier()
        check(sp, cc, rank, size, kind, True, frozen=True)
        cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
