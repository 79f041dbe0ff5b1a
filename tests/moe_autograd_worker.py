"""One process per rank: a MoE layer trained through MoEDispatcher.dispatch_topk_autograd and
combine_topk_autograd, checked against a dense single-process CPU reference over every rank's tokens.
usage: moe_autograd_worker.py STORE_DIR RANK SIZE"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel.strategies import MoEDispatcher  # noqa: E402

E, T, HD, K, ALIGN = 2, 16, 32, 2, 4


def problem(P):
    """The same parameters and tokens in every process: gate (G, HD), one (HD, HD) weight per
    global expert, every rank's tokens and loss weights."""
    g = torch.Generator().manual_seed(2024)
    G = P * E
    gate = torch.randn(G, HD, generator=g) * 0.3
    experts = torch.randn(G, HD, HD, generator=g) * 0.2
    x = torch.randn(P * T, HD, generator=g)
    r = torch.randn(P * T, HD, generator=g)
    return gate, experts, x, r


def routing(gate, x):
    """Top-k indices of softmax(x gate^T), from the CPU so that every process and the reference
    pick the same experts."""
    return torch.topk(torch.softmax(x @ gate.t(), dim=-1), K, dim=-1).indices


def reference(P, dtype):
    """Dense CPU layer over all ranks' tokens: per rank its own copy of the gate (so its gradient is
    the local one), one weight per global expert. Returns x.grad, each rank's gate grad and every
    expert's weight grad."""
    gate, experts, x, r = problem(P)
    idx = routing(gate, x)
    gates = [gate.clone().requires_grad_() for _ in range(P)]
    ws = experts.clone().requires_grad_()
    xs = x.to(dtype).float().clone().requires_grad_()
    loss = 0.0
    for s in range(P):
        xr = xs[s * T:(s + 1) * T]
        p = torch.softmax(xr @ gates[s].t(), dim=-1)
        w = p.gather(1, idx[s * T:(s + 1) * T])
        w = w / w.sum(-1, keepdim=True)
        y = torch.zeros(T, HD)
        for t in range(T):
            for j in range(K):
                e = int(idx[s * T + t, j])
                y[t] = y[t] + w[t, j] * torch.nn.functional.silu(xr[t] @ ws[e].t())
        loss = loss + (y * r[s * T:(s + 1) * T]).sum()
    loss.backward()
    return xs.grad, [g_.grad for g_ in gates], ws.grad


def run(cc, moe, rank, P, dtype):
    gate_w, experts, x_all, r_all = problem(P)
    dev = torch.device("cuda", cc.device)
    idx = routing(gate_w, x_all)[rank * T:(rank + 1) * T].to(dev)
    gate = torch.nn.Linear(HD, P * E, bias=False).to(dev)
    with torch.no_grad():
        gate.weight.copy_(gate_w)
    local = [torch.nn.Linear(HD, HD, bias=False).to(dev) for _ in range(E)]
    with torch.no_grad():
        for e in range(E):
            local[e].weight.copy_(experts[rank * E + e])
    x = x_all[rank * T:(rank + 1) * T].to(dtype).to(dev).requires_grad_()
    r = r_all[rank * T:(rank + 1) * T].to(dev)

    p = torch.softmax(gate(x.float()), dim=-1)
    w = p.gather(1, idx)
    w = w / w.sum(-1, keepdim=True)
    cap = P * T * K + E * ALIGN
    out = torch.empty((cap, HD), dtype=dtype, device=dev)
    expert_in, out_splits, out_offsets, route = moe.dispatch_topk_autograd(x, idx, out, experts=E, align=ALIGN)
    osp, ooff = out_splits.tolist(), out_offsets.tolist()
    rows, ys = [], []
    for e in range(E):
        lo, hi = ooff[e * P], ooff[e * P + P - 1] + osp[e * P + P - 1]
        seg = expert_in[lo:hi]
        ys.append(torch.nn.functional.silu(local[e](seg.float())).to(dtype))
        rows.append(torch.arange(lo, hi, device=dev))
    expert_out = torch.zeros((cap, HD), dtype=dtype, device=dev).index_copy(0, torch.cat(rows), torch.cat(ys))
    y = moe.combine_topk_autograd(expert_out, w, route)
    (y.float() * r).sum().backward()
    cc.synchronize()

    gx, ggate, gexp = reference(P, dtype)
    tol = dict(rtol=1e-4, atol=1e-4) if dtype == torch.float32 else dict(rtol=5e-2, atol=5e-2)
    torch.testing.assert_close(x.grad.float().cpu(), gx[rank * T:(rank + 1) * T], **tol)
    torch.testing.assert_close(gate.weight.grad.cpu(), ggate[rank], **tol)
    for e in range(E):
        torch.testing.assert_close(local[e].weight.grad.cpu(), gexp[rank * E + e], **tol)


def main():
    store_dir, rank, size = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    dev = rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    ctx = gb.init_context(rank, size, path=store_dir, timeout_ms=60000)
    cc = gcu.CudaContext(ctx, dev, stage_bytes=32 << 20)
    moe = MoEDispatcher(ctx, cc)
    for dtype in (torch.float32, torch.bfloat16):
        run(cc, moe, rank, size, dtype)
        cc.pc.host_barrier()
    print(f"WORKER {rank} OK", flush=True)


if __name__ == "__main__":
    main()
