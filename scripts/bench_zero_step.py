#!/usr/bin/env python
"""Time one ZeRO-1 optimizer step of a bf16 model with fp32 master weights, three ways:

  master        ZeroOptimizer(master_dtype=torch.float32).step(): the cast reduce-scatter of the bf16
                gradients into the fp32 shard gradient (1/P fused), AdamW on the fp32 shard, the cast
                allgather of the shard into the bf16 parameters
  bf16_rs       what a user can write without it: bf16 reduce-scatter (1/P fused) into a bf16 shard,
                .float() into the master gradient, AdamW, .to(bf16), bf16 allgather. The gradient
                sum is rounded to bf16 before the optimizer sees it.
  fp32_rs       the exact alternative: flat_grad.float() into a full-size fp32 (symmetric) buffer,
                fp32 reduce-scatter into the master gradient, AdamW, .to(bf16), bf16 allgather

All three use the same flat bf16 buffers (symmetric memory) and torch.optim.AdamW (foreach) on an
fp32 shard. Gradients are filled once; each step is timed with CUDA events on the current stream
after --warmup untimed steps, and the variants alternate over --rounds rounds of --steps steps
(median per round, then the median of the rounds). Wire bytes per rank come from the shapes: the
reduce-scatter brings (P - 1) / P of the flat gradient in at its element size, the allgather sends
(P - 1) / P of the parameters out at theirs.

Run one rank per GPU under torchrun (torchrun --nproc-per-node 8 scripts/bench_zero_step.py), or
--threads P for P ranks as threads on cuda:0: ranks that share a card pay for each other's kernels
and exchange through local memory, so those numbers measure overhead only, not NVLink; the JSON says
so. Rank 0 prints one JSON line with the card name and power limit (and writes it to --out).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel import ZeroOptimizer  # noqa: E402


def gpu_info(device):
    info = {"gpu": torch.cuda.get_device_name(device), "power_limit_w": None}
    try:
        q = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        if q.returncode == 0 and q.stdout.strip():
            info["power_limit_w"] = float(q.stdout.strip().splitlines()[0])
    except Exception as e:  # noqa: BLE001
        info["power_limit_w"] = f"unavailable: {e}"
    return info


def bench_rank(ctx, device, args):
    torch.cuda.set_device(device)
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    P = cc.size
    # transformer-like tensors: hidden x hidden blocks, `params` elements in all
    per = args.hidden * args.hidden
    shapes = [(args.hidden, args.hidden)] * (args.params // per) + ([(args.params % per,)] if args.params % per else [])
    g = torch.Generator(device="cpu").manual_seed(1)
    params = [torch.nn.Parameter((torch.rand(s, generator=g) - 0.5).to(torch.bfloat16).to(device)) for s in shapes]
    opt_kw = {"lr": 1e-4, "foreach": True}
    zo = ZeroOptimizer(ctx, cc, params, torch.optim.AdamW, master_dtype=torch.float32, **opt_kw)
    n, cnt = zo.flat_param.numel(), zo.counts[cc.rank]
    counts = zo.counts
    zo.flat_grad.copy_(((torch.rand(n, device=device) - 0.5) * 1e-2).to(torch.bfloat16))
    sl = slice(zo.start, zo.start + cnt)

    # the two compositions, on the same flat buffers
    master = torch.nn.Parameter(zo.flat_param[sl].float())
    master.grad = torch.zeros_like(master)
    opt = torch.optim.AdamW([master], **opt_kw)
    shard16 = torch.empty(cnt, dtype=torch.bfloat16, device=device)
    grad32 = cc.empty(n, torch.float32)

    def bf16_rs():
        cc.reduce_scatter(shard16, zo.flat_grad, counts, scale=1.0 / P)
        master.grad.copy_(shard16)
        opt.step()
        with torch.no_grad():
            shard16.copy_(master)
        cc.allgatherv(zo.flat_param, shard16, counts)

    def fp32_rs():
        grad32.copy_(zo.flat_grad)
        cc.reduce_scatter(master.grad, grad32, counts, scale=1.0 / P)
        opt.step()
        with torch.no_grad():
            shard16.copy_(master)
        cc.allgatherv(zo.flat_param, shard16, counts)

    variants = {"master": zo.step, "bf16_rs": bf16_rs, "fp32_rs": fp32_rs}
    wire = {"master": (2, 2), "bf16_rs": (2, 2), "fp32_rs": (4, 2)}
    share = n * (P - 1) // P
    for f in variants.values():
        for _ in range(args.warmup):
            f()
    cc.synchronize()
    times = {k: [] for k in variants}
    for _ in range(args.rounds):
        for name, f in variants.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
            cc.pc.host_barrier()
            for a, b in ev:
                a.record()
                f()
                b.record()
            cc.synchronize()
            times[name].append(statistics.median(a.elapsed_time(b) for a, b in ev))
    launches0 = gb._C.cuda.launch_count()
    cc.pc.host_barrier()
    zo.step()
    cc.synchronize()
    cc.pc.host_barrier()
    rows = []
    for name in variants:
        rs_es, ag_es = wire[name]
        rows.append({"variant": name, "step_ms": statistics.median(times[name]), "round_ms": times[name],
                     "wire_bytes_per_rank": share * (rs_es + ag_es), "reduce_scatter_bytes_in": share * rs_es,
                     "allgather_bytes_out": share * ag_es})
    extra = {"params": n, "shard": cnt, "master_step_launches_all_ranks": gb._C.cuda.launch_count() - launches0}
    cc.pc.host_barrier()
    return rows, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--params", type=int, default=350_000_000, help="model parameters (bf16)")
    ap.add_argument("--hidden", type=int, default=4096)
    ap.add_argument("--threads", type=int, default=0, help="this many ranks as threads on cuda:0 (overhead only)")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--stage-mb", type=int, default=64)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if args.steps < 20:
        ap.error("--steps: the median needs at least 20 steps")
    if args.threads:
        world = args.threads
        rows, extra = gb.spawn_threads(world, lambda ctx: bench_rank(ctx, 0, args), cuda_device=0, timeout_ms=600000)[0]
        mode = f"{world} ranks as threads on one GPU: overhead only, not NVLink numbers"
        info, rank = gpu_info(0), 0
    else:
        rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
        local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local)
        ctx = gb.init_context(rank, world, path=f"/tmp/glb_zero_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}",
                              timeout_ms=120000)
        rows, extra = bench_rank(ctx, local, args)
        mode = f"{world} ranks, one per GPU"
        info = gpu_info(local)
    if rank == 0:
        doc = {"benchmark": "zero_step_bf16_fp32_master", "mode": mode, "ranks": world, **info, **extra,
               "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds, "rows": rows}
        text = json.dumps(doc)
        print(text)
        if args.out:
            with open(args.out, "w") as f:
                f.write(text + "\n")


if __name__ == "__main__":
    main()
