#!/usr/bin/env python
"""The fused tensor-parallel step (allreduce + bias + residual add + RMSNorm / LayerNorm, one kernel:
`CudaContext.allreduce_residual_norm`) against the unfused sequence on the same inputs: clone of the
partial, `cc.allreduce`, bias add, residual add, `F.rms_norm` / `F.layer_norm`.

Run one rank per GPU under torch.distributed.run:

    python -m torch.distributed.run --nproc_per_node 8 scripts/bench_allreduce_norm.py --out norm.json

or, for a rehearsal on one GPU, `--threads P` (P ranks as threads sharing cuda:0). Ranks that share
a card pay for each other's kernels and exchange through local memory, so those numbers measure
the per-call overhead only, not the link; the JSON says so.

Time per call: CUDA events around `--iters` back-to-back calls after `--warmup` calls, median over
`--reps` windows, the maximum over ranks. Launches per call: the library's launch counter for the
fused path, kernels counted by torch.profiler for the unfused one (one rank per process only). Prints one JSON document and
writes it to `--out` when given.

`--backward` times the fused backward instead (`CudaContext.allreduce_residual_norm_backward`: the
allreduce of out's gradient, the norm's backward and the add of the residual stream's gradient, one
kernel per chunk plus one that finishes the column sums), with algo auto, one_shot and two_shot,
against the composition TensorParallel's autograd runs without it: clone + `cc.allreduce` of out's
gradient, the norm recomputed under torch autograd, the add and the bias row sum. bf16, with weight
and bias gradients (and the norm bias for layer); T on both sides of the one-shot / two-shot
threshold. Before timing, each shape records how far the two gradients of `partial` lie apart.

`--fp8` times the FP8 form (`allreduce_residual_norm(out_scales=)`: `out` as e4m3 codes with one
fp32 scale per row, in the same launch) against the fused bf16 call followed by the torch
quantisation of its `out` (`strategies.fp8_rows`), at decode T (1-128) and prefill T (4096), bf16,
with the launches per call of each. Each shape first checks that the two give the same bytes.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel.strategies import _norm_input_grad, fp8_rows  # noqa: E402

DECODE_T = (1, 8, 32, 128)
PREFILL_T = (4096,)
HIDDEN = (4096, 8192)


def gpu_info(device):
    name = torch.cuda.get_device_name(device)
    power = None
    try:
        import subprocess

        q = subprocess.run(["nvidia-smi", f"--id={device}", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30)
        power = float(q.stdout.strip().splitlines()[0]) if q.returncode == 0 and q.stdout.strip() else None
    except Exception:  # noqa: BLE001
        power = None
    return {"gpu": name, "power_limit_w": power}


def bench_rank(ctx, device, args, world, profile_unfused=True):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype = torch.bfloat16
    rows = []
    for H in HIDDEN:
        for T in DECODE_T + PREFILL_T:
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            partial = torch.randn(T, H, generator=g).to(dtype).cuda()
            residual = torch.randn(T, H, generator=g).to(dtype).cuda()
            bias = torch.randn(H, generator=g).to(dtype).cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            res_out, out = torch.empty_like(residual), torch.empty_like(residual)
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused():
                    cc.allreduce_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                               residual_out=res_out, out=out)

                def unfused():
                    y = partial.clone()
                    cc.allreduce(y)
                    y = y + bias
                    s = residual + y
                    if norm == "rms":
                        return s, F.rms_norm(s, (H,), weight, 1e-6)
                    return s, F.layer_norm(s, (H,), weight, nb, 1e-6)

                # same results (the unfused sequence rounds after each step, the fused one once)
                s_ref, o_ref = unfused()
                fused()
                torch.cuda.synchronize()
                err = float((out.float() - o_ref.float()).abs().max())
                plan = gb._C.cuda.plan_residual_norm(cc.pc, T, H, int(gb.DataType.BFLOAT16), {"rms": 1, "layer": 2}[norm], 0)
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "bytes": T * H * 2, "variant": plan["variant"],
                       "max_abs_diff_out": err}
                for name, fn in (("fused", fused), ("unfused", unfused)):
                    row[f"{name}_us"] = timed(ctx, cc, fn, stream, args, world)
                row["fused_launches_per_call"] = launches_fused(cc, fused)
                row["unfused_kernels_per_call"] = kernels_unfused(unfused, profile_unfused)
                row["speedup"] = row["unfused_us"] / row["fused_us"]
                rows.append(row)
    return rows


def bench_fp8_rank(ctx, device, args, world, profile_composed=True):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype = torch.bfloat16
    rows = []
    for H in HIDDEN:
        for T in DECODE_T + PREFILL_T:
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            partial = torch.randn(T, H, generator=g).to(dtype).cuda()
            residual = torch.randn(T, H, generator=g).to(dtype).cuda()
            bias = torch.randn(H, generator=g).to(dtype).cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            res_out, out = torch.empty_like(residual), torch.empty_like(residual)
            codes = torch.empty(T, H, dtype=torch.float8_e4m3fn, device="cuda")
            scales = torch.empty(T, 1, dtype=torch.float32, device="cuda")
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused_fp8():
                    cc.allreduce_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                               residual_out=res_out, out=codes, out_scales=scales)

                def composed():
                    cc.allreduce_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                               residual_out=res_out, out=out)
                    return fp8_rows(out)

                want_c, want_s = composed()
                fused_fp8()
                torch.cuda.synchronize()
                same = bool(torch.equal(codes.view(torch.uint8), want_c.view(torch.uint8)) and torch.equal(scales, want_s))
                plan = gb._C.cuda.plan_residual_norm(cc.pc, T, H, int(gb.DataType.BFLOAT16), {"rms": 1, "layer": 2}[norm],
                                                     0, True)
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "variant": plan["variant"],
                       "same_bytes": same}
                row["fp8_fused_us"] = timed(ctx, cc, fused_fp8, stream, args, world)
                row["bf16_fused_plus_torch_quant_us"] = timed(ctx, cc, composed, stream, args, world)
                row["fp8_fused_launches_per_call"] = launches_fused(cc, fused_fp8)
                row["composed_kernels_per_call"] = kernels_unfused(composed, profile_composed)
                row["speedup"] = row["bf16_fused_plus_torch_quant_us"] / row["fp8_fused_us"]
                rows.append(row)
    return rows


BACKWARD_T = (8, 32, 128, 1024, 4096)


def bench_backward_rank(ctx, device, args, world):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype, rank = torch.bfloat16, ctx.rank
    rows = []
    for H in HIDDEN:
        for T in BACKWARD_T:
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            s = torch.randn(T, H, generator=g).to(dtype).cuda()
            g_s = torch.randn(T, H, generator=g).to(dtype).cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            g_out = torch.randn(T, H, generator=torch.Generator().manual_seed(T * 131 + H + 7 + rank)).to(dtype).cuda()
            gp = torch.empty(T, H, dtype=dtype, device="cuda")
            gw, gnb, gb_ = (torch.empty(H, dtype=dtype, device="cuda") for _ in range(3))
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused(algo):
                    return lambda: cc.allreduce_residual_norm_backward(
                        g_out, s, g_s, weight, norm=norm, eps=1e-6, grad_partial=gp, grad_weight=gw,
                        grad_norm_bias=gnb if norm == "layer" else None, grad_bias=gb_, algo=algo)

                def composed():
                    y = g_out.clone()
                    cc.allreduce(y)
                    gs, _, _ = _norm_input_grad(norm, H, 1e-6, s, weight, nb, y)
                    total = g_s + gs
                    total.sum(0)
                    return total

                fused("auto")()
                ref = composed()
                torch.cuda.synchronize()
                vectors = 3 if norm == "layer" else 2
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "bytes": T * H * 2,
                       "max_abs_diff_composed": float((gp.float() - ref.float()).abs().max()),
                       "max_abs_grad": float(ref.float().abs().max())}
                for algo in ("auto", "one_shot", "two_shot"):
                    plan = gb._C.cuda.plan_residual_norm_backward(cc.pc, T, H, int(gb.DataType.BFLOAT16),
                                                                  {"rms": 1, "layer": 2}[norm], vectors,
                                                                  gcu.ALGOS[algo])
                    row[f"{algo}_variant"] = plan["variant"]
                    row[f"{algo}_launches"] = plan["launches"]
                    row[f"{algo}_us"] = timed(ctx, cc, fused(algo), stream, args, world)
                row["composed_us"] = timed(ctx, cc, composed, stream, args, world)
                row["speedup"] = row["composed_us"] / row["auto_us"]
                rows.append(row)
    return rows


def timed(ctx, cc, fn, stream, args, world):
    for _ in range(args.warmup):
        fn()
    per = []
    for _ in range(args.reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        cc.pc.host_barrier()
        a.record(stream)
        for _ in range(args.iters):
            fn()
        b.record(stream)
        b.synchronize()
        per.append(a.elapsed_time(b) * 1e3 / args.iters)
    v = np.asarray([float(np.median(per))], dtype=np.float64)
    if world > 1:
        gb.allreduce(ctx, v, op=gb.ReduceOp.MAX)
    return float(v[0])


def launches_fused(cc, fn):
    torch.cuda.synchronize()
    cc.pc.host_barrier()
    before = gb._C.cuda.launch_count()
    fn()
    torch.cuda.synchronize()
    cc.pc.host_barrier()
    after = gb._C.cuda.launch_count()
    cc.pc.host_barrier()
    return (after - before) // cc.pc.ranks_on_my_device()


def kernels_unfused(fn, count):
    """Device kernels and copies of one call of the unfused sequence (the library's own kernel
    included), from torch.profiler. The profiler must run on the main thread, so with ranks as
    threads it is not run (None) and the call only takes part in the allreduce."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    if not count:
        fn()
        torch.cuda.synchronize()
        return None
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(1 for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--threads", type=int, default=0, help="rehearsal: this many ranks as threads on cuda:0")
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--stage-mb", type=int, default=128)
    ap.add_argument("--backward", action="store_true", help="time the fused backward against its composition")
    ap.add_argument("--fp8", action="store_true", help="time the FP8 out against bf16 + torch quantisation")
    args = ap.parse_args()
    kind = "_backward" if args.backward else "_fp8" if args.fp8 else ""
    if args.threads:
        world = args.threads
        run = bench_backward_rank if args.backward else \
            (lambda ctx, dev, a, w: bench_fp8_rank(ctx, dev, a, w, False)) if args.fp8 else \
            (lambda ctx, dev, a, w: bench_rank(ctx, dev, a, w, False))
        rows = gb.spawn_threads(world, lambda ctx: run(ctx, 0, args, 1), cuda_device=0, timeout_ms=600000)[0]
        mode = f"{world} ranks as threads on one GPU: overhead only, not link numbers"
        info = gpu_info(0)
        rank = 0
    else:
        rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
        local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local)
        ctx = gb.init_context(rank, world, path=f"/tmp/glb_norm_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}",
                              timeout_ms=120000)
        rows = (bench_backward_rank if args.backward else bench_fp8_rank if args.fp8 else bench_rank)(ctx, local, args,
                                                                                                world)
        mode = f"{world} ranks, one per GPU"
        info = gpu_info(local)
    if rank == 0:
        doc = {"benchmark": "allreduce_residual_norm" + kind, "mode": mode, "ranks": world, **info, "iters": args.iters,
               "warmup": args.warmup, "reps": args.reps, "rows": rows}
        text = json.dumps(doc)
        print(text)
        if args.out:
            with open(args.out, "w") as f:
                f.write(text + "\n")


if __name__ == "__main__":
    main()
