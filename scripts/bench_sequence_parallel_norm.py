#!/usr/bin/env python
"""The fused sequence-parallel step (reduce-scatter + bias + residual add + RMSNorm / LayerNorm +
allgather of the normed rows, one kernel: `CudaContext.reduce_scatter_residual_norm`) against the
unfused sequence on the same inputs: `cc.reduce_scatter`, bias add, residual add, `F.rms_norm` /
`F.layer_norm`, `cc.allgather`.

Before timing, every shape checks that the fused call's shard and gathered out equal, byte for
byte, the matching rows of `allreduce_residual_norm` on the same inputs (the same sum order), and
records how far the unfused sequence, which rounds after each step, lands from it.

Run one rank per GPU under torch.distributed.run:

    python -m torch.distributed.run --nproc_per_node 8 scripts/bench_sequence_parallel_norm.py --out sp.json

or, for a rehearsal on one GPU, `--threads P` (P ranks as threads sharing cuda:0). Ranks that share
a card pay for each other's kernels and exchange through local memory, so those numbers measure
the per-call overhead only, not the link; the JSON says so. Timing as in bench_allreduce_norm.py:
CUDA events around `--iters` back-to-back calls after `--warmup`, median over `--reps` windows,
the maximum over ranks. T is the whole sequence (tokens of every rank).

`--backward` times the fused backward instead (`CudaContext.reduce_scatter_residual_norm_backward`:
reduce-scatter of the gathered out's gradient, the norm's backward, the add of the residual
stream's gradient and the allgather, one kernel per chunk plus one that finishes the column sums)
against the composition SequenceParallel's autograd ran before it: `cc.reduce_scatter`, the norm
recomputed under torch autograd, the add, the bias row sum and `cc.allgather`. Before timing, each
shape records how far the two gradients of `partial` lie apart.

`--fp8` times the FP8 form (`reduce_scatter_residual_norm(out_scales=)`: the gathered `out` as e4m3
codes with one fp32 scale per row, in the same launch, so the allgather carries codes) against the
fused bf16 call followed by the torch quantisation of its gathered `out` (`strategies.fp8_rows`),
with the launches per call of each (torch's kernels counted by torch.profiler, one rank per process
only). Each shape first checks that the two give the same bytes.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from bench_allreduce_norm import gpu_info, kernels_unfused, launches_fused, timed  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402
from gloo_b200.parallel.strategies import _norm_input_grad, fp8_rows  # noqa: E402

DECODE_T = (8, 64, 256)
PREFILL_T = (4096,)
HIDDEN = (4096, 8192)


def bench_rank(ctx, device, args, world):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype, P, rank = torch.bfloat16, ctx.size, ctx.rank
    rows = []
    for H in HIDDEN:
        for T in DECODE_T + PREFILL_T:
            Ts = T // P
            shard = slice(rank * Ts, (rank + 1) * Ts)
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            residual_full = torch.randn(T, H, generator=g).to(dtype).cuda()
            bias = torch.randn(H, generator=g).to(dtype).cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            partial = torch.randn(T, H, generator=torch.Generator().manual_seed(T * 131 + H + 7 + rank)).to(dtype).cuda()
            residual = residual_full[shard].contiguous()
            res_out, out = torch.empty_like(residual), torch.empty(T, H, dtype=dtype, device="cuda")
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused():
                    cc.reduce_scatter_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                                    residual_out=res_out, out=out)

                def unfused():
                    y = torch.empty_like(residual)
                    cc.reduce_scatter(y, partial)
                    s = residual + (y + bias)
                    o = F.rms_norm(s, (H,), weight, 1e-6) if norm == "rms" else F.layer_norm(s, (H,), weight, nb, 1e-6)
                    full = torch.empty(T, H, dtype=dtype, device="cuda")
                    cc.allgather(full, o)
                    return full

                s_ar, o_ar = cc.allreduce_residual_norm(partial, residual_full, weight, nb, norm=norm, eps=1e-6,
                                                        bias=bias, residual_out=torch.empty_like(residual_full))
                fused()
                o_ref = unfused()
                torch.cuda.synchronize()
                assert torch.equal(res_out, s_ar[shard]) and torch.equal(out, o_ar), f"T={T} H={H} {norm}: not identical"
                plan = gb._C.cuda.plan_reduce_scatter_norm(cc.pc, T, H, int(gb.DataType.BFLOAT16),
                                                           {"rms": 1, "layer": 2}[norm], True)
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "shard_bytes": Ts * H * 2,
                       "variant": plan["variant"], "launches": plan["launches"],
                       "max_abs_diff_unfused": float((out.float() - o_ref.float()).abs().max())}
                for name, fn in (("fused", fused), ("unfused", unfused)):
                    row[f"{name}_us"] = timed(ctx, cc, fn, stream, args, world)
                row["fused_launches_per_call"] = launches_fused(cc, fused)
                row["speedup"] = row["unfused_us"] / row["fused_us"]
                rows.append(row)
    return rows


def bench_fp8_rank(ctx, device, args, world, profile_composed=True):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype, P, rank = torch.bfloat16, ctx.size, ctx.rank
    rows = []
    for H in HIDDEN:
        for T in DECODE_T + PREFILL_T:
            Ts = T // P
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            residual = torch.randn(T, H, generator=g).to(dtype)[rank * Ts:(rank + 1) * Ts].contiguous().cuda()
            bias = torch.randn(H, generator=g).to(dtype).cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            partial = torch.randn(T, H, generator=torch.Generator().manual_seed(T * 131 + H + 7 + rank)).to(dtype).cuda()
            res_out, out = torch.empty_like(residual), torch.empty(T, H, dtype=dtype, device="cuda")
            codes = torch.empty(T, H, dtype=torch.float8_e4m3fn, device="cuda")
            scales = torch.empty(T, 1, dtype=torch.float32, device="cuda")
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused_fp8():
                    cc.reduce_scatter_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                                    residual_out=res_out, out=codes, out_scales=scales)

                def composed():
                    cc.reduce_scatter_residual_norm(partial, residual, weight, nb, norm=norm, eps=1e-6, bias=bias,
                                                    residual_out=res_out, out=out)
                    return fp8_rows(out)

                want_c, want_s = composed()
                fused_fp8()
                torch.cuda.synchronize()
                same = bool(torch.equal(codes.view(torch.uint8), want_c.view(torch.uint8)) and torch.equal(scales, want_s))
                plans = [gb._C.cuda.plan_reduce_scatter_norm(cc.pc, T, H, int(gb.DataType.BFLOAT16),
                                                             {"rms": 1, "layer": 2}[norm], True, fp8) for fp8 in (False, True)]
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "shard_bytes": Ts * H * 2,
                       "variant": plans[1]["variant"], "same_bytes": same, "bf16_chunk_rows": plans[0]["chunk_rows"],
                       "fp8_chunk_rows": plans[1]["chunk_rows"]}
                row["fp8_fused_us"] = timed(ctx, cc, fused_fp8, stream, args, world)
                row["bf16_fused_plus_torch_quant_us"] = timed(ctx, cc, composed, stream, args, world)
                row["fp8_fused_launches_per_call"] = launches_fused(cc, fused_fp8)
                row["composed_kernels_per_call"] = kernels_unfused(composed, profile_composed)
                row["speedup"] = row["bf16_fused_plus_torch_quant_us"] / row["fp8_fused_us"]
                rows.append(row)
    return rows


BACKWARD_T = (4096, 8192)


def bench_backward_rank(ctx, device, args, world):
    cc = gcu.CudaContext(ctx, device, stage_bytes=args.stage_mb << 20)
    cc.set_timeout(600000)
    stream = torch.cuda.current_stream()
    dtype, P, rank = torch.bfloat16, ctx.size, ctx.rank
    rows = []
    for H in HIDDEN:
        for T in BACKWARD_T:
            Ts = T // P
            g = torch.Generator(device="cpu").manual_seed(T * 131 + H)
            s = torch.randn(T, H, generator=g).to(dtype)[rank * Ts:(rank + 1) * Ts].contiguous().cuda()
            weight = (1 + 0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            norm_bias = (0.1 * torch.randn(H, generator=g)).to(dtype).cuda()
            mine = torch.Generator().manual_seed(T * 131 + H + 7 + rank)
            g_out = torch.randn(T, H, generator=mine).to(dtype).cuda()
            g_s = torch.randn(Ts, H, generator=mine).to(dtype).cuda()
            gp, gr = torch.empty(T, H, dtype=dtype, device="cuda"), torch.empty_like(s)
            gw, gnb, gb_ = (torch.empty(H, dtype=dtype, device="cuda") for _ in range(3))
            for norm in ("rms", "layer"):
                nb = norm_bias if norm == "layer" else None

                def fused():
                    cc.reduce_scatter_residual_norm_backward(g_out, s, g_s, weight, norm=norm, eps=1e-6,
                                                             grad_partial=gp, grad_residual=gr, grad_weight=gw,
                                                             grad_norm_bias=gnb if norm == "layer" else None,
                                                             grad_bias=gb_)

                def composed():
                    y = torch.empty_like(s)
                    cc.reduce_scatter(y, g_out)
                    gs, _, _ = _norm_input_grad(norm, H, 1e-6, s, weight, nb, y)
                    total = g_s + gs
                    total.sum(0)
                    full = torch.empty(T, H, dtype=dtype, device="cuda")
                    cc.allgather(full, total)
                    return full

                fused()
                ref = composed()
                torch.cuda.synchronize()
                vectors = 3 if norm == "layer" else 2
                plan = gb._C.cuda.plan_reduce_scatter_norm_backward(cc.pc, T, H, int(gb.DataType.BFLOAT16),
                                                                    {"rms": 1, "layer": 2}[norm], True, vectors)
                row = {"T": T, "H": H, "dtype": "bfloat16", "norm": norm, "shard_bytes": Ts * H * 2,
                       "variant": plan["variant"], "launches": plan["launches"], "chunk_rows": plan["chunk_rows"],
                       "max_abs_diff_composed": float((gp.float() - ref.float()).abs().max()),
                       "max_abs_grad": float(ref.float().abs().max())}
                for name, fn in (("fused", fused), ("composed", composed)):
                    row[f"{name}_us"] = timed(ctx, cc, fn, stream, args, world)
                row["speedup"] = row["composed_us"] / row["fused_us"]
                rows.append(row)
    return rows


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
    run = bench_backward_rank if args.backward else bench_fp8_rank if args.fp8 else bench_rank
    if args.threads:
        world = args.threads
        thread_run = (lambda ctx, dev, a, w: bench_fp8_rank(ctx, dev, a, w, False)) if args.fp8 else run
        rows = gb.spawn_threads(world, lambda ctx: thread_run(ctx, 0, args, 1), cuda_device=0, timeout_ms=600000)[0]
        mode = f"{world} ranks as threads on one GPU: overhead only, not link numbers"
        info, rank = gpu_info(0), 0
    else:
        rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
        local = int(os.environ.get("LOCAL_RANK", 0))
        torch.cuda.set_device(local)
        ctx = gb.init_context(rank, world, path=f"/tmp/glb_sp_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}",
                              timeout_ms=120000)
        rows = run(ctx, local, args, world)
        mode = f"{world} ranks, one per GPU"
        info = gpu_info(local)
    if rank == 0:
        name = "reduce_scatter_residual_norm" + ("_backward" if args.backward else "_fp8" if args.fp8 else "")
        doc = {"benchmark": name, "mode": mode, "ranks": world, **info, "iters": args.iters,
               "warmup": args.warmup, "reps": args.reps, "rows": rows}
        text = json.dumps(doc)
        print(text)
        if args.out:
            with open(args.out, "w") as f:
                f.write(text + "\n")


if __name__ == "__main__":
    main()
