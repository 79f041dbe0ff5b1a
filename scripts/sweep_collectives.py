#!/usr/bin/env python
"""Bandwidth sweep of the data-movement collectives (configs 4 and 5 of BASELINE.json):
allgather, alltoall, alltoall_v, broadcast, reduce_scatter — 1 KB .. 1 GB per-rank payload,
device-timed, max over ranks, against the NCCL comparator. torchrun, one rank per GPU.
Also the named fp16 schedules (config 3) with --schedules.

--plain (or --threads P) sweeps allgather, reduce_scatter, alltoall, alltoall_v, scatter and
reduce of PLAIN tensors (--plain-ops picks some), 1 MB .. 1 GB of what each rank sends or holds
(allgather output, reduce_scatter / alltoall / scatter root / reduce input), in four arms:
"staged" (payload copied through the staging pool, where it fits), "pipelined" (the pipelined
kernel: the default pool where the payload does not fit it, and a second context whose pool is
smaller than the payload but holds the pipelined slots where it does; alltoall_v always runs it),
"registered" (symmetric buffers, zero copy: the ceiling) and NCCL (more than one GPU, allgather /
reduce_scatter / alltoall). --threads P runs P ranks as threads on ONE GPU, each on its own
gcu.new_stream(): the ranks share that GPU's HBM, so those figures are not NVLink figures."""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402


def _timer(ctx, world, stream, flush):
    def timed(fn, iters):
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        with torch.cuda.stream(stream):
            for _ in range(3):
                fn()
            for a, b in evs:
                flush.fill_(0)
                a.record(stream)
                fn()
                b.record(stream)
        stream.synchronize()
        per = np.asarray([a.elapsed_time(b) * 1e3 for a, b in evs], dtype=np.float64)
        if world > 1:
            gb.allreduce(ctx, per, op=gb.ReduceOp.MAX)
        per.sort()
        return float(per[len(per) // 2])
    return timed


# Launch shape of the pipelined kernels at the defaults (GLB_CUDA_BLOCKS, GLB_CUDA_PIPE_TILE): one
# full-size slot is shares x 128 CTAs x 1024 x 16 bytes.
FULL_SLOT = 128 * 1024 * 16
HALVES = 2 * (256 << 10)      # the pool's two one-shot halves (GLB_CUDA_ONESHOT_MAX)
PLAIN_OPS = ("allgather", "reduce_scatter", "alltoall", "alltoall_v", "scatter", "reduce")


def _plain_shape(op, n, P):
    """(input elements, output elements, pool slots in full-size slot bytes, bytes the staged path
    compares with the bulk region, or None when it has no staged path) of one plain-tensor op, with
    `n` = the elements each rank sends / holds."""
    per = n // P
    if op == "allgather":
        return per, n, 2 * FULL_SLOT, n * 4
    if op == "reduce_scatter":
        return n, per, 2 * P * FULL_SLOT, n * 4
    if op == "alltoall":
        return n, n, 2 * P * FULL_SLOT, n * 4
    if op == "alltoall_v":
        return n, n, 2 * P * FULL_SLOT, None  # always pipelined
    if op == "scatter":
        return n, per, 2 * P * FULL_SLOT, per * 4
    return n, n, 2 * (P + 1) * FULL_SLOT, 2 * n * 4  # reduce: the staged path takes half the bulk region


def plain_rows(ctx, cc, ctx_small, P, rank, stream, iters, max_bytes, nccl, ops=PLAIN_OPS):
    """Rows of the plain-tensor arms. `ctx_small(stage_bytes)` returns a CudaContext with that
    pool on a context of its own (a context has one pool per device)."""
    bulk = cc.pc.stage_bytes() - HALVES
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    timed = _timer(ctx, P, stream, flush)
    F32 = int(gb.DataType.FLOAT32)
    sizes = [m << 20 for m in (1, 4, 16, 64, 256, 1024) if (m << 20) <= max_bytes]
    small = {}
    rows = []
    for op in ops:
        for total in sizes:
            n = total // 4 // P * P
            per = n // P
            n_in, n_out, slots, staged_bytes = _plain_shape(op, n, P)
            # alltoall_v: uneven but balanced split, rank r sends weight w[(j - r) % P] to rank j
            w = [k + 1 for k in range(P)]
            unit = [n * x // sum(w) for x in w]
            unit[-1] += n - sum(unit)
            send = [unit[(j - rank) % P] for j in range(P)]
            recv = [unit[(rank - i) % P] for i in range(P)]
            it = iters if total < (64 << 20) else max(5, iters // 4)
            row = {"op": op + "_plain", "bytes": n * 4}
            big_in = torch.ones(n_in, device="cuda")
            big_out = torch.empty(n_out, device="cuda")

            def call(c, o, i):
                if op == "allgather":
                    return lambda: c.allgather(o, i, stream=stream)
                if op == "reduce_scatter":
                    return lambda: c.reduce_scatter(o, i, [per] * P, stream=stream)
                if op == "alltoall":
                    return lambda: c.alltoall(o, i, stream=stream)
                if op == "alltoall_v":
                    return lambda: c.alltoallv(o, recv, i, send, stream=stream)
                if op == "scatter":
                    return lambda: c.scatter(o, i, root=0, stream=stream)
                return lambda: c.reduce(o, i, root=0, stream=stream)

            try:
                if staged_bytes is not None and staged_bytes <= bulk:
                    row["staged_us"] = round(timed(call(cc, big_out, big_in), it), 2)
                    if staged_bytes > slots:  # a pool that holds the pipelined slots but not the payload
                        if slots not in small:
                            small[slots] = ctx_small(slots + HALVES)
                        row["pipelined_pool_mb"] = round(small[slots].pc.stage_bytes() / 2**20, 1)
                        row["pipelined_us"] = round(timed(call(small[slots], big_out, big_in), it), 2)
                else:
                    row["pipelined_us"] = round(timed(call(cc, big_out, big_in), it), 2)
                sym_in = cc.empty(big_in.numel(), torch.float32)
                sym_in.fill_(1)
                sym_out = cc.empty(big_out.numel(), torch.float32)
                if op in ("allgather", "alltoall", "alltoall_v", "scatter"):
                    row["registered_us"] = round(timed(call(cc, sym_out, big_in), it), 2)
                elif op == "reduce_scatter":
                    row["registered_us"] = round(timed(call(cc, big_out, sym_in), it), 2)
                else:  # reduce: the registered path needs both buffers registered
                    row["registered_us"] = round(timed(call(cc, sym_out, sym_in), it), 2)
                del sym_in, sym_out
                if nccl is not None and op in ("allgather", "reduce_scatter", "alltoall"):
                    if op == "allgather":
                        fn = lambda: nccl.allgather(big_in.data_ptr(), big_out.data_ptr(), per, F32, stream.cuda_stream)  # noqa: E731
                    elif op == "reduce_scatter":
                        fn = lambda: nccl.reduce_scatter(big_in.data_ptr(), big_out.data_ptr(), per, F32, 1, stream.cuda_stream)  # noqa: E731
                    else:
                        fn = lambda: nccl.alltoall(big_in.data_ptr(), big_out.data_ptr(), per, F32, stream.cuda_stream)  # noqa: E731
                    row["nccl_us"] = round(timed(fn, it), 2)
                for k in [k for k in row if k.endswith("_us")]:
                    row[k[:-3] + "_gbs"] = round(n * 4 / (row[k] * 1e-6) / 1e9, 1)
            except Exception as e:  # noqa: BLE001
                row["error"] = f"{type(e).__name__}: {str(e)[:160]}"
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
            del big_in, big_out
            torch.cuda.synchronize()
            gb.barrier(ctx)
    return rows


def card_line():
    """Name and power limit of the card, read in the same run as the numbers."""
    import subprocess

    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()
    except Exception:  # noqa: BLE001
        return torch.cuda.get_device_name()


def threads_main(args):
    P = args.threads
    print(f"card: {card_line()}; {P} ranks as threads on cuda:0 sharing its HBM (not NVLink figures)", flush=True)

    def fn(ctx):
        stream = gcu.new_stream(0)
        made = []

        def ctx_small(stage):
            # A second context over the same threads (a context has one pool per device).
            c2 = gb.init_context(ctx.rank, P, store=store, prefix=f"small{len(made)}", timeout_ms=120000)
            made.append(c2)
            return gcu.CudaContext(c2, 0, stage_bytes=stage)

        cc = gcu.CudaContext(ctx, 0, stage_bytes=128 << 20)
        rows = plain_rows(ctx, cc, ctx_small, P, ctx.rank, stream, args.iters, args.max_bytes, None, args.plain_ops)
        torch.cuda.synchronize()
        for c2 in made:
            gb.barrier(c2)
        return rows

    store = gb._C.HashStore()
    rows = gb.spawn_threads(P, fn, cuda_device=0, timeout_ms=120000)[0]
    if args.out:
        with open(args.out, "w") as f:
            json.dump({"threads": P, "card": card_line(), "rows": rows}, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--max-bytes", type=int, default=1 << 30)
    ap.add_argument("--ops", default="allgather,alltoall,alltoall_v,broadcast,reduce_scatter")
    ap.add_argument("--schedules", action="store_true")
    ap.add_argument("--plain", action="store_true", help="also the plain-tensor arms")
    ap.add_argument("--plain-ops", type=lambda v: tuple(o for o in v.split(",") if o), default=PLAIN_OPS,
                    help="plain-tensor ops to sweep (default: " + ",".join(PLAIN_OPS) + ")")
    ap.add_argument("--threads", type=int, default=0, help="P ranks as threads on one GPU (plain arms only)")
    args = ap.parse_args()
    if args.threads:
        threads_main(args)
        return
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    ctx = gb.init_context(rank, world, path=f"/tmp/glb_swc_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}",
                          timeout_ms=120000)
    cc = gcu.CudaContext(ctx, local, stage_bytes=64 << 20)
    if rank == 0:
        print(cc.describe(), flush=True)
    try:
        nccl = gb._C.cuda.NcclComm.init_rank(ctx, local)
    except Exception as e:  # noqa: BLE001
        nccl = None
        if rank == 0:
            print("NCCL unavailable:", e)
    stream = torch.cuda.Stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    F32 = int(gb.DataType.FLOAT32)
    timed = _timer(ctx, world, stream, flush)

    rows = []
    sizes = []
    b = 1024
    while b <= args.max_bytes:
        sizes.append(b)
        b *= 8
    if sizes[-1] != args.max_bytes:
        sizes.append(args.max_bytes)
    ops = [o for o in args.ops.split(",") if o]
    P = world
    import gc

    maxn = max(P, sizes[-1] // 4 // P * P)
    for op in ops:
        # One symmetric buffer per op, sliced per size: every allocation binds a multicast
        # object, so allocating per size would exhaust them (and waste memory).
        big = cc.empty(maxn, torch.float32)
        big.fill_(1)
        for total in sizes:
            # `total` = bytes each rank ends up holding (allgather/alltoall output, broadcast
            # buffer, reduce_scatter input), i.e. the size that bounds the traffic.
            n = max(P, total // 4 // P * P)  # float32 elements, multiple of P
            per = n // P
            iters = args.iters if total < (64 << 20) else max(5, args.iters // 4)
            row = {"op": op, "bytes": n * 4}
            try:
                if op == "allgather":
                    out = big[:n]
                    inp = torch.ones(per, device="cuda")
                    row["ours_us"] = timed(lambda: cc.allgather(out, inp, stream=stream), iters)
                    if nccl:
                        o2 = torch.empty(n, device="cuda")
                        row["nccl_us"] = timed(lambda: nccl.allgather(inp.data_ptr(), o2.data_ptr(), per, F32, stream.cuda_stream), iters)
                    factor = (P - 1) / P
                elif op in ("alltoall", "alltoall_v"):
                    out = big[:n]
                    inp = torch.ones(n, device="cuda")
                    if op == "alltoall":
                        row["ours_us"] = timed(lambda: cc.alltoall(out, inp, stream=stream), iters)
                    else:
                        # uneven but balanced split: rank r sends weight w[(j - r) % P] to rank j, so
                        # every rank sends and receives n elements in chunks of very different sizes.
                        w = [k + 1 for k in range(P)]
                        unit = [n * x // sum(w) for x in w]
                        unit[-1] += n - sum(unit)
                        send = [unit[(j - rank) % P] for j in range(P)]
                        recv = [unit[(rank - i) % P] for i in range(P)]
                        out_v = big[:n]
                        row["ours_us"] = timed(lambda: cc.alltoallv(out_v, recv, inp, send, stream=stream), iters)
                    if nccl and op == "alltoall":
                        o2 = torch.empty(n, device="cuda")
                        row["nccl_us"] = timed(lambda: nccl.alltoall(inp.data_ptr(), o2.data_ptr(), per, F32, stream.cuda_stream), iters)
                    factor = (P - 1) / P
                elif op == "broadcast":
                    buf = big[:n]
                    row["ours_us"] = timed(lambda: cc.broadcast(buf, root=0, stream=stream), iters)
                    if world > 2 and cc.nvls_available() and n * 4 >= (1 << 20):
                        for m in (0, 1):
                            os.environ["GLB_CUDA_BCAST_MODE"] = str(m)
                            row[f"ours_mode{m}_us"] = round(timed(lambda: cc.broadcast(buf, root=0, stream=stream), iters), 2)
                        os.environ.pop("GLB_CUDA_BCAST_MODE", None)
                    if nccl:
                        o2 = torch.empty(n, device="cuda")
                        row["nccl_us"] = timed(lambda: nccl.broadcast(o2.data_ptr(), o2.data_ptr(), n, F32, 0, stream.cuda_stream), iters)
                    factor = 1.0
                elif op == "reduce_scatter":
                    inp = big[:n]
                    out = torch.empty(per, device="cuda")
                    row["ours_us"] = timed(lambda: cc.reduce_scatter(out, inp, [per] * P, stream=stream), iters)
                    if world > 2 and cc.nvls_available():
                        gb._C.cuda.set_tuning({"nvls_reduce_scatter": False})
                        row["ours_p2p_us"] = round(timed(lambda: cc.reduce_scatter(out, inp, [per] * P, stream=stream), iters), 2)
                        gb._C.cuda.set_tuning({"nvls_reduce_scatter": True})
                    if nccl:
                        i2 = torch.ones(n, device="cuda")
                        row["nccl_us"] = timed(lambda: nccl.reduce_scatter(i2.data_ptr(), out.data_ptr(), per, F32, 1, stream.cuda_stream), iters)
                    factor = (P - 1) / P
                else:
                    continue
                row["ours_busbw_gbs"] = round(n * 4 / (row["ours_us"] * 1e-6) / 1e9 * factor, 2)
                if "nccl_us" in row:
                    row["nccl_busbw_gbs"] = round(n * 4 / (row["nccl_us"] * 1e-6) / 1e9 * factor, 2)
                row["ours_us"] = round(row["ours_us"], 2)
                if "nccl_us" in row:
                    row["nccl_us"] = round(row["nccl_us"], 2)
            except Exception as e:  # noqa: BLE001
                row["error"] = f"{type(e).__name__}: {str(e)[:160]}"
            rows.append(row)
            if rank == 0:
                print(json.dumps(row), flush=True)
            torch.cuda.synchronize()
            gb.barrier(ctx)
        del big
        gc.collect()
    if args.schedules:
        for dtype, name in ((torch.float16, "float16"),):
            for n in (1 << 10, 1 << 16, 1 << 20, 1 << 24, 1 << 27):
                row = {"op": "allreduce_" + name, "elements": n, "bytes": n * 2}
                t = cc.empty(n, dtype)
                t.fill_(0)
                for label, cls, lit in (("auto", gcu.CudaAllreduceHalvingDoubling, False),
                                        ("halving_doubling", gcu.CudaAllreduceHalvingDoubling, True),
                                        ("bcube", gcu.CudaAllreduceBcube, True)):
                    algo = cls(ctx, t, streams=[stream], literal=lit)
                    row[label + "_us"] = round(timed(algo.run, args.iters if n < (1 << 24) else 6), 2)
                    if label == "auto":
                        row["auto_variant"] = algo.resolved_algo()
                if nccl:
                    row["nccl_us"] = round(timed(lambda: nccl.allreduce(t.data_ptr(), t.data_ptr(), n, int(gb.DataType.FLOAT16), 1, stream.cuda_stream), args.iters if n < (1 << 24) else 6), 2)
                best = min(row["auto_us"], row["halving_doubling_us"], row["bcube_us"])
                row["best_busbw_gbs"] = round(n * 2 / (best * 1e-6) / 1e9 * 2 * (P - 1) / P, 2)
                rows.append(row)
                if rank == 0:
                    print(json.dumps(row), flush=True)
                torch.cuda.synchronize()
                gb.barrier(ctx)
    if args.plain:
        if rank == 0:
            print(f"card: {card_line()}", flush=True)
        smalls = []

        def ctx_small(stage):
            c2 = gb.init_context(rank, world, path=f"/tmp/glb_swc_small{len(smalls)}_{os.environ.get('MASTER_PORT', '0')}_"
                                 f"{os.getppid()}", timeout_ms=120000)
            smalls.append(c2)
            return gcu.CudaContext(c2, local, stage_bytes=stage)

        rows += plain_rows(ctx, cc, ctx_small, world, rank, stream, args.iters, args.max_bytes, nccl, args.plain_ops)
    if rank == 0 and args.out:
        with open(args.out, "w") as f:
            json.dump({"world": world, "describe": cc.describe(), "rows": rows}, f, indent=1)
    torch.cuda.synchronize()
    gb.barrier(ctx)
    ctx.close_connections()


if __name__ == "__main__":
    main()
