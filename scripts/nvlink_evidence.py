#!/usr/bin/env python
"""NVLink traffic of the hot allreduce kernels on the REAL multi-GPU path, from the driver's
per-link byte counters (``nvidia-smi nvlink -gt d``): bytes that crossed the links per step,
next to the algorithmic bytes of the variant (Nsight Compute cannot profile kernels of
different ranks that wait for each other). One rank per GPU
(torchrun). Writes one JSON document.
"""
import argparse
import json
import os
import re
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402
from gloo_b200.ops import cuda as gcu  # noqa: E402


def counters(index: int):
    """(tx_bytes, rx_bytes) summed over the links of one GPU, or None. The GPU is named by UUID:
    torch's index is relative to CUDA_VISIBLE_DEVICES, nvidia-smi's is not."""
    try:
        gpu = "GPU-" + str(torch.cuda.get_device_properties(index).uuid)
        out = subprocess.run(["nvidia-smi", "nvlink", "-gt", "d", "-i", gpu], capture_output=True, text=True, timeout=30).stdout
    except Exception:  # noqa: BLE001
        return None
    tx = [int(x) for x in re.findall(r"Data Tx:\s*(\d+)\s*KiB", out)]
    rx = [int(x) for x in re.findall(r"Data Rx:\s*(\d+)\s*KiB", out)]
    if not tx or not rx:
        return None
    return sum(tx) * 1024, sum(rx) * 1024


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="")
    ap.add_argument("--elements", type=int, default=100_000_000)
    ap.add_argument("--steps", type=int, default=50)
    args = ap.parse_args()
    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    ctx = gb.init_context(rank, world, path=f"/tmp/glb_nvl_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}", timeout_ms=120000)
    cc = gcu.CudaContext(ctx, local, stage_bytes=256 << 20)
    stream = torch.cuda.Stream()
    n, S = args.elements, args.elements * 4
    P = world
    rows = []
    sym = cc.empty(n, torch.float32)
    reg = torch.ones(n, device="cuda")
    cc.register(reg)
    plain = torch.ones(n, device="cuda")
    cases = [("two_shot", reg, "two_shot", 2 * S * (P - 1) / P, 2 * S * (P - 1) / P),
             ("pipelined", plain, "pipelined", None, None)]
    if cc.nvls_available():
        cases.insert(0, ("nvls", sym, "nvls", S * (1 + 1 / P), S * (1 + 1 / P)))
        cases[-1] = ("pipelined", plain, "pipelined", S * (1 + 1 / P), S * (1 + 1 / P))
    else:
        cases[-1] = ("pipelined", plain, "pipelined", 2 * S * (P - 1) / P, 2 * S * (P - 1) / P)
    for name, t, algo, alg_tx, alg_rx in cases:
        t.fill_(0.0)   # sums stay finite however many steps run
        if rank == 0:
            t.fill_(1.0)
        for _ in range(3):
            cc.allreduce(t, algo=algo, stream=stream)
        stream.synchronize()
        gb.barrier(ctx)
        # pass 1: time (no nvidia-smi anywhere near: the query takes 0.1-1 s and a different time on
        # every rank, which the first kernel of the loop would wait out)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        for _ in range(args.steps):
            cc.allreduce(t, algo=algo, stream=stream)
        b.record(stream)
        stream.synchronize()
        gb.barrier(ctx)
        # pass 2: the same steps between two counter reads
        torch.cuda.synchronize()
        before = counters(local)
        gb.barrier(ctx)
        for _ in range(args.steps):
            cc.allreduce(t, algo=algo, stream=stream)
        stream.synchronize()
        gb.barrier(ctx)
        after = counters(local)
        ms = np.asarray([a.elapsed_time(b) / args.steps])
        gb.allreduce(ctx, ms, op=gb.ReduceOp.MAX)
        row = {"variant": name, "ms_per_step": round(float(ms[0]), 4), "bytes": S,
               "algorithmic_tx_bytes_per_step": int(alg_tx), "algorithmic_rx_bytes_per_step": int(alg_rx)}
        if before and after:
            row["measured_tx_bytes_per_step"] = int((after[0] - before[0]) / args.steps)
            row["measured_rx_bytes_per_step"] = int((after[1] - before[1]) / args.steps)
            row["tx_over_algorithmic"] = round(row["measured_tx_bytes_per_step"] / alg_tx, 3)
            row["rx_over_algorithmic"] = round(row["measured_rx_bytes_per_step"] / alg_rx, 3)
            row["wire_gbs_tx"] = round(row["measured_tx_bytes_per_step"] / (row["ms_per_step"] * 1e-3) / 1e9, 1)
            row["wire_gbs_rx"] = round(row["measured_rx_bytes_per_step"] / (row["ms_per_step"] * 1e-3) / 1e9, 1)
        else:
            row["counters"] = "nvidia-smi nvlink -gt d unavailable"
        rows.append(row)
        if rank == 0:
            print(json.dumps(row), flush=True)
    if rank == 0 and args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            json.dump({"world": world, "describe": cc.describe(), "rows": rows}, f, indent=1)
    gb.barrier(ctx)
    ctx.close_connections()


if __name__ == "__main__":
    main()
