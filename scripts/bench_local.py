#!/usr/bin/env python
"""How close the single-rank fused step (every buffer := sum of all, one pass) comes to what the
HBM can do, on the benchmark's buffers (2 x 400 MB fp32 on one GPU). Variants, alternated over
3 rounds, each timed as the p50 of 20 device-timed launches after 3 untimed ones:

  fused_ldg_stg   the step through localAllreduceManyKernel (16-byte LDG/STG, shape pinned to the
                  default 4 CTAs/SM x 1 pack)
  fused_bulk      the step as the library runs it at this size: localAllreduceManyBulkKernel
                  (cp.async.bulk tiles through shared memory)
  copy_ldg_stg    the same LDG/STG pattern with no arithmetic: the n = 1 step (A[i] = A[i]) on A,
                  then on B
  copy_bulk       the same through the bulk kernel
  memcpy_d2d      cudaMemcpyAsync device to device, A -> C and B -> D (torch copy_)
  read_only       one read of A and of B (torch sum)
  write_only      one write of A and of B (torch fill_)

The variants that read and write move 1.6 GB (0.8 GB each way), read_only and write_only 0.8 GB;
the rate is bytes moved / p50. Prints the card name, power limit and max SM clock from the same
process, one JSON line per variant and round, and a summary with each variant's median over
the rounds and the bulk step as a fraction of each ceiling. An argument writes the summary there.

--dtype (float32, bfloat16 or float8_e4m3fn; default float32) picks the element type of the step.
The buffers stay 2 x 400 MB whatever the dtype, so every rate compares directly with memcpy_d2d;
read_only and write_only run on a float32 view of the same bytes.

On an H100 80GB HBM3 (SXM, power limit 700 W, max SM clock 1980 MHz), medians of 3 rounds:
fused_ldg_stg 0.574 ms (2.79 TB/s), fused_bulk 0.537 ms (2.98 TB/s), copy_ldg_stg 0.587 ms,
copy_bulk 0.563 ms, memcpy_d2d 0.537 ms (2.98 TB/s), read_only 2.87 TB/s, write_only 3.21 TB/s.
The bulk step runs at 0.999 of the device-to-device copy and 1.07 of the LDG/STG step. Its time
here includes the stream-ordered allocation and zeroing of the tile counter that each
local_allreduce_many call makes for itself (bench.py's step, whose counter lives with the
algorithm object, takes 0.535-0.537 ms).
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import gloo_b200 as gb  # noqa: E402

cu = gb._C.cuda
NBYTES = 400_000_000  # per buffer
DTYPES = {"float32": (torch.float32, gb.DataType.FLOAT32), "bfloat16": (torch.bfloat16, gb.DataType.BFLOAT16),
          "float8_e4m3fn": (torch.float8_e4m3fn, gb.DataType.FLOAT8_E4M3)}
ROUNDS = 3
TIMED = 20


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i",
                              str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), (p.strip() for p in out.strip().split(","))))
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(), "nvidia-smi": f"unavailable: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("summary", nargs="?", help="write the summary JSON here")
    ap.add_argument("--dtype", choices=sorted(DTYPES), default="float32")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_local.py measures on a GPU"
    dtype, glb_dt = DTYPES[args.dtype][0], int(DTYPES[args.dtype][1])
    es = torch.empty((), dtype=dtype).element_size()
    N = NBYTES // es
    a, b = torch.ones(N, device="cuda", dtype=dtype), torch.ones(N, device="cuda", dtype=dtype)
    c, d = torch.empty(N, device="cuda", dtype=dtype), torch.empty(N, device="cuda", dtype=dtype)
    # float32 views of the same bytes for the read / write ceilings (torch reduces no FP8 tensor)
    a32, b32 = a.view(torch.float32), b.view(torch.float32)
    ones32 = torch.ones(4 // es, dtype=dtype).view(torch.float32).item()  # a float32 word of dtype ones
    stream = torch.cuda.current_stream().cuda_stream
    nbytes = N * es

    def step(ptrs, pinned):
        # pinned: the LDG/STG kernel whatever the size; otherwise the library's own choice
        cu.set_local_shape(4, 1, False) if pinned else cu.set_local_shape(0, 0, False)
        for p in ptrs:
            cu.local_allreduce_many(p, N, glb_dt, 1, 0.5 if len(p) > 1 else 1.0, stream)

    both, each = [[a.data_ptr(), b.data_ptr()]], [[a.data_ptr()], [b.data_ptr()]]
    variants = {
        "fused_ldg_stg": (lambda: step(both, True), 4 * nbytes),
        "fused_bulk": (lambda: step(both, False), 4 * nbytes),
        "copy_ldg_stg": (lambda: step(each, True), 4 * nbytes),
        "copy_bulk": (lambda: step(each, False), 4 * nbytes),
        "memcpy_d2d": (lambda: (c.copy_(a), d.copy_(b)), 4 * nbytes),
        "read_only": (lambda: (a32.sum(), b32.sum()), 2 * nbytes),
        "write_only": (lambda: (a32.fill_(ones32), b32.fill_(ones32)), 2 * nbytes),
    }
    info = card()
    print(json.dumps({"card": info, "dtype": args.dtype}), flush=True)
    per = {k: [] for k in variants}
    try:
        for rnd in range(ROUNDS):
            for name, (fn, moved) in variants.items():
                for _ in range(3):
                    fn()
                evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(TIMED)]
                for x, y in evs:
                    x.record()
                    fn()
                    y.record()
                torch.cuda.synchronize()
                ms = sorted(x.elapsed_time(y) for x, y in evs)[TIMED // 2]
                # the inputs are all ones and the fused step scales by 0.5: every variant keeps them so
                ok = all(t[i].float().item() == 1.0 for t in (a, b) for i in (0, N // 3, N - 1))
                assert ok, f"{name} changed the buffers"
                per[name].append(ms)
                print(json.dumps({"round": rnd, "variant": name, "ms": round(ms, 4),
                                  "gbs": round(moved / (ms * 1e-3) / 1e9, 1)}), flush=True)
    finally:
        cu.set_local_shape(0, 0, False)
    med = {k: sorted(v)[len(v) // 2] for k, v in per.items()}
    rate = {k: variants[k][1] / (med[k] * 1e-3) / 1e9 for k in variants}
    summary = {"card": info, "dtype": args.dtype, "rounds": ROUNDS, "launches_per_round": TIMED,
               "ms": {k: round(v, 4) for k, v in med.items()},
               "gbs": {k: round(v, 1) for k, v in rate.items()},
               "fused_bulk_over": {k: round(rate["fused_bulk"] / rate[k], 3) for k in variants if k != "fused_bulk"}}
    print("summary:", json.dumps(summary), flush=True)
    if args.summary:
        with open(args.summary, "w") as f:
            json.dump(summary, f, indent=1)


if __name__ == "__main__":
    main()
