#!/usr/bin/env python
"""Measure the tuning table of the CUDA collectives on this box.

One rank per GPU (torchrun, or the driver's launcher)::

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 8 --master-addr 127.0.0.1 \
        --master-port 29533 -m gloo_b200.tune --out gpurun_out/tune_P8

For every message size of a geometric sweep and every kind of buffer (``sym``: library
symmetric memory with an NVSwitch multicast alias, ``reg``: peer-registered cudaMalloc
memory, ``user``: plain pointer through the pool) every applicable kernel variant is timed
with every launch shape of a small grid (CTAs x unroll, tile for the pipelined kernel):
device-timed with CUDA events, max over ranks, median of the iterations, L2 flushed between
iterations. The fastest candidate per size becomes a table entry; adjacent sizes with the
same choice are merged. ``<out>.tune`` is the table (`GLB_TUNE_FILE`, or copy it to
``gloo_b200/tuning/h100.tune``), ``<out>.json`` keeps every measurement, including the NCCL
comparator at the same sizes, so the table can be audited: AUTO must never be more than a
few percent off the best pinned variant.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np


def geometric_sizes(lo: int, hi: int, per_octave: int = 1):
    out, x = [], float(lo)
    while x <= hi * 1.0001:
        out.append(int(round(x / 16)) * 16 if x >= 64 else int(x))
        x *= 2 ** (1.0 / per_octave)
    return sorted(set(max(4, s) for s in out))


def compress(results, P, dtype_name="float32", device_name="NVIDIA H100 80GB HBM3", cores=132):
    """Measurements -> table lines (see the module docstring)."""
    # ---- compress into a table ---------------------------------------------------------------------------
    # Raw "fastest candidate per size" is noisy: shapes within a few percent of each other trade
    # places from size to size. Per (collective, buffer kind): (1) pick the fastest ALGORITHM per
    # size; (2) for every run of consecutive sizes with the same algorithm pick ONE launch shape
    # if some shape is within TOL of the best at every size of the run, else split the run.
    TOL = 1.04
    lines = [f"# gloo_b200 tuning table: P={P} dtype={dtype_name} device={device_name}",
             f"# measured by gloo_b200.tune ({len(results)} measurements); {cores} SMs; shapes merged within {int((TOL - 1) * 100)} % of the best"]
    by = {}
    for r in results:
        if r.get("us") and r["kind"] != "nccl":
            by.setdefault((r["coll"], r["kind"]), {}).setdefault(r["bytes"], []).append(r)

    def shape(c):
        return (c.get("blocks", 0), c.get("unroll", 0), c.get("tile", 0))

    def pick(run):
        """run: list of (bytes, [candidates of the chosen algo]) -> list of (last_bytes, shape)."""
        common = None
        for _, cands in run:
            best = min(c["us"] for c in cands)
            ok = {shape(c) for c in cands if c["us"] <= best * TOL}
            common = ok if common is None else (common & ok)
        if common:
            # among the shapes good everywhere take the one with the smallest total time
            tot = {sh: sum(min(c["us"] for c in cands if shape(c) == sh) for _, cands in run) for sh in common}
            return [(run[-1][0], min(tot, key=tot.get))]
        if len(run) == 1:
            return [(run[0][0], shape(min(run[0][1], key=lambda c: c["us"])))]
        mid = len(run) // 2
        return pick(run[:mid]) + pick(run[mid:])

    for (coll, kind), per_size in sorted(by.items()):
        sizes_here = sorted(per_size)
        chosen = []  # (bytes, algo, candidates of that algo)
        for nb in sizes_here:
            best = min(per_size[nb], key=lambda c: c["us"])
            chosen.append((nb, best["algo"], [c for c in per_size[nb] if c["algo"] == best["algo"]]))
        entries = []  # (last_bytes, algo, shape)
        i = 0
        while i < len(chosen):
            j = i
            while j + 1 < len(chosen) and chosen[j + 1][1] == chosen[i][1]:
                j += 1
            for last, sh in pick([(c[0], c[2]) for c in chosen[i:j + 1]]):
                entries.append((last, chosen[i][1], sh))
            i = j + 1
        # merge neighbours that ended up identical
        merged = []
        for e in entries:
            if merged and merged[-1][1:] == e[1:]:
                merged[-1] = e
            else:
                merged.append(e)
        for k, (last, algo, (bl, un, tl)) in enumerate(merged):
            if k == len(merged) - 1:
                bound = "inf"
            else:
                nxt = next(x for x in sizes_here if x > last)
                bound = str(int((last * nxt) ** 0.5))  # geometric midpoint between measured sizes
            line = f"{coll} P={P} buf={kind} maxbytes={bound} algo={algo} blocks={bl}"
            if un:
                line += f" unroll={un}"
            if tl:
                line += f" tile={tl}"
            lines.append(line)
    return lines


def merge_tables(base_lines, new_lines, min_bytes):
    """Replace, per (collective, P, buffer kind) that ``new_lines`` covers, the part of ``base_lines`` from
    ``min_bytes`` up with ``new_lines`` (a focused re-tune of the large sizes keeps the small-size rows)."""
    def parse(line):
        f = line.split()
        kv = dict(x.split("=", 1) for x in f[1:])
        mb = float("inf") if kv["maxbytes"] == "inf" else float(kv["maxbytes"])
        return (f[0], kv["P"], kv["buf"]), mb

    new = [ln for ln in new_lines if ln.strip() and not ln.startswith("#")]
    keys = {parse(ln)[0] for ln in new}
    out, clipped = [], set()
    for ln in base_lines:
        if not ln.strip() or ln.startswith("#"):
            out.append(ln)
            continue
        key, mb = parse(ln)
        if key not in keys or mb < min_bytes:
            out.append(ln)
        elif key not in clipped:  # the row that straddles min_bytes keeps its lower part
            clipped.add(key)
            out.append(" ".join(x if not x.startswith("maxbytes=") else f"maxbytes={int(min_bytes) - 1}" for x in ln.split()))
            out.extend(l2 for l2 in new if parse(l2)[0] == key)
    for key in keys - clipped:
        out.extend(l2 for l2 in new if parse(l2)[0] == key)
    return out


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="gpurun_out/tune")
    ap.add_argument("--dtype", default="float32")
    ap.add_argument("--min-bytes", type=int, default=1024)
    ap.add_argument("--max-bytes", type=int, default=512 << 20)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--quick", action="store_true", help="coarser grid (half the shapes, every other size)")
    ap.add_argument("--collectives", default="allreduce,allgather,alltoall,reduce_scatter,broadcast")
    ap.add_argument("--kinds", default="sym,reg,user")
    ap.add_argument("--no-nccl", action="store_true")
    ap.add_argument("--stage-mb", type=int, default=256)
    ap.add_argument("--merge", nargs=3, metavar=("BASE", "NEW", "OUT"), help="no measurement: splice table NEW into BASE from --merge-min-bytes up")
    ap.add_argument("--merge-min-bytes", type=int, default=1 << 20)
    ap.add_argument("--focus", default="", help="'nvls': only the multicast kernels (NVLS with few CTAs, NVLS + P2P hybrid) on symmetric buffers")
    ap.add_argument("--compress-json", default="", help="no measurement: rebuild the table from a saved <out>.json")
    args = ap.parse_args(argv)
    if args.merge:
        base, new, out = args.merge
        with open(base) as f:
            base_lines = f.read().splitlines()
        with open(new) as f:
            new_lines = f.read().splitlines()
        with open(out, "w") as f:
            f.write("\n".join(merge_tables(base_lines, new_lines, args.merge_min_bytes)) + "\n")
        return 0
    if args.compress_json:
        with open(args.compress_json) as f:
            saved = json.load(f)
        print("\n".join(compress(saved["results"], saved["world"], saved.get("dtype", "float32"))))
        return 0

    import torch

    import gloo_b200 as gb
    from gloo_b200.ops import cuda as gcu

    rank, world = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1))
    local = int(os.environ.get("LOCAL_RANK", 0))
    torch.cuda.set_device(local)
    dtype = getattr(torch, args.dtype)
    es = torch.empty((), dtype=dtype).element_size()
    path = f"/tmp/glb_tune_{os.environ.get('MASTER_PORT', '0')}_{os.getppid()}"
    ctx = gb.init_context(rank, world, path=path, timeout_ms=180000)
    cu = gb._C.cuda
    cu.tuning_clear()  # measure with explicit shapes only
    cc = gcu.CudaContext(ctx, local, stage_bytes=args.stage_mb << 20)
    say = (lambda *a: print(*a, flush=True)) if rank == 0 else (lambda *a: None)
    say(cc.describe())
    nccl = None
    if not args.no_nccl and world > 1:
        try:
            nccl = cu.NcclComm.init_rank(ctx, local)
        except Exception as e:  # noqa: BLE001
            say("NCCL comparator unavailable:", e)
    stream = torch.cuda.Stream()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    dt_code = int({torch.float32: gb.DataType.FLOAT32, torch.float16: gb.DataType.FLOAT16,
                   torch.bfloat16: gb.DataType.BFLOAT16}[dtype])

    def timed(fn, nbytes):
        iters = args.iters if nbytes <= (32 << 20) else max(6, args.iters // 3)
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
        with torch.cuda.stream(stream):
            for _ in range(2):
                fn()
            for a, b in evs:
                if nbytes < (128 << 20):
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

    sizes = geometric_sizes(args.min_bytes, args.max_bytes, 1)
    if args.quick:
        sizes = sizes[::2] + ([sizes[-1]] if (len(sizes) - 1) % 2 else [])
    cores = torch.cuda.get_device_properties(local).multi_processor_count
    blocks_bw = [32, 64, 96, 128, cores] if not args.quick else [64, 128, cores]
    blocks_light = [64, cores, cores * 3 // 2, cores * 2] if not args.quick else [cores, cores * 2]
    collectives = [c for c in args.collectives.split(",") if c]
    kinds = [k for k in args.kinds.split(",") if k]
    results = []   # every measurement
    table = []     # (coll, kind, bytes, best dict)
    ll_max = cc.pc.ll_max_bytes()
    P = world

    def record(coll, kind, nbytes, cands):
        """cands: list of dicts with 'us'. Stores all, returns the best."""
        ok = [c for c in cands if c.get("us")]
        for c in cands:
            results.append(dict(c, coll=coll, kind=kind, bytes=nbytes))
        if not ok:
            return None
        best = min(ok, key=lambda c: c["us"])
        table.append((coll, kind, nbytes, best))
        return best

    def attempt(label, fn, nbytes, **shape):
        try:
            us = timed(fn, nbytes)
            return dict(algo=label, us=round(us, 2), **shape)
        except Exception as e:  # noqa: BLE001
            say(f"  {label} {shape} @ {nbytes}: {type(e).__name__}: {str(e)[:160]}")
            return dict(algo=label, us=None, **shape)

    # ---- allreduce ----------------------------------------------------------------------------
    if "allreduce" in collectives and world > 1:
        for nbytes in sizes:
            n = max(1, nbytes // es)
            nb = n * es
            sym = cc.empty(n, dtype)
            sym.fill_(1)
            reg = torch.ones(n, dtype=dtype, device="cuda")
            cc.register(reg)
            plain = torch.ones(n, dtype=dtype, device="cuda")
            torch.cuda.synchronize()
            ref = None
            if nccl is not None:
                ref = attempt("nccl", lambda: nccl.allreduce(plain.data_ptr(), plain.data_ptr(), n, dt_code, 1, stream.cuda_stream), nb)
            for kind in kinds:
                t = {"sym": sym, "reg": reg, "user": plain}[kind]
                cands = []
                focus = args.focus == "nvls"
                if nb <= ll_max and not focus:
                    for b in (1, 4, 16, 64):
                        if b > 1 and nb < b * 512:
                            continue  # more CTAs than 8-byte units to hand out
                        cands.append(attempt("ll", lambda: cc.allreduce(t, algo="ll", stream=stream, blocks=b), nb, blocks=b))
                if nb * P <= (256 << 10) * 2 and nb <= (128 << 10) and not focus:
                    for b in (2, 8, 16):
                        cands.append(attempt("one_shot", lambda: cc.allreduce(t, algo="one_shot", stream=stream, blocks=b), nb, blocks=b))
                if kind in ("sym", "reg") and nb >= 4096 and not focus:
                    unrolls = {2: (2, 4, 8), 4: (1, 2, 4), 8: (1, 2)}.get(P, (0,))
                    for b in blocks_bw:
                        for u in unrolls:
                            cands.append(attempt("two_shot", lambda: cc.allreduce(t, algo="two_shot", stream=stream, blocks=b, unroll=u), nb,
                                                 blocks=b, unroll=u))
                if kind == "sym" and cc.nvls_available() and nb >= 4096:
                    nvls_blocks = [4, 8, 16, 24, 32, 48, 64, 96] if args.focus == "nvls" else blocks_bw + [cores * 3 // 2, cores * 2]
                    for b in nvls_blocks:
                        for u in ((2, 4) if args.focus == "nvls" else (2, 4, 8)):
                            cands.append(attempt("nvls", lambda: cc.allreduce(t, algo="nvls", stream=stream, blocks=b, unroll=u), nb,
                                                 blocks=b, unroll=u))
                if kind == "sym" and cc.nvls_available() and nb >= (1 << 20) and P in (2, 4, 8) and args.focus == "nvls":
                    # blocks = all CTAs, unroll = CTAs of the multicast part, tile = per-mille done peer to peer
                    for b in (64, 96, 128, cores):
                        for nb_mc in (8, 16, 24, 32):
                            for pm in (100, 175, 250, 350, 500):
                                cands.append(attempt("hybrid", lambda: cc.allreduce(t, algo="hybrid", stream=stream, blocks=b,
                                                                                    unroll=nb_mc, tile=pm), nb,
                                                     blocks=b, unroll=nb_mc, tile=pm))
                if kind == "user" and nb >= 32768 and args.focus != "nvls":
                    for b in ([64, 128, cores] if not args.quick else [cores]):
                        for tile in (256, 1024, 4096):
                            for xw in (4, 8, 12):  # exchange warps of the 16 per CTA
                                cands.append(attempt("pipelined", lambda: cc.allreduce(t, algo="pipelined", stream=stream, blocks=b,
                                                                                       tile=tile, unroll=xw), nb,
                                                     blocks=b, tile=tile, unroll=xw))
                best = record("allreduce", kind, nb, cands)
                if best:
                    bus = nb / (best["us"] * 1e-6) / 1e9 * 2 * (P - 1) / P
                    say(f"allreduce {kind:4s} {nb:>11d} B  best {best['algo']:9s} {best}  busbw {bus:8.1f} GB/s"
                        + (f"  nccl {ref['us']} us" if ref and ref.get("us") else ""))
            if ref:
                results.append(dict(ref, coll="allreduce", kind="nccl", bytes=nb))
            del sym, reg, plain
            torch.cuda.synchronize()
            gb.barrier(ctx)

    # ---- data movement: CTA count (and LL vs barrier for the small ones) ----------------------------
    def movement(coll):
        for nbytes in sizes:
            per = max(16, nbytes // P // 16 * 16)  # bytes per rank block
            total = per * P
            if total > (1 << 30):
                continue
            out = cc.empty(total, torch.uint8)
            inp = torch.ones(total, dtype=torch.uint8, device="cuda")
            torch.cuda.synchronize()
            cands = []
            ref = None
            if coll == "allgather":
                call = lambda: cc.allgather(out, inp[:per], stream=stream)  # noqa: E731
                if nccl is not None:
                    ref = attempt("nccl", lambda: nccl.allgather(inp.data_ptr(), out.data_ptr(), per, int(gb.DataType.UINT8), stream.cuda_stream), total)
            elif coll == "alltoall":
                call = lambda: cc.alltoall(out, inp, stream=stream)  # noqa: E731
                if nccl is not None:
                    ref = attempt("nccl", lambda: nccl.alltoall(inp.data_ptr(), out.data_ptr(), per, int(gb.DataType.UINT8), stream.cuda_stream), total)
            elif coll == "broadcast":
                call = lambda: cc.broadcast(out, root=0, stream=stream)  # noqa: E731
                if nccl is not None:
                    ref = attempt("nccl", lambda: nccl.broadcast(out.data_ptr(), out.data_ptr(), total, int(gb.DataType.UINT8), 0, stream.cuda_stream), total)
            else:  # reduce_scatter (float32)
                fin = cc.empty(total // 4, torch.float32)
                fout = torch.empty(per // 4, device="cuda")
                fin.fill_(1)
                call = lambda: cc.reduce_scatter(fout, fin, stream=stream)  # noqa: E731
                if nccl is not None:
                    ref = attempt("nccl", lambda: nccl.reduce_scatter(fin.data_ptr(), fout.data_ptr(), per // 4, int(gb.DataType.FLOAT32), 1, stream.cuda_stream), total)
            small = per <= ll_max and coll in ("allgather", "alltoall", "reduce_scatter")
            if small:
                cu.tuning_clear()
                cu.set_tuning({"ll_max_bytes": ll_max})
                cands.append(attempt("ll", call, total, blocks=0))
                cu.set_tuning({"ll_max_bytes": 0})
            for b in blocks_light:
                cu.tuning_clear()
                cu.tuning_load_string(f"{coll} P={P} buf=reg maxbytes=inf algo=push blocks={b}\n"
                                      f"{coll} P={P} buf=sym maxbytes=inf algo=push blocks={b}\n")
                cu.set_tuning({"copy_blocks": 512, "max_blocks": b})
                cands.append(attempt("push", call, total, blocks=b))
            if coll == "broadcast" and P > 2:
                # the four kernels behind cc.broadcast (planBroadcast honours the algo name of a table row)
                for name in ("direct", "scatter", "nvls", "relay"):
                    if name == "direct" and total * (P - 1) > (1 << 30):
                        continue
                    if name == "nvls" and not cc.nvls_available():
                        continue
                    for b in ([64, cores] if args.quick else [32, 64, cores]):
                        cu.tuning_clear()
                        cu.tuning_load_string(f"broadcast P={P} buf=reg maxbytes=inf algo={name} blocks={b}\n")
                        cu.set_tuning({"copy_blocks": 512, "max_blocks": b})
                        cands.append(attempt(name, call, total, blocks=b))
            if coll == "allgather" and per >= (256 << 10):
                for b in (cores // 4, cores // 2, cores):  # TMA variant: cp.async.bulk through shared memory, 1 CTA per SM
                    cu.tuning_clear()
                    cu.tuning_load_string(f"allgather P={P} buf=reg maxbytes=inf algo=tma blocks={b}\n")
                    cu.set_tuning({"copy_blocks": 512, "max_blocks": cores})
                    cands.append(attempt("tma", call, total, blocks=b))
            cu.tuning_clear()
            cu.set_tuning({"ll_max_bytes": 16384, "copy_blocks": cores * 2, "max_blocks": 128})
            best = record(coll, "reg", per if coll != "broadcast" else total, cands)
            if best:
                bw = total / (best["us"] * 1e-6) / 1e9 * ((P - 1) / P if coll != "broadcast" else 1.0)
                say(f"{coll:14s} {total:>11d} B  best {best}  busbw {bw:8.1f} GB/s" + (f"  nccl {ref['us']} us" if ref and ref.get("us") else ""))
            if ref:
                results.append(dict(ref, coll=coll, kind="nccl", bytes=total))
            del out, inp
            torch.cuda.synchronize()
            gb.barrier(ctx)

    for coll in ("allgather", "alltoall", "reduce_scatter", "broadcast"):
        if coll in collectives and world > 1:
            movement(coll)

    lines = compress(results, P, args.dtype, torch.cuda.get_device_name(local), cores)
    text = "\n".join(lines) + "\n"
    if rank == 0:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out + ".tune", "w") as f:
            f.write(text)
        with open(args.out + ".json", "w") as f:
            json.dump({"world": world, "dtype": args.dtype, "describe": cc.describe(), "results": results}, f)
        print(text, flush=True)
    torch.cuda.synchronize()
    gb.barrier(ctx)
    ctx.close_connections()


if __name__ == "__main__":
    sys.exit(main())
