#!/usr/bin/env python
"""Regenerate profiles/sass_*.txt and profiles/sass_summary.md from the built library
(cuobjdump -sass, sm_90a). One listing per hot kernel + a table of the opcodes that prove what
the kernel does: 128-bit peer loads / stores, sys-scope flag traffic, multimem (LDGMC / STG..MC),
TMA bulk copies (UBLKCP), mbarrier traffic (SYNCS)."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "gloo_b200", "lib", "libglb.so")
OUT = os.path.join(ROOT, "profiles")

# (file tag, regex on the demangled kernel name)
KERNELS = [
    ("barrier", r"barrierKernel"),
    ("ll_allreduce_f32", r"llAllreduceKernel<float, float>"),
    ("ll_allreduce_f32_to_bf16", r"llAllreduceKernel<float, __nv_bfloat16>"),
    ("ll_exchange", r"llExchangeKernel"),
    ("ll_reduce_scatter_f32", r"llReduceScatterKernel<float>"),
    ("one_shot_f32", r"oneShotAllreduceKernel<float>"),
    ("one_shot_push_f32", r"oneShotPushAllreduceKernel<float>"),
    ("two_shot_f32_P2", r"twoShotAllreduceKernel<float, 2, 4>"),
    ("two_shot_f32_P8", r"twoShotAllreduceKernel<float, 8, 2>"),
    ("two_shot_f16_P8", r"twoShotAllreduceKernel<__half, 8, 2>"),
    ("nvls_f32", r"nvlsAllreduceKernel<float, 4>"),
    ("nvls_bf16", r"nvlsAllreduceKernel<__nv_bfloat16, 4>"),
    ("hybrid_nvls_p2p_f32_P8", r"hybridAllreduceKernel<float, 8>"),
    ("cast_f32_to_bf16", r"castAllreduceKernel<float, __nv_bfloat16>"),
    ("pipelined_f32_nvls", r"pipelinedAllreduceKernel<float, true, 0>"),
    ("pipelined_f32_P2", r"pipelinedAllreduceKernel<float, false, 2>"),
    ("pipelined_allgather", r"pipelinedAllgatherKernel"),
    ("pipelined_reduce_scatter_bf16_P8", r"pipelinedReduceScatterKernel<__nv_bfloat16, 8>"),
    ("pipelined_alltoall", r"pipelinedAlltoallKernel"),
    ("pipelined_reduce_bf16_P8", r"pipelinedReduceKernel<__nv_bfloat16, 8>"),
    ("reduce_pull_f32_P8", r"reducePullKernel<float, 8, 2>"),
    ("broadcast", r"broadcastKernel"),
    ("gather_push", r"gatherPushKernel"),
    ("alltoall_push", r"alltoallPushKernel"),
    ("alltoallv_dev", r"alltoallvDevKernel<false>"),
    ("alltoallv_dev_fp8", r"alltoallvDevKernel<true>"),
    ("combine_topk_bf16", r"moeCombineTopkKernel<__nv_bfloat16>"),
    ("combine_topk_f16", r"moeCombineTopkKernel<__half>"),
    ("combine_topk_f32", r"moeCombineTopkKernel<float>"),
    ("combine_topk_backward_bf16", r"moeCombineTopkBackwardKernel<__nv_bfloat16>"),
    ("combine_topk_backward_f16", r"moeCombineTopkBackwardKernel<__half>"),
    ("combine_topk_backward_f32", r"moeCombineTopkBackwardKernel<float>"),
    ("dispatch_topk", r"moeDispatchTopkKernel<false>"),
    ("dispatch_topk_fp8", r"moeDispatchTopkKernel<true>"),
    ("ll_dispatch_topk", r"moeLLDispatchKernel<false>"),
    ("ll_dispatch_topk_fp8", r"moeLLDispatchKernel<true>"),
    ("ll_combine_topk_bf16", r"moeLLCombineKernel<__nv_bfloat16>"),
    ("ll_combine_topk_f16", r"moeLLCombineKernel<__half>"),
    ("ll_combine_topk_f32", r"moeLLCombineKernel<float>"),
    ("reduce_scatter_norm_bf16_rms", r"allreduceNormKernel<__nv_bfloat16, 1, 4, false>"),
    ("reduce_scatter_norm_f32_layer", r"allreduceNormKernel<float, 2, 4, false>"),
    ("reduce_scatter_norm_fp8_bf16_rms", r"allreduceNormKernel<__nv_bfloat16, 1, 4, true>"),
    ("allreduce_norm_fp8_bf16_layer_two_shot", r"allreduceNormKernel<__nv_bfloat16, 2, 2, true>"),
    ("reduce_scatter_norm_backward_bf16_rms", r"normBackwardKernel<__nv_bfloat16, 1, 4>"),
    ("allreduce_norm_backward_bf16_rms_one_shot", r"normBackwardKernel<__nv_bfloat16, 1, 1>"),
    ("allreduce_norm_backward_bf16_rms_two_shot", r"normBackwardKernel<__nv_bfloat16, 1, 2>"),
    ("allreduce_norm_backward_f32_layer_two_shot", r"normBackwardKernel<float, 2, 2>"),
    ("allreduce_norm_backward_finish_bf16", r"normBackwardFinishAllreduceKernel<__nv_bfloat16>"),
    ("p2p_sendrecv", r"p2pKernel"),
    ("exchange_zero_copy", r"exchangeKernel<false>"),
    ("exchange_zero_copy_tma", r"exchangeKernel<true>"),
    ("peer_copy", r"peerCopyKernel"),
    ("peer_bulk_copy_tma", r"peerBulkCopyKernel"),
    ("schedule_f32", r"scheduleKernel<float>"),
    ("local_allreduce_many_f32", r"localAllreduceManyKernel<float>"),
    ("local_reduce_many_f32", r"localReduceManyKernel<float>"),
]


def main():
    sass = subprocess.run(["cuobjdump", "-sass", LIB], capture_output=True, text=True, check=True).stdout
    # split per function
    funcs, cur, name = {}, [], None
    for line in sass.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                funcs[name] = cur
            name, cur = m.group(1), []
        elif name:
            cur.append(line)
    if name:
        funcs[name] = cur
    mangled = list(funcs)
    dem = subprocess.run(["c++filt"], input="\n".join(mangled), capture_output=True, text=True).stdout.splitlines()
    rows = []
    for tag, pat in KERNELS:
        hit = [m for m, d in zip(mangled, dem) if re.search(re.escape(pat), d)]
        if not hit:
            print("missing:", pat, file=sys.stderr)
            continue
        body = funcs[hit[0]]
        ops = [re.sub(r"^\s*/\*[0-9a-f]+\*/\s*", "", ln).split(";")[0] for ln in body if re.match(r"\s*/\*[0-9a-f]{4}\*/", ln)]
        ops = [re.sub(r"^@!?U?P\d+\s+", "", o).split()[0] for o in ops if o.strip()]
        with open(os.path.join(OUT, f"sass_{tag}.txt"), "w") as f:
            f.write(f"// {dem[mangled.index(hit[0])]}\n// cuobjdump -sass gloo_b200/lib/libglb.so (sm_90a)\n")
            f.write("\n".join(body) + "\n")

        def count(rx):
            return sum(1 for o in ops if re.search(rx, o))
        notable = sorted({o for o in ops if re.search(r"LDGMC|MULTIMEM|UBLKCP|SYNCS|UTMA|MEMBAR|STRONG\.SYS|\.MC\b|RED\.|ATOM", o)})
        rows.append((tag, len(ops), count(r"^LDG\.E.*128"), count(r"^STG\.E.*128"), count(r"^LDG.*STRONG\.SYS"),
                     count(r"^STG.*STRONG\.SYS"), count(r"UBLKCP"), ", ".join(notable[:10])))
    with open(os.path.join(OUT, "sass_summary.md"), "w") as f:
        f.write("# SASS evidence (`python scripts/sass_report.py`: cuobjdump -sass gloo_b200/lib/libglb.so, sm_90a)\n\n"
                "Peer traffic is plain `LDG.E.128` / `STG.E.128` on NVLink-mapped addresses in the same kernel as the\n"
                "reduction; flag barriers and flag-in-data lines are `ST/LD.E.STRONG.SYS`; the NVLS kernels show the multimem\n"
                "instructions (`LDGMC.E.ADD…`, stores to the multicast alias); the TMA copy kernels show `UBLKCP.S.G` /\n"
                "`UBLKCP.G.S` (cp.async.bulk) with `SYNCS.*` mbarrier traffic. These are bandwidth / latency kernels: a\n"
                "collectives library has no GEMM, hence no `UTC*MMA`.\n\n"
                "| kernel | instructions | 128-bit loads | 128-bit stores | sys-scope ld | sys-scope st | UBLKCP | notable opcodes |\n"
                "|---|---|---|---|---|---|---|---|\n")
        for r in rows:
            f.write("| " + " | ".join(str(x) for x in r) + " |\n")
    print(f"wrote {len(rows)} listings")


if __name__ == "__main__":
    main()
