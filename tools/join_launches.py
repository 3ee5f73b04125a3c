"""Join the C-ABI call log of tools/profile_step.py (gpurun_out/launch_shapes.json) with an ncu launch list (csv with
gpu__time_duration.sum) and print time per call shape -- which GEMM / conv / attention shapes the step spends its time in.

The join walks both lists in launch order; every C-ABI entry point is described by the sequence of kernel names it may launch
(optional members in brackets), so a planner change inside the library (split-K on/off, query split) cannot shift the alignment.

usage: join_launches.py launch_shapes.json launches.csv [top_n]
"""
import collections
import csv
import json
import re
import sys

calls = json.load(open(sys.argv[1]))
rows = [l for l in open(sys.argv[2]) if not l.startswith("==")]
kern = [(re.sub(r"\(.*", "", r["Kernel Name"]), float(r["Metric Value"].replace(",", "")) / 1e3) for r in csv.DictReader(rows)
        if "hcp::" in r["Kernel Name"]]

# fn -> list of (kernel-name substring, min count, max count), consumed in order
SEQ = {
    "hcp_gemm_bf16": [("gemm_wgmma_kernel", 1, 1), ("splitk_finalize", 0, 1)],
    "hcp_attn_fwd_bf16": [("attn_fwd", 1, 1)],
    # one attn_bwd_kernel launch per 64-column output slice of the head (d <= 192: at most three)
    "hcp_attn_bwd_bf16": [("attn_bwd_prep", 1, 1), ("attn_bwd_kernel", 1, 3), ("attn_bwd_post_kernel", 1, 1), ("attn_bwd_post_kv", 0, 1)],
    "hcp_groupnorm_fwd_bf16": [("gn", 1, 3)],
    "hcp_groupnorm_bwd_bf16": [("gn", 1, 3)],
    # wgrad_tc_kernel<64, true>; launch lists recorded by earlier builds name it lora_grad_tc_kernel
    "hcp_lora_grad_pair": [("grad_tc_kernel", 1, 1)],
    "hcp_lora_grad": [("grad_tc_kernel", 1, 1)],
    "hcp_adamw_flat": [("incr_step", 0, 1), ("adamw", 1, 1)],
    "hcp_adamw_flat_dev": [("incr_step", 1, 1), ("adamw_flat_dev", 1, 1)],
    "hcp_lion_flat_dev": [("lion_flat_dev", 1, 1)],
    "hcp_eps_loss_grouped": [("eps_loss_grouped", 1, 1), ("eps_loss_reduce", 1, 1)],
}


def seq_of(c):
    f = c["fn"]
    if f == "hcp_conv3x3_bf16":
        return [("gemm_wgmma_kernel", 4, 4)] if c.get("mode") == 1 else SEQ["hcp_gemm_bf16"]
    return SEQ.get(f, [("", 1, 1)])


agg = collections.defaultdict(lambda: [0, 0.0])
i = 0
for c in calls:
    t = 0.0
    for name, lo, hi in seq_of(c):
        n = 0
        while n < hi and i < len(kern) and name in kern[i][0]:
            t += kern[i][1]
            i += 1
            n += 1
        if n < lo:
            print(f"!! alignment lost at call {c} (wanted {name!r}, next kernel {kern[i][0] if i < len(kern) else None})")
            sys.exit(1)
    key = json.dumps({k: v for k, v in c.items()}, sort_keys=True)
    agg[key][0] += 1
    agg[key][1] += t
print("kernels consumed", i, "of", len(kern))
tot = sum(v[1] for v in agg.values())
print("total us", round(tot))
for k, (n, t) in sorted(agg.items(), key=lambda x: -x[1][1])[:int(sys.argv[3]) if len(sys.argv) > 3 else 40]:
    c = json.loads(k)
    fl = None
    if c["fn"] == "hcp_gemm_bf16":
        fl = 2.0 * c["M"] * c["N"] * sum(c["K"])
    elif c["fn"] == "hcp_conv3x3_bf16":
        s = c["stride"]
        fl = 2.0 * c["B"] * c["H"] * c["W"] * c["Cout"] * 9 * c["Cin"] / (s * s if c["mode"] == 0 else 1)
    elif c["fn"].startswith("hcp_attn"):
        fl = (4.0 if "fwd" in c["fn"] else 10.0) * c["B"] * c["H"] * c["Lq"] * c["Lkv"] * c["d"]
    tf = f"{fl / (t / n) * 1e-6:7.0f} TF/s" if fl else " " * 12
    print(f"{t:9.1f} us {100 * t / tot:5.1f}%  n={n:3d} avg={t / n:7.1f} {tf}  {k[:150]}")
