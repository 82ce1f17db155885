#!/usr/bin/env python
"""Summarise an `ncu --metrics gpu__time_duration.sum --csv` launch list by kernel family.

usage: python tools/summarize_launches.py launches.csv [--skip N] [--steps K]
Times under ncu are cold-cache and serialised: use the SHARES, never the absolute numbers, as bench values."""
import csv
import re
import sys
from collections import defaultdict


def family(name):
    m = re.search(r"vj::(\w+)", name)
    if m:
        k = m.group(1)
        if k in ("gemm_kernel", "gemm_wgrad_kernel"):
            # gemm_kernel<BN, COOP, B_MN, OUT_F32, EPI, AUX32> (forward / dgrad: ping-pong, or cooperative for long K)
            # gemm_wgrad_kernel<BN, OUT_F32> (weight gradients: both operands MN-major, cooperative, no epilogue op)
            t = re.search(k + r"<([^>]*)>", name)
            a = [x.strip().replace("(bool)", "").replace("(int)", "") for x in t.group(1).split(",")] if t else []
            yes = lambda x: x in ("1", "true")
            if k == "gemm_kernel" and len(a) == 6:
                sched = "coop" if yes(a[1]) else "pingpong"
                epi = {"0": "none", "1": "gelu", "2": "add", "3": "dgelu", "4": "mul", "5": "gelu+grad"}.get(a[4], a[4])
                return (f"gemm {'K-MN' if yes(a[2]) else 'KK'} {sched} bn{a[0]} {epi}"
                        f"{' f32out' if yes(a[3]) else ''}{' aux32' if yes(a[5]) else ''}")
            if k == "gemm_wgrad_kernel" and len(a) == 2:
                return f"gemm MN-MN coop bn{a[0]} none{' f32out' if yes(a[1]) else ''}"
        t = re.search(r"vj::(\w+)<([^>]*)>", name)
        return f"{k}<{t.group(2)}>" if t else k
    if "nccl" in name.lower():
        return "nccl"
    return "torch: " + re.sub(r"<.*", "", name.replace("void ", ""))[:60]


def main():
    path = sys.argv[1]
    skip = int(sys.argv[sys.argv.index("--skip") + 1]) if "--skip" in sys.argv else 0
    steps = int(sys.argv[sys.argv.index("--steps") + 1]) if "--steps" in sys.argv else 1
    with open(path) as f:
        lines = [ln for ln in f if ln.startswith('"')]
    launches = {}   # ID -> [name, time_ns, dram_read_B, dram_write_B]
    unit_scale = {"byte": 1.0, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9, "ns": 1.0, "us": 1e3, "ms": 1e6}
    for r in csv.DictReader(lines):
        rec = launches.setdefault(int(r["ID"]), [r["Kernel Name"], 0.0, 0.0, 0.0])
        val = float(r["Metric Value"].replace(",", "")) * unit_scale.get(r["Metric Unit"], 1.0)
        if r["Metric Name"] == "gpu__time_duration.sum":
            rec[1] = val
        elif r["Metric Name"] == "dram__bytes_read.sum":
            rec[2] = val
        elif r["Metric Name"] == "dram__bytes_write.sum":
            rec[3] = val
    rows = [launches[k] for k in sorted(launches)][skip:]
    agg = defaultdict(lambda: [0, 0.0, 0.0, 0.0])
    for n, t, rd, wr in rows:
        a = agg[family(n)]
        a[0] += 1
        a[1] += t
        a[2] += rd
        a[3] += wr
    total = sum(v[1] for v in agg.values())
    have_dram = any(v[2] or v[3] for v in agg.values())
    print(f"# {path}: {len(rows)} launches, {total / 1e6 / steps:.2f} ms per step (sum of serialised kernel times, {steps} step(s))")
    print(f"{'family':58s} {'launches':>8s} {'ms/step':>9s} {'share':>7s} {'avg us':>8s}" + (f" {'dramR MB':>9s} {'dramW MB':>9s}" if have_dram else ""))
    for k, (c, t, rd, wr) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
        line = f"{k:58s} {c / steps:8.0f} {t / 1e6 / steps:9.3f} {100 * t / total:6.1f}% {t / c / 1e3:8.1f}"
        if have_dram:
            line += f" {rd / 1e6 / steps:9.1f} {wr / 1e6 / steps:9.1f}"
        print(line)
    if have_dram:
        g = [v for k, v in agg.items() if k.startswith("gemm ")]
        print(f"# gemm family: {sum(v[0] for v in g) / steps:.0f} launches, DRAM traffic "
              f"{sum(v[2] + v[3] for v in g) / 1e9 / steps:.2f} GB per step")


if __name__ == "__main__":
    main()
