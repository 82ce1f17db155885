#!/usr/bin/env python
"""Condense an .ncu-rep (ncu --set full) into the handful of numbers the design discussion uses.
usage: python tools/ncu_summary.py report.ncu-rep > profiles/<name>.txt   (needs `ncu` on PATH; runs on CPU)"""
import csv
import io
import subprocess
import sys

KEYS = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_registers", "launch__occupancy_limit_shared_mem", "sm__warps_active.avg.per_cycle_active",
    "sm__issue_active.avg.pct_of_peak_sustained_elapsed", "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_xu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_fma.avg.pct_of_peak_sustained_active",
    "sm__inst_executed_pipe_alu.avg.pct_of_peak_sustained_active", "sm__inst_executed_pipe_lsu.avg.pct_of_peak_sustained_active",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "dram__throughput.avg.pct_of_peak_sustained_elapsed",
    "lts__throughput.avg.pct_of_peak_sustained_elapsed", "l1tex__data_bank_conflicts_pipe_lsu_mem_shared.sum",
    "smsp__average_warps_issue_stalled_long_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_short_scoreboard_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_wait_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_barrier_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_math_pipe_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_mio_throttle_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_branch_resolving_per_issue_active.ratio",
    "smsp__average_warps_issue_stalled_not_selected_per_issue_active.ratio",
]


def main():
    rep = sys.argv[1]
    raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(raw)))
    hdr, units = rows[0], rows[1]
    for r in rows[2:]:
        d = dict(zip(hdr, r))
        u = dict(zip(hdr, units))
        print(f"== {d.get('Kernel Name', '?')}  (from {rep.split('/')[-1]})")
        for k in KEYS:
            if k in d and d[k] != "":
                print(f"  {k:90s} {d[k]:>14s} {u.get(k, '')}")
    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    lines = [ln for ln in src.splitlines() if ln.startswith('"')]
    rows = list(csv.reader(io.StringIO("\n".join(lines))))
    try:
        h = next(i for i, r in enumerate(rows) if "Source" in r and "Address" in r)
    except StopIteration:
        return
    hdr = rows[h]
    isrc, isamp, iex = hdr.index("Source"), hdr.index("Warp Stall Sampling (All Samples)"), hdr.index("Instructions Executed")
    data = rows[h + 1:]
    tot = sum(int(r[isamp] or 0) for r in data)
    mnem = {}
    for r in data:
        m = r[isrc].split()[0] if r[isrc].split() else "?"
        if m.startswith("@"):
            m = r[isrc].split()[1]
        m = m.split(".")[0] + ("." + r[isrc].split(".")[1].split()[0] if m in ("UTCHMMA", "UTMALDG", "UTMASTG", "LDTM", "STTM", "MUFU") and "." in r[isrc] else "")
        mnem[m] = mnem.get(m, 0) + int(r[iex] or 0)
    print(f"  SASS: {len(data)} instructions, {tot} stall samples; top sampled instructions:")
    for r in sorted(data, key=lambda r: -int(r[isamp] or 0))[:12]:
        print(f"    {int(r[isamp] or 0):6d} ({100 * int(r[isamp] or 0) / max(tot, 1):4.1f}%)  {r[isrc][:90]}")
    proof = {k: v for k, v in mnem.items() if k.split(".")[0] in ("UTCHMMA", "UTCQMMA", "UTMALDG", "UTMASTG", "UTMAREDG", "LDTM", "STTM", "UTCBAR", "SYNCS", "MUFU", "FFMA2", "FMUL2", "FADD2", "HMUL2")}
    print("  executed warp-instructions of the architecture-specific kinds:", ", ".join(f"{k}={v}" for k, v in sorted(proof.items())))


if __name__ == "__main__":
    main()
