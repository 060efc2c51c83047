#!/usr/bin/env python
"""Digest of an `ncu --set full` report: one line per profiled launch with the numbers BASELINE.json's
north_star asks for (achieved HBM GB/s, tensor-pipe %, DRAM bytes) next to the duration.

    python tools/ncu_digest.py report.ncu-rep > ncu_ops.txt

Columns: dur_us = gpu__time_duration; dramR/dramW MB = dram__bytes_{read,write}.sum (a kernel's dirty output lines can
still sit in L2 when it ends, so dramW undercounts writes); L2W MB = lts__t_sectors_srcunit_tex_op_write.sum * 32 B (what the kernel
wrote into L2 = what must reach HBM eventually); dram% = gpu__dram_throughput % of peak; tensor% =
sm__pipe_tensor_cycles_active % of peak (while active); warps% = sm__warps_active %; regs; grid."""
import csv
import subprocess
import sys

rep = sys.argv[1]
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], stdout=subprocess.PIPE, text=True).stdout
rows = list(csv.reader(raw.splitlines()))
hdr, units = rows[0], rows[1]


def col(name):
    for i, h in enumerate(hdr):
        if h == name:
            return i
    return None


def val(r, name, scale=None):
    i = col(name)
    if i is None or r[i] in ("", "n/a"):
        return None
    v = float(r[i].replace(",", ""))
    u = units[i]
    if scale == "bytes":
        v *= {"byte": 1, "Kbyte": 1e3, "Mbyte": 1e6, "Gbyte": 1e9}.get(u, 1)
    if scale == "us":
        v *= {"ns": 1e-3, "us": 1, "ms": 1e3, "s": 1e6}.get(u, 1)
    return v


print(f"# {rep}")
print(f"{'kernel':58s} {'grid':>6s} {'regs':>4s} {'dur_us':>8s} {'dramR_MB':>9s} {'dramW_MB':>9s} {'L2W_MB':>8s} "
      f"{'dram%':>6s} {'tensor%':>7s} {'warps%':>6s} {'GB/s(R+L2W)':>11s}")
ik, ig = col("Kernel Name"), col("launch__grid_size")
for r in rows[2:]:
    name = r[ik].replace("b200seg::", "").replace("void ", "").replace("(int)", "").replace("__nv_bfloat16", "bf16")
    name = name.split("(")[0][:58]
    dur = val(r, "gpu__time_duration.sum", "us")
    rd = val(r, "dram__bytes_read.sum", "bytes") or 0.0
    wr = val(r, "dram__bytes_write.sum", "bytes") or 0.0
    l2w = (val(r, "lts__t_sectors_srcunit_tex_op_write.sum") or 0.0) * 32
    dp = val(r, "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed")
    tp = val(r, "sm__pipe_tensor_cycles_active.avg.pct_of_peak_sustained_active")
    wa = val(r, "sm__warps_active.avg.pct_of_peak_sustained_active")
    regs = val(r, "launch__registers_per_thread")
    gbs = (rd + max(wr, l2w)) / dur / 1e3 if dur else 0.0
    print(f"{name:58s} {r[ig]:>6s} {int(regs or 0):4d} {dur:8.1f} {rd / 1e6:9.2f} {wr / 1e6:9.2f} {l2w / 1e6:8.2f} "
          f"{(dp or 0):6.1f} {(tp or 0):7.1f} {(wa or 0):6.1f} {gbs:11.1f}")
