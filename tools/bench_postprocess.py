#!/usr/bin/env python
"""Time the mask post-processing of the reference's dataprocess/utils.py:7-66 (largest connected component, ball
morphology) on the GPU against the scipy restatement on this host's CPU.

    python tools/bench_postprocess.py [--repeats 20] [--cpu-repeats 2] [--out result.json]

Cases: a 96^3 mask and a 300x512x512 CT-sized one, both an ellipsoid with noise islands.  Per case and per operation
(components; open, close, dilate, erode at r in {1, 3, 8}), each the median of repeated calls after a warm-up:
  gpu_ms      the device form (largest_component / binary_morphology) on a device-resident uint8 mask, CUDA events
  wrapper_ms  the reference-named function from a numpy mask to a numpy result (copies and the launches)
  cpu_ms      the scipy restatement (oracle/postprocess.py: ndimage.label + bincount, binary_dilation / erosion with
              the ball) on this machine's CPU, also the check of the GPU result (matches_cpu).  scipy loops over every
              ball offset per voxel, so on the CT-sized case only components and r = 1 are run on the CPU (null
              otherwise).  SimpleITK is not installed here, so ITK's own CPU time is not measured.
The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorchdeeplearing_b200 as b200  # noqa: E402
from oracle import postprocess as opp  # noqa: E402

RADII = (1, 3, 8)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def make_mask(shape, seed=0):
    z, y, x = np.ogrid[tuple(slice(0, s) for s in shape)]
    c = [s / 2 for s in shape]
    m = (((z - c[0]) / (0.36 * shape[0])) ** 2 + ((y - c[1]) / (0.37 * shape[1])) ** 2 +
         ((x - c[2]) / (0.33 * shape[2])) ** 2) <= 1
    m |= np.random.default_rng(seed).random(shape) < 2e-4
    return m.astype(np.uint8)


def gpu_ms(fn, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return statistics.median(times)


def host_ms(fn, repeats):
    times = []
    for _ in range(repeats):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(times)


def bench_case(shape, repeats, cpu_repeats, cpu_radii):
    m = make_mask(shape)
    t = torch.from_numpy(m).cuda()
    wrep = max(3, repeats // 4)
    rows = []
    agree = np.array_equal(b200.largest_component(t)[0].cpu().numpy(), opp.largest_component(m)[0])
    rows.append({"op": "components", "gpu_ms": round(gpu_ms(lambda: b200.largest_component(t), repeats), 4),
                 "wrapper_ms": round(host_ms(lambda: b200.GetLargestConnectedCompont(m), wrep), 3),
                 "cpu_ms": round(host_ms(lambda: opp.largest_component(m), cpu_repeats), 1), "matches_cpu": agree})
    for op in opp.OPS:
        for r in RADII:
            row = {"op": op, "radius": r,
                   "gpu_ms": round(gpu_ms(lambda: b200.binary_morphology(t, r, op), repeats), 4),
                   "wrapper_ms": round(host_ms(lambda: b200.MorphologicalOperation(m, r, op), wrep), 3),
                   "cpu_ms": None, "matches_cpu": None}
            if r in cpu_radii:
                row["matches_cpu"] = np.array_equal(b200.binary_morphology(t, r, op).cpu().numpy(),
                                                    opp.morphology(m, r, op))
                row["cpu_ms"] = round(host_ms(lambda: opp.morphology(m, r, op), cpu_repeats), 1)
            rows.append(row)
    for row in rows:
        row["speedup_gpu_vs_cpu"] = None if row["cpu_ms"] is None else round(row["cpu_ms"] / row["gpu_ms"], 1)
    return {"shape": list(shape), "foreground": int(m.sum()), "rows": rows}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--cpu-repeats", type=int, default=2)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_postprocess needs a CUDA device")
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit, "cpu_threads": os.cpu_count(),
           "cases": [bench_case((96, 96, 96), a.repeats, a.cpu_repeats, RADII),
                     bench_case((300, 512, 512), a.repeats, a.cpu_repeats, (1,))]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
