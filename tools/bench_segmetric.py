#!/usr/bin/env python
"""Time the 3-D segmentation metrics (Seg_Metirc3d, reference model/metric.py:11-142) on the GPU against the
reference's CPU method on the same host.

    python tools/bench_segmetric.py [--repeats 20] [--cpu-repeats 3] [--out result.json]

Cases: a batch-of-one 96^3 volume and the 88x410x512 CT shape the reference's own comment names (metric.py:45), both
two overlapping ellipsoids with spacing (0.78, 0.78, 2.5).  Reported per case, each the median of repeated calls
after a warm-up:
  gpu_ms      seg_metrics3d on device-resident uint8 masks, timed with CUDA events (the nine metrics, no host read)
  class_ms    Seg_Metirc3d from numpy masks: the host-to-device copy, the launches and the one host read
  cpu_ms      the reference's method restated below (scipy binary_erosion with the 18-structure, a cKDTree per
              surface and two nearest-neighbour queries, numpy sums), on this machine's CPU
The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from scipy import ndimage, spatial

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import pytorchdeeplearing_b200 as b200  # noqa: E402


def ellipsoid(shape, centre, radii):
    z, y, x = np.ogrid[tuple(slice(0, s) for s in shape)]
    return (((z - centre[0]) / radii[0]) ** 2 + ((y - centre[1]) / radii[1]) ** 2 +
            ((x - centre[2]) / radii[2]) ** 2) <= 1.0


def reference_method(real, pred, spacing):
    """the reference's CPU computation: erosion-XOR surfaces, cKDTree distances, numpy overlap sums"""
    k = ndimage.generate_binary_structure(3, 2)
    sc = np.array(spacing[::-1]).reshape(1, 3)
    pts = [np.argwhere(ndimage.binary_erosion(m, k) ^ m) * sc for m in (real, pred)]
    r2p, _ = spatial.cKDTree(pts[1]).query(pts[0])
    p2r, _ = spatial.cKDTree(pts[0]).query(pts[1])
    i, u = (real & pred).sum(), (real | pred).sum()
    s = len(pts[0]) + len(pts[1])
    return (2 * i / (real.sum() + pred.sum()), i / u, (p2r.sum() + r2p.sum()) / s,
            math.sqrt(((p2r ** 2).sum() + (r2p ** 2).sum()) / s), max(p2r.max(), r2p.max()))


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def bench_case(shape, repeats, cpu_repeats):
    sh = tuple(shape)
    c = tuple(s / 2 for s in sh)
    r = ellipsoid(sh, c, (0.35 * sh[0], 0.36 * sh[1], 0.37 * sh[2]))
    p = ellipsoid(sh, (c[0] + 0.04 * sh[0], c[1] + 0.03 * sh[1], c[2] + 0.02 * sh[2]),
                  (0.32 * sh[0], 0.34 * sh[1], 0.38 * sh[2]))
    sp = (0.78, 0.78, 2.5)
    rt = torch.from_numpy(r.view(np.uint8)).cuda()
    pt = torch.from_numpy(p.view(np.uint8)).cuda()
    for _ in range(3):
        b200.seg_metrics3d(rt, pt, sp)
    torch.cuda.synchronize()
    times = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        m, _ = b200.seg_metrics3d(rt, pt, sp)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    gpu_ms = statistics.median(times)
    ctimes = []
    for _ in range(max(3, repeats // 4)):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        b200.Seg_Metirc3d(r, p, sp)
        ctimes.append((time.perf_counter() - t0) * 1e3)
    cpu = []
    ref = None
    for _ in range(cpu_repeats):
        t0 = time.perf_counter()
        ref = reference_method(r, p, sp)
        cpu.append((time.perf_counter() - t0) * 1e3)
    mh = m.cpu().numpy()
    agree = max(abs(mh[k] - v) / max(abs(v), 1e-300) for k, v in zip((0, 1, 6, 7, 8), ref))
    return {"shape": list(sh), "surface_points": [int(v) for v in b200.seg_metrics3d(rt, pt, sp)[1][4:].tolist()],
            "gpu_ms": round(gpu_ms, 4), "class_ms": round(statistics.median(ctimes), 3),
            "cpu_ms": round(statistics.median(cpu), 1), "speedup_gpu_vs_cpu": round(statistics.median(cpu) / gpu_ms, 1),
            "max_rel_diff_vs_cpu_method": float(agree)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--cpu-repeats", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_segmetric needs a CUDA device")
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit, "cpu_threads": os.cpu_count(),
           "cases": [bench_case(s, a.repeats, a.cpu_repeats) for s in ((96, 96, 96), (88, 410, 512))]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
