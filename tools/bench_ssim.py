#!/usr/bin/env python
"""Time SSIM / SSIM3D forward plus backward (reference model/lossesSSIM.py) on the GPU: the drop-in's separable kernels
against the reference's operator sequence (five dense depthwise convolutions, autograd backward) on the same device.

    python tools/bench_ssim.py [--repeats 20] [--out result.json]

Cases: 2x1x96^3, 1x1x128x112x112 (the reference's training shape, train.py:34) and 8x1x512^2 (2-D), window 11, mean
form, both inputs requiring gradients.  Each figure is the median of ``--repeats`` forward+backward calls after a
warm-up, timed with CUDA events:
  gpu_ms    pytorchdeeplearing_b200.ssim3D / ssim
  ref_ms    the oracle's fp32 operator sequence (oracle/ssim.py) with torch's default convolution settings
  bytes     the algorithmic DRAM traffic of the kernels, from the shapes: forward reads x, y (8 B per voxel) and writes
            four fp64 coefficients (32 B); backward reads the coefficients and x, y (40 B) and writes two fp32
            gradients (8 B): 88 B per voxel
  gbps      bytes / gpu_ms (an achieved rate, not a peak)
The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pytorchdeeplearing_b200 as b200  # noqa: E402
from oracle import ssim as oss  # noqa: E402

CASES = [("2x1x96^3", (2, 1, 96, 96, 96)), ("1x1x128x112x112", (1, 1, 128, 112, 112)), ("8x1x512^2", (8, 1, 512, 512))]
BYTES_PER_VOXEL = 88


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def time_ms(fn, repeats):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        out.append(a.elapsed_time(b))
    return statistics.median(out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_ssim needs a CUDA device")
    name, limit = gpu_info()
    rows = []
    for label, shape in CASES:
        g = torch.Generator(device="cuda").manual_seed(0)
        x0 = torch.rand(shape, generator=g, device="cuda")
        y0 = (0.7 * x0 + 0.3 * torch.rand(shape, generator=g, device="cuda")).clamp(0, 1)
        x, y = x0.clone().requires_grad_(True), y0.clone().requires_grad_(True)
        dims = len(shape) - 2
        ours = b200.ssim3D if dims == 3 else b200.ssim

        def step(f):
            x.grad = y.grad = None
            v = f(x, y)
            v.backward()
            return v

        gpu_ms = time_ms(lambda: step(ours), args.repeats)
        ref_ms = time_ms(lambda: step(lambda a, b: oss.ssim(a, b, 11, True, dims)), max(3, args.repeats // 4))
        v = step(ours).item()
        gx = x.grad.clone()
        r = step(lambda a, b: oss.ssim(a, b, 11, True, dims)).item()
        grad_rel = ((gx - x.grad).norm() / x.grad.norm()).item()
        nbytes = BYTES_PER_VOXEL * x.numel()
        rows.append({"case": label, "gpu_ms": round(gpu_ms, 4), "ref_ms": round(ref_ms, 3),
                     "speedup": round(ref_ms / gpu_ms, 1), "bytes": nbytes,
                     "gbps": round(nbytes / gpu_ms / 1e6, 1), "value": v, "ref_value": r,
                     "grad_rel_diff": grad_rel})
        print(f"{label:>18}: ssim fwd+bwd {gpu_ms:8.3f} ms ({nbytes / gpu_ms / 1e6:7.1f} GB/s algorithmic), "
              f"reference sequence {ref_ms:9.3f} ms ({ref_ms / gpu_ms:6.1f}x); value {v:.7f} vs {r:.7f}, "
              f"grad rel diff {grad_rel:.2e}")
    res = {"card": name, "power_limit": limit, "cases": rows}
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
