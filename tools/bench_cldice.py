#!/usr/bin/env python
"""Time soft-clDice forward plus backward (reference model/lossescldice.py, repaired) on the GPU: the drop-in's fused
kernels against the torch fp32 restatement (oracle/cldice.py) on the same device.

    python tools/bench_cldice.py [--repeats 20] [--out result.json]

Shapes: 2x1x96^3 and 2x3x96^3 (3-D), 8x1x512^2 (2-D); one binary target per channel (the 3-class shape runs
Mutil_Soft_cldice_loss on integer labels).  Each number is the median of ``--repeats`` timed calls (CUDA events,
after warm-up), with the card's name and power limit printed beside it.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import pytorchdeeplearing_b200 as b200  # noqa: E402
from oracle import cldice as ocl  # noqa: E402

SHAPES = [("2x1x96^3", (2, 1, 96, 96, 96)), ("2x3x96^3", (2, 3, 96, 96, 96)), ("8x1x512^2", (8, 1, 512, 512))]


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
    out.sort()
    return out[len(out) // 2]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_cldice needs a CUDA device")
    g = torch.Generator(device="cuda").manual_seed(0)
    rows = []
    for label, shape in SHAPES:
        n, c = shape[:2]
        pred = torch.rand(shape, generator=g, device="cuda")
        if c == 1:
            target = (torch.rand(shape, generator=g, device="cuda") > 0.6).float()
            ours_fn, ref_fn = b200.Binary_Soft_cldice_loss(), lambda p, t: ocl.binary_loss(p, t)
        else:
            target = torch.randint(0, c, (n,) + shape[2:], generator=g, device="cuda")
            alpha = [1.0] * c
            ours_fn = b200.Mutil_Soft_cldice_loss(alpha)
            a = torch.ones(c, device="cuda")
            ref_fn = lambda p, t: ocl.mutil_loss(p, t, a)  # noqa: E731

        def step(fn):
            p = pred.clone().requires_grad_(True)
            fn(p, target).backward()
            return p.grad

        gpu_ms = time_ms(lambda: step(ours_fn), args.repeats)
        ref_ms = time_ms(lambda: step(ref_fn), max(3, args.repeats // 4))
        err = ((step(ours_fn) - step(ref_fn)).norm() / step(ref_fn).norm()).item()
        vox = pred.numel()
        rows.append({"shape": label, "gpu_ms": gpu_ms, "ref_ms": ref_ms, "voxels": vox, "grad_rel_diff": err})
        print(f"{label:>10}: clDice fwd+bwd {gpu_ms:8.3f} ms, torch restatement {ref_ms:8.3f} ms "
              f"(x{ref_ms / gpu_ms:.1f}), grad rel diff {err:.2e}")
    info = {"card": card(), "rows": rows}
    print(json.dumps(info))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(info, f, indent=1)


if __name__ == "__main__":
    main()
