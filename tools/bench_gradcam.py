#!/usr/bin/env python
"""Time the drop-in's Grad-CAM of ResNet2d (``b200.grad_cam``, bf16 storage) against a torch restatement on the same
device: the functional ResNet2d of ``oracle/gradcam.py`` (cuDNN, fp32) with autograd to the stage outputs, then the
reference's CAM steps (weights, weighted sum, clamp, min-max scale, bilinear resize, mean, scale) in torch ops.

Workloads: ResNet2d(1, 10) at 64x64 (the reference's size), batch 1 and batch 128 (a validation set in one call),
and batch 1 at 512x512; target ``down_tr256``, plus ``down_tr128 + down_tr256`` at 64x64 batch 128.
The card's name and power limit are printed with the numbers.

    python tools/bench_gradcam.py [--repeats 50] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import oracle  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from oracle import gradcam as og  # noqa: E402
from oracle import resnet as ores  # noqa: E402

WORKLOADS = [((64, 64), 1, ("down_tr256",)), ((64, 64), 128, ("down_tr256",)),
             ((64, 64), 128, ("down_tr128", "down_tr256")), ((512, 512), 1, ("down_tr256",))]


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


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


def torch_grad_cam(sd, x, layers):
    """the restatement: arg-max class of each row, hooks replaced by autograd to the stage outputs"""
    A, g, _ = og.stage_grads(sd, x, None, layers)
    H, W = x.shape[2:]

    def scale(m):
        m = m - m.amin(dim=(1, 2), keepdim=True)
        return m / (1e-7 + m.amax(dim=(1, 2), keepdim=True))

    acc = 0
    for a, d in zip(A, g):
        cam = scale((a * d.mean(dim=(2, 3), keepdim=True)).sum(1).clamp_min(0))
        if cam.shape[1:] != (H, W):
            cam = F.interpolate(cam[:, None], size=(H, W), mode="bilinear", align_corners=False)[:, 0]
        acc = acc + cam
    return scale(acc / len(A))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=50)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gradcam needs a CUDA device")
    name, limit = gpu_info()
    b200.set_precision("bf16")
    sd = oracle.init_state_dict(ores.resnet_state_spec(1, 10, dims=2), seed=0, randomize_affine=True)
    model = b200.ResNet2d(1, 10)
    model.load_state_dict(sd)
    model = model.cuda()
    sdc = {k: v.cuda() for k, v in sd.items()}
    rows = []
    for hw, n, layers in WORKLOADS:
        x = torch.randn((n, 1) + hw, generator=torch.Generator().manual_seed(0)).cuda()
        ours = gpu_ms(lambda: b200.grad_cam(model, x, None, layers), a.repeats)
        ref = gpu_ms(lambda: torch_grad_cam(sdc, x, layers), a.repeats)
        diff = float((b200.grad_cam(model, x, None, layers) - torch_grad_cam(sdc, x, layers)).abs().max())
        rows.append({"hw": list(hw), "batch": n, "layers": list(layers), "drop_in_ms": round(ours, 4),
                     "torch_fp32_ms": round(ref, 4), "speedup": round(ref / ours, 2), "max_abs_diff": diff})
        print(rows[-1], flush=True)
    line = json.dumps({"gpu": name, "power_limit": limit, "cases": rows})
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
