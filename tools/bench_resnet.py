"""Training-step throughput of the ResNet2d / ResNet3d classifiers (one GPU, bf16 perf mode, train mode with dropout):
one GraphedStep (Philox masks, forward, loss, backward, FusedAdamW) per step.

    python tools/bench_resnet.py [--iters 20] [--warmup 5] [--rounds 3] [--out results.json]

Workloads:
  resnet2d  ResNet2d(1, 10), 64x64, batch 128, MutilCrossEntropyLoss  (the reference's example.py:204-216 configuration)
  resnet3d  ResNet3d(1, 4), 96^3, batch 2, MutilCrossEntropyLoss
  vnet3d    VNet3d(1, 2), 96^3, batch 2, MutilDiceLoss: the same encoder plus a decoder, timed in the same call; the
            ResNet3d step runs a strict subset of its convolutions and must be faster
Per workload: the median step time of --iters CUDA-event intervals (the workloads alternate for --rounds rounds; the
median over rounds is reported), images per second, the classifier-head kernels' share of device kernel time (from
torch.profiler over eager steps, in a separate pass) and the convolution kernel family (b200seg_conv_path) of every
forward convolution.  The card's name and power limit are printed with the numbers.  Development tool, not a bench
line.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import oracle  # noqa: E402
from oracle import nets as onets  # noqa: E402
from oracle import resnet as ores  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200 import runtime  # noqa: E402
from pytorchdeeplearing_b200.graphed import GraphedStep  # noqa: E402


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def workload(kind):
    """(model, lossfn, x, y) on the device, seeded weights"""
    if kind == "resnet2d":
        k, n, sp, model = 10, 128, (64, 64), b200.ResNet2d(1, 10)
        spec = ores.resnet_state_spec(1, k, 2)
    elif kind == "resnet3d":
        k, n, sp, model = 4, 2, (96, 96, 96), b200.ResNet3d(1, 4)
        spec = ores.resnet_state_spec(1, k, 3)
    else:
        k, n, sp, model = 2, 2, (96, 96, 96), b200.VNet3d(1, 2)
        spec = onets.vnet3d_state_spec(1, 2)
    model.load_state_dict(oracle.init_state_dict(spec, seed=0, randomize_affine=True), strict=True)
    model = model.cuda().train()
    g = torch.Generator().manual_seed(1)
    x = torch.randn((n, 1) + sp, generator=g)
    if kind == "vnet3d":
        y = (torch.rand((n,) + sp, generator=g) > 0.7).long()
        lossfn = b200.MutilDiceLoss(torch.ones(k).cuda())
    else:
        y = torch.randint(0, k, (n,), generator=g)
        lossfn = b200.MutilCrossEntropyLoss(torch.ones(k).cuda())
    return model, lossfn, x.cuda(), y.cuda()


def median_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(iters):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    times.sort()
    return times[len(times) // 2]


class _PathRecorder:
    """the product backend, recording the kernel family of every forward convolution of one pass"""

    def __init__(self, be):
        self._be, self.tag, self.rows = be, "other", []

    def __getattr__(self, name):
        return getattr(self._be, name)

    def conv(self, kind, dims, x, wpk, bias, y, stats, addend):
        if stats is not None:                           # forward convolutions (data gradients carry no statistics)
            self.rows.append({"block": self.tag, "kind": ["3x3", "1x1", "down", "up"][kind],
                              "in": list(x.shape[1:]), "cout": int(y.shape[-1]),
                              "path": self._be.conv_path(kind, dims, x, wpk, y, addend)})
        return self._be.conv(kind, dims, x, wpk, bias, y, stats, addend)


def conv_paths(model, x):
    rec = _PathRecorder(runtime.cuda_backend())
    runtime._set_backend_for_testing(rec)
    try:
        model.eval()
        with torch.no_grad():
            model(x)
    finally:
        runtime._set_backend_for_testing(None)
        model.train()
    torch.cuda.synchronize()
    return rec.rows


def head_share(model, lossfn, x, y, steps=5):
    """share of device kernel time spent in the classifier-head kernels (cls_*), eager GraphedStep phases"""
    from torch.profiler import ProfilerActivity, profile
    step = GraphedStep(model, lossfn, x, y, warmup=2, use_graph=False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            step()
        torch.cuda.synchronize()
    head = total = 0.0
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", None)
        if t is None:
            t = getattr(e, "self_cuda_time_total", 0.0)
        if t <= 0:
            continue
        total += t
        if "cls_" in e.key:
            head += t
    return head / total if total > 0 else float("nan"), head / steps / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_resnet needs a CUDA device")
    b200.set_precision("bf16")
    name, limit = gpu_info()
    print(f"device: {name}, power limit {limit}", flush=True)
    kinds = ("resnet2d", "resnet3d", "vnet3d")
    loads = {k: workload(k) for k in kinds}
    steps = {}
    for k, (model, lossfn, x, y) in loads.items():
        steps[k] = GraphedStep(model, lossfn, x, y, warmup=2,
                               optimizer=b200.FusedAdamW(model.parameters(), lr=1e-4))
    times = {k: [] for k in kinds}
    for _ in range(a.rounds):
        for k in kinds:
            times[k].append(median_ms(lambda: steps[k](), a.iters, a.warmup))
    res = {"device": name, "power_limit": limit, "precision": "bf16", "workloads": {}}
    for k in kinds:
        model, lossfn, x, y = loads[k]
        t = sorted(times[k])[len(times[k]) // 2]
        row = {"batch": int(x.shape[0]), "shape": list(x.shape[2:]), "step_ms": round(t, 4),
               "step_ms_rounds": [round(v, 4) for v in times[k]],
               "images_per_s": round(x.shape[0] / t * 1e3, 1)}
        if k != "vnet3d":
            share, head_ms = head_share(model, lossfn, x, y)
            row["head_share"] = round(share, 5)
            row["head_ms_per_step_profiled"] = round(head_ms, 4)
            row["conv_paths"] = conv_paths(model, x)
        res["workloads"][k] = row
        print(f"{k:9s} B={row['batch']:4d} {str(row['shape']):16s} step {t:8.3f} ms  {row['images_per_s']:10.1f} img/s"
              + (f"  head {100 * row['head_share']:.2f} % of kernel time" if "head_share" in row else ""), flush=True)
    r3, v3 = res["workloads"]["resnet3d"]["step_ms"], res["workloads"]["vnet3d"]["step_ms"]
    print(f"ResNet3d / VNet3d step time at 96^3 B=2: {r3 / v3:.3f}", flush=True)
    for k in ("resnet2d", "resnet3d"):
        for p in res["workloads"][k]["conv_paths"]:
            print(f"  {k:9s} {p['block']:11s} {p['kind']:5s} in {str(p['in']):22s} -> {p['cout']:4d}  {p['path']}")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
