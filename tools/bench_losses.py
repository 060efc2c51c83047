"""Forward + backward time of the Jaccard / ELDice / Tversky / SS / MutilELDice / Lovasz losses (one GPU), against the
reference's torch computation of the same loss on the same logits, and one VNet3d 96^3 batch-2 GraphedStep with
LovaszLoss against one with MutilDiceLoss.

    python tools/bench_losses.py [--iters 20] [--warmup 5] [--out results.json]

The reference side is the fp32 restatement in oracle/losses_ext.py: the same torch operators the reference's
model/losses.py and model/lovasz.py call (sigmoid / softmax, sums, sort, cumsum, dot), run eagerly by the installed
PyTorch on the same device.  Every time is the median of --iters CUDA-event intervals after --warmup calls.
Development tool: prints a table and one JSON line; not a bench line.
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
from oracle import losses_ext as ox  # noqa: E402
from oracle import nets as onets  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200.graphed import GraphedStep  # noqa: E402


def card():
    name = torch.cuda.get_device_name()
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader",
                            f"--id={torch.cuda.current_device()}"], capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


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


def fwd_bwd(loss_fn, z0, t):
    z = z0.clone().requires_grad_(True)

    def run():
        z.grad = None
        loss_fn(z, t).backward()
    return run


def loss_rows(iters, warmup):
    rows = []
    for n, c, sp in ((2, 2, (96, 96, 96)), (1, 5, (128, 112, 112))):
        g = torch.Generator(device="cuda").manual_seed(0)
        zc = torch.randn((n, c) + sp, device="cuda", generator=g)
        zc = zc.permute(0, 2, 3, 4, 1).contiguous().permute(0, 4, 1, 2, 3)      # channels-last, as the networks emit
        tc = torch.randint(0, c, (n,) + sp, device="cuda", generator=g)
        z1 = torch.randn((n, 1) + sp, device="cuda", generator=g)
        t1 = (torch.rand((n,) + sp, device="cuda", generator=g) > 0.7).long()
        alpha = torch.ones(c, device="cuda")
        cases = [
            ("BinaryJaccardLoss", b200.BinaryJaccardLoss(), ox.binary_jaccard, z1, t1),
            ("BinaryELDiceLoss", b200.BinaryELDiceLoss(), ox.binary_eldice, z1, t1),
            ("BinaryTverskyLoss", b200.BinaryTverskyLoss(), ox.binary_tversky, z1, t1),
            ("BinarySSLoss", b200.BinarySSLoss(), ox.binary_ss, z1, t1),
            ("MutilELDiceLoss", b200.MutilELDiceLoss(alpha), lambda z, t: ox.multi_eldice(z, t, alpha), zc, tc),
            ("LovaszLoss", b200.LovaszLoss(), ox.lovasz_softmax, zc, tc),
        ]
        for name, ours, ref, z, t in cases:
            shape = "x".join(str(s) for s in z.shape)
            a = median_ms(fwd_bwd(ours, z, t), iters, warmup)
            b = median_ms(fwd_bwd(ref, z, t), iters, warmup)
            rows.append({"loss": name, "shape": shape, "ours_ms": round(a, 4), "reference_ms": round(b, 4),
                         "speedup": round(b / a, 2)})
            print(f"{name:20s} {shape:18s} ours {a:8.3f} ms   reference ops {b:8.3f} ms   x{b / a:6.1f}", flush=True)
    return rows


def step_ms(lossfn, iters, warmup):
    b200.set_precision("bf16")
    spec = onets.vnet3d_state_spec(1, 2)
    model = b200.VNet3d(1, 2)
    model.load_state_dict(onets.init_state_dict(spec, seed=0, randomize_affine=True), strict=True)
    model = model.cuda().train()
    x, y = oracle.make_inputs(2, 1, (96, 96, 96), 2, seed=1)
    xc, yc = x.cuda(), y.cuda()
    step = GraphedStep(model, lossfn, xc, yc, warmup=2, optimizer=b200.FusedAdamW(model.parameters(), lr=1e-4))
    return median_ms(lambda: step(), iters, warmup)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    name, power = card()
    print(f"device: {name}, power limit {power}", flush=True)
    rows = loss_rows(a.iters, a.warmup)
    s_dice = step_ms(b200.MutilDiceLoss(torch.ones(2).cuda()), a.iters, a.warmup)
    s_lov = step_ms(b200.LovaszLoss(), a.iters, a.warmup)
    print(f"VNet3d 96^3 B=2 GraphedStep: MutilDiceLoss {s_dice:.3f} ms, LovaszLoss {s_lov:.3f} ms "
          f"(+{s_lov - s_dice:.3f} ms)", flush=True)
    res = {"device": name, "power_limit": power, "losses": rows,
           "vnet3d96_step_ms": {"MutilDiceLoss": round(s_dice, 4), "LovaszLoss": round(s_lov, 4)}}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
