"""Forward + backward time of the binary Lovasz hinge (BinaryLovaszLoss, one GPU) at 2x1x96^3, against the reference's
torch computation of the same loss on the same logits, and one VNet3d(1, 1) 96^3 batch-2 GraphedStep with
BinaryLovaszLoss against one with BinaryDiceLoss.

    python tools/bench_lovasz_hinge.py [--iters 20] [--warmup 5] [--out results.json]

The reference side is the fp32 restatement in oracle/lovasz_hinge.py: the same torch operators model/lovasz.py calls
(sort, index, cumsum, relu, dot), run eagerly by the installed PyTorch on the same device.  Every time is the median of
--iters CUDA-event intervals after --warmup calls.  Development tool: prints a table and one JSON line; not a bench line.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)

import oracle  # noqa: E402
from oracle import lovasz_hinge as oh  # noqa: E402
from oracle import nets as onets  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200.graphed import GraphedStep  # noqa: E402
from bench_losses import card, fwd_bwd, median_ms  # noqa: E402


def loss_rows(iters, warmup):
    g = torch.Generator(device="cuda").manual_seed(0)
    z = 2.0 * torch.randn((2, 1, 96, 96, 96), device="cuda", generator=g)
    t = (torch.rand((2, 96, 96, 96), device="cuda", generator=g) > 0.7).long()
    rows = []
    for kw in ({}, {"per_image": True}):
        a = median_ms(fwd_bwd(b200.BinaryLovaszLoss(**kw), z, t), iters, warmup)
        b = median_ms(fwd_bwd(lambda zz, tt: oh.lovasz_hinge(zz, tt, **kw), z, t), iters, warmup)
        name = "BinaryLovaszLoss" + ("(per_image=True)" if kw else "")
        rows.append({"loss": name, "shape": "2x1x96x96x96", "ours_ms": round(a, 4), "reference_ms": round(b, 4),
                     "speedup": round(b / a, 2)})
        print(f"{name:32s} 2x1x96^3   ours {a:8.3f} ms   reference ops {b:8.3f} ms   x{b / a:6.1f}", flush=True)
    return rows


def step_ms(lossfn, iters, warmup):
    b200.set_precision("bf16")
    spec = onets.vnet3d_state_spec(1, 1)
    model = b200.VNet3d(1, 1)
    model.load_state_dict(onets.init_state_dict(spec, seed=0, randomize_affine=True), strict=True)
    model = model.cuda().train()
    x, y = oracle.make_inputs(2, 1, (96, 96, 96), 1, seed=1)
    step = GraphedStep(model, lossfn, x.cuda(), y.cuda(), warmup=2,
                       optimizer=b200.FusedAdamW(model.parameters(), lr=1e-4))
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
    s_dice = step_ms(b200.BinaryDiceLoss(), a.iters, a.warmup)
    s_hinge = step_ms(b200.BinaryLovaszLoss(), a.iters, a.warmup)
    print(f"VNet3d(1, 1) 96^3 B=2 GraphedStep: BinaryDiceLoss {s_dice:.3f} ms, BinaryLovaszLoss {s_hinge:.3f} ms "
          f"(+{s_hinge - s_dice:.3f} ms)", flush=True)
    res = {"device": name, "power_limit": power, "losses": rows,
           "vnet3d96_c1_step_ms": {"BinaryDiceLoss": round(s_dice, 4), "BinaryLovaszLoss": round(s_hinge, 4)}}
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
