#!/usr/bin/env python
"""A/B of the host-side scheduling options (B200SEG_OVERLAP bit mask, engine.py) on ONE box and in ONE process.  For every setting a fresh GraphedStep is captured on the same
model / inputs / dropout draw; its loss and gradients are compared with the first setting (same kernels on the same
data: only atomic ordering may differ -- the list can repeat the baseline to show that noise floor) and the replay is
timed like bench.py times it (device events, 256 MiB L2 flush before every step, median).

  python tools/overlap_ab.py --masks 0,1,2,4,8,15,0 [--workload vnet3d|unet2d|unet3d] [--steps 30] \
         [--choose gpurun_out/chosen_env.sh] >> gpurun_out/overlap_ab.jsonl

``--choose FILE``: write ``export B200SEG_OVERLAP=..`` for the fastest setting whose
results agree with the baseline (bits are kept when they gain on their own; the union must beat the baseline).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200.graphed import GraphedStep  # noqa: E402
import oracle  # noqa: E402

GRAD_TOL = 2e-2        # relative L2 of the flat gradient against the baseline (bf16 kink noise is ~1e-3, see DESIGN 6)
MIN_GAIN_MS = 0.004    # a bit / grid setting is kept only for a median gain above the timing noise


def select(measure, masks):
    """measure(mask) -> record with "mask", "ms_median", "ok".  Returns (mask, summary or None)."""
    recs = [measure(m) for m in masks]
    base = [r for r in recs if r["mask"] == 0]
    if not base:
        return 0, None
    t0 = statistics.median([r["ms_median"] for r in base])
    keep = 0
    for bit in (1, 2, 4, 8):
        rs = [r for r in recs if r["mask"] == bit]
        if rs and all(r["ok"] for r in rs) and t0 - min(r["ms_median"] for r in rs) > MIN_GAIN_MS:
            keep |= bit
    cands = {}
    for r in recs:
        if r["mask"] and r["ok"]:
            cands[r["mask"]] = min(cands.get(r["mask"], 1e9), r["ms_median"])
    if keep and keep not in cands:
        r = measure(keep)
        if r["ok"]:
            cands[keep] = r["ms_median"]
    chosen_mask = 0
    if cands:
        best = min(cands, key=cands.get)
        if t0 - cands[best] > MIN_GAIN_MS:
            chosen_mask = best
    return chosen_mask, {"baseline_ms": t0, "chosen_mask": chosen_mask, "chosen_ms": cands.get(chosen_mask, t0)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--masks", default="0,15")
    ap.add_argument("--workload", default="vnet3d")
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--choose", default="")
    args = ap.parse_args()
    b200.set_precision("bf16")
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    if args.workload == "vnet3d":
        model, ncls, shape = b200.VNet3d(1, 2), 2, (2, 1, 96, 96, 96)
        lossfn = b200.MutilDiceLoss(torch.ones(2, device=dev))
    elif args.workload == "unet3d":
        model, ncls, shape = b200.UNet3d(1, 4), 4, (1, 1, 128, 128, 128)
        lossfn = b200.MutilCrossEntropyDiceLoss(torch.ones(4, device=dev))
    elif args.workload == "unet3dthin":
        model, ncls, shape = b200.UNet3dthin(1, 2), 2, (2, 1, 96, 96, 96)
        lossfn = b200.MutilDiceLoss(torch.ones(2, device=dev))
    elif args.workload == "unet3dthin128":
        model, ncls, shape = b200.UNet3dthin(1, 5), 5, (1, 1, 128, 112, 112)
        lossfn = b200.MutilCrossEntropyDiceLoss(torch.ones(5, device=dev))
    else:
        model, ncls, shape = b200.UNet2d(1, 1), 1, (8, 1, 512, 512)
        lossfn = b200.BinaryDiceFocalLoss()
    model.apply(b200.initialize_weights)
    model = model.to(dev).train()
    x, y = oracle.make_inputs(shape[0], shape[1], shape[2:], ncls)
    x, y = x.to(dev), y.to(dev)
    flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
    ref = [None]

    def measure(mask):
        os.environ["B200SEG_OVERLAP"] = str(mask)
        step = GraphedStep(model, lossfn, x, y, warmup=2)
        for _ in range(5):
            step()
        torch.cuda.manual_seed(1234)             # one replay on a fixed generator state: results to compare
        loss = float(step())
        torch.cuda.synchronize()
        flat = step._flat.detach().clone()
        evs = []
        for _ in range(args.steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            step()
            e1.record()
            evs.append((e0, e1))
        torch.cuda.synchronize()
        ms = [a.elapsed_time(b) for a, b in evs]
        rec = {"workload": args.workload, "mask": mask, "ms_median": statistics.median(ms),
               "ms_min": min(ms), "ms_max": max(ms), "loss": loss, "grad_norm": float(flat.norm()),
               "finite": bool(torch.isfinite(flat).all()), "graphs": len(step.graphs)}
        if ref[0] is None:
            ref[0] = (loss, flat)
            rec["ok"] = rec["finite"]
        else:
            rec["loss_diff_vs_first"] = abs(loss - ref[0][0])
            rec["grad_rel_l2_vs_first"] = float((flat - ref[0][1]).norm() / ref[0][1].norm())
            rec["ok"] = bool(rec["finite"] and rec["grad_rel_l2_vs_first"] < GRAD_TOL
                             and rec["loss_diff_vs_first"] < 1e-3 * max(1.0, abs(ref[0][0])))
        print(json.dumps(rec), flush=True)
        del step
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
        return rec

    chosen_mask, summary = select(measure, [int(m) for m in args.masks.split(",")])
    if summary is not None:
        summary["workload"] = args.workload
        print(json.dumps(summary), flush=True)
    if args.choose:
        with open(args.choose, "w") as f:
            f.write(f"export B200SEG_OVERLAP={chosen_mask}\n")


if __name__ == "__main__":
    main()
