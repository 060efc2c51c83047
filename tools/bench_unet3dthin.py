#!/usr/bin/env python
"""UNet3dthin on the GPU: training-step time against UNet3d and against the reference's operator sequence, and the
per-launch time of the two upsample kernels.

    python tools/bench_unet3dthin.py [--steps 20] [--rounds 3]

Prints the card name and power limit, then one JSON line per measurement:
  * ``step``: GraphedStep (bf16, MutilDiceLoss, FusedAdamW, train mode) ms per step of UNet3dthin and UNet3d, measured
    alternately (``rounds`` windows of ``steps`` steps each, median of the windows) at 2x96^3 and 1x128x112x112;
  * ``oracle_step``: the same step as the reference runs it (oracle.unetthin in fp32 with torch autograd and
    torch.optim.AdamW, cuDNN without TF32) on the same GPU;
  * ``kernel``: us per launch of b200seg_upsample2_add / b200seg_upsample2_bwd at the four joins of 2x96^3 and
    1x128x112x112 in bf16 (CUDA events over 200 launches), with the algorithmic bytes (every operand read once, the
    output written once) over that time against the H100 SXM's 3.35 TB/s.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

import oracle  # noqa: E402
from oracle import nets as onets  # noqa: E402
from oracle import unetthin as othin  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200 import _abi  # noqa: E402
from pytorchdeeplearing_b200.graphed import GraphedStep  # noqa: E402

SIZES = ((2, (96, 96, 96)), (1, (128, 112, 112)))
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, n):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n


def graphed(cls, n, sp, seed=0):
    model = cls(1, 2)
    spec = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    model.load_state_dict(onets.init_state_dict(spec, seed=seed, randomize_affine=True))
    model = model.cuda().train()
    x, y = oracle.make_inputs(n, 1, sp, 2, seed=1)
    opt = b200.FusedAdamW(model.parameters(), lr=1e-4)
    return GraphedStep(model, b200.MutilDiceLoss(torch.ones(2).cuda()), x.cuda(), y.cuda(), warmup=2, optimizer=opt)


def oracle_step(n, sp):
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    sd = onets.init_state_dict(othin.unetthin_state_spec(1, 2), seed=0, randomize_affine=True)
    params = {k: v.cuda().requires_grad_(True) for k, v in sd.items()}
    opt = torch.optim.AdamW(params.values(), lr=1e-4)
    x, y = oracle.make_inputs(n, 1, sp, 2, seed=1)
    x, y = x.cuda(), y.cuda()
    chans = onets.unet_mask_channels(16)

    def step():
        opt.zero_grad()
        masks = [torch.empty((n, c, 1, 1, 1), device="cuda").bernoulli_(0.8).div_(0.8).view(n, c) for c in chans]
        lo, _ = othin.unetthin_forward(params, x, masks)
        oracle.loss_forward("MutilDiceLoss", lo, y, torch.ones(2, device="cuda")).backward()
        opt.step()
    return step


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_unet3dthin needs a CUDA device")
    print(f"# {card()}", flush=True)
    b200.set_precision("bf16")
    for n, sp in SIZES:
        steps = {"UNet3dthin": graphed(b200.UNet3dthin, n, sp), "UNet3d": graphed(b200.UNet3d, n, sp)}
        ms = {k: [] for k in steps}
        for _ in range(args.rounds):
            for k, st in steps.items():
                ms[k].append(timed(st, args.steps))
        for k, v in ms.items():
            print(json.dumps({"what": "step", "net": k, "n": n, "spatial": sp, "ms": round(float(np.median(v)), 3),
                              "windows_ms": [round(t, 3) for t in v]}), flush=True)
        del steps
        st = oracle_step(n, sp)
        for _ in range(2):
            st()
        t = [timed(st, max(3, args.steps // 4)) for _ in range(args.rounds)]
        print(json.dumps({"what": "oracle_step", "net": "UNet3dthin", "n": n, "spatial": sp,
                          "ms": round(float(np.median(t)), 3)}), flush=True)
        del st
        torch.cuda.empty_cache()
    be = _abi.CudaBackend()
    for n, sp in SIZES:
        tot = {"fwd": [0.0, 0], "bwd": [0.0, 0]}
        for lvl in range(4):
            fine = tuple(s >> lvl for s in sp)
            coarse = tuple(s // 2 for s in fine)
            c = 16 << lvl
            a = torch.randn((n,) + coarse + (c,), device="cuda").to(torch.bfloat16)
            e = torch.randn((n,) + fine + (c,), device="cuda").to(torch.bfloat16)
            s = torch.empty_like(e)
            ga = torch.empty_like(a)
            for which, fn, nbytes in (("fwd", lambda: be.upsample_add(a, e, s), 2 * (a.numel() + 2 * e.numel())),
                                      ("bwd", lambda: be.upsample_bwd(e, ga), 2 * (e.numel() + a.numel()))):
                fn()
                us = 1e3 * timed(fn, 200)
                tot[which][0] += us
                tot[which][1] += nbytes
                print(json.dumps({"what": "kernel", "op": which, "n": n, "fine": fine, "C": c, "us": round(us, 2),
                                  "MB": round(nbytes / 1e6, 2), "TB/s": round(nbytes / us / 1e6, 3),
                                  "of_3.35TB/s": round(nbytes / us / 1e6 / 3.35, 3)}), flush=True)
        for which, (us, nbytes) in tot.items():
            print(json.dumps({"what": "kernel_sum", "op": which, "n": n, "spatial": sp, "us": round(us, 2),
                              "MB": round(nbytes / 1e6, 1), "of_3.35TB/s": round(nbytes / us / 1e6 / 3.35, 3)}),
                  flush=True)


if __name__ == "__main__":
    main()
