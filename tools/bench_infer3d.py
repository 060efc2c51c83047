#!/usr/bin/env python
"""Time the whole-volume 3-D inference (XModel.inference, reference model/modelVNet.py:678-698) of a 512x512x300
int16 CT volume through VNet3d(1, 2) at 96^3: where the time of the call goes, on the device and end to end.

    python tools/bench_infer3d.py [--repeats 10] [--precision bf16] [--out result.json]

Device stages (median of ``--repeats`` runs after a warm-up, CUDA events around each stage in one chain):
  upload      numpy int16 volume -> device (pageable host memory, 2 B per voxel)
  resample    linear resample to 96^3 with the fused truncation and partial sums ("vnet") or sort keys ("unet")
  normalize   meanstd ("vnet") or normalize() ("unet": sort, percentiles, two statistics passes, apply)
  network     predict_mask: the eval forward and the fused mask head
  back        nearest-neighbour resample of the uint8 mask to 512x512x300
  download    uint8 mask -> host (1 B per voxel)
End to end: host wall time of ``inference3d`` from the numpy volume to the numpy mask.
Host chain: the same steps done as the reference does them on the host, by the numpy restatement (oracle/resample.py:
fp64 resample, fp32 truncation and float64 statistics, the fp32 network input copied to the device, ``predict``, and the
host NN resample of the mask).  The reference itself needs SimpleITK, which is not installed; its ITK resamples are
multithreaded C++ and will differ from the numpy restatement's times.
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

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200 import inference as inf, runtime  # noqa: E402
from oracle import nets as onets, resample as R  # noqa: E402

SHAPE = (300, 512, 512)      # (D, H, W): ITK size 512 x 512 x 300
NEW = (96, 96, 96)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def device_stages(model, arr, intensity):
    be = runtime.cuda_backend()
    mode = inf._INTENSITY[intensity]
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
    torch.cuda.synchronize()
    ev[0].record()
    vol = torch.from_numpy(arr).cuda()
    ev[1].record()
    ratio = R.size_ratio(SHAPE, NEW)
    x = torch.empty(NEW, dtype=torch.float32, device="cuda")
    ws = be.resample_workspace(mode, NEW, vol.device)
    be.resample_linear(vol, ratio, x, mode, -100.0, 100.0, ws)
    ev[2].record()
    xn = torch.empty_like(x)
    be.normalize(mode, x, ws, xn)
    ev[3].record()
    m = inf.predict_mask(model, xn.view((1, 1) + NEW))[0].contiguous()
    ev[4].record()
    out = torch.empty(SHAPE, dtype=torch.uint8, device="cuda")
    be.resample_nearest_u8(m, R.size_ratio(NEW, SHAPE), SHAPE, out)
    ev[5].record()
    host = out.cpu().numpy()
    ev[6].record()
    ev[6].synchronize()
    names = ("upload", "resample", "normalize", "network", "back", "download")
    return {n: ev[i].elapsed_time(ev[i + 1]) for i, n in enumerate(names)}, host


def host_chain(model, arr):
    t = {}
    t0 = time.perf_counter()
    x = R.resample_linear(arr, NEW, R.size_ratio(SHAPE, NEW))
    t1 = time.perf_counter()
    x = R.meanstd(R.truncate(x, -100.0, 100.0))
    t2 = time.perf_counter()
    m = b200.predict(model, x[None])
    t3 = time.perf_counter()
    mask = R.resample_nearest(m, R.size_ratio(NEW, SHAPE), SHAPE, SHAPE)
    t4 = time.perf_counter()
    t.update(resample=(t1 - t0) * 1e3, normalize=(t2 - t1) * 1e3, predict=(t3 - t2) * 1e3, back=(t4 - t3) * 1e3,
             total=(t4 - t0) * 1e3)
    return t, mask


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=10)
    ap.add_argument("--host-repeats", type=int, default=2)
    ap.add_argument("--precision", default="bf16")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_infer3d needs a CUDA device")
    b200.set_precision(a.precision)
    model = b200.VNet3d(1, 2)
    model.load_state_dict(onets.init_state_dict(onets.vnet3d_state_spec(1, 2), seed=0, randomize_affine=True))
    model = model.cuda().eval()
    arr = np.random.RandomState(0).randint(-1024, 2000, size=SHAPE).astype(np.int16)
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit, "precision": a.precision, "volume": "512x512x300 int16",
           "network": "VNet3d(1, 2) at 96^3"}
    for intensity in ("vnet", "unet"):
        for _ in range(2):
            device_stages(model, arr, intensity)
        runs = [device_stages(model, arr, intensity)[0] for _ in range(a.repeats)]
        res[f"device_ms_{intensity}"] = {k: round(statistics.median(r[k] for r in runs), 4) for k in runs[0]}
    for _ in range(2):
        b200.inference3d(model, arr, NEW)
    torch.cuda.synchronize()
    wall = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        mask = b200.inference3d(model, arr, NEW)
        wall.append((time.perf_counter() - t0) * 1e3)
    res["end_to_end_ms_vnet"] = round(statistics.median(wall), 3)
    host = [host_chain(model, arr) for _ in range(a.host_repeats)]
    res["host_chain_ms"] = {k: round(statistics.median(h[0][k] for h in host), 2) for k in host[0][0]}
    res["host_chain_equal_mask"] = bool(np.array_equal(mask, host[-1][1]))
    res["note"] = ("host_chain is the numpy restatement of the reference's host steps; the reference itself needs "
                   "SimpleITK, which is not installed, so it was not run")
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
