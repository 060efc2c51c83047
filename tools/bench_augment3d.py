#!/usr/bin/env python
"""Time the 3-D augmentation warp (csrc/augment3d.cu: ImageDataGenerator3D's order-0 affine warp, bit-exact scipy)
and the drop-in's entry points against scipy on the host.

    python tools/bench_augment3d.py [--repeats 100] [--out result.json]

kernel_us        one launch warping a batch, C = 1, uint8 labels written as int64 (y != 0): CUDA events around windows
                 of ``--repeats`` back-to-back launches (the statistics launch included when shifting), median of five
                 windows, per batch; GB/s from the bytes the algorithm moves (fp32 image in and out, uint8 label in,
                 int64 label out; the statistics pass reads the image once more), computed from the shapes
transform_batch_ms  ImageDataGenerator3D.transform_batch per call (host draws and matrices, the table copy, the launch),
                 wall time around ``--repeats`` calls ending in a device synchronise
random_transform_ms  the drop-in's random_transform per sample (numpy in and out) and scipy.ndimage.affine_transform on
                 the host on the same matrix (image and label), per sample
Shapes: 2 x 96^3 and 4 x (64, 128, 128).  The card's name and power limit are printed with the numbers.
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
from pytorchdeeplearing_b200 import _abi, augment as A, runtime  # noqa: E402

SHAPES = {"2x96^3": (2, (96, 96, 96)), "4x64x128x128": (4, (64, 128, 128))}
OPTIONS = dict(rotation_range=10, width_shift_range=0.01, height_shift_range=0.01, depth_shift_range=0.01,
               zoom_range=0.01, horizontal_flip=True, rescale=1.1)


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def kernel_us(n, shape, shift, repeats):
    be = runtime.cuda_backend()
    rng = np.random.default_rng(0)
    x = torch.from_numpy(rng.standard_normal((n,) + shape + (1,)).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.integers(0, 2, (n,) + shape).astype(np.uint8)).cuda()
    gen = A.ImageDataGenerator3D(channel_shift_range=0.1 if shift else 0, **OPTIONS)
    np.random.seed(0)
    entries = [A.param_entry(A.draw_transform(gen, shape, 1), shape) for _ in range(n)]
    params = torch.frombuffer(bytearray(_abi.aug3d_param_table(entries)), dtype=torch.uint8).cuda()
    xo, yo = torch.empty_like(x), torch.empty(y.shape, dtype=torch.int64, device="cuda")
    ws = be.augment3d_workspace(n, shape, x.device) if shift else None
    mode, value = A.rescale_form(1.1)

    def run():
        be.augment3d(x, y, params, xo, yo, mode=0, shift=shift, rescale=value, rescale_mode=mode, binarize=True,
                     ws=ws)

    for _ in range(5):
        run()
    times = []
    for _ in range(5):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(repeats):
            run()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / repeats)
    us = statistics.median(times)
    vox = n * int(np.prod(shape))
    nbytes = vox * (4 + 4 + 1 + 8) + (vox * 4 if shift else 0)
    return round(us, 2), round(nbytes / (us * 1e-6) / 1e9, 1), nbytes


def transform_batch_ms(n, shape, repeats):
    rng = np.random.default_rng(1)
    x = torch.from_numpy(rng.standard_normal((n, 1) + shape).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.integers(0, 2, (n,) + shape).astype(np.uint8)).cuda()
    gen = b200.ImageDataGenerator3D(**OPTIONS)
    for _ in range(3):
        gen.transform_batch(x, y)
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(repeats):
        gen.transform_batch(x, y)
    torch.cuda.synchronize()
    return round((time.perf_counter() - t) * 1e3 / repeats, 3)


def random_transform_ms(shape, repeats):
    import scipy.ndimage as ndi
    rng = np.random.default_rng(2)
    x = rng.standard_normal(shape + (1,)).astype(np.float32)
    y = rng.integers(0, 2, shape + (1,)).astype(np.float32)
    gen = b200.ImageDataGenerator3D(**OPTIONS)
    for _ in range(2):
        gen.random_transform(x, y)
    t = time.perf_counter()
    for _ in range(repeats):
        gen.random_transform(x, y)
    dev = (time.perf_counter() - t) * 1e3 / repeats
    np.random.seed(0)
    m = A.compose_matrix(A.draw_transform(gen, shape, 1), shape)
    reps = max(1, repeats // 10)
    t = time.perf_counter()
    for _ in range(reps):
        ndi.affine_transform(x[..., 0], m[:3, :3], m[:3, 3], order=0, mode="nearest", cval=0.0)
        ndi.affine_transform(y[..., 0], m[:3, :3], m[:3, 3], order=0, mode="nearest", cval=0.0)
    host = (time.perf_counter() - t) * 1e3 / reps
    return round(dev, 2), round(host, 2)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_augment3d needs a CUDA device"
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit}
    for key, (n, shape) in SHAPES.items():
        for shift in (False, True):
            us, gbs, nbytes = kernel_us(n, shape, shift, args.repeats)
            tag = f"{key}{'_shift' if shift else ''}"
            res[f"kernel_us_{tag}"] = us
            res[f"kernel_GBps_{tag}"] = gbs
            res[f"bytes_{tag}"] = nbytes
        res[f"transform_batch_ms_{key}"] = transform_batch_ms(n, shape, args.repeats)
    dev, host = random_transform_ms((96, 96, 96), max(10, args.repeats // 5))
    res["random_transform_ms_96^3"] = dev
    res["scipy_affine_transform_ms_96^3"] = host
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
