"""Time the per-step 2-D augmentation (Segmenation_Aug, csrc/augment2d.cu) against the cv2 oracle on every host core.

    python tools/bench_augment2d.py [--iters 200] [--out results/bench_augment2d.json]

Two cases at batch 8: 512 x 512 gray images with masks (``transform_batch``), and a ragged batch of ~1000 x 700 gray
sources with labels resized to 512 x 512 (``InputStager(augment=...)``: draws, one ragged copy, augment, resize,
z-score).  For each: the kernels alone with every stage drawn on every image (CUDA events, a fixed table), the whole
call (host draws and table included, host clock around a device synchronise), and the host path (the oracle's cv2
calls, plus cv2.resize for the ragged case, over a process pool of every core).  Prints one JSON line per case with
the GPU's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import multiprocessing as mp
import os
import random
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import pytorchdeeplearing_b200 as b200  # noqa: E402
from pytorchdeeplearing_b200 import augment2d as A2, runtime  # noqa: E402
from oracle import augment2d as oa  # noqa: E402


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 else "unknown"


def all_stages_draw():
    """a draw with every stage on: flips, a 7-tap motion blur, the warp and the table"""
    return {"hflip": True, "vflip": True, "blur": "motion", "kernel": oa.motion_kernel(7, 0, 1, 6, 5),
            "ssr": (31.0, 1.1, 0.03, -0.02), "bc": (1.2, 0.1)}


def time_kernel(imgs, iters):
    """events around b200seg_augment2d on a fixed all-stages table (images with masks)"""
    dev = torch.device("cuda", 0)
    entries, soff = [], 0
    for img in imgs:
        h, w = img.shape
        e, f = A2.param_entry(all_stages_draw(), h, w, 1, soff, soff, soff, soff, filter_cn=3)
        entries.append((e, f, h * w))
        soff += img.size
    src = torch.from_numpy(np.concatenate([i.reshape(-1) for i in imgs])).to(dev)
    msrc = src.clone()
    out, mout = torch.empty_like(src), torch.empty_like(src)
    be = runtime.get_backend(src)
    params = torch.frombuffer(bytearray(b"".join(e for e, _, _ in entries)), dtype=torch.uint8).to(dev)
    ws = be.augment2d_workspace(out.numel(), dev)
    max_hw = max(hw for _, _, hw in entries)
    for _ in range(10):
        be.augment2d(src, params, len(imgs), max_hw, 31, out, msrc=msrc, mout=mout, ws=ws)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        be.augment2d(src, params, len(imgs), max_hw, 31, out, msrc=msrc, mout=mout, ws=ws)
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) * 1000 / iters


def _host_one(args):
    import cv2
    img, lab, seed, dsize = args
    random.seed(seed)
    d = oa.draw()
    x, y = oa.apply(d, np.repeat(img[..., None], 3, axis=2), lab)
    x = x[..., 0]
    if dsize is not None:
        x, y = cv2.resize(x, dsize), cv2.resize(y, dsize)
    return x, y


def time_host(pool, imgs, labs, dsize, iters):
    jobs = [(im, lb, i, dsize) for i, (im, lb) in enumerate(zip(imgs, labs))]
    pool.map(_host_one, jobs)
    t0 = time.perf_counter()
    for _ in range(iters):
        pool.map(_host_one, jobs)
    return (time.perf_counter() - t0) * 1e6 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_augment2d needs a CUDA device")
    dev = torch.device("cuda", 0)
    rng = np.random.RandomState(0)
    info, lines = gpu_info(), []
    aug = b200.Segmenation_Aug()
    pool = mp.Pool(os.cpu_count())

    # 512 x 512 gray, batch 8, transform_batch
    imgs = [rng.randint(0, 256, (512, 512)).astype(np.uint8) for _ in range(8)]
    labs = [(rng.rand(512, 512) > 0.5).astype(np.uint8) for _ in range(8)]
    x = torch.from_numpy(np.stack(imgs)).to(dev)
    y = torch.from_numpy(np.stack(labs)).to(dev)
    for _ in range(10):
        aug.transform_batch(x, y)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        aug.transform_batch(x, y)
    torch.cuda.synchronize()
    call = (time.perf_counter() - t0) * 1e6 / a.iters
    lines.append(dict(case="512x512 gray x8, transform_batch", gpu=info, kernel_all_stages_us=time_kernel(imgs, a.iters),
                      call_us=call, host_cv2_pool_us=time_host(pool, imgs, labs, None, max(5, a.iters // 20)),
                      host_cores=os.cpu_count()))

    # ragged ~1000 x 700 sources -> 512 x 512, InputStager(augment=...)
    sizes = [(1000, 700), (700, 1000), (980, 720), (1024, 680), (1000, 700), (960, 740), (700, 1000), (1010, 690)]
    imgs = [rng.randint(0, 256, s).astype(np.uint8) for s in sizes]
    labs = [(rng.rand(*s) > 0.5).astype(np.uint8) for s in sizes]
    st = b200.InputStager(dev, (8, 512, 512), max_source_pixels=8 << 20, augment=aug)
    for _ in range(5):
        st.put(imgs, labs)
        st.get()
        st.release()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(a.iters):
        st.put(imgs, labs)
        st.get()
        st.release()
    torch.cuda.synchronize()
    call = (time.perf_counter() - t0) * 1e6 / a.iters
    lines.append(dict(case="ragged ~1000x700 gray x8 -> 512x512, InputStager(augment=...)", gpu=info,
                      kernel_all_stages_us=time_kernel(imgs, a.iters), call_us=call,
                      host_cv2_pool_us=time_host(pool, imgs, labs, (512, 512), max(5, a.iters // 20)),
                      host_cores=os.cpu_count()))
    pool.close()
    pool.join()
    for ln in lines:
        print(json.dumps(ln))
    if a.out:
        os.makedirs(os.path.dirname(a.out), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(json.dumps(ln) for ln in lines) + "\n")


if __name__ == "__main__":
    main()
