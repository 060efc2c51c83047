#!/usr/bin/env python
"""Time the 2-D image resize (csrc/resize2d.cu: cv2.resize INTER_LINEAR, bit-exact) and the resize mode of
InputStager against the host path of the reference's 2-D dataset.

    python tools/bench_resize2d.py [--repeats 200] [--out result.json]

kernel_us      one ragged launch resizing N = 8 images, uint8 and fp32 (/255) outputs: CUDA events around windows of
               ``--repeats`` back-to-back launches, median of five windows, per launch
stager_ms      InputStager(max_source_pixels=...): put (pack into pinned memory, one H2D copy, resize, z-score, label
               widening) + get + release, per batch of 8 images and labels, wall time of ``--repeats`` batches with
               the device work included; stager_put_call_ms: the time put() takes to return (the host packing)
host_ms        the reference's per-batch host work: cv2.resize of every image and label, the float64 z-score, fp32 /
               int64 tensors and their upload (pageable memory), wall time per batch
Sizes: 1024x1024 -> 512x512 and 300x417 -> 512x512.  The card's name and power limit are printed with the numbers.
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

N = 8
TARGET = (512, 512)
SOURCES = {"1024x1024": (1024, 1024), "300x417": (300, 417)}


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = (s.strip() for s in q.split(","))
    except Exception:
        name, limit = torch.cuda.get_device_name(), "unknown"
    return name, limit


def kernel_us(images, dtype, repeats):
    be = runtime.cuda_backend()
    pix = torch.from_numpy(np.concatenate([im.ravel() for im in images])).cuda()
    offs = np.cumsum([0] + [im.size for im in images])[:-1]
    desc = inf.resize_desc(be, [(o, *im.shape) for o, im in zip(offs, images)], pix.device)
    out = torch.empty((len(images),) + TARGET, dtype=dtype, device="cuda")
    for _ in range(5):
        be.resize_linear(pix, desc, out)
    times = []
    for _ in range(5):                          # windows of `repeats` back-to-back launches
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(repeats):
            be.resize_linear(pix, desc, out)
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b) * 1e3 / repeats)
    return round(statistics.median(times), 2)


def stager_ms(images, labels, repeats):
    st = b200.InputStager("cuda", (N,) + TARGET, max_source_pixels=sum(im.size for im in images))
    for _ in range(3):
        st.put(images, labels)
        st.get()
        st.release()
    torch.cuda.synchronize()
    put_s = 0.0
    t0 = time.perf_counter()
    for _ in range(repeats):
        p0 = time.perf_counter()
        st.put(images, labels)
        put_s += time.perf_counter() - p0
        st.get()
        st.release()
    torch.cuda.synchronize()
    return round((time.perf_counter() - t0) * 1e3 / repeats, 3), round(put_s * 1e3 / repeats, 3)


def host_ms(images, labels, repeats):
    try:
        import cv2
        resize, how = (lambda im: cv2.resize(im, (TARGET[1], TARGET[0]))), "cv2"
    except ImportError:                        # the numpy restatement stands in (much slower than cv2)
        from oracle import resize2d as RZ
        resize, how = (lambda im: RZ.resize_u8(im, (TARGET[1], TARGET[0]))), "oracle/resize2d.py (cv2 not installed)"

    def one():
        xs, ys = [], []
        for im, lb in zip(images, labels):
            a = resize(im)
            xs.append(torch.as_tensor(((a - a.mean()) / a.std())[None]).float())
            ys.append(torch.as_tensor(resize(lb)).long())
        x = torch.stack(xs).cuda()
        y = torch.stack(ys)
        y[y != 0] = 1
        y = y.cuda()
        return x, y
    for _ in range(2):
        one()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(repeats):
        one()
    torch.cuda.synchronize()
    return round((time.perf_counter() - t0) * 1e3 / repeats, 3), how


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resize2d needs a CUDA device")
    name, limit = gpu_info()
    res = {"gpu": name, "power_limit": limit, "batch": N, "target": "512x512"}
    rng = np.random.RandomState(0)
    for tag, shape in SOURCES.items():
        images = [rng.randint(0, 256, shape).astype(np.uint8) for _ in range(N)]
        labels = [((rng.rand(*shape) > 0.7) * 255).astype(np.uint8) for _ in range(N)]
        r = {"kernel_us_u8": kernel_us(images, torch.uint8, a.repeats),
             "kernel_us_f32": kernel_us(images, torch.float32, a.repeats)}
        r["stager_ms"], r["stager_put_call_ms"] = stager_ms(images, labels, a.repeats)
        r["host_ms"], res["host_resize"] = host_ms(images, labels, max(5, a.repeats // 20))
        res[tag] = r
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
