#!/usr/bin/env python
"""tests/golden/staging.npz: what the reference's OWN 2-D dataset class returns for a few 8-bit PNG files.

Build container only (needs $PYTORCHDEEPLEARING_REFERENCE and cv2):    python tests/golden/make_golden_staging.py

Writes random 8-bit images / label masks as PNG into a temporary directory, reads them back through the unmodified
``datasetModelSegwithopencv`` (model/dataset.py:120-158; targetsize == file size, so cv2.resize is the identity) and
stores the raw uint8 arrays next to the tensors the dataset returned, after the trainer's label binarisation
(model/modelUnet.py:130).  tests/test_oracle_golden.py checks oracle/staging.py against it; the GPU tests check the
staging kernels against the same arrays."""
import importlib.util
import os
import sys
import tempfile

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE", "reference")


def main():
    spec = importlib.util.spec_from_file_location("ref_dataset", os.path.join(REF, "model", "dataset.py"))
    mod = importlib.util.module_from_spec(spec)
    sys.dont_write_bytecode = True
    spec.loader.exec_module(mod)
    rng = np.random.default_rng(20240923)
    h, w = 64, 64          # square: the reference passes (targetsize[1], targetsize[2]) to cv2.resize as (width, height)
    imgs, labs = [], []
    imgs.append(rng.integers(0, 256, (h, w), dtype=np.uint8))                       # full range
    imgs.append((rng.normal(120, 3, (h, w)).clip(0, 255)).astype(np.uint8))         # low variance around a large mean
    imgs.append((rng.random((h, w)) > 0.97).astype(np.uint8) * 255)                 # sparse
    g = np.zeros((h, w), np.uint8); g[:, : w // 2] = 7                              # two levels
    imgs.append(g)
    for i in range(4):
        labs.append(((rng.random((h, w)) > 0.7) * (255 if i % 2 == 0 else 3)).astype(np.uint8))
    with tempfile.TemporaryDirectory() as d:
        ip, lp = [], []
        for i, (a, b) in enumerate(zip(imgs, labs)):
            ip.append(os.path.join(d, f"img{i}.png")); lp.append(os.path.join(d, f"lab{i}.png"))
            assert cv2.imwrite(ip[-1], a) and cv2.imwrite(lp[-1], b)
        ds = mod.datasetModelSegwithopencv(ip, lp, targetsize=(1, h, w))
        xs, ys = [], []
        for i in range(len(ds)):
            item = ds[i]
            xs.append(item["image"]); ys.append(item["label"])
    x = torch.stack(xs, 0)
    y = torch.stack(ys, 0)
    y[y != 0] = 1                                                                    # modelUnet.py:130
    np.savez_compressed(os.path.join(HERE, "staging.npz"), images_u8=np.stack(imgs), labels_u8=np.stack(labs),
                        x=x.numpy(), y=y.numpy())
    print("wrote staging.npz", x.shape, x.dtype, y.shape, y.dtype, float(x.mean()), float(x.std()))


if __name__ == "__main__":
    main()
