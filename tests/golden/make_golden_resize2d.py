#!/usr/bin/env python
"""tests/golden/resize2d.npz: what cv2 and the reference's own 2-D code return around ``cv2.resize``.

Build container only (needs cv2 and a reference checkout named by $PYTORCHDEEPLEARING_REFERENCE; the wrappers' modules
import SimpleITK, torchsummary, skimage and matplotlib, which tests/ref_harness.py replaces by inert stubs):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/PytorchDeepLearing python tests/golden/make_golden_resize2d.py

Records
  - ``cv2.resize(src, dsize)`` for a fixed list of cases (``rs_<case>_src`` / ``_dsize`` (width, height) / ``_dst``):
    non-integer up- and downscales, exact 2x and 4x downscales, the identity, 1x1 and 1x700 sources, a 1x1
    destination, non-square dsize; random, 0/255 and 0-3 label images;
  - the unmodified ``datasetModelSegwithopencv`` (model/dataset.py:119-158) on PNG files whose sizes differ from the
    target, with the trainer's label binarisation (model/modelUnet.py:130) (``seg_*``), and the unmodified
    ``datasetModelClassifywithopencv`` (dataset.py:42-78) (``cls_*``);
  - the wrappers' own ``inference`` methods (model/modelVNet.py:231-242, model/modelUnet.py:450-461,
    model/modelResNet.py:212-221) with ``predict`` replaced by a recorder that returns a given uint8 mask: the fp32
    network input ``predict`` would build (``torch.as_tensor(full_img).float()``) and ``cv2.resize(mask, image.shape)``
    for a square and a non-square image (``inf_*``)."""
import importlib
import os
import sys
import tempfile

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ref_harness  # noqa: E402


def resize_cases():
    rng = np.random.RandomState(2024)
    rnd = lambda h, w: rng.randint(0, 256, (h, w)).astype(np.uint8)
    binary = lambda h, w: ((rng.rand(h, w) > 0.6) * 255).astype(np.uint8)
    labels = lambda h, w: rng.randint(0, 4, (h, w)).astype(np.uint8)
    return {
        "up_nonint": (rnd(37, 53), (101, 80)),
        "down_nonint": (rnd(300, 417), (128, 96)),
        "down2": (rnd(256, 200), (100, 128)),
        "down4": (rnd(256, 256), (64, 64)),
        "identity": (rnd(64, 48), (48, 64)),
        "src1x1": (rnd(1, 1), (9, 7)),
        "src1x700": (rnd(1, 700), (128, 128)),
        "dst1x1": (rnd(45, 67), (1, 1)),
        "nonsquare": (rnd(120, 80), (64, 96)),
        "binary_up": (binary(50, 60), (173, 131)),
        "binary_down": (binary(200, 150), (96, 96)),
        "labels_up": (labels(90, 70), (256, 256)),
        "labels_down": (labels(333, 251), (64, 80)),
    }


def dataset_inputs(rng, sizes, label_kind):
    imgs = [rng.randint(0, 256, s).astype(np.uint8) for s in sizes]
    labs = []
    for i, s in enumerate(sizes):
        if label_kind == "mixed" and i % 2:
            labs.append(rng.randint(0, 4, s).astype(np.uint8))
        else:
            labs.append(((rng.rand(*s) > 0.7) * 255).astype(np.uint8))
    return imgs, labs


class _Recorder:
    """stands in for the wrapper's predict: keeps the network input it is handed, returns a fixed mask"""

    def __init__(self, mask):
        self.mask, self.x = mask, None

    def __call__(self, full_img, out_threshold=0.5):
        self.x = torch.as_tensor(full_img).float().contiguous().numpy()     # predict's first line
        return self.mask


def run_inference(cls, image, new_size, mask):
    wrapper = object.__new__(cls)             # no network: only the method's own lines run
    wrapper.image_width, wrapper.image_height = new_size
    rec = _Recorder(mask)
    wrapper.predict = rec
    out = wrapper.inference(image)
    return rec.x, out


def main():
    if not ref_harness.available():
        sys.exit("set PYTORCHDEEPLEARING_REFERENCE to a reference checkout")
    ref_harness.import_reference()
    dataset = importlib.import_module("model.dataset")
    m_vnet = importlib.import_module("model.modelVNet")
    m_unet = importlib.import_module("model.modelUnet")
    m_resnet = importlib.import_module("model.modelResNet")
    data, names = {}, []
    for name, (src, dsize) in resize_cases().items():
        data[f"rs_{name}_src"] = src
        data[f"rs_{name}_dsize"] = np.array(dsize, np.int64)
        data[f"rs_{name}_dst"] = cv2.resize(src, dsize)
        names.append(name)
    data["rs_cases"] = np.array(names)

    rng = np.random.RandomState(7)
    seg_sizes = [(100, 80), (50, 70), (64, 64), (33, 129)]
    cls_sizes = [(90, 41), (48, 48), (200, 333)]
    seg_img, seg_lab = dataset_inputs(rng, seg_sizes, "mixed")
    cls_img, _ = dataset_inputs(rng, cls_sizes, "binary")
    with tempfile.TemporaryDirectory() as d:
        def write(prefix, arrays):
            paths = []
            for i, a in enumerate(arrays):
                paths.append(os.path.join(d, f"{prefix}{i}.png"))
                assert cv2.imwrite(paths[-1], a)
            return paths
        ds = dataset.datasetModelSegwithopencv(write("img", seg_img), write("lab", seg_lab), targetsize=(1, 64, 64))
        items = [ds[i] for i in range(len(ds))]
        cds = dataset.datasetModelClassifywithopencv(write("cls", cls_img), [0, 1, 2], targetsize=(1, 48, 48))
        citems = [cds[i] for i in range(len(cds))]
    y = torch.stack([it["label"] for it in items])
    y[y != 0] = 1                                                                    # modelUnet.py:130
    for i, (a, b) in enumerate(zip(seg_img, seg_lab)):
        data[f"seg_img{i}"], data[f"seg_lab{i}"] = a, b
    data["seg_x"] = torch.stack([it["image"] for it in items]).numpy()
    data["seg_y"] = y.numpy()
    for i, a in enumerate(cls_img):
        data[f"cls_img{i}"] = a
    data["cls_x"] = torch.stack([it["image"] for it in citems]).numpy()

    inf = {
        "square": (m_vnet.BinaryVNet2dModel, rng.randint(0, 256, (300, 300)).astype(np.uint8), (64, 64),
                   ((rng.rand(64, 64) > 0.5) * 255).astype(np.uint8)),
        "nonsquare": (m_unet.MutilUNet2dModel, rng.randint(0, 256, (180, 260)).astype(np.uint8), (128, 96),
                      rng.randint(0, 4, (96, 128)).astype(np.uint8)),
    }
    for name, (cls, image, new_size, mask) in inf.items():
        x, out = run_inference(cls, image, new_size, mask)
        data[f"inf_{name}_image"], data[f"inf_{name}_newsize"] = image, np.array(new_size, np.int64)
        data[f"inf_{name}_mask"], data[f"inf_{name}_x"], data[f"inf_{name}_out"] = mask, x, out
    image = rng.randint(0, 256, (150, 210)).astype(np.uint8)
    x, _ = run_inference(m_resnet.BinaryResNet2dModel, image, (64, 48), np.int64(255))
    data["inf_resnet_image"], data["inf_resnet_newsize"], data["inf_resnet_x"] = image, np.array((64, 48)), x
    np.savez_compressed(os.path.join(HERE, "resize2d.npz"), **data)
    print("wrote resize2d.npz:", len(names), "resize cases;", data["seg_x"].shape, data["cls_x"].shape,
          {k: data[f"inf_{k}_out"].shape for k in inf})


if __name__ == "__main__":
    main()
