#!/usr/bin/env python
"""Generate tests/golden/infer3d.npz by RUNNING THE UNMODIFIED REFERENCE ``normalize`` (dataprocess/utils.py:182-204),
the intensity normalisation of the UNet ``XModel.inference`` (model/modelUnet.py:684-705).

Usage (needs a reference checkout named by $PYTORCHDEEPLEARING_REFERENCE; utils.py imports SimpleITK at module level,
which tests/ref_harness.py replaces by an inert stub):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/PytorchDeepLearing python tests/golden/make_golden_infer3d.py

Every case holds the int16 input (the pixel type the UNet inference hands to normalize()) and the fp64 output.  The
resamples have no fixtures: SimpleITK is not available, so oracle/resample.py is their specification.
"""
import importlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ref_harness  # noqa: E402


def cases():
    rng = np.random.RandomState(11)
    out = {}
    out["random"] = rng.randint(-1024, 2000, size=(23, 31, 29)).astype(np.int16)
    z = rng.randint(-200, 300, size=(20, 24, 28)).astype(np.int16)
    z[rng.rand(*z.shape) < 0.7] = 0
    out["zero_heavy"] = z
    out["constant"] = np.full((9, 10, 11), 37, np.int16)
    out["constant_zero"] = np.zeros((6, 7, 8), np.int16)
    # n = 21: the 5th / 95th percentile positions are exactly the order statistics 1 and 19, with ties around them
    out["ties"] = np.array([-5, -5, -5, 0, 0, 1, 2, 2, 2, 3, 3, 3, 3, 4, 7, 7, 7, 9, 9, 9, 9],
                           np.int16).reshape(1, 3, 7)
    t = rng.randint(0, 4, size=(16, 18, 20)).astype(np.int16)
    out["ties_fractional"] = t
    # all nonzero clipped values equal: std of the nonzero voxels is 0
    nz = np.zeros((10, 10, 10), np.int16)
    nz[rng.rand(*nz.shape) < 0.5] = 50
    out["nonzero_constant"] = nz
    return out


def main():
    if not ref_harness.available():
        sys.exit("set PYTORCHDEEPLEARING_REFERENCE to a reference checkout")
    ref_harness.import_reference()
    utils = importlib.import_module("dataprocess.utils")
    data = {}
    names = []
    for name, vol in cases().items():
        res = utils.normalize(vol.copy())
        data[name + "_input"] = vol
        data[name + "_output"] = np.asarray(res, np.float64)
        names.append(name)
    data["cases"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "infer3d.npz"), **data)
    print("wrote", os.path.join(HERE, "infer3d.npz"), names)


if __name__ == "__main__":
    main()
