#!/usr/bin/env python
"""Generate tests/golden/segmetric.npz by RUNNING THE UNMODIFIED REFERENCE ``Seg_Metirc3d`` (model/metric.py:11-142).

Usage (needs a reference checkout named by $PYTORCHDEEPLEARING_REFERENCE; skimage and the other I/O-only modules are
stubbed by tests/ref_harness.py):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/PytorchDeepLearing python tests/golden/make_golden_segmetric.py

For every case the file holds both masks (np.packbits, with shape and dtype), the spacing, the nine metric values,
the dice tuple, the surface counts and, for the small cases, the surface points and both nn distance arrays.  The
``empty`` case records that the constructor raised ValueError.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
import ref_harness  # noqa: E402

SMALL = 20000            # cases up to this many voxels also keep the points and per-point distances


def ellipsoid(shape, centre, radii):
    z, y, x = np.ogrid[tuple(slice(0, s) for s in shape)]
    return (((z - centre[0]) / radii[0]) ** 2 + ((y - centre[1]) / radii[1]) ** 2 +
            ((x - centre[2]) / radii[2]) ** 2) <= 1.0


def cases():
    rng = np.random.RandomState(7)
    out = {}
    sh = (28, 80, 96)
    out["ellipsoids"] = (ellipsoid(sh, (13, 38, 45), (9, 28, 33)), ellipsoid(sh, (15, 42, 50), (8, 25, 36)),
                         (0.78, 0.78, 2.5))
    a = ellipsoid((12, 14, 16), (6, 7, 8), (4, 5, 6))
    out["identical"] = (a, a.copy(), (1.0, 1.5, 2.0))
    r = np.zeros((10, 12, 14), bool)
    p = np.zeros_like(r)
    r[:3, :3, :3] = True
    p[-2:, -3:, -2:] = True
    out["disjoint_corners"] = (r, p, (0.7, 1.1, 1.9))
    r = np.zeros((7, 9, 11), bool)
    r[:, 2:7, :] = True
    r[:, :, 3:8] = True
    r[2:5] = True                                                       # touches all six faces
    out["six_faces"] = (r, ellipsoid(r.shape, (3, 4, 5), (3, 4, 4)), (0.5, 0.5, 1.25))
    out["scattered"] = (rng.rand(9, 10, 11) < 0.08, rng.rand(9, 10, 11) < 0.06, (1.3, 0.9, 0.6))
    r = np.zeros((9, 11, 13), bool)
    r[4, 1:10, 2:12] = True                                             # one-voxel-thick sheet
    p = np.zeros_like(r)
    p[1:8, 6, 7] = True                                                 # a line
    out["sheet_line"] = (r, p, (0.8, 1.0, 3.0))
    r = np.zeros((8, 9, 10), bool)
    r[5, 2, 7] = True
    out["single_voxel"] = (r, ellipsoid(r.shape, (3, 4, 4), (2, 2, 3)), (1.0, 1.0, 1.0))
    out["d1"] = (ellipsoid((1, 30, 40), (0, 14, 19), (1, 10, 14)), ellipsoid((1, 30, 40), (0, 16, 21), (1, 9, 16)),
                 (0.6, 0.6, 5.0))
    out["odd_extents"] = (ellipsoid((13, 7, 37), (6, 3, 17), (5, 3, 14)), ellipsoid((13, 7, 37), (7, 3, 20), (4, 3, 12)),
                          (0.9, 2.1, 1.7))
    r = np.zeros((4, 5, 6), bool)
    r[0:4, 0:3, 0:4] = True                                             # 4x3x4 block touching two faces: 44 surface
    out["block_two_faces"] = (r, ellipsoid(r.shape, (2, 2, 3), (2, 2, 2)), (1.0, 1.0, 1.0))
    # the same masks in three dtypes; pred is smaller than real, so the reference's uint8 RVD wraps around
    r = ellipsoid((14, 16, 18), (7, 8, 9), (5, 6, 7))
    p = ellipsoid((14, 16, 18), (7, 8, 9), (5, 6, 6))
    out["dtype_bool"] = (r, p, (0.9, 0.9, 1.8))
    out["dtype_int64"] = (r.astype(np.int64), p.astype(np.int64), (0.9, 0.9, 1.8))
    out["dtype_uint8"] = (r.astype(np.uint8), p.astype(np.uint8), (0.9, 0.9, 1.8))
    out["empty"] = (np.zeros((5, 6, 7), bool), ellipsoid((5, 6, 7), (2, 3, 3), (2, 2, 2)), (1.0, 1.0, 1.0))
    return out


def main():
    assert ref_harness.available(), "set PYTORCHDEEPLEARING_REFERENCE to a reference checkout"
    M = ref_harness.import_reference()["model.metric"]
    res = {}
    names = []
    for name, (r, p, sp) in cases().items():
        names.append(name)
        res[name + "_shape"] = np.array(r.shape, dtype=np.int64)
        res[name + "_dtype"] = np.array(str(r.dtype))
        res[name + "_real"] = np.packbits(r.astype(bool).ravel())
        res[name + "_pred"] = np.packbits(p.astype(bool).ravel())
        res[name + "_spacing"] = np.array(sp, dtype=np.float64)
        try:
            m = M.Seg_Metirc3d(r, p, sp)
        except ValueError as e:
            res[name + "_raises"] = np.array(str(e))
            print(f"{name}: ValueError {e}")
            continue
        dice = m.get_dice_coefficient()
        vals = [dice[0], m.get_jaccard_index(), m.get_VOE(), m.get_RVD(), m.get_FNR(), m.get_FPR(), m.get_ASSD(),
                m.get_RMSD(), m.get_MSD()]
        res[name + "_metrics"] = np.array([float(v) for v in vals], dtype=np.float64)
        res[name + "_types"] = np.array([type(v).__name__ for v in vals] + [type(dice[1]).__name__,
                                                                           type(dice[2]).__name__])
        res[name + "_dice_tuple"] = np.array([int(dice[1]), int(dice[2])], dtype=np.int64)
        res[name + "_S"] = np.array([len(m.real2pred_nn), len(m.pred2real_nn)], dtype=np.int64)
        if r.size <= SMALL:
            res[name + "_real_pts"] = m.real_mask_surface_pts
            res[name + "_pred_pts"] = m.pred_mask_surface_pts
            res[name + "_real2pred"] = m.real2pred_nn
            res[name + "_pred2real"] = m.pred2real_nn
        print(f"{name}: {r.shape} S={res[name + '_S'].tolist()} " +
              " ".join(f"{v:.6g}" for v in res[name + "_metrics"]))
    res["cases"] = np.array(names)
    np.savez_compressed(os.path.join(HERE, "segmetric.npz"), **res)


if __name__ == "__main__":
    main()
