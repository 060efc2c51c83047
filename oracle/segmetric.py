"""fp64 restatement of the nine 3-D segmentation metrics of ``Seg_Metirc3d`` (reference model/metric.py:11-142) with
scipy, written from their definitions:

- surface of a binary mask: its foreground voxels with background among their 18 neighbours (faces and edges), the
  outside of the volume counting as background -- ``mask & ~binary_erosion(mask, 18-structure, border_value=0)``;
- surface points: C-order voxel indices times the (z, y, x) spacing, the reversed SimpleITK spacing;
- real2pred / pred2real: the exact Euclidean distance in mm from each surface point of one mask to the nearest surface
  point of the other, read from ``distance_transform_edt`` of the other surface's complement;
- overlap metrics from the integer counts I, U, R, P; distance metrics from the two distance lists.
"""
from __future__ import annotations

import math

import numpy as np
from scipy import ndimage

NAMES = ("dice", "jaccard", "VOE", "RVD", "FNR", "FPR", "ASSD", "RMSD", "MSD")
STRUCT18 = ndimage.generate_binary_structure(3, 2)


def surface(mask: np.ndarray) -> np.ndarray:
    m = np.asarray(mask) != 0
    return m & ~ndimage.binary_erosion(m, structure=STRUCT18, border_value=0)


def surface_distances(real: np.ndarray, pred: np.ndarray, voxel_spacing):
    """-> (real surface indices (S_r, 3), pred surface indices (S_p, 3), real2pred (S_r,), pred2real (S_p,))"""
    sp = tuple(float(s) for s in voxel_spacing)[::-1]
    sr, spd = surface(real), surface(pred)
    if not sr.any() or not spd.any():
        raise ValueError("empty mask: surface distances are undefined")
    r2p = ndimage.distance_transform_edt(~spd, sampling=sp)[sr]
    p2r = ndimage.distance_transform_edt(~sr, sampling=sp)[spd]
    return np.argwhere(sr), np.argwhere(spd), r2p, p2r


def counts(real: np.ndarray, pred: np.ndarray):
    """-> (R, P, I, U, S_r, S_p) as Python ints"""
    r, p = np.asarray(real) != 0, np.asarray(pred) != 0
    return (int(r.sum()), int(p.sum()), int((r & p).sum()), int((r | p).sum()), int(surface(r).sum()),
            int(surface(p).sum()))


def seg_metrics(real: np.ndarray, pred: np.ndarray, voxel_spacing):
    """-> (nine metrics in Seg_Metirc3d's order as fp64 array, counts (R, P, I, U, S_r, S_p))"""
    R, P, I, U, Sr, Sp = c = counts(real, pred)
    _, _, r2p, p2r = surface_distances(real, pred, voxel_spacing)
    S = Sr + Sp
    m = [2 * I / (R + P), I / U, 1 - I / U, (P - R) / R, (R - I) / U, (P - I) / U,
         (p2r.sum() + r2p.sum()) / S, math.sqrt(((p2r ** 2).sum() + (r2p ** 2).sum()) / S),
         max(p2r.max(), r2p.max())]
    return np.array(m, dtype=np.float64), c
