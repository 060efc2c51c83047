"""numpy / scipy restatement of the reference's mask post-processing (dataprocess/utils.py:7-66), the oracle of
``pytorchdeeplearing_b200.postprocess``.  SimpleITK is not used; the ITK semantics restated here are:
  - ConnectedComponent (fullyConnected=False): face connectivity, labels in raster order of each component's first
    voxel (scipy's ``ndimage.label`` numbers components in the same order);
  - the default sitkBall of radius r: {d : sum d^2 <= r^2 + r} (FlatStructuringElement::Ball, axes 2r + 1);
  - BinaryDilate: outside is background; BinaryErode: outside is foreground (BoundaryToForeground);
    BinaryMorphologicalClosing: SafeBorder pads by r with background.
Masks are numpy arrays (H, W) or (D, H, W)."""
import numpy as np
from scipy import ndimage

OPS = ("dilate", "erode", "open", "close")


def ball(r: int, dims: int) -> np.ndarray:
    g = np.indices((2 * r + 1,) * dims) - r
    return (g ** 2).sum(axis=0) <= r * r + r


def largest_component(mask: np.ndarray):
    """-> (uint8 mask of the component with the most voxels, ties to the first in C order; number of components;
    voxels of the largest).  All zero without foreground."""
    fg = mask != 0
    lab, n = ndimage.label(fg, structure=ndimage.generate_binary_structure(fg.ndim, 1))
    if n == 0:
        return np.zeros(fg.shape, np.uint8), 0, 0
    counts = np.bincount(lab.ravel())[1:]
    k = int(np.argmax(counts))                  # the first maximum: the component whose first voxel comes first
    return (lab == k + 1).astype(np.uint8), int(n), int(counts[k])


def _dilate(fg, se):
    return ndimage.binary_dilation(fg, structure=se, border_value=0)


def _erode(fg, se):
    return ndimage.binary_erosion(fg, structure=se, border_value=1)


def morphology(mask: np.ndarray, r: int, op: str) -> np.ndarray:
    """MorphologicalOperation(mask, r, op) on ``mask != 0`` -> uint8 0/1, with the ball over the mask's own axes"""
    fg = mask != 0
    se = ball(r, fg.ndim)
    if op == "dilate":
        out = _dilate(fg, se)
    elif op == "erode":
        out = _erode(fg, se)
    elif op == "open":
        out = _dilate(_erode(fg, se), se)
    elif op == "close":
        p = np.pad(fg, r)
        out = _erode(_dilate(p, se), se)[tuple(slice(r, r + s) for s in fg.shape)]
    else:
        raise ValueError(op)
    return out.astype(np.uint8)


def label_bbox(mask: np.ndarray) -> np.ndarray:
    """LabelShapeStatisticsImageFilter.GetBoundingBox(1) in ITK's (x, y, [z]) order followed by the count of voxels
    equal to 1; zeros and count 0 when there is none"""
    idx = np.argwhere(mask == 1)[:, ::-1]       # (x, y, z)
    dims = mask.ndim
    if len(idx) == 0:
        return np.zeros(2 * dims + 1, np.int64)
    lo, hi = idx.min(axis=0), idx.max(axis=0)
    return np.concatenate([lo, hi - lo + 1, [len(idx)]]).astype(np.int64)
