"""Drop-in mask post-processing of the reference's ``dataprocess/utils.py:7-66`` (SimpleITK on the CPU there), on
``b200seg_largest_component`` / ``b200seg_morphology`` / ``b200seg_label_bbox`` (csrc/postprocess.cu).

Device forms take CUDA tensors (H, W) or (D, H, W) and never synchronise, so they can be captured in a CUDA graph and
take ``predict_mask`` / ``inference3d`` output as it is:
  - ``largest_component(mask)`` -> (uint8 mask, int64 (2,) = {components, voxels of the largest});
  - ``binary_morphology(mask, radius, op)`` -> uint8 mask, op one of "open", "close", "dilate", "erode";
  - ``label_bbox(mask)`` -> int64 (2 dims + 1): ITK's box of the voxels equal to 1 and their count.
The reference-named functions take a SimpleITK image or a numpy array and return the same kind, on the current CUDA
device: ``GetLargestConnectedCompont``, ``MorphologicalOperation``, ``GetLargestConnectedCompontBoundingbox``.
"""
from __future__ import annotations

import numpy as np
import torch

from . import runtime
from ._abi import MORPH_MAX_RADIUS, MORPH_OPS
from .inference import _as_result, _is_sitk

_MASK_DTYPES = (torch.bool, torch.uint8, torch.int16, torch.int32, torch.int64)
_MORPH_DTYPES = _MASK_DTYPES + (torch.float32,)
# numpy integer dtypes passed to the device as the same-width type the kernels read: a reinterpretation that keeps
# which values are 0 and which are 1
_NP_VIEW = {np.dtype(np.int8): np.uint8, np.dtype(np.uint16): np.int16, np.dtype(np.uint32): np.int32,
            np.dtype(np.uint64): np.int64}


def _check(mask: torch.Tensor, dtypes, what: str, pad: int = 0) -> torch.Tensor:
    if mask.dim() not in (2, 3):
        raise ValueError(f"{what}: expected a (H, W) or (D, H, W) mask, got shape {tuple(mask.shape)}")
    if mask.dtype not in dtypes:
        raise TypeError(f"{what}: mask dtype must be one of {', '.join(str(d)[6:] for d in dtypes)}, got {mask.dtype}")
    if mask.numel() == 0:
        raise ValueError(f"{what}: empty mask {tuple(mask.shape)}")
    if int(np.prod([s + 2 * pad for s in mask.shape], dtype=np.int64)) >= 2 ** 31:
        raise ValueError(f"{what}: {tuple(mask.shape)}{' padded by %d' % pad if pad else ''} is 2^31 voxels or more")
    return mask.contiguous()


def largest_component(mask: torch.Tensor):
    """The face-connected component (6 neighbours in 3-D, 4 in 2-D) of ``mask != 0`` with the most voxels; on a tie
    the one whose first voxel comes first in C order (ITK's raster-order labels).  -> (uint8 mask of mask's shape,
    int64 (2,) = {number of components, voxels in the largest}); an empty mask gives zeros."""
    m = _check(mask, _MASK_DTYPES, "largest_component")
    out = torch.empty(m.shape, dtype=torch.uint8, device=m.device)
    stats = torch.empty(2, dtype=torch.int64, device=m.device)
    runtime.get_backend(m).largest_component(m, out, stats)
    return out, stats


def _radius(radius) -> int:
    if isinstance(radius, (bool, np.bool_)) or not isinstance(radius, (int, np.integer)):
        raise TypeError(f"radius must be an integer, got {radius!r}")
    r = int(radius)
    if not 0 <= r <= MORPH_MAX_RADIUS:
        raise ValueError(f"radius must be in [0, {MORPH_MAX_RADIUS}], got {r}")
    return r


def binary_morphology(mask: torch.Tensor, radius: int, op: str) -> torch.Tensor:
    """``op`` ("open", "close", "dilate", "erode") of ``mask != 0`` with ITK's ball of ``radius`` (the offsets d with
    |d|^2 <= r^2 + r over the mask's axes).  Dilation treats outside the mask as background, erosion as foreground;
    open = dilate(erode); close pads by ``radius`` with background, dilates, erodes and crops.  -> uint8 0/1 mask."""
    if op not in MORPH_OPS:
        raise ValueError(f"op must be one of {', '.join(MORPH_OPS)}, got {op!r}")
    r = _radius(radius)
    m = _check(mask, _MORPH_DTYPES, "binary_morphology", r if op == "close" else 0)
    out = torch.empty(m.shape, dtype=torch.uint8, device=m.device)
    runtime.get_backend(m).morphology(m, r, MORPH_OPS[op], out)
    return out


def label_bbox(mask: torch.Tensor) -> torch.Tensor:
    """``LabelShapeStatisticsImageFilter.GetBoundingBox(1)`` of the voxels equal to 1, in ITK's order
    (x0, y0, [z0,] size x, size y, [size z]), followed by their count: int64 (2 dims + 1); all zero when no voxel
    equals 1."""
    m = _check(mask, _MASK_DTYPES, "label_bbox")
    box = torch.empty(2 * m.dim() + 1, dtype=torch.int64, device=m.device)
    runtime.get_backend(m).label_bbox(m, box)
    return box


# ------------------------------------------------------------------------------------------ reference-named forms
def _host_mask(image, what: str, allow_float: bool):
    """SimpleITK image or numpy array -> (contiguous numpy mask in a dtype the kernels read, geometry or None)"""
    geom = None
    if _is_sitk(image):
        import SimpleITK as sitk
        geom = (tuple(image.GetOrigin()), tuple(image.GetSpacing()), tuple(image.GetDirection()))
        arr = sitk.GetArrayFromImage(image)
    else:
        arr = image
    arr = np.ascontiguousarray(arr)
    if arr.dtype in _NP_VIEW:
        arr = arr.view(_NP_VIEW[arr.dtype])
    elif arr.dtype.kind == "f" and allow_float and arr.dtype != np.float32:
        arr = (arr != 0).view(np.uint8)            # ITK's != 0, NaN included
    elif arr.dtype.kind not in "biuf" or (arr.dtype.kind == "f" and not allow_float):
        raise TypeError(f"{what}: unsupported pixel type {arr.dtype}")
    if arr.ndim not in (2, 3):
        raise ValueError(f"{what}: expected a 2-D or 3-D image, got shape {arr.shape}")
    return arr, geom


def _device():
    return torch.device("cuda", torch.cuda.current_device())


def GetLargestConnectedCompont(binarysitk_image):
    """Drop-in for the reference's ``GetLargestConnectedCompont`` (dataprocess/utils.py:19-44; the spelling is the
    reference's): the largest face-connected component of the nonzero voxels as a uint32 0/1 image (SimpleITK with
    the input's geometry, or numpy).  As in the reference, a mask without foreground gives an image of all ones."""
    arr, geom = _host_mask(binarysitk_image, "GetLargestConnectedCompont", False)
    out, stats = largest_component(torch.from_numpy(arr).to(_device()))
    if int(stats[0]) == 0:
        mask = np.ones(arr.shape, np.uint32)       # utils.py:38-39 with maxlabel 0: cc == 0 everywhere
    else:
        mask = out.cpu().numpy().astype(np.uint32)
    return _as_result(mask, geom)


def MorphologicalOperation(sitk_maskimg, kernelsize, name="open"):
    """Drop-in for the reference's ``MorphologicalOperation`` (dataprocess/utils.py:47-66): ``name`` in "open",
    "close", "dilate", "erode" of ``image != 0`` with the ball of radius ``kernelsize`` -> uint8 0/1 image (SimpleITK
    with the input's geometry, or numpy); any other name returns None.  Radii above 64 raise ValueError."""
    if name not in MORPH_OPS:
        return None
    r = _radius(kernelsize)
    arr, geom = _host_mask(sitk_maskimg, "MorphologicalOperation", True)
    out = binary_morphology(torch.from_numpy(arr).to(_device()), r, name)
    return _as_result(out.cpu().numpy(), geom)


def GetLargestConnectedCompontBoundingbox(binarysitk_image):
    """Drop-in for the reference's ``GetLargestConnectedCompontBoundingbox`` (dataprocess/utils.py:7-16): the box of
    the voxels equal to 1 (of the image itself, not of its largest component) as ``np.array([x0, y0, z0, sx, sy,
    sz])`` (4 values in 2-D).  No voxel equal to 1 (e.g. a 0/255 mask) raises RuntimeError, as SimpleITK does."""
    arr, _ = _host_mask(binarysitk_image, "GetLargestConnectedCompontBoundingbox", False)
    box = label_bbox(torch.from_numpy(arr).to(_device())).cpu().numpy()
    if box[-1] == 0:
        raise RuntimeError("GetLargestConnectedCompontBoundingbox: no voxel has label 1")
    return np.array(box[:-1], dtype=np.int64)


__all__ = ["largest_component", "binary_morphology", "label_bbox", "GetLargestConnectedCompont",
           "MorphologicalOperation", "GetLargestConnectedCompontBoundingbox"]
