"""Drop-in per-step accuracy functions of the reference ``model/metric.py:146-181`` (called every training /
validation step: model/modelVNet.py:582, modelUnet.py:136,166): ONE pass over ``probs`` + labels producing the
per-sample threshold counts (``b200seg_metric_partials``) and a scalar finalize, instead of ~8 elementwise / reduce
launches and an int64 one-hot tensor.  (Inside a training step the same numbers come for free from the loss pass:
``lossfn.last_dice()`` / ``GraphedStep.dice`` -- SURVEY.md 8f-2.)

The evaluation metrics of ``Seg_Metirc3d`` (model/metric.py:11-142: Dice, Jaccard, VOE, RVD, FNR, FPR, ASSD, RMSD,
MSD) run on ``b200seg_segmetric3d``: ``seg_metrics3d`` is the device-side functional form, ``Seg_Metirc3d`` the
reference's class.
"""
from __future__ import annotations

import numpy as np
import torch

from . import runtime


def _channels_last(t: torch.Tensor) -> torch.Tensor:
    """(N, C, *spatial) -> contiguous (N, *spatial, C) fp32 (free for the tensors the drop-in networks return)"""
    perm = (0,) + tuple(range(2, t.dim())) + (1,)
    t = t.detach().permute(*perm)
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


def _sums(input: torch.Tensor, target: torch.Tensor, binary: bool) -> torch.Tensor:
    if binary:
        n = target.size(0)
        p = input.detach().reshape(n, -1, 1)                     # dice_coeff views (num, -1): metric.py:150
        if p.dtype != torch.float32:
            p = p.float()
        p = p.contiguous()
        t = target.detach().reshape(n, -1)
        t = t.float() if t.is_floating_point() else t.long()
        c = 1
    else:
        p = _channels_last(input)
        n, c = p.shape[0], p.shape[-1]
        t = target.detach().long()
    t = t.contiguous()
    metric = torch.zeros(n, c, 3, dtype=torch.float64, device=p.device)
    runtime.get_backend(p).metric_partials(p, t, 0.5, metric)
    return metric


def _finish(metric: torch.Tensor, which: int) -> torch.Tensor:
    out = torch.empty(2, dtype=torch.float32, device=metric.device)
    runtime.get_backend(metric).metric_finalize(metric, out)
    return out[which]


def dice_coeff(input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """reference model/metric.py:146-155: per-sample Dice of ``input > 0.5`` against ``target``, batch mean"""
    return _finish(_sums(input, target, True), 0)


def iou_coeff(input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """reference model/metric.py:158-167"""
    return _finish(_sums(input, target, True), 1)


def multiclass_dice_coeff(input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """reference model/metric.py:170-181: mean over the non-background classes of ``dice_coeff`` on each class's
    probability map (threshold 0.5) against the one-hot labels"""
    if input.shape[1] < 2:
        raise ValueError("multiclass_dice_coeff needs at least two classes")
    return _finish(_sums(input, target, False), 0)


def multiclass_iou_coeff(input: torch.Tensor, target: torch.Tensor) -> torch.Tensor:
    """the IoU analogue (reference model/metric.py:205-216; its ``assert input.size() == target.size()`` makes the
    original unusable with index labels -- the formula is the one of ``iou_coeff`` per class)"""
    if input.shape[1] < 2:
        raise ValueError("multiclass_iou_coeff needs at least two classes")
    return _finish(_sums(input, target, False), 1)


# ---------------------------------------------------------------------------------------------------------------------
# 3-D segmentation metrics: Seg_Metirc3d (reference model/metric.py:11-142) on b200seg_segmetric3d
# ---------------------------------------------------------------------------------------------------------------------
_MASK_DTYPES = (torch.bool, torch.uint8, torch.int32, torch.int64)
METRIC_NAMES = ("dice", "jaccard", "VOE", "RVD", "FNR", "FPR", "ASSD", "RMSD", "MSD")
COUNT_NAMES = ("R", "P", "I", "U", "S_r", "S_p")


def _spacing_zyx(voxel_spacing, n: int) -> np.ndarray:
    """SimpleITK (x, y, z) spacing, one triple or one per volume -> validated fp64 (n, 3) in (z, y, x) order
    (metric.py:47 reverses it)"""
    sp = np.asarray(voxel_spacing, dtype=np.float64)
    if sp.shape == (3,):
        sp = np.broadcast_to(sp, (n, 3))
    if sp.shape != (n, 3):
        raise ValueError(f"voxel_spacing must be 3 values (x, y, z) or one triple per volume, got shape {sp.shape}")
    if not (np.isfinite(sp).all() and (sp > 0).all()):
        raise ValueError(f"voxel_spacing must be positive and finite, got {sp.tolist()}")
    return np.ascontiguousarray(sp[:, ::-1])


def _upload_spacing(be, sp_zyx: np.ndarray, device) -> torch.Tensor:
    """host spacing -> device fp64 (n, 3) through kernel arguments, so the call stays capturable in a CUDA graph"""
    return be.upload_bytes(sp_zyx.tobytes(), device).view(torch.float64)[:sp_zyx.size].view(-1, 3)


def _launch(real: torch.Tensor, pred: torch.Tensor, voxel_spacing, counts, metrics, flags):
    be = runtime.get_backend(real)
    sp = _upload_spacing(be, _spacing_zyx(voxel_spacing, real.shape[0]), real.device)
    be.segmetric3d(real, pred, sp, counts, metrics, flags)
    return be, sp


def seg_metrics3d(real: torch.Tensor, pred: torch.Tensor, voxel_spacing):
    """The nine metrics of Seg_Metirc3d for device masks of shape (D, H, W) or (N, D, H, W): nonzero is foreground,
    no value check.  ``voxel_spacing``: host (x, y, z), or an (N, 3) array with one spacing per volume.
    -> (metrics fp64 (..., 9) in Seg_Metirc3d's order: dice, jaccard, VOE, RVD, FNR, FPR, ASSD, RMSD, MSD;
        counts int64 (..., 6): R, P, I, U, S_r, S_p).  Both stay on the device; nothing synchronises, so the call can
    be captured in a CUDA graph and takes ``predict_mask`` / ``sliding_window_mask`` output as it is.  Distance metrics
    are NaN where a mask is empty; overlap metrics then follow IEEE division."""
    if real.shape != pred.shape or real.dim() not in (3, 4):
        raise ValueError(f"expected two masks of one shape (D, H, W) or (N, D, H, W), got {tuple(real.shape)} and "
                         f"{tuple(pred.shape)}")
    if real.dtype not in _MASK_DTYPES or pred.dtype not in _MASK_DTYPES:
        raise TypeError(f"masks must be bool, uint8, int32 or int64, got {real.dtype} / {pred.dtype}")
    batched = real.dim() == 4
    r = (real if batched else real.unsqueeze(0)).contiguous()
    p = (pred if batched else pred.unsqueeze(0)).contiguous()
    n = r.shape[0]
    counts = torch.empty((n, 6), dtype=torch.int64, device=r.device)
    metrics = torch.empty((n, 9), dtype=torch.float64, device=r.device)
    flags = torch.empty(n, dtype=torch.int32, device=r.device)
    _launch(r, p, voxel_spacing, counts, metrics, flags)
    return (metrics, counts) if batched else (metrics[0], counts[0])


def _mask_tensor(m, device) -> torch.Tensor:
    """a reference-style mask (numpy array or tensor) -> contiguous device tensor; bool / uint8 arrays go over as one
    byte per voxel, int32 / int64 as they are (a narrowing copy could hide values outside {0, 1})"""
    if isinstance(m, torch.Tensor):
        t = m.detach()
    else:
        a = np.ascontiguousarray(m)
        if a.dtype == np.bool_:
            a = a.view(np.uint8)
        elif a.dtype.kind in "iu" and a.dtype not in (np.uint8, np.int32, np.int64):
            a = a.astype(np.int64)
        t = torch.from_numpy(a)
    if t.dtype not in _MASK_DTYPES:
        raise TypeError(f"Seg_Metirc3d takes bool or integer masks, got {t.dtype}")
    return t.to(device).contiguous()


class Seg_Metirc3d:
    """Drop-in for the reference's ``Seg_Metirc3d(real_mask, pred_mask, voxel_spacing)`` (model/metric.py:11-142; the
    name's spelling is the reference's): nine overlap and surface-distance metrics of two 3-D binary masks, computed on
    the GPU in the constructor with one launch sequence and one host read.

    Masks are numpy arrays (copied to the current CUDA device) or CUDA tensors, of shape (D, H, W); ``voxel_spacing``
    is the SimpleITK (x, y, z) spacing.  Surface distances are exact (a separable Euclidean distance transform in
    fp64), equal to the reference's cKDTree distances up to rounding.  Two deliberate differences:
      - uint8 masks: the reference's RVD subtracts unsigned sums and wraps around when pred is smaller than real; here
        RVD is the signed (P - R) / R for every dtype;
      - values outside {0, 1} (a 0/255 ``predict`` mask): the reference's XOR of the eroded uint8 mask and the mask
        returns meaningless metrics; here the constructor raises ValueError -- binarise first.
    An empty mask raises ValueError, as in the reference's constructor.
    ``real_mask_surface_pts`` / ``pred_mask_surface_pts`` / ``real2pred_nn`` / ``pred2real_nn`` are computed on first
    access (a second launch sequence), with the reference's shapes, order and dtypes."""

    def __init__(self, real_mask, pred_mask, voxel_spacing):
        self.real_mask = real_mask
        self.pred_mask = pred_mask
        self.voxel_sapcing = voxel_spacing
        device = next((m.device for m in (real_mask, pred_mask) if isinstance(m, torch.Tensor) and m.is_cuda), None)
        if device is None:
            device = torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else "cpu"
        r, p = _mask_tensor(real_mask, device), _mask_tensor(pred_mask, device)
        if r.dim() != 3 or p.shape != r.shape:
            raise ValueError(f"Seg_Metirc3d takes two 3-D masks of one shape, got {tuple(r.shape)} and "
                             f"{tuple(p.shape)}")
        self._shape = tuple(r.shape)
        self._r, self._p = r.unsqueeze(0), p.unsqueeze(0)
        # one int64 row: counts [0:6], metrics [6:15] (fp64 bits), flag [15] -> a single device-to-host copy
        buf = torch.empty((1, 16), dtype=torch.int64, device=r.device)
        be, self._sp = _launch(self._r, self._p, voxel_spacing, buf[0, 0:6], buf[0, 6:15].view(torch.float64),
                               buf[0, 15:16].view(torch.int32))
        self._be = be
        host = buf.cpu()[0]
        if int(host[15:16].view(torch.int32)[0]) != 0:
            raise ValueError("Seg_Metirc3d: a mask holds values other than 0 and 1 (e.g. a 0/255 predict mask); "
                             "binarise it first, e.g. mask != 0")
        self._counts = [int(v) for v in host[0:6]]
        R, P = self._counts[0], self._counts[1]
        if R == 0 or P == 0:
            raise ValueError(f"Seg_Metirc3d: empty {'real' if R == 0 else 'pred'} mask: surface distances are "
                             "undefined")
        self._m = host[6:15].clone().view(torch.float64).numpy()
        self._pts = None

    # ------------------------------------------------------------------ lazily computed surface points / distances
    def _points(self):
        if self._pts is None:
            Sr, Sp = self._counts[4], self._counts[5]
            dev = self._r.device
            ri = torch.empty(Sr, dtype=torch.int64, device=dev)
            pi = torch.empty(Sp, dtype=torch.int64, device=dev)
            rn = torch.empty(Sr, dtype=torch.float64, device=dev)
            pn = torch.empty(Sp, dtype=torch.float64, device=dev)
            self._be.segmetric3d_points(self._r, self._p, self._sp, ri, pi, rn, pn)
            self._pts = tuple(t.cpu().numpy() for t in (ri, pi, rn, pn))
        return self._pts

    def _surface_pts(self, idx):
        pts = np.array(np.unravel_index(idx, self._shape)).T.reshape(-1, 3)
        return pts * np.array(self.voxel_sapcing[::-1]).reshape(1, 3)          # metric.py:43-47

    @property
    def real_mask_surface_pts(self):
        return self._surface_pts(self._points()[0])

    @property
    def pred_mask_surface_pts(self):
        return self._surface_pts(self._points()[1])

    @property
    def real2pred_nn(self):
        return self._points()[2]

    @property
    def pred2real_nn(self):
        return self._points()[3]

    # ------------------------------------------------------------------ the nine metrics (metric.py:68-142)
    def get_dice_coefficient(self):
        R, P, I = self._counts[0:3]
        return np.float64(self._m[0]), np.int64(2 * I), np.int64(R + P)

    def get_jaccard_index(self):
        return np.float64(self._m[1])

    def get_VOE(self):
        return np.float64(self._m[2])

    def get_RVD(self):
        return float(self._m[3])

    def get_FNR(self):
        return np.float64(self._m[4])

    def get_FPR(self):
        return np.float64(self._m[5])

    def get_ASSD(self):
        return np.float64(self._m[6])

    def get_RMSD(self):
        return float(self._m[7])

    def get_MSD(self):
        return np.float64(self._m[8])


__all__ = ["dice_coeff", "iou_coeff", "multiclass_dice_coeff", "multiclass_iou_coeff", "seg_metrics3d", "Seg_Metirc3d"]
