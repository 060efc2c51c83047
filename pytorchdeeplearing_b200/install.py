"""Patch the drop-in into an imported reference tree (SURVEY.md section 8b).

The reference wrappers bind the classes at import time (``from networks.VNet3d import VNet3d``
model/modelVNet.py:2-4, model/modelUnet.py:2-4; losses model/modelVNet.py:7-8), so ``install``
rebinds those names in whichever of ``networks``, ``networks.*``, ``model.modelVNet``,
``model.modelUnet``, ``model.modelResNet``, ``model.losses``, ``model.metric``, ``model.lossesSSIM`` are already imported (and in ``sys.modules`` entries
imported later via the same names).  ``uninstall`` restores the originals.
"""
from __future__ import annotations

import sys

_SAVED = []

_NET_NAMES = ("VNet3d", "VNet2d", "UNet3d", "UNet2d", "ResNet2d", "ResNet3d")
_METRIC_NAMES = ("dice_coeff", "iou_coeff", "multiclass_dice_coeff", "multiclass_iou_coeff", "Seg_Metirc3d")
_LOSS_NAMES = ("BinaryDiceLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss", "BinaryCrossEntropyDiceLoss",
               "MutilCrossEntropyLoss", "MutilFocalLoss", "MutilDiceLoss", "MutilCrossEntropyDiceLoss")
# the further model/losses.py classes (bound there, not imported by the wrappers)
_EXT_LOSS_NAMES = ("BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss", "MutilELDiceLoss",
                   "LovaszLoss")
# model/lossesSSIM.py
_SSIM_NAMES = ("SSIM", "SSIM3D", "ssim", "ssim3D")
_MODULES = ("networks", "networks.VNet3d", "networks.VNet2d", "networks.Unet3d", "networks.Unet2d", "model",
            "model.losses", "model.metric", "model.modelVNet", "model.modelUnet", "model.lossesSSIM",
            "networks.ResNet2d", "networks.ResNet3d", "model.modelResNet")


def install() -> int:
    """Rebind the reference's names to the drop-in implementations. Returns the number of bindings changed."""
    from . import networks as nets, losses, metric
    from .ssim import SSIM, SSIM3D, ssim, ssim3D       # the package's ``ssim`` attribute is the function, not the module
    table = {n: getattr(nets, n) for n in _NET_NAMES}
    table.update({n: getattr(losses, n) for n in _LOSS_NAMES + _EXT_LOSS_NAMES})
    table.update({n: getattr(metric, n) for n in _METRIC_NAMES})     # per-step accuracy, model/modelVNet.py:582
    table.update(zip(_SSIM_NAMES, (SSIM, SSIM3D, ssim, ssim3D)))
    count = 0
    for modname in _MODULES:
        mod = sys.modules.get(modname)
        if mod is None:
            continue
        for name, obj in table.items():
            if hasattr(mod, name) and getattr(mod, name) is not obj:
                _SAVED.append((mod, name, getattr(mod, name)))
                setattr(mod, name, obj)
                count += 1
    return count


def uninstall() -> None:
    while _SAVED:
        mod, name, obj = _SAVED.pop()
        setattr(mod, name, obj)
