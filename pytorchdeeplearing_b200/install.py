"""Patch the drop-in into an imported reference tree (SURVEY.md section 8b).

The reference wrappers bind the classes at import time (``from networks.VNet3d import VNet3d``
model/modelVNet.py:2-4, model/modelUnet.py:2-4; losses model/modelVNet.py:7-8), so ``install``
rebinds those names in whichever of ``networks``, ``networks.*`` (``networks.Unet3dthin`` and
``networks.VNet3dregistration`` included), ``model.modelVNet``,
``model.modelUnet``, ``model.modelResNet``, ``model.losses``, ``model.metric``, ``model.lossesSSIM``, ``model.lossescldice`` are already imported (and in ``sys.modules`` entries
imported later via the same names).  The mask post-processing functions are rebound in ``dataprocess.utils``, and
``GradCAM`` in ``model.visualization`` and ``model.modelResNet`` (so ``Grad_CAM_Visual`` runs on the GPU).
``ImageDataGenerator3D`` is rebound in ``dataprocess.Augmentation.
images_masks_3dtransform`` and ``dataprocess.Augmentation.ImageAugmentation`` (which binds it at import,
ImageAugmentation.py:1), so an unmodified ``DataAug3D(...).DataAugmentation(...)`` warps on the GPU, and
``Segmenation_Aug`` in ``dataprocess.AugData`` (the 2-D augmentation).  ``uninstall``
restores the originals.
"""
from __future__ import annotations

import sys

_SAVED = []

_NET_NAMES = ("VNet3d", "VNet2d", "UNet3d", "UNet3dthin", "UNet2d", "ResNet2d", "ResNet3d", "VNet3dRegistration")
_METRIC_NAMES = ("dice_coeff", "iou_coeff", "multiclass_dice_coeff", "multiclass_iou_coeff", "Seg_Metirc3d")
_LOSS_NAMES = ("BinaryDiceLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss", "BinaryCrossEntropyDiceLoss",
               "MutilCrossEntropyLoss", "MutilFocalLoss", "MutilDiceLoss", "MutilCrossEntropyDiceLoss")
# the further model/losses.py classes (bound there, not imported by the wrappers)
_EXT_LOSS_NAMES = ("BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss", "MutilELDiceLoss",
                   "LovaszLoss", "BinaryLovaszLoss")
# model/lossesSSIM.py
_SSIM_NAMES = ("SSIM", "SSIM3D", "ssim", "ssim3D")
# model/lossescldice.py
_CLDICE_NAMES = ("soft_skeletonize", "norm_intersection", "Binary_Soft_cldice_loss", "Mutil_Soft_cldice_loss")
# dataprocess/utils.py
_POSTPROCESS_NAMES = ("GetLargestConnectedCompont", "GetLargestConnectedCompontBoundingbox", "MorphologicalOperation")
_MODULES = ("networks", "networks.VNet3d", "networks.VNet2d", "networks.Unet3d", "networks.Unet3dthin", "networks.Unet2d",
            "model",
            "model.losses", "model.metric", "model.modelVNet", "model.modelUnet", "model.lossesSSIM",
            "model.lossescldice", "networks.ResNet2d", "networks.ResNet3d", "model.modelResNet",
            "dataprocess.Augmentation.images_masks_3dtransform", "dataprocess.Augmentation.ImageAugmentation",
            "dataprocess.utils", "model.visualization", "dataprocess.AugData", "networks.VNet3dregistration")


def install() -> int:
    """Rebind the reference's names to the drop-in implementations. Returns the number of bindings changed."""
    from . import networks as nets, losses, metric
    from .ssim import SSIM, SSIM3D, ssim, ssim3D       # the package's ``ssim`` attribute is the function, not the module
    from .augment import ImageDataGenerator3D
    from . import cldice, postprocess
    from .gradcam import GradCAM
    from .augment2d import Segmenation_Aug
    table = {n: getattr(nets, n) for n in _NET_NAMES}
    table.update({n: getattr(losses, n) for n in _LOSS_NAMES + _EXT_LOSS_NAMES})
    table.update({n: getattr(metric, n) for n in _METRIC_NAMES})     # per-step accuracy, model/modelVNet.py:582
    table.update(zip(_SSIM_NAMES, (SSIM, SSIM3D, ssim, ssim3D)))
    table.update({n: getattr(cldice, n) for n in _CLDICE_NAMES})
    table.update({n: getattr(postprocess, n) for n in _POSTPROCESS_NAMES})
    table["ImageDataGenerator3D"] = ImageDataGenerator3D    # dataprocess/Augmentation (DataAug3D)
    table["GradCAM"] = GradCAM                              # model/visualization.py, model/modelResNet.py
    table["Segmenation_Aug"] = Segmenation_Aug              # dataprocess/AugData.py
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
