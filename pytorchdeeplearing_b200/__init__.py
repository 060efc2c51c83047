"""pytorchdeeplearing_b200 -- H100-native (sm_90a) drop-in for the segmentation hot path of
junqiangchen/PytorchDeepLearing: ``networks/VNet3d.py``, ``networks/Unet3d.py``,
``networks/Unet2d.py`` forward/backward, the ``networks/ResNet3d.py`` / ``ResNet2d.py`` classifiers and the losses of ``model/losses.py`` (Dice / BCE / focal / CE,
Jaccard / Tversky / sensitivity-specificity / exponential-log Dice and Lovasz-Softmax) (SURVEY.md section 8), and the
3-D evaluation metrics of ``model/metric.py`` (``Seg_Metirc3d``, ``seg_metrics3d``) and the SSIM losses of
``model/lossesSSIM.py`` (``SSIM``, ``SSIM3D``, ``ssim``, ``ssim3D``), and the whole-volume 3-D inference of
``XModel.inference`` / ``inference_patch`` with its resamples and normalisations (``inference3d``,
``inference_patch3d``).

    from pytorchdeeplearing_b200 import VNet3d, MutilDiceLoss      # same ctor signatures
    import pytorchdeeplearing_b200 as b200; b200.install()         # or patch the reference in place

Host code is Python/PyTorch (device memory, streams, torch.distributed); every FLOP runs in
hand-written CUDA kernels behind the C ABI of ``include/b200seg.h``.
"""
from .runtime import (set_precision, get_precision, enable_data_parallel, disable_data_parallel)
from .networks import VNet3d, VNet2d, UNet3d, UNet2d, ResNet3d, ResNet2d, initialize_weights
from .losses import (BinaryDiceLoss, BinaryCrossEntropyLoss, BinaryFocalLoss, BinaryCrossEntropyDiceLoss,
                     BinaryDiceFocalLoss, MutilCrossEntropyLoss, MutilFocalLoss, MutilDiceLoss,
                     MutilCrossEntropyDiceLoss, BinaryJaccardLoss, BinaryELDiceLoss, BinarySSLoss, BinaryTverskyLoss,
                     MutilELDiceLoss, LovaszLoss)
from .install import install, uninstall
from .graphed import GraphedStep
from .optim import FusedAdamW, FusedAdam
from .metric import dice_coeff, iou_coeff, multiclass_dice_coeff, multiclass_iou_coeff, seg_metrics3d, Seg_Metirc3d
from .inference import (predict, predict_mask, sliding_window_mask, inference3d, inference_patch3d, resample3d,
                        spacing_size)
from .staging import InputStager, stage_batch
from .ssim import SSIM, SSIM3D, ssim, ssim3D

__all__ = ["VNet3d", "VNet2d", "UNet3d", "UNet2d", "ResNet3d", "ResNet2d", "initialize_weights", "FusedAdamW", "FusedAdam", "dice_coeff",
           "iou_coeff", "multiclass_dice_coeff", "multiclass_iou_coeff", "seg_metrics3d", "Seg_Metirc3d", "predict",
           "predict_mask",
           "sliding_window_mask", "inference3d", "inference_patch3d", "resample3d", "spacing_size", "InputStager", "stage_batch", "set_precision", "get_precision",
           "enable_data_parallel", "disable_data_parallel", "install", "uninstall", "GraphedStep",
           "BinaryDiceLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss", "BinaryCrossEntropyDiceLoss",
           "BinaryDiceFocalLoss", "MutilCrossEntropyLoss", "MutilFocalLoss", "MutilDiceLoss",
           "MutilCrossEntropyDiceLoss", "BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss",
           "MutilELDiceLoss", "LovaszLoss", "SSIM", "SSIM3D", "ssim", "ssim3D"]
