"""pytorchdeeplearing_b200 -- H100-native (sm_90a) drop-in for the segmentation hot path of
junqiangchen/PytorchDeepLearing: ``networks/VNet3d.py``, ``networks/Unet3d.py``,
``networks/Unet3dthin.py``, ``networks/Unet2d.py`` forward/backward, the ``networks/ResNet3d.py`` / ``ResNet2d.py`` classifiers and the losses of ``model/losses.py`` (Dice / BCE / focal / CE,
Jaccard / Tversky / sensitivity-specificity / exponential-log Dice, Lovasz-Softmax and the binary Lovasz hinge)
(SURVEY.md section 8), and the
3-D evaluation metrics of ``model/metric.py`` (``Seg_Metirc3d``, ``seg_metrics3d``) and the SSIM losses of
``model/lossesSSIM.py`` (``SSIM``, ``SSIM3D``, ``ssim``, ``ssim3D``), the soft-clDice losses of ``model/lossescldice.py``
(``soft_skeletonize``, ``norm_intersection``, ``Binary_Soft_cldice_loss``, ``Mutil_Soft_cldice_loss``; the reference
module raises as shipped, so its evident intent runs here, with four documented repairs), and the whole-volume 3-D inference of
``XModel.inference`` / ``inference_patch`` with its resamples and normalisations (``inference3d``,
``inference_patch3d``), and the 2-D ``XModel.inference`` and datasets' bit-exact cv2 bilinear resize (``inference2d``,
``resize2d``, ``InputStager(max_source_pixels=...)``), and the 3-D data augmentation of
``dataprocess/Augmentation`` (``ImageDataGenerator3D``: scipy's order-0 affine warp bit for bit, offline through
``DataAug3D`` or per training step through ``transform_batch``), and the mask post-processing of ``dataprocess/utils.py``
(``largest_component``, ``binary_morphology``, ``label_bbox`` and the reference-named ``GetLargestConnectedCompont``,
``MorphologicalOperation``, ``GetLargestConnectedCompontBoundingbox``), and Grad-CAM of ResNet2d
(``grad_cam`` and the reference-named ``GradCAM`` of ``model/visualization.py``), and the 2-D data augmentation of
``dataprocess/AugData.py`` (``Segmenation_Aug``: cv2's flips, blurs, warp and table byte for byte, offline through
``DataAugmentation`` or per training step through ``transform_batch`` and ``InputStager(augment=...)``), and
voxelmorph's SpatialTransformer as ``networks/VNet3dregistration.py`` uses it (``warp3d``: the trilinear image and
nearest label warp by a displacement field, with d loss / d ddf).

    from pytorchdeeplearing_b200 import VNet3d, MutilDiceLoss      # same ctor signatures
    import pytorchdeeplearing_b200 as b200; b200.install()         # or patch the reference in place

Host code is Python/PyTorch (device memory, streams, torch.distributed); every FLOP runs in
hand-written CUDA kernels behind the C ABI of ``include/b200seg.h``.
"""
from .runtime import (set_precision, get_precision, enable_data_parallel, disable_data_parallel)
from .networks import (VNet3d, VNet2d, UNet3d, UNet3dthin, UNet2d, ResNet3d, ResNet2d, VNet3dRegistration,
                       initialize_weights)
from .losses import (BinaryDiceLoss, BinaryCrossEntropyLoss, BinaryFocalLoss, BinaryCrossEntropyDiceLoss,
                     BinaryDiceFocalLoss, MutilCrossEntropyLoss, MutilFocalLoss, MutilDiceLoss,
                     MutilCrossEntropyDiceLoss, BinaryJaccardLoss, BinaryELDiceLoss, BinarySSLoss, BinaryTverskyLoss,
                     MutilELDiceLoss, LovaszLoss, BinaryLovaszLoss, lovasz_hinge)
from .install import install, uninstall
from .graphed import GraphedStep
from .optim import FusedAdamW, FusedAdam
from .metric import dice_coeff, iou_coeff, multiclass_dice_coeff, multiclass_iou_coeff, seg_metrics3d, Seg_Metirc3d
from .inference import (predict, predict_mask, sliding_window_mask, inference3d, inference_patch3d, resample3d,
                        spacing_size, resize2d, inference2d)
from .staging import InputStager, stage_batch
from .ssim import SSIM, SSIM3D, ssim, ssim3D
from .augment import ImageDataGenerator3D
from .cldice import soft_skeletonize, norm_intersection, Binary_Soft_cldice_loss, Mutil_Soft_cldice_loss
from .postprocess import (largest_component, binary_morphology, label_bbox, GetLargestConnectedCompont,
                          MorphologicalOperation, GetLargestConnectedCompontBoundingbox)
from .gradcam import grad_cam, GradCAM
from .augment2d import Segmenation_Aug
from .warp import warp3d

__all__ = ["VNet3d", "VNet2d", "UNet3d", "UNet3dthin", "UNet2d", "ResNet3d", "ResNet2d", "VNet3dRegistration", "initialize_weights", "FusedAdamW", "FusedAdam", "dice_coeff",
           "iou_coeff", "multiclass_dice_coeff", "multiclass_iou_coeff", "seg_metrics3d", "Seg_Metirc3d", "predict",
           "predict_mask",
           "sliding_window_mask", "inference3d", "inference_patch3d", "resample3d", "spacing_size", "resize2d", "inference2d", "ImageDataGenerator3D", "InputStager", "stage_batch", "set_precision", "get_precision",
           "enable_data_parallel", "disable_data_parallel", "install", "uninstall", "GraphedStep",
           "BinaryDiceLoss", "BinaryCrossEntropyLoss", "BinaryFocalLoss", "BinaryCrossEntropyDiceLoss",
           "BinaryDiceFocalLoss", "MutilCrossEntropyLoss", "MutilFocalLoss", "MutilDiceLoss",
           "MutilCrossEntropyDiceLoss", "BinaryJaccardLoss", "BinaryELDiceLoss", "BinarySSLoss", "BinaryTverskyLoss",
           "MutilELDiceLoss", "LovaszLoss", "BinaryLovaszLoss", "lovasz_hinge", "SSIM", "SSIM3D", "ssim", "ssim3D",
           "soft_skeletonize", "norm_intersection", "Binary_Soft_cldice_loss", "Mutil_Soft_cldice_loss",
           "largest_component", "binary_morphology", "label_bbox", "GetLargestConnectedCompont",
           "MorphologicalOperation", "GetLargestConnectedCompontBoundingbox", "grad_cam", "GradCAM", "Segmenation_Aug",
           "warp3d"]
