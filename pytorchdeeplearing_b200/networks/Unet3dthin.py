"""Drop-in ``UNet3dthin`` (reference networks/Unet3dthin.py:6-86): same ctor, same 56-tensor state_dict.

UNet3d's encoder; each decoder block runs at the coarse resolution of its level and its output is upsampled 2x
(trilinear, align_corners=False) and added to the encoder output -- no transposed convolution, no concat."""
import torch.nn as nn

from ._base import SegNetBase
from ._unet import unet_block, unet_mask_channels


class UNet3dthin(SegNetBase):
    _arch = "unetthin"
    _dims = 3

    def __init__(self, in_channels, out_channels, init_features=16):
        super().__init__()
        self.features = f = init_features
        self.in_channels = in_channels
        self.out_channels = out_channels
        self.encoder1 = unet_block(nn.Conv3d, in_channels, f, "enc1")
        self.encoder2 = unet_block(nn.Conv3d, f, 2 * f, "enc2")
        self.encoder3 = unet_block(nn.Conv3d, 2 * f, 4 * f, "enc3")
        self.encoder4 = unet_block(nn.Conv3d, 4 * f, 8 * f, "enc4")
        self.bottleneck = unet_block(nn.Conv3d, 8 * f, 16 * f, "bottleneck")
        self.decoder4 = unet_block(nn.Conv3d, 16 * f, 8 * f, "dec4")
        self.decoder3 = unet_block(nn.Conv3d, 8 * f, 4 * f, "dec3")
        self.decoder2 = unet_block(nn.Conv3d, 4 * f, 2 * f, "dec2")
        self.decoder1 = unet_block(nn.Conv3d, 2 * f, f, "dec1")
        self.conv = nn.Conv3d(f, out_channels, kernel_size=1)
        self._finish_init()

    def _mask_channels(self):
        return unet_mask_channels(self.features)
