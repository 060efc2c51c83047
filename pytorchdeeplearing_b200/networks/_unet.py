"""Shared builder of the drop-in UNet3d / UNet2d / UNet3dthin (reference networks/Unet3d.py, Unet2d.py,
Unet3dthin.py)."""
from collections import OrderedDict

import torch.nn as nn

from ._base import SegNetBase


def unet_block(Conv, ci, co, name):
    """(conv3 no-bias -> GroupNorm(8) -> Dropout(.2) -> ReLU) x2, Unet3d.py:65-86 (Unet3dthin.py:64-86 is the same
    block); only the stateful members are registered (dropout / relu carry no state_dict entries)"""
    return nn.Sequential(OrderedDict([
        (name + "conv1", Conv(ci, co, kernel_size=3, padding=1, bias=False)),
        (name + "norm1", nn.GroupNorm(8, co)),
        (name + "conv2", Conv(co, co, kernel_size=3, padding=1, bias=False)),
        (name + "norm2", nn.GroupNorm(8, co)),
    ]))


def unet_mask_channels(f):
    """channels of the 18 dropout calls, in module-call order (two per block: encoders, bottleneck, decoders)"""
    ch = []
    for c in (f, 2 * f, 4 * f, 8 * f, 16 * f, 8 * f, 4 * f, 2 * f, f):
        ch += [c, c]
    return ch


class _UNetBase(SegNetBase):
    _arch = "unet"

    def __init__(self, in_channels, out_channels, init_features=16):
        super().__init__()
        Conv = nn.Conv3d if self._dims == 3 else nn.Conv2d
        ConvT = nn.ConvTranspose3d if self._dims == 3 else nn.ConvTranspose2d
        self.features = f = init_features
        self.in_channels = in_channels
        self.out_channels = out_channels

        def block(ci, co, name):
            return unet_block(Conv, ci, co, name)

        self.encoder1 = block(in_channels, f, "enc1")
        self.encoder2 = block(f, 2 * f, "enc2")
        self.encoder3 = block(2 * f, 4 * f, "enc3")
        self.encoder4 = block(4 * f, 8 * f, "enc4")
        self.bottleneck = block(8 * f, 16 * f, "bottleneck")
        self.upconv4 = ConvT(16 * f, 8 * f, kernel_size=2, stride=2)
        self.decoder4 = block(16 * f, 8 * f, "dec4")
        self.upconv3 = ConvT(8 * f, 4 * f, kernel_size=2, stride=2)
        self.decoder3 = block(8 * f, 4 * f, "dec3")
        self.upconv2 = ConvT(4 * f, 2 * f, kernel_size=2, stride=2)
        self.decoder2 = block(4 * f, 2 * f, "dec2")
        self.upconv1 = ConvT(2 * f, f, kernel_size=2, stride=2)
        self.decoder1 = block(2 * f, f, "dec1")
        self.conv = Conv(f, out_channels, kernel_size=1)
        self._finish_init()

    def _mask_channels(self):
        return unet_mask_channels(self.features)
