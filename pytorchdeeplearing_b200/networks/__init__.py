"""Mirror of the reference ``networks`` package for the hot path (networks/__init__.py:1-26)."""
from torch import nn

from .Unet2d import UNet2d
from .Unet3d import UNet3d
from .VNet3d import VNet3d
from .VNet2d import VNet2d
from .ResNet2d import ResNet2d
from .ResNet3d import ResNet3d


def initialize_weights(net):
    """Same dispatch and initialisers as the reference's ``initialize_weights``
    (networks/__init__.py:11-26); used via ``model.apply(initialize_weights)``."""
    convs = (nn.Conv3d, nn.Conv2d, nn.ConvTranspose3d, nn.ConvTranspose2d)
    norms = (nn.BatchNorm1d, nn.BatchNorm2d, nn.BatchNorm3d, nn.GroupNorm)
    if isinstance(net, convs):
        nn.init.kaiming_normal_(net.weight.data, nonlinearity="relu")
        if net.bias is not None:
            nn.init.constant_(net.bias.data, 0)
    elif isinstance(net, norms):
        nn.init.constant_(net.weight.data, 1)
        if net.bias is not None:
            nn.init.constant_(net.bias.data, 0)
    elif isinstance(net, nn.Linear):
        nn.init.kaiming_uniform_(net.weight.data)
        nn.init.constant_(net.bias.data, 0)


__all__ = ["UNet2d", "UNet3d", "VNet3d", "VNet2d", "ResNet2d", "ResNet3d", "initialize_weights"]
