"""Drop-in ``ResNet3d`` (reference networks/ResNet3d.py:72-118)."""
from ._resnet import _ResNetBase


class ResNet3d(_ResNetBase):
    _dims = 3
