"""Drop-in ``ResNet2d`` (reference networks/ResNet2d.py:73-119); runs through the 3-D layer program with a unit
depth."""
from ._resnet import _ResNetBase


class ResNet2d(_ResNetBase):
    _dims = 2
