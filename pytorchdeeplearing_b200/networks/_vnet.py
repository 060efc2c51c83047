"""Shared builder of the drop-in VNet3d / VNet2d (reference networks/VNet3d.py:102-158 and its 2-D twin
networks/VNet2d.py:102-160): same constructor signature, same ``state_dict`` (128 tensors, SURVEY.md App. A),
forward/backward on sm_90a kernels.  The 2-D net runs through the same layer program with a unit depth."""
import torch.nn as nn

from ._base import SegNetBase, _Holder


class _VNetBase(SegNetBase):
    _arch = "vnet"

    def __init__(self, image_channel, numclass, init_features=16):
        super().__init__()
        Conv = nn.Conv3d if self._dims == 3 else nn.Conv2d
        ConvT = nn.ConvTranspose3d if self._dims == 3 else nn.ConvTranspose2d
        self.image_channel = image_channel
        self.numclass = numclass
        self.features = f = init_features

        def lu_stack(nchan, depth):
            # reference: _make_nConv3d -> nn.Sequential of LUConv3d (VNet3d.py:5-22); keys ops.{i}.conv1 / ops.{i}.bn1
            layers = []
            for _ in range(depth):
                lu = _Holder()
                lu.conv1 = Conv(nchan, nchan, kernel_size=3, padding=1)
                lu.bn1 = nn.GroupNorm(8, nchan)
                layers.append(lu)
            return nn.Sequential(*layers)

        self.in_tr = _Holder()                                        # InputTransition3d, VNet3d.py:25-32
        self.in_tr.conv1 = Conv(image_channel, f, kernel_size=3, padding=1)
        self.in_tr.conv2 = Conv(image_channel, f, kernel_size=1)
        self.in_tr.bn1 = nn.GroupNorm(8, f)

        for name, ci, co, n in (("down_tr32", f, 2 * f, 2), ("down_tr64", 2 * f, 4 * f, 3),
                                ("down_tr128", 4 * f, 8 * f, 3), ("down_tr256", 8 * f, 16 * f, 3)):
            blk = _Holder()                                           # DownTransition3d, VNet3d.py:46-53
            blk.down_conv = Conv(ci, co, kernel_size=2, stride=2)
            blk.bn1 = nn.GroupNorm(8, co)
            blk.ops = lu_stack(co, n)
            setattr(self, name, blk)

        for name, ci, co, n in (("up_tr256", 16 * f, 8 * f, 3), ("up_tr128", 8 * f, 4 * f, 3),
                                ("up_tr64", 4 * f, 2 * f, 2), ("up_tr32", 2 * f, f, 1)):
            blk = _Holder()                                           # UpTransition3d, VNet3d.py:62-70
            blk.up_conv = ConvT(ci, co, kernel_size=2, stride=2)
            blk.bn = nn.GroupNorm(8, co)
            blk.ops = lu_stack(co, n)
            blk.conv = Conv(ci, co, kernel_size=1)
            setattr(self, name, blk)

        self.out_tr = _Holder()                                       # OutputTransition3d, VNet3d.py:83-88
        self.out_tr.conv = Conv(f, numclass, kernel_size=1)
        self._finish_init()

    def _mask_channels(self):
        f = self.features
        ch = [f, f]
        for co, n in ((2 * f, 2), (4 * f, 3), (8 * f, 3), (16 * f, 3)):
            ch += [co] * (1 + n)
        for co, n in ((8 * f, 3), (4 * f, 3), (2 * f, 2), (f, 1)):
            ch += [co] * (2 + n)
        return ch
