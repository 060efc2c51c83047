"""Shared builder of the drop-in ResNet3d / ResNet2d classifiers (reference networks/ResNet3d.py:72-118 and
networks/ResNet2d.py:73-119): same constructor signature, same ``state_dict`` (70 tensors), forward/backward on sm_90a
kernels.  ``forward`` returns one tensor, the (N, numclass) fp32 logits, as the reference does.

The reference's ``DownTransition`` reads an undefined global ``prob`` (ResNet3d.py:51), so it cannot be constructed
as shipped; the drop-in uses p = 0.2 (``engine.P_DROP``), the rate of every other Dropout of the reference nets."""
import torch.nn as nn

from ._base import SegNetBase, _ClsNetFunction, _Holder


class _ResNetBase(SegNetBase):
    _arch = "resnet"
    _function = _ClsNetFunction

    def __init__(self, image_channel, numclass):
        super().__init__()
        Conv = nn.Conv3d if self._dims == 3 else nn.Conv2d
        self.image_channel = image_channel
        self.numclass = numclass

        def lu_stack(nchan, depth):
            # reference: _make_nConv3d -> nn.Sequential of LUConv3d (ResNet3d.py:5-21); keys ops.{i}.conv1 / ops.{i}.bn1
            layers = []
            for _ in range(depth):
                lu = _Holder()
                lu.conv1 = Conv(nchan, nchan, kernel_size=3, padding=1)
                lu.bn1 = nn.GroupNorm(8, nchan)
                layers.append(lu)
            return nn.Sequential(*layers)

        self.in_tr = _Holder()                                        # InputTransition3d, ResNet3d.py:24-30
        self.in_tr.conv1 = Conv(image_channel, 16, kernel_size=3, padding=1)
        self.in_tr.conv2 = Conv(image_channel, 16, kernel_size=1)
        self.in_tr.bn1 = nn.GroupNorm(8, 16)

        for name, ci, co, n in (("down_tr32", 16, 32, 2), ("down_tr64", 32, 64, 3),
                                ("down_tr128", 64, 128, 3), ("down_tr256", 128, 256, 3)):
            blk = _Holder()                                           # DownTransition3d, ResNet3d.py:44-51
            blk.down_conv = Conv(ci, co, kernel_size=2, stride=2)
            blk.bn1 = nn.GroupNorm(8, co)
            blk.ops = lu_stack(co, n)
            setattr(self, name, blk)

        # ResNet3d.py:93-96: a Sequential holder, so the keys (fc_layers.0 / fc_layers.2) and initialize_weights match
        self.fc_layers = nn.Sequential(nn.Linear(256, 128), nn.ReLU(inplace=True), nn.Linear(128, numclass))
        self._finish_init()

    def _mask_channels(self):
        # the four DownTransition do1 calls (ResNet3d.py:55); the input transition and LUConv stacks have no dropout
        return [32, 64, 128, 256]
