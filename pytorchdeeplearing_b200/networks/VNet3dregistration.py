"""Drop-in ``VNet3dRegistration`` (reference networks/VNet3dregistration.py:144-208): same constructor, same 110-entry
``state_dict`` (108 parameters in ``nn.Conv3d`` / ``nn.ConvTranspose3d`` / ``nn.InstanceNorm3d`` leaves, then the two
``SpatialTransformer`` grid buffers), forward and backward on sm_90a kernels.

The network is VNet3d's layer program (``engine.Engine.vnet_forward`` with ``engine.REGISTRATION``: InstanceNorm3d as
one GroupNorm group per channel, LeakyReLU(0.01), 2/2/2/2 down and 2/2/2/1 up LUConv ops) on ``cat(moving, fixed)``;
its head writes the displacement field ``ddf`` and one ``csrc/warp3d.cu`` launch warps the moving image (trilinear)
and the moving label (nearest) by it (``warp.py``).  Backward takes d loss / d moved_image and d loss / d ddf (the
caller's own term) together: the warp backward adds the latter as its addend, then the network backward runs.

Differences from the reference, by design: inputs are fp32 CUDA tensors of exactly ``vol_size``; the moving image and
label may not require a gradient; ``numclass`` must be 3 (the reference's broadcast of a ``numclass``-channel field
against its 3-channel grid fails otherwise); at most 512 channels (``init_features <= 32``); no data parallelism (the
loss is the caller's, so a gradient all-reduce would have no defined scale) and no ``GraphedStep``."""
import torch
import torch.nn as nn

from .. import runtime
from ..engine import Engine, REGISTRATION
from ._base import SegNetBase, _Holder, _net_backward


def _grid(size):
    """SpatialTransformergrid's buffer (VNet3dregistration.py:15-26): (1, 3, D, H, W) fp32 meshgrid indices"""
    vectors = [torch.arange(0, s) for s in size]
    return torch.stack(torch.meshgrid(vectors, indexing="ij")).unsqueeze(0).float()


class _RegNetFunction(torch.autograd.Function):
    """forward: (x, moving image, moving label, *params) -> (moved_image, moved_label, ddf);
    backward: d moved_image and d ddf -> d params"""

    @staticmethod
    def forward(ctx, mod, need_grad, x, image, label, masks, *params):
        be = runtime.get_backend(x)
        eng = Engine(be, runtime.act_dtype(), 3)
        eng.want_probs = False
        P = dict(zip(mod._pnames, [p.detach() for p in params]))
        ddf, _ = eng.vnet_forward(P, x, masks, need_grad, spec=REGISTRATION)
        field = ddf.permute(0, 2, 3, 4, 1)                  # the head's (N, D, H, W, 3) buffer
        moved_image = torch.empty_like(image)
        moved_label = torch.empty_like(label)
        be.warp3d(field, image, label, moved_image, moved_label)
        ctx.eng = eng if need_grad else None
        ctx.arch = "vnet"
        ctx.names = mod._pnames
        ctx.save_for_backward(field, image)
        ctx.mark_non_differentiable(moved_label)
        ctx.set_materialize_grads(False)
        return moved_image, moved_label, ddf

    @staticmethod
    def backward(ctx, g_image, g_label, g_ddf):
        eng = ctx.eng
        if eng is None:
            raise RuntimeError("pytorchdeeplearing_b200: backward through the network a second time (the saved "
                               "activations are released after the first backward; retain_graph is not supported)")
        field, image = ctx.saved_tensors
        none = (None,) * (6 + len(ctx.names))
        if g_image is None and g_ddf is None:
            return none
        addend = g_ddf.permute(0, 2, 3, 4, 1).contiguous().float() if g_ddf is not None else None
        if g_image is not None:
            g = torch.empty_like(field)
            runtime.get_backend(field).warp3d_bwd(field, image, g_image.contiguous().float(), addend, g)
        else:
            g = addend
        grads = _net_backward(ctx, eng, g)[4:]
        return (None,) * 6 + tuple(grads)


class VNet3dRegistration(SegNetBase):
    _arch = "vnet"
    _dims = 3

    def __init__(self, image_channel, numclass, vol_size, init_features=16):
        super().__init__()
        self.image_channel = image_channel
        self.numclass = numclass
        self.features = f = init_features
        self.vol_size = tuple(int(s) for s in vol_size)

        def lu_stack(nchan, depth):
            # reference: _make_nConv3d -> nn.Sequential of LUConv3d (VNet3dregistration.py:48-68): ops.{i}.conv / .bn
            layers = []
            for _ in range(depth):
                lu = _Holder()
                lu.conv = nn.Conv3d(nchan, nchan, kernel_size=3, padding=1)
                lu.bn = nn.InstanceNorm3d(nchan, affine=True)
                layers.append(lu)
            return nn.Sequential(*layers)

        # construction order = the reference's, so a seeded construction draws the same initial weights
        self.in_tr = _Holder()                                        # InputTransition3d, :71-78
        self.in_tr.conv1 = nn.Conv3d(image_channel, f, kernel_size=3, padding=1)
        self.in_tr.conv2 = nn.Conv3d(image_channel, f, kernel_size=1)
        self.in_tr.bn = nn.InstanceNorm3d(f, affine=True)
        for name, ci, co, n in (("down_tr32", f, 2 * f, 2), ("down_tr64", 2 * f, 4 * f, 2),
                                ("down_tr128", 4 * f, 8 * f, 2), ("down_tr256", 8 * f, 16 * f, 2)):
            blk = _Holder()                                           # DownTransition3d, :92-99
            blk.down_conv = nn.Conv3d(ci, co, kernel_size=2, stride=2)
            blk.bn = nn.InstanceNorm3d(co, affine=True)
            blk.ops = lu_stack(co, n)
            setattr(self, name, blk)
        for name, ci, co, n in (("up_tr256", 16 * f, 8 * f, 2), ("up_tr128", 8 * f, 4 * f, 2),
                                ("up_tr64", 4 * f, 2 * f, 2), ("up_tr32", 2 * f, f, 1)):
            blk = _Holder()                                           # UpTransition3d, :108-116
            blk.up_conv = nn.ConvTranspose3d(ci, co, kernel_size=2, stride=2)
            blk.bn = nn.InstanceNorm3d(co, affine=True)
            blk.ops = lu_stack(co, n)
            blk.conv = nn.Conv3d(ci, co, kernel_size=1)
            setattr(self, name, blk)
        self.out_tr = _Holder()                                       # OutputTransition3d, :129-134
        self.out_tr.conv = nn.Conv3d(f, numclass, kernel_size=1)
        for name in ("spatial_transformer_image", "spatial_transformer_label"):
            st = _Holder()
            st.register_buffer("grid", _grid(self.vol_size))
            setattr(self, name, st)
        self._finish_init()

    def _mask_channels(self):
        # Dropout3d calls in module-call order: in_tr (both branches), each down block (down conv + ops), each up
        # block (up conv, concat conv, ops)
        f = self.features
        ch = [f, f]
        for co in (2 * f, 4 * f, 8 * f, 16 * f):
            ch += [co] * 3
        for co, n in ((8 * f, 2), (4 * f, 2), (2 * f, 2), (f, 1)):
            ch += [co] * (2 + n)
        return ch

    def _check(self, moving_image, fixed_image, moving_label):
        if runtime.dp_state()[0]:
            raise RuntimeError("VNet3dRegistration does not run data parallel: the loss is the caller's, so the "
                               "gradient all-reduce has no defined scale")
        if self.numclass != 3:
            raise ValueError(f"numclass must be 3 (the displacement field has one channel per axis), got "
                             f"{self.numclass}")
        if 16 * self.features > 512:
            raise ValueError(f"at most 512 channels (init_features <= 32), got init_features={self.features}")
        for name, t in (("moving_image", moving_image), ("fixed_image", fixed_image), ("moving_label", moving_label)):
            if t.dtype != torch.float32:
                raise TypeError(f"{name} must be float32, got {t.dtype}")
            if t.dim() != 5 or tuple(t.shape[2:]) != self.vol_size or t.shape[0] != moving_image.shape[0]:
                raise ValueError(f"{name} must be (N, C, {', '.join(map(str, self.vol_size))}), got {tuple(t.shape)}")
        if any(s % 16 for s in self.vol_size):
            raise ValueError(f"spatial sizes must be multiples of 16 (four stride-2 stages), got {self.vol_size}")
        if self.training and all(s == 16 for s in self.vol_size):
            raise ValueError("training needs more than one voxel at the bottom level (InstanceNorm's rule): "
                             f"vol_size {self.vol_size}")
        if moving_image.shape[1] + fixed_image.shape[1] != self.image_channel:
            raise ValueError(f"moving and fixed images have {moving_image.shape[1]} + {fixed_image.shape[1]} channels, "
                             f"the network takes image_channel={self.image_channel}")
        for name, t in (("moving_image", moving_image), ("moving_label", moving_label)):
            if t.requires_grad:
                raise ValueError(f"{name} requires a gradient; the drop-in computes gradients for the parameters only")
        if fixed_image.requires_grad and torch.is_grad_enabled():
            raise ValueError("fixed_image requires a gradient; the drop-in computes gradients for the parameters only")

    def forward(self, moving_image, fixed_image, moving_label, fixed_label):
        self._check(moving_image, fixed_image, moving_label)
        params = [p for _, p in self.named_parameters()]
        x = torch.cat((moving_image, fixed_image), 1)
        masks = self._draw_masks(x)
        need_grad = torch.is_grad_enabled() and any(p.requires_grad for p in params)
        return _RegNetFunction.apply(self, need_grad, x, moving_image.detach().contiguous(),
                                     moving_label.detach().contiguous(), masks, *params)
