"""Functional restatement of the reference's VNet3dRegistration (networks/VNet3dregistration.py:48-208) and of the
voxelmorph SpatialTransformer it calls, in plain torch ops (fp32 or fp64: the dtype of the inputs), for the tests.

``sd``: a state_dict of the reference layout; ``masks``: the dropout scales (N, C) in module-call order
(``VNet3dRegistration._mask_channels``), or None for eval.  The SpatialTransformer is voxelmorph's layer as recalled:
``F.grid_sample(src, new_locs, align_corners=True, mode=mode)`` over ``SpatialTransformergrid``'s locations."""
import torch
import torch.nn.functional as F

EPS = 1e-5
DOWN_OPS = (2, 2, 2, 2)
UP_OPS = (2, 2, 2, 1)


def sampling_grid(ddf):
    """SpatialTransformergrid.forward (VNet3dregistration.py:28-45) in the dtype of ddf: the normalised locations in
    grid_sample's (x, y, z) order"""
    n, _, D, H, W = ddf.shape
    vectors = [torch.arange(0, s, dtype=ddf.dtype, device=ddf.device) for s in (D, H, W)]
    grid = torch.stack(torch.meshgrid(vectors, indexing="ij")).unsqueeze(0)
    new_locs = grid + ddf
    for i, s in enumerate((D, H, W)):
        new_locs[:, i, ...] = 2 * (new_locs[:, i, ...] / (s - 1) - 0.5)
    return new_locs.permute(0, 2, 3, 4, 1)[..., [2, 1, 0]]


def warp(src, ddf, mode):
    return F.grid_sample(src, sampling_grid(ddf), align_corners=True, mode=mode)


def forward(sd, moving_image, fixed_image, moving_label, masks=None):
    """(moved_image, moved_label, ddf) of VNet3dRegistration.forward"""
    dt = moving_image.dtype
    P = {k: v.to(dtype=dt, device=moving_image.device) for k, v in sd.items()}
    it = iter(masks) if masks is not None else None

    def tail(y, bn):
        y = F.instance_norm(y, weight=P[bn + ".weight"], bias=P[bn + ".bias"], eps=EPS)
        if it is not None:
            y = y * next(it).to(y)[:, :, None, None, None]
        return F.leaky_relu(y, 0.01)

    def conv(x, name, **kw):
        return F.conv3d(x, P[name + ".weight"], P[name + ".bias"], **kw)

    def ops(x, name, n):
        for j in range(n):
            x = tail(conv(x, f"{name}.ops.{j}.conv", padding=1), f"{name}.ops.{j}.bn")
        return x

    x = torch.cat((moving_image, fixed_image), 1)
    out = tail(conv(x, "in_tr.conv1", padding=1), "in_tr.bn") + tail(conv(x, "in_tr.conv2"), "in_tr.bn")
    skips = [out]
    for name, n in zip(("down_tr32", "down_tr64", "down_tr128", "down_tr256"), DOWN_OPS):
        down = tail(conv(out, name + ".down_conv", stride=2), name + ".bn")
        out = ops(down, name, n) + down
        skips.append(out)
    for k, (name, n) in enumerate(zip(("up_tr256", "up_tr128", "up_tr64", "up_tr32"), UP_OPS)):
        up = F.conv_transpose3d(out, P[name + ".up_conv.weight"], P[name + ".up_conv.bias"], stride=2)
        up = tail(up, name + ".bn")
        xcat = tail(conv(torch.cat((up, skips[3 - k]), 1), name + ".conv"), name + ".bn")
        out = ops(xcat, name, n) + xcat
    ddf = conv(out, "out_tr.conv")
    return warp(moving_image, ddf, "bilinear"), warp(moving_label, ddf, "nearest"), ddf
