#!/usr/bin/env python
"""Generate tests/golden/registration.npz by RUNNING THE UNMODIFIED REFERENCE VNet3dRegistration
(networks/VNet3dregistration.py) on the CPU, with ``voxelmorph`` stubbed in ``sys.modules``.

Usage (needs the reference checkout, which the GPU machines do not have):
    PYTORCHDEEPLEARING_REFERENCE=/path/to/reference python tests/golden/make_golden_registration.py

voxelmorph is not installed, so the stub's ``SpatialTransformer`` is voxelmorph's layer as recalled: a subclass of
the reference's own ``SpatialTransformergrid`` whose forward returns ``F.grid_sample(src, new_locs,
align_corners=True, mode=mode)``.  It is NOT verified against voxelmorph.

Weights: the reference's default initialisation after ``torch.manual_seed(<tag>.seed)`` (the drop-in builds its leaves
in the same order, so the same seed gives the same weights).  Per case the file records, under the case tag:
  ``<tag>.cfg``              (batch, image_channel, init_features, D, H, W, seed)
  ``<tag>.moved_image`` / ``<tag>.ddf``   eval-mode outputs at every other voxel per axis
  ``<tag>.moved_label``      the full eval-mode nearest-warped label
  ``<tag>.fp``               sum, mean, std, max |.| of the full moved_image, then of the full ddf
  ``<tag>.loss``             1 - SSIM3D(moved_image, fixed_image) + 0.01 * ddf.pow(2).mean() (lossesSSIM), eval mode
  ``<tag>.grads``            (norm, sum) of every parameter gradient of that loss, in state_dict order
  ``<tag>.params``           (sum, sum of squares) of every state_dict tensor
Inputs come from ``inputs(cfg)`` below (a seeded CPU generator), which the tests import; and ``names`` / ``shapes``: the state_dict layout of VNet3dRegistration(2, 3, (32, 32, 32)).
"""
import importlib.util
import os
import sys
import types

import numpy as np
import torch
import torch.nn.functional as F

sys.dont_write_bytecode = True
HERE = os.path.dirname(os.path.abspath(__file__))

CASES = {
    "cubic_b2_f8": (2, 2, 8, 32, 32, 32, 11),
    "noncubic_f8": (1, 2, 8, 32, 48, 64, 12),
    "cubic_f16": (1, 2, 16, 32, 32, 32, 13),
}


def inputs(cfg):
    """moving image, fixed image (1 channel each), moving label, fixed label (3 classes as float)"""
    n, ic, _, d, h, w, seed = cfg
    g = torch.Generator().manual_seed(1000 + seed)
    sp = (d, h, w)
    mi = torch.randn((n, ic // 2) + sp, generator=g)
    fi = torch.randn((n, ic - ic // 2) + sp, generator=g)
    ml = torch.randint(0, 3, (n, 1) + sp, generator=g).float()
    fl = torch.randint(0, 3, (n, 1) + sp, generator=g).float()
    return mi, fi, ml, fl


def _load(path, name):
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ref = os.environ.get("PYTORCHDEEPLEARING_REFERENCE")
    if not ref:
        sys.exit("set PYTORCHDEEPLEARING_REFERENCE to the reference checkout")
    vxm = types.ModuleType("voxelmorph")
    vxm.torch = types.SimpleNamespace(layers=types.SimpleNamespace())
    sys.modules["voxelmorph"] = vxm
    regmod_src = os.path.join(ref, "networks", "VNet3dregistration.py")

    # the stub needs the reference's SpatialTransformergrid: load the module once with a placeholder, then bind
    vxm.torch.layers.SpatialTransformer = None
    reg = _load(regmod_src, "reference_vnet3dregistration")

    class SpatialTransformer(reg.SpatialTransformergrid):
        def __init__(self, size, mode="bilinear"):
            super().__init__(size)
            self.mode = mode

        def forward(self, src, flow):
            new_locs = super().forward(flow)
            return F.grid_sample(src, new_locs, align_corners=True, mode=self.mode)

    vxm.torch.layers.SpatialTransformer = SpatialTransformer
    ssim = _load(os.path.join(ref, "model", "lossesSSIM.py"), "reference_lossesSSIM")

    out = {}
    for tag, cfg in CASES.items():
        n, ic, f, d, h, w, seed = cfg
        torch.manual_seed(seed)
        net = reg.VNet3dRegistration(ic, 3, (d, h, w), init_features=f).eval()
        mi, fi, ml, fl = inputs(cfg)
        moved, mlab, ddf = net(mi, fi, ml, fl)
        loss = 1 - ssim.SSIM3D()(moved, fi) + 0.01 * ddf.pow(2).mean()
        loss.backward()
        sd = net.state_dict()
        out[tag + ".cfg"] = np.array(cfg, dtype=np.int64)
        out[tag + ".moved_image"] = moved.detach()[:, :, ::2, ::2, ::2].numpy()
        out[tag + ".ddf"] = ddf.detach()[:, :, ::2, ::2, ::2].numpy()
        out[tag + ".moved_label"] = mlab.detach().numpy().astype(np.uint8)
        fp = []
        for t in (moved.detach(), ddf.detach()):
            t = t.double()
            fp += [t.sum().item(), t.mean().item(), t.std().item(), t.abs().max().item()]
        out[tag + ".fp"] = np.array(fp)
        out[tag + ".loss"] = np.array(loss.item())
        out[tag + ".grads"] = np.array([[p.grad.double().norm().item(), p.grad.double().sum().item()]
                                        for _, p in net.named_parameters()])
        out[tag + ".params"] = np.array([[v.double().sum().item(), v.double().pow(2).sum().item()]
                                         for v in sd.values()])
    lay = reg.VNet3dRegistration(2, 3, (32, 32, 32)).state_dict()
    out["names"] = np.array(list(lay.keys()))
    out["shapes"] = np.array([list(v.shape) + [0] * (5 - v.dim()) for v in lay.values()], dtype=np.int64)
    np.savez_compressed(os.path.join(HERE, "registration.npz"), **out)
    print("wrote", os.path.join(HERE, "registration.npz"), {k: v.shape for k, v in out.items() if v.ndim})


if __name__ == "__main__":
    main()
