#!/usr/bin/env python
"""tests/golden/dropin.json from the unmodified reference (PYTORCHDEEPLEARING_REFERENCE=<checkout>): names its modules
bind, digests of its networks' state_dict layouts and of what its initialize_weights leaves in the drop-in's tensors."""
import hashlib
import json
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import ref_harness  # noqa: E402
import pytorchdeeplearing_b200 as b200  # noqa: E402
inst = __import__("importlib").import_module("pytorchdeeplearing_b200.install")


def _digest(lines):
    return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def layout_digest(model):
    sd = model.state_dict()
    return [len(sd), _digest(f"{k} {tuple(v.shape)}" for k, v in sd.items())]


def init_digest(model):
    def value(v):
        u = torch.unique(v)
        return repr(float(u[0])) if u.numel() == 1 else "random"
    return _digest(f"{k} {value(v)}" for k, v in model.state_dict().items())


def main():
    if not ref_harness.available():
        raise SystemExit("set PYTORCHDEEPLEARING_REFERENCE to a checkout of the reference")
    ref = ref_harness.import_reference()
    names = set(inst._NET_NAMES) | set(inst._LOSS_NAMES) | set(inst._METRIC_NAMES)
    bindings = {m: sorted(n for n in names if hasattr(sys.modules[m], n)) for m in inst._MODULES if m in sys.modules}
    nets = ref["networks"]
    VNet3d = ref["networks.VNet3d"].VNet3d

    class VNet3dFixed(VNet3d):
        feature = property(lambda self: self.features)

    torch.manual_seed(0)
    layouts = {"VNet3d(1,2)": layout_digest(VNet3dFixed(1, 2)),
               "VNet2d(1,1)": layout_digest(ref["networks.VNet2d"].VNet2d(1, 1)),
               "UNet3d(1,4)": layout_digest(ref["networks.Unet3d"].UNet3d(1, 4)),
               "UNet2d(1,1)": layout_digest(ref["networks.Unet2d"].UNet2d(1, 1))}
    init = {}
    for key, m in (("VNet3d(1,2)", b200.VNet3d(1, 2)), ("UNet2d(1,1)", b200.UNet2d(1, 1))):
        m.apply(nets.initialize_weights)
        init[key] = init_digest(m)
    with open(os.path.join(HERE, "dropin.json"), "w") as f:
        json.dump({"bindings": bindings, "layouts": layouts, "init": init}, f, indent=1)


if __name__ == "__main__":
    main()
