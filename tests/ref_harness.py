"""Import the UNMODIFIED reference tree (a checkout of junqiangchen/PytorchDeepLearing named by the environment variable
PYTORCHDEEPLEARING_REFERENCE) for drop-in tests -- TEST-ONLY.

The reference's ``model`` package imports four I/O-only modules that are absent here (SimpleITK, torchsummary,
skimage, matplotlib; SURVEY.md 0.10 / App. E).  They are replaced by inert stubs in ``sys.modules``; nothing of the
reference is modified or copied.  Tests using this harness skip when no reference checkout is named."""
import importlib
import os
import sys
import types

REF = os.environ.get("PYTORCHDEEPLEARING_REFERENCE", "")


def available() -> bool:
    return bool(REF) and os.path.isdir(os.path.join(REF, "networks"))


def _stub(name, **attrs):
    m = types.ModuleType(name)
    for k, v in attrs.items():
        setattr(m, k, v)
    sys.modules[name] = m
    return m


def import_reference():
    """-> dict of the reference modules (networks, model.losses, model.metric, model.modelVNet, model.modelUnet)"""
    sys.dont_write_bytecode = True
    if REF not in sys.path:
        sys.path.insert(0, REF)
    noop = lambda *a, **k: None
    if "SimpleITK" not in sys.modules:
        _stub("SimpleITK", sitkLinear=1, sitkNearestNeighbor=0, GetImageFromArray=noop, WriteImage=noop,
              GetArrayFromImage=noop)
    if "torchsummary" not in sys.modules:
        _stub("torchsummary", summary=noop)
    if "skimage" not in sys.modules:
        sk = _stub("skimage")
        sk.metrics = _stub("skimage.metrics", structural_similarity=noop)
    if "matplotlib" not in sys.modules:
        mp = _stub("matplotlib", use=noop)
        class _Style:
            use = staticmethod(noop)
        mp.pyplot = _stub("matplotlib.pyplot", style=_Style, figure=noop, plot=noop, title=noop, xlabel=noop,
                          ylabel=noop, legend=noop, savefig=noop, close=noop, show=noop, imshow=noop, subplot=noop)
    if "model" not in sys.modules or not hasattr(sys.modules["model"], "__path__"):
        pkg = types.ModuleType("model")
        pkg.__path__ = [os.path.join(REF, "model")]          # skip model/__init__.py (drags ResNet/GAN wrappers)
        sys.modules["model"] = pkg
    names = ["networks", "networks.VNet3d", "networks.VNet2d", "networks.Unet3d", "networks.Unet2d", "model.losses",
             "model.metric", "model.modelVNet", "model.modelUnet"]
    return {n: importlib.import_module(n) for n in names}
