"""CPU oracle for the segmentation hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` /
``--impl reference`` legs may import this package.  The product package
``pytorchdeeplearing_b200`` never imports it and has no CPU fallback.

What it is: a functional (state_dict in, tensors out) restatement of the reference's
``networks/VNet3d.py``, ``networks/Unet3d.py``, ``networks/Unet2d.py`` and of the eight
hot-path reductions in ``model/losses.py``, executed by the installed PyTorch on CPU in
fp32 (or fp64 for the noise floor).  The reference itself is pure Python over PyTorch, so
its arithmetic lives in the third-party dependency PyTorch (unpinned by the reference;
README.md:13 says "pytorch1.10.0"; installed here: torch 2.11.0).

Pinning: the reference ships no tests and no golden vectors (SURVEY.md section 4), so the
oracle is pinned against OUTPUTS OF THE REFERENCE ITSELF run in the build container:
``tests/golden/make_golden.py`` imports the reference checkout (``$PYTORCHDEEPLEARING_REFERENCE``) (with the non-invasive
``VNet3d`` constructor shim for the ``networks/VNet3d.py:127`` typo), runs it on seeded
inputs and commits the results as ``tests/golden/*.npz``;  ``tests/test_oracle_golden.py``
checks this restatement against those fixtures on every CPU run.
"""
from .nets import (vnet3d_forward, unet_forward, init_state_dict, vnet3d_state_spec,
                   unet_state_spec, draw_dropout_masks_vnet3d, draw_dropout_masks_unet)
from .losses import LOSSES, loss_forward
from .data import make_inputs

__all__ = ["vnet3d_forward", "unet_forward", "init_state_dict", "vnet3d_state_spec",
           "unet_state_spec", "draw_dropout_masks_vnet3d", "draw_dropout_masks_unet",
           "LOSSES", "loss_forward", "make_inputs"]
