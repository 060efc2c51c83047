"""VNet3dRegistration without a GPU: the state_dict layout and seeded initial weights against what the reference
recorded (tests/golden/registration.npz), the functional oracle against the reference's outputs, install(), and every
input error the drop-in raises before it reaches a kernel."""
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
from make_golden_registration import CASES, inputs  # noqa: E402

import pytorchdeeplearing_b200 as b200  # noqa: E402
from oracle import registration as oreg  # noqa: E402

GOLD = np.load(os.path.join(HERE, "golden", "registration.npz"))


def build(tag):
    n, ic, f, d, h, w, seed = CASES[tag]
    torch.manual_seed(seed)
    return b200.VNet3dRegistration(ic, 3, (d, h, w), init_features=f)


def test_state_dict_layout_matches_the_reference():
    sd = b200.VNet3dRegistration(2, 3, (32, 32, 32)).state_dict()
    assert list(sd.keys()) == [str(k) for k in GOLD["names"]]
    shapes = [[s for s in row if s] for row in GOLD["shapes"].tolist()]
    assert [list(v.shape) for v in sd.values()] == shapes
    assert len(sd) == 110 and sum(1 for _ in b200.VNet3dRegistration(2, 3, (32, 32, 32)).parameters()) == 108
    leaves = {type(m) for m in b200.VNet3dRegistration(2, 3, (32, 32, 32)).modules()}
    assert {torch.nn.Conv3d, torch.nn.ConvTranspose3d, torch.nn.InstanceNorm3d} <= leaves


@pytest.mark.parametrize("tag", sorted(CASES))
def test_seeded_construction_draws_the_reference_weights(tag):
    got = np.array([[v.double().sum().item(), v.double().pow(2).sum().item()] for v in build(tag).state_dict().values()])
    assert np.array_equal(got, GOLD[tag + ".params"])


@pytest.mark.parametrize("tag", sorted(CASES))
def test_oracle_matches_the_reference(tag):
    net = build(tag)
    mi, fi, ml, fl = inputs(CASES[tag])
    moved, mlab, ddf = oreg.forward(net.state_dict(), mi, fi, ml)
    for name, t in (("moved_image", moved), ("ddf", ddf)):
        want = torch.from_numpy(GOLD[f"{tag}.{name}"])
        sub = t[:, :, ::2, ::2, ::2]
        assert (sub - want).abs().max().item() <= 1e-5 * want.abs().max().item(), name
    assert np.array_equal(mlab.numpy().astype(np.uint8), GOLD[tag + ".moved_label"])


def test_install_rebinds_the_reference_module():
    mod = types.ModuleType("networks.VNet3dregistration")
    mod.VNet3dRegistration = object
    sys.modules["networks.VNet3dregistration"] = mod
    try:
        assert b200.install() >= 1
        assert mod.VNet3dRegistration is b200.VNet3dRegistration
    finally:
        b200.uninstall()
        del sys.modules["networks.VNet3dregistration"]
    assert mod.VNet3dRegistration is object


def _args(sp=(32, 32, 32), n=1):
    return (torch.zeros((n, 1) + sp), torch.zeros((n, 1) + sp), torch.zeros((n, 1) + sp), torch.zeros((n, 1) + sp))


def test_errors():
    from pytorchdeeplearing_b200 import runtime
    net = b200.VNet3dRegistration(2, 3, (32, 32, 32), init_features=4)
    with pytest.raises(ValueError, match="must be"):
        net(*_args((32, 32, 48)))
    with pytest.raises(ValueError, match="numclass must be 3"):
        b200.VNet3dRegistration(2, 2, (32, 32, 32), init_features=4)(*_args())
    with pytest.raises(ValueError, match="multiples of 16"):
        b200.VNet3dRegistration(2, 3, (32, 32, 40), init_features=4)(*_args((32, 32, 40)))
    with pytest.raises(ValueError, match="more than one voxel"):
        b200.VNet3dRegistration(2, 3, (16, 16, 16), init_features=4).train()(*_args((16, 16, 16)))
    with pytest.raises(ValueError, match="at most 512"):
        b200.VNet3dRegistration(2, 3, (32, 32, 32), init_features=64)(*_args())
    a = list(_args())
    a[0] = a[0].requires_grad_()
    with pytest.raises(ValueError, match="moving_image requires a gradient"):
        net(*a)
    a = list(_args())
    a[2] = a[2].requires_grad_()
    with pytest.raises(ValueError, match="moving_label requires a gradient"):
        net(*a)
    a = list(_args())
    a[1] = a[1].double()
    with pytest.raises(TypeError):
        net(*a)
    orig = runtime.dp_state
    runtime.dp_state = lambda: (True, None)
    try:
        with pytest.raises(RuntimeError, match="data parallel"):
            net(*_args())
    finally:
        runtime.dp_state = orig
    from pytorchdeeplearing_b200.graphed import GraphedStep
    with pytest.raises(TypeError, match="VNet3dRegistration"):
        GraphedStep(net, None, torch.zeros(1, 2, 32, 32, 32), torch.zeros(1, 32, 32, 32))


def test_mask_channels_follow_the_dropout_calls():
    f = 8
    net = b200.VNet3dRegistration(2, 3, (32, 32, 32), init_features=f)
    # in_tr 2, four down blocks of 1 + 2, up blocks of 2 + (2, 2, 2, 1)
    assert net._mask_channels() == [f, f] + [2 * f] * 3 + [4 * f] * 3 + [8 * f] * 3 + [16 * f] * 3 + \
        [8 * f] * 4 + [4 * f] * 4 + [2 * f] * 4 + [f] * 3
