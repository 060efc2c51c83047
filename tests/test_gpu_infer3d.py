"""Whole-volume 3-D inference kernels (csrc/resample.cu) on the GPU against the fp64 oracle (oracle/resample.py):
the linear resample of every pixel type, both normalisations, the nearest-neighbour back-resample with its crop / pad,
guard bands, bit-identical reruns, graph replay, no host synchronisation, and inference3d / inference_patch3d end to
end against the oracle chain followed by the existing predict."""
import os

import numpy as np
import pytest
import torch

from oracle import nets as onets
from oracle import resample as R
import pytorchdeeplearing_b200 as b200
from pytorchdeeplearing_b200 import inference as inf
from pytorchdeeplearing_b200 import runtime
from pytorchdeeplearing_b200._abi import NORM_MEANSTD, NORM_NONE, NORM_PCTL
from conftest import GOLDEN

pytestmark = pytest.mark.gpu
GOLD = dict(np.load(os.path.join(GOLDEN, "infer3d.npz")))
CASES = [str(c) for c in GOLD["cases"]]
GUARD = 4096


@pytest.fixture(autouse=True)
def _restore_precision():
    prev = b200.get_precision()
    yield
    b200.set_precision(prev)


def be():
    return runtime.cuda_backend()


def guarded(shape, dtype, fill):
    """(view of `shape` inside a buffer with GUARD elements of `fill` on both sides, the buffer)"""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * GUARD,), fill, dtype=dtype, device="cuda")
    return buf[GUARD:GUARD + n].view(shape), buf


def guards_intact(buf, fill):
    g = torch.cat([buf[:GUARD], buf[-GUARD:]]).cpu()
    return bool(torch.isnan(g).all()) if isinstance(fill, float) and fill != fill else bool((g == fill).all())


def volume(shape, dtype, seed=0, lo=-1024, hi=2000):
    rng = np.random.RandomState(seed)
    if dtype == np.float32:
        return (rng.rand(*shape) * (hi - lo) + lo).astype(np.float32)
    if dtype == np.uint8:
        return rng.randint(0, 256, size=shape).astype(np.uint8)
    return rng.randint(lo, hi, size=shape).astype(dtype)


def run_linear(vol, out_zyx, ratio, mode=NORM_NONE, window=(0.0, 0.0)):
    src = torch.from_numpy(vol).cuda()
    out, buf = guarded(out_zyx, torch.float32, float("nan"))
    ws = be().resample_workspace(mode, out_zyx, src.device) if mode != NORM_NONE else None
    be().resample_linear(src, ratio, out, mode, window[0], window[1], ws)
    torch.cuda.synchronize()
    assert guards_intact(buf, float("nan"))
    return out, ws


def ulp_diff(a, b):
    ai, bi = a.astype(np.float32).view(np.int32).astype(np.int64), b.astype(np.float32).view(np.int32).astype(np.int64)
    ai = np.where(ai < 0, -(ai & 0x7fffffff), ai)
    bi = np.where(bi < 0, -(bi & 0x7fffffff), bi)
    return np.abs(ai - bi)


# (input (D, H, W), output (D, H, W)): odd sizes with 2.34x upsampling along W, 2.5x upsampling along every axis, a
# non-integer downsampling, and the CT volume
SHAPES = [((77, 130, 41), (96, 96, 96)), ((20, 24, 16), (50, 60, 40)), ((100, 90, 80), (37, 41, 29)),
          ((300, 512, 512), (96, 96, 96))]


@pytest.mark.parametrize("shape_in,shape_out", SHAPES)
@pytest.mark.parametrize("dtype", [np.float32, np.int16, np.uint8, np.int32])
def test_linear_resample_against_the_oracle(shape_in, shape_out, dtype):
    if shape_in[0] == 300 and dtype != np.int16:
        pytest.skip("the CT volume runs as int16")
    vol = volume(shape_in, dtype)
    ratio = R.size_ratio(shape_in, shape_out)
    out, _ = run_linear(vol, shape_out, ratio)
    got = out.cpu().numpy()
    want = R.resample_linear(vol, shape_out, ratio)
    if dtype == np.float32:
        assert int(ulp_diff(got, want).max()) <= 1
    else:
        # the kernel rounds every fp64 operation as the oracle does, so even samples within 1e-9 of an integer (where
        # the truncating cast would expose a different rounding) agree: the mismatch count is 0
        boundary = R.integer_boundary_points(vol, shape_out, ratio)
        bad = got != want
        assert int(bad.sum()) == 0, (int(bad.sum()), int((bad & boundary).sum()))
    for axis in range(3):
        if shape_out[axis] >= 2 * shape_in[axis]:
            # past the last input sample along this axis: ITK's default pixel value
            assert np.all(np.take(got, -1, axis=axis) == 0.0), axis


@pytest.mark.parametrize("mode", [NORM_MEANSTD, NORM_PCTL])
def test_normalize_is_bit_identical_on_rerun(mode):
    vol = volume((77, 130, 41), np.int16, seed=5, lo=-300, hi=300)
    ratio = R.size_ratio((77, 130, 41), (96, 96, 96))
    runs = [normalize_device(vol, (96, 96, 96), ratio, mode) for _ in range(2)]
    (xa, za, sa), (xb, zb, sb) = runs
    assert np.array_equal(xa, xb)
    assert np.array_equal(za.view(np.int32), zb.view(np.int32))
    # the six stats the kernels write: mean, sigma, p5, p95, unchanged flag, count
    assert np.array_equal(sa[:6].view(np.int64), sb[:6].view(np.int64))


def normalize_device(vol, out_zyx, ratio, mode, window=(-100.0, 100.0)):
    x, ws = run_linear(vol, out_zyx, ratio, mode, window)
    out, buf = guarded(out_zyx, torch.float32, float("nan"))
    be().normalize(mode, x, ws, out)
    torch.cuda.synchronize()
    assert guards_intact(buf, float("nan"))
    return x.cpu().numpy(), out.cpu().numpy(), ws[:64].view(torch.float64).cpu().numpy()


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_meanstd_against_the_oracle(dtype):
    vol = volume((77, 130, 41), dtype, seed=1, lo=-300, hi=300)
    ratio = R.size_ratio((77, 130, 41), (96, 96, 96))
    x, z, st = normalize_device(vol, (96, 96, 96), ratio, NORM_MEANSTD)
    xo = R.truncate(R.resample_linear(vol, (96, 96, 96), ratio), -100.0, 100.0)
    assert np.array_equal(x, xo)
    mean, sd = R.meanstd_stats(xo)
    if dtype == np.int16:            # integer sums are exact in any order
        assert st[0] == mean and st[1] == sd
        assert np.array_equal(z, R.meanstd(xo))
    else:
        assert abs(st[0] - mean) <= 1e-12 * abs(mean) + 1e-12 and abs(st[1] - sd) <= 1e-12 * sd
        assert int(ulp_diff(z, R.meanstd(xo)).max()) <= 1


@pytest.mark.parametrize("case", CASES)
def test_unet_normalize_matches_the_reference_fixture(case):
    vol = GOLD[case + "_input"]
    x, z, st = normalize_device(vol, vol.shape, (1.0, 1.0, 1.0), NORM_PCTL)
    ref = GOLD[case + "_output"]
    t, b, mean, std, unchanged = R.normalize_stats(vol)
    assert st[2] == t and st[3] == b and bool(st[4]) == unchanged
    if not unchanged:
        assert abs(st[0] - mean) <= 1e-13 * abs(mean) and abs(st[1] - std) <= 1e-13 * std
    assert int(ulp_diff(z, ref.astype(np.float32)).max()) <= 1


@pytest.mark.parametrize("shape_in,shape_out", SHAPES[:3])
def test_unet_normalize_against_the_oracle(shape_in, shape_out):
    vol = volume(shape_in, np.int16, seed=2)
    vol[vol < 0] = 0                                  # zero-heavy, as CT background after a window
    ratio = R.size_ratio(shape_in, shape_out)
    x, z, st = normalize_device(vol, shape_out, ratio, NORM_PCTL)
    t, b, mean, std, unchanged = R.normalize_stats(x)
    s = np.sort(x.ravel().astype(np.float64))
    assert st[2] == t == np.percentile(s, 5) and st[3] == b == np.percentile(s, 95)
    assert not unchanged and st[4] == 0.0
    assert abs(st[0] - mean) <= 1e-12 * abs(mean) and abs(st[1] - std) <= 1e-12 * std
    assert int(ulp_diff(z, R.normalize(x).astype(np.float32)).max()) <= 1


@pytest.mark.parametrize("src_zyx,valid,out_zyx", [((96, 96, 96), (77, 130, 41), (77, 130, 41)),
                                                   ((40, 50, 60), (100, 125, 150), (100, 125, 150)),
                                                   ((50, 40, 30), (60, 48, 37), (64, 45, 40)),
                                                   ((50, 40, 30), (60, 48, 37), (55, 50, 30))])
def test_nearest_back_resample_and_crop_pad_are_bit_equal(src_zyx, valid, out_zyx):
    rng = np.random.RandomState(4)
    src = rng.randint(0, 3, size=src_zyx).astype(np.uint8)
    ratio = R.size_ratio(src_zyx, valid)
    out, buf = guarded(out_zyx, torch.uint8, 0xAB)
    be().resample_nearest_u8(torch.from_numpy(src).cuda(), ratio, valid, out)
    torch.cuda.synchronize()
    assert guards_intact(buf, 0xAB)
    assert np.array_equal(out.cpu().numpy(), R.resample_nearest(src, ratio, valid, out_zyx))


def test_argument_checks():
    lib = be().lib
    assert lib.b200seg_resample_workspace(3, 8, 8, 8) == 0 and lib.b200seg_resample_workspace(1, 0, 8, 8) == 0
    src = torch.zeros((4, 4, 4), dtype=torch.int16, device="cuda")
    out = torch.zeros((4, 4, 4), dtype=torch.float32, device="cuda")
    with pytest.raises(TypeError):
        be().resample_linear(src.to(torch.int64), (1.0, 1.0, 1.0), out)
    with pytest.raises(RuntimeError, match="ratios"):
        be().resample_linear(src, (1.0, 0.0, 1.0), out)
    with pytest.raises(RuntimeError, match="workspace"):
        be().resample_linear(src, (1.0, 1.0, 1.0), out, NORM_PCTL, 0.0, 0.0, torch.zeros(8, dtype=torch.uint8,
                                                                                             device="cuda"))
    with pytest.raises(RuntimeError, match="norm_mode"):
        be().normalize(NORM_NONE, out, torch.zeros(256, dtype=torch.uint8, device="cuda"), out.clone())


def seeded(arch, seed=0):
    if arch == "vnet":
        model = b200.VNet3d(1, 2)
        model.load_state_dict(onets.init_state_dict(onets.vnet3d_state_spec(1, 2), seed=seed, randomize_affine=True))
    else:
        model = b200.UNet3d(1, 2)
        model.load_state_dict(onets.init_state_dict(onets.unet_state_spec(1, 2, 3), seed=seed, randomize_affine=True))
    return model.cuda().eval()


def test_graph_replay_of_the_device_chain():
    vol = torch.from_numpy(volume((77, 130, 41), np.int16)).cuda()
    ratio = R.size_ratio((77, 130, 41), (64, 64, 64))
    outs = {}

    def chain():
        res = []
        for mode in (NORM_MEANSTD, NORM_PCTL):
            x, _ = inf._network_input(be(), vol, (64, 64, 64), ratio, mode, (-100.0, 100.0))
            m = (x[0, 0] > 0).to(torch.uint8)
            back = torch.empty((77, 130, 41), dtype=torch.uint8, device="cuda")
            be().resample_nearest_u8(m, R.size_ratio((64, 64, 64), (77, 130, 41)), (77, 130, 41), back)
            res += [x, back]
        return res

    eager = [t.clone() for t in chain()]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        chain()
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        static = chain()
    vol.copy_(torch.from_numpy(volume((77, 130, 41), np.int16, seed=9)))
    g.replay()
    torch.cuda.synchronize()
    assert not all(torch.equal(a, b) for a, b in zip(eager, static))
    vol.copy_(torch.from_numpy(volume((77, 130, 41), np.int16)))
    g.replay()
    torch.cuda.synchronize()
    for a, b in zip(eager, static):
        assert torch.equal(a, b)


@pytest.mark.parametrize("intensity", ["vnet", "unet"])
def test_no_host_synchronisation_between_upload_and_download(intensity):
    b200.set_precision("bf16")
    model = seeded("vnet")
    vol = torch.from_numpy(volume((77, 130, 41), np.int16)).cuda()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        m = inf._inference3d_device(model, vol, (32, 32, 32), inf._INTENSITY[intensity], 0.5, (-100.0, 100.0))
        p = inf._inference_patch3d_device(model, vol, (1.0, 1.0, 1.0), (0.75, 0.75, 0.75), (32, 32, 32),
                                          inf._INTENSITY[intensity], (-100.0, 100.0), 4, 0.5)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    assert m.shape == vol.shape and p.shape == vol.shape


def margin_field(model, x):
    """|logit_1 - logit_0| of the fp32 forward on x (1, 1, D, H, W)"""
    with torch.no_grad():
        logits = model(torch.from_numpy(x).cuda())[0]
    lg = logits.float().cpu().numpy()           # (1, 2, D, H, W)
    return np.abs(lg[0, 1] - lg[0, 0])


@pytest.mark.parametrize("arch", ["vnet", "unet"])
@pytest.mark.parametrize("intensity", ["vnet", "unet", None])
def test_inference3d_end_to_end_equals_the_oracle_chain(arch, intensity):
    b200.set_precision("fp32")
    model = seeded(arch)
    vol = volume((45, 70, 61), np.int16, seed=3, lo=-200, hi=200)
    out_zyx = (32, 32, 32)
    got = b200.inference3d(model, vol, (32, 32, 32), intensity=intensity)
    x = R.resample_linear(vol, out_zyx, R.size_ratio(vol.shape, out_zyx))
    if intensity == "vnet":
        x = R.meanstd(R.truncate(x, -100.0, 100.0))
    elif intensity == "unet":
        x = R.normalize(x).astype(np.float32)
    m = b200.predict(model, x[None])
    back = R.size_ratio(out_zyx, vol.shape)
    want = R.resample_nearest(m, back, vol.shape, vol.shape)
    assert got.dtype == np.uint8 and got.shape == vol.shape
    diff = got != want
    if diff.any():
        margin = R.resample_nearest(margin_field(model, x[None, None]), back, vol.shape, vol.shape)
        assert float(margin[diff].max()) < 1e-4


@pytest.mark.parametrize("arch", ["vnet", "unet"])
def test_inference_patch3d_end_to_end_equals_the_oracle_chain(arch):
    b200.set_precision("fp32")
    model = seeded(arch)
    vol = volume((40, 70, 66), np.int16, seed=6, lo=-1100, hi=-700)
    sp, nsp, patch = (0.8, 0.8, 1.25), (1.0, 1.0, 1.0), (32, 32, 32)
    got = b200.inference_patch3d(model, vol, sp, nsp, patch_size=patch, batch=3)
    rs = R.spacing_size(tuple(reversed(vol.shape)), sp, nsp)
    rs_zyx = tuple(reversed(rs))
    fwd = tuple(n / o for n, o in zip(reversed(nsp), reversed(sp)))
    x = R.meanstd(R.truncate(R.resample_linear(vol, rs_zyx, fwd), -1024.0, -800.0))
    union = b200.sliding_window_mask(model, x[None], (32, 32, 32), step=(32 * 16,) * 3)
    back_zyx = tuple(reversed(R.spacing_size(rs, nsp, sp)))
    bratio = tuple(o / n for n, o in zip(reversed(nsp), reversed(sp)))
    want = R.resample_nearest(union, bratio, back_zyx, vol.shape)
    assert got.dtype == np.uint8 and got.shape == vol.shape and set(np.unique(got)) <= {0, 1}
    assert np.array_equal(got, want)


def test_ct_volume_end_to_end_shape_and_rerun():
    b200.set_precision("bf16")
    model = seeded("vnet")
    vol = volume((300, 512, 512), np.int16, seed=8)
    a = b200.inference3d(model, vol, (96, 96, 96))
    b = b200.inference3d(model, vol, (96, 96, 96))
    assert a.shape == vol.shape and a.dtype == np.uint8 and np.array_equal(a, b)
