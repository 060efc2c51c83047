"""GPU tests of csrc/augment3d.cu and ``ImageDataGenerator3D`` (pytorchdeeplearing_b200/augment.py): bit-exact against
the reference's recorded outputs (tests/golden/augment3d.npz) and against the fp64 oracle (oracle/augment3d.py) at
training sizes, with guard bands and reruns; the drop-in's ``random_transform`` / ``flow`` (also driven as
``DataAug3D`` drives it) and the per-step ``transform_batch``."""
import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from oracle import augment3d as oa  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = np.load(os.path.join(ROOT, "tests", "golden", "augment3d.npz"))
RT_CASES = sorted({k[:-4] for k in GOLD.files if k.startswith("rt_") and k.endswith("_cfg")})
FLOW_CASES = sorted({k[:-4] for k in GOLD.files if k.startswith("flow_") and k.endswith("_cfg")})


@pytest.fixture(scope="module")
def be():
    if not torch.cuda.is_available():
        pytest.skip("needs CUDA")
    from pytorchdeeplearing_b200 import runtime
    return runtime.cuda_backend()


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    if a.dtype == np.float32:
        a = a.view(np.int32)
    if b.dtype == np.float32:
        b = b.view(np.int32)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a, b)


def gen_kwargs(case):
    cfg = json.loads(str(GOLD[f"{case}_cfg"]))
    if cfg.pop("rescale_kind", None) == "float64":
        cfg["rescale"] = np.float64(cfg["rescale"])
    return cfg


def rng_state_is(case):
    st = np.random.get_state()
    return np.array_equal(st[1], GOLD[f"{case}_state_keys"]) and st[2] == int(GOLD[f"{case}_state_pos"])


def launch(be, x, y, entries, mode="nearest", cval=0.0, shift=False, rescale=None, label_out=None, guard=0):
    """x (N, D, H, W, C) fp32, y (N, D, H, W) numpy -> numpy outputs of one launch; ``guard`` elements of sentinel
    before and after each output (which then sits at an unaligned offset), checked untouched"""
    from pytorchdeeplearing_b200 import _abi
    from pytorchdeeplearing_b200.augment import rescale_form
    dev = torch.device("cuda")
    xd = torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    yd = torch.from_numpy(np.ascontiguousarray(y)).to(dev)
    ydt = {None: yd.dtype, "int64": torch.int64, "binary": torch.int64}[label_out]
    xbuf = torch.full((xd.numel() + 2 * guard,), -777.25, dtype=torch.float32, device=dev)
    ybuf = torch.full((yd.numel() + 2 * guard,), 77, dtype=ydt, device=dev)
    xo = xbuf[guard: guard + xd.numel()].view(xd.shape)
    yo = ybuf[guard: guard + yd.numel()].view(yd.shape)
    params = torch.frombuffer(bytearray(_abi.aug3d_param_table(entries)), dtype=torch.uint8).to(dev)
    ws = be.augment3d_workspace(x.shape[0], x.shape[1:4], dev) if shift else None
    rm, rv = rescale_form(rescale)
    be.augment3d(xd, yd, params, xo, yo, mode=_abi.AUG_MODES[mode], cval=cval, shift=shift, rescale=rv,
                 rescale_mode=rm, binarize=label_out == "binary", ws=ws)
    torch.cuda.synchronize()
    if guard:
        assert bool((xbuf[:guard] == -777.25).all()) and bool((xbuf[-guard:] == -777.25).all())
        assert bool((ybuf[:guard] == 77).all()) and bool((ybuf[-guard:] == 77).all())
    return xo.cpu().numpy(), yo.cpu().numpy()


def fixture_entries(case, kw, shape, channels, count):
    """the recorded matrices with the shifts and flips of the host draws (pinned by the CPU tests)"""
    from pytorchdeeplearing_b200 import augment as A
    np.random.seed(int(GOLD[f"{case}_seed"]))
    gen = A.ImageDataGenerator3D(**kw)
    out = []
    for m4 in GOLD[f"{case}_matrices"][:count]:
        d = A.draw_transform(gen, shape, channels)
        shifts = [float(np.float32(u)) for u in d["channel_shift"]] if d["channel_shift"] is not None else []
        out.append((m4[:3, :3].reshape(-1), m4[:3, 3], shifts, A.flip_bits(d["flips"])))
    return out


@pytest.mark.parametrize("label_out", [None, "int64", "binary"])
@pytest.mark.parametrize("case", RT_CASES)
def test_kernel_matches_random_transform_fixture(be, case, label_out):
    kw = gen_kwargs(case)
    x, y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    entries = fixture_entries(case, kw, x.shape[:3], x.shape[3], 1)
    xo, yo = launch(be, x[None], y[None, ..., 0], entries, kw.get("fill_mode", "nearest"), kw.get("cval", 0.0),
                    kw.get("channel_shift_range", 0) != 0, None, label_out, guard=5)
    assert bits_equal(xo[0], GOLD[f"{case}_xo"])
    want = GOLD[f"{case}_yo"][..., 0]
    if label_out == "int64":
        want = np.trunc(want).astype(np.int64) if want.dtype.kind == "f" else want.astype(np.int64)
    elif label_out == "binary":
        want = (want != 0).astype(np.int64)
    assert bits_equal(yo[0], want)


@pytest.mark.parametrize("case", FLOW_CASES)
def test_kernel_matches_flow_fixture(be, case):
    """every sample of the recorded flow batches, in one launch, with standardize's rescale"""
    from pytorchdeeplearing_b200 import augment as A
    kw = gen_kwargs(case)
    X, Y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    gen = A.ImageDataGenerator3D(**kw)
    it = A.NumpyArrayIterator(X, Y, gen, batch_size=int(GOLD[f"{case}_batch_size"]), shuffle=True,
                              seed=int(GOLD[f"{case}_seed"]))
    idx_all, entries, mats = [], [], GOLD[f"{case}_matrices"]
    for size in GOLD[f"{case}_bsizes"]:
        idx, _, cur = next(it.index_generator)
        for j in range(cur):
            d = A.draw_transform(gen, X.shape[1:4], X.shape[4])
            m4 = mats[len(entries)]
            sh = [float(np.float32(u)) for u in d["channel_shift"]] if d["channel_shift"] is not None else []
            entries.append((m4[:3, :3].reshape(-1), m4[:3, 3], sh, A.flip_bits(d["flips"])))
        idx_all.extend(idx.tolist())
    xo, yo = launch(be, X[idx_all], Y[idx_all][..., 0].astype(np.float32), entries, kw.get("fill_mode", "nearest"),
                    kw.get("cval", 0.0), kw.get("channel_shift_range", 0) != 0, kw.get("rescale"), guard=3)
    assert bits_equal(xo.astype(np.float64), GOLD[f"{case}_xo"])
    assert bits_equal(yo[..., None].astype(np.float64), GOLD[f"{case}_yo"])


def _rotation_entries(rng, shape, n, channels):
    from pytorchdeeplearing_b200 import augment as A
    gen = A.ImageDataGenerator3D(rotation_range=15, width_shift_range=0.1, height_shift_range=0.1,
                                 depth_shift_range=0.1, zoom_range=0.15, channel_shift_range=0.5 if channels > 1 else 0,
                                 horizontal_flip=True, vertical_flip=True, depth_flip=True)
    np.random.seed(int(rng.integers(1 << 30)))
    return [A.param_entry(A.draw_transform(gen, shape, channels), shape) for _ in range(n)]


@pytest.mark.parametrize("mode", oa.MODES)
def test_kernel_matches_oracle_at_96(be, mode):
    rng = np.random.default_rng(96)
    shape = (96, 96, 96)
    x = rng.standard_normal((2,) + shape + (1,)).astype(np.float32)
    y = rng.integers(0, 3, (2,) + shape).astype(np.uint8)
    entries = _rotation_entries(rng, shape, 2, 1)
    want = oa.warp_batch(x, y, entries, mode, 1.5, False, 1.1, "binary")
    got = launch(be, x, y, entries, mode, 1.5, False, 1.1, "binary", guard=1)
    assert bits_equal(got[0], want[0]) and bits_equal(got[1], want[1])
    again = launch(be, x, y, entries, mode, 1.5, False, 1.1, "binary")
    assert bits_equal(got[0], again[0]) and bits_equal(got[1], again[1])


@pytest.mark.parametrize("mode", ["nearest", "constant", "mirror"])
def test_kernel_matches_oracle_c3_shift_anisotropic(be, mode):
    rng = np.random.default_rng(64)
    shape = (64, 128, 128)
    x = rng.standard_normal((1,) + shape + (3,)).astype(np.float32)
    y = rng.standard_normal((1,) + shape).astype(np.float32)
    entries = _rotation_entries(rng, shape, 1, 3)
    want = oa.warp_batch(x, y, entries, mode, -4.0, True, np.float64(1.1))
    got = launch(be, x, y, entries, mode, -4.0, True, np.float64(1.1), guard=7)
    assert bits_equal(got[0], want[0]) and bits_equal(got[1], want[1])
    again = launch(be, x, y, entries, mode, -4.0, True, np.float64(1.1), guard=7)
    assert bits_equal(got[0], again[0])


def test_kernel_c4_unaligned_guard_and_rejects_bad_arguments(be):
    rng = np.random.default_rng(4)
    shape = (9, 10, 11)
    x = rng.standard_normal((3,) + shape + (4,)).astype(np.float32)
    y = rng.integers(0, 256, (3,) + shape).astype(np.uint8)
    entries = _rotation_entries(rng, shape, 3, 4)
    want = oa.warp_batch(x, y, entries, "reflect", 0.0, True, None)
    for guard in (0, 1, 2, 4):        # 16-byte aligned and not
        got = launch(be, x, y, entries, "reflect", 0.0, True, None, guard=guard)
        assert bits_equal(got[0], want[0]) and bits_equal(got[1], want[1])
    from pytorchdeeplearing_b200 import _abi
    xd = torch.zeros((1, 2, 2, 2, 2), device="cuda")
    yd = torch.zeros((1, 2, 2, 2), dtype=torch.uint8, device="cuda")
    p = torch.zeros(_abi.AUG3D_PARAM_BYTES, dtype=torch.uint8, device="cuda")
    with pytest.raises(RuntimeError, match="C must be"):
        be.augment3d(xd, yd, p, torch.empty_like(xd), torch.empty_like(yd))
    xd = torch.zeros((1, 2, 2, 2, 1), device="cuda")
    with pytest.raises(RuntimeError, match="workspace"):
        be.augment3d(xd, yd, p, torch.empty_like(xd), torch.empty_like(yd), shift=True)


# ------------------------------------------------------------------------------------------- the drop-in
def _own_matrices_equal_recorded(gen, case, shape, channels, count):
    from pytorchdeeplearing_b200 import augment as A
    np.random.seed(int(GOLD[f"{case}_seed"]))
    return all(np.array_equal(A.compose_matrix(A.draw_transform(gen, shape, channels), shape), m)
               for m in GOLD[f"{case}_matrices"][:count])


@pytest.mark.parametrize("case", RT_CASES)
def test_random_transform_dropin(be, case):
    from pytorchdeeplearing_b200 import ImageDataGenerator3D
    from pytorchdeeplearing_b200 import augment as A
    kw = gen_kwargs(case)
    gen = ImageDataGenerator3D(**kw)
    x, y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    np.random.seed(int(GOLD[f"{case}_seed"]))
    xo, yo = gen.random_transform(x, y)
    assert rng_state_is(case)
    if _own_matrices_equal_recorded(gen, case, x.shape[:3], x.shape[3], 1):
        assert bits_equal(xo, GOLD[f"{case}_xo"]) and bits_equal(yo, GOLD[f"{case}_yo"])
    else:      # this host's BLAS / libm composed a matrix an ulp away: the oracle on the drop-in's own matrix
        np.random.seed(int(GOLD[f"{case}_seed"]))
        e = A.param_entry(A.draw_transform(gen, x.shape[:3], x.shape[3]), x.shape[:3])
        wx, wy = oa.warp_batch(x[None], y[None, ..., 0], [e], gen.fill_mode, gen.cval,
                               gen.channel_shift_range != 0, None)
        assert bits_equal(xo, wx[0]) and bits_equal(yo, wy[0][..., None])


@pytest.mark.parametrize("case", FLOW_CASES)
def test_flow_dropin(be, case):
    from pytorchdeeplearing_b200 import ImageDataGenerator3D
    kw = gen_kwargs(case)
    gen = ImageDataGenerator3D(**kw)
    X, Y = GOLD[f"{case}_x"], GOLD[f"{case}_y"]
    it = gen.flow(X, Y, batch_size=int(GOLD[f"{case}_batch_size"]), seed=int(GOLD[f"{case}_seed"]))
    xs, ys = zip(*[next(it) for _ in GOLD[f"{case}_bsizes"]])
    assert rng_state_is(case)
    from pytorchdeeplearing_b200 import augment as A
    check = A.ImageDataGenerator3D(**kw)
    it2 = A.NumpyArrayIterator(X, Y, check, batch_size=int(GOLD[f"{case}_batch_size"]), shuffle=True,
                               seed=int(GOLD[f"{case}_seed"]))
    same, k = True, 0
    for size in GOLD[f"{case}_bsizes"]:
        next(it2.index_generator)
        for _ in range(size):
            m = A.compose_matrix(A.draw_transform(check, X.shape[1:4], X.shape[4]), X.shape[1:4])
            same &= bool(np.array_equal(m, GOLD[f"{case}_matrices"][k]))
            k += 1
    if not same:
        pytest.skip("this host composes the matrices an ulp away from the recording (covered by the oracle tests)")
    assert bits_equal(np.concatenate(xs), GOLD[f"{case}_xo"]) and bits_equal(np.concatenate(ys), GOLD[f"{case}_yo"])


def test_flow_as_dataaug3d_drives_it_reproduces_the_written_files(be):
    """DataAug3D.DataAugmentation: per volume flow(srcimage, srcmask) with the defaults (batch 32 of one sample,
    shuffle, no seed), ``number`` batches; the image saved as float64, the mask as uint8"""
    from pytorchdeeplearing_b200 import ImageDataGenerator3D
    from pytorchdeeplearing_b200 import augment as A
    cfg = json.loads(str(GOLD["da3d_cfg"]))
    kw = dict(rotation_range=cfg["rotation"], width_shift_range=cfg["width_shift"],
              height_shift_range=cfg["height_shift"], depth_shift_range=cfg["depth_shift"], zoom_range=cfg["zoom_range"],
              rescale=1.1, horizontal_flip=cfg["horizontal_flip"], vertical_flip=cfg["vertical_flip"], depth_flip=False,
              fill_mode="nearest")
    number = int(GOLD["da3d_number"])
    # the matrices this host composes, replayed first
    np.random.seed(int(GOLD["da3d_seed"]))
    mats = []
    for i in range(2):
        shape = GOLD[f"da3d_src_img_{i}"].shape
        g = A.ImageDataGenerator3D(**kw)
        it = g.flow(np.zeros((1,) + shape + (1,), np.float32), np.zeros((1,) + shape + (1,)))
        for _ in range(number):
            next(it.index_generator)
            mats.append(A.compose_matrix(A.draw_transform(g, shape, 1), shape))
    if not all(np.array_equal(a, b) for a, b in zip(mats, GOLD["da3d_matrices"])):
        pytest.skip("this host composes the matrices an ulp away from the recording (covered by the oracle tests)")
    np.random.seed(int(GOLD["da3d_seed"]))
    gen = ImageDataGenerator3D(**kw)
    for i in range(2):
        img, mask = GOLD[f"da3d_src_img_{i}"], GOLD[f"da3d_src_mask_{i}"]
        k = 0
        for bx, by in gen.flow(img.reshape((1,) + img.shape + (1,)), mask.reshape((1,) + mask.shape + (1,))):
            k += 1
            b1 = bx[0].reshape(img.shape)
            b2 = by[0].reshape(mask.shape).astype("uint8")
            assert b1.dtype == GOLD[f"da3d_img_{i}_{k}"].dtype and b1.tobytes() == GOLD[f"da3d_img_{i}_{k}"].tobytes()
            assert b2.tobytes() == GOLD[f"da3d_mask_{i}_{k}"].tobytes()
            if k > number - 1:
                break
    assert rng_state_is("da3d")


def test_transform_batch_equals_per_sample_random_transform(be):
    from pytorchdeeplearing_b200 import ImageDataGenerator3D
    rng = np.random.default_rng(8)
    shape = (40, 48, 56)
    x = torch.from_numpy(rng.standard_normal((3, 1) + shape).astype(np.float32)).cuda()
    y = torch.from_numpy(rng.integers(0, 4, (3,) + shape).astype(np.uint8)).cuda()
    for kw in (dict(rotation_range=10, width_shift_range=0.05, zoom_range=0.1, horizontal_flip=True,
                    vertical_flip=True, rescale=1.1),
               dict(rotation_range=20, fill_mode="constant", cval=0.5, depth_flip=True, channel_shift_range=0.3)):
        gen = ImageDataGenerator3D(**kw)
        np.random.seed(123)
        xo, yo = gen.transform_batch(x, y)
        torch.cuda.synchronize()
        assert xo.shape == x.shape and xo.dtype == torch.float32 and yo.dtype == torch.int64
        np.random.seed(123)
        for s in range(3):
            xs, ys = gen.random_transform(x[s, 0, ..., None].cpu().numpy(), y[s, ..., None].cpu().numpy())
            assert bits_equal(xo[s, 0].cpu().numpy(), oa.rescale_sample(xs, gen.rescale)[..., 0])
            assert bits_equal(yo[s].cpu().numpy(), (ys[..., 0] != 0).astype(np.int64))


def test_training_step_fed_by_transform_batch(be):
    import pytorchdeeplearing_b200 as b200
    torch.manual_seed(0)
    model = b200.VNet3d(1, 2).cuda().train()
    opt = b200.FusedAdamW(model.parameters(), lr=1e-3)
    lossfn = b200.MutilDiceLoss(torch.ones(2).cuda())
    gen = b200.ImageDataGenerator3D(rotation_range=10, width_shift_range=0.01, height_shift_range=0.01,
                                    zoom_range=0.01, horizontal_flip=True, rescale=1.1)
    x = torch.randn(2, 1, 32, 32, 32, device="cuda")
    y = (torch.rand(2, 32, 32, 32, device="cuda") > 0.7).to(torch.uint8) * 255
    np.random.seed(0)
    for _ in range(2):
        xa, ya = gen.transform_batch(x, y)
        opt.zero_grad()
        logits, _ = model(xa)
        loss = lossfn(logits, ya)
        loss.backward()
        opt.step()
    torch.cuda.synchronize()
    assert np.isfinite(loss.item())
    assert set(torch.unique(ya).tolist()) <= {0, 1}
